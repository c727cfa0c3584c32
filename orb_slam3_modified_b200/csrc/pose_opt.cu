// H100 kernel + C-ABI for Optimizer::PoseOptimization (reference src/Optimizer.cc:814-1114, monocular branch):
// one VertexSE3Expmap, one EdgeSE3ProjectXYZOnlyPose per matched keypoint (include/OptimizableTypes.h:31-57,
// src/OptimizableTypes.cpp:49-63), BaseUnaryEdge::constructQuadraticForm (g2o/core/base_unary_edge.hpp:43-72),
// LinearSolverDense (6x6 LDLT), 4 rounds x optimize(10) with outlier re-classification at chi2 > 5.991.
// One CTA per frame (batch over streams), the whole 4-round LM loop on the device, ordered FP64 reductions.
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <string.h>
#include <string>

#include "../../include/orb_b200.h"
#include "staging.h"

using orbx::set_error;

namespace poseopt {

constexpr int NT = 256;

struct Params {
    int count, cap;
    const int* N;                 // [count]
    const double* pose7;          // [count][7] initial pose (frame's Tcw)
    const float* cam4;            // [count][4]
    const double* Xw;             // [count][cap][3]
    const double* obs;            // [count][cap][2]
    const float* invSigma2;       // [count][cap]
    double delta;
    double* err;                  // scratch [count][cap][2]
    double* poseOut;              // [count][7]
    uint8_t* outlier;             // [count][cap]
    int* nInliers;                // [count]
};

__device__ __forceinline__ void qrot(const double* q, const double* v, double* o) {
    double ux = q[2] * v[2] - q[3] * v[1], uy = q[3] * v[0] - q[1] * v[2], uz = q[1] * v[1] - q[2] * v[0];
    ux += ux; uy += uy; uz += uz;
    o[0] = v[0] + q[0] * ux + (q[2] * uz - q[3] * uy);
    o[1] = v[1] + q[0] * uy + (q[3] * ux - q[1] * uz);
    o[2] = v[2] + q[0] * uz + (q[1] * uy - q[2] * ux);
}
__device__ __forceinline__ void qnormalize(double* q) {
    if (q[0] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
__device__ void qfromR(const double* m, double* q) {
    double t = m[0] + m[4] + m[8];
    if (t > 0) {
        t = sqrt(t + 1.0);
        q[0] = 0.5 * t; t = 0.5 / t;
        q[1] = (m[7] - m[5]) * t; q[2] = (m[2] - m[6]) * t; q[3] = (m[3] - m[1]) * t;
    } else {
        int i = 0;
        if (m[4] > m[0]) i = 1;
        if (m[8] > m[i * 3 + i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0);
        double v[3];
        v[i] = 0.5 * t; t = 0.5 / t;
        q[0] = (m[k * 3 + j] - m[j * 3 + k]) * t;
        v[j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
        v[k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
        q[1] = v[0]; q[2] = v[1]; q[3] = v[2];
    }
}
// VertexSE3Expmap::oplusImpl: T <- SE3Quat::exp(upd) * T
__device__ void pose_oplus(double* T, const double* upd) {
    const double om0 = upd[0], om1 = upd[1], om2 = upd[2];
    const double theta = sqrt(om0 * om0 + om1 * om1 + om2 * om2);
    const double O[9] = {0, -om2, om1, om2, 0, -om0, -om1, om0, 0};
    double O2[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) O2[i * 3 + j] = O[i * 3] * O[j] + O[i * 3 + 1] * O[3 + j] + O[i * 3 + 2] * O[6 + j];
    double a, b, c, d;
    if (theta < 0.00001) { a = 1.0; b = 1 / 2.0; c = 1 / 2.0; d = 1 / 6.0; }
    else {
        a = sin(theta) / theta; b = (1 - cos(theta)) / (theta * theta);
        c = b; d = (theta - sin(theta)) / pow(theta, 3.0);
    }
    double R[9], V[9];
    for (int i = 0; i < 9; ++i) {
        const double I = (i % 4 == 0) ? 1.0 : 0.0;
        R[i] = I + a * O[i] + b * O2[i];
        V[i] = I + c * O[i] + d * O2[i];
    }
    double qe[4]; qfromR(R, qe);
    const double te[3] = {V[0] * upd[3] + V[1] * upd[4] + V[2] * upd[5], V[3] * upd[3] + V[4] * upd[4] + V[5] * upd[5],
                          V[6] * upd[3] + V[7] * upd[4] + V[8] * upd[5]};
    qnormalize(qe);
    double rt[3]; qrot(qe, T + 4, rt);
    const double* q2 = T;
    double qn[4] = {qe[0] * q2[0] - qe[1] * q2[1] - qe[2] * q2[2] - qe[3] * q2[3], qe[0] * q2[1] + qe[1] * q2[0] + qe[2] * q2[3] - qe[3] * q2[2],
                    qe[0] * q2[2] + qe[2] * q2[0] + qe[3] * q2[1] - qe[1] * q2[3], qe[0] * q2[3] + qe[3] * q2[0] + qe[1] * q2[2] - qe[2] * q2[1]};
    qnormalize(qn);
    T[0] = qn[0]; T[1] = qn[1]; T[2] = qn[2]; T[3] = qn[3];
    T[4] = te[0] + rt[0]; T[5] = te[1] + rt[1]; T[6] = te[2] + rt[2];
}

// ordered block sum; every thread gets the result
__device__ __forceinline__ double block_sum(double v, double* sm) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    double r = 0;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) r += sm[w];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(NT) pose_opt_kernel(Params P) {
    __shared__ double s_red[NT / 32];
    __shared__ double s_T[7], s_T0[7], s_Tbk[7], s_x[6];
    __shared__ int s_ok2;
    const int f = blockIdx.x, tid = threadIdx.x;
    const int N = min(P.N[f], P.cap);
    if (N < 3) {   // if(nInitialCorrespondences<3) return 0; (src/Optimizer.cc:996-997): pose and outlier flags stay as they are
        if (tid < 7) P.poseOut[7 * (size_t)f + tid] = P.pose7[7 * (size_t)f + tid];
        for (int e = tid; e < N; e += NT) P.outlier[(size_t)f * P.cap + e] = 0;
        if (tid == 0) P.nInliers[f] = 0;
        return;
    }
    const double* Xw = P.Xw + (size_t)f * P.cap * 3;
    const double* obs = P.obs + (size_t)f * P.cap * 2;
    const float* is2 = P.invSigma2 + (size_t)f * P.cap;
    double* err = P.err + (size_t)f * P.cap * 2;
    uint8_t* outlier = P.outlier + (size_t)f * P.cap;
    const double fx = P.cam4[4 * f], fy = P.cam4[4 * f + 1], cx = P.cam4[4 * f + 2], cy = P.cam4[4 * f + 3];
    const double delta = P.delta, dsqr = delta * delta;
    if (tid == 0) {
        for (int i = 0; i < 7; ++i) s_T0[i] = P.pose7[7 * (size_t)f + i];
        qnormalize(s_T0);                                   // SE3Quat(q, t) constructor
        for (int i = 0; i < 6; ++i) s_x[i] = 0.0;
    }
    for (int e = tid; e < N; e += NT) { outlier[e] = 0; err[2 * e] = 0.0; err[2 * e + 1] = 0.0; }
    __syncthreads();
    bool robust = true;
    int nBad = 0;
    // per-edge state lives in `outlier` (== level 1) ; errors in `err`
    auto compute_error = [&](int e) {
        double r[3]; qrot(s_T, Xw + 3 * (size_t)e, r);
        const double X = r[0] + s_T[4], Y = r[1] + s_T[5], Z = r[2] + s_T[6];
        err[2 * e] = obs[2 * e] - (fx * X / Z + cx);
        err[2 * e + 1] = obs[2 * e + 1] - (fy * Y / Z + cy);
    };
    auto rho_of = [&](double e2, double& r0, double& r1) {
        if (!robust || e2 <= dsqr) { r0 = e2; r1 = 1.; }
        else { const double s = sqrt(e2); r0 = 2 * s * delta - dsqr; r1 = delta / s; }
    };
    auto errors_and_chi = [&]() -> double {   // computeActiveErrors + activeRobustChi2 over the level-0 edges
        double acc = 0;
        for (int e = tid; e < N; e += NT) {
            if (outlier[e]) continue;
            compute_error(e);
            double r0, r1;
            rho_of((double)is2[e] * (err[2 * e] * err[2 * e] + err[2 * e + 1] * err[2 * e + 1]), r0, r1);
            acc += r0;
        }
        return block_sum(acc, s_red);
    };
    for (int round = 0; round < 4; ++round) {
        if (tid < 7) s_T[tid] = s_T0[tid];                  // every round restarts from the frame's pose (:1008-1009)
        __syncthreads();
        int nActive = 0;
        for (int e = tid; e < N; e += NT) nActive += !outlier[e];
        nActive = (int)block_sum((double)nActive, s_red);
        double lambda = -1, ni = 2;
        int nBadLM = 0;
        bool ok = true;
        for (int it = 0; it < 10 && ok && nActive > 0; ++it) {
            double currentChi = errors_and_chi();
            double tempChi = currentChi;
            const double iniChi = currentChi;
            // buildSystem: H (21 unique) and b (6)
            double acc[27];
#pragma unroll
            for (int i = 0; i < 27; ++i) acc[i] = 0;
            for (int e = tid; e < N; e += NT) {
                if (outlier[e]) continue;
                double r[3]; qrot(s_T, Xw + 3 * (size_t)e, r);
                const double x = r[0] + s_T[4], y = r[1] + s_T[5], z = r[2] + s_T[6];
                const double J00 = -(fx / z), J02 = fx * x / (z * z), J11 = -(fy / z), J12 = fy * y / (z * z);
                const double B[12] = {J02 * y, J00 * z - J02 * x, -J00 * y, J00, 0, J02, -J11 * z + J12 * y, -J12 * x, J11 * x, 0, J11, J12};
                double r0, r1;
                rho_of((double)is2[e] * (err[2 * e] * err[2 * e] + err[2 * e + 1] * err[2 * e + 1]), r0, r1);
                const double w = r1 * (double)is2[e];
                const double q0 = (double)is2[e] * err[2 * e], q1 = (double)is2[e] * err[2 * e + 1];
                int t = 0;
#pragma unroll
                for (int a = 0; a < 6; ++a)
#pragma unroll
                    for (int c = a; c < 6; ++c) acc[t++] += w * (B[a] * B[c] + B[6 + a] * B[6 + c]);
#pragma unroll
                for (int a = 0; a < 6; ++a) acc[21 + a] -= r1 * (B[a] * q0 + B[6 + a] * q1);
            }
            double H[36], b[6];
            {
                int t = 0;
                for (int a = 0; a < 6; ++a)
                    for (int c = a; c < 6; ++c) { const double v = block_sum(acc[t++], s_red); H[a * 6 + c] = v; H[c * 6 + a] = v; }
                for (int a = 0; a < 6; ++a) b[a] = block_sum(acc[21 + a], s_red);
            }
            if (it == 0) {
                double md = 0;
                for (int a = 0; a < 6; ++a) md = fmax(md, fabs(H[a * 7]));
                lambda = 1e-5 * md; ni = 2; nBadLM = 0;
            }
            double rho = 0;
            int qmax = 0;
            do {
                if (tid == 0) {
                    for (int i = 0; i < 7; ++i) s_Tbk[i] = s_T[i];      // push
                    double A[36];
                    for (int i = 0; i < 36; ++i) A[i] = H[i];
                    for (int a = 0; a < 6; ++a) A[a * 7] += lambda;
                    // 6x6 LDL^T without pivoting; LinearSolverDense rejects a non positive factorisation
                    bool ok2 = true;
                    for (int k = 0; k < 6 && ok2; ++k) {
                        double d = A[k * 6 + k];
                        for (int j = 0; j < k; ++j) d -= A[k * 6 + j] * A[k * 6 + j] * A[j * 6 + j];
                        A[k * 6 + k] = d;
                        if (d == 0.0 || d < 0) { ok2 = false; break; }
                        for (int i = k + 1; i < 6; ++i) {
                            double s = A[i * 6 + k];
                            for (int j = 0; j < k; ++j) s -= A[i * 6 + j] * A[k * 6 + j] * A[j * 6 + j];
                            A[i * 6 + k] = s / d;
                        }
                    }
                    if (ok2) {
                        double y[6];
                        for (int i = 0; i < 6; ++i) { double s = b[i]; for (int j = 0; j < i; ++j) s -= A[i * 6 + j] * y[j]; y[i] = s; }
                        for (int i = 0; i < 6; ++i) y[i] /= A[i * 6 + i];
                        for (int i = 5; i >= 0; --i) { double s = y[i]; for (int j = i + 1; j < 6; ++j) s -= A[j * 6 + i] * s_x[j]; s_x[i] = s; }
                    }
                    s_ok2 = ok2;
                    pose_oplus(s_T, s_x);                                // update (with the stale x when the solve failed)
                }
                __syncthreads();
                const bool ok2 = s_ok2 != 0;
                tempChi = errors_and_chi();
                if (!ok2) tempChi = DBL_MAX;
                rho = currentChi - tempChi;
                double scale = 0;
                for (int a = 0; a < 6; ++a) scale += s_x[a] * (lambda * s_x[a] + b[a]);
                scale += 1e-3;
                rho /= scale;
                if (rho > 0 && isfinite(tempChi)) {
                    double alpha = 1. - pow((2 * rho - 1), 3.0);
                    alpha = fmin(alpha, 2. / 3.);
                    lambda *= fmax(1. / 3., alpha);
                    ni = 2;
                    currentChi = tempChi;
                } else {
                    lambda *= ni; ni *= 2;
                    __syncthreads();
                    if (tid < 7) s_T[tid] = s_Tbk[tid];                  // pop
                    __syncthreads();
                }
                ++qmax;
            } while (rho < 0 && qmax < 10);
            if (qmax == 10 || rho == 0) ok = false;
            else { if ((iniChi - currentChi) * 1e3 < iniChi) ++nBadLM; else nBadLM = 0; if (nBadLM >= 3) ok = false; }
        }
        // classification (:1014-1036): outliers get a fresh error at the round's final pose, inliers keep the last computed one
        int bad = 0;
        for (int e = tid; e < N; e += NT) {
            if (outlier[e]) compute_error(e);
            const double c2 = (double)is2[e] * (err[2 * e] * err[2 * e] + err[2 * e + 1] * err[2 * e + 1]);
            if ((float)c2 > 5.991f) { outlier[e] = 1; ++bad; } else outlier[e] = 0;     // const float chi2 = e->chi2(); chi2 > chi2Mono[it] (float, :1025-1027)
        }
        nBad = (int)block_sum((double)bad, s_red);
        if (round == 2) robust = false;                                   // e->setRobustKernel(0) (:1040-1041)
        if (N < 10) break;                                                // optimizer.edges().size() < 10
    }
    if (tid < 7) P.poseOut[7 * (size_t)f + tid] = s_T[tid];
    if (tid == 0) P.nInliers[f] = N - nBad;
}

}  // namespace poseopt

using namespace poseopt;

extern "C" {

// int Optimizer::PoseOptimization(Frame* pFrame) for `count` frames.  Host pointers; per frame `cap` edge slots.
int pose_optimization_batch(int count, int cap, const int32_t* N, const double* pose7, const float* cam4, const double* Xw,
                            const double* obs, const float* invSigma2, double huberDelta, double* poseOut, uint8_t* outlier,
                            int32_t* nInliers, int device) {
    if (count < 1 || cap < 1 || !N || !pose7 || !cam4 || !Xw || !obs || !invSigma2 || !poseOut || !outlier || !nInliers) {
        set_error("pose_optimization_batch: bad argument"); return ORB_ERR_ARG;
    }
    const size_t C = count, K = cap;
    orbx::ThreadStaging* S;
    int rc = orbx::thread_staging(device, &S);
    if (rc) return rc;
    S->begin();
    const int pN = S->in(N, 4 * C), pP = S->in(pose7, 56 * C), pC = S->in(cam4, 16 * C), pX = S->in(Xw, 24 * C * K), pO = S->in(obs, 16 * C * K),
              pS = S->in(invSigma2, 4 * C * K), pPo = S->out(poseOut, 56 * C), pOut = S->out(outlier, C * K), pNi = S->out(nInliers, 4 * C),
              pE = S->scratch(16 * C * K);
    if ((rc = S->reserve())) return rc;
    cudaStream_t st = S->stream;
    CK(S->upload(st));
    Params P;
    P.count = count; P.cap = cap; P.N = S->dev<int>(pN); P.pose7 = S->dev<double>(pP); P.cam4 = S->dev<float>(pC);
    P.Xw = S->dev<double>(pX); P.obs = S->dev<double>(pO); P.invSigma2 = S->dev<float>(pS); P.delta = huberDelta;
    P.err = S->dev<double>(pE); P.poseOut = S->dev<double>(pPo); P.outlier = S->dev(pOut); P.nInliers = S->dev<int>(pNi);
    pose_opt_kernel<<<count, NT, 0, st>>>(P);
    CK(cudaGetLastError());
    CK(S->download(st));
    return ORB_OK;
}

}  // extern "C"
