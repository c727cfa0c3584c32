// H100 kernel + C-ABI for Optimizer::PoseOptimization (reference src/Optimizer.cc:814-1114, monocular branch):
// one VertexSE3Expmap, one EdgeSE3ProjectXYZOnlyPose per matched keypoint (include/OptimizableTypes.h:31-57,
// src/OptimizableTypes.cpp:49-63), BaseUnaryEdge::constructQuadraticForm (g2o/core/base_unary_edge.hpp:43-72),
// LinearSolverDense (6x6 LDLT), 4 rounds x optimize(10) with outlier re-classification at chi2 > 5.991.
// One CTA per frame (batch over streams), the whole 4-round LM loop on the device, ordered FP64 reductions.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>
#include <string>

#include "../../include/orb_b200.h"
#include "frame_pose.cuh"
#include "inertial_dev.cuh"
#include "pose_opt.h"
#include "staging.h"

using orbx::set_error;

namespace poseopt {

using namespace g2o;
using orbx::block_sum;

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
        if (robust) huber(e2, delta, dsqr, r0, r1);
        else { r0 = e2; r1 = 1.; }
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
        return block_sum<NT>(acc, s_red);
    };
    for (int round = 0; round < 4; ++round) {
        if (tid < 7) s_T[tid] = s_T0[tid];                  // every round restarts from the frame's pose (:1008-1009)
        __syncthreads();
        int nActive = 0;
        for (int e = tid; e < N; e += NT) nActive += !outlier[e];
        nActive = (int)block_sum<NT>((double)nActive, s_red);
        Levenberg lm;
        bool ok = true;
        for (int it = 0; it < 10 && ok && nActive > 0; ++it) {
            double currentChi = errors_and_chi();
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
                    for (int c = a; c < 6; ++c) { const double v = block_sum<NT>(acc[t++], s_red); H[a * 6 + c] = v; H[c * 6 + a] = v; }
                for (int a = 0; a < 6; ++a) b[a] = block_sum<NT>(acc[21 + a], s_red);
            }
            if (it == 0) {
                double md = 0;
                for (int a = 0; a < 6; ++a) md = fmax(md, fabs(H[a * 7]));
                lm.start(0.0, md);
            }
            double rho = 0;
            int qmax = 0;
            do {
                if (tid == 0) {
                    for (int i = 0; i < 7; ++i) s_Tbk[i] = s_T[i];      // push
                    double A[36];
                    for (int i = 0; i < 36; ++i) A[i] = H[i];
                    for (int a = 0; a < 6; ++a) A[a * 7] += lm.lambda;
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
                const double tempChi = errors_and_chi();
                double scale = 0;
                for (int a = 0; a < 6; ++a) scale += s_x[a] * (lm.lambda * s_x[a] + b[a]);
                if (!lm.trial(currentChi, tempChi, scale, ok2, rho)) {
                    __syncthreads();
                    if (tid < 7) s_T[tid] = s_Tbk[tid];                  // pop
                    __syncthreads();
                }
                ++qmax;
            } while (rho < 0 && qmax < Levenberg::maxTrials);
            ok = lm.iteration_done(qmax, rho, iniChi, currentChi);
        }
        // classification (:1014-1036): outliers get a fresh error at the round's final pose, inliers keep the last computed one
        int bad = 0;
        for (int e = tid; e < N; e += NT) {
            if (outlier[e]) compute_error(e);
            const double c2 = (double)is2[e] * (err[2 * e] * err[2 * e] + err[2 * e + 1] * err[2 * e + 1]);
            if ((float)c2 > 5.991f) { outlier[e] = 1; ++bad; } else outlier[e] = 0;     // const float chi2 = e->chi2(); chi2 > chi2Mono[it] (float, :1025-1027)
        }
        nBad = (int)block_sum<NT>((double)bad, s_red);
        if (round == 2) robust = false;                                   // e->setRobustKernel(0) (:1040-1041)
        if (N < 10) break;                                                // optimizer.edges().size() < 10
    }
    if (tid < 7) P.poseOut[7 * (size_t)f + tid] = s_T[tid];
    if (tid == 0) P.nInliers[f] = N - nBad;
}

// ---- The batched tracking calls (pose_opt.h): the matches of every stream are compacted into the packed arrays above, pose_opt_kernel
// runs on them unchanged -- the very instructions pose_optimization_batch runs, so the poses equal its results bit for bit -- and a third
// kernel applies SetPose and the Tracking loop that reads the outlier flags.  One CTA per stream in each.

// Block-wide compaction of the matched keypoints in keypoint order (ballot + warp offsets per tile of NT keypoints), plus the initial
// pose and the camera in pose_opt_kernel's layout.  An inactive stream gets N = 0.
__global__ void __launch_bounds__(NT) gather_edges_kernel(GatherArgs A) {
    __shared__ int s_cnt[NT / 32];
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (A.active && !A.active[f]) { if (tid == 0) A.N[f] = 0; return; }
    const size_t kb = (size_t)f * A.kcap, pb = (size_t)f * A.pstride;
    const int K = min(A.nK[f], A.kcap);
    if (tid < 7) A.poseIn[7 * (size_t)f + tid] = (double)A.TcwIn[7 * (size_t)f + tid];
    if (tid < 4) A.cam4[4 * f + tid] = A.cam[tid];
    int base = 0;
    for (int t0 = 0; t0 < K; t0 += NT) {
        const int i = t0 + tid;
        const int m = i < K ? A.match[kb + i] : -1;
        const unsigned bits = __ballot_sync(0xffffffffu, m >= 0);
        if (lane == 0) s_cnt[wid] = __popc(bits);
        __syncthreads();
        int off = 0, tot = 0;
#pragma unroll
        for (int w = 0; w < NT / 32; ++w) { off += w < wid ? s_cnt[w] : 0; tot += s_cnt[w]; }
        if (m >= 0) {
            const size_t e = kb + base + off + __popc(bits & ((1u << lane) - 1u));
            const OrbKeyPoint kp = A.kps[kb + i];
            const float* X = A.xyz + 3 * (pb + m);
            A.Xw[3 * e] = (double)X[0]; A.Xw[3 * e + 1] = (double)X[1]; A.Xw[3 * e + 2] = (double)X[2];
            A.obs[2 * e] = (double)kp.x; A.obs[2 * e + 1] = (double)kp.y;
            A.invSigma2[e] = A.invLevelSigma2[min(max(kp.octave, 0), A.nlevels - 1)];   // the host entry points reject out-of-range octaves
            A.edgeKp[e] = i;
        }
        base += tot;
        __syncthreads();
    }
    if (tid == 0) A.N[f] = base;
}

// SetPose (none when PoseOptimization returned early with fewer than 3 edges), then the Tracking loop over the frame's matches.
__global__ void __launch_bounds__(NT) gathered_finish_kernel(GatherArgs A) {
    __shared__ int s_n[2];
    const int f = blockIdx.x, tid = threadIdx.x;
    if (A.active && !A.active[f]) return;
    const size_t kb = (size_t)f * A.kcap, pb = (size_t)f * A.pstride;
    const int N = A.N[f];
    if (tid < 2) s_n[tid] = 0;
    if (tid < 7) A.poseOut[7 * (size_t)f + tid] = A.poseTmp[7 * (size_t)f + tid];
    if (tid == 0) A.nInliers[f] = A.nInlTmp[f];
    if (N >= 3) { if (tid == 0) orbm::set_pose_from_double(A.poseTmp + 7 * (size_t)f, A.TcwOut + 7 * (size_t)f); }
    else if (tid < 7) A.TcwOut[7 * (size_t)f + tid] = A.TcwIn[7 * (size_t)f + tid];
    if (A.mode == MOTION_MODEL) for (int p = tid; p < A.pstride; p += NT) A.discarded[pb + p] = 0;
    else for (int i = tid; i < A.kcap; i += NT) A.outlierKp[kb + i] = 0;
    __syncthreads();
    const uint8_t* outl = A.outlier + kb;
    int nOut = 0, nObs = 0;
    for (int e = tid; e < N; e += NT) {
        const int i = A.edgeKp[kb + e];
        const int p = A.match[kb + i];
        if (A.mode == MOTION_MODEL) {
            if (outl[e]) { A.match[kb + i] = -1; A.claimed[kb + i] = 0; A.discarded[pb + p] = 1; ++nOut; }
            else nObs += A.hasObs[pb + p] != 0;
        } else {
            A.outlierKp[kb + i] = outl[e];
            if (!outl[e]) { atomicAdd(&A.found[pb + p], 1); nObs += A.hasObs[pb + p] != 0; }
        }
    }
    if (nOut) atomicAdd(&s_n[0], nOut);
    if (nObs) atomicAdd(&s_n[1], nObs);
    __syncthreads();
    if (tid == 0) {
        if (A.mode == MOTION_MODEL) { A.nmatches[f] -= s_n[0]; A.nmatchesMap[f] = s_n[1]; }
        else A.nMatchesInliers[f] = s_n[1];
    }
}

cudaError_t launch_gathered(const GatherArgs& A, cudaStream_t st) {
    gather_edges_kernel<<<A.batch, NT, 0, st>>>(A);
    Params P;
    memset(&P, 0, sizeof(P));
    P.count = A.batch; P.cap = A.kcap; P.N = A.N; P.pose7 = A.poseIn; P.cam4 = A.cam4;
    P.Xw = A.Xw; P.obs = A.obs; P.invSigma2 = A.invSigma2; P.delta = (double)(float)sqrt(5.991);   // thHuberMono = sqrt(5.991), a float
    P.err = A.err; P.poseOut = A.poseTmp; P.outlier = A.outlier; P.nInliers = A.nInlTmp;
    pose_opt_kernel<<<A.batch, NT, 0, st>>>(P);
    gathered_finish_kernel<<<A.batch, NT, 0, st>>>(A);
    return cudaGetLastError();
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
    int rc = orbx::check_row_counts("pose_optimization_batch", N, count, cap);
    if (rc) return rc;
    const size_t C = count, K = cap;
    orbx::ThreadStaging* S;
    rc = orbx::thread_staging(device, &S);
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
    orbx::zero_row_tails(outlier, N, count, cap);
    return ORB_OK;
}

}  // extern "C"
