// H100 kernels + C-ABI for the inertial edges of the path (SURVEY.md 8f rank 1): what Optimizer::LocalInertialBA
// (reference src/Optimizer.cc:2383-2958) and PoseInertialOptimizationLast{KeyFrame,Frame} (:4491, :4875) evaluate per iteration.
//   IMU::Preintegrated::IntegrateNewMeasurement (src/ImuTypes.cc:177-240)             imu_preintegrate_kernel   thread per interval
//   EdgeInertial ctor information matrix (src/G2oTypes.cc:499-507), EdgeGyroRW / EdgeAccRW information (src/Optimizer.cc:551,559)
//                                                                                       imu_information_kernel    thread per edge
//   EdgeInertial::computeError / linearizeOplus (src/G2oTypes.cc:514-594) + robust chi2  inertial_edges_kernel     thread per edge
//   EdgeMono::computeError / linearizeOplus (include/G2oTypes.h:353, src/G2oTypes.cc:349-373) + robust chi2
//                                                                                       mono_imu_edges_kernel     thread per edge
// Units of work are independent (one interval / edge per thread, batched over all streams of a GPU); the preintegrated terms are
// float like the reference's IMU::Preintegrated, the edges double like g2o.  NormalizeRotation (Eigen::JacobiSVD, U V^T) is a
// one-sided Jacobi SVD; results agree with the CPU oracle to rounding (tests/test_inertial_gpu.py states the tolerances).
// The 15-DoF block solver around these edges is not built yet (DESIGN.md 7).
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>
#include <string>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "inertial_dev.cuh"
#include "pose_inertial.h"
#include "staging.h"

using orbx::set_error;

namespace imu {

using g2o::huber;
using orbx::block_sum;


// ---- Preintegrated::Initialize + IntegrateNewMeasurement over the measurements of one interval; thread per interval ----
__global__ void imu_preintegrate_kernel(int count, const int* __restrict__ nMeas, int maxMeas, const float* __restrict__ acc, const float* __restrict__ gyr,
                                        const float* __restrict__ dts, const float* __restrict__ bias6, float ng2, float na2, float ngw2, float naw2,
                                        float* __restrict__ out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= count) return;
    float dR[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, dV[3] = {0, 0, 0}, dP[3] = {0, 0, 0};
    float JRg[9], JVg[9], JVa[9], JPg[9], JPa[9], C9[81];
    for (int i = 0; i < 9; ++i) JRg[i] = JVg[i] = JVa[i] = JPg[i] = JPa[i] = 0.f;
    for (int i = 0; i < 81; ++i) C9[i] = 0.f;
    float walk[6] = {0, 0, 0, 0, 0, 0};
    const float* b = bias6 + 6 * (size_t)e;
    const float Nga[6] = {ng2, ng2, ng2, na2, na2, na2}, Walk[6] = {ngw2, ngw2, ngw2, naw2, naw2, naw2};
    float dT = 0.f;
    const int n = min(nMeas[e], maxMeas);
    for (int m = 0; m < n; ++m) {
        const size_t o = (size_t)e * maxMeas + m;
        const float dt = dts[o];
        const float a[3] = {acc[3 * o] - b[0], acc[3 * o + 1] - b[1], acc[3 * o + 2] - b[2]};
        float Ra[3];
        m3vec(dR, a, Ra);
        for (int i = 0; i < 3; ++i) dP[i] = dP[i] + dV[i] * dt + 0.5f * Ra[i] * dt * dt;
        for (int i = 0; i < 3; ++i) dV[i] = dV[i] + Ra[i] * dt;
        float Wacc[9], RW[9], RWJ[9];
        hat(a, Wacc);
        m3mul(dR, Wacc, RW);
        m3mul(RW, JRg, RWJ);
        // A = [dRi^T 0 0; -dR dt Wacc, I, 0; -0.5 dR dt^2 Wacc, dt I, I], B = [rightJ dt, 0; 0, dR dt; 0, 0.5 dR dt^2]  (built after the rotation step)
        float A10[9], A20[9], B11[9], B21[9];
        for (int i = 0; i < 9; ++i) { A10[i] = -RW[i] * dt; A20[i] = -0.5f * RW[i] * dt * dt; B11[i] = dR[i] * dt; B21[i] = 0.5f * dR[i] * dt * dt; }
        for (int i = 0; i < 9; ++i) {
            JPa[i] = JPa[i] + JVa[i] * dt - 0.5f * dR[i] * dt * dt;
            JPg[i] = JPg[i] + JVg[i] * dt - 0.5f * RWJ[i] * dt * dt;
            JVa[i] = JVa[i] - dR[i] * dt;
            JVg[i] = JVg[i] - RWJ[i] * dt;
        }
        // IntegratedRotation (:84-107)
        const float w[3] = {(gyr[3 * o] - b[3]) * dt, (gyr[3 * o + 1] - b[4]) * dt, (gyr[3 * o + 2] - b[5]) * dt};
        const float d2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], d = sqrtf(d2);
        float W[9], W2[9], deltaR[9], rightJ[9];
        hat(w, W); m3mul(W, W, W2);
        for (int i = 0; i < 9; ++i) {
            const float I = (i % 4 == 0) ? 1.f : 0.f;
            if (d < 1e-4f) { deltaR[i] = I + W[i]; rightJ[i] = I; }
            else { deltaR[i] = I + W[i] * sinf(d) / d + W2[i] * (1.0f - cosf(d)) / d2; rightJ[i] = I - W[i] * (1.0f - cosf(d)) / d2 + W2[i] * (d - sinf(d)) / (d2 * d); }
        }
        float Rn[9], dRt[9];
        m3mul(dR, deltaR, Rn);
        normalize_rotation(Rn, dR);
        m3T(deltaR, dRt);
        // C9 <- A C9 A^T + B Nga B^T with the block structure of A and B written out row-block by row-block
        float A[81], B[54];
        for (int i = 0; i < 81; ++i) A[i] = (i % 10 == 0) ? 1.f : 0.f;
        for (int i = 0; i < 54; ++i) B[i] = 0.f;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                A[i * 9 + j] = dRt[i * 3 + j]; A[(3 + i) * 9 + j] = A10[i * 3 + j]; A[(6 + i) * 9 + j] = A20[i * 3 + j]; A[(6 + i) * 9 + 3 + j] = i == j ? dt : 0.f;
                B[i * 6 + j] = rightJ[i * 3 + j] * dt; B[(3 + i) * 6 + 3 + j] = B11[i * 3 + j]; B[(6 + i) * 6 + 3 + j] = B21[i * 3 + j];
            }
        float AC[81];
        for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) { float s = 0; for (int k = 0; k < 9; ++k) s += A[i * 9 + k] * C9[k * 9 + j]; AC[i * 9 + j] = s; }
        for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) {
            float s = 0; for (int k = 0; k < 9; ++k) s += AC[i * 9 + k] * A[j * 9 + k];
            float t = 0; for (int k = 0; k < 6; ++k) t += B[i * 6 + k] * Nga[k] * B[j * 6 + k];
            C9[i * 9 + j] = s + t;
        }
        for (int k = 0; k < 6; ++k) walk[k] += Walk[k];
        float T1[9];
        m3mul(dRt, JRg, T1);
        for (int i = 0; i < 9; ++i) JRg[i] = T1[i] - rightJ[i] * dt;
        dT += dt;
    }
    float* P = out + (size_t)P_SIZE * e;
    for (int i = 0; i < P_SIZE; ++i) P[i] = 0.f;
    P[P_DT] = dT;
    for (int i = 0; i < 9; ++i) { P[P_DR + i] = dR[i]; P[P_JRG + i] = JRg[i]; P[P_JVG + i] = JVg[i]; P[P_JVA + i] = JVa[i]; P[P_JPG + i] = JPg[i]; P[P_JPA + i] = JPa[i]; }
    for (int i = 0; i < 3; ++i) { P[P_DV + i] = dV[i]; P[P_DP + i] = dP[i]; }
    for (int i = 0; i < 6; ++i) P[P_B + i] = b[i];
    for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) P[P_C + i * 15 + j] = C9[i * 9 + j];
    for (int k = 0; k < 6; ++k) P[P_C + (9 + k) * 15 + 9 + k] = walk[k];
}

__global__ void imu_information_kernel(int count, const float* __restrict__ preint, double* __restrict__ info9, double* __restrict__ infoG, double* __restrict__ infoA) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= count) return;
    imu_information_dev(preint + (size_t)P_SIZE * e, info9 + 81 * (size_t)e, infoG + 9 * (size_t)e, infoA + 9 * (size_t)e);
}

__global__ void inertial_edges_kernel(int count, const float* __restrict__ preint, const int* __restrict__ preintIndex, const double* __restrict__ states,
                                      const double* __restrict__ info9, double huberDelta, double* __restrict__ errOut, double* __restrict__ Jout,
                                      double* __restrict__ chi2Out, double* __restrict__ rhoOut) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= count) return;
    const int pi = preintIndex ? preintIndex[e] : e;
    double err[9];
    edge_inertial_dev(preint + (size_t)P_SIZE * pi, states + 36 * (size_t)e, err, Jout ? Jout + 216 * (size_t)e : nullptr);
    for (int i = 0; i < 9; ++i) errOut[9 * (size_t)e + i] = err[i];
    if (info9) {   // chi2 = e^T Omega e, Huber rho' (RobustKernelHuber with delta = sqrt(16.92), src/Optimizer.cc:540-542)
        const double* Om = info9 + 81 * (size_t)pi;
        double c2 = 0;
        for (int i = 0; i < 9; ++i) { double s = 0; for (int j = 0; j < 9; ++j) s += Om[i * 9 + j] * err[j]; c2 += err[i] * s; }
        chi2Out[e] = c2;
        if (rhoOut) {
            double r0, r1 = 1.0;                              // huberDelta <= 0: no robust kernel
            if (!(huberDelta <= 0)) huber(c2, huberDelta, huberDelta * huberDelta, r0, r1);
            rhoOut[e] = r1;
        }
    }
}

// ---- EdgeMono with ImuCamPose (body pose + camera extrinsics): residual, Jacobians, chi2, depth sign; thread per edge ----
struct MonoParams {
    int nEdges;
    const double* poses;       // [nPoses][12]: Rwb 9 | twb 3
    const double* extr;        // [24]: Rcb 9 | tcb 3 | Rbc 9 | tbc 3   (Tcb / Tbc of camera 0, IMU::Calib)
    const float* cam;          // [nPoses][4]
    const double* points;      // [nPoints][3]
    const int *edgePoint, *edgePose;
    const double* obs;         // [nEdges][2]
    const float* invSigma2;    // [nEdges]
    double huberDelta;
    double *err, *Jpoint, *Jpose, *chi2, *rho; uint8_t* depthPositive;
};
__global__ void mono_imu_edges_kernel(MonoParams Q) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= Q.nEdges) return;
    const double* Pz = Q.poses + 12 * (size_t)Q.edgePose[e];
    const double *Rwb = Pz, *twb = Pz + 9, *Rcb = Q.extr, *tcb = Q.extr + 9, *Rbc = Q.extr + 12, *tbc = Q.extr + 21;
    const double* Xw = Q.points + 3 * (size_t)Q.edgePoint[e];
    const float* cm = Q.cam + 4 * (size_t)Q.edgePose[e];
    double Rbw[9], tbw[3], Rcw[9], tcw[3], Xc[3];
    m3T(Rwb, Rbw);
    m3vec(Rbw, twb, tbw);
    for (int i = 0; i < 3; ++i) tbw[i] = -tbw[i];
    m3mul(Rcb, Rbw, Rcw);
    m3vec(Rcb, tbw, tcw);
    for (int i = 0; i < 3; ++i) tcw[i] += tcb[i];
    double e0, e1;
    const bool depthPos = mono_residual(Rcw, tcw, Xw, cm, Q.obs[2 * (size_t)e], Q.obs[2 * (size_t)e + 1], Xc, e0, e1);
    Q.err[2 * (size_t)e] = e0; Q.err[2 * (size_t)e + 1] = e1;
    const double c2 = (double)Q.invSigma2[e] * (e0 * e0 + e1 * e1);
    Q.chi2[e] = c2;
    if (Q.rho) {
        double r0, r1 = 1.0;
        if (!(Q.huberDelta <= 0)) huber(c2, Q.huberDelta, Q.huberDelta * Q.huberDelta, r0, r1);
        Q.rho[e] = r1;
    }
    Q.depthPositive[e] = depthPos;
    if (Q.Jpoint) mono_jacobians(Rcw, Rcb, Rbc, tbc, cm, Xc, Q.Jpoint + 6 * (size_t)e, Q.Jpose + 12 * (size_t)e);
}

// ---------------------------------------------------------------------------------------------
// int Optimizer::PoseInertialOptimizationLastKeyFrame(Frame* pFrame, bool bRecInit) (src/Optimizer.cc:4491-4873), monocular frame: the
// tracking-side inertial pose optimiser (Tracking::TrackLocalMap, src/Tracking.cc:2985-2994) for a batch of streams, one CTA per frame.
// 15 unknowns (VertexPose 6, VertexVelocity 3, VertexGyroBias 3, VertexAccBias 3); the last keyframe's vertices are fixed.  Four rounds of
// g2o Gauss-Newton x 10 iterations on the device: the EdgeMonoOnlyPose edges are spread over the threads (pose block: 21 + 6 ordered
// block sums), thread 0 adds EdgeInertial and the two random-walk edges, factors the dense 15 x 15 system (LDLT, LinearSolverDense) and
// applies the update (ImuCamPose::Update; its every-third-update NormalizeRotation call has no effect in the reference, see apply_update15); then the chi2 re-classification of :4713-4778 with
// stale / recomputed errors exactly as g2o leaves them, the recovery of :4783-4810 and the Hessian of the next prior (:4819-4867).
// ---------------------------------------------------------------------------------------------
constexpr int PI_NT = 128;
struct PoseInertialParams {
    int count, cap, recInit;
    const int* N;                       // [count]
    const float *Xw, *obs, *invSigma2, *trackDepth;   // [count][cap][3], [..][2], [..], [..]
    const float* cam4;                  // [count][4]
    const double* extr;                 // [24]
    const float* preint;                // [count][P_SIZE]: EdgeInertial (from the last keyframe / from the previous frame)
    const double* kfState;              // [count][21]: the fixed last keyframe (last-keyframe variant)
    double* state;                      // [count][21] in / out
    double* err;                        // scratch [count][cap][2]
    uint8_t* outlier;                   // [count][cap]
    double* H15;                        // [count][225]
    int* ret;                           // [count]
    // last-frame variant (src/Optimizer.cc:4875-5289): the previous frame is free and held by EdgePriorPoseImu
    const float* preintKF;              // [count][P_SIZE]: mpImuPreintegrated, the source of the two random-walk informations (:5068-5078)
    const double *prior, *priorH;       // [count][21], [count][225]: ConstraintPoseImu of the previous frame
    double* prevState;                  // [count][21] in / out
};
// EdgeMonoOnlyPose at the cached camera pose: residual, depth sign and (optionally) the 2 x 6 Jacobian (src/G2oTypes.cc:375-395)
__device__ __forceinline__ void mono_only_pose(const double* Rcw, const double* tcw, const double* Rcb, const double* Rbc, const double* tbc, const float* cm,
                                               const float* Xwf, const float* of, double& e0, double& e1, bool& depthPos, double* Jp) {
    const double X[3] = {(double)Xwf[0], (double)Xwf[1], (double)Xwf[2]};
    double Xc[3];
    depthPos = mono_residual(Rcw, tcw, X, cm, (double)of[0], (double)of[1], Xc, e0, e1);
    if (Jp) mono_jacobians(Rcw, Rcb, Rbc, tbc, cm, Xc, nullptr, Jp);
}
// vertex updates of one frame: ImuCamPose::Update (twb += Rwb ut; Rwb = Rwb ExpSO3(ur)), v / bg / ba += dx
__device__ void apply_update15(double* st, const double* dx, int& its) {
    double t3[3], E[9], Rn[9];
    m3vec(st, dx + 3, t3);
    for (int i = 0; i < 3; ++i) st[9 + i] += t3[i];
    exp_so3_d(dx, E);
    m3mul(st, E, Rn);
    for (int i = 0; i < 9; ++i) st[i] = Rn[i];
    // ImuCamPose::Update's every-third-update `NormalizeRotation(Rwb);` (src/G2oTypes.cc:202-208) discards the return value of a function that leaves its
    // argument alone (include/G2oTypes.h:67-71): the reference never renormalises Rwb, and neither does this
    (void)its;
    for (int i = 0; i < 3; ++i) { st[12 + i] += dx[6 + i]; st[15 + i] += dx[9 + i]; st[18 + i] += dx[12 + i]; }
}
// EdgePriorPoseImu (src/G2oTypes.cc:731-760): residual 15 and Jacobian 15 x 15 (block diagonal) wrt the previous frame's pose 6, v, bg, ba
__device__ void prior_edge_dev(const double* prior, const double* st, double* e15, double* J) {
    double Rpt[9], dR[9], er[3], d[3], et[3], iJ[9];
    m3T(prior, Rpt); m3mul(Rpt, st, dR);
    log_so3(dR, er);
    for (int i = 0; i < 3; ++i) d[i] = st[9 + i] - prior[9 + i];
    m3vec(Rpt, d, et);
    for (int i = 0; i < 3; ++i) { e15[i] = er[i]; e15[3 + i] = et[i]; e15[6 + i] = st[12 + i] - prior[12 + i]; e15[9 + i] = st[15 + i] - prior[15 + i]; e15[12 + i] = st[18 + i] - prior[18 + i]; }
    for (int i = 0; i < 225; ++i) J[i] = 0;
    inv_right_jacobian(er, iJ);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { J[i * 15 + j] = iJ[i * 3 + j]; J[(3 + i) * 15 + 3 + j] = dR[i * 3 + j]; }
    for (int i = 6; i < 15; ++i) J[i * 15 + i] = 1.0;
}
// Dense LDLT solve of the n x n system in A (shared memory, row-major, n <= 30) by ONE WARP: Eigen::LDLT + isPositive()
// (linear_solver_dense.h:111-118).  Left-looking by columns, lane = row of the column; substitutions column-oriented with the running
// right-hand side in a register per lane.  A is overwritten by L (strictly lower part); d: n doubles of shared memory.
// Returns false (x untouched) when a pivot is not positive.  All 32 lanes call.
__device__ bool ldlt_solve_warp(int n, double* A, const double* b, double* x, double* d) {
    const int lane = threadIdx.x & 31;
    for (int j = 0; j < n; ++j) {
        double dj = A[j * n + j];
        for (int k = 0; k < j; ++k) dj -= A[j * n + k] * A[j * n + k] * d[k];
        if (!(dj > 0)) return false;                         // every lane computed the same dj
        const int i = j + 1 + lane;
        double v = 0;
        if (i < n) { v = A[i * n + j]; for (int k = 0; k < j; ++k) v -= A[i * n + k] * A[j * n + k] * d[k]; }
        __syncwarp();
        if (lane == 0) d[j] = dj;
        if (i < n) A[i * n + j] = v / dj;
        __syncwarp();
    }
    double r = lane < n ? b[lane] : 0.0;                     // forward: L y = b
    for (int k = 0; k < n; ++k) {
        const double yk = __shfl_sync(0xffffffffu, r, k);
        if (lane > k && lane < n) r -= A[lane * n + k] * yk;
    }
    r = lane < n ? r / d[lane] : 0.0;                        // D z = y
    for (int k = n - 1; k >= 0; --k) {                       // backward: L^T x = z
        const double xk = __shfl_sync(0xffffffffu, r, k);
        if (lane < k) r -= A[k * n + lane] * xk;
    }
    if (lane < n) x[lane] = r;
    __syncwarp();
    return true;
}
// LF = false: PoseInertialOptimizationLastKeyFrame (15 unknowns); LF = true: PoseInertialOptimizationLastFrame (30 unknowns: current 15 | previous 15)
template <bool LF>
__global__ void __launch_bounds__(PI_NT) pose_inertial_opt_kernel(PoseInertialParams Q) {
    constexpr int NX = LF ? 30 : 15;
    __shared__ double s_red[PI_NT / 32];
    __shared__ double s_st[21], s_sp[21], s_cam[12], s_info[81 + 9 + 9], s_x[NX], s_H[NX * NX], s_b[NX], s_L[NX * NX], s_d[30];
    __shared__ double s_J[216], s_OJ[216], s_e9[9], s_Jp[225], s_OJp[225], s_e15[15], s_Oe15[15];   // EdgeInertial / EdgePriorPoseImu: Jacobians, Omega J, residuals
    __shared__ int s_ok, s_cnt[2];
    const int f = blockIdx.x, tid = threadIdx.x;
    const int N = min(Q.N[f], Q.cap);
    const float* Xw = Q.Xw + 3 * (size_t)f * Q.cap; const float* ob = Q.obs + 2 * (size_t)f * Q.cap;
    const float* is2 = Q.invSigma2 + (size_t)f * Q.cap; const float* td = Q.trackDepth + (size_t)f * Q.cap;
    const float* cm = Q.cam4 + 4 * (size_t)f; const float* P = Q.preint + (size_t)P_SIZE * f;
    double* err = Q.err + 2 * (size_t)f * Q.cap; uint8_t* outl = Q.outlier + (size_t)f * Q.cap;
    const double *Rcb = Q.extr, *tcb = Q.extr + 9, *Rbc = Q.extr + 12, *tbc = Q.extr + 21;
    const double* prior = LF ? Q.prior + 21 * (size_t)f : nullptr;
    const double* priorH = LF ? Q.priorH + 225 * (size_t)f : nullptr;
    double *Rcw = s_cam, *tcw = s_cam + 9;
    if (tid < 21) { s_st[tid] = Q.state[21 * (size_t)f + tid]; s_sp[tid] = LF ? Q.prevState[21 * (size_t)f + tid] : Q.kfState[21 * (size_t)f + tid]; }
    if (tid < NX) s_x[tid] = 0.0;
    if (tid == 0) {
        if (LF) { imu_information_dev(Q.preintKF + (size_t)P_SIZE * f, s_H, s_info + 81, s_info + 90); imu_information_dev(P, s_info, s_H, s_H + 16); }
        else imu_information_dev(P, s_info, s_info + 81, s_info + 90);
    }
    for (int i = tid; i < N; i += PI_NT) { outl[i] = 0; err[2 * i] = 0; err[2 * i + 1] = 0; }
    __syncthreads();
    auto refresh_camera = [&]() {               // ImuCamPose::Update's camera part: Rcw = Rcb Rbw, tcw = Rcb tbw + tcb   (thread 0)
        double Rbw[9], tbw[3];
        m3T(s_st, Rbw); m3vec(Rbw, s_st + 9, tbw);
        for (int i = 0; i < 3; ++i) tbw[i] = -tbw[i];
        m3mul(Rcb, Rbw, Rcw); m3vec(Rcb, tbw, tcw);
        for (int i = 0; i < 3; ++i) tcw[i] += tcb[i];
    };
    if (tid == 0) refresh_camera();
    __syncthreads();
    const double delta = (double)sqrtf(5.991f), dsqr = delta * delta;
    const float chi2Mono[4] = {LF ? 5.991f : 12.f, LF ? 5.991f : 7.5f, 5.991f, 5.991f};
    bool robust = true;
    int its = 0, itsPrev = 0, nBad = 0, nInliers = 0;        // its / itsPrev: thread 0's copies of ImuCamPose::its of the two VertexPose
    // x column of column c of the EdgeInertial Jacobian (vertex order: previous pose, v, bg, ba | current pose, v)
    auto xi = [](int c) { return c < 15 ? 15 + c : c - 15; };
    for (int it = 0; it < 4; ++it) {
        for (int iter = 0; iter < 10; ++iter) {
            double acc[27];
#pragma unroll
            for (int k = 0; k < 27; ++k) acc[k] = 0;
            for (int i = tid; i < N; i += PI_NT) {
                if (outl[i]) continue;                        // setLevel(1) and mvbOutlier are always set together (:4736-4747)
                double e0, e1, Jp[12]; bool dp;
                mono_only_pose(Rcw, tcw, Rcb, Rbc, tbc, cm, Xw + 3 * i, ob + 2 * i, e0, e1, dp, Jp);
                err[2 * i] = e0; err[2 * i + 1] = e1;
                const double om = (double)is2[i], c2 = om * (e0 * e0 + e1 * e1);
                double r0, w = 1.0;
                if (robust && c2 > dsqr) huber(c2, delta, dsqr, r0, w);       // c2 > dsqr, not huber's e2 <= dsqr: a NaN chi2 weighs 1 here
                const double wo = w * om;
                int t = 0;
#pragma unroll
                for (int a = 0; a < 6; ++a) {
#pragma unroll
                    for (int c = a; c < 6; ++c) acc[t++] += wo * (Jp[a] * Jp[c] + Jp[6 + a] * Jp[6 + c]);
                }
#pragma unroll
                for (int a = 0; a < 6; ++a) acc[21 + a] -= wo * (Jp[a] * e0 + Jp[6 + a] * e1);
            }
            double tot[27];
#pragma unroll
            for (int k = 0; k < 27; ++k) tot[k] = block_sum<PI_NT>(acc[k], s_red);
            // (a) the two multi-vertex edges are linearised by two threads of different warps at the same time
            if (tid == 0) {
                double S36[36];
                for (int k = 0; k < 21; ++k) S36[k] = s_sp[k];
                for (int k = 0; k < 15; ++k) S36[21 + k] = s_st[k];
                edge_inertial_dev(P, S36, s_e9, s_J);
            }
            if (LF && tid == 32) prior_edge_dev(prior, s_sp, s_e15, s_Jp);
            __syncthreads();
            // (b) Omega J, Omega e
            for (int idx = tid; idx < 216; idx += PI_NT) { const int r = idx / 24, c = idx - r * 24; double a = 0; for (int k = 0; k < 9; ++k) a += s_info[r * 9 + k] * s_J[k * 24 + c]; s_OJ[idx] = a; }
            if (LF) {
                for (int idx = tid; idx < 225; idx += PI_NT) { const int r = idx / 15, c = idx - r * 15; double a = 0; for (int k = 0; k < 15; ++k) a += priorH[r * 15 + k] * s_Jp[k * 15 + c]; s_OJp[idx] = a; }
                if (tid < 15) { double a = 0; for (int k = 0; k < 15; ++k) a += priorH[tid * 15 + k] * s_e15[k]; s_Oe15[tid] = a; }
            }
            __syncthreads();
            // (c) the normal equations, one entry per thread.  x index -> column of the EdgeInertial Jacobian: current pose / velocity -> 15..23,
            //     current biases -> none, previous 15 -> 0..14
            double wPrior = 1.0;
            if (LF) {                                           // RobustKernelHuber delta 5 (:5084-5092); a NaN chi2 weighs 1, as at the mono edges
                double c2 = 0, r0;
                for (int k = 0; k < 15; ++k) c2 += s_e15[k] * s_Oe15[k];
                if (c2 > 25.0) huber(c2, 5.0, 25.0, r0, wPrior);
            }
            auto ecol = [](int i) { return i < 9 ? 15 + i : (i < 15 ? -1 : i - 15); };
            for (int idx = tid; idx < NX * NX; idx += PI_NT) {
                const int i = idx / NX, j = idx - i * NX;
                double h = 0;
                if (i < 6 && j < 6) { const int a = min(i, j), c = max(i, j); h += tot[a * 6 - a * (a - 1) / 2 + (c - a)]; }     // packed upper triangle of the mono block
                const int ei = ecol(i), ej = ecol(j);
                if (ei >= 0 && ej >= 0) { double a = 0; for (int r = 0; r < 9; ++r) a += s_J[r * 24 + ei] * s_OJ[r * 24 + ej]; h += a; }
                // EdgeGyroRW / EdgeAccRW: error = b_cur - b_prev, Jacobians +I (current: x 9..14) and -I (previous, when free: x 24..29)
                {
                    const int bi = i >= 9 && i < 15 ? i - 9 : (LF && i >= 24 ? i - 24 : -1), bj = j >= 9 && j < 15 ? j - 9 : (LF && j >= 24 ? j - 24 : -1);
                    if (bi >= 0 && bj >= 0 && (bi / 3) == (bj / 3)) {
                        const double om = s_info[(bi < 3 ? 81 : 90) + (bi % 3) * 3 + (bj % 3)];
                        h += ((i < 15) == (j < 15)) ? om : -om;
                    }
                }
                if (LF && i >= 15 && j >= 15) { double a = 0; for (int r = 0; r < 15; ++r) a += s_Jp[r * 15 + i - 15] * s_OJp[r * 15 + j - 15]; h += wPrior * a; }
                s_H[idx] = h;
            }
            if (tid < NX) {
                const int i = tid;
                double g = i < 6 ? tot[21 + i] : 0.0;
                const int ei = ecol(i);
                if (ei >= 0) { double a = 0; for (int r = 0; r < 9; ++r) a += s_OJ[r * 24 + ei] * s_e9[r]; g -= a; }
                const int bi = i >= 9 && i < 15 ? i - 9 : (LF && i >= 24 ? i - 24 : -1);
                if (bi >= 0) {
                    double a = 0;
                    for (int c = 0; c < 3; ++c) a += s_info[(bi < 3 ? 81 : 90) + (bi % 3) * 3 + c] * (s_st[(bi < 3 ? 15 : 18) + c] - s_sp[(bi < 3 ? 15 : 18) + c]);
                    g += i < 15 ? -a : a;
                }
                if (LF && i >= 15) { double a = 0; for (int r = 0; r < 15; ++r) a += s_Jp[r * 15 + i - 15] * s_Oe15[r]; g -= wPrior * a; }
                s_b[i] = g;
            }
            __syncthreads();
            // (d) dense LDLT by warp 0; a failed solve leaves x of the previous iteration and update() still runs
            if (tid < 32) {
                for (int k = tid; k < NX * NX; k += 32) s_L[k] = s_H[k];
                __syncwarp();
                const bool ok = ldlt_solve_warp(NX, s_L, s_b, s_x, s_d);
                if (tid == 0) s_ok = ok ? 1 : 0;
            }
            __syncthreads();
            // (e) vertex updates, the two frames by two threads
            if (tid == 0) { apply_update15(s_st, s_x, its); refresh_camera(); }
            if (LF && tid == 32) apply_update15(s_sp, s_x + 15, itsPrev);
            __syncthreads();
            if (!s_ok) break;
        }
        // ---- re-classification (:4713-4778 / :5113-5180) ----
        if (tid == 0) { s_cnt[0] = 0; s_cnt[1] = 0; }
        __syncthreads();
        const float chi2close = (float)(1.5 * (double)chi2Mono[it]);
        int bad = 0, good = 0;
        for (int i = tid; i < N; i += PI_NT) {
            double e0, e1; bool dp;
            mono_only_pose(Rcw, tcw, Rcb, Rbc, tbc, cm, Xw + 3 * i, ob + 2 * i, e0, e1, dp, nullptr);
            if (outl[i]) { err[2 * i] = e0; err[2 * i + 1] = e1; }          // e->computeError() only for the outliers
            const float chi2 = (float)((double)is2[i] * (err[2 * i] * err[2 * i] + err[2 * i + 1] * err[2 * i + 1]));
            const bool bClose = td[i] < 10.f;
            if ((chi2 > chi2Mono[it] && !bClose) || (bClose && chi2 > chi2close) || !dp) { outl[i] = 1; ++bad; } else { outl[i] = 0; ++good; }
        }
        atomicAdd(&s_cnt[0], bad); atomicAdd(&s_cnt[1], good);
        __syncthreads();
        nBad = s_cnt[0]; nInliers = s_cnt[1];
        __syncthreads();
        if (it == 2) robust = false;
        if (N + (LF ? 4 : 3) < 10) break;                                   // optimizer.edges().size() < 10
    }
    if (nInliers < 30 && !Q.recInit) {                                       // :4783-4810 / :5183-5211
        if (tid == 0) s_cnt[0] = 0;
        __syncthreads();
        int bad = 0;
        for (int i = tid; i < N; i += PI_NT) {
            double e0, e1; bool dp;
            mono_only_pose(Rcw, tcw, Rcb, Rbc, tbc, cm, Xw + 3 * i, ob + 2 * i, e0, e1, dp, nullptr);
            err[2 * i] = e0; err[2 * i + 1] = e1;
            if ((double)is2[i] * (e0 * e0 + e1 * e1) < (double)18.f) outl[i] = 0; else ++bad;
        }
        atomicAdd(&s_cnt[0], bad);
        __syncthreads();
        nBad = s_cnt[0];
        __syncthreads();
    }
    // ---- the prior of the next frame (:4819-4870 / :5216-5285) ----
    double acc[21];
#pragma unroll
    for (int k = 0; k < 21; ++k) acc[k] = 0;
    for (int i = tid; i < N; i += PI_NT) {
        if (outl[i]) continue;
        double e0, e1, Jp[12]; bool dp;
        mono_only_pose(Rcw, tcw, Rcb, Rbc, tbc, cm, Xw + 3 * i, ob + 2 * i, e0, e1, dp, Jp);
        const double om = (double)is2[i];
        int t = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a) {
#pragma unroll
            for (int c = a; c < 6; ++c) acc[t++] += om * (Jp[a] * Jp[c] + Jp[6 + a] * Jp[6 + c]);
        }
    }
    double tot[21];
#pragma unroll
    for (int k = 0; k < 21; ++k) tot[k] = block_sum<PI_NT>(acc[k], s_red);
    if (tid == 0) {
        double* Hout = Q.H15 + 225 * (size_t)f;
        double S36[36], e9[9], J[216];
        for (int k = 0; k < 21; ++k) S36[k] = s_sp[k];
        for (int k = 0; k < 15; ++k) S36[21 + k] = s_st[k];
        edge_inertial_dev(P, S36, e9, J);
        if constexpr (!LF) {
            for (int k = 0; k < 225; ++k) Hout[k] = 0;
            for (int a = 0; a < 9; ++a) for (int c = 0; c < 9; ++c) {
                double h = 0;
                for (int r = 0; r < 9; ++r) for (int k = 0; k < 9; ++k) h += J[r * 24 + 15 + a] * s_info[r * 9 + k] * J[k * 24 + 15 + c];
                Hout[a * 15 + c] += h;
            }
            for (int a = 0; a < 3; ++a) for (int c = 0; c < 3; ++c) { Hout[(9 + a) * 15 + 9 + c] += s_info[81 + a * 3 + c]; Hout[(12 + a) * 15 + 12 + c] += s_info[90 + a * 3 + c]; }
            int t = 0;
            for (int a = 0; a < 6; ++a) for (int c = a; c < 6; ++c) { Hout[a * 15 + c] += tot[t]; if (c != a) Hout[c * 15 + a] += tot[t]; ++t; }
        } else {
            // 30 x 30 in the reference's order (previous 15 | current 15), then Optimizer::Marginalize(H, 0, 14): H_cc - H_cb pinv(H_bb) H_bc
            double* Hf = s_H;
            for (int k = 0; k < 900; ++k) Hf[k] = 0;
            for (int a = 0; a < 24; ++a) for (int c = 0; c < 24; ++c) {
                double h = 0;
                for (int r = 0; r < 9; ++r) for (int k = 0; k < 9; ++k) h += J[r * 24 + a] * s_info[r * 9 + k] * J[k * 24 + c];
                Hf[a * 30 + c] += h;
            }
            for (int a = 0; a < 3; ++a) for (int c = 0; c < 3; ++c) {
                const double og = s_info[81 + a * 3 + c], oa = s_info[90 + a * 3 + c];
                Hf[(9 + a) * 30 + 9 + c] += og; Hf[(9 + a) * 30 + 24 + c] -= og; Hf[(24 + a) * 30 + 9 + c] -= og; Hf[(24 + a) * 30 + 24 + c] += og;
                Hf[(12 + a) * 30 + 12 + c] += oa; Hf[(12 + a) * 30 + 27 + c] -= oa; Hf[(27 + a) * 30 + 12 + c] -= oa; Hf[(27 + a) * 30 + 27 + c] += oa;
            }
            {
                double e15[15], Jp[225];
                prior_edge_dev(prior, s_sp, e15, Jp);
                for (int a = 0; a < 15; ++a) for (int c = 0; c < 15; ++c) {
                    double h = 0;
                    for (int r = 0; r < 15; ++r) for (int k = 0; k < 15; ++k) h += Jp[r * 15 + a] * priorH[r * 15 + k] * Jp[k * 15 + c];
                    Hf[a * 30 + c] += h;
                }
            }
            int t = 0;
            for (int a = 0; a < 6; ++a) for (int c = a; c < 6; ++c) { Hf[(15 + a) * 30 + 15 + c] += tot[t]; if (c != a) Hf[(15 + c) * 30 + 15 + a] += tot[t]; ++t; }
            // pseudo-inverse of the symmetrised H_bb through cyclic Jacobi (= the SVD of a symmetric matrix), eigenvalues with |w| <= 1e-6 dropped
            double* A = s_L; double* V = s_L + 225; double* Pv = s_L + 450;     // 3 x 225 of the 900-double scratch
            for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) { A[i * 15 + j] = (Hf[i * 30 + j] + Hf[j * 30 + i]) / 2; V[i * 15 + j] = i == j ? 1.0 : 0.0; }
            for (int sweep = 0; sweep < 100; ++sweep) {
                double off = 0, diag = 0;
                for (int p = 0; p < 15; ++p) { diag += A[p * 15 + p] * A[p * 15 + p]; for (int q = p + 1; q < 15; ++q) off += A[p * 15 + q] * A[p * 15 + q]; }
                if (off <= 1e-30 * diag || off < 1e-300) break;
                for (int p = 0; p < 15; ++p)
                    for (int q = p + 1; q < 15; ++q) {
                        const double apq = A[p * 15 + q];
                        if (apq == 0) continue;
                        const double theta = (A[q * 15 + q] - A[p * 15 + p]) / (2 * apq);
                        const double tt = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1));
                        const double cc = 1 / sqrt(tt * tt + 1), sn = tt * cc;
                        for (int k = 0; k < 15; ++k) { const double akp = A[k * 15 + p], akq = A[k * 15 + q]; A[k * 15 + p] = cc * akp - sn * akq; A[k * 15 + q] = sn * akp + cc * akq; }
                        for (int k = 0; k < 15; ++k) { const double apk = A[p * 15 + k], aqk = A[q * 15 + k]; A[p * 15 + k] = cc * apk - sn * aqk; A[q * 15 + k] = sn * apk + cc * aqk; }
                        for (int k = 0; k < 15; ++k) { const double vkp = V[k * 15 + p], vkq = V[k * 15 + q]; V[k * 15 + p] = cc * vkp - sn * vkq; V[k * 15 + q] = sn * vkp + cc * vkq; }
                    }
            }
            for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) {
                double a = 0;
                for (int k = 0; k < 15; ++k) { const double w = A[k * 15 + k]; if (fabs(w) > 1e-6) a += V[i * 15 + k] * V[j * 15 + k] / w; }
                Pv[i * 15 + j] = a;
            }
            for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) {
                double a = 0;
                for (int k = 0; k < 15; ++k) for (int l = 0; l < 15; ++l) a += Hf[(15 + i) * 30 + k] * Pv[k * 15 + l] * Hf[l * 30 + 15 + j];
                Hout[i * 15 + j] = Hf[(15 + i) * 30 + 15 + j] - a;
            }
        }
        Q.ret[f] = N - nBad;
    }
    __syncthreads();
    if (tid < 21) { Q.state[21 * (size_t)f + tid] = s_st[tid]; if (LF) Q.prevState[21 * (size_t)f + tid] = s_sp[tid]; }
}

// The two optimiser launches of the mono-inertial tracking call (pose_inertial.h): pose_inertial_opt_kernel<false> / <true> over the dense
// sub-batches the gather stage of track_inertial.cu wrote, one launch per variant that has streams.
int launch_inertial_optimisers(const ImuTrackArgs& A, cudaStream_t st) {
    int launches = 0;
    for (int v = 0; v < 2; ++v) {
        const int n = A.count[v];
        if (!n) continue;
        const size_t g0 = v ? A.count[0] : 0, K = A.kcap;
        PoseInertialParams Q;
        Q.count = n; Q.cap = A.kcap; Q.recInit = 0;
        Q.N = A.N + g0; Q.Xw = A.Xw + 3 * g0 * K; Q.obs = A.obs + 2 * g0 * K; Q.invSigma2 = A.invSigma2 + g0 * K; Q.trackDepth = A.trackDepth + g0 * K;
        Q.cam4 = A.cam4 + 4 * g0; Q.extr = A.extr; Q.preint = A.preint + (size_t)P_SIZE * g0;
        Q.state = A.state + 21 * g0; Q.err = A.err + 2 * g0 * K; Q.outlier = A.outlier + g0 * K; Q.H15 = A.H15 + 225 * g0; Q.ret = A.ret + g0;
        if (v == 0) {
            Q.kfState = A.fixedState; Q.preintKF = nullptr; Q.prior = nullptr; Q.priorH = nullptr; Q.prevState = nullptr;
            pose_inertial_opt_kernel<false><<<n, PI_NT, 0, st>>>(Q);
        } else {
            Q.kfState = nullptr; Q.preintKF = A.preintKF2 + (size_t)P_SIZE * g0; Q.prior = A.prior + 21 * g0; Q.priorH = A.priorH + 225 * g0;
            Q.prevState = A.fixedState + 21 * g0;          // the previous frame's estimate is discarded afterwards, as in the reference
            pose_inertial_opt_kernel<true><<<n, PI_NT, 0, st>>>(Q);
        }
        ++launches;
    }
    return launches;
}

}  // namespace imu

using namespace imu;
using orbx::ThreadStaging;

extern "C" {

int imu_preintegrate_batch(int count, const int32_t* nMeas, int maxMeas, const float* acc, const float* gyr, const float* dt, const float* bias6,
                           const float* noise4, float* preint, int device) {
    if (count < 1 || maxMeas < 1 || !nMeas || !acc || !gyr || !dt || !bias6 || !noise4 || !preint) { set_error("imu_preintegrate_batch: bad argument"); return ORB_ERR_ARG; }
    const size_t C = count, M = maxMeas;
    ThreadStaging* S;
    int rc = orbx::thread_staging(device, &S);
    if (rc) return rc;
    S->begin();
    const int pN = S->in(nMeas, 4 * C), pA = S->in(acc, 12 * C * M), pG = S->in(gyr, 12 * C * M), pT = S->in(dt, 4 * C * M), pB = S->in(bias6, 24 * C),
              pP = S->out(preint, 4 * P_SIZE * C);
    if ((rc = S->reserve())) return rc;
    cudaStream_t st = S->stream;
    CK(S->upload(st));
    // IMU::Calib::Set (src/ImuTypes.cc:395-407): squares in float
    const float ng2 = noise4[0] * noise4[0], na2 = noise4[1] * noise4[1], ngw2 = noise4[2] * noise4[2], naw2 = noise4[3] * noise4[3];
    imu_preintegrate_kernel<<<(count + 63) / 64, 64, 0, st>>>(count, S->dev<int>(pN), maxMeas, S->dev<float>(pA), S->dev<float>(pG), S->dev<float>(pT),
                                                              S->dev<float>(pB), ng2, na2, ngw2, naw2, S->dev<float>(pP));
    CK(cudaGetLastError());
    CK(S->download(st));
    return ORB_OK;
}

int imu_information_batch(int count, const float* preint, double* info9, double* infoG, double* infoA, int device) {
    if (count < 1 || !preint || !info9 || !infoG || !infoA) { set_error("imu_information_batch: bad argument"); return ORB_ERR_ARG; }
    const size_t C = count;
    ThreadStaging* S;
    int rc = orbx::thread_staging(device, &S);
    if (rc) return rc;
    S->begin();
    const int pP = S->in(preint, 4 * P_SIZE * C), pI = S->out(info9, 648 * C), pG = S->out(infoG, 72 * C), pA = S->out(infoA, 72 * C);
    if ((rc = S->reserve())) return rc;
    cudaStream_t st = S->stream;
    CK(S->upload(st));
    imu_information_kernel<<<(count + 31) / 32, 32, 0, st>>>(count, S->dev<float>(pP), S->dev<double>(pI), S->dev<double>(pG), S->dev<double>(pA));
    CK(cudaGetLastError());
    CK(S->download(st));
    return ORB_OK;
}

int imu_inertial_edges(int count, const float* preint, const double* states36, const double* info9, double huberDelta, double* err9, double* J9x24,
                       double* chi2, double* rho, int device) {
    if (count < 1 || !preint || !states36 || !err9 || (info9 && !chi2)) { set_error("imu_inertial_edges: bad argument"); return ORB_ERR_ARG; }
    const size_t C = count;
    ThreadStaging* S;
    int rc = orbx::thread_staging(device, &S);
    if (rc) return rc;
    S->begin();
    // chi2 is written whether or not the caller asked for it
    const int pP = S->in(preint, 4 * P_SIZE * C), pS = S->in(states36, 288 * C), pI = S->in(info9, info9 ? 648 * C : 0), pE = S->out(err9, 72 * C),
              pJ = S->out(J9x24, J9x24 ? 1728 * C : 0), pC = info9 ? S->out(chi2, 8 * C) : S->scratch(8 * C), pR = S->out(info9 ? rho : nullptr, rho ? 8 * C : 0);
    if ((rc = S->reserve())) return rc;
    cudaStream_t st = S->stream;
    CK(S->upload(st));
    inertial_edges_kernel<<<(count + 31) / 32, 32, 0, st>>>(count, S->dev<float>(pP), nullptr, S->dev<double>(pS), info9 ? S->dev<double>(pI) : nullptr, huberDelta,
                                                            S->dev<double>(pE), J9x24 ? S->dev<double>(pJ) : nullptr, S->dev<double>(pC), rho ? S->dev<double>(pR) : nullptr);
    CK(cudaGetLastError());
    CK(S->download(st));
    return ORB_OK;
}

int pose_inertial_optimization_last_kf_batch(int count, int cap, const int32_t* N, const float* Xw, const float* obs, const float* invSigma2, const float* trackDepth,
                                             const float* cam4, const double* extrinsics24, const float* preint, const double* kfState21, double* state21, int bRecInit,
                                             uint8_t* outlier, double* H15, int32_t* ret, int device) {
    if (count < 1 || cap < 1 || !N || !Xw || !obs || !invSigma2 || !trackDepth || !cam4 || !extrinsics24 || !preint || !kfState21 || !state21 || !outlier || !H15 || !ret) {
        set_error("pose_inertial_optimization_last_kf_batch: bad argument"); return ORB_ERR_ARG;
    }
    int rc = orbx::check_row_counts("pose_inertial_optimization_last_kf_batch", N, count, cap);
    if (rc) return rc;
    const size_t C = count, K = cap;
    ThreadStaging* S;
    rc = orbx::thread_staging(device, &S);
    if (rc) return rc;
    S->begin();
    const int pN = S->in(N, 4 * C), pX = S->in(Xw, 12 * C * K), pO = S->in(obs, 8 * C * K), pS = S->in(invSigma2, 4 * C * K), pT = S->in(trackDepth, 4 * C * K),
              pC = S->in(cam4, 16 * C), pE = S->in(extrinsics24, 192), pP = S->in(preint, 4 * P_SIZE * C), pK = S->in(kfState21, 168 * C),
              pSt = S->inout(state21, 168 * C), pOut = S->out(outlier, C * K), pH = S->out(H15, 1800 * C), pR = S->out(ret, 4 * C), pEr = S->scratch(16 * C * K);
    if ((rc = S->reserve())) return rc;
    cudaStream_t st = S->stream;
    CK(S->upload(st));
    PoseInertialParams Q;
    Q.count = count; Q.cap = cap; Q.recInit = bRecInit;
    Q.N = S->dev<int>(pN); Q.Xw = S->dev<float>(pX); Q.obs = S->dev<float>(pO); Q.invSigma2 = S->dev<float>(pS); Q.trackDepth = S->dev<float>(pT);
    Q.cam4 = S->dev<float>(pC); Q.extr = S->dev<double>(pE); Q.preint = S->dev<float>(pP); Q.kfState = S->dev<double>(pK); Q.state = S->dev<double>(pSt);
    Q.err = S->dev<double>(pEr); Q.outlier = S->dev(pOut); Q.H15 = S->dev<double>(pH); Q.ret = S->dev<int>(pR);
    Q.preintKF = nullptr; Q.prior = nullptr; Q.priorH = nullptr; Q.prevState = nullptr;
    pose_inertial_opt_kernel<false><<<count, PI_NT, 0, st>>>(Q);
    CK(cudaGetLastError());
    CK(S->download(st));
    orbx::zero_row_tails(outlier, N, count, cap);
    return ORB_OK;
}

int pose_inertial_optimization_last_frame_batch(int count, int cap, const int32_t* N, const float* Xw, const float* obs, const float* invSigma2, const float* trackDepth,
                                                const float* cam4, const double* extrinsics24, const float* preintFrame, const float* preintKF, const double* prior21,
                                                const double* priorH, double* prevState21, double* state21, int bRecInit, uint8_t* outlier, double* H15, int32_t* ret,
                                                int device) {
    if (count < 1 || cap < 1 || !N || !Xw || !obs || !invSigma2 || !trackDepth || !cam4 || !extrinsics24 || !preintFrame || !preintKF || !prior21 || !priorH || !prevState21 ||
        !state21 || !outlier || !H15 || !ret) {
        set_error("pose_inertial_optimization_last_frame_batch: bad argument"); return ORB_ERR_ARG;
    }
    int rc = orbx::check_row_counts("pose_inertial_optimization_last_frame_batch", N, count, cap);
    if (rc) return rc;
    const size_t C = count, K = cap;
    ThreadStaging* S;
    rc = orbx::thread_staging(device, &S);
    if (rc) return rc;
    S->begin();
    const int pN = S->in(N, 4 * C), pX = S->in(Xw, 12 * C * K), pO = S->in(obs, 8 * C * K), pS = S->in(invSigma2, 4 * C * K), pT = S->in(trackDepth, 4 * C * K),
              pC = S->in(cam4, 16 * C), pE = S->in(extrinsics24, 192), pP = S->in(preintFrame, 4 * P_SIZE * C), pPk = S->in(preintKF, 4 * P_SIZE * C),
              pPr = S->in(prior21, 168 * C), pPh = S->in(priorH, 1800 * C), pPv = S->inout(prevState21, 168 * C), pSt = S->inout(state21, 168 * C),
              pOut = S->out(outlier, C * K), pH = S->out(H15, 1800 * C), pR = S->out(ret, 4 * C), pEr = S->scratch(16 * C * K);
    if ((rc = S->reserve())) return rc;
    cudaStream_t st = S->stream;
    CK(S->upload(st));
    PoseInertialParams Q;
    Q.count = count; Q.cap = cap; Q.recInit = bRecInit;
    Q.N = S->dev<int>(pN); Q.Xw = S->dev<float>(pX); Q.obs = S->dev<float>(pO); Q.invSigma2 = S->dev<float>(pS); Q.trackDepth = S->dev<float>(pT);
    Q.cam4 = S->dev<float>(pC); Q.extr = S->dev<double>(pE); Q.preint = S->dev<float>(pP); Q.kfState = nullptr; Q.state = S->dev<double>(pSt);
    Q.err = S->dev<double>(pEr); Q.outlier = S->dev(pOut); Q.H15 = S->dev<double>(pH); Q.ret = S->dev<int>(pR);
    Q.preintKF = S->dev<float>(pPk); Q.prior = S->dev<double>(pPr); Q.priorH = S->dev<double>(pPh); Q.prevState = S->dev<double>(pPv);
    pose_inertial_opt_kernel<true><<<count, PI_NT, 0, st>>>(Q);
    CK(cudaGetLastError());
    CK(S->download(st));
    orbx::zero_row_tails(outlier, N, count, cap);
    return ORB_OK;
}

int imu_mono_edges(const ImuMonoEdges* in, double* err2, double* Jpoint2x3, double* Jpose2x6, double* chi2, double* rho, uint8_t* depthPositive, int device) {
    if (!in || in->nEdges < 1 || in->nPoses < 1 || in->nPoints < 1 || !in->poses || !in->extrinsics || !in->cam || !in->points || !in->edgePoint || !in->edgePose ||
        !in->obs || !in->invSigma2 || !err2 || !chi2 || !depthPositive || ((Jpoint2x3 == nullptr) != (Jpose2x6 == nullptr))) {
        set_error("imu_mono_edges: bad argument"); return ORB_ERR_ARG;
    }
    for (int e = 0; e < in->nEdges; ++e)
        if (in->edgePoint[e] < 0 || in->edgePoint[e] >= in->nPoints || in->edgePose[e] < 0 || in->edgePose[e] >= in->nPoses) { set_error("imu_mono_edges: edge index out of range"); return ORB_ERR_ARG; }
    const size_t E = in->nEdges, NP = in->nPoses, NL = in->nPoints;
    ThreadStaging* S;
    int rc = orbx::thread_staging(device, &S);
    if (rc) return rc;
    S->begin();
    const int pPo = S->in(in->poses, 96 * NP), pX = S->in(in->extrinsics, 192), pCm = S->in(in->cam, 16 * NP), pPt = S->in(in->points, 24 * NL),
              pEp = S->in(in->edgePoint, 4 * E), pEk = S->in(in->edgePose, 4 * E), pOb = S->in(in->obs, 16 * E), pIs = S->in(in->invSigma2, 4 * E),
              pEr = S->out(err2, 16 * E), pJp = S->out(Jpoint2x3, Jpoint2x3 ? 48 * E : 0), pJx = S->out(Jpose2x6, Jpose2x6 ? 96 * E : 0), pC2 = S->out(chi2, 8 * E),
              pRh = S->out(rho, rho ? 8 * E : 0), pDp = S->out(depthPositive, E);
    if ((rc = S->reserve())) return rc;
    cudaStream_t st = S->stream;
    CK(S->upload(st));
    MonoParams Q;
    Q.nEdges = in->nEdges; Q.poses = S->dev<double>(pPo); Q.extr = S->dev<double>(pX); Q.cam = S->dev<float>(pCm); Q.points = S->dev<double>(pPt);
    Q.edgePoint = S->dev<int>(pEp); Q.edgePose = S->dev<int>(pEk); Q.obs = S->dev<double>(pOb); Q.invSigma2 = S->dev<float>(pIs);
    Q.huberDelta = in->huberDelta; Q.err = S->dev<double>(pEr); Q.Jpoint = Jpoint2x3 ? S->dev<double>(pJp) : nullptr; Q.Jpose = Jpose2x6 ? S->dev<double>(pJx) : nullptr;
    Q.chi2 = S->dev<double>(pC2); Q.rho = rho ? S->dev<double>(pRh) : nullptr; Q.depthPositive = S->dev(pDp);
    mono_imu_edges_kernel<<<(in->nEdges + 127) / 128, 128, 0, st>>>(Q);
    CK(cudaGetLastError());
    CK(S->download(st));
    return ORB_OK;
}

}  // extern "C"
