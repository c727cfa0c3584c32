// The mono-inertial tracking call (pose_inertial.h, orbm_track_local_map_inertial_batch* in matcher.cu): Tracking::PredictStateIMU
// before the frustum and search stages of matcher.cu; after them the matches are gathered into dense sub-batches,
// pose_inertial_opt_kernel (inertial.cu) runs on them unchanged, and the write-back applies SetImuPoseVelocity, the bias, TrackLocalMap's
// statistics loop and ConstraintPoseImu.  One CTA of PI_NT threads per stream in each kernel; skipped streams leave at once.
#include <cuda_runtime.h>
#include <math.h>

#include "../../include/orb_b200.h"
#include "frame_pose.cuh"
#include "inertial_dev.cuh"
#include "pose_inertial.h"

namespace imu {

constexpr int PI_NT = 128;   // as pose_inertial_opt_kernel


// Tracking::PredictStateIMU (src/Tracking.cc), float like the reference.  Map updated (slot < count[0]): from mpLastKeyFrame with
// mpImuPreintegratedFromLastKF; else from mLastFrame with mpImuPreintegratedFrame; each with the source's bias.
//   Rwb2 = NormalizeRotation(Rwb1 dR(b)), twb2 = ((twb1 + Vwb1 t12) + (0.5 t12 t12) Gz) + Rwb1 dP(b), Vwb2 = (Vwb1 + t12 Gz) + Rwb1 dV(b)
// then Frame::SetImuPoseVelocity (frame_pose.cuh); predState21 is what ImuCamPose(Frame*) reads back, with mImuBias = the source's bias.
__global__ void __launch_bounds__(PI_NT) predict_state_imu_kernel(ImuTrackArgs A) {
    const int b = blockIdx.x, g = A.route[b];
    if (g < 0) return;
    for (int i = threadIdx.x; i < A.kcap; i += PI_NT) A.match[(size_t)b * A.kcap + i] = -1;
    if (threadIdx.x != 0) return;
    const bool fromKF = g < A.count[0];
    const float* S = (fromKF ? A.kfState21 : A.lastState21) + 21 * (size_t)b;
    const float* P = (fromKF ? A.preintKF : A.preintFrame) + (size_t)P_SIZE * b;
    const float *Rwb1 = S, *twb1 = S + 9, *V1 = S + 12;
    const float dbg[3] = {S[15] - P[P_B + 3], S[16] - P[P_B + 4], S[17] - P[P_B + 5]};
    const float dba[3] = {S[18] - P[P_B], S[19] - P[P_B + 1], S[20] - P[P_B + 2]};
    float dR[9], dV[3], dP[3];
    preint_delta_f(P, dbg, dba, dR, dV, dP);
    const float t12 = P[P_DT];
    float M[9], Rwb2[9], RdP[3], RdV[3], twb2[3], Vwb2[3];
    m3mul(Rwb1, dR, M);
    normalize_rotation(M, Rwb2);
    m3vec(Rwb1, dP, RdP); m3vec(Rwb1, dV, RdV);
    const float Gz[3] = {0.f, 0.f, -9.81f};
    const float h = __fmul_rn(__fmul_rn(0.5f, t12), t12);
    for (int i = 0; i < 3; ++i) {
        twb2[i] = __fadd_rn(__fadd_rn(__fadd_rn(twb1[i], __fmul_rn(V1[i], t12)), __fmul_rn(h, Gz[i])), RdP[i]);
        Vwb2[i] = __fadd_rn(__fadd_rn(V1[i], __fmul_rn(t12, Gz[i])), RdV[i]);
    }
    float* out = A.predState21 + 21 * (size_t)b;
    orbm::set_imu_pose(A.Tcb7, Rwb2, twb2, A.predTcw7 + 7 * (size_t)b, out, out + 9);
    for (int i = 0; i < 3; ++i) out[12 + i] = Vwb2[i];
    for (int i = 15; i < 21; ++i) out[i] = S[i];
}

// Block-wide compaction of each routed stream's matches in keypoint order (as gather_edges_kernel in pose_opt.cu) into
// PoseInertialParams' float layout at the stream's slot, plus the per-slot operands: the camera, the current frame's initial state
// (double of predState21), the fixed last keyframe (map updated) or the previous frame and its prior (not updated), the preintegrations.
__global__ void __launch_bounds__(PI_NT) gather_inertial_kernel(ImuTrackArgs A) {
    __shared__ int s_cnt[PI_NT / 32];
    const int b = blockIdx.x, g = A.route[b], tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (g < 0) return;
    const bool fromKF = g < A.count[0];
    const size_t kb = (size_t)b * A.kcap, pb = (size_t)b * A.pstride, sb = (size_t)g * A.kcap;
    const int K = min(A.nK[b], A.kcap);
    if (tid < 21) {
        A.state[21 * (size_t)g + tid] = (double)A.predState21[21 * (size_t)b + tid];
        A.fixedState[21 * (size_t)g + tid] = (double)(fromKF ? A.kfState21 : A.lastState21)[21 * (size_t)b + tid];
        if (!fromKF) A.prior[21 * (size_t)g + tid] = A.priorIn[21 * (size_t)b + tid];
    }
    if (tid < 4) A.cam4[4 * g + tid] = A.cam[tid];
    for (int k = tid; k < P_SIZE; k += PI_NT) {
        A.preint[(size_t)P_SIZE * g + k] = (fromKF ? A.preintKF : A.preintFrame)[(size_t)P_SIZE * b + k];
        if (!fromKF) A.preintKF2[(size_t)P_SIZE * g + k] = A.preintKF[(size_t)P_SIZE * b + k];
    }
    if (!fromKF) for (int k = tid; k < 225; k += PI_NT) A.priorH[225 * (size_t)g + k] = A.priorHIn[225 * (size_t)b + k];
    int base = 0;
    for (int t0 = 0; t0 < K; t0 += PI_NT) {
        const int i = t0 + tid;
        const int m = i < K ? A.match[kb + i] : -1;
        const unsigned bits = __ballot_sync(0xffffffffu, m >= 0);
        if (lane == 0) s_cnt[wid] = __popc(bits);
        __syncthreads();
        int off = 0, tot = 0;
#pragma unroll
        for (int w = 0; w < PI_NT / 32; ++w) { off += w < wid ? s_cnt[w] : 0; tot += s_cnt[w]; }
        if (m >= 0) {
            const size_t e = sb + base + off + __popc(bits & ((1u << lane) - 1u));
            const OrbKeyPoint kp = A.kps[kb + i];
            const float* X = A.xyz + 3 * (pb + m);
            A.Xw[3 * e] = X[0]; A.Xw[3 * e + 1] = X[1]; A.Xw[3 * e + 2] = X[2];
            A.obs[2 * e] = kp.x; A.obs[2 * e + 1] = kp.y;
            A.invSigma2[e] = A.invLevelSigma2[min(max(kp.octave, 0), A.nlevels - 1)];   // the host entry points reject out-of-range octaves
            A.trackDepth[e] = A.depth[pb + m];
            A.edgeKp[e] = i;
        }
        base += tot;
        __syncthreads();
    }
    if (tid == 0) A.N[g] = base;
}

// ConstraintPoseImu's constructor (include/G2oTypes.h:711-722) by one warp, equal bit for bit to the CPU oracle's
// (oracle/inertial_oracle.cpp: orbo_constraint_pose_imu_information, sym_eig): symmetrise, cyclic Jacobi, eigenvalues below 1e-12 set to 0,
// V diag(w) V^T.  Every double operation is an explicit round-to-nearest intrinsic in the oracle's order (the oracle is built with
// -ffp-contract=off; sqrt, fabs and division are correctly rounded on both sides).  The three k loops of a rotation touch disjoint
// elements for different k, so lanes take k and a __syncwarp between the loops keeps each element's serial order.
__device__ void constraint_information_warp(const double* Hin, double* Hout, double* A, double* V) {
    const int lane = threadIdx.x & 31;
    for (int idx = lane; idx < 225; idx += 32) {
        const int i = idx / 15, j = idx - i * 15;
        A[idx] = __ddiv_rn(__dadd_rn(Hin[i * 15 + j], Hin[j * 15 + i]), 2.0);
        V[idx] = i == j ? 1.0 : 0.0;
    }
    __syncwarp();
    for (int sweep = 0; sweep < 100; ++sweep) {
        double off = 0, diag = 0;
        for (int p = 0; p < 15; ++p) {
            diag = __dadd_rn(diag, __dmul_rn(A[p * 15 + p], A[p * 15 + p]));
            for (int q = p + 1; q < 15; ++q) off = __dadd_rn(off, __dmul_rn(A[p * 15 + q], A[p * 15 + q]));
        }
        if (off <= __dmul_rn(1e-30, diag) || off < 1e-300) break;
        for (int p = 0; p < 15; ++p)
            for (int q = p + 1; q < 15; ++q) {
                const double apq = A[p * 15 + q];
                if (apq == 0) continue;
                const double theta = __ddiv_rn(__dsub_rn(A[q * 15 + q], A[p * 15 + p]), __dmul_rn(2.0, apq));
                const double t = __ddiv_rn(theta >= 0 ? 1.0 : -1.0, __dadd_rn(fabs(theta), __dsqrt_rn(__dadd_rn(__dmul_rn(theta, theta), 1.0))));
                const double c = __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(__dmul_rn(t, t), 1.0))), sn = __dmul_rn(t, c);
                __syncwarp();
                const int k = lane;
                if (k < 15) {
                    const double akp = A[k * 15 + p], akq = A[k * 15 + q];
                    A[k * 15 + p] = __dsub_rn(__dmul_rn(c, akp), __dmul_rn(sn, akq)); A[k * 15 + q] = __dadd_rn(__dmul_rn(sn, akp), __dmul_rn(c, akq));
                }
                __syncwarp();
                if (k < 15) {
                    const double apk = A[p * 15 + k], aqk = A[q * 15 + k];
                    A[p * 15 + k] = __dsub_rn(__dmul_rn(c, apk), __dmul_rn(sn, aqk)); A[q * 15 + k] = __dadd_rn(__dmul_rn(sn, apk), __dmul_rn(c, aqk));
                    const double vkp = V[k * 15 + p], vkq = V[k * 15 + q];
                    V[k * 15 + p] = __dsub_rn(__dmul_rn(c, vkp), __dmul_rn(sn, vkq)); V[k * 15 + q] = __dadd_rn(__dmul_rn(sn, vkp), __dmul_rn(c, vkq));
                }
                __syncwarp();
            }
    }
    for (int idx = lane; idx < 225; idx += 32) {
        const int i = idx / 15, j = idx - i * 15;
        double a = 0;
        for (int k = 0; k < 15; ++k) {
            double w = A[k * 15 + k];
            if (w < 1e-12) w = 0;
            a = __dadd_rn(a, __dmul_rn(__dmul_rn(V[i * 15 + k], w), V[j * 15 + k]));
        }
        Hout[idx] = a;
    }
}

// The write-back of PoseInertialOptimizationLast{KeyFrame,Frame} and TrackLocalMap's statistics loop: mvbOutlier scattered to keypoints,
// found += 1 per inlier, mnMatchesInliers = inliers whose point has observations; SetImuPoseVelocity of the float estimate and
// mImuBias = the optimised bias (state21 as the next ImuCamPose(Frame*) reads it, Tcw7); mpcpi = ConstraintPoseImu(double estimate, H).
__global__ void __launch_bounds__(PI_NT) inertial_finish_kernel(ImuTrackArgs A) {
    __shared__ double s_A[225], s_V[225];
    __shared__ int s_n;
    const int b = blockIdx.x, g = A.route[b], tid = threadIdx.x;
    if (g < 0) return;
    const size_t kb = (size_t)b * A.kcap, pb = (size_t)b * A.pstride, sb = (size_t)g * A.kcap;
    const int N = A.N[g];
    if (tid == 0) s_n = 0;
    for (int i = tid; i < A.kcap; i += PI_NT) A.outlierKp[kb + i] = 0;
    __syncthreads();
    int nObs = 0;
    for (int e = tid; e < N; e += PI_NT) {
        const int i = A.edgeKp[sb + e];
        const int p = A.match[kb + i];
        const uint8_t o = A.outlier[sb + e];
        A.outlierKp[kb + i] = o;
        if (!o) { atomicAdd(&A.found[pb + p], 1); nObs += A.hasObs[pb + p] != 0; }
    }
    if (nObs) atomicAdd(&s_n, nObs);
    if (tid < 32) constraint_information_warp(A.H15 + 225 * (size_t)g, A.priorHOut + 225 * (size_t)b, s_A, s_V);
    if (tid == 32) {
        const double* st = A.state + 21 * (size_t)g;
        float Rwb[9], twb[3];
        for (int i = 0; i < 9; ++i) Rwb[i] = (float)st[i];
        for (int i = 0; i < 3; ++i) twb[i] = (float)st[9 + i];
        float* out = A.state21 + 21 * (size_t)b;
        orbm::set_imu_pose(A.Tcb7, Rwb, twb, A.Tcw7 + 7 * (size_t)b, out, out + 9);
        for (int i = 12; i < 21; ++i) out[i] = (float)st[i];
    }
    if (tid < 21) A.priorOut[21 * (size_t)b + tid] = A.state[21 * (size_t)g + tid];
    __syncthreads();
    if (tid == 0) { A.nMatchesInliers[b] = s_n; A.nInliers[b] = A.ret[g]; }
}

cudaError_t launch_predict_imu(const ImuTrackArgs& A, cudaStream_t st) {
    predict_state_imu_kernel<<<A.batch, PI_NT, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t launch_gathered_inertial(const ImuTrackArgs& A, cudaStream_t st, int* launches) {
    gather_inertial_kernel<<<A.batch, PI_NT, 0, st>>>(A);
    const int n = launch_inertial_optimisers(A, st);
    inertial_finish_kernel<<<A.batch, PI_NT, 0, st>>>(A);
    *launches = 2 + n;
    return cudaGetLastError();
}

}  // namespace imu
