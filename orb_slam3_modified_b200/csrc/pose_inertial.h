// The mono-inertial tracking call of matcher.cu (orbm_track_local_map_inertial_batch*): Tracking::PredictStateIMU before its frustum and
// search stages, and after them the inertial pose optimisers of inertial.cu over edges gathered on the device from each stream's matches.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/orb_b200.h"

namespace imu {

// Streams are routed by the host's mode array: route[b] = -1 for a skipped stream (mode 0), else its slot g in the optimiser scratch.
// Slots [0, count[0]) hold the map-updated streams (PoseInertialOptimizationLastKeyFrame), slots [count[0], count[0] + count[1]) the
// others (PoseInertialOptimizationLastFrame), each sub-batch in stream order; the two optimiser launches read dense sub-batches.
struct ImuTrackArgs {
    int batch, kcap, pstride, nlevels;
    int count[2];
    const int* route;                                    // [batch]
    float Tcb7[7];                                       // mImuCalib.mTcb (w, x, y, z, t)
    const double* extr;                                  // [24] Rcb | tcb | Rbc | tbc
    const float *preintKF, *preintFrame;                 // [batch][P_SIZE]
    const float *kfState21, *lastState21;                // [batch][21] Rwb | twb | v | bg | ba (float)
    const double *priorIn, *priorHIn;                    // [batch][21], [batch][225]
    // PredictStateIMU
    float *predState21, *predTcw7;                       // [batch][21], [batch][7]
    int* match;                                          // [batch][kcap]: -1 before the search
    // gather: the frame, its matches and the frustum stage's depths
    const OrbKeyPoint* kps; const int* nK;
    const float* xyz; const uint8_t* hasObs; const float* depth;   // [batch][pstride][3], [batch][pstride], [batch][pstride]
    const float* invLevelSigma2; float cam[4];
    // write-back
    uint8_t* outlierKp; int* found; int *nInliers, *nMatchesInliers;   // [batch][kcap], [batch][pstride], [batch] x 2
    float *Tcw7, *state21; double *priorOut, *priorHOut;                // [batch][7], [batch][21], [batch][21], [batch][225]
    // scratch per slot: edges [slot][kcap] and the optimiser's operands / results
    float *Xw, *obs, *invSigma2, *trackDepth; int* edgeKp; double* err; uint8_t* outlier;
    int* N; float* cam4; float *preint, *preintKF2; double *fixedState, *state, *prior, *priorH, *H15; int* ret;
};
// track_inertial.cu.  One launch: PredictStateIMU + SetImuPoseVelocity for every routed stream (predState21, predTcw7; match = -1).
cudaError_t launch_predict_imu(const ImuTrackArgs& A, cudaStream_t st);
// track_inertial.cu.  Three or four launches: the gather, the optimisers (launch_inertial_optimisers), and the write-back (outlier flags,
// found, the counts, SetImuPoseVelocity, the bias, ConstraintPoseImu).
cudaError_t launch_gathered_inertial(const ImuTrackArgs& A, cudaStream_t st, int* launches);
// inertial.cu, next to the kernel it launches (a kernel in its own translation unit keeps its compiled code): pose_inertial_opt_kernel
// <false> / <true> on the sub-batches that have streams.  Returns the number of launches.
int launch_inertial_optimisers(const ImuTrackArgs& A, cudaStream_t st);

}  // namespace imu
