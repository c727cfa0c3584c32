// Optimizer::PoseOptimization over edges gathered on the device from a frame's matches: the launches the batched tracking calls of
// matcher.cu (orbm_motion_model_pose_batch*, orbm_track_local_map_batch*) make around pose_optimization_batch's kernel (pose_opt.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/orb_b200.h"

namespace poseopt {

// Per stream f (one CTA): the edges are the keypoints i < nK[f] with match[i] >= 0 in ascending i -- the order in which
// PoseOptimization's loop over pFrame->N adds them, so edge e is the edge the host packing of pose_optimization_batch makes -- with Xw = (double)xyz[match[i]],
// obs = (double)kps[i].(x, y) and invSigma2 = invLevelSigma2[kps[i].octave].  The initial pose is (double) of the float Tcw.
// After the four rounds the optimised pose goes to poseOut and, through Frame::SetPose (frame_pose.cuh), to TcwOut (which may
// alias TcwIn); with fewer than three edges PoseOptimization returns before SetPose and TcwOut receives TcwIn unchanged.
// The epilogue is one of the two loops that follow PoseOptimization in Tracking:
//   MOTION_MODEL  TrackWithMotionModel's "discard outliers" loop after its PoseOptimization (src/Tracking.cc:2912): an outlier keypoint loses its match
//                 (match = -1, claimed = 0, nmatches[f]--, discarded[f][point] = 1 for mnLastFrameSeen); nmatchesMap[f] counts the
//                 inliers whose point has observations.  discarded is rewritten over all pstride entries of the row.
//   LOCAL_MAP     the statistics loop after TrackLocalMap's PoseOptimization (src/Tracking.cc:2952 ff.): found[f][point] += 1 per inlier, nMatchesInliers[f] counts
//                 the inliers whose point has observations; outlierKp[f][kcap] = mvbOutlier (0 for keypoints without a match).
enum GatherMode { MOTION_MODEL = 0, LOCAL_MAP = 1 };
struct GatherArgs {
    int batch, kcap, pstride, nlevels, mode;
    const uint8_t* active;                 // [batch] or null (all streams)
    const OrbKeyPoint* kps; const int* nK; // [batch][kcap], [batch]
    int* match; uint8_t* claimed; int* nmatches;        // [batch][kcap] (point index into the xyz rows), [batch][kcap], [batch]
    const float* xyz; const uint8_t* hasObs;            // [batch][pstride][3], [batch][pstride]
    const float* invLevelSigma2; float cam[4];
    const float* TcwIn; float* TcwOut; double* poseOut; int* nInliers;   // [batch][7] x 3, [batch]
    uint8_t* discarded; int* nmatchesMap;                                // MOTION_MODEL
    uint8_t* outlierKp; int* found; int* nMatchesInliers;               // LOCAL_MAP
    // scratch [batch][kcap]: the compacted edges and PoseOptimization's per-edge state; [batch]: its other operands and results
    double *Xw, *obs, *err; float* invSigma2; uint8_t* outlier; int* edgeKp;
    int* N; double *poseIn, *poseTmp; float* cam4; int* nInlTmp;     // [batch], [batch][7] x 2, [batch][4], [batch]
};
// Enqueues three launches (gather, pose_opt_kernel, SetPose + loop; one CTA per stream each) on `st`.
cudaError_t launch_gathered(const GatherArgs& A, cudaStream_t st);

}  // namespace poseopt
