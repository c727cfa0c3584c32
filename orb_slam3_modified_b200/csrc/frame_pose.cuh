// Frame::SetPose / Frame::UpdatePoseMatrices (reference src/Frame.cc) in float, shared by the batched tracking calls
// (orbm_motion_model_pose_batch*, orbm_track_local_map_batch*): the pose kernel hands its double estimate over with set_pose_from_double,
// the frustum stage derives mRcw / mtcw / mOw from the float pose with update_pose_matrices.  Every float operation rounds once (exact_math.h),
// so tests/track_lib.py restates both in numpy float32 bit for bit.
#pragma once
#include "exact_math.h"

namespace orbm {

// PoseOptimization's hand-over at the end of src/Optimizer.cc:814-1114: Sophus::SE3<float>(SE3quat_recov.rotation().cast<float>(),
// SE3quat_recov.translation().cast<float>()).  The SO3 constructor normalises the float quaternion.  Stand-in for Eigen's
// normalize(): n = ((x*x + y*y) + z*z) + w*w summed in storage order (x, y, z, w), every coefficient divided by sqrtf(n).  Eigen's
// vectorised reduction may pair the terms differently; bit agreement with it is not claimed.  T7 / Tcw7: (w, x, y, z, tx, ty, tz).
__device__ __forceinline__ void set_pose_from_double(const double* T7, float* Tcw7) {
    using namespace orbx;
    const float w = (float)T7[0], x = (float)T7[1], y = (float)T7[2], z = (float)T7[3];
    const float n = fadd(fadd(fadd(fmul(x, x), fmul(y, y)), fmul(z, z)), fmul(w, w));
    const float s = __fsqrt_rn(n);
    Tcw7[0] = fdiv(w, s); Tcw7[1] = fdiv(x, s); Tcw7[2] = fdiv(y, s); Tcw7[3] = fdiv(z, s);
    Tcw7[4] = (float)T7[4]; Tcw7[5] = (float)T7[5]; Tcw7[6] = (float)T7[6];
}

// Frame::UpdatePoseMatrices: mRcw = mTcw.rotationMatrix() (Eigen's QuaternionBase::toRotationMatrix, row-major), mtcw = mTcw.translation(),
// mOw = mTcw.inverse().translation() = -(q^-1 * t) with Sophus' quaternion rotation (so3.hpp:358-367; oracle/ref_shim/ref_slam_types.cpp).
__device__ __forceinline__ void update_pose_matrices(const float* T, float* R, float* t, float* Ow) {
    using namespace orbx;
    const float qw = T[0], qx = T[1], qy = T[2], qz = T[3];
    const float tx = fmul(2.0f, qx), ty = fmul(2.0f, qy), tz = fmul(2.0f, qz);
    const float twx = fmul(tx, qw), twy = fmul(ty, qw), twz = fmul(tz, qw);
    const float txx = fmul(tx, qx), txy = fmul(ty, qx), txz = fmul(tz, qx);
    const float tyy = fmul(ty, qy), tyz = fmul(tz, qy), tzz = fmul(tz, qz);
    R[0] = fsub(1.0f, fadd(tyy, tzz)); R[1] = fsub(txy, twz); R[2] = fadd(txz, twy);
    R[3] = fadd(txy, twz); R[4] = fsub(1.0f, fadd(txx, tzz)); R[5] = fsub(tyz, twx);
    R[6] = fsub(txz, twy); R[7] = fadd(tyz, twx); R[8] = fsub(1.0f, fadd(txx, tyy));
    t[0] = T[4]; t[1] = T[5]; t[2] = T[6];
    const float ix = -qx, iy = -qy, iz = -qz, px = T[4], py = T[5], pz = T[6];
    float ux = fsub(fmul(iy, pz), fmul(iz, py)), uy = fsub(fmul(iz, px), fmul(ix, pz)), uz = fsub(fmul(ix, py), fmul(iy, px));
    ux = fadd(ux, ux); uy = fadd(uy, uy); uz = fadd(uz, uz);
    const float cx = fsub(fmul(iy, uz), fmul(iz, uy)), cy = fsub(fmul(iz, ux), fmul(ix, uz)), cz = fsub(fmul(ix, uy), fmul(iy, ux));
    Ow[0] = -fadd(fadd(px, fmul(qw, ux)), cx);
    Ow[1] = -fadd(fadd(py, fmul(qw, uy)), cy);
    Ow[2] = -fadd(fadd(pz, fmul(qw, uz)), cz);
}

}  // namespace orbm
