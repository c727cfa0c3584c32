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

// Sophus::SO3 rotation of a point (so3.hpp:358-367): uv = q.vec x p; uv += uv; (p + w uv) + q.vec x uv
__device__ __forceinline__ void quat_rotate(const float* q, const float* p, float* o) {
    using namespace orbx;
    float ux = fsub(fmul(q[2], p[2]), fmul(q[3], p[1])), uy = fsub(fmul(q[3], p[0]), fmul(q[1], p[2])), uz = fsub(fmul(q[1], p[1]), fmul(q[2], p[0]));
    ux = fadd(ux, ux); uy = fadd(uy, uy); uz = fadd(uz, uz);
    const float cx = fsub(fmul(q[2], uz), fmul(q[3], uy)), cy = fsub(fmul(q[3], ux), fmul(q[1], uz)), cz = fsub(fmul(q[1], uy), fmul(q[2], ux));
    o[0] = fadd(fadd(p[0], fmul(q[0], ux)), cx);
    o[1] = fadd(fadd(p[1], fmul(q[0], uy)), cy);
    o[2] = fadd(fadd(p[2], fmul(q[0], uz)), cz);
}
// SE3f::inverse: (conj q, -(conj q * t))
__device__ __forceinline__ void se3_inverse(const float* T, float* I) {
    I[0] = T[0]; I[1] = -T[1]; I[2] = -T[2]; I[3] = -T[3];
    float r[3];
    quat_rotate(I, T + 4, r);
    I[4] = -r[0]; I[5] = -r[1]; I[6] = -r[2];
}
// Sophus' SE3 action on a point: T * p = q * p + t
__device__ __forceinline__ void se3_transform(const float* T, const float* p, float* o) {
    using namespace orbx;
    quat_rotate(T, p, o);
    o[0] = fadd(o[0], T[4]); o[1] = fadd(o[1], T[5]); o[2] = fadd(o[2], T[6]);
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
    float I[7];
    se3_inverse(T, I);
    Ow[0] = I[4]; Ow[1] = I[5]; Ow[2] = I[6];
}

// ---- Frame::SetImuPoseVelocity and GetImuRotation / GetImuPosition (src/Frame.cc) for the mono-inertial tracking call
//      (orbm_track_local_map_inertial_batch*).  The Sophus operations restate the stand-ins of oracle/ref_shim/ref_slam_types.cpp one
//      rounding per operation: Eigen's matrix-to-quaternion conversion (not normalised, as SO3's matrix constructor keeps it), the SE3
//      inverse, the SE3 product (quaternion product not renormalised) and Matrix3f * Matrix3f / Vector3f summed left to right.  Bit agreement
//      with Eigen / Sophus is not claimed, as for set_pose_from_double. ----

// Sophus::SE3f(Matrix3f R, Vector3f t): Eigen's quaternion from a rotation matrix (R row-major); T = (w, x, y, z, t)
__device__ __forceinline__ void se3_from_matrix(const float* R, const float* t, float* T) {
    using namespace orbx;
    float tr = fadd(fadd(R[0], R[4]), R[8]);
    if (tr > 0) {
        tr = __fsqrt_rn(fadd(tr, 1.0f));
        T[0] = fmul(0.5f, tr); tr = fdiv(0.5f, tr);
        T[1] = fmul(fsub(R[7], R[5]), tr); T[2] = fmul(fsub(R[2], R[6]), tr); T[3] = fmul(fsub(R[3], R[1]), tr);
    } else {
        int i = 0;
        if (R[4] > R[0]) i = 1;
        if (R[8] > R[i * 4]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        tr = __fsqrt_rn(fadd(fsub(fsub(R[i * 4], R[j * 4]), R[k * 4]), 1.0f));
        float q[3];
        q[i] = fmul(0.5f, tr); tr = fdiv(0.5f, tr);
        T[0] = fmul(fsub(R[k * 3 + j], R[j * 3 + k]), tr);
        q[j] = fmul(fadd(R[j * 3 + i], R[i * 3 + j]), tr); q[k] = fmul(fadd(R[k * 3 + i], R[i * 3 + k]), tr);
        T[1] = q[0]; T[2] = q[1]; T[3] = q[2];
    }
    T[4] = t[0]; T[5] = t[1]; T[6] = t[2];
}
// SE3f * SE3f: quaternion product, translation A.q * B.t + A.t
__device__ __forceinline__ void se3_mul(const float* A, const float* B, float* C) {
    using namespace orbx;
    const float w = A[0], x = A[1], y = A[2], z = A[3];
    C[0] = fsub(fsub(fsub(fmul(w, B[0]), fmul(x, B[1])), fmul(y, B[2])), fmul(z, B[3]));
    C[1] = fsub(fadd(fadd(fmul(w, B[1]), fmul(x, B[0])), fmul(y, B[3])), fmul(z, B[2]));
    C[2] = fsub(fadd(fadd(fmul(w, B[2]), fmul(y, B[0])), fmul(z, B[1])), fmul(x, B[3]));
    C[3] = fsub(fadd(fadd(fmul(w, B[3]), fmul(z, B[0])), fmul(x, B[2])), fmul(y, B[1]));
    se3_transform(A, B + 4, C + 4);
}
// Frame::SetImuPoseVelocity's pose part: mTcw = mImuCalib.mTcb * SE3f(Rwb, twb).inverse() (Tcb7 = (w, x, y, z, t)); then UpdatePoseMatrices
// and what ImuCamPose(Frame*) reads back: GetImuRotation = mRwc * mTcb.rotationMatrix(), GetImuPosition = mRwc * mTcb.translation() + mOw
// (mRwc = the rotation matrix of the conjugate quaternion, which is mRcw transposed bit for bit).
__device__ __forceinline__ void set_imu_pose(const float* Tcb7, const float* Rwb, const float* twb, float* Tcw7, float* Rimu, float* timu) {
    using namespace orbx;
    float Twb[7], Tbw[7];
    se3_from_matrix(Rwb, twb, Twb);
    se3_inverse(Twb, Tbw);
    se3_mul(Tcb7, Tbw, Tcw7);
    float Rcw[9], tcw[3], Ow[3], Rcb[9], tcb[3], dummy[3];
    update_pose_matrices(Tcw7, Rcw, tcw, Ow);
    update_pose_matrices(Tcb7, Rcb, tcb, dummy);
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j)
            Rimu[i * 3 + j] = fadd(fadd(fmul(Rcw[i], Rcb[j]), fmul(Rcw[3 + i], Rcb[3 + j])), fmul(Rcw[6 + i], Rcb[6 + j]));
        timu[i] = fadd(fadd(fadd(fmul(Rcw[i], tcb[0]), fmul(Rcw[3 + i], tcb[1])), fmul(Rcw[6 + i], tcb[2])), Ow[i]);
    }
}

}  // namespace orbm
