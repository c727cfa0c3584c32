// Device / host math shared by the optimiser kernels (lba.cu, pose_opt.cu, inertial.cu, local_inertial_ba.cu) and by the host-side emulation
// of the LocalInertialBA kernel (tests/liba_emulate.cpp compiles the same phase functions with g++): SO3 helpers (reference src/G2oTypes.cc:777-861),
// NormalizeRotation (src/ImuTypes.cc:34-37), the information matrices of EdgeInertial / EdgeGyroRW / EdgeAccRW (src/G2oTypes.cc:499-507,
// src/Optimizer.cc:2645-2654), EdgeInertial::computeError / linearizeOplus (src/G2oTypes.cc:514-594), EdgeMono / EdgeMonoOnlyPose with ImuCamPose
// (src/G2oTypes.cc:349-395), and in namespace g2o the g2o pieces every optimiser kernel uses: SE3Quat and VertexSE3Expmap::oplusImpl,
// RobustKernelHuber::robustify and OptimizationAlgorithmLevenberg::solve's damping policy with ORB-SLAM3's nBad stop rule.
#pragma once
#include <float.h>
#include <math.h>
#if defined(__CUDACC__)
#define IMU_HD __host__ __device__
#else
#define IMU_HD
#ifndef __restrict__
#define __restrict__ __restrict
#endif
#endif

namespace imu {

// Product rounded on its own (never fused into a following addition) for the FLOAT arithmetic of IMU::Preintegrated: the bias-corrected
// delta rotation / velocity / position are float in the reference (src/ImuTypes.cc:283-307) and every last-bit difference in them moves
// the optimised states by ~1e-7, so the device evaluates them exactly like the CPU oracle (which is built with -ffp-contract=off).
// Doubles are left to the compiler (their contraction changes results at the 1e-15 level only).
template <class T> IMU_HD inline T pm(T a, T b) { return a * b; }
#if defined(__CUDA_ARCH__)
template <> __device__ inline float pm<float>(float a, float b) { return __fmul_rn(a, b); }
#elif defined(__FMA__)
template <> inline float pm<float>(float a, float b) { float r = a * b; asm volatile("" : "+x"(r)); return r; }
#endif

enum { P_DT = 0, P_DR = 1, P_DV = 10, P_DP = 13, P_JRG = 16, P_JVG = 25, P_JVA = 34, P_JPG = 43, P_JPA = 52, P_B = 61, P_C = 67, P_SIZE = 292 };

template <class T> IMU_HD inline void m3mul(const T* A, const T* B, T* C) {
    T r[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) r[i * 3 + j] = pm(A[i * 3], B[j]) + pm(A[i * 3 + 1], B[3 + j]) + pm(A[i * 3 + 2], B[6 + j]);
#pragma unroll
    for (int i = 0; i < 9; ++i) C[i] = r[i];
}
template <class T> IMU_HD inline void m3T(const T* A, T* B) {
    T r[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) r[i * 3 + j] = A[j * 3 + i];
#pragma unroll
    for (int i = 0; i < 9; ++i) B[i] = r[i];
}
template <class T> IMU_HD inline void m3vec(const T* A, const T* v, T* o) {
    T r[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) r[i] = pm(A[i * 3], v[0]) + pm(A[i * 3 + 1], v[1]) + pm(A[i * 3 + 2], v[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) o[i] = r[i];
}
template <class T> IMU_HD inline void hat(const T* w, T* W) {
    W[0] = 0; W[1] = -w[2]; W[2] = w[1]; W[3] = w[2]; W[4] = 0; W[5] = -w[0]; W[6] = -w[1]; W[7] = w[0]; W[8] = 0;
}
// NormalizeRotation (src/ImuTypes.cc:34-37, Eigen::JacobiSVD): U V^T by one-sided Jacobi
template <class T> IMU_HD inline void normalize_rotation(const T* R, T* out) {
    T A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
#pragma unroll
    for (int i = 0; i < 9; ++i) A[i] = R[i];
    const T tol = sizeof(T) == 4 ? (T)1e-7 : (T)1e-15;
    for (int sweep = 0; sweep < 30; ++sweep) {
        T off = 0;
#pragma unroll
        for (int p = 0; p < 2; ++p)
#pragma unroll
            for (int q = p + 1; q < 3; ++q) {
                T alpha = 0, beta = 0, gamma = 0;
#pragma unroll
                for (int i = 0; i < 3; ++i) { alpha += pm(A[i * 3 + p], A[i * 3 + p]); beta += pm(A[i * 3 + q], A[i * 3 + q]); gamma += pm(A[i * 3 + p], A[i * 3 + q]); }
                const T ab = alpha * beta, tiny = sizeof(T) == 4 ? (T)1e-30 : (T)1e-300;
                off = fmax(off, (T)fabs(gamma) / (T)sqrt(ab > tiny ? ab : tiny));
                if (gamma != 0) {
                    const T zeta = (beta - alpha) / (2 * gamma);
                    const T t = (zeta >= 0 ? (T)1 : (T)-1) / ((T)fabs(zeta) + (T)sqrt(1 + pm(zeta, zeta)));
                    const T c = 1 / (T)sqrt(1 + pm(t, t)), s = c * t;
#pragma unroll
                    for (int i = 0; i < 3; ++i) {
                        const T ap = A[i * 3 + p], aq = A[i * 3 + q];
                        A[i * 3 + p] = pm(c, ap) - pm(s, aq); A[i * 3 + q] = pm(s, ap) + pm(c, aq);
                        const T vp = V[i * 3 + p], vq = V[i * 3 + q];
                        V[i * 3 + p] = pm(c, vp) - pm(s, vq); V[i * 3 + q] = pm(s, vp) + pm(c, vq);
                    }
                }
            }
        if (off < tol) break;
    }
    T U[9];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        T n = 0;
#pragma unroll
        for (int i = 0; i < 3; ++i) n += pm(A[i * 3 + j], A[i * 3 + j]);
        n = (T)sqrt(n);
#pragma unroll
        for (int i = 0; i < 3; ++i) U[i * 3 + j] = n > 0 ? A[i * 3 + j] / n : (T)(i == j);
    }
    T Vt[9];
    m3T(V, Vt);
    m3mul(U, Vt, out);
}

// ---- information matrices: inverse of the covariance blocks (Gauss-Jordan with partial pivoting, like Eigen's PartialPivLU inverse),
//      symmetrised, eigenvalues below 1e-12 clamped to zero (cyclic Jacobi eigen-decomposition) ----
// On an exactly zero pivot (a singular matrix, e.g. the covariance of an interval with one IMU sample) the result is all NaN and false is
// returned: PartialPivLU's inverse divides by that pivot, so the reference's information matrix is not finite either.
template <int N> IMU_HD inline bool invert_n(const double* A, double* out) {
    double M[N * 2 * N];
    for (int i = 0; i < N; ++i) for (int j = 0; j < N; ++j) { M[i * 2 * N + j] = A[i * N + j]; M[i * 2 * N + N + j] = i == j ? 1.0 : 0.0; }
    for (int c = 0; c < N; ++c) {
        int piv = c;
        for (int r = c + 1; r < N; ++r) if (fabs(M[r * 2 * N + c]) > fabs(M[piv * 2 * N + c])) piv = r;
        if (M[piv * 2 * N + c] == 0) { for (int i = 0; i < N * N; ++i) out[i] = NAN; return false; }
        if (piv != c) for (int j = 0; j < 2 * N; ++j) { const double t = M[c * 2 * N + j]; M[c * 2 * N + j] = M[piv * 2 * N + j]; M[piv * 2 * N + j] = t; }
        const double inv = 1.0 / M[c * 2 * N + c];
        for (int j = 0; j < 2 * N; ++j) M[c * 2 * N + j] *= inv;
        for (int r = 0; r < N; ++r) {
            if (r == c) continue;
            const double f = M[r * 2 * N + c];
            if (f != 0) for (int j = 0; j < 2 * N; ++j) M[r * 2 * N + j] -= f * M[c * 2 * N + j];
        }
    }
    for (int i = 0; i < N; ++i) for (int j = 0; j < N; ++j) out[i * N + j] = M[i * 2 * N + N + j];
    return true;
}
IMU_HD inline void imu_information_dev(const float* __restrict__ P, double* __restrict__ I9, double* __restrict__ IG, double* __restrict__ IA) {
    double C9[81], A[81], V[81], w[9];
    for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) C9[i * 9 + j] = (double)P[P_C + i * 15 + j];
    invert_n<9>(C9, A);
    for (int i = 0; i < 9; ++i) for (int j = i; j < 9; ++j) { const double s = (A[i * 9 + j] + A[j * 9 + i]) / 2; A[i * 9 + j] = A[j * 9 + i] = s; }
    for (int i = 0; i < 81; ++i) V[i] = (i % 10 == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0;
        for (int p = 0; p < 9; ++p) for (int q = p + 1; q < 9; ++q) off += A[p * 9 + q] * A[p * 9 + q];
        if (off < 1e-300) break;
        for (int p = 0; p < 9; ++p)
            for (int q = p + 1; q < 9; ++q) {
                const double apq = A[p * 9 + q];
                if (apq == 0) continue;
                const double theta = (A[q * 9 + q] - A[p * 9 + p]) / (2 * apq);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1));
                const double c = 1 / sqrt(t * t + 1), s = t * c;
                for (int k = 0; k < 9; ++k) { const double akp = A[k * 9 + p], akq = A[k * 9 + q]; A[k * 9 + p] = c * akp - s * akq; A[k * 9 + q] = s * akp + c * akq; }
                for (int k = 0; k < 9; ++k) { const double apk = A[p * 9 + k], aqk = A[q * 9 + k]; A[p * 9 + k] = c * apk - s * aqk; A[q * 9 + k] = s * apk + c * aqk; }
                for (int k = 0; k < 9; ++k) { const double vkp = V[k * 9 + p], vkq = V[k * 9 + q]; V[k * 9 + p] = c * vkp - s * vkq; V[k * 9 + q] = s * vkp + c * vkq; }
            }
    }
    for (int i = 0; i < 9; ++i) { w[i] = A[i * 9 + i]; if (w[i] < 1e-12) w[i] = 0; }
    for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) { double s = 0; for (int k = 0; k < 9; ++k) s += V[i * 9 + k] * w[k] * V[j * 9 + k]; I9[i * 9 + j] = s; }
    double G[9], Aa[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { G[i * 3 + j] = (double)P[P_C + (9 + i) * 15 + 9 + j]; Aa[i * 3 + j] = (double)P[P_C + (12 + i) * 15 + 12 + j]; }
    invert_n<3>(G, IG);
    invert_n<3>(Aa, IA);
}
// ---- SO3 helpers in double (src/G2oTypes.cc:777-861) ----
IMU_HD inline void log_so3(const double* R, double* w) {
    const double tr = R[0] + R[4] + R[8];
    w[0] = (R[7] - R[5]) / 2; w[1] = (R[2] - R[6]) / 2; w[2] = (R[3] - R[1]) / 2;
    const double costheta = (tr - 1.0) * 0.5f;
    if (costheta > 1 || costheta < -1) return;
    const double theta = acos(costheta);
    const double s = sin(theta);
    if (fabs(s) < 1e-5) return;
    for (int i = 0; i < 3; ++i) w[i] = theta * w[i] / s;
}
IMU_HD inline void right_jacobian(const double* v, double* J) {
    const double d2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2], d = sqrt(d2);
    double W[9], W2[9];
    hat(v, W); m3mul(W, W, W2);
    for (int i = 0; i < 9; ++i) {
        const double I = (i % 4 == 0) ? 1 : 0;
        J[i] = d < 1e-5 ? I : I - W[i] * (1.0 - cos(d)) / d2 + W2[i] * (d - sin(d)) / (d2 * d);
    }
}
IMU_HD inline void inv_right_jacobian(const double* v, double* J) {
    const double d2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2], d = sqrt(d2);
    double W[9], W2[9];
    hat(v, W); m3mul(W, W, W2);
    for (int i = 0; i < 9; ++i) {
        const double I = (i % 4 == 0) ? 1 : 0;
        J[i] = d < 1e-5 ? I : I + W[i] / 2 + W2[i] * (1.0 / d2 - (1.0 + cos(d)) / (2.0 * d * sin(d)));
    }
}

// IMU::Preintegrated::GetDeltaRotation / Velocity / Position(b) (src/ImuTypes.cc:283-307) in float, like the reference: dbgf / dbaf are
// b - the preintegration's own bias (gyro, acc).  Tracking::PredictStateIMU's deltas (track_inertial.cu).  edge_inertial_dev below
// evaluates the same expressions inline: routing it through this function changed the register allocation and scheduling of
// pose_inertial_opt_kernel, whose compiled code stays as it is.
IMU_HD inline void preint_delta_f(const float* __restrict__ P, const float* dbgf, const float* dbaf, float* Rn, float* dVf, float* dPf) {
    float w[3], W[9], W2[9], E[9], M[9];
    m3vec(P + P_JRG, dbgf, w);
    const float d2 = pm(w[0], w[0]) + pm(w[1], w[1]) + pm(w[2], w[2]), d = sqrtf(d2);
    hat(w, W); m3mul(W, W, W2);
    for (int i = 0; i < 9; ++i) {
        const float I = (i % 4 == 0) ? 1.f : 0.f;
        E[i] = d < 1e-5f ? I + W[i] + pm(0.5f, W2[i]) : I + pm(W[i], sinf(d)) / d + pm(W2[i], 1.0f - cosf(d)) / d2;
    }
    m3mul(P + P_DR, E, M);
    normalize_rotation(M, Rn);
    float g1[3], a1[3], g2[3], a2[3];
    m3vec(P + P_JVG, dbgf, g1); m3vec(P + P_JVA, dbaf, a1); m3vec(P + P_JPG, dbgf, g2); m3vec(P + P_JPA, dbaf, a2);
    for (int i = 0; i < 3; ++i) { dVf[i] = P[P_DV + i] + g1[i] + a1[i]; dPf[i] = P[P_DP + i] + g2[i] + a2[i]; }
}

// ---- EdgeInertial: residual, Jacobians, chi2 and robust weight; thread per edge.  states [count][36] doubles:
//      Rwb1 9 | twb1 3 | v1 3 | bg 3 | ba 3 | Rwb2 9 | twb2 3 | v2 3 ----
// EdgeInertial::computeError + linearizeOplus for one edge: S = Rwb1 9 | twb1 3 | v1 3 | bg 3 | ba 3 | Rwb2 9 | twb2 3 | v2 3; err [9]; J [9][24] or null
IMU_HD inline void edge_inertial_dev(const float* __restrict__ P, const double* S, double* err, double* J) {
    const double *Rwb1 = S, *twb1 = S + 9, *v1 = S + 12, *bg = S + 15, *ba = S + 18, *Rwb2 = S + 21, *twb2 = S + 30, *v2 = S + 33;
    // GetDeltaRotation / Velocity / Position(b1): float, like IMU::Preintegrated (src/ImuTypes.cc:283-307)
    const float b1[6] = {(float)ba[0], (float)ba[1], (float)ba[2], (float)bg[0], (float)bg[1], (float)bg[2]};
    const float dbgf[3] = {b1[3] - P[P_B + 3], b1[4] - P[P_B + 4], b1[5] - P[P_B + 5]};
    const float dbaf[3] = {b1[0] - P[P_B], b1[1] - P[P_B + 1], b1[2] - P[P_B + 2]};
    double dR[9], dV[3], dP[3];
    {
        float w[3], W[9], W2[9], E[9], M[9], Rn[9];
        m3vec(P + P_JRG, dbgf, w);
        const float d2 = pm(w[0], w[0]) + pm(w[1], w[1]) + pm(w[2], w[2]), d = sqrtf(d2);
        hat(w, W); m3mul(W, W, W2);
        for (int i = 0; i < 9; ++i) {
            const float I = (i % 4 == 0) ? 1.f : 0.f;
            E[i] = d < 1e-5f ? I + W[i] + pm(0.5f, W2[i]) : I + pm(W[i], sinf(d)) / d + pm(W2[i], 1.0f - cosf(d)) / d2;
        }
        m3mul(P + P_DR, E, M);
        normalize_rotation(M, Rn);
        float g1[3], a1[3], g2[3], a2[3];
        m3vec(P + P_JVG, dbgf, g1); m3vec(P + P_JVA, dbaf, a1); m3vec(P + P_JPG, dbgf, g2); m3vec(P + P_JPA, dbaf, a2);
        for (int i = 0; i < 9; ++i) dR[i] = (double)Rn[i];
        for (int i = 0; i < 3; ++i) { dV[i] = (double)(P[P_DV + i] + g1[i] + a1[i]); dP[i] = (double)(P[P_DP + i] + g2[i] + a2[i]); }
    }
    const double dt = (double)P[P_DT];
    const double g[3] = {0, 0, -(double)9.81f};
    double Rbw1[9], dRt[9], T[9], eR[9], er[3];
    m3T(Rwb1, Rbw1); m3T(dR, dRt);
    m3mul(dRt, Rbw1, T); m3mul(T, Rwb2, eR);
    log_so3(eR, er);
    double dv[3], dp[3], rv[3], rp[3];
    for (int i = 0; i < 3; ++i) { dv[i] = v2[i] - v1[i] - g[i] * dt; dp[i] = twb2[i] - twb1[i] - v1[i] * dt - g[i] * dt * dt / 2; }
    m3vec(Rbw1, dv, rv); m3vec(Rbw1, dp, rp);
    for (int i = 0; i < 3; ++i) { err[i] = er[i]; err[3 + i] = rv[i] - dV[i]; err[6 + i] = rp[i] - dP[i]; }
    if (!J) return;
    for (int i = 0; i < 216; ++i) J[i] = 0;
    double invJr[9], A[9], H[9], Rwb2t[9];
    inv_right_jacobian(er, invJr);
    auto put = [&](int r0, int c0, const double* M, double s) { for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) J[(r0 + i) * 24 + c0 + j] = s * M[i * 3 + j]; };
    m3T(Rwb2, Rwb2t);
    m3mul(Rwb2t, Rwb1, A); m3mul(invJr, A, A);
    put(0, 0, A, -1.0);
    hat(rv, H); put(3, 0, H, 1.0);
    hat(rp, H); put(6, 0, H, 1.0);
    const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    put(6, 3, I3, -1.0);
    put(3, 6, Rbw1, -1.0); put(6, 6, Rbw1, -dt);
    double JRg[9], M9[9], w[3], Jr[9], eRt[9];
    const double dbg[3] = {(double)dbgf[0], (double)dbgf[1], (double)dbgf[2]};
    for (int i = 0; i < 9; ++i) JRg[i] = (double)P[P_JRG + i];
    m3vec(JRg, dbg, w);
    right_jacobian(w, Jr);
    m3T(eR, eRt);
    m3mul(invJr, eRt, A); m3mul(A, Jr, A); m3mul(A, JRg, A);
    put(0, 9, A, -1.0);
    for (int i = 0; i < 9; ++i) M9[i] = (double)P[P_JVG + i];
    put(3, 9, M9, -1.0);
    for (int i = 0; i < 9; ++i) M9[i] = (double)P[P_JPG + i];
    put(6, 9, M9, -1.0);
    for (int i = 0; i < 9; ++i) M9[i] = (double)P[P_JVA + i];
    put(3, 12, M9, -1.0);
    for (int i = 0; i < 9; ++i) M9[i] = (double)P[P_JPA + i];
    put(6, 12, M9, -1.0);
    put(0, 15, invJr, 1.0);
    m3mul(Rbw1, Rwb2, A); put(6, 18, A, 1.0);
    put(3, 21, Rbw1, 1.0);
}
// ---- EdgeMono / EdgeMonoOnlyPose with ImuCamPose (src/G2oTypes.cc:349-395), at the camera pose Rcw, tcw that ImuCamPose caches ----
// computeError: the camera point Xc = Rcw X + tcw and the residual obs - Pinhole::project(Xc) (cam = fx fy cx cy); returns isDepthPositive
IMU_HD inline bool mono_residual(const double* Rcw, const double* tcw, const double* X, const float* cam, double obs0, double obs1, double* Xc,
                                 double& e0, double& e1) {
    m3vec(Rcw, X, Xc);
    for (int i = 0; i < 3; ++i) Xc[i] += tcw[i];
    const double fx = cam[0], fy = cam[1], cx = cam[2], cy = cam[3];
    e0 = obs0 - (fx * Xc[0] / Xc[2] + cx);
    e1 = obs1 - (fy * Xc[1] / Xc[2] + cy);
    return (Rcw[6] * X[0] + Rcw[7] * X[1] + Rcw[8] * X[2] + tcw[2]) > 0.0;
}
// linearizeOplus at the camera point Xc: Jpoint (2 x 3; null for EdgeMonoOnlyPose) = -proj_jac Rcw, Jpose (2 x 6) = proj_jac Rcb [[Xb]x | I]
// with Xb = Rbc Xc + tbc the point in the body frame
IMU_HD inline void mono_jacobians(const double* Rcw, const double* Rcb, const double* Rbc, const double* tbc, const float* cam, const double* Xc,
                                  double* Jpoint, double* Jpose) {
    const double fx = cam[0], fy = cam[1];
    const double pj[6] = {fx / Xc[2], 0, -fx * Xc[0] / (Xc[2] * Xc[2]), 0, fy / Xc[2], -fy * Xc[1] / (Xc[2] * Xc[2])};
    if (Jpoint)
        for (int i = 0; i < 2; ++i) for (int j = 0; j < 3; ++j) Jpoint[i * 3 + j] = -(pj[i * 3] * Rcw[j] + pj[i * 3 + 1] * Rcw[3 + j] + pj[i * 3 + 2] * Rcw[6 + j]);
    double Xb[3];
    m3vec(Rbc, Xc, Xb);
    for (int i = 0; i < 3; ++i) Xb[i] += tbc[i];
    const double x = Xb[0], y = Xb[1], z = Xb[2];
    const double Sd[18] = {0.0, z, -y, 1.0, 0.0, 0.0, -z, 0.0, x, 0.0, 1.0, 0.0, y, -x, 0.0, 0.0, 0.0, 1.0};
    double PR[6];
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 3; ++j) PR[i * 3 + j] = pj[i * 3] * Rcb[j] + pj[i * 3 + 1] * Rcb[3 + j] + pj[i * 3 + 2] * Rcb[6 + j];
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 6; ++j) Jpose[i * 6 + j] = PR[i * 3] * Sd[j] + PR[i * 3 + 1] * Sd[6 + j] + PR[i * 3 + 2] * Sd[12 + j];
}
IMU_HD inline void exp_so3_d(const double* w, double* R) {      // ExpSO3(double) with its NormalizeRotation (src/G2oTypes.cc:782-798)
    const double d2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], d = sqrt(d2);
    double W[9], W2[9], res[9];
    hat(w, W); m3mul(W, W, W2);
    for (int i = 0; i < 9; ++i) {
        const double I = (i % 4 == 0) ? 1.0 : 0.0;
        res[i] = d < 1e-5 ? I + W[i] + 0.5 * W2[i] : I + W[i] * sin(d) / d + W2[i] * (1.0 - cos(d)) / d2;
    }
    normalize_rotation(res, R);
}

}  // namespace imu

// ---- the g2o pieces of every optimiser kernel: lba.cu and pose_opt.cu use the SE3Quat part, all five kernels the Huber kernel, and
//      lba.cu, pose_opt.cu and liba_core.cuh the Levenberg-Marquardt policy ----
namespace g2o {

// ---- SE3Quat (g2o/types/se3quat.h), quaternion q = (w, x, y, z), pose T = q 4 | t 3 ----
IMU_HD inline void qrot(const double* q, const double* v, double* o) {   // Eigen::Quaternion * Vector3
    double ux = q[2] * v[2] - q[3] * v[1], uy = q[3] * v[0] - q[1] * v[2], uz = q[1] * v[1] - q[2] * v[0];
    ux += ux; uy += uy; uz += uz;
    o[0] = v[0] + q[0] * ux + (q[2] * uz - q[3] * uy);
    o[1] = v[1] + q[0] * uy + (q[3] * ux - q[1] * uz);
    o[2] = v[2] + q[0] * uz + (q[1] * uy - q[2] * ux);
}
IMU_HD inline void qnormalize(double* q) {
    if (q[0] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
IMU_HD inline void qtoR(const double* q, double* R) {
    const double tx = 2 * q[1], ty = 2 * q[2], tz = 2 * q[3];
    const double twx = tx * q[0], twy = ty * q[0], twz = tz * q[0], txx = tx * q[1], txy = ty * q[1], txz = tz * q[1];
    const double tyy = ty * q[2], tyz = tz * q[2], tzz = tz * q[3];
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
IMU_HD inline void qfromR(const double* m, double* q) {
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
// VertexSE3Expmap::oplusImpl: T <- SE3Quat::exp(upd) * T   (g2o/types/se3quat.h:223-256, :101-110)
IMU_HD inline void pose_oplus(double* T, const double* upd) {
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

// RobustKernelHuber::robustify (robust_kernel_impl.cpp:78-91) with dsqr = delta * delta: rho0 = rho(e2), rho1 = rho'(e2).  A NaN e2 takes
// the second branch, as in g2o.  dsqr is an argument so that a caller can keep it out of its per-edge loop.
IMU_HD inline void huber(double e2, double delta, double dsqr, double& rho0, double& rho1) {
    if (e2 <= dsqr) { rho0 = e2; rho1 = 1.0; }
    else { const double s = sqrt(e2); rho0 = 2 * s * delta - dsqr; rho1 = delta / s; }
}

// OptimizationAlgorithmLevenberg::solve's damping (optimization_algorithm_levenberg.cpp:61-194) and the stop rule ORB-SLAM3 adds to it
// (nBad: three iterations in a row that lower chi2 by less than a 1e-3 fraction).  Only the scalar policy: the caller builds and solves the
// system, applies and undoes the step, and evaluates chi2.
struct Levenberg {
    static constexpr int maxTrials = 10;
    double lambda = -1, ni = 2;
    int nBad = 0;
    // first iteration: the user's lambda when it is set, else computeLambdaInit = tau * the largest diagonal entry of H
    IMU_HD void start(double userLambda, double maxDiag) {
        lambda = userLambda > 0 ? userLambda : 1e-5 * maxDiag;
        ni = 2; nBad = 0;
    }
    // one trial: rho = (currentChi - tempChi) / (x^T (lambda x + b) + 1e-3), a failed solve counting as tempChi = DBL_MAX.  On a good step
    // lambda shrinks and currentChi takes tempChi (returns true); otherwise lambda grows and the caller undoes the step.
    IMU_HD bool trial(double& currentChi, double tempChi, double xLxb, bool solved, double& rho) {
        if (!solved) tempChi = DBL_MAX;
        rho = currentChi - tempChi;
        const double scale = xLxb + 1e-3;
        rho /= scale;
        if (rho > 0 && tempChi <= DBL_MAX && tempChi >= -DBL_MAX) {      // tempChi finite (NaN and +-inf fail)
            double alpha = 1. - pow((2 * rho - 1), 3.0);
            alpha = fmin(alpha, 2. / 3.);
            lambda *= fmax(1. / 3., alpha);
            ni = 2;
            currentChi = tempChi;
            return true;
        }
        lambda *= ni;
        ni *= 2;
        return false;
    }
    // end of an iteration of qmax trials: false when the optimisation stops
    IMU_HD bool iteration_done(int qmax, double rho, double iniChi, double currentChi) {
        if (qmax == maxTrials || rho == 0) return false;
        if ((iniChi - currentChi) * 1e3 < iniChi) ++nBad; else nBad = 0;
        return nBad < 3;
    }
};

}  // namespace g2o
