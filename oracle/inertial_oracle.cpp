// TEST INFRASTRUCTURE ONLY (see oracle_common.h).  CPU restatement of the inertial part of the path (SURVEY.md 8f rank 1):
//   IMU::Preintegrated::IntegrateNewMeasurement / IntegratedRotation        reference src/ImuTypes.cc:177-240, :84-107   (float, as the reference)
//   IMU::Preintegrated::GetDeltaRotation / GetDeltaVelocity / GetDeltaPosition / GetDeltaBias     :276-307
//   IMU::NormalizeRotation (Eigen::JacobiSVD U V^T)                                               :34-37
//   EdgeInertial ctor (information = inverse of the 9x9 covariance, symmetrised, eigenvalues < 1e-12 clamped)  src/G2oTypes.cc:492-509
//   EdgeInertial::computeError / linearizeOplus                                                   :514-594
//   EdgeMono::computeError (include/G2oTypes.h:353-358), linearizeOplus (src/G2oTypes.cc:349-373), ImuCamPose::Project :170-175
//   EdgeGyroRW / EdgeAccRW (include/G2oTypes.h:635-700): error = b2 - b1, information = inverse of the 3x3 walk covariance
//   ExpSO3 / LogSO3 / RightJacobianSO3 / InverseRightJacobianSO3                                  :777-861
//   ImuCamPose::Update (VertexPose::oplusImpl)                                                    :192-220
// PARITY: the double-precision edge functions below equal the reference's own function bodies compiled against a small Eigen stand-in
// (oracle/ref_shim/ref_wrap_inertial.cpp -> oracle/_ref/libref_inertial.so, tests/test_ref_pins_inertial_cpu.py) to 1e-12; ImuTypes.cc needs Sophus::SO3f::exp
// and Eigen::JacobiSVD and is not compiled.  Independently of that, the analytic Jacobians
// below are pinned by numerical differentiation of the residuals under the reference's own update rules
// (tests/test_inertial_cpu.py), the SVD / eigen pieces by their defining properties.  The solver loops around these edges are "parity unpinned" by the reference itself.
#include "oracle_common.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace orbo {
namespace imu {

template <class T> static void mat3_mul(const T* A, const T* B, T* C) {
    T r[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
    for (int i = 0; i < 9; ++i) C[i] = r[i];
}
template <class T> static void mat3_T(const T* A, T* B) { T r[9]; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r[i * 3 + j] = A[j * 3 + i]; for (int i = 0; i < 9; ++i) B[i] = r[i]; }
template <class T> static void mat3_vec(const T* A, const T* v, T* o) { T r[3]; for (int i = 0; i < 3; ++i) r[i] = A[i * 3] * v[0] + A[i * 3 + 1] * v[1] + A[i * 3 + 2] * v[2]; for (int i = 0; i < 3; ++i) o[i] = r[i]; }
template <class T> static void hat(const T* w, T* W) { W[0] = 0; W[1] = -w[2]; W[2] = w[1]; W[3] = w[2]; W[4] = 0; W[5] = -w[0]; W[6] = -w[1]; W[7] = w[0]; W[8] = 0; }

// One-sided Jacobi SVD of a 3x3 matrix (what Eigen::JacobiSVD computes, up to rounding): returns U V^T = the nearest rotation.
template <class T> static void normalize_rotation(const T* R, T* out) {
    T A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int i = 0; i < 9; ++i) A[i] = R[i];
    for (int sweep = 0; sweep < 30; ++sweep) {
        T off = 0;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                T alpha = 0, beta = 0, gamma = 0;       // column p, q of A
                for (int i = 0; i < 3; ++i) { alpha += A[i * 3 + p] * A[i * 3 + p]; beta += A[i * 3 + q] * A[i * 3 + q]; gamma += A[i * 3 + p] * A[i * 3 + q]; }
                off = std::max(off, (T)std::fabs(gamma) / (T)std::sqrt(std::max(alpha * beta, sizeof(T) == 4 ? (T)1e-30 : (T)1e-300)));
                if (gamma == 0) continue;
                const T zeta = (beta - alpha) / (2 * gamma);
                const T t = (zeta >= 0 ? (T)1 : (T)-1) / ((T)std::fabs(zeta) + (T)std::sqrt(1 + zeta * zeta));
                const T c = 1 / (T)std::sqrt(1 + t * t), s = c * t;
                for (int i = 0; i < 3; ++i) {
                    const T ap = A[i * 3 + p], aq = A[i * 3 + q];
                    A[i * 3 + p] = c * ap - s * aq; A[i * 3 + q] = s * ap + c * aq;
                    const T vp = V[i * 3 + p], vq = V[i * 3 + q];
                    V[i * 3 + p] = c * vp - s * vq; V[i * 3 + q] = s * vp + c * vq;
                }
            }
        if (off < (sizeof(T) == 4 ? (T)1e-7 : (T)1e-15)) break;
    }
    T U[9];   // columns of A are sigma_j u_j
    for (int j = 0; j < 3; ++j) {
        T n = 0;
        for (int i = 0; i < 3; ++i) n += A[i * 3 + j] * A[i * 3 + j];
        n = (T)std::sqrt(n);
        for (int i = 0; i < 3; ++i) U[i * 3 + j] = n > 0 ? A[i * 3 + j] / n : (i == j ? 1 : 0);
    }
    T Vt[9];
    mat3_T(V, Vt);
    mat3_mul(U, Vt, out);
}

// src/G2oTypes.cc:782-798 (double) / Sophus::SO3f::exp(...).matrix() (float: Rodrigues through the quaternion; same rotation to rounding)
template <class T> static void exp_so3(const T* w, T* R, bool normalise) {
    const T x = w[0], y = w[1], z = w[2];
    const T d2 = x * x + y * y + z * z, d = (T)std::sqrt(d2);
    T W[9], W2[9];
    hat(w, W);
    mat3_mul(W, W, W2);
    T res[9];
    for (int i = 0; i < 9; ++i) {
        const T I = (i % 4 == 0) ? 1 : 0;
        res[i] = d < (T)1e-5 ? I + W[i] + (T)0.5 * W2[i] : I + W[i] * (T)std::sin(d) / d + W2[i] * ((T)1.0 - (T)std::cos(d)) / d2;
    }
    if (normalise) normalize_rotation(res, R);
    else for (int i = 0; i < 9; ++i) R[i] = res[i];
}
static void log_so3(const double* R, double* w) {   // :800-814
    const double tr = R[0] + R[4] + R[8];
    w[0] = (R[7] - R[5]) / 2; w[1] = (R[2] - R[6]) / 2; w[2] = (R[3] - R[1]) / 2;
    const double costheta = (tr - 1.0) * 0.5f;
    if (costheta > 1 || costheta < -1) return;
    const double theta = std::acos(costheta);
    const double s = std::sin(theta);
    if (std::fabs(s) < 1e-5) return;
    for (int i = 0; i < 3; ++i) w[i] = theta * w[i] / s;
}
template <class T> static void right_jacobian(const T* v, T* J, T eps) {   // G2oTypes.cc:839-854 / ImuTypes.cc:39-55
    const T d2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2], d = (T)std::sqrt(d2);
    T W[9], W2[9];
    hat(v, W); mat3_mul(W, W, W2);
    for (int i = 0; i < 9; ++i) {
        const T I = (i % 4 == 0) ? 1 : 0;
        J[i] = d < eps ? I : I - W[i] * ((T)1.0 - (T)std::cos(d)) / d2 + W2[i] * (d - (T)std::sin(d)) / (d2 * d);
    }
}
static void inv_right_jacobian(const double* v, double* J) {   // G2oTypes.cc:821-832
    const double d2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2], d = std::sqrt(d2);
    double W[9], W2[9];
    hat(v, W); mat3_mul(W, W, W2);
    for (int i = 0; i < 9; ++i) {
        const double I = (i % 4 == 0) ? 1 : 0;
        J[i] = d < 1e-5 ? I : I + W[i] / 2 + W2[i] * (1.0 / d2 - (1.0 + std::cos(d)) / (2.0 * d * std::sin(d)));
    }
}

}  // namespace imu
}  // namespace orbo

using namespace orbo::imu;

extern "C" {

// Layout of one IMU::Preintegrated as 292 floats (include/orb_b200.h: ImuPreintegrated):
//   [0] dT | [1..9] dR | [10..12] dV | [13..15] dP | [16..24] JRg | [25..33] JVg | [34..42] JVa | [43..51] JPg | [52..60] JPa |
//   [61..66] b = (bax, bay, baz, bwx, bwy, bwz) | [67..291] C (15 x 15, row-major)
enum { P_DT = 0, P_DR = 1, P_DV = 10, P_DP = 13, P_JRG = 16, P_JVG = 25, P_JVA = 34, P_JPG = 43, P_JPA = 52, P_B = 61, P_C = 67, P_SIZE = 292 };

// Preintegrated::Initialize(b) + IntegrateNewMeasurement for n measurements (acc, gyro, dt); noise4 = (ng, na, ngw, naw) of IMU::Calib::Set.
void orbo_imu_preintegrate(int n, const float* acc, const float* gyr, const float* dts, const float* bias6, const float* noise4, float* P) {
    std::memset(P, 0, sizeof(float) * P_SIZE);
    float* dR = P + P_DR; float* dV = P + P_DV; float* dP = P + P_DP;
    float *JRg = P + P_JRG, *JVg = P + P_JVG, *JVa = P + P_JVA, *JPg = P + P_JPG, *JPa = P + P_JPA, *C = P + P_C;
    dR[0] = dR[4] = dR[8] = 1.f;
    for (int i = 0; i < 6; ++i) P[P_B + i] = bias6[i];
    const float ng2 = noise4[0] * noise4[0], na2 = noise4[1] * noise4[1], ngw2 = noise4[2] * noise4[2], naw2 = noise4[3] * noise4[3];
    const float Nga[6] = {ng2, ng2, ng2, na2, na2, na2}, Walk[6] = {ngw2, ngw2, ngw2, naw2, naw2, naw2};
    float dT = 0.f;
    for (int m = 0; m < n; ++m) {
        const float dt = dts[m];
        float A[81], B[54];
        for (int i = 0; i < 81; ++i) A[i] = (i % 10 == 0) ? 1.f : 0.f;
        for (int i = 0; i < 54; ++i) B[i] = 0.f;
        const float a[3] = {acc[3 * m] - bias6[0], acc[3 * m + 1] - bias6[1], acc[3 * m + 2] - bias6[2]};
        float Ra[3];
        mat3_vec(dR, a, Ra);
        for (int i = 0; i < 3; ++i) { dP[i] = dP[i] + dV[i] * dt + 0.5f * Ra[i] * dt * dt; }
        for (int i = 0; i < 3; ++i) dV[i] = dV[i] + Ra[i] * dt;
        float Wacc[9], RW[9];
        hat(a, Wacc);
        mat3_mul(dR, Wacc, RW);
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
            A[(3 + i) * 9 + j] = -RW[i * 3 + j] * dt;                 // A.block<3,3>(3,0) = -dR*dt*Wacc
            A[(6 + i) * 9 + j] = -0.5f * RW[i * 3 + j] * dt * dt;     // A.block<3,3>(6,0)
            A[(6 + i) * 9 + 3 + j] = i == j ? dt : 0.f;               // A.block<3,3>(6,3)
            B[(3 + i) * 6 + 3 + j] = dR[i * 3 + j] * dt;              // B.block<3,3>(3,3)
            B[(6 + i) * 6 + 3 + j] = 0.5f * dR[i * 3 + j] * dt * dt;  // B.block<3,3>(6,3)
        }
        float RWJ[9];
        mat3_mul(RW, JRg, RWJ);
        for (int i = 0; i < 9; ++i) {
            JPa[i] = JPa[i] + JVa[i] * dt - 0.5f * dR[i] * dt * dt;
            JPg[i] = JPg[i] + JVg[i] * dt - 0.5f * RWJ[i] * dt * dt;
            JVa[i] = JVa[i] - dR[i] * dt;
            JVg[i] = JVg[i] - RWJ[i] * dt;
        }
        // IntegratedRotation (ImuTypes.cc:84-107)
        const float w[3] = {(gyr[3 * m] - bias6[3]) * dt, (gyr[3 * m + 1] - bias6[4]) * dt, (gyr[3 * m + 2] - bias6[5]) * dt};
        const float d2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], d = std::sqrt(d2);
        float W[9], W2[9], deltaR[9], rightJ[9];
        hat(w, W); mat3_mul(W, W, W2);
        for (int i = 0; i < 9; ++i) {
            const float I = (i % 4 == 0) ? 1.f : 0.f;
            if (d < 1e-4f) { deltaR[i] = I + W[i]; rightJ[i] = I; }
            else { deltaR[i] = I + W[i] * std::sin(d) / d + W2[i] * (1.0f - std::cos(d)) / d2; rightJ[i] = I - W[i] * (1.0f - std::cos(d)) / d2 + W2[i] * (d - std::sin(d)) / (d2 * d); }
        }
        float Rn[9];
        mat3_mul(dR, deltaR, Rn);
        normalize_rotation(Rn, dR);
        float dRt[9];
        mat3_T(deltaR, dRt);
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { A[i * 9 + j] = dRt[i * 3 + j]; B[i * 6 + j] = rightJ[i * 3 + j] * dt; }
        // C.block<9,9>(0,0) = A C A^T + B Nga B^T ; C.block<6,6>(9,9) += NgaWalk
        float C9[81], AC[81], N9[81];
        for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) C9[i * 9 + j] = C[i * 15 + j];
        for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) { float s = 0; for (int k = 0; k < 9; ++k) s += A[i * 9 + k] * C9[k * 9 + j]; AC[i * 9 + j] = s; }
        for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) {
            float s = 0; for (int k = 0; k < 9; ++k) s += AC[i * 9 + k] * A[j * 9 + k];
            float t = 0; for (int k = 0; k < 6; ++k) t += B[i * 6 + k] * Nga[k] * B[j * 6 + k];
            N9[i * 9 + j] = s + t;
        }
        for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) C[i * 15 + j] = N9[i * 9 + j];
        for (int k = 0; k < 6; ++k) C[(9 + k) * 15 + 9 + k] += Walk[k];
        float T1[9];
        mat3_mul(dRt, JRg, T1);
        for (int i = 0; i < 9; ++i) JRg[i] = T1[i] - rightJ[i] * dt;
        dT += dt;
    }
    P[P_DT] = dT;
}

// GetDeltaRotation / Velocity / Position (b1), float like the reference, returned as the doubles EdgeInertial casts them to.
void orbo_imu_delta(const float* P, const double* bg, const double* ba, double* dR9, double* dV3, double* dP3) {
    // const IMU::Bias b1(VA1[0..2], VG1[0..2]): double -> float
    const float b1[6] = {(float)ba[0], (float)ba[1], (float)ba[2], (float)bg[0], (float)bg[1], (float)bg[2]};
    const float dbg[3] = {b1[3] - P[P_B + 3], b1[4] - P[P_B + 4], b1[5] - P[P_B + 5]};
    const float dba[3] = {b1[0] - P[P_B], b1[1] - P[P_B + 1], b1[2] - P[P_B + 2]};
    float w[3], E[9], M[9], Rn[9];
    mat3_vec(P + P_JRG, dbg, w);
    exp_so3(w, E, false);
    mat3_mul(P + P_DR, E, M);
    normalize_rotation(M, Rn);
    float g1[3], a1[3], g2[3], a2[3];
    mat3_vec(P + P_JVG, dbg, g1); mat3_vec(P + P_JVA, dba, a1); mat3_vec(P + P_JPG, dbg, g2); mat3_vec(P + P_JPA, dba, a2);
    for (int i = 0; i < 9; ++i) dR9[i] = (double)Rn[i];
    for (int i = 0; i < 3; ++i) { dV3[i] = (double)(P[P_DV + i] + g1[i] + a1[i]); dP3[i] = (double)(P[P_DP + i] + g2[i] + a2[i]); }
}

// symmetric eigen-decomposition by cyclic Jacobi (n <= 9): A = V diag(w) V^T
static void jacobi_eig(int n, double* A, double* V, double* w) {
    for (int i = 0; i < n * n; ++i) V[i] = (i % (n + 1) == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0;
        for (int p = 0; p < n; ++p) for (int q = p + 1; q < n; ++q) off += A[p * n + q] * A[p * n + q];
        if (off < 1e-300) break;
        for (int p = 0; p < n; ++p)
            for (int q = p + 1; q < n; ++q) {
                const double apq = A[p * n + q];
                if (apq == 0) continue;
                const double theta = (A[q * n + q] - A[p * n + p]) / (2 * apq);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1));
                const double c = 1 / std::sqrt(t * t + 1), s = t * c;
                for (int k = 0; k < n; ++k) { const double akp = A[k * n + p], akq = A[k * n + q]; A[k * n + p] = c * akp - s * akq; A[k * n + q] = s * akp + c * akq; }
                for (int k = 0; k < n; ++k) { const double apk = A[p * n + k], aqk = A[q * n + k]; A[p * n + k] = c * apk - s * aqk; A[q * n + k] = s * apk + c * aqk; }
                for (int k = 0; k < n; ++k) { const double vkp = V[k * n + p], vkq = V[k * n + q]; V[k * n + p] = c * vkp - s * vkq; V[k * n + q] = s * vkp + c * vkq; }
            }
    }
    for (int i = 0; i < n; ++i) w[i] = A[i * n + i];
}
static bool invert(int n, const double* A, double* out) {   // Gauss-Jordan with partial pivoting (Eigen: PartialPivLU)
    double M[9 * 18];
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) { M[i * 2 * n + j] = A[i * n + j]; M[i * 2 * n + n + j] = i == j ? 1.0 : 0.0; }
    for (int c = 0; c < n; ++c) {
        int piv = c;
        for (int r = c + 1; r < n; ++r) if (std::fabs(M[r * 2 * n + c]) > std::fabs(M[piv * 2 * n + c])) piv = r;
        if (M[piv * 2 * n + c] == 0) { for (int i = 0; i < n * n; ++i) out[i] = NAN; return false; }   // PartialPivLU divides by the zero pivot: not finite
        if (piv != c) for (int j = 0; j < 2 * n; ++j) std::swap(M[c * 2 * n + j], M[piv * 2 * n + j]);
        const double inv = 1.0 / M[c * 2 * n + c];
        for (int j = 0; j < 2 * n; ++j) M[c * 2 * n + j] *= inv;
        for (int r = 0; r < n; ++r) {
            if (r == c) continue;
            const double f = M[r * 2 * n + c];
            if (f != 0) for (int j = 0; j < 2 * n; ++j) M[r * 2 * n + j] -= f * M[c * 2 * n + j];
        }
    }
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) out[i * n + j] = M[i * 2 * n + n + j];
    return true;
}
// EdgeInertial ctor (G2oTypes.cc:499-507): Info (9x9) ; EdgeGyroRW / EdgeAccRW information (Optimizer.cc:551,559): InfoG, InfoA (3x3)
void orbo_imu_information(const float* P, double* Info9, double* InfoG3, double* InfoA3) {
    double C9[81], Inv[81], V[81], w[9];
    for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) C9[i * 9 + j] = (double)P[P_C + i * 15 + j];
    invert(9, C9, Inv);
    for (int i = 0; i < 9; ++i) for (int j = i; j < 9; ++j) { const double s = (Inv[i * 9 + j] + Inv[j * 9 + i]) / 2; Inv[i * 9 + j] = Inv[j * 9 + i] = s; }
    double A[81];
    std::memcpy(A, Inv, sizeof(A));
    jacobi_eig(9, A, V, w);
    for (int i = 0; i < 9; ++i) if (w[i] < 1e-12) w[i] = 0;
    for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) { double s = 0; for (int k = 0; k < 9; ++k) s += V[i * 9 + k] * w[k] * V[j * 9 + k]; Info9[i * 9 + j] = s; }
    double G[9], Aa[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { G[i * 3 + j] = (double)P[P_C + (9 + i) * 15 + 9 + j]; Aa[i * 3 + j] = (double)P[P_C + (12 + i) * 15 + 12 + j]; }
    invert(3, G, InfoG3); invert(3, Aa, InfoA3);
}

// EdgeInertial::computeError + linearizeOplus for one edge.  State: Rwb1[9], twb1[3], v1[3], bg[3], ba[3], Rwb2[9], twb2[3], v2[3].
// err[9] = (er, ev, ep); J[9][24] columns: pose1 (rot 3, trans 3) | v1 | gyro bias | acc bias | pose2 (rot 3, trans 3) | v2.
void orbo_imu_edge_inertial(const float* P, const double* Rwb1, const double* twb1, const double* v1, const double* bg, const double* ba,
                            const double* Rwb2, const double* twb2, const double* v2, double* err, double* J) {
    double dR[9], dV[3], dP[3];
    orbo_imu_delta(P, bg, ba, dR, dV, dP);
    const double dt = (double)P[P_DT];
    const double g[3] = {0, 0, -(double)9.81f};                 // g << 0, 0, -IMU::GRAVITY_VALUE (const float 9.81)
    double Rbw1[9], dRt[9], T[9], eR[9], er[3];
    mat3_T(Rwb1, Rbw1); mat3_T(dR, dRt);
    mat3_mul(dRt, Rbw1, T); mat3_mul(T, Rwb2, eR);
    log_so3(eR, er);
    double dv[3], dp[3], rv[3], rp[3];
    for (int i = 0; i < 3; ++i) { dv[i] = v2[i] - v1[i] - g[i] * dt; dp[i] = twb2[i] - twb1[i] - v1[i] * dt - g[i] * dt * dt / 2; }
    mat3_vec(Rbw1, dv, rv); mat3_vec(Rbw1, dp, rp);
    for (int i = 0; i < 3; ++i) { err[i] = er[i]; err[3 + i] = rv[i] - dV[i]; err[6 + i] = rp[i] - dP[i]; }
    if (!J) return;
    for (int i = 0; i < 9 * 24; ++i) J[i] = 0;
    double invJr[9];
    inv_right_jacobian(er, invJr);
    // dbg of GetDeltaBias(b1) (float), JRg etc. cast to double
    const float b1g[3] = {(float)bg[0], (float)bg[1], (float)bg[2]};
    const double dbg[3] = {(double)(b1g[0] - P[P_B + 3]), (double)(b1g[1] - P[P_B + 4]), (double)(b1g[2] - P[P_B + 5])};
    double JRg[9], JVg[9], JVa[9], JPg[9], JPa[9];
    for (int i = 0; i < 9; ++i) { JRg[i] = P[P_JRG + i]; JVg[i] = P[P_JVG + i]; JVa[i] = P[P_JVA + i]; JPg[i] = P[P_JPG + i]; JPa[i] = P[P_JPA + i]; }
    auto put = [&](int r0, int c0, const double* M, double s) { for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) J[(r0 + i) * 24 + c0 + j] = s * M[i * 3 + j]; };
    double Rwb2t[9], A[9], H[9];
    mat3_T(Rwb2, Rwb2t);
    mat3_mul(Rwb2t, Rwb1, A); mat3_mul(invJr, A, A);
    put(0, 0, A, -1.0);                                         // -invJr*Rwb2^T*Rwb1
    hat(rv, H); put(3, 0, H, 1.0);                              // hat(Rbw1*(v2 - v1 - g dt))
    // NOTE the reference uses 0.5*g*dt*dt here and g*dt*dt/2 in computeError: the same value
    hat(rp, H); put(6, 0, H, 1.0);
    const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    put(6, 3, I3, -1.0);
    put(3, 6, Rbw1, -1.0); put(6, 6, Rbw1, -dt);                // velocity 1
    double w[3], Jr[9], eRt[9];
    mat3_vec(JRg, dbg, w);
    right_jacobian(w, Jr, 1e-5);
    mat3_T(eR, eRt);
    mat3_mul(invJr, eRt, A); mat3_mul(A, Jr, A); mat3_mul(A, JRg, A);
    put(0, 9, A, -1.0); put(3, 9, JVg, -1.0); put(6, 9, JPg, -1.0);   // gyro bias
    put(3, 12, JVa, -1.0); put(6, 12, JPa, -1.0);               // acc bias
    put(0, 15, invJr, 1.0);                                     // pose 2
    mat3_mul(Rbw1, Rwb2, A); put(6, 18, A, 1.0);
    put(3, 21, Rbw1, 1.0);                                      // velocity 2
}

// EdgeMono for one edge.  Body pose (Rwb, twb), extrinsics Tcb = (Rcb, tcb), Tbc = (Rbc, tbc); pinhole cam4 (float promoted).
// err[2]; Jpoint[2][3] (_jacobianOplusXi); Jpose[2][6] (_jacobianOplusXj, tangent = (rotation, translation) of ImuCamPose::Update).
void orbo_imu_edge_mono(const double* Rwb, const double* twb, const double* Rcb, const double* tcb, const double* Rbc, const double* tbc,
                        const float* cam4, const double* Xw, const double* obs, double* err, double* Jpoint, double* Jpose, int* depthPositive) {
    double Rbw[9], tbw[3], Rcw[9], tcw[3];
    mat3_T(Rwb, Rbw);
    mat3_vec(Rbw, twb, tbw);
    for (int i = 0; i < 3; ++i) tbw[i] = -tbw[i];
    mat3_mul(Rcb, Rbw, Rcw);                                    // ImuCamPose::Update: Rcw = Rcb*Rbw, tcw = Rcb*tbw + tcb
    mat3_vec(Rcb, tbw, tcw);
    for (int i = 0; i < 3; ++i) tcw[i] += tcb[i];
    double Xc[3];
    mat3_vec(Rcw, Xw, Xc);
    for (int i = 0; i < 3; ++i) Xc[i] += tcw[i];
    const double fx = cam4[0], fy = cam4[1], cx = cam4[2], cy = cam4[3];
    err[0] = obs[0] - (fx * Xc[0] / Xc[2] + cx);
    err[1] = obs[1] - (fy * Xc[1] / Xc[2] + cy);
    if (depthPositive) *depthPositive = (Rcw[6] * Xw[0] + Rcw[7] * Xw[1] + Rcw[8] * Xw[2] + tcw[2]) > 0.0;
    if (!Jpoint) return;
    // Pinhole::projectJac (src/CameraModels/Pinhole.cpp:71-81)
    const double pj[6] = {fx / Xc[2], 0, -fx * Xc[0] / (Xc[2] * Xc[2]), 0, fy / Xc[2], -fy * Xc[1] / (Xc[2] * Xc[2])};
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 3; ++j) Jpoint[i * 3 + j] = -(pj[i * 3] * Rcw[j] + pj[i * 3 + 1] * Rcw[3 + j] + pj[i * 3 + 2] * Rcw[6 + j]);
    double Xb[3];
    mat3_vec(Rbc, Xc, Xb);
    for (int i = 0; i < 3; ++i) Xb[i] += tbc[i];
    const double x = Xb[0], y = Xb[1], z = Xb[2];
    const double S[18] = {0.0, z, -y, 1.0, 0.0, 0.0, -z, 0.0, x, 0.0, 1.0, 0.0, y, -x, 0.0, 0.0, 0.0, 1.0};
    double PR[6];
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 3; ++j) PR[i * 3 + j] = pj[i * 3] * Rcb[j] + pj[i * 3 + 1] * Rcb[3 + j] + pj[i * 3 + 2] * Rcb[6 + j];
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 6; ++j) Jpose[i * 6 + j] = PR[i * 3] * S[j] + PR[i * 3 + 1] * S[6 + j] + PR[i * 3 + 2] * S[12 + j];
}

// ImuCamPose::Update (VertexPose::oplusImpl): twb += Rwb*ut; Rwb = Rwb*ExpSO3(ur)   (the periodic re-normalisation left out)
void orbo_imu_pose_update(double* Rwb, double* twb, const double* pu) {
    double t[3], E[9];
    mat3_vec(Rwb, pu + 3, t);
    for (int i = 0; i < 3; ++i) twb[i] += t[i];
    exp_so3(pu, E, true);
    mat3_mul(Rwb, E, Rwb);
}

void orbo_normalize_rotation_f(const float* R, float* out) { normalize_rotation(R, out); }   // IMU::NormalizeRotation (float), for oracle/ref_shim/ref_wrap_preint.cpp

void orbo_so3(int what, const double* in, double* out) {   // 0 Exp, 1 Log, 2 RightJacobian, 3 InverseRightJacobian, 4 NormalizeRotation
    if (what == 0) exp_so3(in, out, true);
    else if (what == 1) log_so3(in, out);
    else if (what == 2) right_jacobian(in, out, 1e-5);
    else if (what == 3) inv_right_jacobian(in, out);
    else normalize_rotation(in, out);
}

// int Optimizer::PoseInertialOptimizationLastKeyFrame(Frame* pFrame, bool bRecInit) (src/Optimizer.cc:4491-4873), monocular frame:
// the tracking-side inertial pose optimiser (Tracking::TrackLocalMap, src/Tracking.cc:2985-2994).  Unknowns: the frame's VertexPose (6: rotation,
// translation of ImuCamPose::Update), VertexVelocity, VertexGyroBias, VertexAccBias = 15; the last keyframe's four vertices are fixed.
// Edges: EdgeMonoOnlyPose per map point (Huber sqrt(5.991), dropped after round 2), EdgeInertial (preintegration from the last keyframe,
// biases of the keyframe), EdgeGyroRW, EdgeAccRW.  Four rounds of g2o Gauss-Newton (OptimizationAlgorithmGaussNewton::solve: computeActiveErrors,
// buildSystem, dense LDLT, update; 10 iterations each, no restart of the estimate) with the chi2 re-classification of :4713-4778 (thresholds
// 12 / 7.5 / 5.991 / 5.991, x1.5 for points closer than 10 m, stale errors for edges that were active, recomputed ones for outliers), the
// recovery of :4783-4810, and the Hessian of the new prior (:4819-4867).
// state15: Rwb 9 | twb 3 | v 3 | bg 3 | ba 3 (in/out for the frame; the keyframe's is read only).  Returns nInitialCorrespondences - nBad.
static bool ldlt_solve(int n, const double* A, const double* b, double* x) {   // Eigen::LDLT + isPositive() (linear_solver_dense.h:111-118)
    std::vector<double> L(A, A + (size_t)n * n), d(n), y(n);
    for (int j = 0; j < n; ++j) {
        double dj = L[j * n + j];
        for (int k = 0; k < j; ++k) dj -= L[j * n + k] * L[j * n + k] * d[k];
        if (!(dj > 0)) return false;
        d[j] = dj;
        for (int i = j + 1; i < n; ++i) {
            double v = L[i * n + j];
            for (int k = 0; k < j; ++k) v -= L[i * n + k] * L[j * n + k] * d[k];
            L[i * n + j] = v / dj;
        }
    }
    for (int i = 0; i < n; ++i) { double v = b[i]; for (int k = 0; k < i; ++k) v -= L[i * n + k] * y[k]; y[i] = v; }
    for (int i = n - 1; i >= 0; --i) { double v = y[i] / d[i]; for (int k = i + 1; k < n; ++k) v -= L[k * n + i] * x[k]; x[i] = v; }
    return true;
}
// the problem as a state with the operations g2o performs on it (shared by the solver below and by its step-by-step form, OrboLmBackend)
struct PoseInertialKF {
    int N; const float *invSigma2, *trackDepth, *cam4, *P; const double *Rcb, *tcb, *Rbc, *tbc;
    const double *Rwbk, *twbk, *vk, *bgk, *bak;
    double *Rwb, *twb, *v, *bg, *ba;
    double Info9[81], InfoG[9], InfoA[9], delta, dsqr;
    std::vector<double> Xd, od, err;
    std::vector<uint8_t> level, robust;
    int its = 0;                                                            // ImuCamPose::its
    double x[15], H[225], b[15];
    void edge_error(int i, double* e2, int* dpos) const { orbo_imu_edge_mono(Rwb, twb, Rcb, tcb, Rbc, tbc, cam4, &Xd[3 * i], &od[2 * i], e2, nullptr, nullptr, dpos); }
    void compute_error(int i) { edge_error(i, &err[2 * i], nullptr); }
    double chi2(int i) const { return (double)invSigma2[i] * (err[2 * i] * err[2 * i] + err[2 * i + 1] * err[2 * i + 1]); }
    void build() {                                                          // computeActiveErrors + buildSystem
        for (double& q : H) q = 0;
        for (double& q : b) q = 0;
        for (int i = 0; i < N; ++i) {
            if (level[i]) continue;
            double Jpt[6], Jp[12];
            orbo_imu_edge_mono(Rwb, twb, Rcb, tcb, Rbc, tbc, cam4, &Xd[3 * i], &od[2 * i], &err[2 * i], Jpt, Jp, nullptr);
            const double om = (double)invSigma2[i];
            const double c2 = om * (err[2 * i] * err[2 * i] + err[2 * i + 1] * err[2 * i + 1]);
            double w = 1.0;
            if (robust[i] && c2 > dsqr) w = delta / std::sqrt(c2);
            for (int a = 0; a < 6; ++a) {
                b[a] -= w * om * (Jp[a] * err[2 * i] + Jp[6 + a] * err[2 * i + 1]);
                for (int c = 0; c < 6; ++c) H[a * 15 + c] += w * om * (Jp[a] * Jp[c] + Jp[6 + a] * Jp[6 + c]);
            }
        }
        {   // EdgeInertial: only the Jacobians of the frame's pose (columns 15..20) and velocity (21..23) count, the keyframe is fixed
            double e9[9], J[216], Jc[81], OJ[81];
            orbo_imu_edge_inertial(P, Rwbk, twbk, vk, bgk, bak, Rwb, twb, v, e9, J);
            for (int r = 0; r < 9; ++r) for (int c = 0; c < 9; ++c) Jc[r * 9 + c] = J[r * 24 + 15 + c];
            for (int r = 0; r < 9; ++r) for (int c = 0; c < 9; ++c) { double s = 0; for (int k = 0; k < 9; ++k) s += Info9[r * 9 + k] * Jc[k * 9 + c]; OJ[r * 9 + c] = s; }
            for (int a = 0; a < 9; ++a) {
                double s = 0;
                for (int r = 0; r < 9; ++r) s += OJ[r * 9 + a] * e9[r];            // J^T Omega e (Omega symmetric)
                b[a] -= s;
                for (int c = 0; c < 9; ++c) { double h = 0; for (int r = 0; r < 9; ++r) h += Jc[r * 9 + a] * OJ[r * 9 + c]; H[a * 15 + c] += h; }
            }
        }
        for (int a = 0; a < 3; ++a) {                                   // EdgeGyroRW / EdgeAccRW: error = b2 - b1, Jacobian of the free vertex = I
            double sg = 0, sa = 0;
            for (int c = 0; c < 3; ++c) { sg += InfoG[a * 3 + c] * (bg[c] - bgk[c]); sa += InfoA[a * 3 + c] * (ba[c] - bak[c]); H[(9 + a) * 15 + 9 + c] += InfoG[a * 3 + c]; H[(12 + a) * 15 + 12 + c] += InfoA[a * 3 + c]; }
            b[9 + a] -= sg; b[12 + a] -= sa;
        }
    }
    bool solve() { return ldlt_solve(15, H, b, x); }                    // a failed solve leaves x from the previous iteration, update() still runs
    void update() {
        orbo_imu_pose_update(Rwb, twb, x);
        // `NormalizeRotation(Rwb);` every third update (src/G2oTypes.cc:202-208) has no effect: the function (include/G2oTypes.h:67-71) returns the
        // normalised matrix and the call discards it
        if (++its >= 3) its = 0;
        for (int k = 0; k < 3; ++k) { v[k] += x[6 + k]; bg[k] += x[9 + k]; ba[k] += x[12 + k]; }
    }
    void init(int N_, const float* Xw, const float* obs, const float* invSigma2_, const float* trackDepth_, const float* cam4_, const double* extr24, const float* P_,
              const double* kfState15, double* state15) {
        N = N_; invSigma2 = invSigma2_; trackDepth = trackDepth_; cam4 = cam4_; P = P_;
        Rcb = extr24; tcb = extr24 + 9; Rbc = extr24 + 12; tbc = extr24 + 21;
        Rwb = state15; twb = state15 + 9; v = state15 + 12; bg = state15 + 15; ba = state15 + 18;
        Rwbk = kfState15; twbk = kfState15 + 9; vk = kfState15 + 12; bgk = kfState15 + 15; bak = kfState15 + 18;
        orbo_imu_information(P, Info9, InfoG, InfoA);
        delta = (double)sqrtf(5.991f); dsqr = delta * delta;            // const float thHuberMono = sqrt(5.991); rk->setDelta(thHuberMono)
        Xd.resize(3 * (size_t)N); od.resize(2 * (size_t)N); err.assign(2 * (size_t)N, 0.0);
        for (int i = 0; i < 3 * N; ++i) Xd[i] = (double)Xw[i];
        for (int i = 0; i < 2 * N; ++i) od[i] = (double)obs[i];
        level.assign(N, 0); robust.assign(N, 1);
        its = 0;
        for (double& q : x) q = 0;
    }
};
// `rounds` x `iters`: 4 x 10 in the reference; the tests also run a single Gauss-Newton step
int orbo_pose_inertial_opt_last_kf_n(int N, const float* Xw, const float* obs, const float* invSigma2, const float* trackDepth, const float* cam4, const double* extr24,
                                     const float* P, const double* kfState15, double* state15, int bRecInit, uint8_t* outlier, double* H15, int rounds, int iters) {
    PoseInertialKF S;
    S.init(N, Xw, obs, invSigma2, trackDepth, cam4, extr24, P, kfState15, state15);
    const double *Rcb = S.Rcb, *tcb = S.tcb, *Rbc = S.Rbc, *tbc = S.tbc;
    double *Rwb = S.Rwb, *twb = S.twb, *v = S.v;
    const double *Rwbk = S.Rwbk, *twbk = S.twbk, *vk = S.vk, *bgk = S.bgk, *bak = S.bak;
    const double *Info9 = S.Info9, *InfoG = S.InfoG, *InfoA = S.InfoA;
    const std::vector<double>&Xd = S.Xd, &od = S.od;
    for (int i = 0; i < N; ++i) outlier[i] = 0;
    const float chi2Mono[4] = {12, 7.5, 5.991, 5.991};
    int nBad = 0, nInliers = 0;
    for (int it = 0; it < rounds; ++it) {
        for (int iter = 0; iter < iters; ++iter) {                          // optimizer.optimize(its[it]) with OptimizationAlgorithmGaussNewton
            S.build();
            const bool ok = S.solve();
            S.update();
            if (!ok) break;
        }
        int nBadMono = 0, nInliersMono = 0;
        const float chi2close = 1.5 * chi2Mono[it];
        for (int i = 0; i < N; ++i) {
            int dpos = 0;
            double e2[2];
            S.edge_error(i, e2, &dpos);
            if (outlier[i]) { S.err[2 * i] = e2[0]; S.err[2 * i + 1] = e2[1]; }     // e->computeError() only for the outliers; the others keep their last active error
            const float chi2 = (float)S.chi2(i);
            const bool bClose = trackDepth[i] < 10.f;
            if ((chi2 > chi2Mono[it] && !bClose) || (bClose && chi2 > chi2close) || !dpos) { outlier[i] = 1; S.level[i] = 1; ++nBadMono; }
            else { outlier[i] = 0; S.level[i] = 0; ++nInliersMono; }
            if (it == 2) S.robust[i] = 0;
        }
        nInliers = nInliersMono; nBad = nBadMono;
        if (N + 3 < 10) break;                                              // optimizer.edges().size() < 10
    }
    if (nInliers < 30 && !bRecInit) {
        nBad = 0;
        for (int i = 0; i < N; ++i) {
            double e2[2];
            S.edge_error(i, e2, nullptr);
            S.err[2 * i] = e2[0]; S.err[2 * i + 1] = e2[1];
            if ((double)invSigma2[i] * (e2[0] * e2[0] + e2[1] * e2[1]) < (double)18.f) outlier[i] = 0; else ++nBad;
        }
    }
    // the prior of the next frame (:4819-4867): H = EdgeInertial::GetHessian2 + the two random-walk informations + the inliers' EdgeMonoOnlyPose Hessians
    for (int i = 0; i < 225; ++i) H15[i] = 0;
    {
        double e9[9], J[216];
        orbo_imu_edge_inertial(P, Rwbk, twbk, vk, bgk, bak, Rwb, twb, v, e9, J);
        for (int a = 0; a < 9; ++a) for (int c = 0; c < 9; ++c) {
            double h = 0;
            for (int r = 0; r < 9; ++r) for (int k = 0; k < 9; ++k) h += J[r * 24 + 15 + a] * Info9[r * 9 + k] * J[k * 24 + 15 + c];
            H15[a * 15 + c] += h;
        }
    }
    for (int a = 0; a < 3; ++a) for (int c = 0; c < 3; ++c) { H15[(9 + a) * 15 + 9 + c] += InfoG[a * 3 + c]; H15[(12 + a) * 15 + 12 + c] += InfoA[a * 3 + c]; }
    for (int i = 0; i < N; ++i) {
        if (outlier[i]) continue;
        double e2[2], Jpt[6], Jp[12];
        orbo_imu_edge_mono(Rwb, twb, Rcb, tcb, Rbc, tbc, cam4, &Xd[3 * i], &od[2 * i], e2, Jpt, Jp, nullptr);
        const double om = (double)invSigma2[i];
        for (int a = 0; a < 6; ++a) for (int c = 0; c < 6; ++c) H15[a * 15 + c] += om * (Jp[a] * Jp[c] + Jp[6 + a] * Jp[6 + c]);
    }
    return N - nBad;
}
// ---- the last-keyframe problem opened step by step: OrboLmBackend for g2o's Gauss-Newton / optimize() text + the per-edge operations the four rounds of
//      Optimizer::PoseInertialOptimizationLastKeyFrame (src/Optimizer.cc:4698-4823) perform (oracle/ref_shim/ref_wrap_g2o_lm.cpp compiles that text verbatim) ----
namespace {
struct PiKfOpen { PoseInertialKF S; std::vector<float> Xw, obs, is2, td, cam, P; std::vector<double> extr, kf, st; double diag[15]; };
void pik_compute_errors(void* p) { PoseInertialKF& S = ((PiKfOpen*)p)->S; for (int i = 0; i < S.N; ++i) if (!S.level[i]) S.compute_error(i); }
double pik_robust_chi2(void*) { return 0.0; }                             // Gauss-Newton does not look at the cost
void pik_build_system(void* p) { PiKfOpen* o = (PiKfOpen*)p; o->S.build(); for (int a = 0; a < 15; ++a) o->diag[a] = o->S.H[a * 16]; }
int pik_solve(void* p, double) { return ((PiKfOpen*)p)->S.solve() ? 1 : 0; }
void pik_update(void* p) { ((PiKfOpen*)p)->S.update(); }
void pik_nop(void*) {}
int pik_vector_size(void*) { return 15; }
const double* pik_x(void* p) { return ((PiKfOpen*)p)->S.x; }
const double* pik_b(void* p) { return ((PiKfOpen*)p)->S.b; }
int pik_n_diag(void*) { return 15; }
const double* pik_diag(void* p) { return ((PiKfOpen*)p)->diag; }
}  // namespace
void orbo_pikf_open(int N, const float* Xw, const float* obs, const float* invSigma2, const float* trackDepth, const float* cam4, const double* extr24, const float* P,
                    const double* kfState15, const double* state15, OrboLmBackend* out) {
    PiKfOpen* o = new PiKfOpen;
    o->Xw.assign(Xw, Xw + 3 * (size_t)N); o->obs.assign(obs, obs + 2 * (size_t)N); o->is2.assign(invSigma2, invSigma2 + N); o->td.assign(trackDepth, trackDepth + N);
    o->cam.assign(cam4, cam4 + 4); o->P.assign(P, P + P_SIZE); o->extr.assign(extr24, extr24 + 24); o->kf.assign(kfState15, kfState15 + 21); o->st.assign(state15, state15 + 21);
    o->S.init(N, o->Xw.data(), o->obs.data(), o->is2.data(), o->td.data(), o->cam.data(), o->extr.data(), o->P.data(), o->kf.data(), o->st.data());
    for (double& d : o->diag) d = 0;
    *out = OrboLmBackend{o, pik_compute_errors, pik_robust_chi2, pik_build_system, pik_solve, pik_update, pik_nop, pik_nop, pik_vector_size, pik_x, pik_b, pik_n_diag, pik_diag};
}
void orbo_pikf_edge_compute_error(void* h, int e) { ((PiKfOpen*)h)->S.compute_error(e); }
double orbo_pikf_edge_chi2(void* h, int e) { return ((PiKfOpen*)h)->S.chi2(e); }
int orbo_pikf_edge_depth_positive(void* h, int e) { double e2[2]; int d = 0; ((PiKfOpen*)h)->S.edge_error(e, e2, &d); return d; }
void orbo_pikf_edge_set_level(void* h, int e, int level) { ((PiKfOpen*)h)->S.level[e] = (uint8_t)level; }
void orbo_pikf_edge_set_robust(void* h, int e, int on) { ((PiKfOpen*)h)->S.robust[e] = (uint8_t)on; }
void orbo_pikf_close(void* h, double* stateOut21) { PiKfOpen* o = (PiKfOpen*)h; for (int i = 0; i < 21; ++i) stateOut21[i] = o->st[i]; delete o; }

int orbo_pose_inertial_opt_last_kf(int N, const float* Xw, const float* obs, const float* invSigma2, const float* trackDepth, const float* cam4, const double* extr24,
                                   const float* P, const double* kfState15, double* state15, int bRecInit, uint8_t* outlier, double* H15) {
    return orbo_pose_inertial_opt_last_kf_n(N, Xw, obs, invSigma2, trackDepth, cam4, extr24, P, kfState15, state15, bRecInit, outlier, H15, 4, 10);
}

// int Optimizer::PoseInertialOptimizationLastFrame(Frame* pFrame, bool bRecInit) (src/Optimizer.cc:4875-5289), monocular frame: like the
// last-keyframe variant, but the PREVIOUS FRAME's four vertices are free too (30 unknowns), held by EdgePriorPoseImu (its ConstraintPoseImu:
// state + 15 x 15 information, Huber delta 5; src/G2oTypes.cc:720-760); EdgeInertial uses mpImuPreintegratedFrame (frame to frame), the two
// random-walk informations come from mpImuPreintegrated (since the last keyframe) (:5068-5078).  Thresholds 5.991 in all four rounds.
// Afterwards the 30 x 30 Hessian is assembled in the order (previous 15 | current 15) and the previous frame is marginalised
// (Optimizer::Marginalize, :2960-3043: Schur complement with the SVD pseudo-inverse, singular values <= 1e-6 dropped).
// x layout here: current pose 6, v 3, bg 3, ba 3 | previous pose 6, v 3, bg 3, ba 3.
static void sym_eig(int n, const double* Ain, double* V, double* w) {   // cyclic Jacobi, A = V diag(w) V^T
    std::vector<double> A(Ain, Ain + (size_t)n * n);
    for (int i = 0; i < n * n; ++i) V[i] = (i % (n + 1) == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 100; ++sweep) {
        double off = 0, diag = 0;
        for (int p = 0; p < n; ++p) { diag += A[p * n + p] * A[p * n + p]; for (int q = p + 1; q < n; ++q) off += A[p * n + q] * A[p * n + q]; }
        if (off <= 1e-30 * diag || off < 1e-300) break;
        for (int p = 0; p < n; ++p)
            for (int q = p + 1; q < n; ++q) {
                const double apq = A[p * n + q];
                if (apq == 0) continue;
                const double theta = (A[q * n + q] - A[p * n + p]) / (2 * apq);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1));
                const double c = 1 / std::sqrt(t * t + 1), sn = t * c;
                for (int k = 0; k < n; ++k) { const double akp = A[k * n + p], akq = A[k * n + q]; A[k * n + p] = c * akp - sn * akq; A[k * n + q] = sn * akp + c * akq; }
                for (int k = 0; k < n; ++k) { const double apk = A[p * n + k], aqk = A[q * n + k]; A[p * n + k] = c * apk - sn * aqk; A[q * n + k] = sn * apk + c * aqk; }
                for (int k = 0; k < n; ++k) { const double vkp = V[k * n + p], vkq = V[k * n + q]; V[k * n + p] = c * vkp - sn * vkq; V[k * n + q] = sn * vkp + c * vkq; }
            }
    }
    for (int i = 0; i < n; ++i) w[i] = A[i * n + i];
}
// ConstraintPoseImu's constructor (include/G2oTypes.h:711-722): symmetrise, clamp eigenvalues < 1e-12 to 0
void orbo_constraint_pose_imu_information(const double* Hin, double* Hout) {
    double S[225], V[225], w[15];
    for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) S[i * 15 + j] = (Hin[i * 15 + j] + Hin[j * 15 + i]) / 2;
    sym_eig(15, S, V, w);
    for (int i = 0; i < 15; ++i) if (w[i] < 1e-12) w[i] = 0;
    for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) { double a = 0; for (int k = 0; k < 15; ++k) a += V[i * 15 + k] * w[k] * V[j * 15 + k]; Hout[i * 15 + j] = a; }
}
// EdgePriorPoseImu: residual (15) and the diagonal-block Jacobian (15 x 15 wrt pose 6, v, bg, ba) of the previous frame
static void prior_edge(const double* prior21, const double* st21, double* e15, double* J225) {
    const double *Rp = prior21, *tp = prior21 + 9;
    double Rpt[9], dR[9], er[3], d[3], et[3];
    mat3_T(Rp, Rpt); mat3_mul(Rpt, st21, dR);
    log_so3(dR, er);
    for (int i = 0; i < 3; ++i) d[i] = st21[9 + i] - tp[i];
    mat3_vec(Rpt, d, et);
    for (int i = 0; i < 3; ++i) { e15[i] = er[i]; e15[3 + i] = et[i]; e15[6 + i] = st21[12 + i] - prior21[12 + i]; e15[9 + i] = st21[15 + i] - prior21[15 + i]; e15[12 + i] = st21[18 + i] - prior21[18 + i]; }
    if (!J225) return;
    for (int i = 0; i < 225; ++i) J225[i] = 0;
    double iJ[9];
    inv_right_jacobian(er, iJ);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { J225[i * 15 + j] = iJ[i * 3 + j]; J225[(3 + i) * 15 + 3 + j] = dR[i * 3 + j]; }
    for (int i = 6; i < 15; ++i) J225[i * 15 + i] = 1.0;
}
// the problem as a state with the operations g2o performs on it (shared by the solver below and by its step-by-step form, OrboLmBackend); unknowns: current 15 | previous 15
struct PoseInertialLF {
    int N; const float *invSigma2, *trackDepth, *cam4, *Pframe; const double *Rcb, *tcb, *Rbc, *tbc, *prior21, *priorH;
    double* S[2];                                    // current, previous
    double Info9[81], InfoG[9], InfoA[9], delta, dsqr;
    std::vector<double> Xd, od, err, H;
    std::vector<uint8_t> level, robust;
    int its[2];
    double x[30], b[30];
    static int xi(int c) { return c < 15 ? 15 + c : c - 15; }   // column of x for column c of the EdgeInertial Jacobian (vertex order: previous pose, v, bg, ba, current pose, v)
    void inertial(double* e9, double* J) const { orbo_imu_edge_inertial(Pframe, S[1], S[1] + 9, S[1] + 12, S[1] + 15, S[1] + 18, S[0], S[0] + 9, S[0] + 12, e9, J); }
    void edge_error(int i, double* e2, int* dpos) const { orbo_imu_edge_mono(S[0], S[0] + 9, Rcb, tcb, Rbc, tbc, cam4, &Xd[3 * i], &od[2 * i], e2, nullptr, nullptr, dpos); }
    void compute_error(int i) { edge_error(i, &err[2 * i], nullptr); }
    double chi2(int i) const { return (double)invSigma2[i] * (err[2 * i] * err[2 * i] + err[2 * i + 1] * err[2 * i + 1]); }
    void build() {
        std::fill(H.begin(), H.end(), 0.0);
        for (double& q : b) q = 0;
        for (int i = 0; i < N; ++i) {
            if (level[i]) continue;
            double Jpt[6], Jp[12];
            orbo_imu_edge_mono(S[0], S[0] + 9, Rcb, tcb, Rbc, tbc, cam4, &Xd[3 * i], &od[2 * i], &err[2 * i], Jpt, Jp, nullptr);
            const double om = (double)invSigma2[i];
            const double c2 = om * (err[2 * i] * err[2 * i] + err[2 * i + 1] * err[2 * i + 1]);
            const double w = (robust[i] && c2 > dsqr) ? delta / std::sqrt(c2) : 1.0;
            for (int a = 0; a < 6; ++a) {
                b[a] -= w * om * (Jp[a] * err[2 * i] + Jp[6 + a] * err[2 * i + 1]);
                for (int c = 0; c < 6; ++c) H[a * 30 + c] += w * om * (Jp[a] * Jp[c] + Jp[6 + a] * Jp[6 + c]);
            }
        }
        {
            double e9[9], J[216], OJ[216];
            inertial(e9, J);
            for (int r = 0; r < 9; ++r) for (int c = 0; c < 24; ++c) { double a = 0; for (int k = 0; k < 9; ++k) a += Info9[r * 9 + k] * J[k * 24 + c]; OJ[r * 24 + c] = a; }
            for (int a = 0; a < 24; ++a) {
                double g = 0;
                for (int r = 0; r < 9; ++r) g += OJ[r * 24 + a] * e9[r];
                b[xi(a)] -= g;
                for (int c = 0; c < 24; ++c) { double h = 0; for (int r = 0; r < 9; ++r) h += J[r * 24 + a] * OJ[r * 24 + c]; H[xi(a) * 30 + xi(c)] += h; }
            }
        }
        for (int a = 0; a < 3; ++a) {           // EdgeGyroRW (VGk, VG), EdgeAccRW (VAk, VA): error = b_cur - b_prev, Jacobians -I / +I
            double sg = 0, sa = 0;
            for (int c = 0; c < 3; ++c) {
                const double og = InfoG[a * 3 + c], oa = InfoA[a * 3 + c];
                sg += og * (S[0][15 + c] - S[1][15 + c]); sa += oa * (S[0][18 + c] - S[1][18 + c]);
                H[(9 + a) * 30 + 9 + c] += og; H[(24 + a) * 30 + 24 + c] += og; H[(9 + a) * 30 + 24 + c] -= og; H[(24 + a) * 30 + 9 + c] -= og;
                H[(12 + a) * 30 + 12 + c] += oa; H[(27 + a) * 30 + 27 + c] += oa; H[(12 + a) * 30 + 27 + c] -= oa; H[(27 + a) * 30 + 12 + c] -= oa;
            }
            b[9 + a] -= sg; b[24 + a] += sg; b[12 + a] -= sa; b[27 + a] += sa;
        }
        {   // EdgePriorPoseImu on the previous frame, Huber delta 5
            double e15[15], J[225], OJ[225], Oe[15];
            prior_edge(prior21, S[1], e15, J);
            double c2 = 0;
            for (int r = 0; r < 15; ++r) { double a = 0; for (int k = 0; k < 15; ++k) a += priorH[r * 15 + k] * e15[k]; Oe[r] = a; c2 += e15[r] * a; }
            const double w = c2 > 25.0 ? 5.0 / std::sqrt(c2) : 1.0;
            for (int r = 0; r < 15; ++r) for (int c = 0; c < 15; ++c) { double a = 0; for (int k = 0; k < 15; ++k) a += priorH[r * 15 + k] * J[k * 15 + c]; OJ[r * 15 + c] = a; }
            for (int a = 0; a < 15; ++a) {
                double g = 0;
                for (int r = 0; r < 15; ++r) g += J[r * 15 + a] * Oe[r];
                b[15 + a] -= w * g;
                for (int c = 0; c < 15; ++c) { double h = 0; for (int r = 0; r < 15; ++r) h += J[r * 15 + a] * OJ[r * 15 + c]; H[(15 + a) * 30 + 15 + c] += w * h; }
            }
        }
    }
    bool solve() { return ldlt_solve(30, H.data(), b, x); }
    void update() {
        for (int k = 0; k < 2; ++k) {
            const double* dx = x + 15 * k;
            orbo_imu_pose_update(S[k], S[k] + 9, dx);
            if (++its[k] >= 3) its[k] = 0;      // the reference's NormalizeRotation(Rwb) call discards its result (see the last-keyframe variant)
            for (int q = 0; q < 3; ++q) { S[k][12 + q] += dx[6 + q]; S[k][15 + q] += dx[9 + q]; S[k][18 + q] += dx[12 + q]; }
        }
    }
    void init(int N_, const float* Xw, const float* obs, const float* invSigma2_, const float* trackDepth_, const float* cam4_, const double* extr24, const float* Pframe_,
              const float* Pkf, const double* prior21_, const double* priorH_, double* prevState21, double* state21) {
        N = N_; invSigma2 = invSigma2_; trackDepth = trackDepth_; cam4 = cam4_; Pframe = Pframe_; prior21 = prior21_; priorH = priorH_;
        Rcb = extr24; tcb = extr24 + 9; Rbc = extr24 + 12; tbc = extr24 + 21;
        S[0] = state21; S[1] = prevState21;
        double tmpI[81];
        orbo_imu_information(Pframe, Info9, tmpI, tmpI);
        orbo_imu_information(Pkf, tmpI, InfoG, InfoA);
        delta = (double)sqrtf(5.991f); dsqr = delta * delta;
        Xd.resize(3 * (size_t)N); od.resize(2 * (size_t)N); err.assign(2 * (size_t)N, 0.0); H.assign(900, 0.0);
        for (int i = 0; i < 3 * N; ++i) Xd[i] = (double)Xw[i];
        for (int i = 0; i < 2 * N; ++i) od[i] = (double)obs[i];
        level.assign(N, 0); robust.assign(N, 1);
        its[0] = its[1] = 0;
        for (double& q : x) q = 0;
    }
};
int orbo_pose_inertial_opt_last_frame_n(int N, const float* Xw, const float* obs, const float* invSigma2, const float* trackDepth, const float* cam4, const double* extr24,
                                        const float* Pframe, const float* Pkf, const double* prior21, const double* priorH, double* prevState21, double* state21,
                                        int bRecInit, uint8_t* outlier, double* H15, int rounds, int iters) {
    PoseInertialLF Q;
    Q.init(N, Xw, obs, invSigma2, trackDepth, cam4, extr24, Pframe, Pkf, prior21, priorH, prevState21, state21);
    const double *Rcb = Q.Rcb, *tcb = Q.tcb, *Rbc = Q.Rbc, *tbc = Q.tbc;
    double** S = Q.S;
    const double *Info9 = Q.Info9, *InfoG = Q.InfoG, *InfoA = Q.InfoA;
    const std::vector<double>&Xd = Q.Xd, &od = Q.od;
    auto inertial = [&](double* e9, double* J) { Q.inertial(e9, J); };
    for (int i = 0; i < N; ++i) outlier[i] = 0;
    const float chi2Mono[4] = {5.991, 5.991, 5.991, 5.991};
    int nBad = 0, nInliers = 0;
    for (int it = 0; it < rounds; ++it) {
        for (int iter = 0; iter < iters; ++iter) {
            Q.build();
            const bool ok = Q.solve();
            Q.update();
            if (!ok) break;
        }
        int nBadMono = 0, nInliersMono = 0;
        const float chi2close = 1.5 * chi2Mono[it];
        for (int i = 0; i < N; ++i) {
            int dpos = 0; double e2[2];
            Q.edge_error(i, e2, &dpos);
            if (outlier[i]) { Q.err[2 * i] = e2[0]; Q.err[2 * i + 1] = e2[1]; }
            const float chi2 = (float)Q.chi2(i);
            const bool bClose = trackDepth[i] < 10.f;
            if ((chi2 > chi2Mono[it] && !bClose) || (bClose && chi2 > chi2close) || !dpos) { outlier[i] = 1; Q.level[i] = 1; ++nBadMono; } else { outlier[i] = 0; Q.level[i] = 0; ++nInliersMono; }
            if (it == 2) Q.robust[i] = 0;
        }
        nInliers = nInliersMono; nBad = nBadMono;
        if (N + 4 < 10) break;                                              // optimizer.edges().size() < 10 (N mono + inertial + 2 random walk + prior)
    }
    if (nInliers < 30 && !bRecInit) {
        nBad = 0;
        for (int i = 0; i < N; ++i) {
            double e2[2];
            Q.edge_error(i, e2, nullptr);
            if ((double)invSigma2[i] * (e2[0] * e2[0] + e2[1] * e2[1]) < (double)18.f) outlier[i] = 0; else ++nBad;
        }
    }
    // 30 x 30 Hessian in the reference's order (previous 15 | current 15) (:5216-5266), then Marginalize(H, 0, 14) and the current 15 x 15 block
    std::vector<double> Hf(900, 0.0);
    {
        double e9[9], J[216];
        inertial(e9, J);
        for (int a = 0; a < 24; ++a) for (int c = 0; c < 24; ++c) {
            double h = 0;
            for (int r = 0; r < 9; ++r) for (int k = 0; k < 9; ++k) h += J[r * 24 + a] * Info9[r * 9 + k] * J[k * 24 + c];
            Hf[a * 30 + c] += h;
        }
        for (int a = 0; a < 3; ++a) for (int c = 0; c < 3; ++c) {
            const double og = InfoG[a * 3 + c], oa = InfoA[a * 3 + c];
            Hf[(9 + a) * 30 + 9 + c] += og; Hf[(9 + a) * 30 + 24 + c] -= og; Hf[(24 + a) * 30 + 9 + c] -= og; Hf[(24 + a) * 30 + 24 + c] += og;
            Hf[(12 + a) * 30 + 12 + c] += oa; Hf[(12 + a) * 30 + 27 + c] -= oa; Hf[(27 + a) * 30 + 12 + c] -= oa; Hf[(27 + a) * 30 + 27 + c] += oa;
        }
        double e15[15], Jp[225];
        prior_edge(prior21, S[1], e15, Jp);
        for (int a = 0; a < 15; ++a) for (int c = 0; c < 15; ++c) {
            double h = 0;
            for (int r = 0; r < 15; ++r) for (int k = 0; k < 15; ++k) h += Jp[r * 15 + a] * priorH[r * 15 + k] * Jp[k * 15 + c];
            Hf[a * 30 + c] += h;
        }
    }
    for (int i = 0; i < N; ++i) {
        if (outlier[i]) continue;
        double e2[2], Jpt[6], Jp[12];
        orbo_imu_edge_mono(S[0], S[0] + 9, Rcb, tcb, Rbc, tbc, cam4, &Xd[3 * i], &od[2 * i], e2, Jpt, Jp, nullptr);
        const double om = (double)invSigma2[i];
        for (int a = 0; a < 6; ++a) for (int c = 0; c < 6; ++c) Hf[(15 + a) * 30 + 15 + c] += om * (Jp[a] * Jp[c] + Jp[6 + a] * Jp[6 + c]);
    }
    {   // H_cc - H_cb pinv(H_bb) H_bc, pinv through the eigen-decomposition of the symmetrised block (= the SVD of a symmetric matrix)
        double Hbb[225], V[225], w[15], pinv[225];
        for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) Hbb[i * 15 + j] = (Hf[i * 30 + j] + Hf[j * 30 + i]) / 2;
        sym_eig(15, Hbb, V, w);
        for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) {
            double a = 0;
            for (int k = 0; k < 15; ++k) if (std::fabs(w[k]) > 1e-6) a += V[i * 15 + k] * V[j * 15 + k] / w[k];
            pinv[i * 15 + j] = a;
        }
        for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) {
            double a = 0;
            for (int k = 0; k < 15; ++k) for (int l = 0; l < 15; ++l) a += Hf[(15 + i) * 30 + k] * pinv[k * 15 + l] * Hf[l * 30 + 15 + j];
            H15[i * 15 + j] = Hf[(15 + i) * 30 + 15 + j] - a;
        }
    }
    return N - nBad;
}
// ---- the last-frame problem opened step by step (as orbo_pikf_* for the last-keyframe variant): Optimizer.cc:5098-5221 ----
namespace {
struct PiLfOpen { PoseInertialLF Q; std::vector<float> Xw, obs, is2, td, cam, Pf, Pk; std::vector<double> extr, prior, priorH, prev, st; double diag[30]; };
void pil_compute_errors(void* p) { PoseInertialLF& Q = ((PiLfOpen*)p)->Q; for (int i = 0; i < Q.N; ++i) if (!Q.level[i]) Q.compute_error(i); }
double pil_robust_chi2(void*) { return 0.0; }
void pil_build_system(void* p) { PiLfOpen* o = (PiLfOpen*)p; o->Q.build(); for (int a = 0; a < 30; ++a) o->diag[a] = o->Q.H[a * 31]; }
int pil_solve(void* p, double) { return ((PiLfOpen*)p)->Q.solve() ? 1 : 0; }
void pil_update(void* p) { ((PiLfOpen*)p)->Q.update(); }
void pil_nop(void*) {}
int pil_vector_size(void*) { return 30; }
const double* pil_x(void* p) { return ((PiLfOpen*)p)->Q.x; }
const double* pil_b(void* p) { return ((PiLfOpen*)p)->Q.b; }
int pil_n_diag(void*) { return 30; }
const double* pil_diag(void* p) { return ((PiLfOpen*)p)->diag; }
}  // namespace
void orbo_pilf_open(int N, const float* Xw, const float* obs, const float* invSigma2, const float* trackDepth, const float* cam4, const double* extr24, const float* Pframe,
                    const float* Pkf, const double* prior21, const double* priorH, const double* prevState21, const double* state21, OrboLmBackend* out) {
    PiLfOpen* o = new PiLfOpen;
    o->Xw.assign(Xw, Xw + 3 * (size_t)N); o->obs.assign(obs, obs + 2 * (size_t)N); o->is2.assign(invSigma2, invSigma2 + N); o->td.assign(trackDepth, trackDepth + N);
    o->cam.assign(cam4, cam4 + 4); o->Pf.assign(Pframe, Pframe + P_SIZE); o->Pk.assign(Pkf, Pkf + P_SIZE); o->extr.assign(extr24, extr24 + 24);
    o->prior.assign(prior21, prior21 + 21); o->priorH.assign(priorH, priorH + 225); o->prev.assign(prevState21, prevState21 + 21); o->st.assign(state21, state21 + 21);
    o->Q.init(N, o->Xw.data(), o->obs.data(), o->is2.data(), o->td.data(), o->cam.data(), o->extr.data(), o->Pf.data(), o->Pk.data(), o->prior.data(), o->priorH.data(), o->prev.data(), o->st.data());
    for (double& d : o->diag) d = 0;
    *out = OrboLmBackend{o, pil_compute_errors, pil_robust_chi2, pil_build_system, pil_solve, pil_update, pil_nop, pil_nop, pil_vector_size, pil_x, pil_b, pil_n_diag, pil_diag};
}
void orbo_pilf_edge_compute_error(void* h, int e) { ((PiLfOpen*)h)->Q.compute_error(e); }
double orbo_pilf_edge_chi2(void* h, int e) { return ((PiLfOpen*)h)->Q.chi2(e); }
int orbo_pilf_edge_depth_positive(void* h, int e) { double e2[2]; int d = 0; ((PiLfOpen*)h)->Q.edge_error(e, e2, &d); return d; }
void orbo_pilf_edge_set_level(void* h, int e, int level) { ((PiLfOpen*)h)->Q.level[e] = (uint8_t)level; }
void orbo_pilf_edge_set_robust(void* h, int e, int on) { ((PiLfOpen*)h)->Q.robust[e] = (uint8_t)on; }
void orbo_pilf_close(void* h, double* prevOut21, double* stateOut21) { PiLfOpen* o = (PiLfOpen*)h; for (int i = 0; i < 21; ++i) { prevOut21[i] = o->prev[i]; stateOut21[i] = o->st[i]; } delete o; }

int orbo_pose_inertial_opt_last_frame(int N, const float* Xw, const float* obs, const float* invSigma2, const float* trackDepth, const float* cam4, const double* extr24,
                                      const float* Pframe, const float* Pkf, const double* prior21, const double* priorH, double* prevState21, double* state21,
                                      int bRecInit, uint8_t* outlier, double* H15) {
    return orbo_pose_inertial_opt_last_frame_n(N, Xw, obs, invSigma2, trackDepth, cam4, extr24, Pframe, Pkf, prior21, priorH, prevState21, state21, bRecInit, outlier, H15, 4, 10);
}

}  // extern "C"
