// Optimizer::LocalInertialBA (reference src/Optimizer.cc:2383-2958, monocular-inertial branch) -- the numeric core as ONE persistent
// CTA per local map: the whole g2o Levenberg-Marquardt loop (OptimizationAlgorithmLevenberg::solve, optimization_algorithm_levenberg.cpp:61-194;
// BlockSolverX::buildSystem / solve with the Schur complement over the marginalised points, block_solver.hpp:354-604) runs on the device.
//
// The algorithm is written once, as a sequence of CTA-wide phases driven through an executor `Exec`:
//     ex.par(f)   every thread t of the CTA runs f(t), then a CTA barrier;
//     ex.sum(f)   CTA-wide ordered sum of f(t) (fixed reduction tree), the same value returned to every thread;
//     ex.panel()  CTA-shared storage for the LDL^T panel (MAXN * LW doubles);
//     ex.tag(k)   marks the start of phase group k for the optional time profile (0 errors, 1 buildSystem, 2 Dinv / Y, 3 Schur, 4 LDL^T,
//                 5 point back-substitution, 6 push / update / pop, 7 the rest).
// Everything between two phases is uniform control flow (LM state replicated per thread).  On the GPU Exec is DeviceExec
// (local_inertial_ba.cu: threadIdx + __syncthreads + shuffles); tests/liba_emulate.cpp instantiates the very same code with a serial
// HostExec (g++), which checks the logic against the CPU oracle in this GPU-less container.  It is a test vehicle: the product library
// does not contain it and has no CPU path.
//
// Unknown layout of the reduced system: keyframe k of the temporal window (k < nOpt) owns rows 15 k .. 15 k + 14 =
// VertexPose (rotation 3, translation 3: tangent of ImuCamPose::Update) | VertexVelocity | VertexGyroBias | VertexAccBias.
// Sums run in fixed orders (edges of a point / of a keyframe in edge-index order), so a solve is run-to-run reproducible.
#pragma once
#include <stdint.h>

#include "inertial_dev.cuh"

namespace liba {

using namespace imu;
using g2o::huber;
using g2o::Levenberg;

#ifndef LIBA_NT
#define LIBA_NT 512
#endif
constexpr int NT = LIBA_NT;      // threads per CTA
constexpr int EJ = 24;           // per mono edge: A 2x3 | B 2x6 | w | r0 | r1 | 3 pad (192 B = six 32-byte vectors)
constexpr int WS = 20;           // per mono edge: the 6 x 3 block W (and Y) + 2 pad (160 B = five 32-byte vectors)
constexpr int LW = 5;            // panel width of the blocked LDL^T (15 = 3 * 5)
constexpr int SL = 32;           // slices of a keyframe's edge list in the Schur phase
constexpr int MAXN = 15 * 64;    // largest reduced system (liba_pack.h: check() admits at most 64 keyframes in the window)

// One problem, device (or emulation) view.  Inputs are written by the host packer (liba_pack.h); scratch is uninitialised.
struct Dev {
    int nKF, nOpt, nI, nL, nE, iterations, bLarge;
    double lambdaInit;
    // ---- inputs ----
    double* kfState;              // [nKF][21]  Rwb 9 | twb 3 | v 3 | bg 3 | ba 3        (current estimate)
    double* kfTcw;                // [nKF][12]  Rcw 9 | tcw 3                             (ImuCamPose's cached camera pose)
    const float* cam;             // [nKF][4]
    const double* extr;           // Rcb 9 | tcb 3 | Rbc 9 | tbc 3
    const int *ieKf1, *ieKf2;     // [nI]
    const float* preint;          // [nI][292]
    const uint8_t* ieRobust;      // [nI]
    const double* ieInfoScale;    // [nI]
    double* pts;                  // [nL][3]
    const float* trackDepth;      // [nL]
    const int *ePt, *eKf;         // [nE]
    const double* obs;            // [nE][2]
    const float* invSigma2;       // [nE]
    const int *ptStart, *ptEdges; // CSR point -> its edges (ascending edge index)
    const int *kfStart, *kfEdges; // CSR free keyframe -> its edges
    // ---- scratch ----
    int* pk;                      // [nL][nOpt] edge of (point, free keyframe) or -1
    double *info9, *infoG, *infoA;          // [nI][81], [nI][9], [nI][9]
    double *errM, *errI, *errG, *errA;      // the edges' _error
    double *ejac, *W, *Y;                   // [nE][EJ], [nE][WS], [nE][WS]
    double *Hll, *bl, *Dinv, *db;           // [nL][9], [nL][3], [nL][9], [nL][3]
    double *H, *b, *Hs, *bs, *dvec, *x;     // [n][n], [n], [n][n], [n], [n], [n + 3 nL]
    double *He, *be;                        // [nI][900], [nI][30]
    double *part, *partb;                   // [nPairs][SL][36], [nOpt][SL][6]: partial Schur sums
    double *Jin, *OJ, *Oe, *win;            // [nI][216], [nI][216], [nI][9], [nI]: EdgeInertial Jacobians, Omega J, Omega e, robust weight
    double *kfBk, *tcwBk, *ptsBk;           // push() / pop()
    // ---- outputs ----
    double *outState, *outTcw, *outPts;     // [nKF][21], [nKF][12], [nL][3]
    uint8_t* erase;                         // [nE]
    double* chi2;                           // [nE]
    double* stats;                          // [8]: err, err_end, failed, lambda, trials, iterations, solver ns
    double* prof;                           // [8]: nanoseconds per phase group (ex.tag)
};

// n32 consecutive 32-byte vectors (two LDG.E.128 each on the device, the widest sm_90 has -- the gathers of the per-edge records are bound
// by look-ups per instruction, not by bytes); p must be 32-byte aligned
template <int N32> IMU_HD inline void ldvec(const double* p, double* r) {
#if defined(__CUDA_ARCH__)
#pragma unroll
    for (int k = 0; k < 2 * N32; ++k)
        asm volatile("ld.global.v2.f64 {%0, %1}, [%2];" : "=d"(r[2 * k]), "=d"(r[2 * k + 1]) : "l"(p + 2 * k));
#else
    for (int k = 0; k < 4 * N32; ++k) r[k] = p[k];
#endif
}
template <int N32> IMU_HD inline void stvec(double* p, const double* r) {
#if defined(__CUDA_ARCH__)
#pragma unroll
    for (int k = 0; k < 2 * N32; ++k)
        asm volatile("st.global.v2.f64 [%0], {%1, %2};" ::"l"(p + 2 * k), "d"(r[2 * k]), "d"(r[2 * k + 1]) : "memory");
#else
    for (int k = 0; k < 4 * N32; ++k) p[k] = r[k];
#endif
}
template <int N> IMU_HD inline double quad(const double* M, const double* e) {
    double s = 0;
    for (int i = 0; i < N; ++i) { double t = 0; for (int j = 0; j < N; ++j) t += M[i * N + j] * e[j]; s += e[i] * t; }
    return s;
}
IMU_HD inline void inv3_cof(const double* m, double* o) {                            // Eigen fixed-size 3x3 inverse: cofactors / determinant
    const double c00 = m[4] * m[8] - m[5] * m[7], c10 = m[5] * m[6] - m[3] * m[8], c20 = m[3] * m[7] - m[4] * m[6];
    const double det = m[0] * c00 + m[1] * c10 + m[2] * c20;
    const double id = 1.0 / det;
    o[0] = c00 * id; o[1] = (m[2] * m[7] - m[1] * m[8]) * id; o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
    o[3] = c10 * id; o[4] = (m[0] * m[8] - m[2] * m[6]) * id; o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
    o[6] = c20 * id; o[7] = (m[1] * m[6] - m[0] * m[7]) * id; o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
}
// EdgeInertial's information matrix (src/G2oTypes.cc:499-507): inverse of the 9 x 9 covariance, symmetrised, then V diag(max(w, 0 if w < 1e-12)) V^T
// of its eigen-decomposition.  The eigen step only changes the matrix when an eigenvalue is below 1e-12.  lambda_min(Info) = 1 / lambda_max(C) >=
// 1 / trace(C), so for a positive definite Info (Cholesky succeeds) and trace(C) < 1e11 nothing is clamped and V diag(w) V^T reproduces the
// symmetrised inverse up to rounding: the serial Jacobi sweeps (~3 ms on one thread) are then skipped.  Otherwise the full path runs.
// information_fast_path: that test; true leaves the symmetrised inverse in A.
IMU_HD inline bool information_fast_path(const float* __restrict__ P, double* __restrict__ A) {
    double C9[81], Lc[81];
    double trace = 0;
    for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) C9[i * 9 + j] = (double)P[P_C + i * 15 + j];
    for (int i = 0; i < 9; ++i) trace += C9[i * 10];
    bool ok = invert_n<9>(C9, A) && trace < 1e11;
    if (ok) {
        for (int i = 0; i < 9; ++i) for (int j = i; j < 9; ++j) { const double v = (A[i * 9 + j] + A[j * 9 + i]) / 2; A[i * 9 + j] = A[j * 9 + i] = v; }
        for (int j = 0; j < 9 && ok; ++j) {                      // Cholesky: positive definite?
            double dj = A[j * 9 + j];
            for (int k = 0; k < j; ++k) dj -= Lc[j * 9 + k] * Lc[j * 9 + k];
            if (!(dj > 0)) { ok = false; break; }
            dj = sqrt(dj);
            Lc[j * 9 + j] = dj;
            for (int i = j + 1; i < 9; ++i) {
                double v = A[i * 9 + j];
                for (int k = 0; k < j; ++k) v -= Lc[i * 9 + k] * Lc[j * 9 + k];
                Lc[i * 9 + j] = v / dj;
            }
        }
    }
    return ok;
}
IMU_HD inline void information_matrices(const float* __restrict__ P, double* __restrict__ I9, double* __restrict__ IG, double* __restrict__ IA) {
    double A[81];
    if (!information_fast_path(P, A)) { imu_information_dev(P, I9, IG, IA); return; }
    for (int i = 0; i < 81; ++i) I9[i] = A[i];
    double G[9], Aa[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { G[i * 3 + j] = (double)P[P_C + (9 + i) * 15 + 9 + j]; Aa[i * 3 + j] = (double)P[P_C + (12 + i) * 15 + 12 + j]; }
    invert_n<3>(G, IG);
    invert_n<3>(Aa, IA);
}
IMU_HD inline void edge_states(const Dev& D, int i, double* S) {                     // the six vertices of EdgeInertial i
    const double* a = D.kfState + 21 * (size_t)D.ieKf1[i];
    const double* c = D.kfState + 21 * (size_t)D.ieKf2[i];
    for (int k = 0; k < 21; ++k) S[k] = a[k];
    for (int k = 0; k < 15; ++k) S[21 + k] = c[k];
}
IMU_HD inline void mono_camera_point(const Dev& D, int e, double* Xc) {
    const double* T = D.kfTcw + 12 * (size_t)D.eKf[e];
    const double* X = D.pts + 3 * (size_t)D.ePt[e];
    for (int i = 0; i < 3; ++i) Xc[i] = T[i * 3] * X[0] + T[i * 3 + 1] * X[1] + T[i * 3 + 2] * X[2] + T[9 + i];
}

// computeActiveErrors + activeRobustChi2
template <class Exec> IMU_HD inline double compute_errors(const Dev& D, Exec& ex, double deltaMono, double deltaInertial) {
    ex.tag(0);
    return ex.sum([&](int tid) {
        double v = 0;
        for (int e = tid; e < D.nE; e += NT) {
            double Xc[3];
            mono_camera_point(D, e, Xc);
            const float* c = D.cam + 4 * (size_t)D.eKf[e];
            const double e0 = D.obs[2 * (size_t)e] - ((double)c[0] * Xc[0] / Xc[2] + (double)c[2]);
            const double e1 = D.obs[2 * (size_t)e + 1] - ((double)c[1] * Xc[1] / Xc[2] + (double)c[3]);
            D.errM[2 * (size_t)e] = e0; D.errM[2 * (size_t)e + 1] = e1;
            double r0, r1;
            huber((double)D.invSigma2[e] * (e0 * e0 + e1 * e1), deltaMono, deltaMono * deltaMono, r0, r1);
            v += r0;
        }
        for (int i = tid; i < D.nI; i += NT) {
            double S[36];
            edge_states(D, i, S);
            double* e9 = D.errI + 9 * (size_t)i;
            edge_inertial_dev(D.preint + (size_t)P_SIZE * i, S, e9, nullptr);
            double* eg = D.errG + 3 * (size_t)i; double* ea = D.errA + 3 * (size_t)i;
            const double* k1 = D.kfState + 21 * (size_t)D.ieKf1[i];
            const double* k2 = D.kfState + 21 * (size_t)D.ieKf2[i];
            for (int k = 0; k < 3; ++k) { eg[k] = k2[15 + k] - k1[15 + k]; ea[k] = k2[18 + k] - k1[18 + k]; }
            const double c = quad<9>(D.info9 + 81 * (size_t)i, e9);
            if (D.ieRobust[i]) { double r0, r1; huber(c, deltaInertial, deltaInertial * deltaInertial, r0, r1); v += r0; } else v += c;
            v += quad<3>(D.infoG + 9 * (size_t)i, eg) + quad<3>(D.infoA + 9 * (size_t)i, ea);
        }
        return v;
    });
}

// BlockSolver::buildSystem: linearizeOplus + constructQuadraticForm of every edge
template <class Exec> IMU_HD inline void build_system(const Dev& D, Exec& ex, double deltaMono, double deltaInertial) {
    ex.tag(1);
    const int n = 15 * D.nOpt;
    const double *Rcb = D.extr, *Rbc = D.extr + 12, *tbc = D.extr + 21;
    ex.par([&](int tid) {
        for (size_t i = tid; i < (size_t)n * n; i += NT) D.H[i] = 0.0;
        for (int i = tid; i < n; i += NT) D.b[i] = 0.0;
        // EdgeMono::linearizeOplus (src/G2oTypes.cc:349-373) + the robust weights of constructQuadraticForm
        for (int e = tid; e < D.nE; e += NT) {
            const double* T = D.kfTcw + 12 * (size_t)D.eKf[e];
            double Xc[3];
            mono_camera_point(D, e, Xc);
            double J[EJ];
            double* A = J; double* B = J + 6;
            mono_jacobians(T, Rcb, Rbc, tbc, D.cam + 4 * (size_t)D.eKf[e], Xc, A, B);
            const double e0 = D.errM[2 * (size_t)e], e1 = D.errM[2 * (size_t)e + 1], om = (double)D.invSigma2[e];
            double r0, r1;
            huber(om * (e0 * e0 + e1 * e1), deltaMono, deltaMono * deltaMono, r0, r1);
            const double w = r1 * om;
            J[18] = w; J[19] = -om * e0 * r1; J[20] = -om * e1 * r1; J[21] = 0.0; J[22] = 0.0; J[23] = 0.0;
            stvec<6>(D.ejac + (size_t)EJ * e, J);
            if (D.eKf[e] < D.nOpt) {
                double We[WS];
                for (int a = 0; a < 6; ++a) for (int k = 0; k < 3; ++k) We[a * 3 + k] = w * (B[a] * A[k] + B[6 + a] * A[3 + k]);
                We[18] = 0.0; We[19] = 0.0;
                stvec<5>(D.W + WS * (size_t)e, We);
            }
        }
        // EdgeInertial::linearizeOplus (one thread per edge; the products with the information matrix are spread over the CTA below)
        for (int i = tid; i < D.nI; i += NT) {
            double S[36], e9[9];
            edge_states(D, i, S);
            edge_inertial_dev(D.preint + (size_t)P_SIZE * i, S, e9, D.Jin + 216 * (size_t)i);
            double w = 1.0;
            if (D.ieRobust[i]) { double r0; huber(quad<9>(D.info9 + 81 * (size_t)i, D.errI + 9 * (size_t)i), deltaInertial, deltaInertial * deltaInertial, r0, w); }
            D.win[i] = w;
        }
    });
    ex.par([&](int tid) {
        // inertial edges: Omega J (one task per edge and Jacobian column) and Omega e
        for (int t = tid; t < D.nI * 25; t += NT) {
            const int i = t / 25, c = t % 25;
            const double* Om = D.info9 + 81 * (size_t)i;
            if (c < 24) {
                const double* J = D.Jin + 216 * (size_t)i;
                for (int r = 0; r < 9; ++r) { double sacc = 0; for (int k = 0; k < 9; ++k) sacc += Om[r * 9 + k] * J[k * 24 + c]; D.OJ[216 * (size_t)i + r * 24 + c] = sacc; }
            } else {
                const double* er = D.errI + 9 * (size_t)i;
                for (int r = 0; r < 9; ++r) { double sacc = 0; for (int k = 0; k < 9; ++k) sacc += Om[r * 9 + k] * er[k]; D.Oe[9 * (size_t)i + r] = sacc; }
            }
        }
        // points: Hll, bl in the order of the point's edge list
        for (int p = tid; p < D.nL; p += NT) {
            double h[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, b3[3] = {0, 0, 0};
            for (int j = D.ptStart[p]; j < D.ptStart[p + 1]; ++j) {
                double J[8], Jw[8];                              // record entries 0 .. 7 (A) and 16 .. 23 (w r0 r1 at 18 .. 20)
                ldvec<2>(D.ejac + (size_t)EJ * D.ptEdges[j], J);
                ldvec<2>(D.ejac + (size_t)EJ * D.ptEdges[j] + 16, Jw);
                const double w = Jw[2], r0 = Jw[3], r1 = Jw[4];
                for (int a = 0; a < 3; ++a) {
                    b3[a] += J[a] * r0 + J[3 + a] * r1;
                    for (int c = 0; c < 3; ++c) h[a * 3 + c] += w * (J[a] * J[c] + J[3 + a] * J[3 + c]);
                }
            }
            for (int k = 0; k < 9; ++k) D.Hll[9 * (size_t)p + k] = h[k];
            for (int k = 0; k < 3; ++k) D.bl[3 * (size_t)p + k] = b3[k];
        }
        // keyframes, step 1: partial sums of the 6 x 6 pose block (lower triangle) and of its b over a slice of the keyframe's edge list
        for (int t = tid; t < D.nOpt * SL; t += NT) {
            const int k = t / SL, sl = t % SL;
            double acc[27];
            for (int q = 0; q < 27; ++q) acc[q] = 0.0;
            for (int j = D.kfStart[k] + sl; j < D.kfStart[k + 1]; j += SL) {
                double Jv[20];                                  // record entries 4 .. 23: A[4], A[5] | B 12 | w r0 r1 | pad
                ldvec<5>(D.ejac + (size_t)EJ * D.kfEdges[j] + 4, Jv);
                const double* B = Jv + 2;
                const double w = Jv[14], r0 = Jv[15], r1 = Jv[16];
#pragma unroll
                for (int a = 0; a < 6; ++a)
#pragma unroll
                    for (int c = 0; c <= a; ++c) acc[a * (a + 1) / 2 + c] += w * (B[a] * B[c] + B[6 + a] * B[6 + c]);
#pragma unroll
                for (int a = 0; a < 6; ++a) acc[21 + a] += B[a] * r0 + B[6 + a] * r1;
            }
            for (int q = 0; q < 27; ++q) D.part[27 * (size_t)t + q] = acc[q];
        }
    });
    ex.par([&](int tid) {
        // inertial edges: the local 30 x 30 Hessian over (keyframe 1's 15 | keyframe 2's 15) and its b, one task per row; EdgeGyroRW / EdgeAccRW
        // (error = b2 - b1, Jacobians -I / +I, include/G2oTypes.h:635-700) add to the bias rows
        for (int t = tid; t < D.nI * 30; t += NT) {
            const int i = t / 30, a = t % 30;
            const double* J = D.Jin + 216 * (size_t)i;
            const double* OJ = D.OJ + 216 * (size_t)i;
            const double w = D.win[i];
            double* He = D.He + 900 * (size_t)i + 30 * a;
            double bacc = 0;
            for (int c = 0; c < 30; ++c) He[c] = 0.0;
            if (a < 24) {
                for (int r = 0; r < 9; ++r) bacc += J[r * 24 + a] * D.Oe[9 * (size_t)i + r];
                bacc = -w * bacc;
                for (int c = 0; c < 24; ++c) { double h = 0; for (int r = 0; r < 9; ++r) h += J[r * 24 + a] * OJ[r * 24 + c]; He[c] = w * h; }
            }
            const int blk = (a >= 9 && a < 15) ? (a - 9) / 3 : (a >= 24 ? (a - 24) / 3 : -1);      // 0 gyro, 1 acc
            if (blk >= 0) {
                const bool first = a < 15;                                                         // vertex 0 (Jacobian -I) or vertex 1 (+I)
                const int q = (a - (first ? 9 : 24)) % 3;
                const double* Inf = blk == 0 ? D.infoG + 9 * (size_t)i : D.infoA + 9 * (size_t)i;
                const double* e3 = blk == 0 ? D.errG + 3 * (size_t)i : D.errA + 3 * (size_t)i;
                const int g1 = blk == 0 ? 9 : 12, g2 = blk == 0 ? 24 : 27;
                double sacc = 0;
                for (int c = 0; c < 3; ++c) sacc += Inf[q * 3 + c] * e3[c];
                if (first) {
                    bacc += sacc;
                    for (int c = 0; c < 3; ++c) { He[g1 + c] += Inf[q * 3 + c]; He[g2 + c] -= Inf[q * 3 + c]; }
                } else {
                    bacc -= sacc;
                    for (int c = 0; c < 3; ++c) { He[g2 + c] += Inf[q * 3 + c]; He[g1 + c] -= Inf[c * 3 + q]; }
                }
            }
            D.be[30 * (size_t)i + a] = bacc;
        }
        // step 2: the slices in order; the block is mirrored
        for (int t = tid; t < D.nOpt * 27; t += NT) {
            const int k = t / 27, q = t % 27;
            double acc = 0;
            for (int sl = 0; sl < SL; ++sl) acc += D.part[27 * ((size_t)k * SL + sl) + q];
            if (q < 21) {
                int a = 0, r = q;
                while (r > a) { r -= a + 1; ++a; }
                D.H[(size_t)(15 * k + a) * n + 15 * k + r] = acc; D.H[(size_t)(15 * k + r) * n + 15 * k + a] = acc;
            } else D.b[15 * k + q - 21] = acc;
        }
    });
    ex.par([&](int tid) {
        // inertial edges into H, b: one task per row of the reduced system, edges in index order
        for (int g = tid; g < n; g += NT) {
            const int k = g / 15, r = g % 15;
            for (int i = 0; i < D.nI; ++i) {
                int lr;
                if (D.ieKf1[i] == k) lr = r; else if (D.ieKf2[i] == k) lr = 15 + r; else continue;
                const double* He = D.He + 900 * (size_t)i;
                for (int lc = 0; lc < 30; ++lc) {
                    const int kc = lc < 15 ? D.ieKf1[i] : D.ieKf2[i];
                    if (kc >= D.nOpt) continue;
                    D.H[(size_t)g * n + 15 * kc + lc % 15] += He[lr * 30 + lc];
                }
                D.b[g] += D.be[30 * (size_t)i + lr];
            }
        }
    });
}

// dense blocked LDL^T of Hs (lower triangle) + the solve of Hs x = bs; false on an exactly zero pivot (x untouched)
template <class Exec> IMU_HD inline bool ldlt_solve(const Dev& D, Exec& ex) {
    const int n = 15 * D.nOpt;
    double* A = D.Hs; double* y = D.bs;
    double* P = ex.panel();             // (n - LW) x LW doubles of CTA-shared storage
    for (int k0 = 0; k0 < n; k0 += LW) {
        // uniform: factor the diagonal block, forward-substitute the block's right-hand side
        double L11[LW * LW], d[LW], z[LW];
        bool bad = false;
        for (int j = 0; j < LW; ++j) {
            double dj = A[(size_t)(k0 + j) * n + k0 + j];
            for (int k = 0; k < j; ++k) dj -= L11[j * LW + k] * L11[j * LW + k] * d[k];
            d[j] = dj;
            if (dj == 0.0) { bad = true; break; }
            for (int i = j + 1; i < LW; ++i) {
                double v = A[(size_t)(k0 + i) * n + k0 + j];
                for (int k = 0; k < j; ++k) v -= L11[i * LW + k] * L11[j * LW + k] * d[k];
                L11[i * LW + j] = v / dj;
            }
        }
        if (bad) return false;
        for (int c = 0; c < LW; ++c) { double v = y[k0 + c]; for (int j = 0; j < c; ++j) v -= L11[c * LW + j] * z[j]; z[c] = v; }
        double dinv[LW];
        for (int c = 0; c < LW; ++c) dinv[c] = 1.0 / d[c];
        ex.par([&](int tid) {
            // panel: X = A21 L11^-T (kept unscaled in place), y2 -= (X D^-1) z
            for (int i = k0 + LW + tid; i < n; i += NT) {
                double* row = A + (size_t)i * n + k0;
                double xr[LW], s = 0;
                for (int c = 0; c < LW; ++c) {
                    double v = row[c];
                    for (int j = 0; j < c; ++j) v -= xr[j] * L11[c * LW + j];
                    xr[c] = v;
                    s += v * dinv[c] * z[c];
                }
                for (int c = 0; c < LW; ++c) { row[c] = xr[c]; P[(i - k0 - LW) * LW + c] = xr[c]; }      // in place for the back-substitution, and in the CTA's panel buffer
                y[i] -= s;
            }
        });
        const int r0 = k0 + LW, m = n - r0;
        ex.par([&](int tid) {
                // (every thread has left the uniform section above: only now may the block and its right-hand side be overwritten)
                if (tid == 0) {
                    for (int c = 0; c < LW; ++c) {
                        y[k0 + c] = z[c]; D.dvec[k0 + c] = d[c];
                        for (int j = 0; j < c; ++j) A[(size_t)(k0 + c) * n + k0 + j] = L11[c * LW + j];      // the block keeps the scaled L11
                    }
                }
                // trailing update of the lower triangle: A22[i][j] -= sum_c X[i][c] X[j][c] / d[c]
                for (int idx = tid; idx < m * (m + 1) / 2; idx += NT) {
                    int i = (int)((sqrt(8.0 * idx + 1.0) - 1.0) * 0.5);
                    while ((i + 1) * (i + 2) / 2 <= idx) ++i;
                    while (i * (i + 1) / 2 > idx) --i;
                    const int j = idx - i * (i + 1) / 2;
                    const double* xi = P + i * LW;      // the panel rows come from shared memory (in A they are n doubles apart: 32 lanes = 32 lines per load)
                    const double* xj = P + j * LW;
                    double s = 0;
                    for (int c = 0; c < LW; ++c) s += xi[c] * (xj[c] * dinv[c]);
                    A[(size_t)(r0 + i) * n + r0 + j] -= s;
                }
            });
    }
    ex.par([&](int tid) { for (int i = tid; i < n; i += NT) y[i] /= D.dvec[i]; });
    for (int k0 = n - LW; k0 >= 0; k0 -= LW) {
        double xs[LW];
        for (int c = LW - 1; c >= 0; --c) {
            double v = y[k0 + c];
            for (int j = c + 1; j < LW; ++j) v -= A[(size_t)(k0 + j) * n + k0 + c] * xs[j];
            xs[c] = v;
        }
        ex.par([&](int tid) {
            for (int j = tid; j < k0; j += NT) {
                double s = 0;
                for (int c = 0; c < LW; ++c) s += A[(size_t)(k0 + c) * n + j] * xs[c];
                y[j] -= s / D.dvec[j];
            }
            if (tid < LW) D.x[k0 + tid] = xs[tid];
        });
    }
    return true;
}

// BlockSolver::solve (Schur branch) with lambda folded into the diagonals of copies (setLambda / restoreDiagonal)
template <class Exec> IMU_HD inline bool solve_system(const Dev& D, Exec& ex, double lambda) {
    ex.tag(2);
    const int n = 15 * D.nOpt, nO = D.nOpt;
    ex.par([&](int tid) {
        for (int p = tid; p < D.nL; p += NT) {
            double Dm[9];
            for (int k = 0; k < 9; ++k) Dm[k] = D.Hll[9 * (size_t)p + k];
            Dm[0] += lambda; Dm[4] += lambda; Dm[8] += lambda;
            double* Di = D.Dinv + 9 * (size_t)p;
            inv3_cof(Dm, Di);
            const double* b3 = D.bl + 3 * (size_t)p;
            for (int a = 0; a < 3; ++a) D.db[3 * (size_t)p + a] = Di[a * 3] * b3[0] + Di[a * 3 + 1] * b3[1] + Di[a * 3 + 2] * b3[2];
        }
        for (int i = tid; i < n * n; i += NT) D.Hs[i] = D.H[i] + ((i / n == i % n) ? lambda : 0.0);
        for (int i = tid; i < n; i += NT) D.bs[i] = D.b[i];
    });
    ex.par([&](int tid) {
        for (int e = tid; e < D.nE; e += NT) {
            if (D.eKf[e] >= nO) continue;
            double We[WS], Ye[WS];
            ldvec<5>(D.W + WS * (size_t)e, We);
            const double* Di = D.Dinv + 9 * (size_t)D.ePt[e];
            for (int a = 0; a < 6; ++a) for (int c = 0; c < 3; ++c) Ye[a * 3 + c] = We[a * 3] * Di[c] + We[a * 3 + 1] * Di[3 + c] + We[a * 3 + 2] * Di[6 + c];
            Ye[18] = 0.0; Ye[19] = 0.0;
            stvec<5>(D.Y + WS * (size_t)e, Ye);
        }
    });
    const int nPairs = nO * (nO + 1) / 2;
    ex.tag(3);
    ex.par([&](int tid) {
        // Hschur, step 1: one task per (keyframe pair i1 <= i2, slice of keyframe i1's edge list): partial 6 x 6 blocks
        for (int t = tid; t < nPairs * SL; t += NT) {
            int pidx = t / SL;
            const int sl = t % SL;
            int i1 = 0;
            while (pidx >= nO - i1) { pidx -= nO - i1; ++i1; }
            const int i2 = i1 + pidx;
            double acc[36];
            for (int k = 0; k < 36; ++k) acc[k] = 0.0;
            // the indices of the next pair are fetched before the blocks of the current one (two dependent look-ups hide behind the block loads)
            int j = D.kfStart[i1] + sl;
            const int jend = D.kfStart[i1 + 1];
            int e1n = -1, e2n = -1;
            if (j < jend) { e1n = D.kfEdges[j]; e2n = i1 == i2 ? e1n : D.pk[(size_t)D.ePt[e1n] * nO + i2]; }
            while (j < jend) {
                const int e1 = e1n, e2 = e2n;
                j += SL;
                if (j < jend) { e1n = D.kfEdges[j]; e2n = i1 == i2 ? e1n : D.pk[(size_t)D.ePt[e1n] * nO + i2]; }
                if (e2 < 0) continue;
                // block += Y1 W2^T, with W2 consumed vector by vector (element m = 3 c + k of W2 meets column k of Y1): Y1, one vector of W2 and the
                // 36 accumulators stay within the 128 registers a thread of a 512-thread CTA has
                double Y1[WS];
                ldvec<5>(D.Y + WS * (size_t)e1, Y1);
                const double* W2p = D.W + WS * (size_t)e2;
#pragma unroll
                for (int v = 0; v < 5; ++v) {
                    double w4[4];
                    ldvec<1>(W2p + 4 * v, w4);
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int m = 4 * v + u;
                        if (m < 18) {
#pragma unroll
                            for (int a = 0; a < 6; ++a) acc[a * 6 + m / 3] += Y1[a * 3 + m % 3] * w4[u];
                        }
                    }
                }
            }
            double* out = D.part + 36 * (size_t)t;
            for (int k = 0; k < 36; ++k) out[k] = acc[k];
        }
        // bschur, step 1: (keyframe, slice)
        for (int t = tid; t < nO * SL; t += NT) {
            const int k = t / SL, sl = t % SL;
            double acc[6] = {0, 0, 0, 0, 0, 0};
            for (int j = D.kfStart[k] + sl; j < D.kfStart[k + 1]; j += SL) {
                const int e = D.kfEdges[j];
                double We[WS];
                ldvec<5>(D.W + WS * (size_t)e, We);
                const double* d3 = D.db + 3 * (size_t)D.ePt[e];
                for (int a = 0; a < 6; ++a) acc[a] += We[a * 3] * d3[0] + We[a * 3 + 1] * d3[1] + We[a * 3 + 2] * d3[2];
            }
            for (int a = 0; a < 6; ++a) D.partb[6 * (size_t)t + a] = acc[a];
        }
    });
    ex.par([&](int tid) {
        // step 2: the slices in order
        for (int t = tid; t < nPairs * 36; t += NT) {
            int pidx = t / 36;
            const int q = t % 36, a = q / 6, c = q % 6;
            const double* src = D.part + 36 * (size_t)pidx * SL + q;
            double acc = 0;
            for (int sl = 0; sl < SL; ++sl) acc += src[36 * sl];
            int i1 = 0;
            while (pidx >= nO - i1) { pidx -= nO - i1; ++i1; }
            const int i2 = i1 + pidx;
            D.Hs[(size_t)(15 * i1 + a) * n + 15 * i2 + c] -= acc;
            if (i1 != i2) D.Hs[(size_t)(15 * i2 + c) * n + 15 * i1 + a] -= acc;
        }
        for (int t = tid; t < nO * 6; t += NT) {
            const int k = t / 6, a = t % 6;
            double acc = 0;
            for (int sl = 0; sl < SL; ++sl) acc += D.partb[6 * ((size_t)k * SL + sl) + a];
            D.bs[15 * k + a] -= acc;
        }
    });
    ex.tag(4);
    if (n > 0 && !ldlt_solve(D, ex)) return false;
    ex.tag(5);
    ex.par([&](int tid) {
        // landmarks: xl = Dinv (bl - Hpl^T xp)
        for (int p = tid; p < D.nL; p += NT) {
            double cl[3] = {D.bl[3 * (size_t)p], D.bl[3 * (size_t)p + 1], D.bl[3 * (size_t)p + 2]};
            for (int j = D.ptStart[p]; j < D.ptStart[p + 1]; ++j) {
                const int e = D.ptEdges[j];
                if (D.eKf[e] >= nO) continue;
                double We[WS];
                ldvec<5>(D.W + WS * (size_t)e, We);
                const double* xp = D.x + 15 * (size_t)D.eKf[e];
                for (int c = 0; c < 3; ++c) for (int a = 0; a < 6; ++a) cl[c] -= We[a * 3 + c] * xp[a];
            }
            const double* Di = D.Dinv + 9 * (size_t)p;
            for (int a = 0; a < 3; ++a) D.x[n + 3 * (size_t)p + a] = Di[a * 3] * cl[0] + Di[a * 3 + 1] * cl[1] + Di[a * 3 + 2] * cl[2];
        }
    });
    return true;
}

// push() + SparseOptimizer::update: VertexPose::oplusImpl = ImuCamPose::Update (src/G2oTypes.cc:192-221), additive velocity / biases / points
template <class Exec> IMU_HD inline void push_and_update(const Dev& D, Exec& ex) {
    ex.tag(6);
    const int n = 15 * D.nOpt;
    const double *Rcb = D.extr, *tcb = D.extr + 9;
    ex.par([&](int tid) {
        for (int k = tid; k < D.nOpt; k += NT) {
            double* st = D.kfState + 21 * (size_t)k; double* T = D.kfTcw + 12 * (size_t)k;
            for (int i = 0; i < 21; ++i) D.kfBk[21 * (size_t)k + i] = st[i];
            for (int i = 0; i < 12; ++i) D.tcwBk[12 * (size_t)k + i] = T[i];
            const double* u = D.x + 15 * (size_t)k;
            double t3[3], E[9], Rn[9];
            m3vec(st, u + 3, t3);
            for (int i = 0; i < 3; ++i) st[9 + i] += t3[i];
            exp_so3_d(u, E);
            m3mul(st, E, Rn);
            for (int i = 0; i < 9; ++i) st[i] = Rn[i];
            // (ImuCamPose::Update's every-third-update `NormalizeRotation(Rwb);`, src/G2oTypes.cc:202-208, discards the function's return value -- the
            //  template of include/G2oTypes.h:67-71 returns the normalised matrix and leaves its argument alone -- so the reference never renormalises Rwb)
            double tbw[3];
            for (int i = 0; i < 3; ++i) tbw[i] = -(st[i] * st[9] + st[3 + i] * st[10] + st[6 + i] * st[11]);
            for (int i = 0; i < 3; ++i) {
                for (int j = 0; j < 3; ++j) T[i * 3 + j] = Rcb[i * 3] * st[j * 3] + Rcb[i * 3 + 1] * st[j * 3 + 1] + Rcb[i * 3 + 2] * st[j * 3 + 2];
                T[9 + i] = Rcb[i * 3] * tbw[0] + Rcb[i * 3 + 1] * tbw[1] + Rcb[i * 3 + 2] * tbw[2] + tcb[i];
            }
            for (int i = 0; i < 3; ++i) { st[12 + i] += u[6 + i]; st[15 + i] += u[9 + i]; st[18 + i] += u[12 + i]; }
        }
        for (size_t i = tid; i < (size_t)3 * D.nL; i += NT) { D.ptsBk[i] = D.pts[i]; D.pts[i] += D.x[n + i]; }
    });
}
template <class Exec> IMU_HD inline void pop(const Dev& D, Exec& ex) {
    ex.tag(6);
    ex.par([&](int tid) {
        for (int i = tid; i < 21 * D.nOpt; i += NT) D.kfState[i] = D.kfBk[i];
        for (int i = tid; i < 12 * D.nOpt; i += NT) D.kfTcw[i] = D.tcwBk[i];
        for (size_t i = tid; i < (size_t)3 * D.nL; i += NT) D.pts[i] = D.ptsBk[i];
    });
}

// initializeOptimization(); computeActiveErrors(); err; optimize(opt_it); err_end; the EdgeMono chi2 / depth test; the FAIL test
template <class Exec> IMU_HD inline void run(const Dev& D, Exec& ex) {
    const int n = 15 * D.nOpt, nO = D.nOpt;
    const double deltaMono = (double)sqrtf(5.991f);      // const float thHuberMono = sqrt(5.991)
    const double deltaInertial = sqrt(16.92);
    ex.tag(7);
    ex.par([&](int tid) {
        for (int i = tid; i < D.nI; i += NT) {
            double* I9 = D.info9 + 81 * (size_t)i;
            information_matrices(D.preint + (size_t)P_SIZE * i, I9, D.infoG + 9 * (size_t)i, D.infoA + 9 * (size_t)i);
            for (int k = 0; k < 81; ++k) I9[k] *= D.ieInfoScale[i];      // vei[i]->setInformation(information() * 1e-2), :2641
        }
        for (size_t i = tid; i < (size_t)D.nL * nO; i += NT) D.pk[i] = -1;
        for (int i = tid; i < n + 3 * D.nL; i += NT) D.x[i] = 0.0;
    });
    ex.par([&](int tid) {
        for (int e = tid; e < D.nE; e += NT) if (D.eKf[e] < nO) D.pk[(size_t)D.ePt[e] * nO + D.eKf[e]] = e;
    });
    double chiNow = compute_errors(D, ex, deltaMono, deltaInertial);      // the robust chi2 of the errors the edges hold for the current estimate
    const float err = (float)chiNow;

    Levenberg lm;
    int cj = 0, trials = 0;
    bool ok = true;
    for (int it = 0; it < D.iterations && ok; ++it) {
        // solve() starts with computeActiveErrors(): the estimate has not changed since the last evaluation (the optimize() call itself, or the
        // accepted trial that ended the previous iteration), so the edges already hold exactly these errors
        double currentChi = chiNow;
        const double iniChi = currentChi;
        build_system(D, ex, deltaMono, deltaInertial);
        if (it == 0) {
            double maxDiag = 0;
            if (!(D.lambdaInit > 0))
                maxDiag = ex.max([&](int tid) {
                    double m = 0;
                    for (int i = tid; i < n; i += NT) m = fmax(m, fabs(D.H[(size_t)i * n + i]));
                    for (int i = tid; i < 3 * D.nL; i += NT) m = fmax(m, fabs(D.Hll[9 * (size_t)(i / 3) + 4 * (i % 3)]));
                    return m;
                });
            lm.start(D.lambdaInit, maxDiag);
        }
        double rho = 0;
        int qmax = 0;
        do {
            const bool ok2 = solve_system(D, ex, lm.lambda);
            push_and_update(D, ex);
            const double tempChi = compute_errors(D, ex, deltaMono, deltaInertial);
            ex.tag(7);
            const double scale = ex.sum([&](int tid) {
                double s = 0;
                for (int j = tid; j < n; j += NT) s += D.x[j] * (lm.lambda * D.x[j] + D.b[j]);
                for (int j = tid; j < 3 * D.nL; j += NT) s += D.x[n + j] * (lm.lambda * D.x[n + j] + D.bl[j]);
                return s;
            });
            if (lm.trial(currentChi, tempChi, scale, ok2, rho)) chiNow = currentChi;
            else pop(D, ex);
            ++qmax; ++trials;
        } while (rho < 0 && qmax < Levenberg::maxTrials);
        ++cj;
        ok = lm.iteration_done(qmax, rho, iniChi, currentChi);
    }
    ex.tag(7);
    // err_end = activeRobustChi2() of the errors the edges hold (those of a rejected last trial included)
    const float errEnd = (float)ex.sum([&](int tid) {
        double v = 0;
        for (int e = tid; e < D.nE; e += NT) {
            const double e0 = D.errM[2 * (size_t)e], e1 = D.errM[2 * (size_t)e + 1];
            double r0, r1;
            huber((double)D.invSigma2[e] * (e0 * e0 + e1 * e1), deltaMono, deltaMono * deltaMono, r0, r1);
            v += r0;
        }
        for (int i = tid; i < D.nI; i += NT) {
            const double c = quad<9>(D.info9 + 81 * (size_t)i, D.errI + 9 * (size_t)i);
            if (D.ieRobust[i]) { double r0, r1; huber(c, deltaInertial, deltaInertial * deltaInertial, r0, r1); v += r0; } else v += c;
            v += quad<3>(D.infoG + 9 * (size_t)i, D.errG + 3 * (size_t)i) + quad<3>(D.infoA + 9 * (size_t)i, D.errA + 3 * (size_t)i);
        }
        return v;
    });
    const bool failed = (2 * err < errEnd || err != err || errEnd != errEnd) && !D.bLarge;      // :2884
    ex.par([&](int tid) {
        const float chi2Mono2 = 5.991f;
        for (int e = tid; e < D.nE; e += NT) {
            const double e0 = D.errM[2 * (size_t)e], e1 = D.errM[2 * (size_t)e + 1];
            const double c2 = (double)D.invSigma2[e] * (e0 * e0 + e1 * e1);
            D.chi2[e] = c2;
            const bool bClose = D.trackDepth[D.ePt[e]] < 10.f;
            const double* T = D.kfTcw + 12 * (size_t)D.eKf[e];
            const double* X = D.pts + 3 * (size_t)D.ePt[e];
            const bool depthPos = (T[6] * X[0] + T[7] * X[1] + T[8] * X[2] + T[11]) > 0.0;
            D.erase[e] = ((c2 > chi2Mono2 && !bClose) || (c2 > 1.5f * chi2Mono2 && bClose) || !depthPos) ? 1 : 0;
        }
        for (int i = tid; i < 21 * D.nKF; i += NT) D.outState[i] = D.kfState[i];
        for (int i = tid; i < 12 * D.nKF; i += NT) D.outTcw[i] = D.kfTcw[i];
        for (size_t i = tid; i < (size_t)3 * D.nL; i += NT) D.outPts[i] = D.pts[i];
        if (tid == 0) {
            D.stats[0] = err; D.stats[1] = errEnd; D.stats[2] = failed ? 1.0 : 0.0; D.stats[3] = lm.lambda; D.stats[4] = trials; D.stats[5] = cj;
            D.stats[6] = 0; D.stats[7] = 0;
        }
    });
}

}  // namespace liba
