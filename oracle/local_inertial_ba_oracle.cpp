// TEST INFRASTRUCTURE ONLY (see oracle_common.h).  CPU restatement of the numeric core of
// void Optimizer::LocalInertialBA(KeyFrame*, bool*, Map*, int&, int&, int&, int&, bool bLarge, bool bRecInit)
// (reference src/Optimizer.cc:2383-2958; SURVEY.md 8f rank 1), monocular-inertial branch, between the graph set-up and the write-back:
//   vertices  VertexPose (ImuCamPose, 6) + VertexVelocity / VertexGyroBias / VertexAccBias (3 each) per keyframe of the temporal window
//             (:2524-2548), fixed keyframes (:2562-2586), VertexSBAPointXYZ marginalised (:2710-2717)
//   edges     EdgeInertial (6 vertices; Huber sqrt(16.92) + information * 1e-2 on the link to the fixed keyframe, Huber on all with bRecInit)
//             + EdgeGyroRW + EdgeAccRW per consecutive pair (:2593-2656), EdgeMono per observation with Huber sqrt(5.991) (:2737-2763)
//   solve     optimizer.initializeOptimization(); computeActiveErrors(); err = activeRobustChi2(); optimize(opt_it); err_end (:2835-2839)
//             = g2o Levenberg-Marquardt with setUserLambdaInit(1e0 | 1e-2), BlockSolverX + Schur complement over the points,
//             LinearSolverEigen on the reduced system (same g2o semantics as lba_oracle.cpp, which cites the g2o lines)
//   after     chi2 / depth test of every EdgeMono (:2848-2862), the FAIL test (:2884-2888)
// The graph walk that collects keyframes, points and observations (:2385-2478) is host code of the caller; arrays arrive flattened.
// ImuCamPose keeps the keyframe's own camera pose (float Tcw cast to double, src/G2oTypes.cc:46-47) until its first Update(), after which
// Rcw / tcw derive from the body pose (:213-221): both are inputs here.  BaseMultiEdge / BaseBinaryEdge::constructQuadraticForm with a
// robust kernel scale information and b by rho'(chi2) (g2o/core/base_multi_edge.hpp:41-54, base_edge.h:96-102).
// PARITY UNPINNED by the reference (g2o / G2oTypes need Eigen): pinned by a dense Levenberg step built from numerical derivatives of the
// whitened residuals (tests/test_local_inertial_ba_cpu.py); the edge functions are those of inertial_oracle.cpp (pinned there).
#include "oracle_common.h"

#include <cfloat>
#include <cstring>
#include <vector>

extern "C" {
void orbo_imu_information(const float* P, double* Info9, double* InfoG3, double* InfoA3);
void orbo_imu_edge_inertial(const float* P, const double* Rwb1, const double* twb1, const double* v1, const double* bg, const double* ba,
                            const double* Rwb2, const double* twb2, const double* v2, double* err, double* J);
void orbo_imu_pose_update(double* Rwb, double* twb, const double* pu);
void orbo_so3(int what, const double* in, double* out);
}

namespace orbo {
namespace liba {

enum { P_SIZE = 292 };

struct KF {
    double Rwb[9], twb[3], v[3], bg[3], ba[3];
    double Rcw[9], tcw[3];
    int its;
};

static inline void mv3(const double* A, const double* x, double* o) {
    for (int i = 0; i < 3; ++i) o[i] = A[i * 3] * x[0] + A[i * 3 + 1] * x[1] + A[i * 3 + 2] * x[2];
}

static bool inv3(const double* m, double* o) {
    const double c00 = m[4] * m[8] - m[5] * m[7], c10 = m[5] * m[6] - m[3] * m[8], c20 = m[3] * m[7] - m[4] * m[6];
    const double det = m[0] * c00 + m[1] * c10 + m[2] * c20;
    const double id = 1.0 / det;
    o[0] = c00 * id; o[1] = (m[2] * m[7] - m[1] * m[8]) * id; o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
    o[3] = c10 * id; o[4] = (m[0] * m[8] - m[2] * m[6]) * id; o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
    o[6] = c20 * id; o[7] = (m[1] * m[6] - m[0] * m[7]) * id; o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
    return true;
}

// dense LDL^T without pivoting; false on an exactly zero pivot (SimplicialLDLT's failure mode)
static bool ldlt_solve(std::vector<double>& A, int n, const double* b, double* x) {
    for (int k = 0; k < n; ++k) {
        double d = A[(size_t)k * n + k];
        for (int j = 0; j < k; ++j) d -= A[(size_t)k * n + j] * A[(size_t)k * n + j] * A[(size_t)j * n + j];
        A[(size_t)k * n + k] = d;
        if (d == 0.0) return false;
        for (int i = k + 1; i < n; ++i) {
            double s = A[(size_t)i * n + k];
            for (int j = 0; j < k; ++j) s -= A[(size_t)i * n + j] * A[(size_t)k * n + j] * A[(size_t)j * n + j];
            A[(size_t)i * n + k] = s / d;
        }
    }
    std::vector<double> y(n);
    for (int i = 0; i < n; ++i) { double s = b[i]; for (int j = 0; j < i; ++j) s -= A[(size_t)i * n + j] * y[j]; y[i] = s; }
    for (int i = 0; i < n; ++i) y[i] /= A[(size_t)i * n + i];
    for (int i = n - 1; i >= 0; --i) { double s = y[i]; for (int j = i + 1; j < n; ++j) s -= A[(size_t)j * n + i] * x[j]; x[i] = s; }
    return true;
}

struct Problem {
    int nKF, nOpt, nI, nL, nE;
    std::vector<KF> kf, kfBk;
    std::vector<double> pts, ptsBk;
    const float* cam;                    // 4 per keyframe
    const double *Rcb, *tcb, *Rbc, *tbc;
    const int *ieKf1, *ieKf2;
    const float* preint;
    const uint8_t* ieRobust;
    std::vector<double> info9, infoG, infoA;   // per inertial edge (info9 already scaled)
    const int *ePt, *eKf;
    const double* obs;
    const float* invSigma2;
    double deltaMono, deltaInertial;
    // errors kept by the edges
    std::vector<double> errM, errI, errG, errA;
    // linear system: reduced matrix index of keyframe k = 15 k (pose 6 | v 3 | bg 3 | ba 3), k < nOpt
    std::vector<double> H, b, Hll, bl, W, x, Dinv;

    static void huber(double e2, double delta, double* rho) {
        const double dsqr = delta * delta;
        if (e2 <= dsqr) { rho[0] = e2; rho[1] = 1.; rho[2] = 0.; }
        else { const double s = std::sqrt(e2); rho[0] = 2 * s * delta - dsqr; rho[1] = delta / s; rho[2] = -0.5 * rho[1] / e2; }
    }
    void mono_project(int e, double* Xc) const {
        const KF& k = kf[eKf[e]];
        mv3(k.Rcw, &pts[3 * (size_t)ePt[e]], Xc);
        for (int i = 0; i < 3; ++i) Xc[i] += k.tcw[i];
    }
    void inertial(int i, double* e9, double* J) const {
        const KF &a = kf[ieKf1[i]], &c = kf[ieKf2[i]];
        orbo_imu_edge_inertial(preint + (size_t)P_SIZE * i, a.Rwb, a.twb, a.v, a.bg, a.ba, c.Rwb, c.twb, c.v, e9, J);
    }
    void compute_errors() {
        for (int e = 0; e < nE; ++e) {
            double Xc[3];
            mono_project(e, Xc);
            const float* c = cam + 4 * (size_t)eKf[e];
            errM[2 * (size_t)e] = obs[2 * (size_t)e] - ((double)c[0] * Xc[0] / Xc[2] + (double)c[2]);
            errM[2 * (size_t)e + 1] = obs[2 * (size_t)e + 1] - ((double)c[1] * Xc[1] / Xc[2] + (double)c[3]);
        }
        for (int i = 0; i < nI; ++i) {
            inertial(i, &errI[9 * (size_t)i], nullptr);
            const KF &a = kf[ieKf1[i]], &c = kf[ieKf2[i]];
            for (int k = 0; k < 3; ++k) { errG[3 * (size_t)i + k] = c.bg[k] - a.bg[k]; errA[3 * (size_t)i + k] = c.ba[k] - a.ba[k]; }
        }
    }
    double chi2_mono(int e) const { return (double)invSigma2[e] * (errM[2 * (size_t)e] * errM[2 * (size_t)e] + errM[2 * (size_t)e + 1] * errM[2 * (size_t)e + 1]); }
    static double quad(const double* M, const double* e, int n) {
        double s = 0;
        for (int i = 0; i < n; ++i) { double t = 0; for (int j = 0; j < n; ++j) t += M[i * n + j] * e[j]; s += e[i] * t; }
        return s;
    }
    double robust_chi2() const {
        double chi = 0, rho[3];
        for (int e = 0; e < nE; ++e) { huber(chi2_mono(e), deltaMono, rho); chi += rho[0]; }
        for (int i = 0; i < nI; ++i) {
            const double c = quad(&info9[81 * (size_t)i], &errI[9 * (size_t)i], 9);
            if (ieRobust[i]) { huber(c, deltaInertial, rho); chi += rho[0]; } else chi += c;
            chi += quad(&infoG[9 * (size_t)i], &errG[3 * (size_t)i], 3) + quad(&infoA[9 * (size_t)i], &errA[3 * (size_t)i], 3);
        }
        return chi;
    }
    void mono_jac(int e, double* Jpt, double* Jp) const {   // EdgeMono::linearizeOplus, src/G2oTypes.cc:349-373
        const KF& k = kf[eKf[e]];
        double Xc[3];
        mono_project(e, Xc);
        const float* c = cam + 4 * (size_t)eKf[e];
        const double fx = c[0], fy = c[1];
        const double pj[6] = {fx / Xc[2], 0, -fx * Xc[0] / (Xc[2] * Xc[2]), 0, fy / Xc[2], -fy * Xc[1] / (Xc[2] * Xc[2])};
        for (int i = 0; i < 2; ++i) for (int j = 0; j < 3; ++j) Jpt[i * 3 + j] = -(pj[i * 3] * k.Rcw[j] + pj[i * 3 + 1] * k.Rcw[3 + j] + pj[i * 3 + 2] * k.Rcw[6 + j]);
        double Xb[3];
        mv3(Rbc, Xc, Xb);
        for (int i = 0; i < 3; ++i) Xb[i] += tbc[i];
        const double x = Xb[0], y = Xb[1], z = Xb[2];
        const double S[18] = {0.0, z, -y, 1.0, 0.0, 0.0, -z, 0.0, x, 0.0, 1.0, 0.0, y, -x, 0.0, 0.0, 0.0, 1.0};
        double PR[6];
        for (int i = 0; i < 2; ++i) for (int j = 0; j < 3; ++j) PR[i * 3 + j] = pj[i * 3] * Rcb[j] + pj[i * 3 + 1] * Rcb[3 + j] + pj[i * 3 + 2] * Rcb[6 + j];
        for (int i = 0; i < 2; ++i) for (int j = 0; j < 6; ++j) Jp[i * 6 + j] = PR[i * 3] * S[j] + PR[i * 3 + 1] * S[6 + j] + PR[i * 3 + 2] * S[12 + j];
    }
    void build_system() {
        const int n = 15 * nOpt;
        std::fill(H.begin(), H.end(), 0.0); std::fill(b.begin(), b.end(), 0.0);
        std::fill(Hll.begin(), Hll.end(), 0.0); std::fill(bl.begin(), bl.end(), 0.0);
        for (int e = 0; e < nE; ++e) {
            const int ip = ePt[e], ik = eKf[e];
            double A[6], B[12], rho[3];
            mono_jac(e, A, B);
            huber(chi2_mono(e), deltaMono, rho);
            const double w = rho[1] * (double)invSigma2[e];
            const double r0 = -(double)invSigma2[e] * errM[2 * (size_t)e] * rho[1], r1 = -(double)invSigma2[e] * errM[2 * (size_t)e + 1] * rho[1];
            double* hl = &Hll[9 * (size_t)ip]; double* b3 = &bl[3 * (size_t)ip];
            for (int a = 0; a < 3; ++a) {
                b3[a] += A[a] * r0 + A[3 + a] * r1;
                for (int c = 0; c < 3; ++c) hl[a * 3 + c] += w * (A[a] * A[c] + A[3 + a] * A[3 + c]);
            }
            double* We = &W[18 * (size_t)e];
            if (ik < nOpt) {
                const int h0 = 15 * ik;
                for (int a = 0; a < 6; ++a) {
                    b[h0 + a] += B[a] * r0 + B[6 + a] * r1;
                    for (int c = 0; c < 6; ++c) H[(size_t)(h0 + a) * n + h0 + c] += w * (B[a] * B[c] + B[6 + a] * B[6 + c]);
                    for (int c = 0; c < 3; ++c) We[a * 3 + c] = w * (B[a] * A[c] + B[6 + a] * A[3 + c]);
                }
            } else std::memset(We, 0, 18 * sizeof(double));
        }
        for (int i = 0; i < nI; ++i) {
            double e9[9], J[216];
            inertial(i, e9, J);
            const double* Om = &info9[81 * (size_t)i];
            const double* er = &errI[9 * (size_t)i];
            double w = 1.0;
            if (ieRobust[i]) { double rho[3]; huber(quad(Om, er, 9), deltaInertial, rho); w = rho[1]; }
            const int k1 = ieKf1[i], k2 = ieKf2[i];
            int g[24];
            for (int c = 0; c < 24; ++c) g[c] = c < 15 ? (k1 < nOpt ? 15 * k1 + c : -1) : (k2 < nOpt ? 15 * k2 + (c - 15) : -1);
            double OJ[216], Oe[9];
            for (int r = 0; r < 9; ++r) {
                double t = 0;
                for (int k = 0; k < 9; ++k) t += Om[r * 9 + k] * er[k];
                Oe[r] = t;
                for (int c = 0; c < 24; ++c) { double s = 0; for (int k = 0; k < 9; ++k) s += Om[r * 9 + k] * J[k * 24 + c]; OJ[r * 24 + c] = s; }
            }
            for (int a = 0; a < 24; ++a) {
                if (g[a] < 0) continue;
                double s = 0;
                for (int r = 0; r < 9; ++r) s += J[r * 24 + a] * Oe[r];
                b[g[a]] -= w * s;
                for (int c = 0; c < 24; ++c) {
                    if (g[c] < 0) continue;
                    double h = 0;
                    for (int r = 0; r < 9; ++r) h += J[r * 24 + a] * OJ[r * 24 + c];
                    H[(size_t)g[a] * n + g[c]] += w * h;
                }
            }
            // EdgeGyroRW / EdgeAccRW: error = b2 - b1, Jacobians -I, +I (include/G2oTypes.h:635-700)
            for (int which = 0; which < 2; ++which) {
                const double* Inf = which == 0 ? &infoG[9 * (size_t)i] : &infoA[9 * (size_t)i];
                const double* er3 = which == 0 ? &errG[3 * (size_t)i] : &errA[3 * (size_t)i];
                const int off = which == 0 ? 9 : 12;
                const int g1 = k1 < nOpt ? 15 * k1 + off : -1, g2 = k2 < nOpt ? 15 * k2 + off : -1;
                for (int a = 0; a < 3; ++a) {
                    double s = 0;
                    for (int c = 0; c < 3; ++c) s += Inf[a * 3 + c] * er3[c];
                    if (g1 >= 0) b[g1 + a] += s;        // -(-I)^T Omega e
                    if (g2 >= 0) b[g2 + a] -= s;
                    for (int c = 0; c < 3; ++c) {
                        if (g1 >= 0) H[(size_t)(g1 + a) * n + g1 + c] += Inf[a * 3 + c];
                        if (g2 >= 0) H[(size_t)(g2 + a) * n + g2 + c] += Inf[a * 3 + c];
                        if (g1 >= 0 && g2 >= 0) { H[(size_t)(g1 + a) * n + g2 + c] -= Inf[a * 3 + c]; H[(size_t)(g2 + a) * n + g1 + c] -= Inf[c * 3 + a]; }
                    }
                }
            }
        }
    }
    bool solve(double lambda) {
        const int n = 15 * nOpt;
        std::vector<double> Hs(H), bs(b);
        for (int i = 0; i < n; ++i) Hs[(size_t)i * n + i] += lambda;
        std::vector<std::vector<int>> edgesOf(nL);
        for (int e = 0; e < nE; ++e) if (eKf[e] < nOpt) edgesOf[ePt[e]].push_back(e);
        for (int p = 0; p < nL; ++p) {
            double D[9];
            for (int i = 0; i < 9; ++i) D[i] = Hll[9 * (size_t)p + i];
            D[0] += lambda; D[4] += lambda; D[8] += lambda;
            double* Di = &Dinv[9 * (size_t)p];
            inv3(D, Di);
            double db[3];
            mv3(Di, &bl[3 * (size_t)p], db);
            for (int e1 : edgesOf[p]) {
                const int i1 = 15 * eKf[e1];
                const double* B1 = &W[18 * (size_t)e1];
                double BD[18];
                for (int a = 0; a < 6; ++a) for (int c = 0; c < 3; ++c) BD[a * 3 + c] = B1[a * 3] * Di[c] + B1[a * 3 + 1] * Di[3 + c] + B1[a * 3 + 2] * Di[6 + c];
                for (int a = 0; a < 6; ++a) bs[i1 + a] -= B1[a * 3] * db[0] + B1[a * 3 + 1] * db[1] + B1[a * 3 + 2] * db[2];
                for (int e2 : edgesOf[p]) {
                    const int i2 = 15 * eKf[e2];
                    const double* B2 = &W[18 * (size_t)e2];
                    for (int a = 0; a < 6; ++a) for (int c = 0; c < 6; ++c)
                        Hs[(size_t)(i1 + a) * n + i2 + c] -= BD[a * 3] * B2[c * 3] + BD[a * 3 + 1] * B2[c * 3 + 1] + BD[a * 3 + 2] * B2[c * 3 + 2];
                }
            }
        }
        if (n > 0 && !ldlt_solve(Hs, n, bs.data(), x.data())) return false;
        for (int p = 0; p < nL; ++p) {
            double cl[3] = {bl[3 * (size_t)p], bl[3 * (size_t)p + 1], bl[3 * (size_t)p + 2]};
            for (int e : edgesOf[p]) {
                const int i1 = 15 * eKf[e];
                const double* B1 = &W[18 * (size_t)e];
                for (int c = 0; c < 3; ++c) for (int a = 0; a < 6; ++a) cl[c] -= B1[a * 3 + c] * x[i1 + a];
            }
            mv3(&Dinv[9 * (size_t)p], cl, &x[n + 3 * (size_t)p]);
        }
        return true;
    }
    void update() {
        for (int k = 0; k < nOpt; ++k) {
            KF& f = kf[k];
            const double* u = &x[15 * (size_t)k];
            orbo_imu_pose_update(f.Rwb, f.twb, u);                          // twb += Rwb ut; Rwb = Rwb ExpSO3(ur)
            if (++f.its >= 3) f.its = 0;      // its `NormalizeRotation(Rwb);` (src/G2oTypes.cc:202-208) discards the returned matrix: Rwb is never renormalised
            double tbw[3];
            for (int i = 0; i < 3; ++i) tbw[i] = -(f.Rwb[i] * f.twb[0] + f.Rwb[3 + i] * f.twb[1] + f.Rwb[6 + i] * f.twb[2]);   // -Rbw twb
            for (int i = 0; i < 3; ++i) {
                for (int j = 0; j < 3; ++j) f.Rcw[i * 3 + j] = Rcb[i * 3] * f.Rwb[j * 3] + Rcb[i * 3 + 1] * f.Rwb[j * 3 + 1] + Rcb[i * 3 + 2] * f.Rwb[j * 3 + 2];   // Rcb Rbw
                f.tcw[i] = Rcb[i * 3] * tbw[0] + Rcb[i * 3 + 1] * tbw[1] + Rcb[i * 3 + 2] * tbw[2] + tcb[i];
            }
            for (int i = 0; i < 3; ++i) { f.v[i] += u[6 + i]; f.bg[i] += u[9 + i]; f.ba[i] += u[12 + i]; }
        }
        const int n = 15 * nOpt;
        for (size_t k = 0; k < (size_t)3 * nL; ++k) pts[k] += x[n + k];
    }
};

}  // namespace liba
}  // namespace orbo

using namespace orbo::liba;

extern "C" {

// Keyframes [0, nOpt) are the temporal window (all four vertices free), [nOpt, nKF) are fixed.
//   kfState21 [nKF][21] in/out: Rwb 9 | twb 3 | velocity 3 | gyro bias 3 | acc bias 3;  kfTcw12 [nKF][12] in/out: Rcw 9 | tcw 3 (the keyframe's own
//   camera pose, what ImuCamPose(KeyFrame*) loads);  cam4 [nKF][4];  extr24: Rcb 9 | tcb 3 | Rbc 9 | tbc 3.
//   inertial edge i: keyframes ieKf1[i] -> ieKf2[i], preint [nI][292] (already SetNewBias'ed: only b / the Jacobians / C are read),
//   ieRobust[i] (Huber sqrt(16.92)), ieInfoScale[i] (1e-2 on the link to the fixed keyframe, else 1).
//   mono edge e: point ePt[e], keyframe eKf[e], obs2, invSigma2; trackDepth [nL] = pMP->mTrackDepth.
//   eraseOut [nE]: the (keyframe, point) pairs of vToErase; edgeChi2Out [nE].
//   stats [8]: err, err_end (as the reference's floats), failed, final lambda, LM trials, outer iterations.
// Returns optimize()'s iteration count.  When the FAIL test fires the states and points are left as they came in and eraseOut is all zero (the reference
// returns before the erasure and the write-back).
int orbo_local_inertial_ba(int nKF, int nOpt, double* kfState21, double* kfTcw12, const float* cam4, const double* extr24, int nI, const int* ieKf1, const int* ieKf2,
                           const float* preint, const uint8_t* ieRobust, const double* ieInfoScale, int nL, double* points3, const float* trackDepth, int nE,
                           const int* ePt, const int* eKf, const double* obs2, const float* invSigma2, int iterations, double lambdaInit, int bLarge,
                           uint8_t* eraseOut, double* edgeChi2Out, double* stats) {
    Problem L;
    L.nKF = nKF; L.nOpt = nOpt; L.nI = nI; L.nL = nL; L.nE = nE;
    L.kf.resize(nKF);
    for (int k = 0; k < nKF; ++k) {
        const double* s = kfState21 + 21 * (size_t)k;
        KF& f = L.kf[k];
        std::memcpy(f.Rwb, s, 9 * sizeof(double)); std::memcpy(f.twb, s + 9, 3 * sizeof(double)); std::memcpy(f.v, s + 12, 3 * sizeof(double));
        std::memcpy(f.bg, s + 15, 3 * sizeof(double)); std::memcpy(f.ba, s + 18, 3 * sizeof(double));
        std::memcpy(f.Rcw, kfTcw12 + 12 * (size_t)k, 9 * sizeof(double)); std::memcpy(f.tcw, kfTcw12 + 12 * (size_t)k + 9, 3 * sizeof(double));
        f.its = 0;
    }
    L.pts.assign(points3, points3 + 3 * (size_t)nL);
    L.cam = cam4; L.Rcb = extr24; L.tcb = extr24 + 9; L.Rbc = extr24 + 12; L.tbc = extr24 + 21;
    L.ieKf1 = ieKf1; L.ieKf2 = ieKf2; L.preint = preint; L.ieRobust = ieRobust;
    L.info9.resize(81 * (size_t)nI); L.infoG.resize(9 * (size_t)nI); L.infoA.resize(9 * (size_t)nI);
    for (int i = 0; i < nI; ++i) {
        orbo_imu_information(preint + (size_t)P_SIZE * i, &L.info9[81 * (size_t)i], &L.infoG[9 * (size_t)i], &L.infoA[9 * (size_t)i]);
        for (int k = 0; k < 81; ++k) L.info9[81 * (size_t)i + k] *= ieInfoScale[i];
    }
    L.ePt = ePt; L.eKf = eKf; L.obs = obs2; L.invSigma2 = invSigma2;
    L.deltaMono = (double)(float)std::sqrt(5.991);       // const float thHuberMono = sqrt(5.991); rk->setDelta(thHuberMono)
    L.deltaInertial = std::sqrt(16.92);                  // rki->setDelta(sqrt(16.92))
    L.errM.assign(2 * (size_t)nE, 0.0); L.errI.assign(9 * (size_t)nI, 0.0); L.errG.assign(3 * (size_t)nI, 0.0); L.errA.assign(3 * (size_t)nI, 0.0);
    const int n = 15 * nOpt;
    L.H.assign((size_t)n * n, 0.0); L.b.assign(n, 0.0); L.Hll.assign(9 * (size_t)nL, 0.0); L.bl.assign(3 * (size_t)nL, 0.0);
    L.W.assign(18 * (size_t)nE, 0.0); L.x.assign(n + 3 * (size_t)nL, 0.0); L.Dinv.assign(9 * (size_t)nL, 0.0);
    if (stats) std::memset(stats, 0, 8 * sizeof(double));
    const std::vector<KF> kf0 = L.kf;
    const std::vector<double> pts0 = L.pts;

    L.compute_errors();
    const float err = (float)L.robust_chi2();

    double lambda = -1, ni = 2;
    int nBad = 0, cj = 0, trials = 0;
    const int maxTrials = 10;
    bool ok = true;
    for (int it = 0; it < iterations && ok; ++it) {
        L.compute_errors();
        double currentChi = L.robust_chi2();
        double tempChi = currentChi;
        const double iniChi = currentChi;
        L.build_system();
        if (it == 0) {
            if (lambdaInit > 0) lambda = lambdaInit;
            else {
                double maxDiag = 0;
                for (int i = 0; i < n; ++i) maxDiag = std::max(std::fabs(L.H[(size_t)i * n + i]), maxDiag);
                for (int p = 0; p < nL; ++p) for (int j = 0; j < 3; ++j) maxDiag = std::max(std::fabs(L.Hll[9 * (size_t)p + 4 * j]), maxDiag);
                lambda = 1e-5 * maxDiag;
            }
            ni = 2; nBad = 0;
        }
        double rho = 0;
        int qmax = 0;
        do {
            L.kfBk = L.kf; L.ptsBk = L.pts;
            const bool ok2 = L.solve(lambda);
            L.update();
            L.compute_errors();
            tempChi = L.robust_chi2();
            if (!ok2) tempChi = DBL_MAX;
            rho = currentChi - tempChi;
            double scale = 0;
            for (int j = 0; j < n; ++j) scale += L.x[j] * (lambda * L.x[j] + L.b[j]);
            for (size_t j = 0; j < (size_t)3 * nL; ++j) scale += L.x[n + j] * (lambda * L.x[n + j] + L.bl[j]);
            scale += 1e-3;
            rho /= scale;
            if (rho > 0 && std::isfinite(tempChi)) {
                double alpha = 1. - std::pow((2 * rho - 1), 3);
                alpha = std::min(alpha, 2. / 3.);
                lambda *= std::max(1. / 3., alpha);
                ni = 2;
                currentChi = tempChi;
            } else {
                lambda *= ni;
                ni *= 2;
                L.kf = L.kfBk; L.pts = L.ptsBk;
            }
            ++qmax; ++trials;
        } while (rho < 0 && qmax < maxTrials);
        ++cj;
        if (qmax == maxTrials || rho == 0) ok = false;
        else {
            if ((iniChi - currentChi) * 1e3 < iniChi) ++nBad; else nBad = 0;
            if (nBad >= 3) ok = false;
        }
    }
    const float errEnd = (float)L.robust_chi2();          // from the errors the edges hold (stale after a rejected last trial)
    const float chi2Mono2 = 5.991f;
    for (int e = 0; e < nE; ++e) {
        const double c2 = L.chi2_mono(e);
        if (edgeChi2Out) edgeChi2Out[e] = c2;
        const bool bClose = trackDepth[ePt[e]] < 10.f;
        const KF& k = L.kf[eKf[e]];
        const double* X = &L.pts[3 * (size_t)ePt[e]];
        const bool depthPos = (k.Rcw[6] * X[0] + k.Rcw[7] * X[1] + k.Rcw[8] * X[2] + k.tcw[2]) > 0.0;
        eraseOut[e] = ((c2 > chi2Mono2 && !bClose) || (c2 > 1.5f * chi2Mono2 && bClose) || !depthPos) ? 1 : 0;
    }
    const bool failed = (2 * err < errEnd || std::isnan(err) || std::isnan(errEnd)) && !bLarge;
    // on FAIL the reference returns before it erases any observation (:2884-2888): no flag is set
    if (failed) { L.kf = kf0; L.pts = pts0; if (nE) std::memset(eraseOut, 0, (size_t)nE); }
    for (int k = 0; k < nKF; ++k) {
        double* s = kfState21 + 21 * (size_t)k;
        const KF& f = L.kf[k];
        std::memcpy(s, f.Rwb, 9 * sizeof(double)); std::memcpy(s + 9, f.twb, 3 * sizeof(double)); std::memcpy(s + 12, f.v, 3 * sizeof(double));
        std::memcpy(s + 15, f.bg, 3 * sizeof(double)); std::memcpy(s + 18, f.ba, 3 * sizeof(double));
        std::memcpy(kfTcw12 + 12 * (size_t)k, f.Rcw, 9 * sizeof(double)); std::memcpy(kfTcw12 + 12 * (size_t)k + 9, f.tcw, 3 * sizeof(double));
    }
    std::memcpy(points3, L.pts.data(), sizeof(double) * 3 * (size_t)nL);
    if (stats) { stats[0] = err; stats[1] = errEnd; stats[2] = failed; stats[3] = lambda; stats[4] = trials; stats[5] = cj; }
    return cj;
}

// ---- the same state opened step by step (OrboLmBackend, oracle_common.h) ----
namespace {
struct LibaOpen {
    Problem L;
    std::vector<float> cam, preint, is2; std::vector<double> extr, obs; std::vector<int> k1, k2, ePt, eKf; std::vector<uint8_t> rob;
    std::vector<double> bcat, diag;
};
void lio_compute_errors(void* p) { ((LibaOpen*)p)->L.compute_errors(); }
double lio_robust_chi2(void* p) { return ((LibaOpen*)p)->L.robust_chi2(); }
void lio_build_system(void* p) {
    LibaOpen* o = (LibaOpen*)p; Problem& L = o->L;
    L.build_system();
    const int n = 15 * L.nOpt;
    o->bcat.assign(L.b.begin(), L.b.end()); o->bcat.insert(o->bcat.end(), L.bl.begin(), L.bl.end());
    o->diag.clear();
    for (int i = 0; i < n; ++i) o->diag.push_back(L.H[(size_t)i * n + i]);
    for (int q = 0; q < L.nL; ++q) for (int j = 0; j < 3; ++j) o->diag.push_back(L.Hll[9 * (size_t)q + 4 * j]);
}
int lio_solve(void* p, double lambda) { return ((LibaOpen*)p)->L.solve(lambda) ? 1 : 0; }
void lio_update(void* p) { ((LibaOpen*)p)->L.update(); }
void lio_push(void* p) { Problem& L = ((LibaOpen*)p)->L; L.kfBk = L.kf; L.ptsBk = L.pts; }
void lio_pop(void* p) { Problem& L = ((LibaOpen*)p)->L; L.kf = L.kfBk; L.pts = L.ptsBk; }
int lio_vector_size(void* p) { Problem& L = ((LibaOpen*)p)->L; return 15 * L.nOpt + 3 * L.nL; }
const double* lio_x(void* p) { return ((LibaOpen*)p)->L.x.data(); }
const double* lio_b(void* p) { return ((LibaOpen*)p)->bcat.data(); }
int lio_n_diag(void* p) { return (int)((LibaOpen*)p)->diag.size(); }
const double* lio_diag(void* p) { return ((LibaOpen*)p)->diag.data(); }
}  // namespace

void orbo_liba_backend_open(int nKF, int nOpt, const double* kfState21, const double* kfTcw12, const float* cam4, const double* extr24, int nI, const int* ieKf1, const int* ieKf2,
                            const float* preint, const uint8_t* ieRobust, const double* ieInfoScale, int nL, const double* points3, int nE, const int* ePt, const int* eKf,
                            const double* obs2, const float* invSigma2, OrboLmBackend* out) {
    LibaOpen* o = new LibaOpen;
    o->cam.assign(cam4, cam4 + 4 * (size_t)nKF); o->extr.assign(extr24, extr24 + 24); o->k1.assign(ieKf1, ieKf1 + nI); o->k2.assign(ieKf2, ieKf2 + nI);
    o->preint.assign(preint, preint + (size_t)P_SIZE * nI); o->rob.assign(ieRobust, ieRobust + nI); o->ePt.assign(ePt, ePt + nE); o->eKf.assign(eKf, eKf + nE);
    o->obs.assign(obs2, obs2 + 2 * (size_t)nE); o->is2.assign(invSigma2, invSigma2 + nE);
    Problem& L = o->L;
    L.nKF = nKF; L.nOpt = nOpt; L.nI = nI; L.nL = nL; L.nE = nE;
    L.kf.resize(nKF);
    for (int k = 0; k < nKF; ++k) {
        const double* s = kfState21 + 21 * (size_t)k;
        KF& f = L.kf[k];
        std::memcpy(f.Rwb, s, 9 * sizeof(double)); std::memcpy(f.twb, s + 9, 3 * sizeof(double)); std::memcpy(f.v, s + 12, 3 * sizeof(double));
        std::memcpy(f.bg, s + 15, 3 * sizeof(double)); std::memcpy(f.ba, s + 18, 3 * sizeof(double));
        std::memcpy(f.Rcw, kfTcw12 + 12 * (size_t)k, 9 * sizeof(double)); std::memcpy(f.tcw, kfTcw12 + 12 * (size_t)k + 9, 3 * sizeof(double));
        f.its = 0;
    }
    L.pts.assign(points3, points3 + 3 * (size_t)nL);
    L.cam = o->cam.data(); L.Rcb = o->extr.data(); L.tcb = o->extr.data() + 9; L.Rbc = o->extr.data() + 12; L.tbc = o->extr.data() + 21;
    L.ieKf1 = o->k1.data(); L.ieKf2 = o->k2.data(); L.preint = o->preint.data(); L.ieRobust = o->rob.data();
    L.info9.resize(81 * (size_t)nI); L.infoG.resize(9 * (size_t)nI); L.infoA.resize(9 * (size_t)nI);
    for (int i = 0; i < nI; ++i) {
        orbo_imu_information(L.preint + (size_t)P_SIZE * i, &L.info9[81 * (size_t)i], &L.infoG[9 * (size_t)i], &L.infoA[9 * (size_t)i]);
        for (int k = 0; k < 81; ++k) L.info9[81 * (size_t)i + k] *= ieInfoScale[i];
    }
    L.ePt = o->ePt.data(); L.eKf = o->eKf.data(); L.obs = o->obs.data(); L.invSigma2 = o->is2.data();
    L.deltaMono = (double)(float)std::sqrt(5.991); L.deltaInertial = std::sqrt(16.92);
    L.errM.assign(2 * (size_t)nE, 0.0); L.errI.assign(9 * (size_t)nI, 0.0); L.errG.assign(3 * (size_t)nI, 0.0); L.errA.assign(3 * (size_t)nI, 0.0);
    const int n = 15 * nOpt;
    L.H.assign((size_t)n * n, 0.0); L.b.assign(n, 0.0); L.Hll.assign(9 * (size_t)nL, 0.0); L.bl.assign(3 * (size_t)nL, 0.0);
    L.W.assign(18 * (size_t)nE, 0.0); L.x.assign(n + 3 * (size_t)nL, 0.0); L.Dinv.assign(9 * (size_t)nL, 0.0);
    *out = OrboLmBackend{o, lio_compute_errors, lio_robust_chi2, lio_build_system, lio_solve, lio_update, lio_push, lio_pop, lio_vector_size, lio_x, lio_b, lio_n_diag, lio_diag};
}
// per-edge accessors for the post-optimisation text of Optimizer::LocalInertialBA (src/Optimizer.cc:2840-2895), which oracle/ref_shim/ref_wrap_g2o_lm.cpp compiles verbatim
double orbo_liba_edge_chi2(void* h, int e) { return ((LibaOpen*)h)->L.chi2_mono(e); }
int orbo_liba_edge_depth_positive(void* h, int e) {
    const Problem& L = ((LibaOpen*)h)->L;
    const KF& k = L.kf[L.eKf[e]];
    const double* X = &L.pts[3 * (size_t)L.ePt[e]];
    return (k.Rcw[6] * X[0] + k.Rcw[7] * X[1] + k.Rcw[8] * X[2] + k.tcw[2]) > 0.0;
}
int orbo_liba_edge_point(void* h, int e) { return ((LibaOpen*)h)->L.ePt[e]; }
void orbo_liba_backend_close(OrboLmBackend* be, double* kfStateOut21, double* pointsOut3) {
    LibaOpen* o = (LibaOpen*)be->self; Problem& L = o->L;
    for (int k = 0; k < L.nKF; ++k) {
        double* s = kfStateOut21 + 21 * (size_t)k; const KF& f = L.kf[k];
        std::memcpy(s, f.Rwb, 9 * sizeof(double)); std::memcpy(s + 9, f.twb, 3 * sizeof(double)); std::memcpy(s + 12, f.v, 3 * sizeof(double));
        std::memcpy(s + 15, f.bg, 3 * sizeof(double)); std::memcpy(s + 18, f.ba, 3 * sizeof(double));
    }
    std::memcpy(pointsOut3, L.pts.data(), sizeof(double) * 3 * (size_t)L.nL);
    delete o;
    be->self = nullptr;
}

// reprojection residuals of a state (for the 1e-4 px bar): obs - project(Rcw X + tcw)
void orbo_local_inertial_ba_residuals(int nE, const int* ePt, const int* eKf, const double* kfTcw12, const float* cam4, const double* points3, const double* obs2, double* res2) {
    for (int e = 0; e < nE; ++e) {
        const double* T = kfTcw12 + 12 * (size_t)eKf[e];
        const double* X = points3 + 3 * (size_t)ePt[e];
        double Xc[3];
        mv3(T, X, Xc);
        for (int i = 0; i < 3; ++i) Xc[i] += T[9 + i];
        const float* c = cam4 + 4 * (size_t)eKf[e];
        res2[2 * (size_t)e] = obs2[2 * (size_t)e] - ((double)c[0] * Xc[0] / Xc[2] + (double)c[2]);
        res2[2 * (size_t)e + 1] = obs2[2 * (size_t)e + 1] - ((double)c[1] * Xc[1] / Xc[2] + (double)c[3]);
    }
}

}  // extern "C"
