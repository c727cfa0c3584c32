// TEST INFRASTRUCTURE ONLY (see oracle_common.h).  CPU restatement of the numeric core of
// Optimizer::LocalBundleAdjustment (reference src/Optimizer.cc:1116-1498, between optimizer.optimize(10)
// at :1411 and the outlier test at :1417-1430) and of Optimizer::PoseOptimization (:814-1114) with g2o semantics:
//   SparseOptimizer::optimize / update / computeActiveErrors / activeRobustChi2   g2o/core/sparse_optimizer.cpp:354-435,61-113
//   OptimizationAlgorithmLevenberg::solve / computeLambdaInit / computeScale      g2o/core/optimization_algorithm_levenberg.cpp:61-194
//   BlockSolver<6,3>::buildSystem / setLambda / solve (Schur) / restoreDiagonal   g2o/core/block_solver.hpp:354-486,502-604
//   BaseBinaryEdge::constructQuadraticForm, RobustKernelHuber::robustify           g2o/core/base_binary_edge.hpp:55-120, robust_kernel_impl.cpp:78-91
//   EdgeSE3ProjectXYZ::computeError / linearizeOplus / isDepthPositive             include/OptimizableTypes.h:99-110, src/OptimizableTypes.cpp:139-160
//   Pinhole::project(Vector3d) / projectJac                                        src/CameraModels/Pinhole.cpp:35-41,71-81
//   SE3Quat::exp / operator* / map / normalizeRotation, VertexSE3Expmap::oplusImpl g2o/types/se3quat.h:62-120,223-256, types_six_dof_expmap.h:73-76
//   LinearSolverEigen::solve (SimplicialLDLT)                                      g2o/solvers/linear_solver_eigen.h:94-125
// Eigen is absent here, so the small fixed-size algebra is written out; the reduced camera system is factorised by
// a dense LDL^T without pivoting (what SimplicialLDLT computes up to the fill-reducing permutation, i.e. up to rounding).
// Summation order over edges is free (the reference's own order depends on pointer values, SURVEY.md 8a'); control
// flow (accept/reject, lambda schedule, stop rules, stale errors after a rejected last trial) is reproduced exactly.
// PARITY: the edge errors / Jacobians, VertexSE3Expmap::oplusImpl, the Huber kernel and the LM control flow equal the reference's own text compiled into oracle/_ref
// (tests/test_ref_pins_lba_edges_cpu.py, tests/test_ref_pins_lm_cpu.py); BlockSolver's Schur / linear solve (needs Eigen) stays pinned by an independent dense solve
// with numerical Jacobians (tests/test_lba_dense_cpu.py), the whole LM loop additionally by a second transcription (tests/test_lba_lm_transcription_cpu.py).
#include "oracle_common.h"

#include <cfloat>
#include <cstring>
#include <vector>

namespace orbo {

struct Quat { double w, x, y, z; };
struct Pose { Quat q; double t[3]; };

static inline void qrot(const Quat& q, const double* v, double* o) {   // Eigen QuaternionBase::_transformVector
    double ux = q.y * v[2] - q.z * v[1], uy = q.z * v[0] - q.x * v[2], uz = q.x * v[1] - q.y * v[0];
    ux += ux; uy += uy; uz += uz;
    o[0] = v[0] + q.w * ux + (q.y * uz - q.z * uy);
    o[1] = v[1] + q.w * uy + (q.z * ux - q.x * uz);
    o[2] = v[2] + q.w * uz + (q.x * uy - q.y * ux);
}
static inline Quat qmul(const Quat& a, const Quat& b) {
    return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}
static inline void qnormalize(Quat& q) {   // SE3Quat::normalizeRotation
    if (q.w < 0) { q.w = -q.w; q.x = -q.x; q.y = -q.y; q.z = -q.z; }
    const double n = std::sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    q.w /= n; q.x /= n; q.y /= n; q.z /= n;
}
static inline void qtoR(const Quat& q, double R[9]) {   // Eigen toRotationMatrix
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w, txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
static inline Quat qfromR(const double m[9]) {   // Eigen quaternion from rotation matrix
    Quat q;
    double t = m[0] + m[4] + m[8];
    if (t > 0) {
        t = std::sqrt(t + 1.0);
        q.w = 0.5 * t; t = 0.5 / t;
        q.x = (m[7] - m[5]) * t; q.y = (m[2] - m[6]) * t; q.z = (m[3] - m[1]) * t;
    } else {
        int i = 0;
        if (m[4] > m[0]) i = 1;
        if (m[8] > m[i * 3 + i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0);
        double v[3];
        v[i] = 0.5 * t; t = 0.5 / t;
        q.w = (m[k * 3 + j] - m[j * 3 + k]) * t;
        v[j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
        v[k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
        q.x = v[0]; q.y = v[1]; q.z = v[2];
    }
    return q;
}
static inline void mat3mul(const double* a, const double* b, double* c) {
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) c[i * 3 + j] = a[i * 3] * b[j] + a[i * 3 + 1] * b[3 + j] + a[i * 3 + 2] * b[6 + j];
}
// SE3Quat::exp(update) * T   (VertexSE3Expmap::oplusImpl)
static void pose_oplus(Pose& T, const double* upd) {
    const double om[3] = {upd[0], upd[1], upd[2]}, up[3] = {upd[3], upd[4], upd[5]};
    const double theta = std::sqrt(om[0] * om[0] + om[1] * om[1] + om[2] * om[2]);
    const double O[9] = {0, -om[2], om[1], om[2], 0, -om[0], -om[1], om[0], 0};
    double O2[9]; mat3mul(O, O, O2);
    double R[9], V[9];
    double a, b, c, d;
    if (theta < 0.00001) { a = 1.0; b = 1 / 2.0; c = 1 / 2.0; d = 1 / 6.0; }
    else {
        a = std::sin(theta) / theta; b = (1 - std::cos(theta)) / (theta * theta);
        c = b; d = (theta - std::sin(theta)) / std::pow(theta, 3);
    }
    for (int i = 0; i < 9; ++i) {
        const double I = (i % 4 == 0) ? 1.0 : 0.0;
        R[i] = I + a * O[i] + b * O2[i];
        V[i] = I + c * O[i] + d * O2[i];
    }
    Quat qe = qfromR(R);
    double te[3] = {V[0] * up[0] + V[1] * up[1] + V[2] * up[2], V[3] * up[0] + V[4] * up[1] + V[5] * up[2], V[6] * up[0] + V[7] * up[1] + V[8] * up[2]};
    qnormalize(qe);   // SE3Quat(Quaterniond(R), V*upsilon) constructor
    double rt[3]; qrot(qe, T.t, rt);   // operator*: result._t += _r*tr2._t; result._r *= tr2._r; normalize
    Pose Rn;
    Rn.t[0] = te[0] + rt[0]; Rn.t[1] = te[1] + rt[1]; Rn.t[2] = te[2] + rt[2];
    Rn.q = qmul(qe, T.q);
    qnormalize(Rn.q);
    T = Rn;
}

static bool inv3(const double* m, double* o) {   // Eigen fixed-size 3x3 inverse: cofactors / determinant
    const double c00 = m[4] * m[8] - m[5] * m[7], c10 = m[5] * m[6] - m[3] * m[8], c20 = m[3] * m[7] - m[4] * m[6];
    const double det = m[0] * c00 + m[1] * c10 + m[2] * c20;
    const double id = 1.0 / det;
    o[0] = c00 * id; o[1] = (m[2] * m[7] - m[1] * m[8]) * id; o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
    o[3] = c10 * id; o[4] = (m[0] * m[8] - m[2] * m[6]) * id; o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
    o[6] = c20 * id; o[7] = (m[1] * m[6] - m[0] * m[7]) * id; o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
    return true;
}

// dense LDL^T (no pivoting) of the symmetric n x n matrix A (full storage, modified in place); solves A x = b.
// Returns false when a pivot is exactly zero (SimplicialLDLT's only failure mode).
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

// EdgeSE3ProjectXYZ::linearizeOplus (src/OptimizableTypes.cpp:139-160) at the camera-frame point Xc = T.map(xyz)
static void edge_jacobians(const Quat& q, const float* c, const double* Xc, double* A, double* B) {
    const double x = Xc[0], y = Xc[1], z = Xc[2];
    // -projectJac
    const double J[6] = {-((double)c[0] / z), -0.0, -(-(double)c[0] * x / (z * z)), -0.0, -((double)c[1] / z), -(-(double)c[1] * y / (z * z))};
    double R[9]; qtoR(q, R);
    for (int r = 0; r < 2; ++r) for (int k = 0; k < 3; ++k) A[r * 3 + k] = J[r * 3] * R[k] + J[r * 3 + 1] * R[3 + k] + J[r * 3 + 2] * R[6 + k];      // 2x3 = J * R
    const double S[18] = {0, z, -y, 1, 0, 0, -z, 0, x, 0, 1, 0, y, -x, 0, 0, 0, 1};
    for (int r = 0; r < 2; ++r) for (int k = 0; k < 6; ++k) B[r * 6 + k] = J[r * 3] * S[k] + J[r * 3 + 1] * S[6 + k] + J[r * 3 + 2] * S[12 + k];   // 2x6 = J * SE3deriv
}

struct Lba {
    int nP, nL, nE;
    std::vector<Pose> poses, posesBk;
    std::vector<uint8_t> fixed;
    std::vector<int> hidx;            // Hessian block index of each pose (-1 fixed)
    int nF = 0;
    std::vector<double> pts, ptsBk;   // 3 per point
    const float* cam;                 // 4 per pose
    const int *ePt, *ePose;
    const double* obs;
    const float* invSigma2;
    double delta, dsqr;
    std::vector<double> err;          // 2 per edge (EdgeSE3ProjectXYZ::_error)
    // linear system
    std::vector<double> Hpp, bp, Hll, bl, W, x, Dinv;   // Hpp: dense (6nF)^2 holding only diagonal blocks; W: 18 per edge (6x3)
    volatile const int* stop;

    bool terminate() const { return stop && *stop; }

    void project_edge(int e, double* Xc, double* uv) const {
        const Pose& T = poses[ePose[e]];
        double r[3]; qrot(T.q, &pts[3 * (size_t)ePt[e]], r);
        Xc[0] = r[0] + T.t[0]; Xc[1] = r[1] + T.t[1]; Xc[2] = r[2] + T.t[2];
        const float* c = cam + 4 * (size_t)ePose[e];
        uv[0] = (double)c[0] * Xc[0] / Xc[2] + (double)c[2];
        uv[1] = (double)c[1] * Xc[1] / Xc[2] + (double)c[3];
    }
    void compute_errors() {   // computeActiveErrors
        for (int e = 0; e < nE; ++e) {
            double Xc[3], uv[2];
            project_edge(e, Xc, uv);
            err[2 * (size_t)e] = obs[2 * (size_t)e] - uv[0];
            err[2 * (size_t)e + 1] = obs[2 * (size_t)e + 1] - uv[1];
        }
    }
    double chi2(int e) const { return (double)invSigma2[e] * (err[2 * (size_t)e] * err[2 * (size_t)e] + err[2 * (size_t)e + 1] * err[2 * (size_t)e + 1]); }
    void robustify(double e2, double* rho) const {
        if (e2 <= dsqr) { rho[0] = e2; rho[1] = 1.; rho[2] = 0.; }
        else { const double s = std::sqrt(e2); rho[0] = 2 * s * delta - dsqr; rho[1] = delta / s; rho[2] = -0.5 * rho[1] / e2; }
    }
    double robust_chi2() const {
        double chi = 0, rho[3];
        for (int e = 0; e < nE; ++e) { robustify(chi2(e), rho); chi += rho[0]; }
        return chi;
    }
    void build_system() {
        const int n = 6 * nF;
        std::fill(Hpp.begin(), Hpp.end(), 0.0); std::fill(bp.begin(), bp.end(), 0.0);
        std::fill(Hll.begin(), Hll.end(), 0.0); std::fill(bl.begin(), bl.end(), 0.0);
        for (int e = 0; e < nE; ++e) {
            const int ip = ePt[e], ic = ePose[e], h = hidx[ic];
            double Xc[3], uv[2];
            project_edge(e, Xc, uv);
            double A[6], B[12];   // _jacobianOplusXi (2x3), _jacobianOplusXj (2x6)
            edge_jacobians(poses[ic].q, cam + 4 * (size_t)ic, Xc, A, B);
            double rho[3]; robustify(chi2(e), rho);
            const double w = rho[1] * (double)invSigma2[e];
            const double r0 = -(double)invSigma2[e] * err[2 * (size_t)e] * rho[1], r1 = -(double)invSigma2[e] * err[2 * (size_t)e + 1] * rho[1];
            double* hl = &Hll[9 * (size_t)ip]; double* b3 = &bl[3 * (size_t)ip];
            for (int a = 0; a < 3; ++a) {
                b3[a] += A[a] * r0 + A[3 + a] * r1;
                for (int b = 0; b < 3; ++b) hl[a * 3 + b] += w * (A[a] * A[b] + A[3 + a] * A[3 + b]);
            }
            double* We = &W[18 * (size_t)e];
            if (h >= 0) {
                for (int a = 0; a < 6; ++a) {
                    bp[6 * (size_t)h + a] += B[a] * r0 + B[6 + a] * r1;
                    for (int b = 0; b < 6; ++b) Hpp[(size_t)(6 * h + a) * n + 6 * h + b] += w * (B[a] * B[b] + B[6 + a] * B[6 + b]);
                    for (int b = 0; b < 3; ++b) We[a * 3 + b] = w * (B[a] * A[b] + B[6 + a] * A[3 + b]);
                }
            } else std::memset(We, 0, 18 * sizeof(double));
        }
    }
    // BlockSolver::solve with lambda already folded into the diagonals of local copies
    bool solve(double lambda) {
        const int n = 6 * nF;
        std::vector<double> Hs(Hpp), bs(bp);
        for (int i = 0; i < n; ++i) Hs[(size_t)i * n + i] += lambda;
        // per landmark: Dinv, Schur complement
        std::vector<std::vector<int>> edgesOf(nL);
        for (int e = 0; e < nE; ++e) if (hidx[ePose[e]] >= 0) edgesOf[ePt[e]].push_back(e);
        for (int p = 0; p < nL; ++p) {
            double D[9];
            for (int i = 0; i < 9; ++i) D[i] = Hll[9 * (size_t)p + i];
            D[0] += lambda; D[4] += lambda; D[8] += lambda;
            double* Di = &Dinv[9 * (size_t)p];
            inv3(D, Di);
            const double* b3 = &bl[3 * (size_t)p];
            const double db[3] = {Di[0] * b3[0] + Di[1] * b3[1] + Di[2] * b3[2], Di[3] * b3[0] + Di[4] * b3[1] + Di[5] * b3[2], Di[6] * b3[0] + Di[7] * b3[1] + Di[8] * b3[2]};
            for (int e1 : edgesOf[p]) {
                const int i1 = hidx[ePose[e1]];
                const double* B1 = &W[18 * (size_t)e1];
                double BD[18];
                for (int a = 0; a < 6; ++a) for (int b = 0; b < 3; ++b) BD[a * 3 + b] = B1[a * 3] * Di[b] + B1[a * 3 + 1] * Di[3 + b] + B1[a * 3 + 2] * Di[6 + b];
                for (int a = 0; a < 6; ++a) bs[6 * (size_t)i1 + a] -= B1[a * 3] * db[0] + B1[a * 3 + 1] * db[1] + B1[a * 3 + 2] * db[2];
                for (int e2 : edgesOf[p]) {
                    const int i2 = hidx[ePose[e2]];
                    const double* B2 = &W[18 * (size_t)e2];
                    for (int a = 0; a < 6; ++a) for (int b = 0; b < 6; ++b)
                        Hs[(size_t)(6 * i1 + a) * n + 6 * i2 + b] -= BD[a * 3] * B2[b * 3] + BD[a * 3 + 1] * B2[b * 3 + 1] + BD[a * 3 + 2] * B2[b * 3 + 2];
                }
            }
        }
        if (n > 0 && !ldlt_solve(Hs, n, bs.data(), x.data())) return false;
        // landmarks: xl = Dinv (bl - Hpl^T xp)
        for (int p = 0; p < nL; ++p) {
            double cl[3] = {bl[3 * (size_t)p], bl[3 * (size_t)p + 1], bl[3 * (size_t)p + 2]};
            for (int e : edgesOf[p]) {
                const int i1 = hidx[ePose[e]];
                const double* B1 = &W[18 * (size_t)e];
                for (int b = 0; b < 3; ++b) for (int a = 0; a < 6; ++a) cl[b] -= B1[a * 3 + b] * x[6 * (size_t)i1 + a];
            }
            const double* Di = &Dinv[9 * (size_t)p];
            for (int a = 0; a < 3; ++a) x[n + 3 * (size_t)p + a] = Di[a * 3] * cl[0] + Di[a * 3 + 1] * cl[1] + Di[a * 3 + 2] * cl[2];
        }
        return true;
    }
    void update() {
        for (int i = 0; i < nP; ++i) if (hidx[i] >= 0) pose_oplus(poses[i], &x[6 * (size_t)hidx[i]]);
        const int n = 6 * nF;
        for (size_t k = 0; k < (size_t)3 * nL; ++k) pts[k] += x[n + k];
    }
};

}  // namespace orbo

using namespace orbo;

static void only_pose_jacobian(const float* cam4, double x, double y, double z, double* B);

extern "C" {

// Returns the number of outer iterations performed (SparseOptimizer::optimize's return value), or -1 when there is
// nothing to optimise.  Arrays are in g2o's Hessian order (poses by id, points by id).
//   posesInOut: nP x 7 (qw,qx,qy,qz,tx,ty,tz); pointsInOut: nL x 3; edgeChi2Out / edgeDepthPosOut: nE
//   stats (optional, 8 doubles): final lambda, final robust chi2, initial robust chi2, total LM trials, ...
int orbo_lba_solve(int nP, double* posesInOut, const uint8_t* fixed, const float* cam4, int nL, double* pointsInOut, int nE,
                   const int* edgePoint, const int* edgePose, const double* obs2, const float* invSigma2, double huberDelta,
                   int iterations, double userLambdaInit, const int* stopFlag, double* edgeChi2Out, uint8_t* edgeDepthPosOut,
                   double* stats) {
    Lba L;
    L.nP = nP; L.nL = nL; L.nE = nE;
    L.poses.resize(nP); L.fixed.assign(fixed, fixed + nP); L.hidx.assign(nP, -1);
    for (int i = 0; i < nP; ++i) {
        const double* p = posesInOut + 7 * (size_t)i;
        L.poses[i].q = {p[0], p[1], p[2], p[3]};
        qnormalize(L.poses[i].q);   // SE3Quat(q, t) constructor normalises
        L.poses[i].t[0] = p[4]; L.poses[i].t[1] = p[5]; L.poses[i].t[2] = p[6];
        if (!fixed[i]) L.hidx[i] = L.nF++;
    }
    L.pts.assign(pointsInOut, pointsInOut + 3 * (size_t)nL);
    L.cam = cam4; L.ePt = edgePoint; L.ePose = edgePose; L.obs = obs2; L.invSigma2 = invSigma2;
    L.delta = huberDelta; L.dsqr = huberDelta * huberDelta;
    L.stop = stopFlag;
    L.err.assign(2 * (size_t)nE, 0.0);
    const int n = 6 * L.nF;
    L.Hpp.assign((size_t)n * n, 0.0); L.bp.assign(n, 0.0); L.Hll.assign(9 * (size_t)nL, 0.0); L.bl.assign(3 * (size_t)nL, 0.0);
    L.W.assign(18 * (size_t)nE, 0.0); L.x.assign(n + 3 * (size_t)nL, 0.0); L.Dinv.assign(9 * (size_t)nL, 0.0);
    if (stats) std::memset(stats, 0, 8 * sizeof(double));
    if (L.nF + nL == 0) return -1;

    double lambda = -1, ni = 2;
    int nBad = 0, cj = 0, trials = 0;
    const int maxTrials = 10;
    const double goodUpper = 2. / 3., goodLower = 1. / 3., tau = 1e-5;
    bool ok = true;
    double firstChi = 0;
    for (int it = 0; it < iterations && !L.terminate() && ok; ++it) {
        // OptimizationAlgorithmLevenberg::solve
        L.compute_errors();
        double currentChi = L.robust_chi2();
        double tempChi = currentChi;
        const double iniChi = currentChi;
        if (it == 0) firstChi = iniChi;
        L.build_system();
        if (it == 0) {
            if (userLambdaInit > 0) lambda = userLambdaInit;
            else {
                double maxDiag = 0;
                for (int i = 0; i < n; ++i) maxDiag = std::max(std::fabs(L.Hpp[(size_t)i * n + i]), maxDiag);
                for (int p = 0; p < nL; ++p) for (int j = 0; j < 3; ++j) maxDiag = std::max(std::fabs(L.Hll[9 * (size_t)p + 4 * j]), maxDiag);
                lambda = tau * maxDiag;
            }
            ni = 2; nBad = 0;
        }
        double rho = 0;
        int qmax = 0;
        do {
            L.posesBk = L.poses; L.ptsBk = L.pts;           // push
            const bool ok2 = L.solve(lambda);                // setLambda + solve (+ restoreDiagonal: copies are used)
            L.update();
            L.compute_errors();
            tempChi = L.robust_chi2();
            if (!ok2) tempChi = DBL_MAX;
            rho = currentChi - tempChi;
            double scale = 0;
            for (int j = 0; j < n; ++j) scale += L.x[j] * (lambda * L.x[j] + L.bp[j]);
            for (size_t j = 0; j < (size_t)3 * nL; ++j) scale += L.x[n + j] * (lambda * L.x[n + j] + L.bl[j]);
            scale += 1e-3;
            rho /= scale;
            if (rho > 0 && std::isfinite(tempChi)) {
                double alpha = 1. - std::pow((2 * rho - 1), 3);
                alpha = std::min(alpha, goodUpper);
                const double scaleFactor = std::max(goodLower, alpha);
                lambda *= scaleFactor;
                ni = 2;
                currentChi = tempChi;
            } else {
                lambda *= ni;
                ni *= 2;
                L.poses = L.posesBk; L.pts = L.ptsBk;      // pop (the edges keep the errors of the rejected state)
            }
            ++qmax; ++trials;
        } while (rho < 0 && qmax < maxTrials && !L.terminate());
        ++cj;
        if (qmax == maxTrials || rho == 0) { ok = false; }
        else {
            if ((iniChi - currentChi) * 1e3 < iniChi) ++nBad; else nBad = 0;
            if (nBad >= 3) ok = false;
        }
        if (stats) { stats[0] = lambda; stats[1] = currentChi; }
    }
    for (int i = 0; i < nP; ++i) {
        double* p = posesInOut + 7 * (size_t)i;
        p[0] = L.poses[i].q.w; p[1] = L.poses[i].q.x; p[2] = L.poses[i].q.y; p[3] = L.poses[i].q.z;
        p[4] = L.poses[i].t[0]; p[5] = L.poses[i].t[1]; p[6] = L.poses[i].t[2];
    }
    std::memcpy(pointsInOut, L.pts.data(), sizeof(double) * 3 * (size_t)nL);
    for (int e = 0; e < nE; ++e) {
        if (edgeChi2Out) edgeChi2Out[e] = L.chi2(e);       // e->chi2(): from the last computed _error (Optimizer.cc:1425)
        if (edgeDepthPosOut) { double Xc[3], uv[2]; L.project_edge(e, Xc, uv); edgeDepthPosOut[e] = Xc[2] > 0.0; }
    }
    if (stats) { stats[2] = firstChi; stats[3] = trials; stats[4] = cj; }
    return cj;
}

// ---- the same state opened step by step (OrboLmBackend, oracle_common.h) ----
namespace {
struct LbaOpen {
    Lba L;
    std::vector<float> cam, is2; std::vector<int> ePt, ePose; std::vector<double> obs;
    std::vector<double> bcat, diag;
};
void lbo_compute_errors(void* p) { ((LbaOpen*)p)->L.compute_errors(); }
double lbo_robust_chi2(void* p) { return ((LbaOpen*)p)->L.robust_chi2(); }
void lbo_build_system(void* p) {
    LbaOpen* o = (LbaOpen*)p; Lba& L = o->L;
    L.build_system();
    const int n = 6 * L.nF;
    o->bcat.assign(L.bp.begin(), L.bp.end()); o->bcat.insert(o->bcat.end(), L.bl.begin(), L.bl.end());
    o->diag.clear();
    for (int i = 0; i < n; ++i) o->diag.push_back(L.Hpp[(size_t)i * n + i]);
    for (int q = 0; q < L.nL; ++q) for (int j = 0; j < 3; ++j) o->diag.push_back(L.Hll[9 * (size_t)q + 4 * j]);
}
int lbo_solve(void* p, double lambda) { return ((LbaOpen*)p)->L.solve(lambda) ? 1 : 0; }
void lbo_update(void* p) { ((LbaOpen*)p)->L.update(); }
void lbo_push(void* p) { Lba& L = ((LbaOpen*)p)->L; L.posesBk = L.poses; L.ptsBk = L.pts; }
void lbo_pop(void* p) { Lba& L = ((LbaOpen*)p)->L; L.poses = L.posesBk; L.pts = L.ptsBk; }
int lbo_vector_size(void* p) { Lba& L = ((LbaOpen*)p)->L; return 6 * L.nF + 3 * L.nL; }
const double* lbo_x(void* p) { return ((LbaOpen*)p)->L.x.data(); }
const double* lbo_b(void* p) { return ((LbaOpen*)p)->bcat.data(); }
int lbo_n_diag(void* p) { return (int)((LbaOpen*)p)->diag.size(); }
const double* lbo_diag(void* p) { return ((LbaOpen*)p)->diag.data(); }
}  // namespace

// arguments as orbo_lba_solve (copied: the caller's arrays need not outlive the call)
void orbo_lba_backend_open(int nP, const double* poses7, const uint8_t* fixed, const float* cam4, int nL, const double* points3, int nE, const int* edgePoint, const int* edgePose,
                           const double* obs2, const float* invSigma2, double huberDelta, OrboLmBackend* out) {
    LbaOpen* o = new LbaOpen;
    o->cam.assign(cam4, cam4 + 4 * (size_t)nP); o->is2.assign(invSigma2, invSigma2 + nE); o->ePt.assign(edgePoint, edgePoint + nE); o->ePose.assign(edgePose, edgePose + nE);
    o->obs.assign(obs2, obs2 + 2 * (size_t)nE);
    Lba& L = o->L;
    L.nP = nP; L.nL = nL; L.nE = nE;
    L.poses.resize(nP); L.fixed.assign(fixed, fixed + nP); L.hidx.assign(nP, -1);
    for (int i = 0; i < nP; ++i) {
        const double* p = poses7 + 7 * (size_t)i;
        L.poses[i].q = {p[0], p[1], p[2], p[3]};
        qnormalize(L.poses[i].q);
        L.poses[i].t[0] = p[4]; L.poses[i].t[1] = p[5]; L.poses[i].t[2] = p[6];
        if (!fixed[i]) L.hidx[i] = L.nF++;
    }
    L.pts.assign(points3, points3 + 3 * (size_t)nL);
    L.cam = o->cam.data(); L.ePt = o->ePt.data(); L.ePose = o->ePose.data(); L.obs = o->obs.data(); L.invSigma2 = o->is2.data();
    L.delta = huberDelta; L.dsqr = huberDelta * huberDelta; L.stop = nullptr;
    L.err.assign(2 * (size_t)nE, 0.0);
    const int n = 6 * L.nF;
    L.Hpp.assign((size_t)n * n, 0.0); L.bp.assign(n, 0.0); L.Hll.assign(9 * (size_t)nL, 0.0); L.bl.assign(3 * (size_t)nL, 0.0);
    L.W.assign(18 * (size_t)nE, 0.0); L.x.assign(n + 3 * (size_t)nL, 0.0); L.Dinv.assign(9 * (size_t)nL, 0.0);
    *out = OrboLmBackend{o, lbo_compute_errors, lbo_robust_chi2, lbo_build_system, lbo_solve, lbo_update, lbo_push, lbo_pop, lbo_vector_size, lbo_x, lbo_b, lbo_n_diag, lbo_diag};
}
void orbo_lba_backend_close(OrboLmBackend* be, double* posesOut7, double* pointsOut3) {
    LbaOpen* o = (LbaOpen*)be->self; Lba& L = o->L;
    for (int i = 0; i < L.nP; ++i) {
        double* p = posesOut7 + 7 * (size_t)i;
        p[0] = L.poses[i].q.w; p[1] = L.poses[i].q.x; p[2] = L.poses[i].q.y; p[3] = L.poses[i].q.z; p[4] = L.poses[i].t[0]; p[5] = L.poses[i].t[1]; p[6] = L.poses[i].t[2];
    }
    std::memcpy(pointsOut3, L.pts.data(), sizeof(double) * 3 * (size_t)L.nL);
    delete o;
    be->self = nullptr;
}

// the per-edge numerics on their own, for tests/test_ref_pins_lba_edges_cpu.py (the functions the solvers above call)
//   err [2] = obs - project(T.map(X)); Jpoint [2][3], Jpose [2][6] = EdgeSE3ProjectXYZ::linearizeOplus; JposeOnly [2][6] = EdgeSE3ProjectXYZOnlyPose::linearizeOplus
void orbo_lba_edge(const double* pose7, const float* cam4, const double* X3, const double* obs2, double* err2, double* Jpoint, double* Jpose, double* JposeOnly, int* depthPositive) {
    Quat q = {pose7[0], pose7[1], pose7[2], pose7[3]};
    qnormalize(q);
    double r[3]; qrot(q, X3, r);
    const double Xc[3] = {r[0] + pose7[4], r[1] + pose7[5], r[2] + pose7[6]};
    err2[0] = obs2[0] - ((double)cam4[0] * Xc[0] / Xc[2] + (double)cam4[2]);
    err2[1] = obs2[1] - ((double)cam4[1] * Xc[1] / Xc[2] + (double)cam4[3]);
    edge_jacobians(q, cam4, Xc, Jpoint, Jpose);
    only_pose_jacobian(cam4, Xc[0], Xc[1], Xc[2], JposeOnly);
    *depthPositive = Xc[2] > 0.0;
}
void orbo_huber(double delta, double e, double* rho3) { Lba L; L.delta = delta; L.dsqr = delta * delta; L.robustify(e, rho3); }
// SE3Quat::exp(update) * T (VertexSE3Expmap::oplusImpl), pose7 in/out
void orbo_lba_pose_oplus(double* pose7, const double* update6) {
    Pose T; T.q = {pose7[0], pose7[1], pose7[2], pose7[3]}; qnormalize(T.q); T.t[0] = pose7[4]; T.t[1] = pose7[5]; T.t[2] = pose7[6];
    pose_oplus(T, update6);
    pose7[0] = T.q.w; pose7[1] = T.q.x; pose7[2] = T.q.y; pose7[3] = T.q.z; pose7[4] = T.t[0]; pose7[5] = T.t[1]; pose7[6] = T.t[2];
}

// reprojection residuals (obs - proj) of a state, for the 1e-4 px parity bar
void orbo_lba_residuals(int nP, const double* poses7, const float* cam4, int nL, const double* points3, int nE, const int* edgePoint,
                        const int* edgePose, const double* obs2, double* res2) {
    for (int e = 0; e < nE; ++e) {
        const double* p = poses7 + 7 * (size_t)edgePose[e];
        Quat q = {p[0], p[1], p[2], p[3]};
        double r[3]; qrot(q, points3 + 3 * (size_t)edgePoint[e], r);
        const double X = r[0] + p[4], Y = r[1] + p[5], Z = r[2] + p[6];
        const float* c = cam4 + 4 * (size_t)edgePose[e];
        res2[2 * (size_t)e] = obs2[2 * (size_t)e] - ((double)c[0] * X / Z + (double)c[2]);
        res2[2 * (size_t)e + 1] = obs2[2 * (size_t)e + 1] - ((double)c[1] * Y / Z + (double)c[3]);
    }
    (void)nP; (void)nL;
}


// ---------------------------------------------------------------------------------------------------------
// Optimizer::PoseOptimization (reference src/Optimizer.cc:814-1114, monocular branch): one VertexSE3Expmap,
// EdgeSE3ProjectXYZOnlyPose per matched keypoint (include/OptimizableTypes.h:31-57, src/OptimizableTypes.cpp:49-63),
// BaseUnaryEdge::constructQuadraticForm (g2o/core/base_unary_edge.hpp:43-72), LinearSolverDense (6x6 LDLT).
// 4 rounds x optimize(10), every round restarts from the frame's pose; outliers (chi2 > 5.991) leave the active set
// (level 1) and can come back; the Huber kernel is removed after the third round (:1040-1041).
// Returns nInitialCorrespondences - nBad.  pose7 in/out, outlier[N] out.  stats (optional, 4 doubles): LM trials, LM iterations that
// ended after maxTrials rejected trials (qmax == 10), iterations that ended with rho == 0, rounds run.
// ---------------------------------------------------------------------------------------------------------
}  // extern "C" (reopened below: the pose-only problem is a struct shared by the solver and its step-by-step form)

namespace orbo {
struct PoseOpt {
    int N; const float* cam4; const double *Xw3, *obs2; const float* invSigma2; double delta, dsqr;
    Pose T, Tbk;
    std::vector<double> err; std::vector<uint8_t> level, robust;
    double H[36], b[6], xs[6];      // xs: the solver's x vector keeps its previous content when the factorisation fails
    void compute_error(int e) {
        double r[3]; qrot(T.q, Xw3 + 3 * (size_t)e, r);
        const double X = r[0] + T.t[0], Y = r[1] + T.t[1], Z = r[2] + T.t[2];
        err[2 * (size_t)e] = obs2[2 * (size_t)e] - ((double)cam4[0] * X / Z + (double)cam4[2]);
        err[2 * (size_t)e + 1] = obs2[2 * (size_t)e + 1] - ((double)cam4[1] * Y / Z + (double)cam4[3]);
    }
    double chi2(int e) const { return (double)invSigma2[e] * (err[2 * (size_t)e] * err[2 * (size_t)e] + err[2 * (size_t)e + 1] * err[2 * (size_t)e + 1]); }
    void robustify(int e, double e2, double* rho) const {
        if (!robust[e] || e2 <= dsqr) { rho[0] = e2; rho[1] = 1.; }
        else { const double s = std::sqrt(e2); rho[0] = 2 * s * delta - dsqr; rho[1] = delta / s; }
    }
    void compute_active_errors() { for (int e = 0; e < N; ++e) if (!level[e]) compute_error(e); }
    double active_chi2() const { double c = 0, rho[2]; for (int e = 0; e < N; ++e) if (!level[e]) { robustify(e, chi2(e), rho); c += rho[0]; } return c; }
    int n_active() const { int n = 0; for (int e = 0; e < N; ++e) n += !level[e]; return n; }
    void build() {
        for (double& v : H) v = 0;
        for (double& v : b) v = 0;
        for (int e = 0; e < N; ++e) {
            if (level[e]) continue;
            double r[3]; qrot(T.q, Xw3 + 3 * (size_t)e, r);
            const double x = r[0] + T.t[0], y = r[1] + T.t[1], z = r[2] + T.t[2];
            double B[12];
            only_pose_jacobian(cam4, x, y, z, B);
            double rho[2]; robustify(e, chi2(e), rho);
            const double w = rho[1] * (double)invSigma2[e];
            const double r0 = (double)invSigma2[e] * err[2 * (size_t)e], r1 = (double)invSigma2[e] * err[2 * (size_t)e + 1];
            for (int a = 0; a < 6; ++a) {
                b[a] -= rho[1] * (B[a] * r0 + B[6 + a] * r1);
                for (int c = 0; c < 6; ++c) H[a * 6 + c] += w * (B[a] * B[c] + B[6 + a] * B[6 + c]);
            }
        }
    }
    bool solve(double lambda) {         // LinearSolverDense: Eigen::LDLT + isPositive(); x untouched on failure
        std::vector<double> A(H, H + 36); for (int a = 0; a < 6; ++a) A[a * 7] += lambda;
        double x6[6] = {0, 0, 0, 0, 0, 0};
        bool ok2 = ldlt_solve(A, 6, b, x6);
        if (ok2) for (int a = 0; a < 6; ++a) if (A[a * 7] < 0) ok2 = false;
        if (ok2) for (int a = 0; a < 6; ++a) xs[a] = x6[a];
        return ok2;
    }
    void update() { pose_oplus(T, xs); }
};
}  // namespace orbo

extern "C" {

int orbo_pose_optimization(double* pose7, const float* cam4, int N, const double* Xw3, const double* obs2, const float* invSigma2,
                           double huberDelta, uint8_t* outlier, double* stats) {
    if (N < 3) {   // if(nInitialCorrespondences<3) return 0; (src/Optimizer.cc:996-997): the frame's pose is not touched
        for (int i = 0; i < N; ++i) outlier[i] = 0;
        if (stats) for (int i = 0; i < 4; ++i) stats[i] = 0;
        return 0;
    }
    PoseOpt P;
    P.N = N; P.cam4 = cam4; P.Xw3 = Xw3; P.obs2 = obs2; P.invSigma2 = invSigma2; P.delta = huberDelta; P.dsqr = huberDelta * huberDelta;
    Pose T0; T0.q = {pose7[0], pose7[1], pose7[2], pose7[3]}; qnormalize(T0.q); T0.t[0] = pose7[4]; T0.t[1] = pose7[5]; T0.t[2] = pose7[6];
    P.T = T0;
    P.err.assign(2 * (size_t)N, 0.0); P.level.assign(N, 0); P.robust.assign(N, 1);
    for (double& v : P.xs) v = 0;
    for (int i = 0; i < N; ++i) outlier[i] = 0;
    int nBad = 0, totalTrials = 0, nExhausted = 0, nRhoZero = 0, rounds = 0;
    for (int round = 0; round < 4; ++round) {
        ++rounds;
        P.T = T0;
        const int nActive = P.n_active();
        // optimizer.optimize(10)
        double lambda = -1, ni = 2; int nBadLM = 0; bool ok = true;
        for (int it = 0; it < 10 && ok && nActive > 0; ++it) {
            P.compute_active_errors();
            double currentChi = P.active_chi2(), tempChi = currentChi; const double iniChi = currentChi;
            P.build();
            if (it == 0) { double md = 0; for (int a = 0; a < 6; ++a) md = std::max(md, std::fabs(P.H[a * 7])); lambda = 1e-5 * md; ni = 2; nBadLM = 0; }
            double rho = 0; int qmax = 0;
            do {
                P.Tbk = P.T;
                const bool ok2 = P.solve(lambda);
                P.update();
                P.compute_active_errors();
                tempChi = P.active_chi2();
                if (!ok2) tempChi = DBL_MAX;
                rho = currentChi - tempChi;
                double scale = 0; for (int a = 0; a < 6; ++a) scale += P.xs[a] * (lambda * P.xs[a] + P.b[a]);
                scale += 1e-3; rho /= scale;
                if (rho > 0 && std::isfinite(tempChi)) {
                    double alpha = 1. - std::pow((2 * rho - 1), 3); alpha = std::min(alpha, 2. / 3.);
                    lambda *= std::max(1. / 3., alpha); ni = 2; currentChi = tempChi;
                } else { lambda *= ni; ni *= 2; P.T = P.Tbk; }
                ++qmax; ++totalTrials;
            } while (rho < 0 && qmax < 10);
            nExhausted += qmax == 10; nRhoZero += rho == 0;
            if (qmax == 10 || rho == 0) ok = false;
            else { if ((iniChi - currentChi) * 1e3 < iniChi) ++nBadLM; else nBadLM = 0; if (nBadLM >= 3) ok = false; }
        }
        nBad = 0;
        for (int e = 0; e < N; ++e) {
            if (outlier[e]) P.compute_error(e);
            if ((float)P.chi2(e) > 5.991f) { outlier[e] = 1; P.level[e] = 1; ++nBad; }     // const float chi2 = e->chi2(); chi2 > chi2Mono[it] (:1025-1027)
            else { outlier[e] = 0; P.level[e] = 0; }
            if (round == 2) P.robust[e] = 0;
        }
        if (N < 10) break;
    }
    pose7[0] = P.T.q.w; pose7[1] = P.T.q.x; pose7[2] = P.T.q.y; pose7[3] = P.T.q.z; pose7[4] = P.T.t[0]; pose7[5] = P.T.t[1]; pose7[6] = P.T.t[2];
    if (stats) { stats[0] = totalTrials; stats[1] = nExhausted; stats[2] = nRhoZero; stats[3] = rounds; }
    return N - nBad;
}

// ---- the pose-only problem opened step by step: OrboLmBackend for g2o's optimize() text + the per-edge operations the four-round loop of
//      Optimizer::PoseOptimization (src/Optimizer.cc:1005-1104) performs (oracle/ref_shim/ref_wrap_g2o_lm.cpp compiles that loop verbatim) ----
namespace {
struct PoseOptOpen { PoseOpt P; std::vector<float> cam, is2; std::vector<double> X, obs; double diag[6]; };
void ppo_compute_errors(void* p) { ((PoseOptOpen*)p)->P.compute_active_errors(); }
double ppo_robust_chi2(void* p) { return ((PoseOptOpen*)p)->P.active_chi2(); }
void ppo_build_system(void* p) { PoseOptOpen* o = (PoseOptOpen*)p; o->P.build(); for (int a = 0; a < 6; ++a) o->diag[a] = o->P.H[a * 7]; }
int ppo_solve(void* p, double lambda) { return ((PoseOptOpen*)p)->P.solve(lambda) ? 1 : 0; }
void ppo_update(void* p) { ((PoseOptOpen*)p)->P.update(); }
void ppo_push(void* p) { PoseOpt& P = ((PoseOptOpen*)p)->P; P.Tbk = P.T; }
void ppo_pop(void* p) { PoseOpt& P = ((PoseOptOpen*)p)->P; P.T = P.Tbk; }
int ppo_vector_size(void*) { return 6; }
const double* ppo_x(void* p) { return ((PoseOptOpen*)p)->P.xs; }
const double* ppo_b(void* p) { return ((PoseOptOpen*)p)->P.b; }
int ppo_n_diag(void*) { return 6; }
const double* ppo_diag(void* p) { return ((PoseOptOpen*)p)->diag; }
}  // namespace
void orbo_poseopt_open(const float* cam4, int N, const double* Xw3, const double* obs2, const float* invSigma2, double huberDelta, OrboLmBackend* out) {
    PoseOptOpen* o = new PoseOptOpen;
    o->cam.assign(cam4, cam4 + 4); o->is2.assign(invSigma2, invSigma2 + N); o->X.assign(Xw3, Xw3 + 3 * (size_t)N); o->obs.assign(obs2, obs2 + 2 * (size_t)N);
    PoseOpt& P = o->P;
    P.N = N; P.cam4 = o->cam.data(); P.Xw3 = o->X.data(); P.obs2 = o->obs.data(); P.invSigma2 = o->is2.data(); P.delta = huberDelta; P.dsqr = huberDelta * huberDelta;
    P.T.q = {1, 0, 0, 0}; P.T.t[0] = P.T.t[1] = P.T.t[2] = 0;
    P.err.assign(2 * (size_t)N, 0.0); P.level.assign(N, 0); P.robust.assign(N, 1);
    for (double& v : P.xs) v = 0;
    for (double& v : o->diag) v = 0;
    *out = OrboLmBackend{o, ppo_compute_errors, ppo_robust_chi2, ppo_build_system, ppo_solve, ppo_update, ppo_push, ppo_pop, ppo_vector_size, ppo_x, ppo_b, ppo_n_diag, ppo_diag};
}
void orbo_poseopt_set_estimate(void* h, const double* pose7) {      // vSE3->setEstimate(g2o::SE3Quat(q, t)): the constructor normalises
    PoseOpt& P = ((PoseOptOpen*)h)->P;
    P.T.q = {pose7[0], pose7[1], pose7[2], pose7[3]}; qnormalize(P.T.q); P.T.t[0] = pose7[4]; P.T.t[1] = pose7[5]; P.T.t[2] = pose7[6];
}
void orbo_poseopt_get_estimate(void* h, double* pose7) {
    const PoseOpt& P = ((PoseOptOpen*)h)->P;
    pose7[0] = P.T.q.w; pose7[1] = P.T.q.x; pose7[2] = P.T.q.y; pose7[3] = P.T.q.z; pose7[4] = P.T.t[0]; pose7[5] = P.T.t[1]; pose7[6] = P.T.t[2];
}
void orbo_poseopt_edge_compute_error(void* h, int e) { ((PoseOptOpen*)h)->P.compute_error(e); }
double orbo_poseopt_edge_chi2(void* h, int e) { return ((PoseOptOpen*)h)->P.chi2(e); }
void orbo_poseopt_edge_set_level(void* h, int e, int level) { ((PoseOptOpen*)h)->P.level[e] = (uint8_t)level; }
void orbo_poseopt_edge_set_robust(void* h, int e, int on) { ((PoseOptOpen*)h)->P.robust[e] = (uint8_t)on; }
int orbo_poseopt_active(void* h) { return ((PoseOptOpen*)h)->P.n_active(); }
void orbo_poseopt_close(void* h) { delete (PoseOptOpen*)h; }

}  // extern "C"

// EdgeSE3ProjectXYZOnlyPose::linearizeOplus (src/OptimizableTypes.cpp:49-63): -projectJac * SE3deriv, written out
static void only_pose_jacobian(const float* cam4, double x, double y, double z, double* B) {
    const double fx = cam4[0], fy = cam4[1];
    const double J00 = -(fx / z), J02 = fx * x / (z * z), J11 = -(fy / z), J12 = fy * y / (z * z);
    const double v[12] = {J02 * y, J00 * z - J02 * x, -J00 * y, J00, 0, J02, -J11 * z + J12 * y, -J12 * x, J11 * x, 0, J11, J12};
    for (int i = 0; i < 12; ++i) B[i] = v[i];
}
