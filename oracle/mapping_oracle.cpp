// TEST INFRASTRUCTURE ONLY -- CPU oracle of LocalMapping::CreateNewMapPoints (src/LocalMapping.cc, the vpNeighKFs loop from :296) for
// monocular keyframes, with GeometricTools::Triangulate (src/GeometricTools.cc) and the part of MapPoint::UpdateNormalAndDepth
// (src/MapPoint.cc) a new two-observation point needs.
//
// Evaluation order.  The Eigen / Sophus expressions are evaluated uncontracted (this file is built with -ffp-contract=off):
//   * unprojectEig: xn = ((u - cx) / fx, (v - cy) / fy, 1);
//   * a matrix-vector product and a dot product sum their terms in ascending index order: ((a0 b0 + a1 b1) + a2 b2);
//   * norm() = sqrt of the squared norm summed the same way;
//   * Triangulate's rows are x * T.row(2) - T.row(0), element by element (one product, one difference).
// The plain float statements of the function body are contracted as the reference's -O3 -march=native build contracts them: of the
// statements on this path only errX*errX + errY*errY has a product feeding an addition; it is fmaf(errX, errX, errY * errY), as
// `ex*ex+ey*ey` in Fuse (DESIGN.md section 2).  Constants written as double literals (0.9998, 0.9996, 5.991) compare in double.
//
// Triangulate's Eigen::JacobiSVD<Matrix4f>(A, ComputeFullV) is restated as Eigen's two-sided cyclic Jacobi SVD in float: scale by the
// largest |a_ij|, sweep the pairs (p, q) with p = 1..3, q < p while an off-diagonal entry exceeds max(FLT_MIN, 2 eps maxDiagEntry),
// each pair diagonalised by real_2x2_jacobi_svd (one rotation to make the block symmetric, then makeJacobi), then the singular values
// sorted in decreasing order (first maximum wins, columns of V swapped with them).  Eigen has no sweep limit; this restatement stops
// after NP_MAX_SWEEPS sweeps, which a float 4x4 never reaches (it converges in a handful).  Without Eigen here, bit agreement with
// Eigen's build is not claimed: the same standing as NormalizeRotation (DESIGN.md section 2).
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "oracle_common.h"

using orbo::KeyPoint;

extern "C" int orbo_search_for_triangulation(int N1, const KeyPoint* kps1, const uint8_t* desc1, const uint8_t* hasMP1, int E1, const int* fvNode1, const int* fvFeat1,
                                  int N2, const KeyPoint* kps2, const uint8_t* desc2, const uint8_t* hasMP2, int E2, const int* fvNode2, const int* fvFeat2,
                                  const float* scaleFactors2, const float* levelSigma2_2, const float* ep, const float* F12, int bCoarse, int checkOri,
                                  int* matches12);

extern "C" {
// Layout-compatible with OrbmTriFrame / OrbmNewPointsIn / OrbmNewPoint (include/orb_b200.h).
typedef struct OrboTriFrame {
    int N; const KeyPoint* keypoints; const uint8_t* descriptors; const uint8_t* hasMapPoint;
    int nEntries; const int32_t* fvNode; const int32_t* fvFeature;
} OrboTriFrame;
typedef struct OrboNewPointsIn {
    const OrboTriFrame* KF1; int nKF2; const OrboTriFrame* KF2;
    const float* ep2; const float* F12;
    const float* scaleFactors; const float* levelSigma2; int nlevels;
    const float* Tcw; const float* Ow; const float* cam;
    float scaleFactor; int bCoarse; int bInertial; float thFarPoints;
} OrboNewPointsIn;
typedef struct OrboNewPoint {
    int32_t kf2, idx1, idx2; float x3D[3]; float normal[3]; float minDistance, maxDistance;
} OrboNewPoint;
}

namespace {

// Reason codes of one (neighbour, idx1) match, in the order the reference tests them.
enum : uint8_t { NP_NO_MATCH = 0, NP_LOW_PARALLAX, NP_SVD_W0, NP_DEPTH1, NP_DEPTH2, NP_REPROJ1, NP_REPROJ2, NP_ZERO_DIST, NP_FAR, NP_SCALE, NP_CREATED,
                 NP_TAKEN };      // NP_TAKEN: the static search matched idx1, but an earlier neighbour created its point (the reference never sees it)
constexpr int NP_MAX_SWEEPS = 64;

struct Rot { float c, s; };

// Eigen: JacobiRotation::makeJacobi(x, y, z) for real scalars (Jacobi.h)
Rot make_jacobi(float x, float y, float z) {
    const float deno = 2.0f * std::fabs(y);
    if (deno < FLT_MIN) return {1.0f, 0.0f};
    const float tau = (x - z) / deno;
    const float w = std::sqrt(tau * tau + 1.0f);
    const float t = tau > 0.0f ? 1.0f / (tau + w) : 1.0f / (tau - w);
    const float sign_t = t > 0.0f ? 1.0f : -1.0f;
    const float n = 1.0f / std::sqrt(t * t + 1.0f);
    return {n, -sign_t * (y / std::fabs(y)) * std::fabs(t) * n};
}

// x = c x + s y, y = -s x + c y over row (left) or column (right) p, q
void rot_rows(float W[4][4], int p, int q, Rot j) {
    for (int i = 0; i < 4; ++i) { const float x = W[p][i], y = W[q][i]; W[p][i] = j.c * x + j.s * y; W[q][i] = -j.s * x + j.c * y; }
}
void rot_cols(float W[4][4], int p, int q, Rot j) {
    for (int i = 0; i < 4; ++i) { const float x = W[i][p], y = W[i][q]; W[i][p] = j.c * x + j.s * y; W[i][q] = -j.s * x + j.c * y; }
}

}  // namespace

extern "C" {

// GeometricTools::Triangulate(x_c1, x_c2, Tc1w, Tc2w, x3D): 1 and x3D, or 0 when V(3, 3) of the smallest singular value is 0.
// Tc1w / Tc2w: float 3x4 row-major.  V [16] (optional, row-major): V after sorting.
int orbo_triangulate(float x1, float y1, float x2, float y2, const float* T1, const float* T2, float* x3D, float* Vout) {
    float A[4][4];
    for (int j = 0; j < 4; ++j) {
        A[0][j] = x1 * T1[8 + j] - T1[j];
        A[1][j] = y1 * T1[8 + j] - T1[4 + j];
        A[2][j] = x2 * T2[8 + j] - T2[j];
        A[3][j] = y2 * T2[8 + j] - T2[4 + j];
    }
    // JacobiSVD::compute (JacobiSVD.h): square input, so no QR preconditioner
    float scale = 0.0f;
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) scale = std::max(scale, std::fabs(A[i][j]));
    if (scale == 0.0f) scale = 1.0f;
    float W[4][4], V[4][4];
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) { W[i][j] = A[i][j] / scale; V[i][j] = i == j ? 1.0f : 0.0f; }
    const float considerAsZero = FLT_MIN, precision = 2.0f * FLT_EPSILON;
    float maxDiagEntry = 0.0f;
    for (int i = 0; i < 4; ++i) maxDiagEntry = std::max(maxDiagEntry, std::fabs(W[i][i]));
    bool finished = false;
    for (int sweep = 0; !finished && sweep < NP_MAX_SWEEPS; ++sweep) {
        finished = true;
        for (int p = 1; p < 4; ++p) for (int q = 0; q < p; ++q) {
            const float threshold = std::max(considerAsZero, precision * maxDiagEntry);
            if (!(std::fabs(W[p][q]) > threshold || std::fabs(W[q][p]) > threshold)) continue;
            finished = false;
            // real_2x2_jacobi_svd(W, p, q, &j_left, &j_right)
            float m00 = W[p][p], m01 = W[p][q], m10 = W[q][p], m11 = W[q][q];
            Rot rot1;
            const float t = m00 + m11, d = m10 - m01;
            if (std::fabs(d) < FLT_MIN) rot1 = {1.0f, 0.0f};
            else {
                const float u = t / d;
                const float tmp = std::sqrt(1.0f + u * u);
                rot1 = {u / tmp, 1.0f / tmp};
            }
            // m.applyOnTheLeft(0, 1, rot1)
            const float n00 = rot1.c * m00 + rot1.s * m10, n01 = rot1.c * m01 + rot1.s * m11;
            const float n11 = -rot1.s * m01 + rot1.c * m11;
            m00 = n00; m01 = n01; m11 = n11;
            const Rot jr = make_jacobi(m00, m01, m11);
            // j_left = rot1 * j_right.transpose(): (c1 c2 - s1 s2', c1 s2' + s1 c2) with s2' = -s2
            const Rot jrt = {jr.c, -jr.s};
            const Rot jl = {rot1.c * jrt.c - rot1.s * jrt.s, rot1.c * jrt.s + rot1.s * jrt.c};
            rot_rows(W, p, q, jl);                                 // W.applyOnTheLeft(p, q, j_left)
            rot_cols(W, p, q, {jr.c, -jr.s});                      // W.applyOnTheRight(p, q, j_right): the transposed rotation on the columns
            rot_cols(V, p, q, {jr.c, -jr.s});                      // V.applyOnTheRight(p, q, j_right)
            maxDiagEntry = std::max(maxDiagEntry, std::max(std::fabs(W[p][p]), std::fabs(W[q][q])));
        }
    }
    float s[4];
    for (int i = 0; i < 4; ++i) s[i] = std::fabs(W[i][i]);
    for (int i = 0; i < 4; ++i) {                                   // sort, first maximum wins
        int pos = i;
        for (int k = i + 1; k < 4; ++k) if (s[k] > s[pos]) pos = k;
        if (s[pos] == 0.0f) break;
        if (pos != i) {
            std::swap(s[i], s[pos]);
            for (int r = 0; r < 4; ++r) std::swap(V[r][i], V[r][pos]);
        }
    }
    if (Vout) for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) Vout[4 * i + j] = V[i][j];
    const float w = V[3][3];
    if (w == 0.0f) return 0;
    x3D[0] = V[0][3] / w; x3D[1] = V[1][3] / w; x3D[2] = V[2][3] / w;
    return 1;
}

// The checks of src/LocalMapping.cc CreateNewMapPoints for one match (idx1 of KF1, idx2 of neighbour k), monocular keyframes: the reason code,
// and for NP_CREATED the new point with MapPoint::UpdateNormalAndDepth's normal and distances (reference keyframe = KF1).
int orbo_new_point_for_match(const OrboNewPointsIn* in, int k, int idx1, int idx2, OrboNewPoint* rec) {
    const KeyPoint& kp1 = in->KF1->keypoints[idx1];
    const KeyPoint& kp2 = in->KF2[k].keypoints[idx2];
    const float* T1 = in->Tcw; const float* T2 = in->Tcw + 12 * (size_t)(k + 1);
    const float* O1 = in->Ow; const float* O2 = in->Ow + 3 * (size_t)(k + 1);
    const float* c1 = in->cam; const float* c2 = in->cam + 4 * (size_t)(k + 1);
    // Pinhole::unprojectEig, ray = Rwc * xn with Rwc = Rcw^T
    const float xn1[3] = {(kp1.x - c1[2]) / c1[0], (kp1.y - c1[3]) / c1[1], 1.0f};
    const float xn2[3] = {(kp2.x - c2[2]) / c2[0], (kp2.y - c2[3]) / c2[1], 1.0f};
    float ray1[3], ray2[3];
    for (int i = 0; i < 3; ++i) {
        ray1[i] = (T1[i] * xn1[0] + T1[4 + i] * xn1[1]) + T1[8 + i] * xn1[2];
        ray2[i] = (T2[i] * xn2[0] + T2[4 + i] * xn2[1]) + T2[8 + i] * xn2[2];
    }
    const float dot = (ray1[0] * ray2[0] + ray1[1] * ray2[1]) + ray1[2] * ray2[2];
    const float n1 = std::sqrt((ray1[0] * ray1[0] + ray1[1] * ray1[1]) + ray1[2] * ray1[2]);
    const float n2 = std::sqrt((ray2[0] * ray2[0] + ray2[1] * ray2[1]) + ray2[2] * ray2[2]);
    const float cosParallaxRays = dot / (n1 * n2);
    const float cosParallaxStereo = cosParallaxRays + 1;                                          // no stereo: min(cosParallaxStereo1, 2) = this
    if (!(cosParallaxRays < cosParallaxStereo && cosParallaxRays > 0 &&
          ((in->bInertial && cosParallaxRays < 0.9996) || (!in->bInertial && cosParallaxRays < 0.9998))))
        return NP_LOW_PARALLAX;
    float x3D[3];
    if (!orbo_triangulate(xn1[0], xn1[1], xn2[0], xn2[1], T1, T2, x3D, nullptr)) return NP_SVD_W0;
    auto row = [&](const float* T, int r) { return ((T[4 * r] * x3D[0] + T[4 * r + 1] * x3D[1]) + T[4 * r + 2] * x3D[2]) + T[4 * r + 3]; };
    const float z1 = row(T1, 2);
    if (z1 <= 0) return NP_DEPTH1;
    const float z2 = row(T2, 2);
    if (z2 <= 0) return NP_DEPTH2;
    {
        const float sigmaSquare1 = in->levelSigma2[kp1.octave];
        const float x1 = row(T1, 0), y1 = row(T1, 1);
        const float u = c1[0] * x1 / z1 + c1[2], v = c1[1] * y1 / z1 + c1[3];                  // Pinhole::project(cv::Point3f)
        const float errX1 = u - kp1.x, errY1 = v - kp1.y;
        if (fmaf(errX1, errX1, errY1 * errY1) > 5.991 * sigmaSquare1) return NP_REPROJ1;
    }
    {
        const float sigmaSquare2 = in->levelSigma2[kp2.octave];
        const float x2 = row(T2, 0), y2 = row(T2, 1);
        const float u = c2[0] * x2 / z2 + c2[2], v = c2[1] * y2 / z2 + c2[3];
        const float errX2 = u - kp2.x, errY2 = v - kp2.y;
        if (fmaf(errX2, errX2, errY2 * errY2) > 5.991 * sigmaSquare2) return NP_REPROJ2;
    }
    const float nv1[3] = {x3D[0] - O1[0], x3D[1] - O1[1], x3D[2] - O1[2]};
    const float nv2[3] = {x3D[0] - O2[0], x3D[1] - O2[1], x3D[2] - O2[2]};
    const float dist1 = std::sqrt((nv1[0] * nv1[0] + nv1[1] * nv1[1]) + nv1[2] * nv1[2]);
    const float dist2 = std::sqrt((nv2[0] * nv2[0] + nv2[1] * nv2[1]) + nv2[2] * nv2[2]);
    if (dist1 == 0 || dist2 == 0) return NP_ZERO_DIST;
    if (in->thFarPoints > 0 && (dist1 >= in->thFarPoints || dist2 >= in->thFarPoints)) return NP_FAR;
    const float ratioDist = dist2 / dist1;
    const float ratioOctave = in->scaleFactors[kp1.octave] / in->scaleFactors[kp2.octave];
    const float ratioFactor = 1.5f * in->scaleFactor;
    if (ratioDist * ratioFactor < ratioOctave || ratioDist > ratioOctave * ratioFactor) return NP_SCALE;
    // MapPoint::UpdateNormalAndDepth: normal = (0 + n1/|n1| + n2/|n2|) / 2, PC = Pos - Ow(refKF = KF1)
    rec->kf2 = k; rec->idx1 = idx1; rec->idx2 = idx2;
    for (int i = 0; i < 3; ++i) {
        rec->x3D[i] = x3D[i];
        rec->normal[i] = ((0.0f + nv1[i] / dist1) + nv2[i] / dist2) / 2.0f;
    }
    rec->maxDistance = dist1 * in->scaleFactors[kp1.octave];
    rec->minDistance = rec->maxDistance / in->scaleFactors[in->nlevels - 1];
    return NP_CREATED;
}

// The whole vpNeighKFs loop for one new keyframe, restated for parallel evaluation (DESIGN.md section 4): every neighbour is searched with
// the STATIC hasMapPoint of KF1, every match is triangulated, and the point of idx1 comes from the first neighbour whose match passes.
// out [KF1.N] in (k, idx1) order; nmatches [nKF2] = vMatchedIndices.size() after the sequential exclusion; ncreated [nKF2];
// reason [nKF2][KF1.N] (optional): NP_* of every (k, idx1).
int orbo_create_new_map_points(const OrboNewPointsIn* in, OrboNewPoint* out, int* nNew, int* nmatches, int* ncreated, uint8_t* reason) {
    const OrboTriFrame& F1 = *in->KF1;
    const int N1 = F1.N, K = in->nKF2;
    std::vector<int> m12((size_t)K * N1, -1), winner(N1, -1);
    std::vector<uint8_t> why((size_t)K * N1, NP_NO_MATCH);
    std::vector<OrboNewPoint> recs((size_t)K * N1);
    for (int k = 0; k < K; ++k) {
        const OrboTriFrame& F2 = in->KF2[k];
        orbo_search_for_triangulation(N1, F1.keypoints, F1.descriptors, F1.hasMapPoint, F1.nEntries, F1.fvNode, F1.fvFeature, F2.N, F2.keypoints, F2.descriptors,
                                      F2.hasMapPoint, F2.nEntries, F2.fvNode, F2.fvFeature, in->scaleFactors, in->levelSigma2, in->ep2 + 2 * (size_t)k,
                                      in->F12 + 9 * (size_t)k, in->bCoarse, 0, m12.data() + (size_t)k * N1);
        for (int i = 0; i < N1; ++i) {
            const int j = m12[(size_t)k * N1 + i];
            if (j >= 0) why[(size_t)k * N1 + i] = (uint8_t)orbo_new_point_for_match(in, k, i, j, &recs[(size_t)k * N1 + i]);
        }
    }
    for (int i = 0; i < N1; ++i)
        for (int k = 0; k < K; ++k) if (why[(size_t)k * N1 + i] == NP_CREATED) { winner[i] = k; break; }
    int n = 0;
    for (int k = 0; k < K; ++k) {
        nmatches[k] = 0; ncreated[k] = 0;
        for (int i = 0; i < N1; ++i) {
            uint8_t& w = why[(size_t)k * N1 + i];
            if (w == NP_NO_MATCH) continue;
            if (winner[i] >= 0 && winner[i] < k) { w = NP_TAKEN; continue; }
            ++nmatches[k];
            if (winner[i] == k) { out[n++] = recs[(size_t)k * N1 + i]; ++ncreated[k]; }
        }
    }
    *nNew = n;
    if (reason) std::memcpy(reason, why.data(), why.size());
    return 0;
}

}  // extern "C"
