// TEST INFRASTRUCTURE ONLY -- CPU oracle of Frame::UndistortKeyPoints (reference src/Frame.cc:747) and Frame::ComputeImageBounds (called
// at src/Frame.cc:793).
//
// orbo_undistort_points restates OpenCV's cvUndistortPointsInternal for the reference's call cv::undistortPoints(mat, mat, K, mDistCoef,
// cv::Mat(), mK): R = I, P = K, no tilt (fewer than 14 coefficients), criteria COUNT 5, double arithmetic, float in and out.  Built with
// -ffp-contract=off, so every operation below rounds on its own as it does in OpenCV's build.  The k1 == 0 rule is the reference's Frame
// code, not OpenCV's, so it lives in orbo_undistort_keypoints / orbo_image_bounds only.
#include <algorithm>
#include <cstdint>
#include <cstring>

#include "oracle_common.h"

namespace {

// OpenCV's Matx33d * Vec3d (Matx_MatMulOp: s = 0; s += a(i, k) * b(k))
void matvec(const double A[9], const double b[3], double out[3]) {
    for (int i = 0; i < 3; ++i) {
        double s = 0;
        for (int k = 0; k < 3; ++k) s += A[i * 3 + k] * b[k];
        out[i] = s;
    }
}

void undistort_one(float px, float py, const double A[9], const double k[14], const double RR[9], float* ox, float* oy) {
    const double fx = A[0], fy = A[4], ifx = 1. / fx, ify = 1. / fy, cx = A[2], cy = A[5];
    static const double invMatTilt[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    double x = px, y = py, x0 = 0, y0 = 0, u, v;
    u = x; v = y;
    x = (x - cx) * ifx;
    y = (y - cy) * ify;
    const double in[3] = {x, y, 1};
    double vecUntilt[3];
    matvec(invMatTilt, in, vecUntilt);
    double invProj = vecUntilt[2] ? 1. / vecUntilt[2] : 1;
    x0 = x = invProj * vecUntilt[0];
    y0 = y = invProj * vecUntilt[1];
    for (int j = 0; j < 5; j++) {                        // criteria = TermCriteria(COUNT, 5, 0.01): COUNT only
        double r2 = x * x + y * y;
        double icdist = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2);
        if (icdist < 0) {
            x = (u - cx) * ifx;
            y = (v - cy) * ify;
            break;
        }
        double deltaX = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x) + k[8] * r2 + k[9] * r2 * r2;
        double deltaY = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y + k[10] * r2 + k[11] * r2 * r2;
        x = (x0 - deltaX) * icdist;
        y = (y0 - deltaY) * icdist;
    }
    double xx = RR[0] * x + RR[1] * y + RR[2];
    double yy = RR[3] * x + RR[4] * y + RR[5];
    double ww = 1. / (RR[6] * x + RR[7] * y + RR[8]);
    x = xx * ww;
    y = yy * ww;
    *ox = (float)x;
    *oy = (float)y;
}

// K as CV_32F converted to double, and RR = P * I computed as cvMatMul does (sum of three products per entry, in order)
void setup(const float K4[4], const float* D, int nD, double A[9], double k[14], double RR[9]) {
    const double a[9] = {K4[0], 0, K4[2], 0, K4[1], K4[3], 0, 0, 1};
    memcpy(A, a, sizeof(a));
    for (int i = 0; i < 14; ++i) k[i] = i < nD ? (double)D[i] : 0.0;
    static const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) RR[i * 3 + j] = A[i * 3] * I[j] + A[i * 3 + 1] * I[3 + j] + A[i * 3 + 2] * I[6 + j];
}

}  // namespace

extern "C" {

// cv::undistortPoints(pts, out, K, D, cv::Mat(), K) on n float (x, y) pairs; K4 = fx fy cx cy, D = nD (4 or 5) coefficients.
void orbo_undistort_points(const float* pts, int n, const float* K4, const float* D, int nD, float* out) {
    double A[9], k[14], RR[9];
    setup(K4, D, nD, A, k, RR);
    for (int i = 0; i < n; ++i) undistort_one(pts[2 * i], pts[2 * i + 1], A, k, RR, &out[2 * i], &out[2 * i + 1]);
}

// Frame::UndistortKeyPoints on n keypoints: cam9 = fx fy cx cy k1 k2 p1 p2 k3.  k1 == 0 copies mvKeys; otherwise each mvKeysUn[i] is
// mvKeys[i] with pt replaced.
void orbo_undistort_keypoints(const orbo::KeyPoint* kps, int n, const float* cam9, orbo::KeyPoint* out) {
    if (cam9[4] == 0.0) {
        if (n > 0) memcpy(out, kps, sizeof(orbo::KeyPoint) * n);
        return;
    }
    double A[9], k[14], RR[9];
    setup(cam9, cam9 + 4, 5, A, k, RR);
    for (int i = 0; i < n; ++i) {
        out[i] = kps[i];
        undistort_one(kps[i].x, kps[i].y, A, k, RR, &out[i].x, &out[i].y);
    }
}

// Frame::ComputeImageBounds: bounds4 = mnMinX, mnMaxX, mnMinY, mnMaxY.
void orbo_image_bounds(const float* cam9, int cols, int rows, float* bounds4) {
    if (cam9[4] != 0.0) {
        const float mat[8] = {0.0f, 0.0f, (float)cols, 0.0f, 0.0f, (float)rows, (float)cols, (float)rows};
        float u[8];
        orbo_undistort_points(mat, 4, cam9, cam9 + 4, 5, u);
        bounds4[0] = std::min(u[0], u[4]);
        bounds4[1] = std::max(u[2], u[6]);
        bounds4[2] = std::min(u[1], u[3]);
        bounds4[3] = std::max(u[5], u[7]);
    } else {
        bounds4[0] = 0.0f; bounds4[1] = (float)cols; bounds4[2] = 0.0f; bounds4[3] = (float)rows;
    }
}

}  // extern "C"
