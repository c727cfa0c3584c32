// Frame::UndistortKeyPoints (reference src/Frame.cc:747) / Frame::ComputeImageBounds for one point, shared by the CUDA kernel
// (csrc/undistort.cu) and the host (tests/undistort_host.cpp compiles it with g++ for the CPU tests).
//
// The reference calls cv::undistortPoints(mat, mat, K, mDistCoef, cv::Mat(), mK).  For that call (R = I, P = K, no tilt, default
// criteria COUNT 5) OpenCV's cvUndistortPointsInternal works in double; undistort_point restates it expression for expression, in
// OpenCV's order of operations, so that the float result has the same bits:
//   * every product and sum is one dmul / dadd / dsub (exact_math.h): nvcc cannot contract them into DFMA;
//   * every quotient is ddiv_rn below, IEEE round-to-nearest-even division done in integer arithmetic.  The device's own IEEE division
//     (__ddiv_rn) is a Newton iteration built from DFMA, so it would put DFMA back into the kernel; the integer form has none;
//   * the zero coefficients OpenCV carries (k4..k6, s1..s4, the identity tilt, the zeros of R and P) are kept in the expressions,
//     so non-finite intermediates propagate as they do there.
#pragma once
#include <stdint.h>
#if !defined(__CUDACC__)
#include <string.h>
#endif

#include "exact_math.h"

namespace orbx {

#if defined(__CUDA_ARCH__)
ORB_HD uint64_t dbits(double v) { return (uint64_t)__double_as_longlong(v); }
ORB_HD double dfrom(uint64_t u) { return __longlong_as_double((long long)u); }
#else
ORB_HD uint64_t dbits(double v) { uint64_t u; memcpy(&u, &v, 8); return u; }
ORB_HD double dfrom(uint64_t u) { double v; memcpy(&v, &u, 8); return v; }
#endif

// a / b rounded to nearest, ties to even, as IEEE 754 binary64 division: subnormal operands and results, signed zeros and infinities
// included.  A NaN result is the quiet NaN 0x7ff8000000000000 (or the NaN operand, quieted); NaN bits are not part of the contract.
ORB_HD double ddiv_rn(double a, double b) {
    const uint64_t ua = dbits(a), ub = dbits(b), M52 = (1ull << 52) - 1, INF = 0x7ffull << 52, QNAN = 0x7ff8ull << 48;
    const uint64_t sign = (ua ^ ub) & (1ull << 63);
    int ea = (int)((ua >> 52) & 0x7ff), eb = (int)((ub >> 52) & 0x7ff);
    uint64_t ma = ua & M52, mb = ub & M52;
    if (ea == 0x7ff && ma) return dfrom(ua | (1ull << 51));
    if (eb == 0x7ff && mb) return dfrom(ub | (1ull << 51));
    if (ea == 0x7ff) return dfrom(eb == 0x7ff ? QNAN : sign | INF);           // inf / inf, inf / x
    if (eb == 0x7ff) return dfrom(sign);                                       // x / inf
    if (eb == 0 && mb == 0) return dfrom(ea == 0 && ma == 0 ? QNAN : sign | INF);   // 0 / 0, x / 0
    if (ea == 0 && ma == 0) return dfrom(sign);                                // 0 / x
    if (ea) ma |= 1ull << 52; else for (ea = 1; !(ma >> 52); --ea) ma <<= 1;   // mantissas in [2^52, 2^53)
    if (eb) mb |= 1ull << 52; else for (eb = 1; !(mb >> 52); --eb) mb <<= 1;
    int e = ea - eb + 1023;                                                    // biased exponent of a quotient in [1, 2)
    if (ma < mb) { ma <<= 1; --e; }
    uint64_t q = 0, r = ma;                                                    // q = floor(ma * 2^54 / mb): 55 bits, top bit set
    for (int i = 0; i < 55; ++i) {
        q <<= 1;
        if (r >= mb) { r -= mb; q |= 1; }
        r <<= 1;
    }
    if (e >= 0x7ff) return dfrom(sign | INF);
    const int s = e >= 1 ? 2 : (3 - e < 63 ? 3 - e : 63);                     // bits below the result's last place
    uint64_t m = q >> s;
    const uint64_t rem = q & ((1ull << s) - 1), half = 1ull << (s - 1);
    if (rem > half || (rem == half && (r != 0 || (m & 1)))) ++m;
    // a normal result carries its implicit bit in m, so the exponent field is (e - 1) + that bit; a carry out of the last place moves
    // into the exponent (up to infinity), and a subnormal that rounds up to 2^52 becomes the smallest normal
    return dfrom(sign | (e >= 1 ? ((uint64_t)(e - 1) << 52) + m : m));
}

// One point of cvUndistortPointsInternal with R = I, P = K, 4 or 5 coefficients (k1 k2 p1 p2 k3; a 4-coefficient call equals k3 = 0)
// and criteria COUNT 5.  fx fy cx cy k1 k2 p1 p2 k3 are the calibration's floats; (u, v) the distorted pixel.
ORB_HD void undistort_point(float u_, float v_, float fx_, float fy_, float cx_, float cy_, float k1, float k2, float p1, float p2, float k3,
                            float* ou, float* ov) {
    const double fx = fx_, fy = fy_, cx = cx_, cy = cy_;
    const double k[12] = {k1, k2, p1, p2, k3, 0, 0, 0, 0, 0, 0, 0};
    const double ifx = ddiv_rn(1.0, fx), ify = ddiv_rn(1.0, fy);
    const double u = u_, v = v_;
    double x = dmul(dsub(u, cx), ifx), y = dmul(dsub(v, cy), ify);
    // vecUntilt = invMatTilt * Vec3d(x, y, 1) with invMatTilt = I: Matx's s = 0; s += a(i, k) * b(k)
    const double ux = dadd(dadd(dadd(0.0, dmul(1.0, x)), dmul(0.0, y)), dmul(0.0, 1.0));
    const double uy = dadd(dadd(dadd(0.0, dmul(0.0, x)), dmul(1.0, y)), dmul(0.0, 1.0));
    const double uz = dadd(dadd(dadd(0.0, dmul(0.0, x)), dmul(0.0, y)), dmul(1.0, 1.0));
    const double invProj = uz != 0.0 ? ddiv_rn(1.0, uz) : 1.0;
    const double x0 = x = dmul(invProj, ux), y0 = y = dmul(invProj, uy);
    for (int j = 0; j < 5; ++j) {
        const double r2 = dadd(dmul(x, x), dmul(y, y));
        const double num = dadd(1.0, dmul(dadd(dmul(dadd(dmul(k[7], r2), k[6]), r2), k[5]), r2));
        const double den = dadd(1.0, dmul(dadd(dmul(dadd(dmul(k[4], r2), k[1]), r2), k[0]), r2));
        const double icdist = ddiv_rn(num, den);
        if (icdist < 0) {                                   // OpenCV's regression_14583 guard: back to the normalised input
            x = dmul(dsub(u, cx), ifx);
            y = dmul(dsub(v, cy), ify);
            break;
        }
        // 2*k[2]*x*y + k[3]*(r2 + 2*x*x) + k[8]*r2 + k[9]*r2*r2
        const double deltaX = dadd(dadd(dadd(dmul(dmul(dmul(2.0, k[2]), x), y), dmul(k[3], dadd(r2, dmul(dmul(2.0, x), x)))), dmul(k[8], r2)),
                                   dmul(dmul(k[9], r2), r2));
        // k[2]*(r2 + 2*y*y) + 2*k[3]*x*y + k[10]*r2 + k[11]*r2*r2
        const double deltaY = dadd(dadd(dadd(dmul(k[2], dadd(r2, dmul(dmul(2.0, y), y))), dmul(dmul(dmul(2.0, k[3]), x), y)), dmul(k[10], r2)),
                                   dmul(dmul(k[11], r2), r2));
        x = dmul(dsub(x0, deltaX), icdist);
        y = dmul(dsub(y0, deltaY), icdist);
    }
    // RR = P * R = K: xx = RR[0][0]*x + RR[0][1]*y + RR[0][2], yy likewise, ww = 1./(RR[2][0]*x + RR[2][1]*y + RR[2][2])
    const double xx = dadd(dadd(dmul(fx, x), dmul(0.0, y)), cx);
    const double yy = dadd(dadd(dmul(0.0, x), dmul(fy, y)), cy);
    const double ww = ddiv_rn(1.0, dadd(dadd(dmul(0.0, x), dmul(0.0, y)), 1.0));
    *ou = d2f(dmul(xx, ww));
    *ov = d2f(dmul(yy, ww));
}

// Frame::ComputeImageBounds (called at src/Frame.cc:793) from the four undistorted corners; bounds = mnMinX, mnMaxX, mnMinY, mnMaxY.
// k1 == 0 (either sign of zero) gives 0, cols, 0, rows, as the reference's `if(mDistCoef.at<float>(0)!=0.0)` does.  std::min(a, b) is
// (b < a) ? b : a and std::max(a, b) is (a < b) ? b : a, which decides signed zeros.
ORB_HD void image_bounds(const float cam[9], int cols, int rows, float bounds[4]) {
    if (cam[4] == 0.0f) {
        bounds[0] = 0.0f; bounds[1] = (float)cols; bounds[2] = 0.0f; bounds[3] = (float)rows;
        return;
    }
    float cx[4], cy[4];
    const float px[4] = {0.0f, (float)cols, 0.0f, (float)cols}, py[4] = {0.0f, 0.0f, (float)rows, (float)rows};
    for (int i = 0; i < 4; ++i)
        undistort_point(px[i], py[i], cam[0], cam[1], cam[2], cam[3], cam[4], cam[5], cam[6], cam[7], cam[8], &cx[i], &cy[i]);
    bounds[0] = cx[2] < cx[0] ? cx[2] : cx[0];     // min(mat.at<float>(0,0), mat.at<float>(2,0))
    bounds[1] = cx[1] < cx[3] ? cx[3] : cx[1];     // max(mat.at<float>(1,0), mat.at<float>(3,0))
    bounds[2] = cy[1] < cy[0] ? cy[1] : cy[0];     // min(mat.at<float>(0,1), mat.at<float>(1,1))
    bounds[3] = cy[2] < cy[3] ? cy[3] : cy[2];     // max(mat.at<float>(2,1), mat.at<float>(3,1))
}

}  // namespace orbx
