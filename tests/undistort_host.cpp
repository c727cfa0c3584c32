// Host-side build of csrc/undistort.h for tests/test_undistort_cpu.py: the per-point function the undistortion kernel runs, compiled with
// g++ -ffp-contract=off, so the CPU tests can pin it (and its integer IEEE division) against the oracle, cv2 and the host's own division.
#include "../orb_slam3_modified_b200/csrc/undistort.h"

extern "C" {

void uh_ddiv_n(const double* a, const double* b, double* out, int n) {
    for (int i = 0; i < n; ++i) out[i] = orbx::ddiv_rn(a[i], b[i]);
}

void uh_undistort_points(const float* pts, int n, const float* cam9, float* out) {
    for (int i = 0; i < n; ++i)
        orbx::undistort_point(pts[2 * i], pts[2 * i + 1], cam9[0], cam9[1], cam9[2], cam9[3], cam9[4], cam9[5], cam9[6], cam9[7], cam9[8],
                              &out[2 * i], &out[2 * i + 1]);
}

void uh_image_bounds(const float* cam9, int cols, int rows, float* bounds4) { orbx::image_bounds(cam9, cols, rows, bounds4); }

}  // extern "C"
