// MapPoint::UpdateNormalAndDepth (src/MapPoint.cc) on one thread, monocular observations, shared by update_connections_kernel and
// local_ba_finish_kernel.  Float rules (the oracles evaluate the same expressions with -ffp-contract=off): |v| = sqrtf((x*x + y*y) + z*z),
// every operation rounded; the normal is the running sum of v / |v| element-wise from zero in key order, then / (float)n; mfMaxDistance =
// dist * scaleFactors[level of the reference keyframe's observation], mfMinDistance = mfMaxDistance / scaleFactors[nlevels - 1].
#pragma once
#include <cuda_runtime.h>

namespace orbx {

__device__ __forceinline__ float norm3(float x, float y, float z) {
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

// next(k, oct) yields the point's observations in key order (observer k with Ow [k][3], keypoint octave) and returns false after the
// last; ref must be among them.
template <class Next>
__device__ __forceinline__ void update_normal_and_depth(const float* pos, const float* Ow, int ref, const float* scaleFactors, int nlevels, Next next,
                                                        float* normal, float* minDistance, float* maxDistance) {
    const float px = pos[0], py = pos[1], pz = pos[2];
    float nx = 0.f, ny = 0.f, nz = 0.f;
    int n = 0, level = 0, k, oct;
    while (next(k, oct)) {
        const float vx = __fsub_rn(px, Ow[3 * k]), vy = __fsub_rn(py, Ow[3 * k + 1]), vz = __fsub_rn(pz, Ow[3 * k + 2]);
        const float d = norm3(vx, vy, vz);
        nx = __fadd_rn(nx, __fdiv_rn(vx, d)); ny = __fadd_rn(ny, __fdiv_rn(vy, d)); nz = __fadd_rn(nz, __fdiv_rn(vz, d));
        ++n;
        if (k == ref) level = oct;
    }
    const float fn = (float)n;
    normal[0] = __fdiv_rn(nx, fn); normal[1] = __fdiv_rn(ny, fn); normal[2] = __fdiv_rn(nz, fn);
    const float dist = norm3(__fsub_rn(px, Ow[3 * ref]), __fsub_rn(py, Ow[3 * ref + 1]), __fsub_rn(pz, Ow[3 * ref + 2]));
    const float dmax = __fmul_rn(dist, scaleFactors[level]);
    *maxDistance = dmax;
    *minDistance = __fdiv_rn(dmax, scaleFactors[nlevels - 1]);
}

}  // namespace orbx
