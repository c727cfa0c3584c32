// What the whole-function map walks share (local_ba.cu: LocalBundleAdjustment, local_inertial_ba_map.cu: LocalInertialBA): the
// first-appearance compaction over a position space, and a local point's EraseObservation cascade followed by UpdateNormalAndDepth.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "normal_depth.cuh"

namespace orbx {

// the segment r of base [0..R] (ascending, base[0] = 0, base[R] > q) with base[r] <= q < base[r + 1]
__device__ __forceinline__ int segment(const int* base, int R, int q) {
    int lo = 0, hi = R;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (base[mid] <= q) lo = mid; else hi = mid; }
    return lo;
}

// Numbers the positions q in [0, Q) with flag(q) in order: emit(q, rank).  Returns the count.  All NT threads.
template <int NT, class Flag, class Emit>
__device__ int compact(int Q, int* sm, Flag flag, Emit emit) {
    int carry = 0;
    for (int b = 0; b < Q; b += NT) {
        const int q = b + (int)threadIdx.x;
        const bool f = q < Q && flag(q);
        int tot;
        const int r = block_scan_excl<NT>(f ? 1 : 0, sm, tot);
        if (f) emit(q, carry + r);
        carry += tot;
    }
    return carry;
}

// One local point after the solve, on one thread: the erase loop over its observations [o0, o1) in key order (vToErase holds a point's
// pairs in key order, and points are independent), then SetWorldPos and UpdateNormalAndDepth.  flag(o) is observation o's LBA_OBS_*;
// it is written to obsFlag[o], which holds no LBA_OBS_ERASED on entry.  EraseObservation drops nObs, moves mpRefKF to the first
// observation left when its own goes, and turns the point bad at nObs <= 2 (SetBadFlag clears the observations, so later erasures find
// nothing).  Ow [nKF][3] are the camera centres after SetPose.  Writes *bad, *ref (-1 once no observation remains) and, for a good point
// with observations, normal / minDistance / maxDistance.
template <class Flag>
__device__ __forceinline__ void finish_point(const int* obsKF, const int* obsOctave, int o0, int o1, uint8_t* obsFlag, int ref, Flag flag,
                                             const float* pos, const float* Ow, const float* scaleFactors, int nlevels, uint8_t* badOut,
                                             int* refOut, float* normal, float* minDistance, float* maxDistance) {
    int nObs = o1 - o0;
    bool bad = false;
    for (int o = o0; o < o1; ++o) {
        const uint8_t f = flag(o);
        obsFlag[o] = f;
        if (f != LBA_OBS_ERASED || bad) continue;      // EraseObservation of a bad point finds no observation
        --nObs;
        if (obsKF[o] == ref) {                         // mpRefKF = mObservations.begin()->first
            ref = -1;
            for (int j = o0; j < o1 && ref < 0; ++j)
                if (obsFlag[j] != LBA_OBS_ERASED) ref = obsKF[j];
        }
        if (nObs <= 2) bad = true;                     // SetBadFlag: the observations are cleared
    }
    *badOut = bad; *refOut = ref;
    if (bad || o1 == o0) return;                       // UpdateNormalAndDepth returns on a bad point or an empty mObservations
    int o = o0;
    auto next = [&](int& k, int& oct) {
        while (o < o1 && obsFlag[o] == LBA_OBS_ERASED) ++o;
        if (o == o1) return false;
        k = obsKF[o]; oct = obsOctave[o]; ++o;
        return true;
    };
    update_normal_and_depth(pos, Ow, ref, scaleFactors, nlevels, next, normal, minDistance, maxDistance);
}

}  // namespace orbx
