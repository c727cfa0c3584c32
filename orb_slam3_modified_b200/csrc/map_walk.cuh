// What the whole-function map walks share (local_ba.cu: LocalBundleAdjustment, local_inertial_ba_map.cu: LocalInertialBA): the map table
// LbaLocalMap and LocalInertialBAMap have in common, with its host check, staging and device view; the first-appearance compaction over a
// position space; the walk to the local points and their observations; and the local points' EraseObservation cascade and write-back.
#pragma once
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include <vector>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "normal_depth.cuh"
#include "staging.h"

namespace orbx {

// The map table as the kernels see it: the caller's arrays, the outputs both entry points write and the scratch of the walk and the
// write-back, in the staging buffer.  Each caller's Map derives from it and adds its own fields.
struct MapTable {
    int nKF, nPoints, nObs, nlevels;
    const float *Ow, *cam4;
    const int *slotStart, *slotPoint;
    const uint8_t* pointFlags; const float* pos; const int* refKF;
    const int *obsStart, *obsKF, *obsOctave; const float* obsPt;
    const float *invLevelSigma2, *scaleFactors;
    // outputs
    int* localPoint; uint8_t* obsFlag;
    float *kfPose7, *kfCenter, *pointPos; uint8_t* pointBad; int* pointRefKF; float *normal, *minDistance, *maxDistance;
    double *optPoint, *edgeChi2;      // optional
    // scratch
    int* firstPt;                     // [nPoints] first slot position of a local point
    int* lpBase;                      // [nPoints + 1] observation base of the local points
    int* obsEdge;                     // [nObs] edge of an observation, -1 none
    float* Ow2;                       // [nKF][3] camera centres after SetPose
};

// The table's pieces on a Staging, declared from the caller's LbaLocalMap or LocalInertialBAMap, whose slot CSR holds nLists lists.  A
// null optPoint / edgeChi2 stages nothing (piece -1) and binds nullptr.
class MapTablePieces {
    int nKF, nPoints, nObs, nlevels;
    int Ow, cam, slotStart, slotPoint, pflags, pos, ref, obsStart, obsKF, obsPt, obsOct, isg, sf,
        localPoint, obsFlag, kfPose, kfCenter, pointPos, pointBad, pointRef, normal, minD, maxD, optPoint, chi2, firstPt, lpBase, obsEdge, Ow2;
public:
    template <class Table> MapTablePieces(Staging& S, const Table& m, int nLists)
        : nKF(m.nKF), nPoints(m.nPoints), nObs(m.nPoints ? m.obsStart[m.nPoints] : 0), nlevels(m.nlevels) {
        const size_t K = nKF, P = nPoints, NS = m.slotStart[nLists], O = nObs, L = nlevels;
        Ow = S.in(m.cameraCenter, 12 * K); cam = S.in(m.cam4, 16 * K); slotStart = S.in(m.slotStart, 4 * ((size_t)nLists + 1));
        slotPoint = S.in(m.slotPoint, 4 * NS);
        pflags = S.in(m.pointFlags, P); pos = S.in(m.worldPos, 12 * P); ref = S.in(m.refKF, 4 * P);
        obsStart = S.in(P ? m.obsStart : nullptr, P ? 4 * (P + 1) : 0); obsKF = S.in(m.obsKF, 4 * O); obsPt = S.in(m.obsPt, 8 * O);
        obsOct = S.in(m.obsOctave, 4 * O); isg = S.in(m.invLevelSigma2, 4 * L); sf = S.in(m.scaleFactors, 4 * L);
        localPoint = S.out(m.localPoint, 4 * P); obsFlag = S.out(m.obsFlag, O);
        kfPose = S.out(m.kfPose7, 28 * K); kfCenter = S.out(m.kfCenter, 12 * K); pointPos = S.out(m.pointPos, 12 * P);
        pointBad = S.out(m.pointBad, P); pointRef = S.out(m.pointRefKF, 4 * P); normal = S.out(m.normal, 12 * P);
        minD = S.out(m.minDistance, 4 * P); maxD = S.out(m.maxDistance, 4 * P);
        optPoint = m.optPoint ? S.out(m.optPoint, 24 * P) : -1; chi2 = m.edgeChi2 ? S.out(m.edgeChi2, 8 * O) : -1;
        firstPt = S.scratch(4 * P); lpBase = S.scratch(4 * (P + 1)); obsEdge = S.scratch(4 * O); Ow2 = S.scratch(12 * K);
    }
    // Points the device view `d` at the staged pieces.  The staging is reserved.
    void bind(const Staging& S, MapTable& d) const {
        d.nKF = nKF; d.nPoints = nPoints; d.nObs = nObs; d.nlevels = nlevels;
        d.Ow = S.dev<float>(Ow); d.cam4 = S.dev<float>(cam); d.slotStart = S.dev<int>(slotStart); d.slotPoint = S.dev<int>(slotPoint);
        d.pointFlags = S.dev(pflags); d.pos = S.dev<float>(pos); d.refKF = S.dev<int>(ref);
        d.obsStart = S.dev<int>(obsStart); d.obsKF = S.dev<int>(obsKF); d.obsOctave = S.dev<int>(obsOct); d.obsPt = S.dev<float>(obsPt);
        d.invLevelSigma2 = S.dev<float>(isg); d.scaleFactors = S.dev<float>(sf);
        d.localPoint = S.dev<int>(localPoint); d.obsFlag = S.dev(obsFlag);
        d.kfPose7 = S.dev<float>(kfPose); d.kfCenter = S.dev<float>(kfCenter); d.pointPos = S.dev<float>(pointPos); d.pointBad = S.dev(pointBad);
        d.pointRefKF = S.dev<int>(pointRef); d.normal = S.dev<float>(normal); d.minDistance = S.dev<float>(minD); d.maxDistance = S.dev<float>(maxD);
        d.optPoint = optPoint < 0 ? nullptr : S.dev<double>(optPoint); d.edgeChi2 = chi2 < 0 ? nullptr : S.dev<double>(chi2);
        d.firstPt = S.dev<int>(firstPt); d.lpBase = S.dev<int>(lpBase); d.obsEdge = S.dev<int>(obsEdge); d.Ow2 = S.dev<float>(Ow2);
    }
};

// The host checks of the table, each returning bad(message) (ORB_ERR_ARG naming the map) or ORB_OK.  The slots: slotStart [nLists + 1]
// a CSR, slotPoint in [-1, nPoints).
template <class Table, class Bad> int check_slots(const Table& m, int nLists, Bad bad) {
    if (!csr_ok(nLists, m.slotStart)) return bad("slotStart must start at 0 and not decrease");
    const int nSlots = m.slotStart[nLists];
    if (nSlots > 0 && !m.slotPoint) return bad("slotPoint is null");
    for (int s = 0; s < nSlots; ++s)
        if (m.slotPoint[s] < -1 || m.slotPoint[s] >= m.nPoints) return bad("slotPoint out of range");
    return ORB_OK;
}
// The observations: obsStart a CSR, the arrays present, indices and octaves in range, no keyframe twice among a point's observers, and a
// good point's mpRefKF among them.
template <class Table, class Bad> int check_observations(const Table& m, Bad bad) {
    if (m.nPoints == 0) return ORB_OK;
    if (!csr_ok(m.nPoints, m.obsStart)) return bad("obsStart must start at 0 and not decrease");
    const int nObs = m.obsStart[m.nPoints];
    if (nObs > 0 && (!m.obsKF || !m.obsIdx || !m.obsPt || !m.obsOctave || !m.obsFlag)) return bad("an observation array is null");
    std::vector<int> stamp(m.nKF, -1);             // the last point each keyframe was seen observing
    for (int p = 0; p < m.nPoints; ++p) {
        bool refSeen = false;
        for (int o = m.obsStart[p]; o < m.obsStart[p + 1]; ++o) {
            if (m.obsKF[o] < 0 || m.obsKF[o] >= m.nKF) return bad("obsKF out of range");
            if (m.obsIdx[o] < 0) return bad("obsIdx negative");
            if (m.obsOctave[o] < 0 || m.obsOctave[o] >= m.nlevels) return bad("obsOctave outside [0, nlevels)");
            if (stamp[m.obsKF[o]] == p) return bad("a keyframe observes a point twice");
            stamp[m.obsKF[o]] = p;
            refSeen |= m.obsKF[o] == m.refKF[p];
        }
        if (!(m.pointFlags[p] & ORBM_KF_BAD) && m.obsStart[p + 1] > m.obsStart[p] && !refSeen) return bad("a point's mpRefKF is not among its observers");
    }
    return ORB_OK;
}

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

// lLocalMapPoints: clears the point and observation scratch (firstPt, localPoint, obsEdge, obsFlag), then numbers into localPoint, in order
// of first appearance, the points in the slots of nLists keyframe lists (list r is slot list slotList(r); base [nLists + 1] gets the lists'
// slot bases), leaving out NULL slots and points with a flag of skip.  Then concatenates the local points' observations in list order (each
// point's in key order) into one position space of Qo positions, lpBase [nL + 1] getting the points' bases (obs_at).  Returns nL.
template <int NT, class SlotList>
__device__ __forceinline__ int local_points(const MapTable& M, int nLists, SlotList slotList, int* base, int* sm, uint8_t skip, int& Qo) {
    const int tid = threadIdx.x;
    for (int p = tid; p < M.nPoints; p += NT) { M.firstPt[p] = INT_MAX; M.localPoint[p] = -1; }
    for (int o = tid; o < M.nObs; o += NT) { M.obsEdge[o] = -1; M.obsFlag[o] = LBA_OBS_NO_EDGE; }
    // block_prefix ends in a __syncthreads, which orders the clear before the atomicMin below
    const int Qs = block_prefix<NT>(nLists, base, sm, [&](int r) { const int c = slotList(r); return M.slotStart[c + 1] - M.slotStart[c]; });
    if (tid == 0) base[nLists] = Qs;
    auto slotPt = [&](int q) {
        const int r = segment(base, nLists, q);
        const int p = M.slotPoint[M.slotStart[slotList(r)] + q - base[r]];
        return p >= 0 && !(M.pointFlags[p] & skip) ? p : -1;
    };
    for (int q = tid; q < Qs; q += NT) { const int p = slotPt(q); if (p >= 0) atomicMin(&M.firstPt[p], q); }
    __syncthreads();
    const int nL = compact<NT>(Qs, sm, [&](int q) { const int p = slotPt(q); return p >= 0 && M.firstPt[p] == q; },
                               [&](int q, int r) { M.localPoint[r] = slotPt(q); });
    __syncthreads();
    Qo = block_prefix<NT>(nL, M.lpBase, sm, [&](int r) { const int p = M.localPoint[r]; return M.obsStart[p + 1] - M.obsStart[p]; });
    if (tid == 0) M.lpBase[nL] = Qo;
    return nL;
}
// the observation at position q of the local points' observations
__device__ __forceinline__ int obs_at(const MapTable& M, int nL, int q) {
    const int r = segment(M.lpBase, nL, q);
    return M.obsStart[M.localPoint[r]] + q - M.lpBase[r];
}

// The write-back's starting state: every point output and every kfPose7 / kfCenter row 0 (the rows past the lists, and every row of a map
// that writes nothing back, stay so), and Ow2 = Ow until SetPose moves the local keyframes' centres.
template <int NT> __device__ __forceinline__ void clear_write_back(const MapTable& M) {
    for (int i = threadIdx.x; i < M.nKF; i += NT) {
        for (int c = 0; c < 7; ++c) M.kfPose7[7 * i + c] = 0.f;
        for (int c = 0; c < 3; ++c) { M.kfCenter[3 * i + c] = 0.f; M.Ow2[3 * i + c] = M.Ow[3 * i + c]; }
    }
    for (int i = threadIdx.x; i < M.nPoints; i += NT) {
        for (int c = 0; c < 3; ++c) { M.pointPos[3 * i + c] = 0.f; M.normal[3 * i + c] = 0.f; }
        M.pointBad[i] = 0; M.pointRefKF[i] = -1; M.minDistance[i] = M.maxDistance[i] = 0.f;
        if (M.optPoint) for (int c = 0; c < 3; ++c) M.optPoint[3 * i + c] = 0.0;
    }
}

// Per local point i < nL, on one thread each, after SetPose has written Ow2: the solver's estimate point(i, X) to optPoint, SetWorldPos,
// the erase loop over its observations in key order (vToErase holds a point's pairs in key order, and points are independent), then
// UpdateNormalAndDepth.  flag(o) is observation o's LBA_OBS_*; it is written to obsFlag[o], which holds no LBA_OBS_ERASED on entry.
// EraseObservation drops nObs, moves mpRefKF to the first observation left when its own goes, and turns the point bad at nObs <= 2
// (SetBadFlag clears the observations, so later erasures find nothing).  Writes pointBad, pointRefKF (-1 once no observation remains)
// and, for a good point with observations, normal / minDistance / maxDistance.
template <int NT, class Point, class Flag>
__device__ __forceinline__ void write_back_points(const MapTable& M, int nL, Point point, Flag flag) {
    for (int i = threadIdx.x; i < nL; i += NT) {
        const int p = M.localPoint[i], o0 = M.obsStart[p], o1 = M.obsStart[p + 1];
        double X[3];
        point(i, X);
        if (M.optPoint) for (int c = 0; c < 3; ++c) M.optPoint[3 * i + c] = X[c];
        float pos[3] = {(float)X[0], (float)X[1], (float)X[2]};
        for (int c = 0; c < 3; ++c) M.pointPos[3 * i + c] = pos[c];
        int nObs = o1 - o0, ref = M.refKF[p];
        bool bad = false;
        for (int o = o0; o < o1; ++o) {
            const uint8_t f = flag(o);
            M.obsFlag[o] = f;
            if (f != LBA_OBS_ERASED || bad) continue;      // EraseObservation of a bad point finds no observation
            --nObs;
            if (M.obsKF[o] == ref) {                       // mpRefKF = mObservations.begin()->first
                ref = -1;
                for (int j = o0; j < o1 && ref < 0; ++j)
                    if (M.obsFlag[j] != LBA_OBS_ERASED) ref = M.obsKF[j];
            }
            if (nObs <= 2) bad = true;                     // SetBadFlag: the observations are cleared
        }
        M.pointBad[i] = bad; M.pointRefKF[i] = ref;
        if (bad || o1 == o0) continue;                     // UpdateNormalAndDepth returns on a bad point or an empty mObservations
        int o = o0;
        auto next = [&](int& k, int& oct) {
            while (o < o1 && M.obsFlag[o] == LBA_OBS_ERASED) ++o;
            if (o == o1) return false;
            k = M.obsKF[o]; oct = M.obsOctave[o]; ++o;
            return true;
        };
        update_normal_and_depth(pos, M.Ow2, ref, M.scaleFactors, M.nlevels, next, M.normal + 3 * i, M.minDistance + i, M.maxDistance + i);
    }
}

}  // namespace orbx
