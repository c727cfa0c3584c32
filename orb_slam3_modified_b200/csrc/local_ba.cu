// Optimizer::LocalBundleAdjustment (src/Optimizer.cc:1116-1498, monocular observations) as a whole, for a batch of maps
// (lba_local_bundle_adjustment_batch, include/orb_b200.h).  One call:
//   1. local_ba_walk_kernel, one CTA per map: the graph walk of :1125-1403 and the problem g2o would see (vertices sorted by mnId,
//      edges in insertion order), written in LbaProblem's layout into the staging buffer;
//   2. one small copy of the built sizes to the host, which lays the solver's slots out (lba.cu: Solver::layout) and reads the stop flags;
//   3. lba_fill_kernel copies the built problems into the slots, then lba.cu's structure and cluster kernels solve them;
//   4. local_ba_finish_kernel, one CTA per map: the outlier test, EraseObservation's cascade, SetPose, SetWorldPos, UpdateNormalAndDepth.
// Every order the reference defines by list walks is rebuilt as a first-appearance order: a position space (the local keyframes' slots, or
// the local points' observations, concatenated in list order) is scanned once with atomicMin for each item's first position, then one
// ordered block scan over the positions numbers the items.
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "frame_pose.cuh"
#include "local_ba.h"
#include "map_walk.cuh"
#include "staging.h"

namespace lba_local {

using orbx::set_error;
using orbx::csr_ok;
using orbx::all_distinct;
using orbx::segment;

constexpr int WT = 512;
constexpr unsigned char KF_SKIP = ORBM_KF_BAD | ORBM_KF_OTHER_MAP;   // isBad() || GetMap() != pCurrentMap

// One map as the kernels see it: the caller's arrays, its outputs and its scratch in the staging buffer.
struct Map {
    int nKF, nCov, nPoints, nObs, nlevels, sortCap;
    const unsigned long long* mnId; const uint8_t* kfFlags; const float *pose7, *Ow, *cam4;
    const int *cov, *slotStart, *slotPoint;
    const unsigned long long* pointId; const uint8_t* pointFlags; const float* pos; const int* refKF;
    const int *obsStart, *obsKF, *obsOctave; const float* obsPt;
    const float *invLevelSigma2, *scaleFactors;
    // outputs
    int* sizes;                       // [8] walk verdict (0 built, 1 no fixed keyframe), nP, nL, nE, nF
    int *counts, *nLists, *localKF, *fixedKF, *localPoint; uint8_t* obsFlag;
    float *kfPose7, *kfCenter, *pointPos; uint8_t* pointBad; int* pointRefKF; float *normal, *minDistance, *maxDistance; double* lmStats;
    double *optPose, *optPoint, *edgeChi2; uint8_t* edgeDepthPos;      // optional
    // the built problem (LbaProblem's layout)
    double* bPoses; uint8_t* bFixed; float* bCam; double* bPts; int *bEPt, *bEPose; double* bObs; float* bIsg;
    // scratch
    int *kfRank;                      // [nKF] local rank, -2 for the other entries of the covisible list (mnBALocalForKF), else -1
    int *kfVert, *ptVert;             // vertex of a keyframe / point, -1 none
    int *firstFix, *firstPt;          // first position of a fixed-camera candidate / local point
    int *obsEdge;                     // [nObs] edge of an observation, -1 none
    int *locCand, *locBase, *lpBase;  // candidate of a local keyframe, slot base of the local keyframes, observation base of the local points
    unsigned long long* key; int* val;   // [sortCap] sort buffers
    float* Ow2;                       // [nKF][3] camera centres after SetPose
};

// What the finish kernel reads of the solve: status (LBA_LOCAL_*), solved (0: nothing was optimised), the slot's results.
struct Solve { int status, solved; lba::SlotOut r; };

// ascending bitonic sort of key / val [n2], n2 a power of two, in global memory.  All threads.
__device__ void bitonic(unsigned long long* key, int* val, int n2) {
    for (int k = 2; k <= n2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2; i += WT) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned long long a = key[i], b = key[l];
                    if ((a > b) == ((i & k) == 0)) { key[i] = b; key[l] = a; const int t = val[i]; val[i] = val[l]; val[l] = t; }
                }
            }
            __syncthreads();
        }
}

__global__ void __launch_bounds__(WT) local_ba_walk_kernel(const Map* __restrict__ maps) {
    __shared__ Map M;
    __shared__ int sm[33];
    __shared__ int s_nLocal, s_init;
    const int tid = threadIdx.x;
    if (tid == 0) M = maps[blockIdx.x];
    __syncthreads();
    // every output starts empty: lists -1, no edge, no estimate
    for (int k = tid; k < M.nKF; k += WT) { M.kfRank[k] = -1; M.kfVert[k] = -1; M.firstFix[k] = INT_MAX; M.localKF[k] = -1; M.fixedKF[k] = -1; }
    for (int p = tid; p < M.nPoints; p += WT) { M.ptVert[p] = -1; M.firstPt[p] = INT_MAX; M.localPoint[p] = -1; }
    for (int o = tid; o < M.nObs; o += WT) { M.obsEdge[o] = -1; M.obsFlag[o] = LBA_OBS_NO_EDGE; }
    __syncthreads();
    // lLocalKeyFrames: pKF, then the covisibles that are not bad and in the current map; every covisible is marked (mnBALocalForKF)
    if (tid == 0) {
        int n = 0;
        M.kfRank[0] = 0; M.localKF[0] = 0; M.locCand[0] = 0; ++n;
        for (int i = 0; i < M.nCov; ++i) {
            const int k = M.cov[i];
            if (M.kfFlags[k] & KF_SKIP) { M.kfRank[k] = -2; continue; }
            M.kfRank[k] = n; M.localKF[n] = k; M.locCand[n] = 1 + i; ++n;
        }
        int init = 0;
        for (int r = 0; r < n; ++r) init |= (M.kfFlags[M.localKF[r]] & ORBM_KF_INIT) != 0;
        s_nLocal = n; s_init = init;
    }
    __syncthreads();
    const int nLocal = s_nLocal;
    // lLocalMapPoints: first appearance over the local keyframes' slots, bad and other-map points skipped
    const int Qs = orbx::block_prefix<WT>(nLocal, M.locBase, sm, [&](int r) { const int c = M.locCand[r]; return M.slotStart[c + 1] - M.slotStart[c]; });
    if (tid == 0) M.locBase[nLocal] = Qs;
    auto slotPt = [&](int q) {
        const int r = segment(M.locBase, nLocal, q);
        const int p = M.slotPoint[M.slotStart[M.locCand[r]] + q - M.locBase[r]];
        return p >= 0 && !(M.pointFlags[p] & KF_SKIP) ? p : -1;
    };
    for (int q = tid; q < Qs; q += WT) { const int p = slotPt(q); if (p >= 0) atomicMin(&M.firstPt[p], q); }
    __syncthreads();
    const int nL = orbx::compact<WT>(Qs, sm, [&](int q) { const int p = slotPt(q); return p >= 0 && M.firstPt[p] == q; },
                           [&](int q, int r) { M.localPoint[r] = slotPt(q); });
    __syncthreads();
    // lFixedCameras: first appearance over (local point, observation) of the unmarked observers, kept when good and in the current map
    const int Qo = orbx::block_prefix<WT>(nL, M.lpBase, sm, [&](int r) { const int p = M.localPoint[r]; return M.obsStart[p + 1] - M.obsStart[p]; });
    if (tid == 0) M.lpBase[nL] = Qo;
    auto obsAt = [&](int q) { const int r = segment(M.lpBase, nL, q); return M.obsStart[M.localPoint[r]] + q - M.lpBase[r]; };
    for (int q = tid; q < Qo; q += WT) {
        const int k = M.obsKF[obsAt(q)];
        if (M.kfRank[k] == -1 && !(M.kfFlags[k] & KF_SKIP)) atomicMin(&M.firstFix[k], q);
    }
    __syncthreads();
    const int nFix = orbx::compact<WT>(Qo, sm, [&](int q) { const int k = M.obsKF[obsAt(q)]; return M.kfRank[k] == -1 && M.firstFix[k] == q; },
                             [&](int q, int r) { M.fixedKF[r] = M.obsKF[obsAt(q)]; });
    __syncthreads();
    const int numFixed = nFix + s_init;
    if (numFixed == 0) {                              // :1178-1182: return before the optimiser is set up
        if (tid == 0) {
            M.sizes[0] = 1; M.sizes[1] = M.sizes[2] = M.sizes[3] = M.sizes[4] = 0;
            M.counts[0] = M.counts[1] = M.counts[2] = M.counts[3] = 0;
            M.nLists[0] = nLocal; M.nLists[1] = 0; M.nLists[2] = nL;
        }
        return;
    }
    // vertices in g2o's order: keyframes by mnId, then points by mnId
    const int nP = nLocal + nFix;
    for (int i = tid; i < M.sortCap; i += WT) {
        M.key[i] = i < nP ? M.mnId[i < nLocal ? M.localKF[i] : M.fixedKF[i - nLocal]] : ~0ull;
        M.val[i] = i < nP ? (i < nLocal ? M.localKF[i] : M.fixedKF[i - nLocal]) : -1;
    }
    __syncthreads();
    int n2 = 1;
    while (n2 < nP) n2 <<= 1;
    bitonic(M.key, M.val, n2);
    for (int v = tid; v < nP; v += WT) {
        const int k = M.val[v];
        M.kfVert[k] = v;
        for (int c = 0; c < 7; ++c) M.bPoses[7 * v + c] = (double)M.pose7[7 * k + c];
        for (int c = 0; c < 4; ++c) M.bCam[4 * v + c] = M.cam4[4 * k + c];
        M.bFixed[v] = M.kfRank[k] < 0 || (M.kfFlags[k] & ORBM_KF_INIT);   // fixed camera, or vSE3->setFixed(mnId == GetInitKFid())
    }
    __syncthreads();
    for (int i = tid; i < M.sortCap; i += WT) {
        M.key[i] = i < nL ? M.pointId[M.localPoint[i]] : ~0ull;
        M.val[i] = i < nL ? M.localPoint[i] : -1;
    }
    __syncthreads();
    n2 = 1;
    while (n2 < nL) n2 <<= 1;
    bitonic(M.key, M.val, n2);
    for (int v = tid; v < nL; v += WT) {
        const int p = M.val[v];
        M.ptVert[p] = v;
        for (int c = 0; c < 3; ++c) M.bPts[3 * v + c] = (double)M.pos[3 * p + c];
    }
    __syncthreads();
    // edges in insertion order: local points in list order, observations in key order, observers good and in the current map
    const int nE = orbx::compact<WT>(Qo, sm, [&](int q) { return !(M.kfFlags[M.obsKF[obsAt(q)]] & KF_SKIP); }, [&](int q, int e) {
        const int r = segment(M.lpBase, nL, q);
        const int p = M.localPoint[r], o = M.obsStart[p] + q - M.lpBase[r], k = M.obsKF[o];
        M.bEPt[e] = M.ptVert[p]; M.bEPose[e] = M.kfVert[k];
        M.bObs[2 * e] = (double)M.obsPt[2 * o]; M.bObs[2 * e + 1] = (double)M.obsPt[2 * o + 1];
        M.bIsg[e] = M.invLevelSigma2[M.obsOctave[o]];
        M.obsEdge[o] = e;
    });
    int nFree = 0;
    for (int v = tid; v < nP; v += WT) nFree += !M.bFixed[v];
    int nF;
    orbx::block_scan_excl<WT>(nFree, sm, nF);
    if (tid == 0) {
        M.sizes[0] = 0; M.sizes[1] = nP; M.sizes[2] = nL; M.sizes[3] = nE; M.sizes[4] = nF;
        M.counts[0] = numFixed; M.counts[1] = nLocal; M.counts[2] = nL; M.counts[3] = nE;
        M.nLists[0] = nLocal; M.nLists[1] = nFix; M.nLists[2] = nL;
    }
}

__global__ void __launch_bounds__(WT) local_ba_finish_kernel(const Map* __restrict__ maps, const Solve* __restrict__ solves) {
    __shared__ Map M;
    __shared__ Solve V;
    const int tid = threadIdx.x;
    if (tid == 0) { M = maps[blockIdx.x]; V = solves[blockIdx.x]; }
    __syncthreads();
    const int nLocal = M.nLists[0], nL = M.nLists[2];
    const bool ran = V.status == LBA_LOCAL_RAN;
    if (tid == 0) {
        const double* st = V.solved ? V.r.stats : nullptr;
        M.lmStats[0] = st ? st[0] : -1.0;
        for (int i = 1; i < 5; ++i) M.lmStats[i] = st ? st[i] : 0.0;
    }
    // the solver's estimates per local keyframe / point (the initial ones when nothing was optimised)
    auto posePtr = [&](int i, double* T) {
        const int k = M.localKF[i];
        if (V.solved) for (int c = 0; c < 7; ++c) T[c] = V.r.poses[7 * M.kfVert[k] + c];
        else for (int c = 0; c < 7; ++c) T[c] = (double)M.pose7[7 * k + c];
    };
    auto pointOf = [&](int i, double* X) {
        const int p = M.localPoint[i];
        if (V.solved) for (int c = 0; c < 3; ++c) X[c] = V.r.points[3 * M.ptVert[p] + c];
        else for (int c = 0; c < 3; ++c) X[c] = (double)M.pos[3 * p + c];
    };
    // every output slot past the lists, and every slot of a map that did not run, holds zeros
    for (int i = tid; i < M.nKF; i += WT) {
        for (int c = 0; c < 7; ++c) M.kfPose7[7 * i + c] = 0.f;
        for (int c = 0; c < 3; ++c) M.kfCenter[3 * i + c] = 0.f;
        if (M.optPose) for (int c = 0; c < 7; ++c) M.optPose[7 * i + c] = 0.0;
        for (int c = 0; c < 3; ++c) M.Ow2[3 * i + c] = M.Ow[3 * i + c];
    }
    for (int i = tid; i < M.nPoints; i += WT) {
        for (int c = 0; c < 3; ++c) { M.pointPos[3 * i + c] = 0.f; M.normal[3 * i + c] = 0.f; }
        M.pointBad[i] = 0; M.pointRefKF[i] = -1; M.minDistance[i] = M.maxDistance[i] = 0.f;
        if (M.optPoint) for (int c = 0; c < 3; ++c) M.optPoint[3 * i + c] = 0.0;
    }
    for (int o = tid; o < M.nObs; o += WT) {
        if (M.edgeChi2) M.edgeChi2[o] = 0.0;
        if (M.edgeDepthPos) M.edgeDepthPos[o] = 0;
    }
    __syncthreads();
    if (!ran) return;
    // SetPose (:1464-1471): the float pose and its camera centre
    for (int i = tid; i < nLocal; i += WT) {
        double T[7];
        posePtr(i, T);
        if (M.optPose) for (int c = 0; c < 7; ++c) M.optPose[7 * i + c] = T[c];
        float Tf[7], R[9], t[3], Ow[3];
        orbm::set_pose_from_double(T, Tf);
        orbm::update_pose_matrices(Tf, R, t, Ow);
        for (int c = 0; c < 7; ++c) M.kfPose7[7 * i + c] = Tf[c];
        const int k = M.localKF[i];
        for (int c = 0; c < 3; ++c) { M.kfCenter[3 * i + c] = Ow[c]; M.Ow2[3 * k + c] = Ow[c]; }
    }
    __syncthreads();
    // per local point: the outlier test and the erase loop (:1417-1460) in edge order -- the point's observations in key order, points
    // being independent -- then SetWorldPos and UpdateNormalAndDepth (:1474-1481)
    for (int i = tid; i < nL; i += WT) {
        const int p = M.localPoint[i];
        double X[3];
        pointOf(i, X);
        if (M.optPoint) for (int c = 0; c < 3; ++c) M.optPoint[3 * i + c] = X[c];
        float pos[3] = {(float)X[0], (float)X[1], (float)X[2]};
        for (int c = 0; c < 3; ++c) M.pointPos[3 * i + c] = pos[c];
        orbx::finish_point(M.obsKF, M.obsOctave, M.obsStart[p], M.obsStart[p + 1], M.obsFlag, M.refKF[p], [&](int o) -> uint8_t {
            const int e = M.obsEdge[o];
            if (e < 0) return LBA_OBS_NO_EDGE;
            const double chi2 = V.solved ? V.r.chi2[e] : 0.0;
            const uint8_t dpos = V.solved ? V.r.depthPos[e] : 1;
            if (M.edgeChi2) { M.edgeChi2[o] = chi2; M.edgeDepthPos[o] = dpos; }
            return chi2 > 5.991 || !dpos ? LBA_OBS_ERASED : LBA_OBS_KEPT;
        }, pos, M.Ow2, M.scaleFactors, M.nlevels, M.pointBad + i, M.pointRefKF + i, M.normal + 3 * i, M.minDistance + i, M.maxDistance + i);
    }
}

// ORB_ERR_ARG with a message naming the map, or ORB_OK
int check_map(const LbaLocalMap& m, int j) {
    auto bad = [j](const std::string& what) { set_error("lba_local_bundle_adjustment_batch: map " + std::to_string(j) + ": " + what); return ORB_ERR_ARG; };
    if (m.nKF < 1 || m.nCov < 0 || m.nPoints < 0 || m.nlevels < 1) return bad("nKF < 1, nlevels < 1 or a negative count");
    if (!m.mnId || !m.kfFlags || !m.pose7 || !m.cameraCenter || !m.cam4 || !m.slotStart || !m.invLevelSigma2 || !m.scaleFactors)
        return bad("a keyframe or map array is null");
    if (m.nCov > 0 && !m.cov) return bad("cov is null");
    if (!m.status || !m.counts || !m.nLists || !m.localKF || !m.fixedKF || !m.kfPose7 || !m.kfCenter || !m.lmStats) return bad("a keyframe output is null");
    if (m.nPoints > 0 && (!m.pointId || !m.pointFlags || !m.worldPos || !m.refKF || !m.obsStart || !m.localPoint || !m.pointPos || !m.pointBad ||
                          !m.pointRefKF || !m.normal || !m.minDistance || !m.maxDistance)) return bad("a point array is null");
    if ((m.edgeChi2 == nullptr) != (m.edgeDepthPositive == nullptr)) return bad("edgeChi2 and edgeDepthPositive go together");
    if (m.kfFlags[0] & ORBM_KF_OTHER_MAP) return bad("pKF (entry 0) cannot be of another map");
    if (!all_distinct(m.mnId, m.nKF)) return bad("keyframe mnIds repeat");
    std::vector<char> seen(m.nKF, 0);
    seen[0] = 1;
    for (int i = 0; i < m.nCov; ++i) {
        if (m.cov[i] < 1 || m.cov[i] >= m.nKF) return bad("cov out of range [1, nKF)");
        if (seen[m.cov[i]]) return bad("cov repeats a keyframe");
        seen[m.cov[i]] = 1;
    }
    if (!csr_ok(m.nCov + 1, m.slotStart)) return bad("slotStart must start at 0 and not decrease");
    const int nSlots = m.slotStart[m.nCov + 1];
    if (nSlots > 0 && !m.slotPoint) return bad("slotPoint is null");
    for (int s = 0; s < nSlots; ++s)
        if (m.slotPoint[s] < -1 || m.slotPoint[s] >= m.nPoints) return bad("slotPoint out of range");
    if (m.nPoints > 0) {
        if (!all_distinct(m.pointId, m.nPoints)) return bad("point mnIds repeat");
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
    }
    return ORB_OK;
}

}  // namespace lba_local

using namespace lba_local;

extern "C" int lba_local_bundle_adjustment_batch(lba_handle* h, int nMaps, const LbaLocalMap* maps) {
    if (!h || nMaps < 0 || (nMaps > 0 && !maps)) { set_error("lba_local_bundle_adjustment_batch: bad argument"); return ORB_ERR_ARG; }
    for (int j = 0; j < nMaps; ++j)
        if (int rc = check_map(maps[j], j)) return rc;
    int maxP, maxL, maxE, maxBatch;
    lba::solver_limits(h, &maxP, &maxL, &maxE, &maxBatch);
    if (nMaps > maxBatch) { set_error("lba_local_bundle_adjustment_batch: " + std::to_string(nMaps) + " maps, max_batch " + std::to_string(maxBatch)); return ORB_ERR_CAPACITY; }
    lba::solver_set_local_launches(h, 0);
    if (nMaps == 0) return ORB_OK;
    const cudaStream_t st = lba::solver_stream(h);
    orbx::Staging& S = lba::solver_staging(h);
    S.begin();
    struct Pieces { int mnId, flags, pose, Ow, cam, cov, slotStart, slotPoint, pid, pflags, pos, ref, obsStart, obsKF, obsPt, obsOct, isg, sf,
                    sizes, counts, nLists, localKF, fixedKF, localPoint, obsFlag, kfPose, kfCenter, pointPos, pointBad, pointRef, normal, minD, maxD,
                    lm, optPose, optPoint, chi2, dpos, bPoses, bFixed, bCam, bPts, bEPt, bEPose, bObs, bIsg, kfRank, kfVert, ptVert, firstFix,
                    firstPt, obsEdge, locCand, locBase, lpBase, key, val, Ow2; int sortCap; };
    std::vector<Pieces> pc(nMaps);
    const int sizesAll = S.out(nullptr, 32 * (size_t)nMaps);       // one piece, so that one small copy brings every map's sizes
    for (int j = 0; j < nMaps; ++j) {
        const LbaLocalMap& m = maps[j];
        const size_t K = m.nKF, C = m.nCov, P = m.nPoints, NS = m.slotStart[m.nCov + 1], O = P ? m.obsStart[m.nPoints] : 0, L = m.nlevels;
        Pieces& q = pc[j];
        q.sortCap = 1;
        while (q.sortCap < std::max<int>(m.nKF, m.nPoints)) q.sortCap <<= 1;
        q.mnId = S.in(m.mnId, 8 * K); q.flags = S.in(m.kfFlags, K); q.pose = S.in(m.pose7, 28 * K); q.Ow = S.in(m.cameraCenter, 12 * K);
        q.cam = S.in(m.cam4, 16 * K); q.cov = S.in(m.cov, 4 * C); q.slotStart = S.in(m.slotStart, 4 * (C + 2)); q.slotPoint = S.in(m.slotPoint, 4 * NS);
        q.pid = S.in(m.pointId, 8 * P); q.pflags = S.in(m.pointFlags, P); q.pos = S.in(m.worldPos, 12 * P); q.ref = S.in(m.refKF, 4 * P);
        q.obsStart = S.in(P ? m.obsStart : nullptr, P ? 4 * (P + 1) : 0); q.obsKF = S.in(m.obsKF, 4 * O); q.obsPt = S.in(m.obsPt, 8 * O);
        q.obsOct = S.in(m.obsOctave, 4 * O); q.isg = S.in(m.invLevelSigma2, 4 * L); q.sf = S.in(m.scaleFactors, 4 * L);
        q.sizes = j; q.counts = S.out(m.counts, 16); q.nLists = S.out(m.nLists, 12);
        q.localKF = S.out(m.localKF, 4 * K); q.fixedKF = S.out(m.fixedKF, 4 * K); q.localPoint = S.out(m.localPoint, 4 * P); q.obsFlag = S.out(m.obsFlag, O);
        q.kfPose = S.out(m.kfPose7, 28 * K); q.kfCenter = S.out(m.kfCenter, 12 * K); q.pointPos = S.out(m.pointPos, 12 * P);
        q.pointBad = S.out(m.pointBad, P); q.pointRef = S.out(m.pointRefKF, 4 * P); q.normal = S.out(m.normal, 12 * P);
        q.minD = S.out(m.minDistance, 4 * P); q.maxD = S.out(m.maxDistance, 4 * P); q.lm = S.out(m.lmStats, 40);
        q.optPose = S.out(m.optPose, m.optPose ? 56 * K : 0); q.optPoint = S.out(m.optPoint, m.optPoint ? 24 * P : 0);
        q.chi2 = S.out(m.edgeChi2, m.edgeChi2 ? 8 * O : 0); q.dpos = S.out(m.edgeDepthPositive, m.edgeChi2 ? O : 0);
        q.bPoses = S.scratch(56 * K); q.bFixed = S.scratch(K); q.bCam = S.scratch(16 * K); q.bPts = S.scratch(24 * P);
        q.bEPt = S.scratch(4 * O); q.bEPose = S.scratch(4 * O); q.bObs = S.scratch(16 * O); q.bIsg = S.scratch(4 * O);
        q.kfRank = S.scratch(4 * K); q.kfVert = S.scratch(4 * K); q.ptVert = S.scratch(4 * P); q.firstFix = S.scratch(4 * K); q.firstPt = S.scratch(4 * P);
        q.obsEdge = S.scratch(4 * O); q.locCand = S.scratch(4 * (C + 1)); q.locBase = S.scratch(4 * (C + 2)); q.lpBase = S.scratch(4 * (P + 1));
        q.key = S.scratch(8 * (size_t)q.sortCap); q.val = S.scratch(4 * (size_t)q.sortCap); q.Ow2 = S.scratch(12 * K);
    }
    const int tab = S.in(nullptr, sizeof(Map) * nMaps), fillTab = S.scratch(sizeof(lba::FillSrc) * nMaps), solveTab = S.scratch(sizeof(Solve) * nMaps);
    if (int rc = S.reserve()) return rc;
    Map* T = S.host<Map>(tab);
    for (int j = 0; j < nMaps; ++j) {
        const LbaLocalMap& m = maps[j];
        const Pieces& q = pc[j];
        Map d;
        d.nKF = m.nKF; d.nCov = m.nCov; d.nPoints = m.nPoints; d.nObs = m.nPoints ? m.obsStart[m.nPoints] : 0; d.nlevels = m.nlevels; d.sortCap = q.sortCap;
        d.mnId = S.dev<unsigned long long>(q.mnId); d.kfFlags = S.dev(q.flags); d.pose7 = S.dev<float>(q.pose); d.Ow = S.dev<float>(q.Ow);
        d.cam4 = S.dev<float>(q.cam); d.cov = S.dev<int>(q.cov); d.slotStart = S.dev<int>(q.slotStart); d.slotPoint = S.dev<int>(q.slotPoint);
        d.pointId = S.dev<unsigned long long>(q.pid); d.pointFlags = S.dev(q.pflags); d.pos = S.dev<float>(q.pos); d.refKF = S.dev<int>(q.ref);
        d.obsStart = S.dev<int>(q.obsStart); d.obsKF = S.dev<int>(q.obsKF); d.obsOctave = S.dev<int>(q.obsOct); d.obsPt = S.dev<float>(q.obsPt);
        d.invLevelSigma2 = S.dev<float>(q.isg); d.scaleFactors = S.dev<float>(q.sf);
        d.sizes = S.dev<int>(sizesAll) + 8 * j; d.counts = S.dev<int>(q.counts); d.nLists = S.dev<int>(q.nLists); d.localKF = S.dev<int>(q.localKF);
        d.fixedKF = S.dev<int>(q.fixedKF); d.localPoint = S.dev<int>(q.localPoint); d.obsFlag = S.dev(q.obsFlag);
        d.kfPose7 = S.dev<float>(q.kfPose); d.kfCenter = S.dev<float>(q.kfCenter); d.pointPos = S.dev<float>(q.pointPos); d.pointBad = S.dev(q.pointBad);
        d.pointRefKF = S.dev<int>(q.pointRef); d.normal = S.dev<float>(q.normal); d.minDistance = S.dev<float>(q.minD); d.maxDistance = S.dev<float>(q.maxD);
        d.lmStats = S.dev<double>(q.lm);
        d.optPose = m.optPose ? S.dev<double>(q.optPose) : nullptr; d.optPoint = m.optPoint ? S.dev<double>(q.optPoint) : nullptr;
        d.edgeChi2 = m.edgeChi2 ? S.dev<double>(q.chi2) : nullptr; d.edgeDepthPos = m.edgeChi2 ? S.dev(q.dpos) : nullptr;
        d.bPoses = S.dev<double>(q.bPoses); d.bFixed = S.dev(q.bFixed); d.bCam = S.dev<float>(q.bCam); d.bPts = S.dev<double>(q.bPts);
        d.bEPt = S.dev<int>(q.bEPt); d.bEPose = S.dev<int>(q.bEPose); d.bObs = S.dev<double>(q.bObs); d.bIsg = S.dev<float>(q.bIsg);
        d.kfRank = S.dev<int>(q.kfRank); d.kfVert = S.dev<int>(q.kfVert); d.ptVert = S.dev<int>(q.ptVert); d.firstFix = S.dev<int>(q.firstFix);
        d.firstPt = S.dev<int>(q.firstPt); d.obsEdge = S.dev<int>(q.obsEdge); d.locCand = S.dev<int>(q.locCand); d.locBase = S.dev<int>(q.locBase);
        d.lpBase = S.dev<int>(q.lpBase); d.key = S.dev<unsigned long long>(q.key); d.val = S.dev<int>(q.val); d.Ow2 = S.dev<float>(q.Ow2);
        T[j] = d;
    }
    CK(S.upload(st));
    local_ba_walk_kernel<<<nMaps, WT, 0, st>>>(S.dev<Map>(tab));
    CK(cudaGetLastError());
    int launches = 1;
    // the built sizes: they decide the solver slots' layout
    CK(cudaMemcpyAsync(S.host(sizesAll), S.dev(sizesAll), 32 * (size_t)nMaps, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    std::vector<int> status(nMaps);
    std::vector<int4> sizes;
    std::vector<double> lambdaInit;
    std::vector<lba::FillSrc> fill;
    std::vector<const volatile uint8_t*> flags;
    std::vector<int> slotOf(nMaps, -1);
    for (int j = 0; j < nMaps; ++j) {
        const int* z = S.host<int>(sizesAll) + 8 * j;
        if (z[0] == 1) { status[j] = LBA_LOCAL_NO_FIXED; continue; }
        if (maps[j].stopFlag && *maps[j].stopFlag) { status[j] = LBA_LOCAL_STOPPED; continue; }   // :1406-1408
        status[j] = LBA_LOCAL_RAN;
        if (z[1] > maxP || z[2] > maxL || z[3] > maxE) {
            set_error("lba_local_bundle_adjustment_batch: map " + std::to_string(j) + ": " + std::to_string(z[1]) + " poses, " + std::to_string(z[2]) +
                      " points, " + std::to_string(z[3]) + " edges exceed the handle");
            return ORB_ERR_CAPACITY;
        }
        if (z[4] + z[2] == 0) continue;                // nothing to optimise (g2o's optimize returns without an iteration)
        slotOf[j] = (int)sizes.size();
        sizes.push_back(make_int4(z[1], z[2], z[3], z[4]));
        lambdaInit.push_back(maps[j].inertial ? 100.0 : 0.0);
        const Map& d = T[j];
        fill.push_back(lba::FillSrc{d.bPoses, d.bFixed, d.bCam, d.bPts, d.bEPt, d.bEPose, d.bObs, d.bIsg});
        flags.push_back(maps[j].stopFlag);
    }
    std::vector<lba::SlotOut> outs(sizes.size());
    if (!sizes.empty()) {
        CK(cudaMemcpyAsync(S.dev(fillTab), fill.data(), sizeof(lba::FillSrc) * fill.size(), cudaMemcpyHostToDevice, st));
        if (int rc = lba::solver_load_device(h, (int)sizes.size(), sizes.data(), lambdaInit.data(), S.dev<lba::FillSrc>(fillTab), outs.data())) return rc;
        if (int rc = lba::solver_check_structure(h, (int)sizes.size())) return rc;   // no LM run on a graph the structure kernel refused
        if (int rc = lba::solver_run(h, flags.data())) return rc;
        launches += 3;
    }
    std::vector<Solve> solves(nMaps);
    for (int j = 0; j < nMaps; ++j) {
        solves[j].status = status[j]; solves[j].solved = slotOf[j] >= 0;
        solves[j].r = slotOf[j] >= 0 ? outs[slotOf[j]] : lba::SlotOut{};
    }
    CK(cudaMemcpyAsync(S.dev(solveTab), solves.data(), sizeof(Solve) * nMaps, cudaMemcpyHostToDevice, st));
    local_ba_finish_kernel<<<nMaps, WT, 0, st>>>(S.dev<Map>(tab), S.dev<Solve>(solveTab));
    CK(cudaGetLastError());
    ++launches;
    CK(S.download(st));
    for (int j = 0; j < nMaps; ++j) *maps[j].status = status[j];
    lba::solver_set_local_launches(h, launches);
    return ORB_OK;
}
