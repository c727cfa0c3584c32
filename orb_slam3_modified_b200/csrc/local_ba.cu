// Optimizer::LocalBundleAdjustment (src/Optimizer.cc:1116-1498, monocular observations) as a whole, for a batch of maps
// (lba_local_bundle_adjustment_batch, include/orb_b200.h).  One call:
//   1. local_ba_walk_kernel, one CTA per map: the graph walk of :1125-1403 and the problem g2o would see (vertices sorted by mnId,
//      edges in insertion order), written in LbaProblem's layout into the staging buffer;
//   2. one small copy of the built sizes to the host, which lays the solver's slots out (lba.cu: Solver::layout) and reads the stop flags;
//   3. lba_fill_kernel copies the built problems into the slots, then lba.cu's structure and cluster kernels solve them;
//   4. local_ba_finish_kernel, one CTA per map: the outlier test, EraseObservation's cascade, SetPose, SetWorldPos, UpdateNormalAndDepth.
// Every order the reference defines by list walks is rebuilt as a first-appearance order: a position space (the local keyframes' slots, or
// the local points' observations, concatenated in list order) is scanned once with atomicMin for each item's first position, then one
// ordered block scan over the positions numbers the items.  The map table's check, staging, local-point walk and write-back of the local
// points are map_walk.cuh's, shared with local_inertial_ba_map.cu.
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
using orbx::all_distinct;
using orbx::segment;

constexpr int WT = 512;
constexpr unsigned char KF_SKIP = ORBM_KF_BAD | ORBM_KF_OTHER_MAP;   // isBad() || GetMap() != pCurrentMap

// One map as the kernels see it: the table (map_walk.cuh), and the caller's arrays, outputs and scratch only this function has.
struct Map : orbx::MapTable {
    int nCov, sortCap;
    const unsigned long long* mnId; const uint8_t* kfFlags; const float* pose7; const int* cov;
    const unsigned long long* pointId;
    // outputs
    int* sizes;                       // [8] walk verdict (0 built, 1 no fixed keyframe), nP, nL, nE, nF
    int *counts, *nLists, *localKF, *fixedKF; double* lmStats;
    double* optPose; uint8_t* edgeDepthPos;      // optional
    // the built problem (LbaProblem's layout)
    double* bPoses; uint8_t* bFixed; float* bCam; double* bPts; int *bEPt, *bEPose; double* bObs; float* bIsg;
    // scratch
    int *kfRank;                      // [nKF] local rank, -2 for the other entries of the covisible list (mnBALocalForKF), else -1
    int *kfVert, *ptVert;             // vertex of a keyframe / point, -1 none
    int *firstFix;                    // first position of a fixed-camera candidate
    int *locCand, *locBase;           // candidate of a local keyframe, slot base of the local keyframes
    unsigned long long* key; int* val;   // [sortCap] sort buffers
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
    for (int p = tid; p < M.nPoints; p += WT) M.ptVert[p] = -1;
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
    int Qo;
    const int nL = orbx::local_points<WT>(M, nLocal, [&](int r) { return M.locCand[r]; }, M.locBase, sm, KF_SKIP, Qo);
    // lFixedCameras: first appearance over (local point, observation) of the unmarked observers, kept when good and in the current map
    for (int q = tid; q < Qo; q += WT) {
        const int k = M.obsKF[orbx::obs_at(M, nL, q)];
        if (M.kfRank[k] == -1 && !(M.kfFlags[k] & KF_SKIP)) atomicMin(&M.firstFix[k], q);
    }
    __syncthreads();
    const int nFix = orbx::compact<WT>(Qo, sm, [&](int q) { const int k = M.obsKF[orbx::obs_at(M, nL, q)]; return M.kfRank[k] == -1 && M.firstFix[k] == q; },
                             [&](int q, int r) { M.fixedKF[r] = M.obsKF[orbx::obs_at(M, nL, q)]; });
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
    const int nE = orbx::compact<WT>(Qo, sm, [&](int q) { return !(M.kfFlags[M.obsKF[orbx::obs_at(M, nL, q)]] & KF_SKIP); }, [&](int q, int e) {
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
    orbx::clear_write_back<WT>(M);
    if (M.optPose) for (int i = tid; i < M.nKF; i += WT) for (int c = 0; c < 7; ++c) M.optPose[7 * i + c] = 0.0;
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
    orbx::write_back_points<WT>(M, nL, pointOf, [&](int o) -> uint8_t {
        const int e = M.obsEdge[o];
        if (e < 0) return LBA_OBS_NO_EDGE;
        const double chi2 = V.solved ? V.r.chi2[e] : 0.0;
        const uint8_t dpos = V.solved ? V.r.depthPos[e] : 1;
        if (M.edgeChi2) { M.edgeChi2[o] = chi2; M.edgeDepthPos[o] = dpos; }
        return chi2 > 5.991 || !dpos ? LBA_OBS_ERASED : LBA_OBS_KEPT;
    });
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
    // ~0ull pads the vertex sort's keys: an mnId equal to it could sort behind a padding entry and lose its vertex
    for (int k = 0; k < m.nKF; ++k)
        if (m.mnId[k] == ~0ull) return bad("a keyframe mnId is 2^64 - 1");
    std::vector<char> seen(m.nKF, 0);
    seen[0] = 1;
    for (int i = 0; i < m.nCov; ++i) {
        if (m.cov[i] < 1 || m.cov[i] >= m.nKF) return bad("cov out of range [1, nKF)");
        if (seen[m.cov[i]]) return bad("cov repeats a keyframe");
        seen[m.cov[i]] = 1;
    }
    if (int rc = orbx::check_slots(m, m.nCov + 1, bad)) return rc;
    if (m.nPoints > 0 && !all_distinct(m.pointId, m.nPoints)) return bad("point mnIds repeat");
    for (int p = 0; p < m.nPoints; ++p)
        if (m.pointId[p] == ~0ull) return bad("a point mnId is 2^64 - 1");
    return orbx::check_observations(m, bad);
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
    struct Pieces { orbx::MapTablePieces tab; int mnId, flags, pose, cov, pid, counts, nLists, localKF, fixedKF, lm, optPose, dpos, bPoses, bFixed,
                    bCam, bPts, bEPt, bEPose, bObs, bIsg, kfRank, kfVert, ptVert, firstFix, locCand, locBase, key, val, sortCap; };
    std::vector<Pieces> pc;
    const int sizesAll = S.out(nullptr, 32 * (size_t)nMaps);       // one piece, so that one small copy brings every map's sizes
    for (int j = 0; j < nMaps; ++j) {
        const LbaLocalMap& m = maps[j];
        const size_t K = m.nKF, C = m.nCov, P = m.nPoints, O = P ? m.obsStart[m.nPoints] : 0;
        pc.push_back({orbx::MapTablePieces(S, m, m.nCov + 1)});
        Pieces& q = pc.back();
        q.sortCap = 1;
        while (q.sortCap < std::max<int>(m.nKF, m.nPoints)) q.sortCap <<= 1;
        q.mnId = S.in(m.mnId, 8 * K); q.flags = S.in(m.kfFlags, K); q.pose = S.in(m.pose7, 28 * K); q.cov = S.in(m.cov, 4 * C); q.pid = S.in(m.pointId, 8 * P);
        q.counts = S.out(m.counts, 16); q.nLists = S.out(m.nLists, 12); q.localKF = S.out(m.localKF, 4 * K); q.fixedKF = S.out(m.fixedKF, 4 * K);
        q.lm = S.out(m.lmStats, 40); q.optPose = S.out(m.optPose, m.optPose ? 56 * K : 0); q.dpos = S.out(m.edgeDepthPositive, m.edgeChi2 ? O : 0);
        q.bPoses = S.scratch(56 * K); q.bFixed = S.scratch(K); q.bCam = S.scratch(16 * K); q.bPts = S.scratch(24 * P);
        q.bEPt = S.scratch(4 * O); q.bEPose = S.scratch(4 * O); q.bObs = S.scratch(16 * O); q.bIsg = S.scratch(4 * O);
        q.kfRank = S.scratch(4 * K); q.kfVert = S.scratch(4 * K); q.ptVert = S.scratch(4 * P); q.firstFix = S.scratch(4 * K);
        q.locCand = S.scratch(4 * (C + 1)); q.locBase = S.scratch(4 * (C + 2));
        q.key = S.scratch(8 * (size_t)q.sortCap); q.val = S.scratch(4 * (size_t)q.sortCap);
    }
    const int tab = S.in(nullptr, sizeof(Map) * nMaps), fillTab = S.scratch(sizeof(lba::FillSrc) * nMaps), solveTab = S.scratch(sizeof(Solve) * nMaps);
    if (int rc = S.reserve()) return rc;
    Map* T = S.host<Map>(tab);
    for (int j = 0; j < nMaps; ++j) {
        const LbaLocalMap& m = maps[j];
        const Pieces& q = pc[j];
        Map d;
        q.tab.bind(S, d);
        d.nCov = m.nCov; d.sortCap = q.sortCap;
        d.mnId = S.dev<unsigned long long>(q.mnId); d.kfFlags = S.dev(q.flags); d.pose7 = S.dev<float>(q.pose); d.cov = S.dev<int>(q.cov);
        d.pointId = S.dev<unsigned long long>(q.pid);
        d.sizes = S.dev<int>(sizesAll) + 8 * j; d.counts = S.dev<int>(q.counts); d.nLists = S.dev<int>(q.nLists); d.localKF = S.dev<int>(q.localKF);
        d.fixedKF = S.dev<int>(q.fixedKF); d.lmStats = S.dev<double>(q.lm);
        d.optPose = m.optPose ? S.dev<double>(q.optPose) : nullptr; d.edgeDepthPos = m.edgeChi2 ? S.dev(q.dpos) : nullptr;
        d.bPoses = S.dev<double>(q.bPoses); d.bFixed = S.dev(q.bFixed); d.bCam = S.dev<float>(q.bCam); d.bPts = S.dev<double>(q.bPts);
        d.bEPt = S.dev<int>(q.bEPt); d.bEPose = S.dev<int>(q.bEPose); d.bObs = S.dev<double>(q.bObs); d.bIsg = S.dev<float>(q.bIsg);
        d.kfRank = S.dev<int>(q.kfRank); d.kfVert = S.dev<int>(q.kfVert); d.ptVert = S.dev<int>(q.ptVert); d.firstFix = S.dev<int>(q.firstFix);
        d.locCand = S.dev<int>(q.locCand); d.locBase = S.dev<int>(q.locBase); d.key = S.dev<unsigned long long>(q.key); d.val = S.dev<int>(q.val);
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
