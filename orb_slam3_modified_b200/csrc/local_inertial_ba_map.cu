// Optimizer::LocalInertialBA (src/Optimizer.cc:2383-2958, monocular observations) as a whole, for a batch of maps
// (local_inertial_ba_map_batch, include/orb_b200.h).  One upload, three launches, one download:
//   1. local_inertial_ba_walk_kernel, one CTA per map: the window, the local points, lFixedKeyFrames and the edges (:2385-2478,
//      :2593-2763), written as a LocalInertialBAProblem straight into the solver's input region (liba_pack.h's layout, laid out on the host
//      from bounds), with the CSR lists pack_inputs builds and the problem's sizes in the map's Dev entry;
//   2. local_inertial_ba_kernel (local_inertial_ba.cu), unchanged, on those entries;
//   3. local_inertial_ba_map_finish_kernel, one CTA per map: the FAIL test, the write-back of the window, and per local point the erase
//      cascade, SetWorldPos and UpdateNormalAndDepth.
// The map table's check, staging, local-point walk (a first-appearance order over the window's slots) and write-back of the local points
// are map_walk.cuh's, shared with local_ba.cu.  The rule that fills lFixedKeyFrames is sequential: each point's observers are marked as
// far as the first good one, so a point's effect depends on every earlier point.  Only points with an observer outside the window and its
// predecessor can mark anything; the kernel compacts those, then repeatedly finds the first one that still has an unmarked observer (one
// parallel probe per 512 candidates) and lets one thread apply the rule to it.  Each such step marks at least one keyframe.
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "frame_pose.cuh"
#include "liba_pack.h"
#include "map_walk.cuh"
#include "staging.h"

namespace liba {
cudaError_t launch_solver(const Dev* probs, int count, cudaStream_t st);   // local_inertial_ba.cu
}

namespace liba_map {

using orbx::set_error;

constexpr int WT = 512;
constexpr int MAXW = 25;          // maxOpt with bLarge: the window never holds more
constexpr int MAXFIX = 200;       // maxFixKF
constexpr uint8_t MARK_LOCAL = 1, MARK_FIXED = 2;   // mnBALocalForKF / mnBAFixedForKF == pKF->mnId

thread_local int t_launches = 0;

// One map as the kernels see it: the table (map_walk.cuh), the caller's arrays, outputs and scratch only this function has, and its Dev entry.
struct Map : orbx::MapTable {
    int Nd, bRecInit;
    const uint8_t* kfFlags; const int* prevKF; const float *state21, *tcw12, *preint; const double* extr;
    const float* trackDepth;
    // outputs
    int *status, *nLists, *optKF, *fixedKF; uint8_t* ieLinked;
    float *kfVelocity, *kfBias6;
    double* stats8; double *optState21, *optTcw12;   // optional, with optPoint and edgeChi2
    // scratch
    uint8_t* mark;                    // [nKF] MARK_LOCAL / MARK_FIXED, 0 unmarked
    int* kfIdx;                       // [nKF] problem keyframe, -1 none
    int* cand;                        // [nPoints] local points with an observer left unmarked by the window and its predecessor
    liba::Dev* D;                     // the map's solver problem
};

__global__ void __launch_bounds__(WT) local_inertial_ba_walk_kernel(const Map* __restrict__ maps) {
    __shared__ Map M;
    __shared__ liba::Dev D;
    __shared__ int sm[33];
    __shared__ int s_win[MAXW], s_winBase[MAXW + 1], s_ieSrc[MAXW];
    __shared__ int s_nWin, s_N, s_nFix, s_nI, s_first;
    __shared__ int s_kfBase[MAXW], s_wcnt[WT / 32][MAXW];
    const int tid = threadIdx.x;
    if (tid == 0) { M = maps[blockIdx.x]; D = *M.D; }
    __syncthreads();
    for (int k = tid; k < M.nKF; k += WT) { M.mark[k] = 0; M.kfIdx[k] = -1; M.optKF[k] = -1; M.fixedKF[k] = -1; M.ieLinked[k] = 0; }
    // vpOptimizableKFs (:2395-2410): pKF, then mPrevKF while it exists, Nd keyframes at most
    if (tid == 0) {
        int n = 0;
        s_win[n++] = 0;
        for (int i = 1; i < M.Nd; ++i) {
            const int p = M.prevKF[s_win[n - 1]];
            if (p < 0) break;
            s_win[n++] = p;
        }
        s_nWin = n;
    }
    __syncthreads();
    const int nWin = s_nWin;
    for (int i = tid; i < nWin; i += WT) M.mark[s_win[i]] = MARK_LOCAL;
    // lLocalMapPoints (:2413-2428): first appearance over the slots of the whole window (before the pop below), NULL and bad points skipped
    int Qo;
    const int nL = orbx::local_points<WT>(M, nWin, [&](int i) { return s_win[i]; }, s_winBase, sm, ORBM_KF_BAD, Qo);
    // lFixedKeyFrames' first entry (:2431-2442): the window's predecessor, or the window's last keyframe popped
    if (tid == 0) {
        const int back = s_win[nWin - 1], pred = M.prevKF[back];
        if (pred >= 0) { M.fixedKF[0] = pred; M.mark[pred] = MARK_FIXED; s_N = nWin; }
        else { M.fixedKF[0] = back; M.mark[back] = MARK_FIXED; s_N = nWin - 1; }
        s_nFix = 1;
    }
    __syncthreads();
    const int N = s_N;
    // the other fixed keyframes (:2458-2478): per local point in list order, its observers in key order are marked up to the first good one,
    // which joins the list; the loop ends once the list holds maxFixKF.  Points whose observers are all marked by now never mark anything.
    auto unmarked = [&](int r) {
        const int p = M.localPoint[r];
        for (int o = M.obsStart[p]; o < M.obsStart[p + 1]; ++o) if (!M.mark[M.obsKF[o]]) return true;
        return false;
    };
    const int nCand = orbx::compact<WT>(nL, sm, unmarked, [&](int r, int c) { M.cand[c] = r; });
    __syncthreads();
    for (int c0 = 0; c0 < nCand && s_nFix < MAXFIX;) {
        if (tid == 0) s_first = INT_MAX;
        __syncthreads();
        const int c = c0 + tid;
        if (c < nCand && unmarked(M.cand[c])) atomicMin(&s_first, c);
        __syncthreads();
        const int f = s_first;
        __syncthreads();
        if (f == INT_MAX) { c0 += WT; continue; }
        if (tid == 0) {
            const int p = M.localPoint[M.cand[f]];
            for (int o = M.obsStart[p]; o < M.obsStart[p + 1]; ++o) {
                const int k = M.obsKF[o];
                if (M.mark[k]) continue;
                M.mark[k] = MARK_FIXED;
                if (!(M.kfFlags[k] & ORBM_KF_BAD)) { M.fixedKF[s_nFix++] = k; break; }
            }
        }
        __syncthreads();
        c0 = f + 1;
    }
    const int nFix = s_nFix;
    // the problem's keyframes: the window (newest first), then lFixedKeyFrames
    const int nK = N + nFix;
    for (int v = tid; v < nK; v += WT) {
        const int k = v < N ? s_win[v] : M.fixedKF[v - N];
        if (v < N) M.optKF[v] = k;
        M.kfIdx[k] = v;
        for (int c = 0; c < 21; ++c) D.kfState[21 * v + c] = (double)M.state21[21 * k + c];
        for (int c = 0; c < 12; ++c) D.kfTcw[12 * v + c] = (double)M.tcw12[12 * k + c];
        for (int c = 0; c < 4; ++c) const_cast<float*>(D.cam)[4 * v + c] = M.cam4[4 * k + c];
    }
    if (tid < 24) const_cast<double*>(D.extr)[tid] = M.extr[tid];
    for (int r = tid; r < nL; r += WT) {
        const int p = M.localPoint[r];
        for (int c = 0; c < 3; ++c) D.pts[3 * r + c] = (double)M.pos[3 * p + c];
        const_cast<float*>(D.trackDepth)[r] = M.trackDepth[p];
    }
    __syncthreads();
    // inertial edges (:2593-2656), keyed on the window index: bImu && mPrevKF->bImu && mpImuPreintegrated; Huber for i == N-1 or bRecInit,
    // information x 1e-2 for i == N-1
    if (tid == 0) {
        int nI = 0;
        for (int i = 0; i < N; ++i) {
            const int k = s_win[i], p = M.prevKF[k];
            if (p < 0 || !(M.kfFlags[p] & ORBM_KF_IMU) || !(M.kfFlags[k] & ORBM_KF_PREINT)) continue;
            const_cast<int*>(D.ieKf1)[nI] = M.kfIdx[p]; const_cast<int*>(D.ieKf2)[nI] = i;
            const_cast<uint8_t*>(D.ieRobust)[nI] = (i == N - 1 || M.bRecInit) ? 1 : 0;
            const_cast<double*>(D.ieInfoScale)[nI] = i == N - 1 ? 1e-2 : 1.0;
            M.ieLinked[i] = 1;
            s_ieSrc[nI++] = k;
        }
        s_nI = nI;
    }
    __syncthreads();
    const int nI = s_nI;
    for (int x = tid; x < nI * IMU_PREINT_FLOATS; x += WT)
        const_cast<float*>(D.preint)[x] = M.preint[(size_t)IMU_PREINT_FLOATS * s_ieSrc[x / IMU_PREINT_FLOATS] + x % IMU_PREINT_FLOATS];
    // mono edges (:2690-2763): local points in list order, observations in key order, observers marked, good and in the current map
    const int nE = orbx::compact<WT>(Qo, sm, [&](int q) {
        const int k = M.obsKF[orbx::obs_at(M, nL, q)];
        return M.mark[k] && !(M.kfFlags[k] & (ORBM_KF_BAD | ORBM_KF_OTHER_MAP));
    }, [&](int q, int e) {
        const int r = orbx::segment(M.lpBase, nL, q);
        const int o = M.obsStart[M.localPoint[r]] + q - M.lpBase[r];
        const_cast<int*>(D.ePt)[e] = r; const_cast<int*>(D.eKf)[e] = M.kfIdx[M.obsKF[o]];
        const_cast<double*>(D.obs)[2 * e] = (double)M.obsPt[2 * o]; const_cast<double*>(D.obs)[2 * e + 1] = (double)M.obsPt[2 * o + 1];
        const_cast<float*>(D.invSigma2)[e] = M.invLevelSigma2[M.obsOctave[o]];   // / uncertainty2, 1 for Pinhole
        M.obsEdge[o] = e;
    });
    __syncthreads();
    // CSR point -> edges: a point's edges are consecutive
    int* ptStart = const_cast<int*>(D.ptStart);
    orbx::block_prefix<WT>(nL, ptStart, sm, [&](int r) {
        const int p = M.localPoint[r];
        int n = 0;
        for (int o = M.obsStart[p]; o < M.obsStart[p + 1]; ++o) n += M.obsEdge[o] >= 0;
        return n;
    });
    if (tid == 0) ptStart[nL] = nE;
    for (int e = tid; e < nE; e += WT) const_cast<int*>(D.ptEdges)[e] = e;
    // CSR window keyframe -> edges in ascending edge order: per tile of WT edges, ranks among a warp's equal keyframes, then per keyframe
    // an exclusive scan over the warps
    int* kfStart = const_cast<int*>(D.kfStart);
    if (tid < N) s_kfBase[tid] = 0;
    __syncthreads();
    for (int e = tid; e < nE; e += WT) if (D.eKf[e] < N) atomicAdd(&s_kfBase[D.eKf[e]], 1);
    __syncthreads();
    if (tid == 0) {
        int run = 0;
        for (int i = 0; i < N; ++i) { kfStart[i] = run; const int n = s_kfBase[i]; s_kfBase[i] = run; run += n; }
        kfStart[N] = run;
    }
    __syncthreads();
    const int lane = tid & 31, warp = tid >> 5;
    for (int b = 0; b < nE; b += WT) {
        const int e = b + tid;
        const int k = e < nE && D.eKf[e] < N ? D.eKf[e] : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, k);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        if (lane < N) s_wcnt[warp][lane] = 0;
        __syncwarp();
        if (k >= 0 && rank == 0) s_wcnt[warp][k] = __popc(peers);
        __syncthreads();
        if (tid < N) {
            int run = s_kfBase[tid];
            for (int w = 0; w < WT / 32; ++w) { const int n = s_wcnt[w][tid]; s_wcnt[w][tid] = run; run += n; }
            s_kfBase[tid] = run;
        }
        __syncthreads();
        if (k >= 0) const_cast<int*>(D.kfEdges)[s_wcnt[warp][k] + rank] = e;
        __syncthreads();
    }
    if (tid == 0) {
        M.D->nKF = nK; M.D->nOpt = N; M.D->nI = nI; M.D->nL = nL; M.D->nE = nE;
        M.nLists[0] = N; M.nLists[1] = nFix; M.nLists[2] = nL; M.nLists[3] = nE;
    }
}

__global__ void __launch_bounds__(WT) local_inertial_ba_map_finish_kernel(const Map* __restrict__ maps) {
    __shared__ Map M;
    __shared__ liba::Dev D;
    const int tid = threadIdx.x;
    if (tid == 0) { M = maps[blockIdx.x]; D = *M.D; }
    __syncthreads();
    const bool failed = D.stats[2] != 0.0;             // (2 err < err_end || isnan) && !bLarge, :2884-2888
    const int N = D.nOpt, nK = D.nKF, nL = D.nL;
    if (tid < 8) M.stats8[tid] = D.stats[tid];
    if (tid == 0) *M.status = failed ? LIBA_LOCAL_FAILED : LIBA_LOCAL_RAN;
    // every output slot past the lists, and every slot of a FAILED map, holds zeros
    orbx::clear_write_back<WT>(M);
    for (int i = tid; i < M.nKF; i += WT) {
        for (int c = 0; c < 3; ++c) M.kfVelocity[3 * i + c] = 0.f;
        for (int c = 0; c < 6; ++c) M.kfBias6[6 * i + c] = 0.f;
        if (M.optState21) {
            for (int c = 0; c < 21; ++c) M.optState21[21 * i + c] = !failed && i < nK ? D.outState[21 * i + c] : 0.0;
            for (int c = 0; c < 12; ++c) M.optTcw12[12 * i + c] = !failed && i < nK ? D.outTcw[12 * i + c] : 0.0;
        }
    }
    for (int o = tid; o < M.nObs; o += WT) {
        const int e = M.obsEdge[o];
        if (M.edgeChi2) M.edgeChi2[o] = e >= 0 ? D.chi2[e] : 0.0;
        if (failed && e >= 0) M.obsFlag[o] = LBA_OBS_KEPT;
    }
    __syncthreads();
    if (failed) return;
    // the window (:2905-2930): SetPose(SE3f(Rcw.cast<float>(), tcw.cast<float>())), SetVelocity, SetNewBias(IMU::Bias(ba, bg))
    for (int i = tid; i < N; i += WT) {
        float R[9], t[3], T[7], Rr[9], tr[3], Ow[3];
        for (int c = 0; c < 9; ++c) R[c] = (float)D.outTcw[12 * i + c];
        for (int c = 0; c < 3; ++c) t[c] = (float)D.outTcw[12 * i + 9 + c];
        orbm::se3_from_matrix(R, t, T);
        orbm::update_pose_matrices(T, Rr, tr, Ow);
        const int k = M.optKF[i];
        for (int c = 0; c < 7; ++c) M.kfPose7[7 * i + c] = T[c];
        for (int c = 0; c < 3; ++c) {
            M.kfCenter[3 * i + c] = Ow[c]; M.Ow2[3 * k + c] = Ow[c];
            M.kfVelocity[3 * i + c] = (float)D.outState[21 * i + 12 + c];
            M.kfBias6[6 * i + c] = (float)D.outState[21 * i + 18 + c];
            M.kfBias6[6 * i + 3 + c] = (float)D.outState[21 * i + 15 + c];
        }
    }
    __syncthreads();
    // per local point (:2848-2902, :2935-2950): the erase loop in vToErase order -- points in list order, each point's edges in key order,
    // points being independent -- then SetWorldPos and UpdateNormalAndDepth against the new camera centres
    orbx::write_back_points<WT>(M, nL, [&](int i, double* X) { for (int c = 0; c < 3; ++c) X[c] = D.outPts[3 * i + c]; }, [&](int o) -> uint8_t {
        const int e = M.obsEdge[o];
        return e < 0 ? LBA_OBS_NO_EDGE : D.erase[e] ? LBA_OBS_ERASED : LBA_OBS_KEPT;
    });
}

// ORB_ERR_ARG with a message naming the map, or ORB_OK; *nWin = the window's length before the pop (a bound on N)
int check_map(const LocalInertialBAMap& m, int j, int* nWin) {
    auto bad = [j](const std::string& what) { set_error("local_inertial_ba_map_batch: map " + std::to_string(j) + ": " + what); return ORB_ERR_ARG; };
    if (m.nKF < 1 || m.nPoints < 0 || m.nlevels < 1) return bad("nKF < 1, nlevels < 1 or a negative count");
    if (!m.kfFlags || !m.prevKF || !m.state21 || !m.tcw12 || !m.cameraCenter || !m.cam4 || !m.extrinsics24 || !m.slotStart || !m.invLevelSigma2 ||
        !m.scaleFactors) return bad("a keyframe or map array is null");
    if (!m.status || !m.nLists || !m.optKF || !m.fixedKF || !m.ieLinked || !m.kfPose7 || !m.kfCenter || !m.kfVelocity || !m.kfBias6 || !m.stats8)
        return bad("a keyframe output is null");
    if (m.nPoints > 0 && (!m.pointFlags || !m.worldPos || !m.trackDepth || !m.refKF || !m.obsStart || !m.localPoint || !m.pointPos || !m.pointBad ||
                          !m.pointRefKF || !m.normal || !m.minDistance || !m.maxDistance)) return bad("a point array is null");
    const int nOpt = (m.optState21 != nullptr) + (m.optTcw12 != nullptr) + (m.optPoint != nullptr) + (m.edgeChi2 != nullptr);
    if (nOpt != 0 && nOpt != 4) return bad("optState21, optTcw12, optPoint and edgeChi2 go together");
    bool preint = false;
    for (int k = 0; k < m.nKF; ++k) {
        if (m.prevKF[k] < -1 || m.prevKF[k] >= m.nKF) return bad("prevKF out of range");
        preint |= (m.kfFlags[k] & ORBM_KF_PREINT) != 0;
    }
    if (preint && !m.preint) return bad("preint is null");
    if (m.kfFlags[0] & ORBM_KF_OTHER_MAP) return bad("pKF (entry 0) cannot be of another map");
    if (m.prevKF[0] < 0) return bad("pKF (entry 0) has no mPrevKF: the window would be empty");
    // the window as the kernel walks it, with its predecessor: Nd = min(KeyFramesInMap() - 2, maxOpt)
    const int Nd = std::min(m.keyFramesInMap - 2, m.bLarge ? 25 : 10);
    std::vector<int> chain(1, 0);
    for (int i = 1; i < Nd && m.prevKF[chain.back()] >= 0; ++i) chain.push_back(m.prevKF[chain.back()]);
    *nWin = (int)chain.size();
    const bool popped = m.prevKF[chain.back()] < 0;    // the last one moves to lFixedKeyFrames
    for (size_t i = 0; i + popped < chain.size(); ++i)
        if (!(m.kfFlags[chain[i]] & ORBM_KF_IMU)) return bad("a window keyframe has no ORBM_KF_IMU");
    if (!popped) chain.push_back(m.prevKF[chain.back()]);
    std::vector<int> sorted(chain);
    std::sort(sorted.begin(), sorted.end());
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) return bad("the mPrevKF chain revisits a keyframe within Nd + 1 steps");
    if (int rc = orbx::check_slots(m, m.nKF, bad)) return rc;
    return orbx::check_observations(m, bad);
}

}  // namespace liba_map

using namespace liba_map;

extern "C" int local_inertial_ba_map_last_launches(void) { return t_launches; }

extern "C" int local_inertial_ba_map_batch(int nMaps, const LocalInertialBAMap* maps, int device) {
    t_launches = 0;
    if (nMaps < 0 || (nMaps > 0 && !maps)) { set_error("local_inertial_ba_map_batch: bad argument"); return ORB_ERR_ARG; }
    std::vector<int> nWin(nMaps);
    for (int j = 0; j < nMaps; ++j)
        if (int rc = check_map(maps[j], j, &nWin[j])) return rc;
    orbx::ThreadStaging* S;
    if (int rc = orbx::thread_staging(device, &S)) return rc;
    if (nMaps == 0) return ORB_OK;
    S->begin();
    struct Pieces { orbx::MapTablePieces tab; int flags, prev, state, tcw, preint, extr, td, status, nLists, optKF, fixedKF, ieLinked, kfVel, kfBias,
                    stats, optState, optTcw, mark, kfIdx, cand, in, sc, out; liba::Layout lay; };
    std::vector<Pieces> pc;
    for (int j = 0; j < nMaps; ++j) {
        const LocalInertialBAMap& m = maps[j];
        const size_t K = m.nKF, P = m.nPoints, O = P ? m.obsStart[m.nPoints] : 0;
        bool preint = false;
        for (int k = 0; k < m.nKF; ++k) preint |= (m.kfFlags[k] & ORBM_KF_PREINT) != 0;
        pc.push_back({orbx::MapTablePieces(*S, m, m.nKF)});
        Pieces& q = pc.back();
        q.flags = S->in(m.kfFlags, K); q.prev = S->in(m.prevKF, 4 * K); q.state = S->in(m.state21, 84 * K); q.tcw = S->in(m.tcw12, 48 * K);
        q.preint = S->in(preint ? m.preint : nullptr, preint ? 4 * IMU_PREINT_FLOATS * K : 0); q.extr = S->in(m.extrinsics24, 24 * 8);
        q.td = S->in(m.trackDepth, 4 * P);
        q.status = S->out(m.status, 4); q.nLists = S->out(m.nLists, 16); q.optKF = S->out(m.optKF, 4 * K); q.fixedKF = S->out(m.fixedKF, 4 * K);
        q.ieLinked = S->out(m.ieLinked, K); q.kfVel = S->out(m.kfVelocity, 12 * K); q.kfBias = S->out(m.kfBias6, 24 * K); q.stats = S->out(m.stats8, 64);
        const bool dbg = m.optState21 != nullptr;
        q.optState = S->out(m.optState21, dbg ? 168 * K : 0); q.optTcw = S->out(m.optTcw12, dbg ? 96 * K : 0);
        q.mark = S->scratch(K); q.kfIdx = S->scratch(4 * K); q.cand = S->scratch(4 * P);
        // the solver's regions, laid out from bounds: N <= nWin keyframes in the window and as many inertial edges, at most every table
        // keyframe, point and observation in the problem
        q.lay = liba::make_layout(K, nWin[j], nWin[j], P, O, (int)O);
        q.in = S->scratch(q.lay.inBytes); q.sc = S->scratch(q.lay.scBytes); q.out = S->scratch(q.lay.outBytes);
    }
    const int devTab = S->in(nullptr, sizeof(liba::Dev) * nMaps), mapTab = S->in(nullptr, sizeof(Map) * nMaps);
    if (int rc = S->reserve()) return rc;
    liba::Dev* hDev = S->host<liba::Dev>(devTab);
    Map* T = S->host<Map>(mapTab);
    for (int j = 0; j < nMaps; ++j) {
        const LocalInertialBAMap& m = maps[j];
        const Pieces& q = pc[j];
        LocalInertialBAProblem bound{};                 // the sizes are the walk kernel's to write
        bound.iterations = m.bLarge ? 4 : 10; bound.bLarge = m.bLarge ? 1 : 0; bound.lambdaInit = m.bLarge ? 1e-2 : 1e0;
        liba::bind(hDev[j], bound, q.lay, S->dev(q.in), S->dev(q.sc), S->dev(q.out));
        Map d;
        q.tab.bind(*S, d);
        d.Nd = std::min(m.keyFramesInMap - 2, m.bLarge ? 25 : 10); d.bRecInit = m.bRecInit != 0;
        d.kfFlags = S->dev(q.flags); d.prevKF = S->dev<int>(q.prev); d.state21 = S->dev<float>(q.state); d.tcw12 = S->dev<float>(q.tcw);
        d.preint = S->dev<float>(q.preint); d.extr = S->dev<double>(q.extr); d.trackDepth = S->dev<float>(q.td);
        d.status = S->dev<int>(q.status); d.nLists = S->dev<int>(q.nLists); d.optKF = S->dev<int>(q.optKF); d.fixedKF = S->dev<int>(q.fixedKF);
        d.ieLinked = S->dev(q.ieLinked); d.kfVelocity = S->dev<float>(q.kfVel); d.kfBias6 = S->dev<float>(q.kfBias); d.stats8 = S->dev<double>(q.stats);
        const bool dbg = m.optState21 != nullptr;
        d.optState21 = dbg ? S->dev<double>(q.optState) : nullptr; d.optTcw12 = dbg ? S->dev<double>(q.optTcw) : nullptr;
        d.mark = S->dev(q.mark); d.kfIdx = S->dev<int>(q.kfIdx); d.cand = S->dev<int>(q.cand);
        d.D = S->dev<liba::Dev>(devTab) + j;
        T[j] = d;
    }
    CK(S->upload(S->stream));
    local_inertial_ba_walk_kernel<<<nMaps, WT, 0, S->stream>>>(S->dev<Map>(mapTab));
    CK(cudaGetLastError());
    CK(liba::launch_solver(S->dev<liba::Dev>(devTab), nMaps, S->stream));
    local_inertial_ba_map_finish_kernel<<<nMaps, WT, 0, S->stream>>>(S->dev<Map>(mapTab));
    CK(cudaGetLastError());
    CK(S->download(S->stream));
    t_launches = 3;
    return ORB_OK;
}
