// LocalMapping::KeyFrameCulling() (src/LocalMapping.cc; monocular and mono-inertial, redundant_th = 0.9, Nd = 21) for a batch of maps:
// one CTA per map.  The walk over the local keyframes is sequential, as in the reference: culling keyframe k erases its observations,
// which can make a point bad and changes the counts of every later keyframe (DESIGN.md §4).  Each keyframe's step is parallel over its
// map-point slots: the redundancy counts, a block reduction, one thread for the decision (with the inertial guards and the prev / next
// links), then the erasures of the cull.  The map's live state -- point bad flags, Observations(), culled keyframes, links -- lives in
// device memory from the matcher's staging buffer; KeyFramesInMap() in shared memory.
//
// Float rules (the oracle evaluates the same expressions with -ffp-contract=off):
//   * nRedundantObservations > redundant_th * nMPs: both sides in float, one rounded product;
//   * t = mNextKF->mTimeStamp - mPrevKF->mTimeStamp: the difference in double, rounded to float;
//   * (GetImuPosition() - mPrevKF->GetImuPosition()).norm(): sqrtf((dx*dx + dy*dy) + dz*dz), every operation rounded, compared in
//     double with 0.02.
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "matcher_context.h"
#include "staging.h"

namespace orbm {

using orbx::set_error;
using orbx::csr_ok;

constexpr int KFC_NT = 256;
constexpr int KFC_ND = 21;
constexpr float KFC_REDUNDANT_TH = 0.9f;

// One map as the kernel sees it: the caller's arrays in the staging buffer, its outputs, and the live state (scratch).
struct KfcMap {
    int nKF, nLocal, nPoints, inertial, imuInit, inertialBA2, abortBA, keyFramesInMap;
    unsigned long long currentId, lastId;
    const unsigned long long* mnId; const uint8_t* kfFlags; const int *prev0, *next0; const double* ts; const float* pos;
    const int *local, *slotStart, *slotPoint, *slotOctave;
    const uint8_t* pointBad0; const int *obsStart, *obsKF, *obsOctave;
    uint8_t* status; int *nMPs, *nRedundant, *visited;
    uint8_t* kfGone;            // culled by this call: isBad(), its observations erased
    int *prev, *next;           // mPrevKF / mNextKF after the relinks so far (inertial)
    uint8_t* pointBad; int* nObs;
};

enum { KFC_CONTINUE = 0, KFC_FALL_THROUGH = 1, KFC_ERASE = 2 };

__global__ void __launch_bounds__(KFC_NT) keyframe_culling_kernel(const KfcMap* __restrict__ maps) {
    __shared__ KfcMap M;
    __shared__ int s_mps[KFC_NT / 32], s_red[KFC_NT / 32];
    __shared__ int s_decision, s_kfInMap;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { M = maps[blockIdx.x]; s_kfInMap = maps[blockIdx.x].keyFramesInMap; }
    __syncthreads();
    for (int k = tid; k < M.nKF; k += KFC_NT) {
        M.kfGone[k] = 0;
        if (M.inertial) { M.prev[k] = M.prev0[k]; M.next[k] = M.next0[k]; }
    }
    for (int p = tid; p < M.nPoints; p += KFC_NT) { M.pointBad[p] = M.pointBad0[p]; M.nObs[p] = M.obsStart[p + 1] - M.obsStart[p]; }
    for (int l = tid; l < M.nLocal; l += KFC_NT) { M.status[l] = ORBM_KFC_NOT_VISITED; M.nMPs[l] = -1; M.nRedundant[l] = -1; }
    __syncthreads();
    int count = 0;
    for (int l = 0; l < M.nLocal; ++l) {
        count = l + 1;
        const int k = M.local[l];
        if ((M.kfFlags[k] & (ORBM_KF_INIT | ORBM_KF_BAD)) || M.kfGone[k]) {
            if (tid == 0) M.status[l] = ORBM_KFC_SKIPPED;
            continue;
        }
        const int s0 = M.slotStart[l], s1 = M.slotStart[l + 1];
        int mps = 0, red = 0;
        for (int s = s0 + tid; s < s1; s += KFC_NT) {
            const int p = M.slotPoint[s];
            if (M.pointBad[p]) continue;
            ++mps;
            if (M.nObs[p] > 3) {
                const int level = M.slotOctave[s] + 1;
                int n = 0;
                for (int o = M.obsStart[p], oe = M.obsStart[p + 1]; o < oe; ++o) {
                    const int kfi = M.obsKF[o];
                    if (kfi == k || M.kfGone[kfi]) continue;
                    n += M.obsOctave[o] <= level;
                }
                red += n > 3;
            }
        }
        for (int d = 16; d; d >>= 1) { mps += __shfl_down_sync(0xffffffffu, mps, d); red += __shfl_down_sync(0xffffffffu, red, d); }
        if (lane == 0) { s_mps[warp] = mps; s_red[warp] = red; }
        __syncthreads();
        if (tid == 0) {
            mps = 0; red = 0;
            for (int w = 0; w < KFC_NT / 32; ++w) { mps += s_mps[w]; red += s_red[w]; }
            M.nMPs[l] = mps; M.nRedundant[l] = red;
            int st = ORBM_KFC_KEPT, dec = KFC_FALL_THROUGH;
            if ((float)red > __fmul_rn(KFC_REDUNDANT_TH, (float)mps)) {
                if (!M.inertial) {
                    st = ORBM_KFC_CULLED; dec = KFC_ERASE;
                } else if (s_kfInMap <= KFC_ND) {
                    st = ORBM_KFC_KEPT_FEW_KFS; dec = KFC_CONTINUE;
                } else if (M.mnId[k] > M.currentId - 2ull) {
                    st = ORBM_KFC_KEPT_RECENT; dec = KFC_CONTINUE;
                } else {
                    const int pv = M.prev[k], nx = M.next[k];
                    if (pv < 0 || nx < 0) {
                        st = ORBM_KFC_KEPT_NO_LINK;
                    } else {
                        const float t = __double2float_rn(__dsub_rn(M.ts[nx], M.ts[pv]));
                        const bool byTime = (M.imuInit && M.mnId[k] < M.lastId && t < 3.0f) || t < 0.5f;
                        bool still = false;
                        if (!byTime && !M.inertialBA2 && t < 3.0f) {
                            const float dx = __fsub_rn(M.pos[3 * k], M.pos[3 * pv]), dy = __fsub_rn(M.pos[3 * k + 1], M.pos[3 * pv + 1]),
                                        dz = __fsub_rn(M.pos[3 * k + 2], M.pos[3 * pv + 2]);
                            const float norm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
                            still = (double)norm < 0.02;
                        }
                        if (byTime || still) {
                            st = byTime ? ORBM_KFC_CULLED_TIME : ORBM_KFC_CULLED_STILL; dec = KFC_ERASE;
                            M.prev[nx] = pv; M.next[pv] = nx; M.prev[k] = -1; M.next[k] = -1;
                        } else {
                            st = ORBM_KFC_KEPT_IMU;
                        }
                    }
                }
            }
            if (dec == KFC_ERASE) {                      // KeyFrame::SetBadFlag
                if (M.kfFlags[k] & ORBM_KF_NOT_ERASE) { st = ORBM_KFC_NOT_ERASE; dec = KFC_FALL_THROUGH; }
                else { M.kfGone[k] = 1; --s_kfInMap; }
            }
            M.status[l] = (uint8_t)st;
            s_decision = dec;
        }
        __syncthreads();
        const int dec = s_decision;
        if (dec == KFC_ERASE) {                          // MapPoint::EraseObservation of every point of the keyframe
            for (int s = s0 + tid; s < s1; s += KFC_NT) {
                const int p = M.slotPoint[s];
                if (M.pointBad[p]) continue;
                if (--M.nObs[p] <= 2) M.pointBad[p] = 1;    // MapPoint::SetBadFlag: gone from every keyframe that held it
            }
            __syncthreads();
        }
        if (dec == KFC_CONTINUE) continue;
        if ((count > 20 && M.abortBA) || count > 100) break;
    }
    if (tid == 0) *M.visited = count;
}

}  // namespace orbm

using namespace orbm;

namespace {

// ORB_ERR_ARG with a message naming the map, or ORB_OK.
int check_map(const OrbmCullingMap& m, int j) {
    auto bad = [j](const char* what) { set_error("orbm_keyframe_culling_batch: map " + std::to_string(j) + ": " + what); return ORB_ERR_ARG; };
    if (m.nKF < 0 || m.nLocal < 0 || m.nPoints < 0) return bad("negative count");
    if (m.nLocal > m.nKF) return bad("nLocal > nKF");
    if (!m.visited) return bad("visited is null");
    if (m.nKF > 0 && (!m.mnId || !m.kfFlags)) return bad("mnId / kfFlags is null");
    if (m.inertial && m.nKF > 0 && (!m.prevKF || !m.nextKF || !m.timeStamp || !m.imuPosition)) return bad("an inertial array is null");
    if (m.nLocal > 0 && (!m.local || !m.slotStart || !m.status || !m.nMPs || !m.nRedundant)) return bad("local / slotStart / an output is null");
    if (m.nPoints > 0 && (!m.pointBad || !m.obsStart)) return bad("pointBad / obsStart is null");
    if (m.inertial)
        for (int k = 0; k < m.nKF; ++k)
            if (m.prevKF[k] < -1 || m.prevKF[k] >= m.nKF || m.nextKF[k] < -1 || m.nextKF[k] >= m.nKF) return bad("prevKF / nextKF out of range");
    for (int l = 0; l < m.nLocal; ++l) if (m.local[l] < 0 || m.local[l] >= m.nKF) return bad("local index out of range");
    if (m.nLocal > 0) {
        if (!csr_ok(m.nLocal, m.slotStart)) return bad("slotStart must start at 0 and not decrease");
        const int nSlots = m.slotStart[m.nLocal];
        if (nSlots > 0 && (!m.slotPoint || !m.slotOctave)) return bad("slotPoint / slotOctave is null");
        for (int s = 0; s < nSlots; ++s) {
            if (m.slotPoint[s] < 0 || m.slotPoint[s] >= m.nPoints) return bad("slotPoint out of range");
            if (m.slotOctave[s] < 0 || m.slotOctave[s] >= 256) return bad("slotOctave outside [0, 256)");
        }
    }
    if (m.nPoints > 0) {
        if (!csr_ok(m.nPoints, m.obsStart)) return bad("obsStart must start at 0 and not decrease");
        const int nObs = m.obsStart[m.nPoints];
        if (nObs > 0 && (!m.obsKF || !m.obsOctave)) return bad("obsKF / obsOctave is null");
        for (int o = 0; o < nObs; ++o) {
            if (m.obsKF[o] < 0 || m.obsKF[o] >= m.nKF) return bad("obsKF out of range");
            if (m.obsOctave[o] < 0 || m.obsOctave[o] >= 256) return bad("obsOctave outside [0, 256)");
        }
    }
    return ORB_OK;
}

}  // namespace

extern "C" int orbm_keyframe_culling_batch(orbm_handle* h, int nMaps, const OrbmCullingMap* maps) {
    if (!h || nMaps < 0 || (nMaps > 0 && !maps)) { set_error("orbm_keyframe_culling_batch: bad argument"); return ORB_ERR_ARG; }
    for (int j = 0; j < nMaps; ++j)
        if (int rc = check_map(maps[j], j)) return rc;
    const MatcherContext ctx = matcher_context(h);
    *ctx.launches = 0;
    std::vector<int> live;
    for (int j = 0; j < nMaps; ++j) {
        if (maps[j].nLocal > 0) live.push_back(j);
        else *maps[j].visited = 0;
    }
    if (live.empty()) return ORB_OK;
    CK(cudaSetDevice(ctx.device));
    orbx::Staging& S = *ctx.staging;
    S.begin();
    struct Pieces { int mnId, flags, prev0, next0, ts, pos, local, slotStart, slotPoint, slotOctave, bad0, obsStart, obsKF, obsOctave,
                    status, nMPs, nRed, visited, gone, prev, next, bad, nObs; };
    std::vector<Pieces> pc(live.size());
    for (size_t i = 0; i < live.size(); ++i) {
        const OrbmCullingMap& m = maps[live[i]];
        const size_t K = (size_t)m.nKF, L = (size_t)m.nLocal, P = (size_t)m.nPoints, NS = (size_t)m.slotStart[m.nLocal],
                     NO = P ? (size_t)m.obsStart[m.nPoints] : 0, KI = m.inertial ? K : 0;
        Pieces& q = pc[i];
        q.mnId = S.in(m.mnId, 8 * K); q.flags = S.in(m.kfFlags, K);
        q.prev0 = S.in(m.prevKF, 4 * KI); q.next0 = S.in(m.nextKF, 4 * KI); q.ts = S.in(m.timeStamp, 8 * KI); q.pos = S.in(m.imuPosition, 12 * KI);
        q.local = S.in(m.local, 4 * L); q.slotStart = S.in(m.slotStart, 4 * (L + 1)); q.slotPoint = S.in(m.slotPoint, 4 * NS);
        q.slotOctave = S.in(m.slotOctave, 4 * NS);
        q.bad0 = S.in(m.pointBad, P); q.obsStart = S.in(P ? m.obsStart : nullptr, P ? 4 * (P + 1) : 0); q.obsKF = S.in(m.obsKF, 4 * NO);
        q.obsOctave = S.in(m.obsOctave, 4 * NO);
        q.status = S.out(m.status, L); q.nMPs = S.out(m.nMPs, 4 * L); q.nRed = S.out(m.nRedundant, 4 * L); q.visited = S.out(m.visited, 4);
        q.gone = S.scratch(K); q.prev = S.scratch(4 * KI); q.next = S.scratch(4 * KI); q.bad = S.scratch(P); q.nObs = S.scratch(4 * P);
    }
    const int tab = S.in(nullptr, sizeof(KfcMap) * live.size());
    if (int rc = S.reserve()) return rc;
    KfcMap* T = S.host<KfcMap>(tab);
    for (size_t i = 0; i < live.size(); ++i) {
        const OrbmCullingMap& m = maps[live[i]];
        const Pieces& q = pc[i];
        KfcMap d;
        d.nKF = m.nKF; d.nLocal = m.nLocal; d.nPoints = m.nPoints; d.inertial = m.inertial ? 1 : 0; d.imuInit = m.imuInitialized ? 1 : 0;
        d.inertialBA2 = m.inertialBA2 ? 1 : 0; d.abortBA = m.abortBA ? 1 : 0; d.keyFramesInMap = m.keyFramesInMap;
        d.currentId = m.currentId; d.lastId = m.lastId;
        d.mnId = S.dev<unsigned long long>(q.mnId); d.kfFlags = S.dev(q.flags); d.prev0 = S.dev<int>(q.prev0); d.next0 = S.dev<int>(q.next0);
        d.ts = S.dev<double>(q.ts); d.pos = S.dev<float>(q.pos);
        d.local = S.dev<int>(q.local); d.slotStart = S.dev<int>(q.slotStart); d.slotPoint = S.dev<int>(q.slotPoint); d.slotOctave = S.dev<int>(q.slotOctave);
        d.pointBad0 = S.dev(q.bad0); d.obsStart = S.dev<int>(q.obsStart); d.obsKF = S.dev<int>(q.obsKF); d.obsOctave = S.dev<int>(q.obsOctave);
        d.status = S.dev(q.status); d.nMPs = S.dev<int>(q.nMPs); d.nRedundant = S.dev<int>(q.nRed); d.visited = S.dev<int>(q.visited);
        d.kfGone = S.dev(q.gone); d.prev = S.dev<int>(q.prev); d.next = S.dev<int>(q.next); d.pointBad = S.dev(q.bad); d.nObs = S.dev<int>(q.nObs);
        T[i] = d;
    }
    CK(S.upload(ctx.stream));
    keyframe_culling_kernel<<<(unsigned)live.size(), KFC_NT, 0, ctx.stream>>>(S.dev<KfcMap>(tab));
    CK(cudaGetLastError());
    *ctx.launches = 1;
    CK(S.download(ctx.stream));
    return ORB_OK;
}
