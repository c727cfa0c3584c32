// LocalMapping::ProcessNewKeyFrame's map-point loop and the tail of LocalMapping::SearchInNeighbors (src/LocalMapping.cc; monocular
// observations), each followed by KeyFrame::UpdateConnections (src/KeyFrame.cc), for a batch of keyframes: one CTA per keyframe.
// Within a keyframe the reference's order does not matter (DESIGN.md §4): UpdateNormalAndDepth and ComputeDistinctiveDescriptors of a
// point read only that point and the keyframes' fixed fields, and UpdateConnections skips the current keyframe's own observations, so it
// counts the call-start observations.  The steps of a CTA:
//   1. the slot statuses; a point's first slot is the smallest slot holding it (atomicMin);
//   2. warp per updated point: the normal and distances on lane 0 (the sum in key order), the distinctive descriptor over the warp
//      (distinctive_best, the function distinctive_kernel calls), with the new observation inserted at its key position;
//   3. KFcounter in shared memory (in the counter output beyond UC_SMEM_KF keyframes), atomics over (slot, observation);
//   4. the selection (th = 15, else the first strict maximum in key order), the ordered list by rank over (weight, key), the parent;
//   5. warp per AddConnection target: its new weight map re-sorted by (weight, key) without bad keyframes, unless the weight is equal.
// UpdateNormalAndDepth's float rules are normal_depth.cuh's.
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "matcher_context.h"
#include "normal_depth.cuh"
#include "staging.h"

namespace orbm {

using orbx::distinctive_best;
using orbx::update_normal_and_depth;
using orbx::set_error;
using orbx::csr_ok;
using orbx::all_distinct;

constexpr int UC_NT = 256;
constexpr int UC_TH = 15;
constexpr int UC_SMEM_KF = 4096;
constexpr int UC_MAX_OBS = 65534;      // + the new observation: distinctive_best's 16-bit row index

// One keyframe as the kernel sees it: the caller's arrays in the staging buffer, its outputs and its scratch.
struct UcItem {
    int mode, nKF, nSlots, nPoints, nlevels, firstConnection;
    const unsigned long long *order, *mnId; const uint8_t* kfFlags; const float* Ow;
    const int *connStart, *connKF, *connWeight; const float* scaleFactors;
    const int *slotPoint, *slotOctave; const uint8_t* slotDesc;
    const uint8_t* pointBad; const float* pos; const int *refKF, *obsStart, *obsKF, *obsIdx, *obsOctave; const uint8_t* obsDesc;
    uint8_t *slotStatus, *pointUpdated; float *normal, *minDistance, *maxDistance; int *descKF, *descIdx;
    int *counter, *nConnected, *orderedKF, *orderedWeight, *parent, *nbrCount, *nbrKF, *nbrWeight;
    int* firstSlot;          // [nPoints] the point's first good slot
    int* rows;               // [obsStart[nPoints] + nPoints] per point from obsStart[p] + p: its descriptor rows (observation, -1 = new)
    int* cand;               // [nKF] the keyframes of vPairs
};

// (w1, key1) > (w2, key2): the order of the ordered lists (sort ascending by pair<int, KeyFrame*>, then push_front)
__device__ __forceinline__ bool heavier(int w1, unsigned long long k1, int w2, unsigned long long k2) { return w1 > w2 || (w1 == w2 && k1 > k2); }

__global__ void __launch_bounds__(UC_NT) update_connections_kernel(const UcItem* __restrict__ items) {
    __shared__ UcItem I;
    __shared__ int s_cnt[UC_SMEM_KF];
    __shared__ int s_nmax, s_nCand;
    __shared__ unsigned long long s_maxKey;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { I = items[blockIdx.x]; s_nmax = 0; s_nCand = 0; s_maxKey = ~0ull; }
    __syncthreads();
    int* cnt = I.nKF <= UC_SMEM_KF ? s_cnt : I.counter;
    const int nNbr = I.connStart[I.nKF] + I.nKF;
    for (int k = tid; k < I.nKF; k += UC_NT) { cnt[k] = 0; I.orderedKF[k] = -1; I.orderedWeight[k] = 0; I.nbrCount[k] = -1; }
    for (int e = tid; e < nNbr; e += UC_NT) { I.nbrKF[e] = -1; I.nbrWeight[e] = 0; }
    for (int p = tid; p < I.nPoints; p += UC_NT) {
        I.firstSlot[p] = INT_MAX; I.pointUpdated[p] = 0;
        I.normal[3 * p] = I.normal[3 * p + 1] = I.normal[3 * p + 2] = 0.f; I.minDistance[p] = I.maxDistance[p] = 0.f;
        I.descKF[p] = I.descIdx[p] = -1;
    }
    __syncthreads();
    for (int s = tid; s < I.nSlots; s += UC_NT) {
        const int p = I.slotPoint[s];
        if (p >= 0 && !I.pointBad[p]) atomicMin(&I.firstSlot[p], s);
    }
    __syncthreads();
    // 1 + 3: slot statuses, KFcounter
    const unsigned long long curId = I.mnId[0];
    for (int s = tid; s < I.nSlots; s += UC_NT) {
        const int p = I.slotPoint[s];
        if (p < 0 || I.pointBad[p]) { I.slotStatus[s] = ORBM_UC_SLOT_NONE; continue; }
        const int o0 = I.obsStart[p], o1 = I.obsStart[p + 1];
        const bool first = s == I.firstSlot[p];
        uint8_t st = ORBM_UC_SLOT_UPDATED;
        if (I.mode == ORBM_UC_PROCESS_NEW_KEYFRAME) {
            bool inKF = !first;                          // a later slot finds the observation its first slot added
            for (int o = o0; o < o1 && !inKF; ++o) inKF = I.obsKF[o] == 0;
            st = inKF ? ORBM_UC_SLOT_IN_KEYFRAME : ORBM_UC_SLOT_ADDED;
        }
        I.slotStatus[s] = st;
        if (first && st != ORBM_UC_SLOT_IN_KEYFRAME) I.pointUpdated[p] = 1;
        for (int o = o0; o < o1; ++o) {
            const int k = I.obsKF[o];
            if (I.mnId[k] != curId && !(I.kfFlags[k] & (ORBM_KF_BAD | ORBM_KF_OTHER_MAP))) atomicAdd(&cnt[k], 1);
        }
    }
    __syncthreads();
    // 2: UpdateNormalAndDepth and ComputeDistinctiveDescriptors, warp per updated point
    for (int p = warp; p < I.nPoints; p += UC_NT / 32) {
        if (!I.pointUpdated[p]) continue;
        const int o0 = I.obsStart[p], o1 = I.obsStart[p + 1];
        const int ns = I.mode == ORBM_UC_PROCESS_NEW_KEYFRAME ? I.firstSlot[p] : -1;     // the slot of the new observation
        int* rows = I.rows + o0 + p;
        int nRows = 0;
        if (lane == 0) {
            const unsigned long long newKey = I.order[0];
            bool pending = ns >= 0;
            int o = o0;
            // the observations in key order with the new one inserted at its key; the descriptor rows of the good observers on the way
            auto next = [&](int& k, int& oct) {
                int row;
                if (pending && (o == o1 || I.order[I.obsKF[o]] > newKey)) { k = 0; oct = I.slotOctave[ns]; row = -1; pending = false; }
                else if (o == o1) return false;
                else { k = I.obsKF[o]; oct = I.obsOctave[o]; row = o; ++o; }
                if (!(I.kfFlags[k] & ORBM_KF_BAD)) rows[nRows++] = row;
                return true;
            };
            update_normal_and_depth(I.pos + 3 * p, I.Ow, I.refKF[p], I.scaleFactors, I.nlevels, next, I.normal + 3 * p, I.minDistance + p, I.maxDistance + p);
        }
        nRows = __shfl_sync(0xffffffffu, nRows, 0);
        __syncwarp();
        if (nRows == 0) continue;                       // every observer bad: mDescriptor unchanged
        const uint8_t *obsDesc = I.obsDesc, *newRow = ns >= 0 ? I.slotDesc + (size_t)ns * 32 : nullptr;
        const int b = distinctive_best(nRows, lane, [&](int j) { const int r = rows[j]; return r >= 0 ? obsDesc + (size_t)r * 32 : newRow; });
        if (lane == 0) {
            const int r = rows[b];
            I.descKF[p] = r >= 0 ? I.obsKF[r] : 0;
            I.descIdx[p] = r >= 0 ? I.obsIdx[r] : ns;
        }
    }
    // 4: the selection, the ordered list, the parent
    for (int k = tid; k < I.nKF; k += UC_NT) {
        const int c = cnt[k];
        if (cnt != I.counter) I.counter[k] = c;
        if (c > 0) atomicMax(&s_nmax, c);
    }
    __syncthreads();
    const int nmax = s_nmax;
    if (nmax == 0) {                                     // KFcounter.empty(): return
        if (tid == 0) { *I.nConnected = -1; *I.parent = -1; }
        return;
    }
    for (int k = tid; k < I.nKF; k += UC_NT)
        if (cnt[k] == nmax) atomicMin(&s_maxKey, I.order[k]);
    __syncthreads();
    for (int k = tid; k < I.nKF; k += UC_NT) {
        const int c = cnt[k];
        if (c >= UC_TH || (nmax < UC_TH && c == nmax && I.order[k] == s_maxKey)) I.cand[atomicAdd(&s_nCand, 1)] = k;
    }
    __syncthreads();
    const int nCand = s_nCand;
    for (int i = tid; i < nCand; i += UC_NT) {
        const int k = I.cand[i], w = cnt[k];
        const unsigned long long key = I.order[k];
        int r = 0;
        for (int j = 0; j < nCand; ++j) { const int kj = I.cand[j]; r += heavier(cnt[kj], I.order[kj], w, key); }
        I.orderedKF[r] = k; I.orderedWeight[r] = w;
    }
    __syncthreads();
    if (tid == 0) {
        *I.nConnected = nCand;
        *I.parent = I.firstConnection && !(I.kfFlags[0] & ORBM_KF_INIT) ? I.orderedKF[0] : -1;
    }
    // 5: AddConnection(KF, w) on every keyframe of vPairs, warp per keyframe
    for (int i = warp; i < nCand; i += UC_NT / 32) {
        const int k = I.cand[i], w = cnt[k], c0 = I.connStart[k], c1 = I.connStart[k + 1];
        int old = -1;
        for (int c = c0 + lane; c < c1; c += 32)
            if (I.connKF[c] == 0) old = I.connWeight[c];
        old = __reduce_max_sync(0xffffffffu, old);
        if (old == w) continue;                          // an equal weight: AddConnection returns before UpdateBestCovisibles
        const int m = c1 - c0 + (old < 0);               // the weight map with the current keyframe set (or inserted at the end)
        auto entry = [&](int e, int& kk, int& ww) {
            if (e < c1 - c0) { kk = I.connKF[c0 + e]; ww = kk == 0 ? w : I.connWeight[c0 + e]; }
            else { kk = 0; ww = w; }
        };
        int good = 0;
        for (int e = lane; e < m; e += 32) {
            int kk, ww;
            entry(e, kk, ww);
            if (I.kfFlags[kk] & ORBM_KF_BAD) continue;
            ++good;
            const unsigned long long key = I.order[kk];
            int r = 0;
            for (int f = 0; f < m; ++f) {
                int kf, wf;
                entry(f, kf, wf);
                r += !(I.kfFlags[kf] & ORBM_KF_BAD) && heavier(wf, I.order[kf], ww, key);
            }
            I.nbrKF[c0 + k + r] = kk; I.nbrWeight[c0 + k + r] = ww;
        }
        good = __reduce_add_sync(0xffffffffu, good);
        if (lane == 0) I.nbrCount[k] = good;
    }
}

}  // namespace orbm

using namespace orbm;

namespace {

// ORB_ERR_ARG / ORB_ERR_CAPACITY with a message naming the item, or ORB_OK.
int check_item(const OrbmConnectionsItem& it, int j) {
    auto fail = [j](int rc, const char* what) { set_error("orbm_update_connections_batch: item " + std::to_string(j) + ": " + what); return rc; };
    auto bad = [&](const char* what) { return fail(ORB_ERR_ARG, what); };
    if (it.mode != ORBM_UC_PROCESS_NEW_KEYFRAME && it.mode != ORBM_UC_SEARCH_IN_NEIGHBORS) return bad("unknown mode");
    if (it.nKF < 1 || it.nSlots < 0 || it.nPoints < 0 || it.nlevels < 1) return bad("nKF < 1, nlevels < 1 or a negative count");
    if (!it.order || !it.mnId || !it.kfFlags || !it.cameraCenter || !it.connStart || !it.scaleFactors) return bad("a keyframe array is null");
    if (!it.counter || !it.nConnected || !it.orderedKF || !it.orderedWeight || !it.parent || !it.nbrCount) return bad("a connection output is null");
    if (it.nSlots > 0 && (!it.slotPoint || !it.slotOctave || !it.slotDesc || !it.slotStatus)) return bad("a slot array is null");
    if (it.nPoints > 0 && (!it.pointBad || !it.pointPos || !it.pointRefKF || !it.obsStart || !it.pointUpdated || !it.normal || !it.minDistance ||
                           !it.maxDistance || !it.descKF || !it.descIdx)) return bad("a point array is null");
    if (!all_distinct(it.order, it.nKF)) return bad("order keys are not distinct");
    if (!csr_ok(it.nKF, it.connStart)) return bad("connStart must start at 0 and not decrease");
    const int nConn = it.connStart[it.nKF];
    if (!it.nbrKF || !it.nbrWeight) return bad("nbrKF / nbrWeight is null");
    if (nConn > 0 && (!it.connKF || !it.connWeight)) return bad("connKF / connWeight is null");
    for (int k = 0; k < it.nKF; ++k)
        for (int c = it.connStart[k]; c < it.connStart[k + 1]; ++c) {
            if (it.connKF[c] < 0 || it.connKF[c] >= it.nKF) return bad("connKF out of range");
            if (c > it.connStart[k] && it.order[it.connKF[c]] <= it.order[it.connKF[c - 1]]) return bad("a connection map is not in key order");
        }
    for (int s = 0; s < it.nSlots; ++s) {
        if (it.slotPoint[s] < -1 || it.slotPoint[s] >= it.nPoints) return bad("slotPoint out of range");
        if (it.slotOctave[s] < 0 || it.slotOctave[s] >= it.nlevels) return bad("slotOctave outside [0, nlevels)");
    }
    if (it.nPoints > 0) {
        if (!csr_ok(it.nPoints, it.obsStart)) return bad("obsStart must start at 0 and not decrease");
        if (it.obsStart[it.nPoints] > 0 && (!it.obsKF || !it.obsIdx || !it.obsOctave || !it.obsDesc)) return bad("an observation array is null");
        for (int p = 0; p < it.nPoints; ++p) {
            const int o0 = it.obsStart[p], o1 = it.obsStart[p + 1];
            if (o1 - o0 > UC_MAX_OBS) return fail(ORB_ERR_CAPACITY, "a point has more than 65534 observations");
            bool refSeen = false;
            for (int o = o0; o < o1; ++o) {
                if (it.obsKF[o] < 0 || it.obsKF[o] >= it.nKF) return bad("obsKF out of range");
                if (it.obsIdx[o] < 0) return bad("obsIdx negative");
                if (it.obsOctave[o] < 0 || it.obsOctave[o] >= it.nlevels) return bad("obsOctave outside [0, nlevels)");
                if (o > o0 && it.order[it.obsKF[o]] <= it.order[it.obsKF[o - 1]]) return bad("observations not in key order");
                refSeen |= it.obsKF[o] == it.pointRefKF[p];
            }
            if (!it.pointBad[p] && !refSeen) return bad("a good point's mpRefKF is not among its observers");
        }
    }
    return ORB_OK;
}

// What UpdateConnections leaves of an item without slots: an empty counter, nothing changed.
void write_empty(const OrbmConnectionsItem& it) {
    const int nNbr = it.connStart[it.nKF] + it.nKF;
    std::fill(it.counter, it.counter + it.nKF, 0);
    std::fill(it.orderedKF, it.orderedKF + it.nKF, -1);
    std::fill(it.orderedWeight, it.orderedWeight + it.nKF, 0);
    std::fill(it.nbrCount, it.nbrCount + it.nKF, -1);
    std::fill(it.nbrKF, it.nbrKF + nNbr, -1);
    std::fill(it.nbrWeight, it.nbrWeight + nNbr, 0);
    *it.nConnected = -1; *it.parent = -1;
    for (int p = 0; p < it.nPoints; ++p) {
        it.pointUpdated[p] = 0;
        it.normal[3 * p] = it.normal[3 * p + 1] = it.normal[3 * p + 2] = 0.f; it.minDistance[p] = it.maxDistance[p] = 0.f;
        it.descKF[p] = it.descIdx[p] = -1;
    }
}

}  // namespace

extern "C" int orbm_update_connections_batch(orbm_handle* h, int nItems, const OrbmConnectionsItem* items) {
    if (!h || nItems < 0 || (nItems > 0 && !items)) { set_error("orbm_update_connections_batch: bad argument"); return ORB_ERR_ARG; }
    for (int j = 0; j < nItems; ++j)
        if (int rc = check_item(items[j], j)) return rc;
    const MatcherContext ctx = matcher_context(h);
    *ctx.launches = 0;
    std::vector<int> live;
    for (int j = 0; j < nItems; ++j) {
        if (items[j].nSlots > 0) live.push_back(j);
        else write_empty(items[j]);
    }
    if (live.empty()) return ORB_OK;
    CK(cudaSetDevice(ctx.device));
    orbx::Staging& S = *ctx.staging;
    S.begin();
    struct Pieces { int order, mnId, flags, Ow, connStart, connKF, connW, sf, slotPoint, slotOct, slotDesc, bad, pos, ref, obsStart, obsKF, obsIdx,
                    obsOct, obsDesc, slotStatus, updated, normal, minD, maxD, descKF, descIdx, counter, nConn, ordKF, ordW, parent, nbrCount, nbrKF,
                    nbrW, first, rows, cand; };
    std::vector<Pieces> pc(live.size());
    for (size_t i = 0; i < live.size(); ++i) {
        const OrbmConnectionsItem& it = items[live[i]];
        const size_t K = (size_t)it.nKF, NC = (size_t)it.connStart[it.nKF], NS = (size_t)it.nSlots, P = (size_t)it.nPoints,
                     NO = P ? (size_t)it.obsStart[it.nPoints] : 0, NB = NC + K;
        Pieces& q = pc[i];
        q.order = S.in(it.order, 8 * K); q.mnId = S.in(it.mnId, 8 * K); q.flags = S.in(it.kfFlags, K); q.Ow = S.in(it.cameraCenter, 12 * K);
        q.connStart = S.in(it.connStart, 4 * (K + 1)); q.connKF = S.in(it.connKF, 4 * NC); q.connW = S.in(it.connWeight, 4 * NC);
        q.sf = S.in(it.scaleFactors, 4 * (size_t)it.nlevels);
        q.slotPoint = S.in(it.slotPoint, 4 * NS); q.slotOct = S.in(it.slotOctave, 4 * NS); q.slotDesc = S.in(it.slotDesc, 32 * NS);
        q.bad = S.in(it.pointBad, P); q.pos = S.in(it.pointPos, 12 * P); q.ref = S.in(it.pointRefKF, 4 * P);
        q.obsStart = S.in(P ? it.obsStart : nullptr, P ? 4 * (P + 1) : 0); q.obsKF = S.in(it.obsKF, 4 * NO); q.obsIdx = S.in(it.obsIdx, 4 * NO);
        q.obsOct = S.in(it.obsOctave, 4 * NO); q.obsDesc = S.in(it.obsDesc, 32 * NO);
        q.slotStatus = S.out(it.slotStatus, NS); q.updated = S.out(it.pointUpdated, P); q.normal = S.out(it.normal, 12 * P);
        q.minD = S.out(it.minDistance, 4 * P); q.maxD = S.out(it.maxDistance, 4 * P); q.descKF = S.out(it.descKF, 4 * P); q.descIdx = S.out(it.descIdx, 4 * P);
        q.counter = S.out(it.counter, 4 * K); q.nConn = S.out(it.nConnected, 4); q.ordKF = S.out(it.orderedKF, 4 * K);
        q.ordW = S.out(it.orderedWeight, 4 * K); q.parent = S.out(it.parent, 4); q.nbrCount = S.out(it.nbrCount, 4 * K);
        q.nbrKF = S.out(it.nbrKF, 4 * NB); q.nbrW = S.out(it.nbrWeight, 4 * NB);
        q.first = S.scratch(4 * P); q.rows = S.scratch(4 * (NO + P)); q.cand = S.scratch(4 * K);
    }
    const int tab = S.in(nullptr, sizeof(UcItem) * live.size());
    if (int rc = S.reserve()) return rc;
    UcItem* T = S.host<UcItem>(tab);
    for (size_t i = 0; i < live.size(); ++i) {
        const OrbmConnectionsItem& it = items[live[i]];
        const Pieces& q = pc[i];
        UcItem d;
        d.mode = it.mode; d.nKF = it.nKF; d.nSlots = it.nSlots; d.nPoints = it.nPoints; d.nlevels = it.nlevels; d.firstConnection = it.firstConnection ? 1 : 0;
        d.order = S.dev<unsigned long long>(q.order); d.mnId = S.dev<unsigned long long>(q.mnId); d.kfFlags = S.dev(q.flags); d.Ow = S.dev<float>(q.Ow);
        d.connStart = S.dev<int>(q.connStart); d.connKF = S.dev<int>(q.connKF); d.connWeight = S.dev<int>(q.connW); d.scaleFactors = S.dev<float>(q.sf);
        d.slotPoint = S.dev<int>(q.slotPoint); d.slotOctave = S.dev<int>(q.slotOct); d.slotDesc = S.dev(q.slotDesc);
        d.pointBad = S.dev(q.bad); d.pos = S.dev<float>(q.pos); d.refKF = S.dev<int>(q.ref); d.obsStart = S.dev<int>(q.obsStart);
        d.obsKF = S.dev<int>(q.obsKF); d.obsIdx = S.dev<int>(q.obsIdx); d.obsOctave = S.dev<int>(q.obsOct); d.obsDesc = S.dev(q.obsDesc);
        d.slotStatus = S.dev(q.slotStatus); d.pointUpdated = S.dev(q.updated); d.normal = S.dev<float>(q.normal); d.minDistance = S.dev<float>(q.minD);
        d.maxDistance = S.dev<float>(q.maxD); d.descKF = S.dev<int>(q.descKF); d.descIdx = S.dev<int>(q.descIdx);
        d.counter = S.dev<int>(q.counter); d.nConnected = S.dev<int>(q.nConn); d.orderedKF = S.dev<int>(q.ordKF); d.orderedWeight = S.dev<int>(q.ordW);
        d.parent = S.dev<int>(q.parent); d.nbrCount = S.dev<int>(q.nbrCount); d.nbrKF = S.dev<int>(q.nbrKF); d.nbrWeight = S.dev<int>(q.nbrW);
        d.firstSlot = S.dev<int>(q.first); d.rows = S.dev<int>(q.rows); d.cand = S.dev<int>(q.cand);
        T[i] = d;
    }
    CK(S.upload(ctx.stream));
    update_connections_kernel<<<(unsigned)live.size(), UC_NT, 0, ctx.stream>>>(S.dev<UcItem>(tab));
    CK(cudaGetLastError());
    *ctx.launches = 1;
    CK(S.download(ctx.stream));
    return ORB_OK;
}
