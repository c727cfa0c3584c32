// Tracking::UpdateLocalMap's UpdateLocalKeyFrames and UpdateLocalPoints (reference src/Tracking.cc; monocular and mono-inertial) for a
// batch of streams: one CTA per stream (DESIGN.md §4).  Integer and ordering work only, so the result is the reference's byte for byte.
//   * Votes: parallel over the vote source, atomics into the stream's keyframeCounter.
//   * Voters and pKFmax: a block scan over the keyframe table, which is in the std::map's key order.
//   * Expansion and temporal walk: one warp; a ballot per covisibility / children list finds the first qualifying entry.  The walk over the
//     voters is sequential by definition (each push can change what the next voter adds) and ends after about 80 pushes.
//   * UpdateLocalPoints: an occurrence (local keyframe at reverse rank r, slot s) has the key (keys of the keyframes visited before it) + s,
//     which is its position in the reference's visit order.  atomicMin gives each good point its first occurrence; a block prefix count
//     over the occurrences in key order then numbers the points that are taken there, and the slab rows are gathered per point.
// The counter, the keyframe marks and the per-point keys are scratch: the matcher's staging in the host form, which ends in a stream
// synchronise, and a scratch buffer of the handle's own in the device form.
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include <string>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "matcher_context.h"
#include "staging.h"

namespace orbm {

using orbx::set_error;
using orbx::csr_ok;

constexpr int ULM_NT = 256;
constexpr int ULM_MAX_LOCAL_KF = 80;    // if(mvpLocalKeyFrames.size()>80) break;  /  mvpLocalKeyFrames.size()<80
constexpr int ULM_COVISIBLES = 10;      // GetBestCovisibilityKeyFrames(10)
constexpr int ULM_ND = 20;              // the temporal walk's const int Nd = 20

struct UlmArgs {
    OrbmUpdateLocalMapBatch in;
    OrbmUpdateLocalMapResult out;
    int* counter;        // [nKF] keyframeCounter
    uint8_t* mark;       // [nKF] mnTrackReferenceForFrame == mCurrentFrame.mnId
    int* key;            // [nPoints] first occurrence in UpdateLocalPoints' order (INT_MAX: none), then -2 - the point's local index
};

// Warp 0: appends the first keyframe of list[0, n) that is not bad and not marked, if any (the covisibles' and the children's loops, each
// of which pushes one keyframe and breaks).  Returns whether it pushed.
__device__ __forceinline__ bool push_first(const int* list, int n, const uint8_t* flags, volatile uint8_t* mark, int* localKF, int& nL) {
    const int lane = threadIdx.x & 31;
    for (int base = 0; base < n; base += 32) {
        const int e = base + lane;
        int k = -1;
        bool ok = false;
        if (e < n) { k = list[e]; ok = !(flags[k] & ORBM_KF_BAD) && !mark[k]; }
        const unsigned ball = __ballot_sync(0xffffffffu, ok);
        if (ball) {
            const int first = __shfl_sync(0xffffffffu, k, __ffs(ball) - 1);
            if (lane == 0) { localKF[nL] = first; mark[first] = 1; }
            ++nL;
            __syncwarp();
            return true;
        }
    }
    return false;
}

__global__ void __launch_bounds__(ULM_NT) update_local_map_kernel(const UlmArgs A) {
    const OrbmUpdateLocalMapBatch& I = A.in;
    const OrbmUpdateLocalMapResult& O = A.out;
    __shared__ int s_warp[33], s_bestC[ULM_NT / 32], s_bestK[ULM_NT / 32];
    __shared__ int s_nLocal, s_ref;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int k0 = I.kfStart[b], nk = I.kfStart[b + 1] - k0, p0 = I.pointStart[b], np = I.pointStart[b + 1] - p0;
    const uint8_t* flags = I.kfFlags + k0;
    const uint8_t* pointBad = I.pointBad + p0;
    int* counter = A.counter + k0;
    uint8_t* mark = A.mark + k0;
    int* key = A.key + p0;
    int* localKF = O.localKF + k0;
    for (int k = tid; k < nk; k += ULM_NT) { counter[k] = 0; mark[k] = 0; localKF[k] = -1; }
    for (int p = tid; p < np; p += ULM_NT) key[p] = INT_MAX;
    __syncthreads();

    // 1. keyframeCounter: every good point of the vote source, once per keypoint that holds it
    const int nSrc = I.nSrc[b];
    const int* src = I.srcPoint + (size_t)b * I.mcapLast;
    const bool lastFrame = I.voteLastFrame[b] != 0;
    const int nVote = lastFrame ? nSrc : I.nK[b];
    for (int i = tid; i < nVote; i += ULM_NT) {
        int j = i;
        if (!lastFrame) {
            j = I.match[(size_t)b * I.kcap + i];
            if (j < 0 || j >= nSrc) continue;
        }
        const int p = src[j];
        if (p < 0 || pointBad[p]) continue;
        for (int o = I.obsStart[p0 + p], oe = I.obsStart[p0 + p + 1]; o < oe; ++o) atomicAdd(&counter[I.obsKF[o]], 1);
    }
    __syncthreads();

    // 2. the good voters in key order, and pKFmax: the first of them with the largest count (strict >)
    int nL = 0, bestC = 0, bestK = -1;
    for (int base = 0; base < nk; base += ULM_NT) {
        const int k = base + tid;
        const int c = k < nk ? counter[k] : 0;
        const bool voter = c > 0 && !(flags[k] & ORBM_KF_BAD);
        int total;
        const int pos = orbx::block_scan_excl<ULM_NT>(voter ? 1 : 0, s_warp, total);
        if (voter) {
            localKF[nL + pos] = k;
            mark[k] = 1;
            if (c > bestC) { bestC = c; bestK = k; }
        }
        nL += total;
    }
    for (int d = 16; d; d >>= 1) {
        const int oc = __shfl_down_sync(0xffffffffu, bestC, d), ok = __shfl_down_sync(0xffffffffu, bestK, d);
        if (oc > bestC || (oc == bestC && oc > 0 && ok < bestK)) { bestC = oc; bestK = ok; }
    }
    if (lane == 0) { s_bestC[warp] = bestC; s_bestK[warp] = bestK; }
    __syncthreads();

    // 3. + 4. one warp: the neighbours of the voters (only the voters: the end iterator is taken before the loop), then the temporal walk
    if (warp == 0) {
        volatile uint8_t* vmark = mark;
        const int nVoters = nL;
        for (int v = 0; v < nVoters; ++v) {
            if (nL > ULM_MAX_LOCAL_KF) break;
            const int kf = localKF[v];
            const int c0 = I.covStart[k0 + kf], c1 = I.covStart[k0 + kf + 1];
            push_first(I.covKF + c0, c1 - c0, flags, vmark, localKF, nL);
            const int h0 = I.childStart[k0 + kf], h1 = I.childStart[k0 + kf + 1];
            push_first(I.childKF + h0, h1 - h0, flags, vmark, localKF, nL);
            const int pa = I.parent[k0 + kf];
            if (pa >= 0 && !vmark[pa]) {                  // the parent's isBad() is not tested
                if (lane == 0) { localKF[nL] = pa; vmark[pa] = 1; }
                ++nL;
                __syncwarp();
                break;
            }
        }
        if (lane == 0) {
            if (I.inertial[b] && nL < ULM_MAX_LOCAL_KF) {
                int t = I.lastKF[b];
                for (int i = 0; i < ULM_ND; ++i) {
                    if (t < 0) break;
                    if (!vmark[t]) {                      // a marked keyframe stalls the walk for the remaining steps
                        localKF[nL++] = t;
                        vmark[t] = 1;
                        t = I.prevKF[k0 + t];
                    }
                }
            }
            int c = 0, k = -1;
            for (int w = 0; w < ULM_NT / 32; ++w)
                if (s_bestC[w] > c || (s_bestC[w] == c && c > 0 && s_bestK[w] < k)) { c = s_bestC[w]; k = s_bestK[w]; }
            s_nLocal = nL;
            s_ref = k;
        }
    }
    __syncthreads();
    nL = s_nLocal;

    // 5. UpdateLocalPoints: first occurrence of every good point in (reverse local rank, slot) order ...
    int off = 0;
    for (int r = nL - 1; r >= 0; --r) {
        const int kf = localKF[r];
        const int s0 = I.slotStart[k0 + kf], n = I.slotStart[k0 + kf + 1] - s0;
        for (int s = tid; s < n; s += ULM_NT) {
            const int p = I.slotPoint[s0 + s];
            if (!pointBad[p]) atomicMin(&key[p], off + s);
        }
        off += n;
    }
    __syncthreads();
    // ... then the points numbered in that order: an occurrence takes its point when its key is the point's minimum
    int nM = 0;
    off = 0;
    for (int r = nL - 1; r >= 0; --r) {
        const int kf = localKF[r];
        const int s0 = I.slotStart[k0 + kf], n = I.slotStart[k0 + kf + 1] - s0;
        for (int base = 0; base < n; base += ULM_NT) {
            const int s = base + tid;
            int p = -1;
            bool first = false;
            if (s < n) { p = I.slotPoint[s0 + s]; first = !pointBad[p] && key[p] == off + s; }
            int total;
            const int pos = orbx::block_scan_excl<ULM_NT>(first ? 1 : 0, s_warp, total);
            if (first) key[p] = -2 - (nM + pos);       // read by no later occurrence as a match: keys are >= 0
            nM += total;
        }
        off += n;
    }
    __syncthreads();

    // the slabs: rows [0, nM) gathered per point, the rest zero; lastToLocal
    const int mcap = I.mcap;
    const bool fits = nM <= mcap;
    const size_t row0 = (size_t)b * mcap;
    if (fits) {
        for (int p = tid; p < np; p += ULM_NT) {
            const int v = key[p];
            if (v > -2) continue;
            const size_t l = row0 + (size_t)(-2 - v), q = (size_t)(p0 + p);
            O.localPoint[l] = p;
            for (int c = 0; c < 3; ++c) { O.worldPos[3 * l + c] = I.worldPos[3 * q + c]; O.normal[3 * l + c] = I.normal[3 * q + c]; }
            O.minDistInv[l] = I.minDistInv[q]; O.maxDistInv[l] = I.maxDistInv[q]; O.maxDistance[l] = I.maxDistance[q];
            for (int c = 0; c < 32; ++c) O.mpDesc[32 * l + c] = I.mpDesc[32 * q + c];
            O.hasObs[l] = I.hasObs[q];
            O.bad[l] = 0;
        }
    }
    for (int r = (fits ? nM : 0) + tid; r < mcap; r += ULM_NT) {
        const size_t l = row0 + r;
        O.localPoint[l] = -1;
        for (int c = 0; c < 3; ++c) { O.worldPos[3 * l + c] = 0.0f; O.normal[3 * l + c] = 0.0f; }
        O.minDistInv[l] = 0.0f; O.maxDistInv[l] = 0.0f; O.maxDistance[l] = 0.0f;
        for (int c = 0; c < 32; ++c) O.mpDesc[32 * l + c] = 0;
        O.hasObs[l] = 0;
        O.bad[l] = 0;
    }
    for (int j = tid; j < I.mcapLast; j += ULM_NT) {
        int v = -1;
        if (fits && j < nSrc && src[j] >= 0) {
            const int kv = key[src[j]];
            if (kv <= -2) v = -2 - kv;
        }
        O.lastToLocal[(size_t)b * I.mcapLast + j] = v;
    }
    if (tid == 0) { O.nLocalKF[b] = nL; O.refKF[b] = s_ref; O.nM[b] = nM; }
}

}  // namespace orbm

using namespace orbm;

namespace {

// The pointers and sizes every form needs.
int ulm_shape(const OrbmUpdateLocalMapBatch* in, const OrbmUpdateLocalMapResult* out, const char* who) {
    auto bad = [who](const char* what) { set_error(std::string(who) + ": " + what); return ORB_ERR_ARG; };
    if (!in || !out) return bad("null argument");
    if (in->batch < 1 || in->kcap < 1 || in->mcap < 1 || in->mcapLast < 1 || in->nKF < 0 || in->nPoints < 0) return bad("bad sizes");
    if (!in->kfStart || !in->pointStart || !in->nSrc || !in->srcPoint || !in->voteLastFrame || !in->inertial || !in->lastKF)
        return bad("a per-stream input is null");
    if (in->nKF > 0 && (!in->kfFlags || !in->covStart || !in->childStart || !in->parent || !in->prevKF || !in->slotStart))
        return bad("a keyframe table array is null");
    if (in->nPoints > 0 && (!in->pointBad || !in->obsStart || !in->worldPos || !in->normal || !in->minDistInv || !in->maxDistInv ||
                            !in->maxDistance || !in->mpDesc || !in->hasObs))
        return bad("a point array is null");
    if (!out->localKF && in->nKF > 0) return bad("localKF is null");
    if (!out->nLocalKF || !out->refKF || !out->localPoint || !out->nM || !out->worldPos || !out->normal || !out->minDistInv || !out->maxDistInv ||
        !out->maxDistance || !out->mpDesc || !out->hasObs || !out->bad || !out->lastToLocal)
        return bad("an output is null");
    return ORB_OK;
}

// The host form's data checks, before anything is staged.
int ulm_check(const OrbmUpdateLocalMapBatch& I) {
    const char* who = "orbm_update_local_map_batch";
    auto bad = [who](int b, const char* what) {
        set_error(std::string(who) + ": " + (b >= 0 ? "stream " + std::to_string(b) + ": " : std::string()) + what);
        return ORB_ERR_ARG;
    };
    const int B = I.batch;
    if (!csr_ok(B, I.kfStart) || I.kfStart[B] != I.nKF) return bad(-1, "kfStart must start at 0, not decrease and end at nKF");
    if (!csr_ok(B, I.pointStart) || I.pointStart[B] != I.nPoints) return bad(-1, "pointStart must start at 0, not decrease and end at nPoints");
    if (I.nKF > 0) {
        if (!csr_ok(I.nKF, I.covStart) || !csr_ok(I.nKF, I.childStart) || !csr_ok(I.nKF, I.slotStart))
            return bad(-1, "covStart / childStart / slotStart must start at 0 and not decrease");
        if ((I.covStart[I.nKF] > 0 && !I.covKF) || (I.childStart[I.nKF] > 0 && !I.childKF) || (I.slotStart[I.nKF] > 0 && !I.slotPoint))
            return bad(-1, "covKF / childKF / slotPoint is null");
    }
    if (I.nPoints > 0) {
        if (!csr_ok(I.nPoints, I.obsStart)) return bad(-1, "obsStart must start at 0 and not decrease");
        if (I.obsStart[I.nPoints] > 0 && !I.obsKF) return bad(-1, "obsKF is null");
    }
    bool needMatch = false;
    for (int b = 0; b < B; ++b) needMatch |= I.voteLastFrame[b] == 0;
    if (needMatch && (!I.match || !I.nK)) return bad(-1, "match / nK is null and a stream votes with the frame's matches");
    for (int b = 0; b < B; ++b) {
        const int k0 = I.kfStart[b], nk = I.kfStart[b + 1] - k0, p0 = I.pointStart[b], np = I.pointStart[b + 1] - p0;
        auto kf_ok = [nk](int k) { return k >= 0 && k < nk; };
        for (int k = k0; k < k0 + nk; ++k) {
            if (I.covStart[k + 1] - I.covStart[k] > ULM_COVISIBLES) return bad(b, "more than 10 covisibles");
            for (int e = I.covStart[k]; e < I.covStart[k + 1]; ++e) if (!kf_ok(I.covKF[e])) return bad(b, "covKF out of range");
            for (int e = I.childStart[k]; e < I.childStart[k + 1]; ++e) {
                if (!kf_ok(I.childKF[e])) return bad(b, "childKF out of range");
                if (e > I.childStart[k] && I.childKF[e] <= I.childKF[e - 1]) return bad(b, "children not in ascending order");
            }
            if (I.parent[k] < -1 || I.parent[k] >= nk || I.prevKF[k] < -1 || I.prevKF[k] >= nk) return bad(b, "parent / prevKF out of range");
            for (int s = I.slotStart[k]; s < I.slotStart[k + 1]; ++s)
                if (I.slotPoint[s] < 0 || I.slotPoint[s] >= np) return bad(b, "slotPoint out of range");
        }
        for (int p = p0; p < p0 + np; ++p)
            for (int o = I.obsStart[p]; o < I.obsStart[p + 1]; ++o) if (!kf_ok(I.obsKF[o])) return bad(b, "obsKF out of range");
        const int nSrc = I.nSrc[b];
        if (nSrc < 0 || nSrc > I.mcapLast) return bad(b, "nSrc outside [0, mcapLast]");
        for (int j = 0; j < nSrc; ++j) {
            const int p = I.srcPoint[(size_t)b * I.mcapLast + j];
            if (p < -1 || p >= np) return bad(b, "srcPoint out of range");
        }
        if (I.lastKF[b] < -1 || I.lastKF[b] >= nk) return bad(b, "lastKF out of range");
        if (I.voteLastFrame[b] == 0) {
            if (I.nK[b] < 0 || I.nK[b] > I.kcap) return bad(b, "nK outside [0, kcap]");
            for (int i = 0; i < I.nK[b]; ++i) {
                const int m = I.match[(size_t)b * I.kcap + i];
                if (m < -1 || m >= nSrc) return bad(b, "match outside [-1, nSrc)");
            }
        }
    }
    return ORB_OK;
}

// Launches over the scratch: counter [nKF] int, mark [nKF] u8, key [nPoints] int.
int ulm_launch(int* counter, uint8_t* mark, int* key, const OrbmUpdateLocalMapBatch& in, const OrbmUpdateLocalMapResult& out, cudaStream_t st) {
    UlmArgs A;
    A.in = in; A.out = out;
    A.counter = counter; A.mark = mark; A.key = key;
    update_local_map_kernel<<<(unsigned)in.batch, ULM_NT, 0, st>>>(A);
    CK(cudaGetLastError());
    return ORB_OK;
}

}  // namespace

extern "C" int orbm_update_local_map_batch_device(orbm_handle* h, const OrbmUpdateLocalMapBatch* in, const OrbmUpdateLocalMapResult* out, void* stream) {
    const char* who = "orbm_update_local_map_batch_device";
    if (!h) { set_error(std::string(who) + ": bad argument"); return ORB_ERR_ARG; }
    if (int rc = ulm_shape(in, out, who)) return rc;
    const MatcherContext ctx = matcher_context(h);
    CK(cudaSetDevice(ctx.device));
    const size_t align = 256, NK = (size_t)in->nKF, NP = (size_t)in->nPoints;
    const size_t oMark = (4 * NK + align - 1) / align * align, oKey = oMark + (NK + align - 1) / align * align;
    DeviceScratch& D = *ctx.localMapScratch;
    if (int rc = D.reserve(oKey + 4 * NP + 1)) return rc;
    if (int rc = ulm_launch((int*)D.ptr, D.ptr + oMark, (int*)(D.ptr + oKey), *in, *out, (cudaStream_t)stream)) return rc;
    *ctx.launches = 1;
    return ORB_OK;
}

extern "C" int orbm_update_local_map_batch(orbm_handle* h, const OrbmUpdateLocalMapBatch* in, const OrbmUpdateLocalMapResult* out) {
    const char* who = "orbm_update_local_map_batch";
    if (!h) { set_error(std::string(who) + ": bad argument"); return ORB_ERR_ARG; }
    if (int rc = ulm_shape(in, out, who)) return rc;
    if (int rc = ulm_check(*in)) return rc;
    const MatcherContext ctx = matcher_context(h);
    *ctx.launches = 0;
    const size_t B = in->batch, K = in->kcap, M = in->mcap, ML = in->mcapLast, NK = in->nKF, NP = in->nPoints;
    if (NK == 0) {                                        // every table is empty: no local keyframe, no local point
        for (size_t b = 0; b < B; ++b) { out->nLocalKF[b] = 0; out->refKF[b] = -1; out->nM[b] = 0; }
        for (size_t r = 0; r < B * M; ++r) {
            out->localPoint[r] = -1;
            for (int c = 0; c < 3; ++c) { out->worldPos[3 * r + c] = 0.0f; out->normal[3 * r + c] = 0.0f; }
            out->minDistInv[r] = out->maxDistInv[r] = out->maxDistance[r] = 0.0f;
            memset(out->mpDesc + 32 * r, 0, 32);
            out->hasObs[r] = out->bad[r] = 0;
        }
        for (size_t j = 0; j < B * ML; ++j) out->lastToLocal[j] = -1;
        return ORB_OK;
    }
    CK(cudaSetDevice(ctx.device));
    orbx::Staging& S = *ctx.staging;
    S.begin();
    bool needMatch = false;
    for (size_t b = 0; b < B; ++b) needMatch |= in->voteLastFrame[b] == 0;
    const size_t NC = in->covStart[NK], NH = in->childStart[NK], NS = in->slotStart[NK], NO = NP ? (size_t)in->obsStart[NP] : 0;
    const int iKf = S.in(in->kfStart, 4 * (B + 1)), iFlags = S.in(in->kfFlags, NK), iCovS = S.in(in->covStart, 4 * (NK + 1)),
              iCov = S.in(in->covKF, 4 * NC), iChS = S.in(in->childStart, 4 * (NK + 1)), iCh = S.in(in->childKF, 4 * NH),
              iPar = S.in(in->parent, 4 * NK), iPrev = S.in(in->prevKF, 4 * NK), iSlS = S.in(in->slotStart, 4 * (NK + 1)),
              iSl = S.in(in->slotPoint, 4 * NS), iPs = S.in(in->pointStart, 4 * (B + 1)), iBad = S.in(in->pointBad, NP),
              iObS = S.in(NP ? in->obsStart : nullptr, NP ? 4 * (NP + 1) : 0), iOb = S.in(in->obsKF, 4 * NO), iWp = S.in(in->worldPos, 12 * NP),
              iNo = S.in(in->normal, 12 * NP), iMin = S.in(in->minDistInv, 4 * NP), iMax = S.in(in->maxDistInv, 4 * NP),
              iRaw = S.in(in->maxDistance, 4 * NP), iDesc = S.in(in->mpDesc, 32 * NP), iObs = S.in(in->hasObs, NP), iNSrc = S.in(in->nSrc, 4 * B),
              iSrc = S.in(in->srcPoint, 4 * B * ML), iVote = S.in(in->voteLastFrame, B), iMatch = S.in(needMatch ? in->match : nullptr, needMatch ? 4 * B * K : 0),
              iNK = S.in(needMatch ? in->nK : nullptr, needMatch ? 4 * B : 0), iIn = S.in(in->inertial, B), iLast = S.in(in->lastKF, 4 * B);
    const int oKf = S.out(out->localKF, 4 * NK), oNL = S.out(out->nLocalKF, 4 * B), oRef = S.out(out->refKF, 4 * B), oLp = S.out(out->localPoint, 4 * B * M),
              oNM = S.out(out->nM, 4 * B), oWp = S.out(out->worldPos, 12 * B * M), oNo = S.out(out->normal, 12 * B * M), oMin = S.out(out->minDistInv, 4 * B * M),
              oMax = S.out(out->maxDistInv, 4 * B * M), oRaw = S.out(out->maxDistance, 4 * B * M), oDesc = S.out(out->mpDesc, 32 * B * M),
              oObs = S.out(out->hasObs, B * M), oBad = S.out(out->bad, B * M), oL2l = S.out(out->lastToLocal, 4 * B * ML);
    const int pCounter = S.scratch(4 * NK), pMark = S.scratch(NK), pKey = S.scratch(4 * NP);
    if (int rc = S.reserve()) return rc;
    OrbmUpdateLocalMapBatch d = *in;
    d.kfStart = S.dev<int>(iKf); d.kfFlags = S.dev(iFlags); d.covStart = S.dev<int>(iCovS); d.covKF = S.dev<int>(iCov); d.childStart = S.dev<int>(iChS);
    d.childKF = S.dev<int>(iCh); d.parent = S.dev<int>(iPar); d.prevKF = S.dev<int>(iPrev); d.slotStart = S.dev<int>(iSlS); d.slotPoint = S.dev<int>(iSl);
    d.pointStart = S.dev<int>(iPs); d.pointBad = S.dev(iBad); d.obsStart = S.dev<int>(iObS); d.obsKF = S.dev<int>(iOb); d.worldPos = S.dev<float>(iWp);
    d.normal = S.dev<float>(iNo); d.minDistInv = S.dev<float>(iMin); d.maxDistInv = S.dev<float>(iMax); d.maxDistance = S.dev<float>(iRaw);
    d.mpDesc = S.dev(iDesc); d.hasObs = S.dev(iObs); d.nSrc = S.dev<int>(iNSrc); d.srcPoint = S.dev<int>(iSrc); d.voteLastFrame = S.dev(iVote);
    d.match = S.dev<int>(iMatch); d.nK = S.dev<int>(iNK); d.inertial = S.dev(iIn); d.lastKF = S.dev<int>(iLast);
    const OrbmUpdateLocalMapResult o = {S.dev<int>(oKf), S.dev<int>(oNL), S.dev<int>(oRef), S.dev<int>(oLp), S.dev<int>(oNM), S.dev<float>(oWp),
                                        S.dev<float>(oNo), S.dev<float>(oMin), S.dev<float>(oMax), S.dev<float>(oRaw), S.dev(oDesc), S.dev(oObs),
                                        S.dev(oBad), S.dev<int>(oL2l)};
    CK(S.upload(ctx.stream));
    if (int rc = ulm_launch(S.dev<int>(pCounter), S.dev(pMark), S.dev<int>(pKey), d, o, ctx.stream)) return rc;
    *ctx.launches = 1;
    CK(S.download(ctx.stream));
    for (size_t b = 0; b < B; ++b)
        if (out->nM[b] > in->mcap) {
            set_error(std::string(who) + ": stream " + std::to_string(b) + ": the local map has " + std::to_string(out->nM[b]) + " points, more than mcap " +
                      std::to_string(in->mcap));
            return ORB_ERR_CAPACITY;
        }
    return ORB_OK;
}
