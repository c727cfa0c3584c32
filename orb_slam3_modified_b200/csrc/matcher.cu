// H100 kernels + C-ABI for the per-frame matchers of ORBmatcher (reference src/ORBmatcher.cc):
//   SearchByProjection(Frame&, const vector<MapPoint*>&, ...)  :43-213   -> orbm_search_local_map
//   SearchByProjection(Frame&, const Frame&, th, bMono)        :1676-1887 -> orbm_search_last_frame[_batch_device]
//   DescriptorDistance                                          :2058-2074 -> hamming256 / orbm_descriptor_distance
//   cv::BFMatcher(NORM_HAMMING).knnMatch(k=2) (src/Frame.cc:1144)          -> orbm_bf_knn2
// plus Frame::AssignFeaturesToGrid / GetFeaturesInArea (src/Frame.cc:385-416,657-723) rebuilt on the device.
//
// Parallelisation of the reference's sequential claim rule (a keypoint that already holds a map point with
// observations is skipped by later map points, :84-86 / :1747-1749):
//   pass 1 (warp per map point, all streams at once): top-2 candidates by (Hamming distance, enumeration order)
//           against the claim state at entry;
//   pass 2 (one warp per stream, map points in index order): a pass-1 result is still exact unless its best or
//           second-best keypoint has been claimed meanwhile -- only then the warp rescans that map point against
//           the current claim state.  Claims live in a shared-memory bitset.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <string.h>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "exact_math.h"
#include "frame_pose.cuh"
#include "matcher_context.h"
#include "pose_inertial.h"
#include "pose_opt.h"
#include "staging.h"

using orbx::set_error;

namespace orbm {

using namespace orbx;
namespace cg = cooperative_groups;

constexpr int GRID_COLS = 64, GRID_ROWS = 48, GRID_CELLS = GRID_COLS * GRID_ROWS;   // include/Frame.h:44-45
constexpr int TH_HIGH = 100;       // src/ORBmatcher.cc:35
constexpr int HISTO_LENGTH = 30;   // :37

struct MatchParams {
    int batch, kcap, mcap, nlevels, mode;   // mode 0 = local map, 1 = last frame
    const OrbKeyPoint* kps; const uint8_t* desc; const int* nK;
    float minX, minY, maxX, maxY, gridWInv, gridHInv;
    const float* scaleFactors;
    const int* nM;
    const uint8_t *inView, *bad, *hasObs, *mpDesc, *valid;
    const float *depth, *projX, *projY, *viewCos, *xyz, *angle, *Tcw7;
    const int *level, *octave;
    float cam[4];
    float th, nnratio, thFar;
    int bFar, checkOri, resetState;
    const float* thBatch;      // mode 0: per-stream th [batch] instead of th (orbm_track_local_map_batch*); null otherwise
    const uint8_t* active;     // [batch] streams to run, or null (all)
    int ks, ms, descInSmem;   // shared-memory capacities of match_frame_kernel (keypoints, map points) and where the descriptors live
    // scratch
    float4* query;       // [batch][mcap]  u, v, r, bits(minLevel+1 | (maxLevel+1) << 8 | valid << 16)
    int4 *resultIdx, *resultDist;   // [batch][mcap]  the four best (keypoint index, distance) of pass 1, ascending
    // in/out
    int* match; uint8_t* claimed; int* nmatches;
    int* status;
};

// ---------------------------------------------------------------------------------------------
// Fused per-frame matcher.  One thread-block CLUSTER per frame (stream); every CTA of the cluster holds the frame in
// shared memory -- the 64x48 grid of Frame::AssignFeaturesToGrid (src/Frame.cc:385-416, cell lists in keypoint order
// = the reference's push_back order), keypoint positions / octaves and (when they fit) the descriptors -- and scans
// its share of the map points (pass 1, warp per map point).  CTA 0 of the cluster then resolves the reference's
// sequential claim rule in parallel (pass 2) and applies the rotation-histogram filter.
//
// Pass 1: the four smallest (Hamming distance, Frame::GetFeaturesInArea enumeration order) keys of every map point
//         among the keypoints that are not claimed at entry.
// Pass 2: the reference visits map points in index order; a keypoint assigned to a map point with observations is
//         skipped by all later map points (src/ORBmatcher.cc:84-86, :1747-1749).  With s_i the choice of map point i,
//         s_i = first candidate of i that no j < i with observations chose.  That recurrence is solved by fixed-point
//         iteration: every map point re-decides in parallel against minClaimer[c] = min{ j : s_j = c, j has
//         observations }; after iteration t the first t map points are final, and an iteration without a change is the
//         sequential result (induction over i).  Contention is rare, so it converges in a handful of sweeps instead of
//         the M dependent steps of a serial walk.  A map point whose four candidates are all taken (while more exist)
//         is rescanned by a warp against the current claims -- removing keys ranked after the second never changes
//         (best, second), so this is exact.
// ---------------------------------------------------------------------------------------------
constexpr int MF_NT = 512;
constexpr unsigned NONE16 = 0xFFFFu;

struct FrameSmem {          // carved from dynamic shared memory (layout computed by frame_smem_bytes)
    int* cnt;               // [GRID_CELLS] build counters; reused as histogram / scratch afterwards
    uint16_t* cellStart;    // [GRID_CELLS + 1]
    uint16_t* cellIdx;      // [Ks]
    float *kx, *ky;         // [Ks]
    uint8_t* koct;          // [Ks]
    uint32_t* initBits;     // [(Ks + 31) / 32] claimed at entry
    int* minClaimer;        // [Ks]
    uint16_t* choice;       // [Ms] chosen keypoint of every map point (NONE16: none / not accepted)
    uint8_t* mflags;        // [Ms] bit0 = has observations, bits 2.. = rotation bin + 1 (0: none)
    uint16_t* queue;        // [Ms] map points that need a rescan in the current sweep
    uint32_t* desc;         // [Ks][8] or nullptr (descriptors stay in global memory)
};

__host__ __device__ inline size_t al16(size_t v) { return (v + 15) & ~(size_t)15; }
__host__ __device__ inline size_t frame_smem_bytes(int Ks, int Ms, bool descInSmem) {
    size_t b = 0;
    b += al16(sizeof(int) * GRID_CELLS);
    b += al16(sizeof(uint16_t) * (GRID_CELLS + 1));
    b += al16(sizeof(uint16_t) * Ks);
    b += 2 * al16(sizeof(float) * Ks);
    b += al16(Ks);
    b += al16(sizeof(uint32_t) * ((Ks + 31) / 32));
    b += al16(sizeof(int) * Ks);
    b += 2 * al16(sizeof(uint16_t) * Ms);
    b += al16(Ms);
    if (descInSmem) b += al16((size_t)32 * Ks);
    return b;
}
// The opt-in maximum of dynamic shared memory per CTA (227 KB on sm_90) less 2 KB for the frame kernels' static shared memory
constexpr size_t FRAME_SMEM_LIMIT = 227 * 1024 - 2048;
__device__ __forceinline__ FrameSmem carve_frame_smem(uint8_t* p, int Ks, int Ms, bool descInSmem) {
    FrameSmem S;
    S.cnt = (int*)p; p += al16(sizeof(int) * GRID_CELLS);
    S.cellStart = (uint16_t*)p; p += al16(sizeof(uint16_t) * (GRID_CELLS + 1));
    S.cellIdx = (uint16_t*)p; p += al16(sizeof(uint16_t) * Ks);
    S.kx = (float*)p; p += al16(sizeof(float) * Ks);
    S.ky = (float*)p; p += al16(sizeof(float) * Ks);
    S.koct = p; p += al16(Ks);
    S.initBits = (uint32_t*)p; p += al16(sizeof(uint32_t) * ((Ks + 31) / 32));
    S.minClaimer = (int*)p; p += al16(sizeof(int) * Ks);
    S.choice = (uint16_t*)p; p += al16(sizeof(uint16_t) * Ms);
    S.mflags = p; p += al16(Ms);
    S.queue = (uint16_t*)p; p += al16(sizeof(uint16_t) * Ms);
    S.desc = descInSmem ? (uint32_t*)p : nullptr;
    return S;
}

template <int K>
struct TopK {   // the K smallest keys seen, ascending
    unsigned long long k[K];
    int i[K];
    __device__ __forceinline__ void init() {
#pragma unroll
        for (int j = 0; j < K; ++j) { k[j] = ~0ull; i[j] = -1; }
    }
    __device__ __forceinline__ void insert(unsigned long long key, int idx) {
        if (key >= k[K - 1]) return;
        k[K - 1] = key; i[K - 1] = idx;
#pragma unroll
        for (int j = K - 1; j > 0; --j) {
            if (k[j] < k[j - 1]) {
                const unsigned long long tk = k[j]; k[j] = k[j - 1]; k[j - 1] = tk;
                const int ti = i[j]; i[j] = i[j - 1]; i[j - 1] = ti;
            }
        }
    }
    // Afterwards every lane holds the K smallest keys of the whole warp.  Keys are unique (they carry the candidate's enumeration
    // rank), every lane's list is sorted, so the warp minimum is the minimum of the heads: K rounds of a 64-bit warp minimum (two
    // REDUX.MIN on the halves), the winning lane pops its head.
    __device__ __forceinline__ void warp_merge() {
        unsigned long long rk[K]; int ri[K];
#pragma unroll
        for (int j = 0; j < K; ++j) {
            const unsigned hi = (unsigned)(k[0] >> 32), lo = (unsigned)k[0];
            const unsigned mhi = __reduce_min_sync(0xffffffffu, hi);
            const unsigned mlo = __reduce_min_sync(0xffffffffu, hi == mhi ? lo : 0xffffffffu);
            const unsigned long long mk = ((unsigned long long)mhi << 32) | mlo;
            const bool won = k[0] == mk;
            const int src = __ffs(__ballot_sync(0xffffffffu, won)) - 1;
            rk[j] = mk; ri[j] = __shfl_sync(0xffffffffu, i[0], src);
            if (won && mk != ~0ull) {
#pragma unroll
                for (int q = 0; q + 1 < K; ++q) { k[q] = k[q + 1]; i[q] = i[q + 1]; }
                k[K - 1] = ~0ull; i[K - 1] = -1;
            }
        }
#pragma unroll
        for (int j = 0; j < K; ++j) { k[j] = rk[j]; i[j] = ri[j]; }
    }
};
typedef TopK<2> Top2;

// Warp-wide scan of the candidates of one query in Frame::GetFeaturesInArea order (src/Frame.cc:657-723): (ix, iy, position in
// the cell).  key = dist << 40 | cellRank << 20 | position; keeps the K smallest keys among keypoints that pass `usable`.
struct AnyDist { __device__ __forceinline__ bool operator()(int, int) const { return true; } };
template <int K, class UsableFn, class UsableDistFn = AnyDist>
__device__ __forceinline__ TopK<K> scan_candidates(const MatchParams& P, const FrameSmem& S, int f, float u, float v, float r, int minLevel,
                                                   int maxLevel, const uint32_t* mpd, UsableFn usable, UsableDistFn usableDist = AnyDist()) {
    const int lane = threadIdx.x & 31;
    TopK<K> t; t.init();
    const int nMinCellX = max(0, (int)floorf(fmul(fsub(fsub(u, P.minX), r), P.gridWInv)));
    const int nMaxCellX = min(GRID_COLS - 1, (int)ceilf(fmul(fadd(fsub(u, P.minX), r), P.gridWInv)));
    const int nMinCellY = max(0, (int)floorf(fmul(fsub(fsub(v, P.minY), r), P.gridHInv)));
    const int nMaxCellY = min(GRID_ROWS - 1, (int)ceilf(fmul(fadd(fsub(v, P.minY), r), P.gridHInv)));
    if (nMinCellX < GRID_COLS && nMaxCellX >= 0 && nMinCellY < GRID_ROWS && nMaxCellY >= 0) {
        const int ny = nMaxCellY - nMinCellY + 1, nx = nMaxCellX - nMinCellX + 1;
        const uint8_t* gdesc = P.desc + (size_t)f * P.kcap * 32;
        const bool bCheckLevels = (minLevel > 0) || (maxLevel >= 0);
        // c / ny by multiply-high (exact: c * ny < 2^32).  For ny = 1 (a window clipped to the first or last grid row) the magic
        // wraps to 0, so the quotient is c itself.
        const unsigned nyMagic = 0xFFFFFFFFu / (unsigned)ny + 1u;
        for (int c = lane; c < nx * ny; c += 32) {
            const int cq = ny > 1 ? (int)__umulhi((unsigned)c, nyMagic) : c;
            const int ix = nMinCellX + cq, iy = nMinCellY + (c - cq * ny);
            const int cell = ix * GRID_ROWS + iy;
            const int a = S.cellStart[cell], b = S.cellStart[cell + 1];
            for (int e = a; e < b; ++e) {
                const int idx = S.cellIdx[e];
                const int oct = S.koct[idx];
                if (bCheckLevels) {
                    if (oct < minLevel) continue;
                    if (maxLevel >= 0 && oct > maxLevel) continue;
                }
                const float dx = fsub(S.kx[idx], u), dy = fsub(S.ky[idx], v);
                if (!(fabsf(dx) < r && fabsf(dy) < r)) continue;
                if (!usable(idx)) continue;
                uint32_t dd[8];
                if (S.desc) {
                    const uint4* dp = reinterpret_cast<const uint4*>(S.desc + (size_t)idx * 8);
                    const uint4 d0 = dp[0], d1 = dp[1];
                    dd[0] = d0.x; dd[1] = d0.y; dd[2] = d0.z; dd[3] = d0.w; dd[4] = d1.x; dd[5] = d1.y; dd[6] = d1.z; dd[7] = d1.w;
                } else {
                    load_desc(gdesc + (size_t)idx * 32, dd);
                }
                const int dist = hamming256(mpd, dd);
                if (!usableDist(idx, dist)) continue;
                t.insert(((unsigned long long)dist << 40) | ((unsigned long long)c << 20) | (unsigned)(e - a), idx);
            }
        }
    }
    t.warp_merge();
    return t;
}

__device__ __forceinline__ void load_mp_desc(const MatchParams& P, int f, int i, uint32_t (&mpd)[8]) {
    load_desc(P.mpDesc + ((size_t)f * P.mcap + i) * 32, mpd);
}

// Query of map point i: search centre, radius and level window; returns false when the reference `continue`s.
__device__ __forceinline__ bool make_query(const MatchParams& P, int f, int i, float& u, float& v, float& r, int& minL, int& maxL) {
    const size_t o = (size_t)f * P.mcap + i;
    if (P.mode == 0) {   // src/ORBmatcher.cc:50-72
        if (!P.inView[o]) return false;
        if (P.bFar && P.depth[o] > P.thFar) return false;
        if (P.bad[o]) return false;
        const int lvl = min(max(P.level[o], 0), P.nlevels - 1);   // the host entry points reject out-of-range levels; device callers are clamped
        float rr = ((double)P.viewCos[o] > 0.998) ? 2.5f : 4.0f;   // RadiusByViewingCos :215-221
        const float th = P.thBatch ? P.thBatch[f] : P.th;
        if (th != 1.0f) rr = fmul(rr, th);
        u = P.projX[o]; v = P.projY[o];
        r = fmul(rr, P.scaleFactors[lvl]);
        minL = lvl - 1; maxL = lvl;
        return true;
    }
    // last frame, mono (:1702-1741): x3Dc = Tcw * x3Dw with Sophus' quaternion form (so3.hpp:358-367)
    if (!P.valid[o]) return false;
    float xc3[3];
    se3_transform(P.Tcw7 + (size_t)f * 7, P.xyz + 3 * o, xc3);
    const float xc = xc3[0], yc = xc3[1], zc = xc3[2];
    const float invzc = (float)(1.0 / (double)zc);
    if (invzc < 0) return false;
    u = fadd(fdiv(fmul(P.cam[0], xc), zc), P.cam[2]);   // Pinhole::project, Pinhole.cpp:43-49
    v = fadd(fdiv(fmul(P.cam[1], yc), zc), P.cam[3]);
    if (u < P.minX || u > P.maxX) return false;
    if (v < P.minY || v > P.maxY) return false;
    if (!(u == u) || !(v == v)) return false;   // NaN projections (zc == 0) fail every comparison above in the reference too
    const int oct = min(max(P.octave[o], 0), P.nlevels - 1);
    r = fmul(P.th, P.scaleFactors[oct]);
    minL = oct - 1; maxL = oct + 1;
    return true;
}

// rotation histogram bin (:1779-1789)
__device__ __forceinline__ int rot_bin(float lastAngle, float curAngle) {
    float rot = fsub(lastAngle, curAngle);
    if (rot < 0.0f) rot = fadd(rot, 360.0f);
    int bin = (int)roundf(fmul(rot, 1.0f / HISTO_LENGTH));
    if (bin == HISTO_LENGTH) bin = 0;
    return min(max(bin, 0), HISTO_LENGTH - 1);
}

// ComputeThreeMaxima (:2012-2053): the three fullest bins of the rotation histogram, -1 for the second and third when they hold less
// than a tenth of the first
__device__ __forceinline__ void three_maxima(const int* hist, int ind[3]) {
    int ind1 = -1, ind2 = -1, ind3 = -1, max1 = 0, max2 = 0, max3 = 0;
    for (int b = 0; b < HISTO_LENGTH; ++b) {
        const int s = hist[b];
        if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = b; }
        else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = b; }
        else if (s > max3) { max3 = s; ind3 = b; }
    }
    if ((float)max2 < fmul(0.1f, (float)max1)) { ind2 = -1; ind3 = -1; }
    else if ((float)max3 < fmul(0.1f, (float)max1)) { ind3 = -1; }
    ind[0] = ind1; ind[1] = ind2; ind[2] = ind3;
}
// the matches of bin b survive the rotation filter
__device__ __forceinline__ bool rot_kept(int b, const int ind[3]) { return b == ind[0] || b == ind[1] || b == ind[2]; }

// The rotation events of SearchByBoW and SearchForTriangulation: match i's bin + 1 in evBin[i], counted in the histogram
__device__ __forceinline__ void rot_event(int* hist, uint8_t* evBin, int i, float angle1, float angle2) {
    const int b = rot_bin(angle1, angle2);
    evBin[i] = (uint8_t)(b + 1);
    atomicAdd(&hist[b], 1);
}

// Frame::AssignFeaturesToGrid + PosInGrid (src/Frame.cc:385-416, :725-735): counting sort of the keypoints into the 64x48 grid held in
// shared memory, cell lists in increasing keypoint index (= the reference's push_back order); also stages positions, octaves and
// (when S.desc is set) the descriptors.  All threads of the CTA call; ends with a barrier.
__device__ void build_frame_smem(const FrameSmem& S, const OrbKeyPoint* kps, const uint8_t* gdesc, int K, float minX, float minY, float gridWInv,
                                 float gridHInv, int* s_warp) {
    const int tid = threadIdx.x;
    for (int c = tid; c < GRID_CELLS; c += MF_NT) S.cnt[c] = 0;
    __syncthreads();
    for (int i = tid; i < K; i += MF_NT) {
        const OrbKeyPoint kp = kps[i];
        S.kx[i] = kp.x; S.ky[i] = kp.y; S.koct[i] = (uint8_t)min(max(kp.octave, 0), 255);
        const int px = (int)roundf(fmul(fsub(kp.x, minX), gridWInv));
        const int py = (int)roundf(fmul(fsub(kp.y, minY), gridHInv));
        if (px >= 0 && px < GRID_COLS && py >= 0 && py < GRID_ROWS) atomicAdd(&S.cnt[px * GRID_ROWS + py], 1);
    }
    if (S.desc) {
        const uint4* src = reinterpret_cast<const uint4*>(gdesc);
        uint4* dst = reinterpret_cast<uint4*>(S.desc);
        for (int i = tid; i < 2 * K; i += MF_NT) dst[i] = __ldg(src + i);
    }
    __syncthreads();
    const int total = block_prefix<MF_NT>(GRID_CELLS, S.cnt, s_warp, [&](int c) { return S.cnt[c]; });
    for (int c = tid; c < GRID_CELLS; c += MF_NT) S.cellStart[c] = (uint16_t)S.cnt[c];
    if (tid == 0) S.cellStart[GRID_CELLS] = (uint16_t)total;
    __syncthreads();
    for (int i = tid; i < K; i += MF_NT) {
        const int px = (int)roundf(fmul(fsub(S.kx[i], minX), gridWInv));
        const int py = (int)roundf(fmul(fsub(S.ky[i], minY), gridHInv));
        if (px >= 0 && px < GRID_COLS && py >= 0 && py < GRID_ROWS) S.cellIdx[atomicAdd(&S.cnt[px * GRID_ROWS + py], 1)] = (uint16_t)i;
    }
    __syncthreads();
    for (int c = tid; c < GRID_CELLS; c += MF_NT) {    // restore insertion order inside each cell (lists are short)
        const int a = S.cellStart[c], b = S.cnt[c];     // cnt now holds the end offset
        for (int i = a + 1; i < b; ++i) {
            const uint16_t v = S.cellIdx[i];
            int j = i - 1;
            while (j >= a && S.cellIdx[j] > v) { S.cellIdx[j + 1] = S.cellIdx[j]; --j; }
            S.cellIdx[j + 1] = v;
        }
    }
    __syncthreads();
}

// Phase stamps of match_frame_kernel (build with -DMF_PHASES, read by tools/match_phases.py through orbm_match_phases): thread 0 of
// every CTA adds the clock64() spans between the kernel's barriers.  [0] grid build, [1] pass 1 (to the cluster barrier), both summed
// over all CTAs; [2] pass 2, [3] outcome / histogram, summed over the CTAs 0; [4] pass-2 sweeps, [5] map points queued for a rescan,
// [6] CTAs, [7] frames.
#ifdef MF_PHASES
__device__ unsigned long long mf_phase[8];
#define MF_STAMP(t) long long t = 0; if (tid == 0) t = clock64()
#define MF_ADD(k, v) if (tid == 0) atomicAdd(&mf_phase[k], (unsigned long long)(v))
#else
#define MF_STAMP(t)
#define MF_ADD(k, v)
#endif

// 64 registers: two 512-thread CTAs per SM when the frame's shared memory allows it (frame_smem_bytes <= 100 KB).
__global__ void __launch_bounds__(MF_NT, 2) match_frame_kernel(MatchParams P) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ int s_warp[33];
    __shared__ int s_changed, s_nq, s_nAcc, s_nRemoved, s_ind[3];
    cg::cluster_group cluster = cg::this_cluster();
    const int C = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
    const int f = blockIdx.x / C, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (P.active && !P.active[f]) return;          // the whole cluster of an inactive stream leaves before its first cluster barrier
    MF_STAMP(t0);
    const int K = min(P.nK[f], P.kcap), M = min(P.nM[f], P.mcap);
    const FrameSmem S = carve_frame_smem(smem_raw, P.ks, P.ms, P.descInSmem != 0);
    const OrbKeyPoint* kps = P.kps + (size_t)f * P.kcap;
    int* match = P.match + (size_t)f * P.kcap;
    uint8_t* claimed = P.claimed + (size_t)f * P.kcap;
    const bool reset = P.resetState != 0;

    // ---- the frame in shared memory: grid, positions, octaves, descriptors; claims at entry ----
    for (int w = tid; w < (P.ks + 31) / 32; w += MF_NT) S.initBits[w] = 0;
    build_frame_smem(S, kps, P.desc + (size_t)f * P.kcap * 32, K, P.minX, P.minY, P.gridWInv, P.gridHInv, s_warp);
    if (!reset) {
        for (int i = tid; i < K; i += MF_NT)
            if (match[i] >= 0 && claimed[i]) atomicOr(&S.initBits[i >> 5], 1u << (i & 31));
        __syncthreads();
    }
    MF_STAMP(t1);

    // ---- pass 1: this CTA's share of the map points, warp per map point ----
    // The warp's map points are i = first + j * stride.  They are taken 32 at a time: lane j makes the query of the j-th point and
    // prefetches its descriptor into L1, so the dependent loads of make_query (valid, then pose / position / octave) are in flight
    // for 32 points at once; the warp then scans the points in order with the query broadcast from lane j.  Holding the descriptors
    // in registers instead measured no faster and spills at the 64-register bound.
    auto notInit = [&](int idx) { return !((S.initBits[idx >> 5] >> (idx & 31)) & 1u); };
    const int stride = C * (MF_NT / 32);
    for (int first = rank * (MF_NT / 32) + wid; first < M; first += 32 * stride) {
        const int il = first + lane * stride;
        float qu = 0, qv = 0, qr = 0; int minL = 0, maxL = 0;
        bool qok = false;
        if (il < M) {
            const size_t o = (size_t)f * P.mcap + il;
            qok = make_query(P, f, il, qu, qv, qr, minL, maxL);
            if (qok) asm volatile("prefetch.global.L1 [%0];" :: "l"(P.mpDesc + o * 32));
            P.query[o] = make_float4(qu, qv, qr, __int_as_float((minL + 1) | ((maxL + 1) << 8) | ((qok ? 1 : 0) << 16)));
        }
        const unsigned okMask = __ballot_sync(0xffffffffu, qok);
        const int levels = (minL + 1) | ((maxL + 1) << 8);
        const int n = min(32, (M - first + stride - 1) / stride);
        for (int j = 0; j < n; ++j) {
            const size_t o = (size_t)f * P.mcap + first + j * stride;
            int4 ri = make_int4(-1, -1, -1, -1), rd = make_int4(256, 256, 256, 256);
            if ((okMask >> j) & 1u) {
                const float u = __shfl_sync(0xffffffffu, qu, j), v = __shfl_sync(0xffffffffu, qv, j), r = __shfl_sync(0xffffffffu, qr, j);
                const int lv = __shfl_sync(0xffffffffu, levels, j);
                uint32_t mpd[8];
                load_mp_desc(P, f, first + j * stride, mpd);
                const TopK<4> t = scan_candidates<4>(P, S, f, u, v, r, (lv & 0xff) - 1, (lv >> 8) - 1, mpd, notInit);
                ri = make_int4(t.i[0], t.i[1], t.i[2], t.i[3]);
                rd = make_int4(t.i[0] >= 0 ? (int)(t.k[0] >> 40) : 256, t.i[1] >= 0 ? (int)(t.k[1] >> 40) : 256,
                               t.i[2] >= 0 ? (int)(t.k[2] >> 40) : 256, t.i[3] >= 0 ? (int)(t.k[3] >> 40) : 256);
            }
            if (lane == 0) { P.resultIdx[o] = ri; P.resultDist[o] = rd; }
        }
    }
    if (C > 1) { __threadfence(); cluster.sync(); }     // the lists of all CTAs are visible to CTA 0
    else __syncthreads();
    MF_STAMP(t2);
    MF_ADD(0, t1 - t0); MF_ADD(1, t2 - t1); MF_ADD(6, 1);
    if (rank != 0) return;

    // ---- pass 2 (CTA 0): fixed-point resolution of the sequential claim rule ----
    const int4* RI = P.resultIdx + (size_t)f * P.mcap;
    const int4* RD = P.resultDist + (size_t)f * P.mcap;
    for (int i = tid; i < M; i += MF_NT) { S.choice[i] = (uint16_t)NONE16; S.mflags[i] = P.hasObs[(size_t)f * P.mcap + i] ? 1 : 0; }
    for (int c = tid; c < K; c += MF_NT) S.minClaimer[c] = 0x7fffffff;
    if (tid == 0) { s_changed = 0; s_nq = 0; }
    __syncthreads();
    // decision of map point i from (best, second) among the usable candidates
    auto decide = [&](int bIdx, int bDist, int sIdx, int sDist) -> unsigned {
        if (bIdx < 0 || bDist > TH_HIGH) return NONE16;
        if (P.mode == 0) {   // ratio test only when best and second come from the same level (:123-128)
            const int lv1 = S.koct[bIdx], lv2 = sIdx >= 0 ? (int)S.koct[sIdx] : -1;
            if (lv1 == lv2 && (float)bDist > fmul(P.nnratio, (float)sDist)) return NONE16;
        }
        return (unsigned)bIdx;
    };
    const bool need2 = P.mode == 0;
    for (int sweep = 0; sweep <= M; ++sweep) {
        // A. thread per map point: walk the four candidates against the claims of lower-index map points
        for (int i = tid; i < M; i += MF_NT) {
            const int4 ri = RI[i];
            unsigned ch = NONE16;
            if (ri.x >= 0) {
                const int4 rd = RD[i];
                const int ids[4] = {ri.x, ri.y, ri.z, ri.w};
                const int ds[4] = {rd.x, rd.y, rd.z, rd.w};
                int bIdx = -1, bDist = 256, sIdx = -1, sDist = 256;
                bool exhausted = false;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    if (ids[c] < 0) { exhausted = true; continue; }
                    if (S.minClaimer[ids[c]] < i) continue;
                    if (bIdx < 0) { bIdx = ids[c]; bDist = ds[c]; }
                    else if (sIdx < 0) { sIdx = ids[c]; sDist = ds[c]; }
                }
                if (!exhausted && (bIdx < 0 || (need2 && sIdx < 0))) {
                    S.queue[atomicAdd(&s_nq, 1)] = (uint16_t)i;            // decided in phase B
                    continue;
                }
                ch = decide(bIdx, bDist, sIdx, sDist);
            }
            if (ch != S.choice[i]) { S.choice[i] = (uint16_t)ch; s_changed = 1; }
        }
        __syncthreads();
        // B. warp per queued map point: exact rescan against the current claims
        const int nq = s_nq;
        MF_ADD(4, 1); MF_ADD(5, nq);
        for (int q = wid; q < nq; q += MF_NT / 32) {
            const int i = S.queue[q];
            const float4 qq = P.query[(size_t)f * P.mcap + i];
            const int bits = __float_as_int(qq.w);
            uint32_t mpd[8];
            load_mp_desc(P, f, i, mpd);
            const Top2 t = scan_candidates<2>(P, S, f, qq.x, qq.y, qq.z, (bits & 0xff) - 1, ((bits >> 8) & 0xff) - 1, mpd,
                                              [&](int idx) { return notInit(idx) && !(S.minClaimer[idx] < i); });
            const unsigned ch = decide(t.i[0], t.i[0] >= 0 ? (int)(t.k[0] >> 40) : 256, t.i[1], t.i[1] >= 0 ? (int)(t.k[1] >> 40) : 256);
            if (lane == 0 && ch != S.choice[i]) { S.choice[i] = (uint16_t)ch; s_changed = 1; }
        }
        __syncthreads();
        const int changed = s_changed;
        __syncthreads();
        if (!changed) break;
        // C. claims of this sweep's choices
        for (int c = tid; c < K; c += MF_NT) S.minClaimer[c] = 0x7fffffff;
        if (tid == 0) { s_changed = 0; s_nq = 0; }
        __syncthreads();
        for (int i = tid; i < M; i += MF_NT) {
            const unsigned ch = S.choice[i];
            if (ch != NONE16 && (S.mflags[i] & 1)) atomicMin(&S.minClaimer[ch], i);
        }
        __syncthreads();
    }
    MF_STAMP(t3);
    MF_ADD(2, t3 - t2); MF_ADD(7, 1);

    // ---- outcome: nmatches++ per accepted map point (:1762-1776), rotation histogram, ComputeThreeMaxima (:2012-2053) ----
    const bool hist = P.mode == 1 && P.checkOri;
    int* s_hist = S.cnt;                      // [HISTO_LENGTH]
    int* lastWriter = S.minClaimer;           // [K] highest-index accepted map point that chose the keypoint
    uint32_t* removedBits = S.initBits;       // [K bits] keypoints cleared by the rotation filter
    if (tid < HISTO_LENGTH) s_hist[tid] = 0;
    if (tid == 0) { s_nAcc = 0; s_nRemoved = 0; }
    for (int c = tid; c < K; c += MF_NT) lastWriter[c] = -1;
    for (int w = tid; w < (K + 31) / 32; w += MF_NT) removedBits[w] = 0;
    __syncthreads();
    int nAcc = 0;
    for (int i = tid; i < M; i += MF_NT) {
        const unsigned ch = S.choice[i];
        if (ch == NONE16) continue;
        ++nAcc;
        atomicMax(&lastWriter[ch], i);
        if (hist) {
            const int b = rot_bin(P.angle[(size_t)f * P.mcap + i], kps[ch].angle);
            S.mflags[i] = (uint8_t)((S.mflags[i] & 1) | ((b + 1) << 2));
            atomicAdd(&s_hist[b], 1);
        }
    }
    if (nAcc) atomicAdd(&s_nAcc, nAcc);
    __syncthreads();
    if (hist) {
        if (tid == 0) three_maxima(s_hist, s_ind);
        __syncthreads();
        int removed = 0;
        for (int i = tid; i < M; i += MF_NT) {      // every event of a rejected bin clears its keypoint (:1868-1884)
            const unsigned ch = S.choice[i];
            if (ch == NONE16) continue;
            const int b = (S.mflags[i] >> 2) - 1;
            if (!rot_kept(b, s_ind)) { atomicOr(&removedBits[ch >> 5], 1u << (ch & 31)); ++removed; }
        }
        if (removed) atomicAdd(&s_nRemoved, removed);
        __syncthreads();
    }
    for (int c = tid; c < K; c += MF_NT) {
        const int w = lastWriter[c];
        if ((removedBits[c >> 5] >> (c & 31)) & 1u) { match[c] = -1; claimed[c] = 0; }
        else if (w >= 0) { match[c] = w; claimed[c] = S.mflags[w] & 1; }
        else if (reset) { match[c] = -1; claimed[c] = 0; }
    }
    if (reset) for (int c = K + tid; c < P.kcap; c += MF_NT) { match[c] = -1; claimed[c] = 0; }
    if (tid == 0) P.nmatches[f] = s_nAcc - s_nRemoved;
    MF_STAMP(t4);
    MF_ADD(3, t4 - t3);
}

// ---------------------------------------------------------------------------------------------
// ORBmatcher::SearchForInitialization (src/ORBmatcher.cc:648-763): windowed brute force between the two frames of the monocular
// initialiser.  Same cluster layout as match_frame_kernel with F2 as the frame in shared memory:
//   pass 1 (all CTAs, warp per level-0 keypoint of F1): the four smallest (distance, enumeration order) keys among the level-0
//           keypoints of F2 inside the window around vbPrevMatched[i1];
//   pass 2 (one warp of CTA 0, F1 keypoints in index order -- the vMatchedDistance / vnMatches21 overwrite rule is order dependent):
//           best and second-best among the candidates i2 whose current match is worse (vMatchedDistance[i2] > dist, :686), TH_LOW,
//           ratio test, re-assignment of an already matched F2 keypoint (:706-714); a keypoint whose four candidates do not
//           settle it is rescanned against the live vMatchedDistance;
//   then the rotation histogram on F1 indices (:716-726, :733-754) and the vbPrevMatched update (:757-759).
// MatchParams reuse: kps/desc/nK = F2, mpDesc/nM = descriptors / count of F1, projX/projY = vbPrevMatched (in), level = F1 octaves,
// angle = F1 angles, th = windowSize, nnratio; outputs: match = vnMatches12 [K1], query = updated vbPrevMatched (xy), nmatches.
// ---------------------------------------------------------------------------------------------
constexpr int TH_LOW = 50;         // src/ORBmatcher.cc:36
__global__ void __launch_bounds__(MF_NT) init_match_kernel(MatchParams P) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ int s_warp[33];
    __shared__ int s_hist[HISTO_LENGTH], s_ind[3], s_nm;
    cg::cluster_group cluster = cg::this_cluster();
    const int C = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int K2 = min(P.nK[0], P.kcap), K1 = min(P.nM[0], P.mcap);
    const FrameSmem S = carve_frame_smem(smem_raw, P.ks, P.ms, P.descInSmem != 0);
    uint16_t* m21 = reinterpret_cast<uint16_t*>(smem_raw + frame_smem_bytes(P.ks, P.ms, P.descInSmem != 0));   // vnMatches21 [K2]
    int* matchedDist = S.minClaimer;                                                                             // vMatchedDistance [K2]
    build_frame_smem(S, P.kps, P.desc, K2, P.minX, P.minY, P.gridWInv, P.gridHInv, s_warp);
    auto anyIdx = [](int) { return true; };
    // ---- pass 1 ----
    for (int i = rank * (MF_NT / 32) + wid; i < K1; i += C * (MF_NT / 32)) {
        int4 ri = make_int4(-1, -1, -1, -1), rd = make_int4(256, 256, 256, 256);
        const int level1 = P.level[i];
        if (!(level1 > 0)) {                                        // :663-665
            uint32_t mpd[8];
            load_mp_desc(P, 0, i, mpd);
            const TopK<4> t = scan_candidates<4>(P, S, 0, P.projX[i], P.projY[i], P.th, level1, level1, mpd, anyIdx);
            ri = make_int4(t.i[0], t.i[1], t.i[2], t.i[3]);
            rd = make_int4(t.i[0] >= 0 ? (int)(t.k[0] >> 40) : 256, t.i[1] >= 0 ? (int)(t.k[1] >> 40) : 256,
                           t.i[2] >= 0 ? (int)(t.k[2] >> 40) : 256, t.i[3] >= 0 ? (int)(t.k[3] >> 40) : 256);
        }
        if (lane == 0) { P.resultIdx[i] = ri; P.resultDist[i] = rd; }
    }
    if (C > 1) { __threadfence(); cluster.sync(); }
    else __syncthreads();
    if (rank != 0) return;
    // ---- pass 2 ----
    for (int c = tid; c < K2; c += MF_NT) { matchedDist[c] = 0x7fffffff; m21[c] = (uint16_t)NONE16; }
    for (int i = tid; i < K1; i += MF_NT) { S.choice[i] = (uint16_t)NONE16; S.mflags[i] = 0; }
    if (tid < HISTO_LENGTH) s_hist[tid] = 0;
    if (tid == 0) s_nm = 0;
    __syncthreads();
    if (wid == 0) {
        for (int base = 0; base < K1; base += 32) {
            const int i = base + lane;
            int4 ri = make_int4(-1, -1, -1, -1), rd = make_int4(256, 256, 256, 256);
            if (i < K1) { ri = P.resultIdx[i]; rd = P.resultDist[i]; }
            const int cnt = min(32, K1 - base);
            for (int j = 0; j < cnt; ++j) {
                const int c0 = __shfl_sync(0xffffffffu, ri.x, j);
                if (c0 < 0) continue;                                 // level > 0 or no candidate (:671-672)
                const int ids[4] = {c0, __shfl_sync(0xffffffffu, ri.y, j), __shfl_sync(0xffffffffu, ri.z, j), __shfl_sync(0xffffffffu, ri.w, j)};
                const int ds[4] = {__shfl_sync(0xffffffffu, rd.x, j), __shfl_sync(0xffffffffu, rd.y, j), __shfl_sync(0xffffffffu, rd.z, j),
                                   __shfl_sync(0xffffffffu, rd.w, j)};
                const int i1 = base + j;
                int bIdx = -1, bDist = 0x7fffffff, sDist = 0x7fffffff, found = 0;
                bool exhausted = false;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    if (ids[c] < 0) { exhausted = true; continue; }
                    if (matchedDist[ids[c]] <= ds[c]) continue;       // :686-687
                    if (found == 0) { bIdx = ids[c]; bDist = ds[c]; }
                    else if (found == 1) sDist = ds[c];
                    ++found;
                }
                if (!exhausted && found < 2) {                        // the four do not settle best and second: exact rescan
                    uint32_t mpd[8];
                    load_mp_desc(P, 0, i1, mpd);
                    const int level1 = P.level[i1];
                    const Top2 t = scan_candidates<2>(P, S, 0, P.projX[i1], P.projY[i1], P.th, level1, level1, mpd, anyIdx,
                                                      [&](int idx, int dist) { return !(matchedDist[idx] <= dist); });
                    bIdx = t.i[0]; bDist = t.i[0] >= 0 ? (int)(t.k[0] >> 40) : 0x7fffffff;
                    sDist = t.i[1] >= 0 ? (int)(t.k[1] >> 40) : 0x7fffffff;
                }
                if (bIdx < 0 || bDist > TH_LOW) continue;             // :702
                if (!((float)bDist < fmul((float)sDist, P.nnratio))) continue;    // :704
                __syncwarp();                                         // every lane has read matchedDist[] for this keypoint before lane 0 updates it
                if (lane == 0) {
                    const unsigned prev = m21[bIdx];
                    if (prev != NONE16) S.choice[prev] = (uint16_t)NONE16;        // :706-710
                    S.choice[i1] = (uint16_t)bIdx; m21[bIdx] = (uint16_t)i1; matchedDist[bIdx] = bDist;
                    if (P.checkOri) {                                             // :716-726
                        const int b = rot_bin(P.angle[i1], P.kps[bIdx].angle);
                        S.mflags[i1] = (uint8_t)(b + 1);
                        s_hist[b]++;
                    }
                }
                __syncwarp();
            }
        }
    }
    __syncthreads();
    if (P.checkOri && tid == 0) three_maxima(s_hist, s_ind);
    __syncthreads();
    int n = 0;
    for (int i = tid; i < K1; i += MF_NT) {
        unsigned ch = S.choice[i];
        if (ch != NONE16 && P.checkOri) {                             // :733-754: events of rejected bins lose their match if they still hold one
            if (!rot_kept((int)S.mflags[i] - 1, s_ind)) ch = NONE16;
        }
        P.match[i] = ch == NONE16 ? -1 : (int)ch;
        float px = P.projX[i], py = P.projY[i];
        if (ch != NONE16) { ++n; px = S.kx[ch]; py = S.ky[ch]; }      // :757-759
        P.query[i] = make_float4(px, py, 0.f, 0.f);
    }
    if (n) atomicAdd(&s_nm, n);
    __syncthreads();
    if (tid == 0) P.nmatches[0] = s_nm;
}

// ---------------------------------------------------------------------------------------------
// ORBmatcher::SearchByBoW(KeyFrame*, Frame&, vector<MapPoint*>&) (src/ORBmatcher.cc:223-425, monocular branch; Tracking::TrackReferenceKeyFrame
// src/Tracking.cc:2730 and relocalisation).  Features are matched only inside the same vocabulary node, so nodes are independent: one warp per
// keyframe node walks its features in order (the claim rule "a frame feature that already holds a match is skipped" is sequential inside a
// node only), lanes over the frame features of that node: top-2 by (distance, position).  The rotation histogram is resolved by the CTA.
// One CTA per (keyframe, frame) pair: CTA f reads its operands at f times the strides (the single-pair entry points are the batch of one).
// ---------------------------------------------------------------------------------------------
struct BowMatchParams {
    const int *nKF, *nF, *eKF, *eF;               // [grid]: features and FeatureVector entries of each keyframe / frame
    int kfStride, fStride;                        // per-CTA stride of the keyframe-side / frame-side operands
    const OrbKeyPoint *kpsKF, *kpsF; const uint8_t *descKF, *descF, *kfPoint;
    const int *fvNodeKF, *fvFeatKF, *fvNodeF, *fvFeatF;
    float nnratio; int checkOri;
    int* match; int* nmatches; int* groupStart; uint8_t* evBin;   // match [fStride], nmatches [1]; scratch: groupStart [kfStride + 1], evBin [fStride]
    // SearchByBoW(KeyFrame*, KeyFrame*) (src/ORBmatcher.cc:765-905): the second side is a keyframe too -- its features need a good map point
    // (fPoint, null for a Frame), the distance test is strict (bestDist1 < TH_LOW, :859) and the result is indexed by the first side (match12)
    const uint8_t* fPoint; int strictLow; int* match12;
    // the batched TrackReferenceKeyFrame (orbm_track_reference_keyframe_batch*): streams not in `active` are skipped (null: all);
    // poseActive[f] = the stream is active and nmatches >= gate, nmatchesCopy[f] = nmatches (both null elsewhere)
    const uint8_t* active; uint8_t* poseActive; int* nmatchesCopy; int gate;
    // orbm_common_regions_bow_batch: CTA f matches the table entries pairEntry[f] = (keyframe side, frame side), whose operands start at
    // entryBase[entry] and whose counts nKF / nF / eKF / eF are indexed by entry; the outputs and scratch stay at f times the strides.
    // Null elsewhere: the operands and counts are CTA f's own.
    const int2* pairEntry; const int* entryBase;
};
constexpr int BM_NT = 256;
__global__ void __launch_bounds__(BM_NT) bow_match_kernel(BowMatchParams Q) {
    __shared__ int s_hist[HISTO_LENGTH], s_ind[3], s_acc, s_rem, s_ng;
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (Q.active && !Q.active[f]) { if (tid == 0 && Q.poseActive) Q.poseActive[f] = 0; return; }
    const size_t kb = (size_t)f * Q.kfStride, fb = (size_t)f * Q.fStride;
    int cKF = f, cF = f;
    size_t kIn = kb, fIn = fb;
    if (Q.pairEntry) { const int2 pe = Q.pairEntry[f]; cKF = pe.x; cF = pe.y; kIn = (size_t)Q.entryBase[cKF]; fIn = (size_t)Q.entryBase[cF]; }
    const int nKF = min(Q.nKF[cKF], Q.kfStride), nF = min(Q.nF[cF], Q.fStride), eKF = min(Q.eKF[cKF], nKF), eF = min(Q.eF[cF], nF);
    const OrbKeyPoint *kpsKF = Q.kpsKF + kIn, *kpsF = Q.kpsF + fIn;
    const uint8_t *descKF = Q.descKF + 32 * kIn, *descF = Q.descF + 32 * fIn, *kfPoint = Q.kfPoint + kIn, *fPoint = Q.fPoint ? Q.fPoint + fIn : nullptr;
    const int *fvNodeKF = Q.fvNodeKF + kIn, *fvFeatKF = Q.fvFeatKF + kIn, *fvNodeF = Q.fvNodeF + fIn, *fvFeatF = Q.fvFeatF + fIn;
    int *match = Q.match + fb, *match12 = Q.match12 ? Q.match12 + kb : nullptr, *groupStart = Q.groupStart + (size_t)f * (Q.kfStride + 1);
    uint8_t* evBin = Q.evBin + fb;
    for (int i = tid; i < Q.fStride; i += BM_NT) { match[i] = -1; evBin[i] = 0; }
    if (match12) for (int i = tid; i < nKF; i += BM_NT) match12[i] = -1;
    if (tid < HISTO_LENGTH) s_hist[tid] = 0;
    if (tid == 0) { s_acc = 0; s_rem = 0; s_ng = 0; }
    __syncthreads();
    // group heads of the keyframe's feature vector (entries are sorted by node id)
    for (int e = tid; e < eKF; e += BM_NT)
        if (e == 0 || fvNodeKF[e] != fvNodeKF[e - 1]) groupStart[atomicAdd(&s_ng, 1)] = e;     // order of groups is irrelevant: nodes are independent
    __syncthreads();
    const int ng = s_ng;
    int acc = 0;
    for (int g = wid; g < ng; g += BM_NT / 32) {
        const int a = groupStart[g];
        const int node = fvNodeKF[a];
        int a1 = a;
        while (a1 < eKF && fvNodeKF[a1] == node) ++a1;
        const int b = lower_bound(fvNodeF, 0, eF, node), b1 = upper_bound(fvNodeF, b, eF, node);   // `node` in the frame's vector
        if (b1 == b) continue;
        for (int iKF = a; iKF < a1; ++iKF) {
            const int realIdxKF = fvFeatKF[iKF];
            if (kfPoint[realIdxKF] != 1) continue;               // no map point, or a bad one (:255-259)
            uint32_t dk[8];
            load_desc(descKF + (size_t)realIdxKF * 32, dk);
            Top2 t; t.init();
            for (int iF = b + lane; iF < b1; iF += 32) {
                const int realIdxF = fvFeatF[iF];
                if (match[realIdxF] >= 0) continue;              // already matched by an earlier keyframe feature of this node (:275-276)
                if (fPoint && fPoint[realIdxF] != 1) continue;
                uint32_t dfw[8];
                load_desc(descF + (size_t)realIdxF * 32, dfw);
                t.insert(((unsigned long long)hamming256(dk, dfw) << 32) | (unsigned)(iF - b), realIdxF);
            }
            t.warp_merge();
            const int bestDist1 = t.i[0] >= 0 ? (int)(t.k[0] >> 32) : 256, bestDist2 = t.i[1] >= 0 ? (int)(t.k[1] >> 32) : 256;
            if ((Q.strictLow ? bestDist1 < TH_LOW : bestDist1 <= TH_LOW) && (float)bestDist1 < fmul(Q.nnratio, (float)bestDist2)) {
                if (lane == 0) {
                    match[t.i[0]] = realIdxKF;
                    if (match12) match12[realIdxKF] = t.i[0];
                    if (Q.checkOri) rot_event(s_hist, evBin, t.i[0], kpsKF[realIdxKF].angle, kpsF[t.i[0]].angle);
                }
                ++acc;
            }
            __syncwarp();
        }
    }
    if (lane == 0 && acc) atomicAdd(&s_acc, acc);
    __syncthreads();
    if (Q.checkOri) {
        if (tid == 0) three_maxima(s_hist, s_ind);
        __syncthreads();
        int rem = 0;
        for (int i = tid; i < nF; i += BM_NT) {
            const int bb = (int)evBin[i] - 1;
            if (bb >= 0 && !rot_kept(bb, s_ind)) { if (match12) match12[match[i]] = -1; match[i] = -1; ++rem; }
        }
        if (rem) atomicAdd(&s_rem, rem);
        __syncthreads();
    }
    if (tid == 0) {
        const int n = s_acc - s_rem;
        Q.nmatches[f] = n;
        if (Q.nmatchesCopy) Q.nmatchesCopy[f] = n;
        if (Q.poseActive) Q.poseActive[f] = n >= Q.gate ? 1 : 0;
    }
}

// ---------------------------------------------------------------------------------------------
// The merge of LoopClosing::DetectCommonRegionsFromBoW (step 5 of orbm_common_regions_bow_batch): one CTA per RAN candidate over the
// matches of its sweep pairs.  Pair t of the candidate holds vpCovKFi[j] with j ascending in t, so the sequential walk "j, k ascending,
// insert a point not yet in spMatchedMPi" keeps match (t, k) of point p iff t * N0 + k is the least position of p among the candidate's
// matches.  Pass 1 takes that minimum per point with atomicMin into an open-addressing hash (capacity a power of two >= twice the match
// bound, so every probe ends); pass 2 counts the kept matches and gives slot k the largest t among them (the last write of the walk);
// pass 3 resolves slot k's pair into (j, point).  Nothing depends on thread order.
// ---------------------------------------------------------------------------------------------
struct CrMergeItem {
    int pairBegin, nPairs, N0, hashCap;
    const uint8_t* pointBad;                 // the query's point table
    int *matchedCov, *matchedPoint, *numBoW; // outputs [N0], [N0], [1]
    int *hashKey, *hashPos;                  // scratch [hashCap]
};
struct CrMergeParams {
    const CrMergeItem* items;
    const int* match12; int kfStride;        // the sweep's result: pair f's match12 at f * kfStride
    const int2* pairEntry; const int* entryBase; const int* slotPoint; const int* pairJ;
};
constexpr int CRM_NT = 256;
__device__ __forceinline__ unsigned cr_hash(int p) { unsigned x = (unsigned)p * 0x9E3779B1u; return x ^ (x >> 15); }
__global__ void __launch_bounds__(CRM_NT) common_regions_merge_kernel(CrMergeParams P) {
    __shared__ int s_n;
    const CrMergeItem& C = P.items[blockIdx.x];
    const int tid = threadIdx.x, N0 = C.N0, total = C.nPairs * N0;
    const unsigned mask = (unsigned)C.hashCap - 1u;
    // the good point pair t brings to current-keyframe feature k, or -1
    auto pointAt = [&](int t, int k) -> int {
        const int f = C.pairBegin + t;
        const int i2 = P.match12[(size_t)f * P.kfStride + k];
        if (i2 < 0) return -1;
        const int p = P.slotPoint[P.entryBase[P.pairEntry[f].y] + i2];
        return (p < 0 || C.pointBad[p]) ? -1 : p;
    };
    for (int i = tid; i < C.hashCap; i += CRM_NT) { C.hashKey[i] = -1; C.hashPos[i] = 0x7fffffff; }
    for (int k = tid; k < N0; k += CRM_NT) C.matchedCov[k] = -1;
    if (tid == 0) s_n = 0;
    __syncthreads();
    for (int i = tid; i < total; i += CRM_NT) {
        const int p = pointAt(i / N0, i % N0);
        if (p < 0) continue;
        for (unsigned s = cr_hash(p) & mask;; s = (s + 1) & mask) {
            const int prev = atomicCAS(&C.hashKey[s], -1, p);
            if (prev == -1 || prev == p) { atomicMin(&C.hashPos[s], i); break; }
        }
    }
    __syncthreads();
    int n = 0;
    for (int i = tid; i < total; i += CRM_NT) {
        const int p = pointAt(i / N0, i % N0);
        if (p < 0) continue;
        unsigned s = cr_hash(p) & mask;
        while (C.hashKey[s] != p) s = (s + 1) & mask;
        if (C.hashPos[s] != i) continue;
        ++n;
        atomicMax(&C.matchedCov[i % N0], i / N0);
    }
    if (n) atomicAdd(&s_n, n);
    __syncthreads();
    for (int k = tid; k < N0; k += CRM_NT) {
        const int t = C.matchedCov[k];
        C.matchedPoint[k] = t >= 0 ? pointAt(t, k) : -1;
        C.matchedCov[k] = t >= 0 ? P.pairJ[C.pairBegin + t] : -1;
    }
    if (tid == 0) *C.numBoW = s_n;
}

// ---------------------------------------------------------------------------------------------
// ORBmatcher::Fuse(KeyFrame*, vector<MapPoint*>, th) (src/ORBmatcher.cc:1148-1338), the search: the keyframe's grid in shared memory (every CTA
// builds its own copy), one warp per map point: projection with the keyframe pose, KeyFrame::IsInImage, distance and viewing-angle tests,
// MapPoint::PredictScale, then the radius search of KeyFrame::GetFeaturesInArea (src/KeyFrame.cc:704-753) with the level window
// [predicted - 1, predicted] and the chi-square gate e2 * invSigma2 > 5.99; first smallest distance wins.  No search depends on what Fuse does
// with another map point's hit, so the AddObservation / Replace bookkeeping stays with the caller (in map-point order).
// One launch serves a table of independent searches (items: keyframe, pose, points, outputs); item j owns CTAs
// [ctaBegin, ctaBegin + nCta) and each of them builds that item's grid.  Single searches are tables of one.
// ---------------------------------------------------------------------------------------------
struct FuseParams {
    MatchParams P;          // keyframe: kps, desc, bounds, scaleFactors, nlevels, ks, descInSmem
    int K, M;
    const uint8_t *state, *mpDesc;
    const float *xyz, *normal, *minD, *maxD, *invSigma2;
    float Tcw[7], Ow[3], logSF;
    int mode, gate;         // mode 0: world point + pose + normal test (Fuse); 2: point given in the camera frame (SearchBySim3).  gate: chi-square test
    int *bestIdx, *bestDist;
    int ctaBegin, nCta;
};
__global__ void __launch_bounds__(MF_NT) fuse_search_kernel(const FuseParams* __restrict__ items, const int* __restrict__ ctaItem) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ int s_warp[33];
    const FuseParams& Q = items[ctaItem[blockIdx.x]];
    const MatchParams& P = Q.P;
    const int tid = threadIdx.x, lane = tid & 31;
    const FrameSmem S = carve_frame_smem(smem_raw, P.ks, 1, P.descInSmem != 0);
    build_frame_smem(S, P.kps, P.desc, Q.K, P.minX, P.minY, P.gridWInv, P.gridHInv, s_warp);
    const int nw = Q.nCta * (MF_NT / 32);
    for (int i = (blockIdx.x - Q.ctaBegin) * (MF_NT / 32) + (tid >> 5); i < Q.M; i += nw) {
        int bestIdx = -1, bestDist = 256;
        bool go = Q.state[i] == 1;
        float u = 0.f, v = 0.f, r = 0.f; int lvl = 0;
        if (go) {
            const float px = Q.xyz[3 * i], py = Q.xyz[3 * i + 1], pz = Q.xyz[3 * i + 2];
            const float maxRaw = Q.maxD[i];
            const float maxDist = fmul(1.2f, maxRaw), minDist = fmul(0.8f, Q.minD[i]);
            float dist3D;
            if (Q.mode == 0) {
                const float pw[3] = {px, py, pz};
                float xc3[3];
                se3_transform(Q.Tcw, pw, xc3);
                const float xc = xc3[0], yc = xc3[1], zc = xc3[2];
                go = !(zc < 0.0f);
                u = fadd(fdiv(fmul(P.cam[0], xc), zc), P.cam[2]);
                v = fadd(fdiv(fmul(P.cam[1], yc), zc), P.cam[3]);
                go = go && (u >= P.minX && u < P.maxX && v >= P.minY && v < P.maxY);                                 // KeyFrame::IsInImage
                const float ox = fsub(px, Q.Ow[0]), oy = fsub(py, Q.Ow[1]), oz = fsub(pz, Q.Ow[2]);
                dist3D = __fsqrt_rn(fadd(fadd(fmul(ox, ox), fmul(oy, oy)), fmul(oz, oz)));
                go = go && !(dist3D < minDist || dist3D > maxDist);
                const float dot = fadd(fadd(fmul(ox, Q.normal[3 * i]), fmul(oy, Q.normal[3 * i + 1])), fmul(oz, Q.normal[3 * i + 2]));
                go = go && !((double)dot < 0.5 * (double)dist3D);
            } else {                                                   // src/ORBmatcher.cc:1510-1532 (and :1589-1611)
                go = !(pz < 0.0f);
                const float invz = (float)(1.0 / (double)pz);
                u = __fmaf_rn(P.cam[0], fmul(px, invz), P.cam[2]);       // fx*x+cx: one FMA in the reference build, see oracle
                v = __fmaf_rn(P.cam[1], fmul(py, invz), P.cam[3]);
                go = go && (u >= P.minX && u < P.maxX && v >= P.minY && v < P.maxY);
                dist3D = __fsqrt_rn(fadd(fadd(fmul(px, px), fmul(py, py)), fmul(pz, pz)));
                go = go && !(dist3D < minDist || dist3D > maxDist);
            }
            if (go) {
                lvl = (int)ceilf(fdiv(orbx::logf_glibc(fdiv(maxRaw, dist3D)), Q.logSF));
                if (lvl < 0) lvl = 0; else if (lvl >= P.nlevels) lvl = P.nlevels - 1;
                r = fmul(P.th, P.scaleFactors[lvl]);
            }
        }
        if (go) {      // warp-uniform: every lane computed the same query
            uint32_t mpd[8];
            load_desc(Q.mpDesc + (size_t)i * 32, mpd);
            const float* isg = Q.invSigma2;
            const bool gate = Q.gate != 0;
            const TopK<1> t = scan_candidates<1>(P, S, 0, u, v, r, lvl - 1, lvl, mpd, [&](int idx) {
                if (!gate) return true;
                const float ex = fsub(u, S.kx[idx]), ey = fsub(v, S.ky[idx]);
                const float e2 = __fmaf_rn(ex, ex, fmul(ey, ey));                     // one FMA in the reference build, see oracle
                return !((double)fmul(e2, isg[S.koct[idx]]) > 5.99);
            });
            if (t.i[0] >= 0) { bestIdx = t.i[0]; bestDist = (int)(t.k[0] >> 40); }
        }
        if (lane == 0) { Q.bestIdx[i] = bestIdx; Q.bestDist[i] = bestDist; }
    }
}

// ---------------------------------------------------------------------------------------------
// ORBmatcher::SearchForTriangulation(pKF1, pKF2, vMatchedPairs, bOnlyStereo = false, bCoarse) (src/ORBmatcher.cc:907-1146, monocular keyframes;
// LocalMapping::CreateNewMapPoints, src/LocalMapping.cc:340-344) with Pinhole::epipolarConstrain (src/CameraModels/Pinhole.cpp:107-129).
// One CTA per (KF1, KF2) pair, one warp per KF1 feature without a map point: lanes over the KF2 features of the same vocabulary node (binary
// search in KF2's feature vector); a candidate passes with distance <= TH_LOW, no map point, the epipole-distance test and the epipolar test;
// the smallest distance wins, the last candidate on ties (:1008 is strict).  The reference never sets vbMatched2, so KF1 features are
// independent.  The epipole and the fundamental matrix are inputs (Eigen / Sophus expressions in the caller); the scalar float expressions
// are contracted as the reference's build contracts them (oracle/matcher_oracle.cpp: orbo_search_for_triangulation).
// The pairs may belong to several new keyframes (items): each pair names its item, whose KF1 operands sit in the item table.
// ---------------------------------------------------------------------------------------------
struct TriItem {
    int N1, E1, coarse;
    const OrbKeyPoint* kps1; const uint8_t *desc1, *hasMP1; const int *fvNode1, *fvFeat1;
    const float *scaleFactors, *levelSigma2;
};
struct TriPair {
    int item, N2, E2;
    const OrbKeyPoint* kps2; const uint8_t *desc2, *hasMP2; const int *fvNode2, *fvFeat2;
    float ep[2], F12[9];
    int* matches12; int* nmatches; uint8_t* evBin;
};
struct TriParams {
    int checkOri;
    const TriItem* items;
    const TriPair* pairs;
};
constexpr int TM_NT = 256;
__global__ void __launch_bounds__(TM_NT) tri_match_kernel(TriParams P) {
    __shared__ int s_hist[HISTO_LENGTH], s_ind[3], s_acc, s_rem;
    const TriPair& R = P.pairs[blockIdx.x];
    const TriItem& Q = P.items[R.item];
    const int checkOri = P.checkOri;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int i = tid; i < Q.N1; i += TM_NT) { R.matches12[i] = -1; R.evBin[i] = 0; }
    if (tid < HISTO_LENGTH) s_hist[tid] = 0;
    if (tid == 0) { s_acc = 0; s_rem = 0; }
    __syncthreads();
    int acc = 0;
    for (int e1 = wid; e1 < Q.E1; e1 += TM_NT / 32) {
        const int idx1 = Q.fvFeat1[e1];
        if (Q.hasMP1[idx1]) continue;
        const int node = Q.fvNode1[e1];
        const int b = lower_bound(R.fvNode2, 0, R.E2, node), b1 = upper_bound(R.fvNode2, b, R.E2, node);
        if (b1 == b) continue;
        const OrbKeyPoint kp1 = Q.kps1[idx1];
        uint32_t d1[8];
        load_desc(Q.desc1 + (size_t)idx1 * 32, d1);
        // epipolar line of kp1 in the second image, l = x1' F12 = [a b c]
        const float ea = fadd(__fmaf_rn(kp1.x, R.F12[0], fmul(kp1.y, R.F12[3])), R.F12[6]);
        const float eb = fadd(__fmaf_rn(kp1.x, R.F12[1], fmul(kp1.y, R.F12[4])), R.F12[7]);
        const float ec = fadd(__fmaf_rn(kp1.x, R.F12[2], fmul(kp1.y, R.F12[5])), R.F12[8]);
        const float den = __fmaf_rn(ea, ea, fmul(eb, eb));
        unsigned long long best = ~0ull;
        for (int i2 = b + lane; i2 < b1; i2 += 32) {
            const int idx2 = R.fvFeat2[i2];
            if (R.hasMP2[idx2]) continue;
            uint32_t d2[8];
            load_desc(R.desc2 + (size_t)idx2 * 32, d2);
            const int dist = hamming256(d1, d2);
            if (dist > TH_LOW) continue;
            const OrbKeyPoint kp2 = R.kps2[idx2];
            const int oct = min(max(kp2.octave, 0), 255);
            const float distex = fsub(R.ep[0], kp2.x), distey = fsub(R.ep[1], kp2.y);
            if (__fmaf_rn(distex, distex, fmul(distey, distey)) < fmul(100.0f, Q.scaleFactors[oct])) continue;
            if (!Q.coarse) {
                if (den == 0.0f) continue;
                const float num = fadd(__fmaf_rn(ea, kp2.x, fmul(eb, kp2.y)), ec);
                const float dsqr = fdiv(fmul(num, num), den);
                if (!((double)dsqr < 3.84 * (double)Q.levelSigma2[oct])) continue;
            }
            const unsigned long long key = ((unsigned long long)dist << 32) | (0xFFFFFFFFu - (unsigned)(i2 - b));
            best = key < best ? key : best;
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o); best = t < best ? t : best; }
        if (best != ~0ull) {
            if (lane == 0) {
                const int idx2 = R.fvFeat2[b + (int)(0xFFFFFFFFu - (unsigned)best)];
                R.matches12[idx1] = idx2;
                if (checkOri) rot_event(s_hist, R.evBin, idx1, kp1.angle, R.kps2[idx2].angle);
            }
            ++acc;
        }
    }
    if (lane == 0 && acc) atomicAdd(&s_acc, acc);
    __syncthreads();
    if (checkOri) {
        if (tid == 0) three_maxima(s_hist, s_ind);
        __syncthreads();
        int rem = 0;
        for (int i = tid; i < Q.N1; i += TM_NT) {
            const int bb = (int)R.evBin[i] - 1;
            if (bb >= 0 && !rot_kept(bb, s_ind)) { R.matches12[i] = -1; ++rem; }
        }
        if (rem) atomicAdd(&s_rem, rem);
        __syncthreads();
    }
    if (tid == 0) *R.nmatches = s_acc - s_rem;
}

// ---------------------------------------------------------------------------------------------
// LocalMapping::CreateNewMapPoints (src/LocalMapping.cc, the vpNeighKFs loop from :296; monocular keyframes) after the search:
// new_points_kernel checks one (neighbour k, idx1) match per thread -- ray parallax, GeometricTools::Triangulate (Eigen's two-sided
// Jacobi SVD of the 4x4 in registers), depth, reprojection, far points, scale -- and fills the record MapPoint::UpdateNormalAndDepth gives.
// new_points_commit_kernel applies the sequential rule (DESIGN.md section 4): the point of idx1 comes from the first k whose match
// passes, and a match of a later neighbour at that idx1 is one the reference never sees.  Every rounding and contraction is the
// oracle's (oracle/mapping_oracle.cpp), which documents the evaluation order.
// A launch serves several new keyframes (items) of different maps: the pairs of tri_match_kernel, item after item, carry the item; each
// item owns the [nKF2][N1] block of slots from `slot0` in matches12 / reason / recs and its own outputs.
// ---------------------------------------------------------------------------------------------
enum : uint8_t { NP_NO_MATCH = 0, NP_LOW_PARALLAX, NP_SVD_W0, NP_DEPTH1, NP_DEPTH2, NP_REPROJ1, NP_REPROJ2, NP_ZERO_DIST, NP_FAR, NP_SCALE, NP_CREATED };
constexpr int NP_MAX_SWEEPS = 64;       // Eigen has no limit; a float 4x4 converges in a handful of sweeps (oracle)
constexpr int NP_NT = 128, NPC_NT = 1024;

struct NpItem {
    int pair0, nKF2, nlevels, bInertial;                                     // pair0: the item's first pair
    float ratioFactor, thFar;
    size_t slot0;
    const float *Tcw, *Ow, *cam;                                             // [1 + nKF2] keyframes, KF1 first
    int* winner; int* counts; OrbmNewPoint* out;                             // [N1]; nNew, nmatches [nKF2], ncreated [nKF2]; out [N1]
};
struct NewPointsParams {
    const TriItem* tri; const NpItem* items; const TriPair* pairs;
    const int* matches12; uint8_t* reason; OrbmNewPoint* recs;               // every item's slots
};

struct NpRot { float c, s; };
__device__ __forceinline__ float fmaxe(float a, float b) { return a < b ? b : a; }   // std::max
__device__ __forceinline__ NpRot np_make_jacobi(float x, float y, float z) {           // Eigen JacobiRotation::makeJacobi (real)
    const float deno = fmul(2.0f, fabsf(y));
    if (deno < FLT_MIN) return {1.0f, 0.0f};
    const float tau = fdiv(fsub(x, z), deno);
    const float w = __fsqrt_rn(fadd(fmul(tau, tau), 1.0f));
    const float t = tau > 0.0f ? fdiv(1.0f, fadd(tau, w)) : fdiv(1.0f, fsub(tau, w));
    const float sign_t = t > 0.0f ? 1.0f : -1.0f;
    const float n = fdiv(1.0f, __fsqrt_rn(fadd(fmul(t, t), 1.0f)));
    return {n, fmul(fmul(fmul(-sign_t, fdiv(y, fabsf(y))), fabsf(t)), n)};
}
template <int P, int Q> __device__ __forceinline__ void np_rot_rows(float (&W)[4][4], NpRot j) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float x = W[P][i], y = W[Q][i];
        W[P][i] = fadd(fmul(j.c, x), fmul(j.s, y)); W[Q][i] = fadd(fmul(-j.s, x), fmul(j.c, y));
    }
}
template <int P, int Q> __device__ __forceinline__ void np_rot_cols(float (&W)[4][4], NpRot j) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float x = W[i][P], y = W[i][Q];
        W[i][P] = fadd(fmul(j.c, x), fmul(j.s, y)); W[i][Q] = fadd(fmul(-j.s, x), fmul(j.c, y));
    }
}
// One pair (p, q) of a Jacobi sweep (JacobiSVD::compute + real_2x2_jacobi_svd).
template <int P, int Q> __device__ __forceinline__ void np_jacobi_pair(float (&W)[4][4], float (&V)[4][4], float& maxDiag, bool& finished) {
    const float threshold = fmaxe(FLT_MIN, fmul(2.0f * FLT_EPSILON, maxDiag));
    if (!(fabsf(W[P][Q]) > threshold || fabsf(W[Q][P]) > threshold)) return;
    finished = false;
    const float m00 = W[P][P], m01 = W[P][Q], m10 = W[Q][P], m11 = W[Q][Q];
    NpRot r1;
    const float t = fadd(m00, m11), d = fsub(m10, m01);
    if (fabsf(d) < FLT_MIN) r1 = {1.0f, 0.0f};
    else {
        const float u = fdiv(t, d);
        const float tmp = __fsqrt_rn(fadd(1.0f, fmul(u, u)));
        r1 = {fdiv(u, tmp), fdiv(1.0f, tmp)};
    }
    const float n00 = fadd(fmul(r1.c, m00), fmul(r1.s, m10)), n01 = fadd(fmul(r1.c, m01), fmul(r1.s, m11));
    const float n11 = fadd(fmul(-r1.s, m01), fmul(r1.c, m11));
    const NpRot jr = np_make_jacobi(n00, n01, n11);
    const NpRot jrt = {jr.c, -jr.s};
    const NpRot jl = {fsub(fmul(r1.c, jrt.c), fmul(r1.s, jrt.s)), fadd(fmul(r1.c, jrt.s), fmul(r1.s, jrt.c))};
    np_rot_rows<P, Q>(W, jl);
    np_rot_cols<P, Q>(W, jrt);
    np_rot_cols<P, Q>(V, jrt);
    maxDiag = fmaxe(maxDiag, fmaxe(fabsf(W[P][P]), fabsf(W[Q][Q])));
}
// GeometricTools::Triangulate: false when V(3, 3) of the smallest singular value is 0.
__device__ __forceinline__ bool np_triangulate(float x1, float y1, float x2, float y2, const float* T1, const float* T2, float* x3D) {
    float W[4][4], V[4][4];
    float scale = 0.0f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        W[0][j] = fsub(fmul(x1, T1[8 + j]), T1[j]);
        W[1][j] = fsub(fmul(y1, T1[8 + j]), T1[4 + j]);
        W[2][j] = fsub(fmul(x2, T2[8 + j]), T2[j]);
        W[3][j] = fsub(fmul(y2, T2[8 + j]), T2[4 + j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) scale = fmaxe(scale, fabsf(W[i][j]));
    if (scale == 0.0f) scale = 1.0f;
    float maxDiag = 0.0f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { W[i][j] = fdiv(W[i][j], scale); V[i][j] = i == j ? 1.0f : 0.0f; }
        maxDiag = fmaxe(maxDiag, fabsf(W[i][i]));
    }
    bool finished = false;
    for (int sweep = 0; !finished && sweep < NP_MAX_SWEEPS; ++sweep) {
        finished = true;
        np_jacobi_pair<1, 0>(W, V, maxDiag, finished);
        np_jacobi_pair<2, 0>(W, V, maxDiag, finished);
        np_jacobi_pair<2, 1>(W, V, maxDiag, finished);
        np_jacobi_pair<3, 0>(W, V, maxDiag, finished);
        np_jacobi_pair<3, 1>(W, V, maxDiag, finished);
        np_jacobi_pair<3, 2>(W, V, maxDiag, finished);
    }
    // sort the singular values in decreasing order (first maximum wins); only the permutation of V's columns is kept
    float s[4];
    int perm[4] = {0, 1, 2, 3};
#pragma unroll
    for (int i = 0; i < 4; ++i) s[i] = fabsf(W[i][i]);
    bool stop = false;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int pos = i;
#pragma unroll
        for (int k = i + 1; k < 4; ++k) {
            float sp = s[i];
#pragma unroll
            for (int l = i + 1; l < 4; ++l) if (l == pos) sp = s[l];
            if (s[k] > sp) pos = k;
        }
        float smax = s[i];
#pragma unroll
        for (int l = i + 1; l < 4; ++l) if (l == pos) smax = s[l];
        stop = stop || smax == 0.0f;
        if (!stop) {
#pragma unroll
            for (int l = i + 1; l < 4; ++l)
                if (l == pos) { const float ts = s[i]; s[i] = s[l]; s[l] = ts; const int tp = perm[i]; perm[i] = perm[l]; perm[l] = tp; }
        }
    }
    float v[4] = {V[0][0], V[1][0], V[2][0], V[3][0]};
#pragma unroll
    for (int c = 1; c < 4; ++c)
        if (perm[3] == c) { v[0] = V[0][c]; v[1] = V[1][c]; v[2] = V[2][c]; v[3] = V[3][c]; }
    if (v[3] == 0.0f) return false;
    x3D[0] = fdiv(v[0], v[3]); x3D[1] = fdiv(v[1], v[3]); x3D[2] = fdiv(v[2], v[3]);
    return true;
}

__device__ __forceinline__ float np_row(const float* T, int r, const float* x) {
    return fadd(fadd(fadd(fmul(T[4 * r], x[0]), fmul(T[4 * r + 1], x[1])), fmul(T[4 * r + 2], x[2])), T[4 * r + 3]);
}
__device__ __forceinline__ float np_norm(const float* a) { return __fsqrt_rn(fadd(fadd(fmul(a[0], a[0]), fmul(a[1], a[1])), fmul(a[2], a[2]))); }

// Grid (x: idx1 blocks of the widest item, y: pair); a thread beyond its item's N1 exits.
__global__ void __launch_bounds__(NP_NT) new_points_kernel(NewPointsParams P) {
    const TriPair* R = P.pairs + blockIdx.y;
    const int it = R->item, N1 = P.tri[it].N1, idx1 = blockIdx.x * NP_NT + threadIdx.x;
    if (idx1 >= N1) return;
    const NpItem* I = P.items + it;
    const int k = (int)blockIdx.y - I->pair0;
    const size_t slot = I->slot0 + (size_t)k * N1 + idx1;
    const int idx2 = P.matches12[slot];
    uint8_t why = NP_NO_MATCH;
    if (idx2 >= 0) {
        const float *scaleFactors = P.tri[it].scaleFactors, *levelSigma2 = P.tri[it].levelSigma2;
        const OrbKeyPoint kp1 = P.tri[it].kps1[idx1], kp2 = R->kps2[idx2];
        const float *Tcw = I->Tcw, *Ow = I->Ow, *cam = I->cam;
        float T1[12], T2[12], O1[3], O2[3], c1[4], c2[4];
#pragma unroll
        for (int i = 0; i < 12; ++i) { T1[i] = Tcw[i]; T2[i] = Tcw[12 * (k + 1) + i]; }
#pragma unroll
        for (int i = 0; i < 3; ++i) { O1[i] = Ow[i]; O2[i] = Ow[3 * (k + 1) + i]; }
#pragma unroll
        for (int i = 0; i < 4; ++i) { c1[i] = cam[i]; c2[i] = cam[4 * (k + 1) + i]; }
        const float xn1[3] = {fdiv(fsub(kp1.x, c1[2]), c1[0]), fdiv(fsub(kp1.y, c1[3]), c1[1]), 1.0f};
        const float xn2[3] = {fdiv(fsub(kp2.x, c2[2]), c2[0]), fdiv(fsub(kp2.y, c2[3]), c2[1]), 1.0f};
        float ray1[3], ray2[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            ray1[i] = fadd(fadd(fmul(T1[i], xn1[0]), fmul(T1[4 + i], xn1[1])), fmul(T1[8 + i], xn1[2]));
            ray2[i] = fadd(fadd(fmul(T2[i], xn2[0]), fmul(T2[4 + i], xn2[1])), fmul(T2[8 + i], xn2[2]));
        }
        const float dot = fadd(fadd(fmul(ray1[0], ray2[0]), fmul(ray1[1], ray2[1])), fmul(ray1[2], ray2[2]));
        const float cp = fdiv(dot, fmul(np_norm(ray1), np_norm(ray2)));
        float x3D[3];
        const int bInertial = I->bInertial;
        if (!(cp < fadd(cp, 1.0f) && cp > 0.0f && ((bInertial && (double)cp < 0.9996) || (!bInertial && (double)cp < 0.9998)))) why = NP_LOW_PARALLAX;
        else if (!np_triangulate(xn1[0], xn1[1], xn2[0], xn2[1], T1, T2, x3D)) why = NP_SVD_W0;
        else {
            const float z1 = np_row(T1, 2, x3D), z2 = np_row(T2, 2, x3D);
            const float u1 = fadd(fdiv(fmul(c1[0], np_row(T1, 0, x3D)), z1), c1[2]), v1 = fadd(fdiv(fmul(c1[1], np_row(T1, 1, x3D)), z1), c1[3]);
            const float ex1 = fsub(u1, kp1.x), ey1 = fsub(v1, kp1.y);
            const float u2 = fadd(fdiv(fmul(c2[0], np_row(T2, 0, x3D)), z2), c2[2]), v2 = fadd(fdiv(fmul(c2[1], np_row(T2, 1, x3D)), z2), c2[3]);
            const float ex2 = fsub(u2, kp2.x), ey2 = fsub(v2, kp2.y);
            const float nv1[3] = {fsub(x3D[0], O1[0]), fsub(x3D[1], O1[1]), fsub(x3D[2], O1[2])};
            const float nv2[3] = {fsub(x3D[0], O2[0]), fsub(x3D[1], O2[1]), fsub(x3D[2], O2[2])};
            const float dist1 = np_norm(nv1), dist2 = np_norm(nv2);
            const float sf1 = scaleFactors[kp1.octave], thFar = I->thFar;
            if (z1 <= 0.0f) why = NP_DEPTH1;
            else if (z2 <= 0.0f) why = NP_DEPTH2;
            else if ((double)__fmaf_rn(ex1, ex1, fmul(ey1, ey1)) > 5.991 * (double)levelSigma2[kp1.octave]) why = NP_REPROJ1;   // one FMA, see oracle
            else if ((double)__fmaf_rn(ex2, ex2, fmul(ey2, ey2)) > 5.991 * (double)levelSigma2[kp2.octave]) why = NP_REPROJ2;
            else if (dist1 == 0.0f || dist2 == 0.0f) why = NP_ZERO_DIST;
            else if (thFar > 0.0f && (dist1 >= thFar || dist2 >= thFar)) why = NP_FAR;
            else {
                const float ratioFactor = I->ratioFactor;
                const float ratioDist = fdiv(dist2, dist1), ratioOctave = fdiv(sf1, scaleFactors[kp2.octave]);
                if (fmul(ratioDist, ratioFactor) < ratioOctave || ratioDist > fmul(ratioOctave, ratioFactor)) why = NP_SCALE;
                else {
                    why = NP_CREATED;
                    OrbmNewPoint r;
                    r.kf2 = k; r.idx1 = idx1; r.idx2 = idx2;
#pragma unroll
                    for (int i = 0; i < 3; ++i) { r.x3D[i] = x3D[i]; r.normal[i] = fdiv(fadd(fadd(0.0f, fdiv(nv1[i], dist1)), fdiv(nv2[i], dist2)), 2.0f); }
                    r.maxDistance = fmul(dist1, sf1);
                    r.minDistance = fdiv(r.maxDistance, scaleFactors[I->nlevels - 1]);
                    P.recs[slot] = r;
                }
            }
        }
    }
    P.reason[slot] = why;
}

// One CTA per item: winner[idx1] = first neighbour that created idx1's point; then per neighbour, in order, the counts and the records
// compacted in idx1 order (thread t owns a contiguous run of idx1, a block scan gives each run its place).
__global__ void __launch_bounds__(NPC_NT) new_points_commit_kernel(NewPointsParams P) {
    __shared__ int s_warp[33];
    const NpItem& I = P.items[blockIdx.x];
    const int tid = threadIdx.x, N1 = P.tri[blockIdx.x].N1, K = I.nKF2;
    const int* matches12 = P.matches12 + I.slot0;
    const uint8_t* reason = P.reason + I.slot0;
    const OrbmNewPoint* recs = P.recs + I.slot0;
    int* winner = I.winner;
    for (int i = tid; i < N1; i += NPC_NT) {
        int w = -1;
        for (int k = 0; k < K && w < 0; ++k) if (reason[(size_t)k * N1 + i] == NP_CREATED) w = k;
        winner[i] = w;
    }
    __syncthreads();
    const int per = (N1 + NPC_NT - 1) / NPC_NT, i0 = min(N1, tid * per), i1 = min(N1, i0 + per);
    int base = 0;
    for (int k = 0; k < K; ++k) {
        int c = 0, mt = 0;
        for (int i = i0; i < i1; ++i) {
            const int w = winner[i];
            c += w == k;
            mt += matches12[(size_t)k * N1 + i] >= 0 && (w < 0 || w >= k);     // the reference's search skips idx1 once an earlier k made its point
        }
        int created, matched;
        int pos = base + block_scan_excl<NPC_NT>(c, s_warp, created);
        block_scan_excl<NPC_NT>(mt, s_warp, matched);
        for (int i = i0; i < i1; ++i) if (winner[i] == k) I.out[pos++] = recs[(size_t)k * N1 + i];
        if (tid == 0) { I.counts[1 + k] = matched; I.counts[1 + K + k] = created; }
        base += created;
    }
    if (tid == 0) I.counts[0] = base;
}

// ---------------------------------------------------------------------------------------------
// MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:329-403) for a batch of map points: warp per map point, lane per observation row
// (distinctive_best, device_utils.cuh).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) distinctive_kernel(int nPoints, const int* __restrict__ ptStart, const uint8_t* __restrict__ desc, int* __restrict__ best) {
    const int p = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (p >= nPoints) return;
    const int a = ptStart[p], n = ptStart[p + 1] - a;
    if (n <= 0) { if (lane == 0) best[p] = -1; return; }
    const int b = distinctive_best(n, lane, [&](int j) { return desc + (size_t)(a + j) * 32; });
    if (lane == 0) best[p] = b;
}

// cv::BFMatcher(NORM_HAMMING).knnMatch(k=2): warp per query, lanes over train rows
constexpr int BF_NT = 256;
__global__ void __launch_bounds__(BF_NT) bf_knn2_kernel(const uint8_t* __restrict__ q, int Q, const uint8_t* __restrict__ t, int T,
                                                        int* __restrict__ idx, int* __restrict__ dist) {
    const int qi = blockIdx.x * (BF_NT / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (qi >= Q) return;
    uint32_t qd[8];
    load_desc(q + (size_t)qi * 32, qd);
    Top2 tt; tt.init();
    for (int j = lane; j < T; j += 32) {
        uint32_t td[8];
        load_desc(t + (size_t)j * 32, td);
        tt.insert(((unsigned long long)hamming256(qd, td) << 32) | (unsigned)j, j);
    }
    tt.warp_merge();
    if (lane == 0) {
        idx[2 * qi] = tt.i[0]; idx[2 * qi + 1] = tt.i[1];
        dist[2 * qi] = tt.i[0] >= 0 ? (int)(tt.k[0] >> 32) : -1;
        dist[2 * qi + 1] = tt.i[1] >= 0 ? (int)(tt.k[1] >> 32) : -1;
    }
}

__global__ void hamming_pairs_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int n, int* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint4* pa = reinterpret_cast<const uint4*>(a + (size_t)i * 32);
    const uint4* pb = reinterpret_cast<const uint4*>(b + (size_t)i * 32);
    const uint4 a0 = pa[0], a1 = pa[1], b0 = pb[0], b1 = pb[1];
    const uint32_t x[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    const uint32_t y[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    out[i] = hamming256(x, y);
}

// Frame::AssignFeaturesToGrid's cell scale (src/Frame.cc:342-343) and the shared-memory layout of a frame of P.ks keypoints and P.ms
// map points with `extra` bytes behind it: the descriptors are staged (P.descInSmem) when the whole then takes at most descLimit bytes.
// Returns the dynamic shared memory, or 0 with `tooLarge` as the error when even without the descriptors it exceeds FRAME_SMEM_LIMIT.
static size_t frame_layout(MatchParams& P, size_t extra, size_t descLimit, const char* tooLarge) {
    P.gridWInv = (float)GRID_COLS / (P.maxX - P.minX);
    P.gridHInv = (float)GRID_ROWS / (P.maxY - P.minY);
    P.descInSmem = frame_smem_bytes(P.ks, P.ms, true) + extra <= descLimit ? 1 : 0;
    const size_t sm = frame_smem_bytes(P.ks, P.ms, P.descInSmem != 0) + extra;
    if (sm > FRAME_SMEM_LIMIT) { set_error(tooLarge); return 0; }
    return sm;
}

// The launch of match_frame_kernel / init_match_kernel: one cluster of MF_NT-thread CTAs per frame, `sm` bytes of dynamic shared memory.
struct ClusterLaunch {
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute at[1];
    ClusterLaunch(size_t sm, cudaStream_t st) {
        cfg.blockDim = dim3(MF_NT); cfg.dynamicSmemBytes = sm; cfg.stream = st;
        at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
    }
    ClusterLaunch(const ClusterLaunch&) = delete;
    // clusters of C CTAs for `frames` frames
    const cudaLaunchConfig_t* shape(int frames, int C) { at[0].val.clusterDim.x = C; cfg.gridDim = dim3((unsigned)(frames * C)); return &cfg; }
};

struct Matcher {
    int device, maxBatch, kcap, mcap;
    cudaStream_t stream = nullptr;
    cudaEvent_t evWait = nullptr;      // blocking-sync event of the batch host entry points (device_utils.cuh)
    // scratch
    float4* d_query = nullptr; int4 *d_resultIdx = nullptr, *d_resultDist = nullptr;
    int* d_status = nullptr;
    int numSMs = 132;
    uint8_t* d_track = nullptr;                          // scratch of the batched tracking calls, allocated by their first call (track_scratch)
    orbm::DeviceScratch ulm;                             // scratch of orbm_update_local_map_batch_device, grown by its calls
    Staging staging;                                     // the single-call host entry points' operands
    uint8_t* d_batch = nullptr; size_t batchBytes = 0;   // device staging of search_last_frame_batch_host (copied straight from the caller)
    int launches = 0;
    // the device form of the mono-inertial call: pinned mirror of its route / active tables ([maxBatch] int + [maxBatch] u8) and the event
    // of the copy that last read it (a new call waits for that copy only, never for the caller's stream)
    uint8_t* h_route = nullptr; cudaEvent_t evRoute = nullptr;

    ~Matcher() {
        cudaSetDevice(device);
        void* ptrs[] = {d_query, d_resultIdx, d_resultDist, d_status, d_batch, d_track, ulm.ptr};
        for (void* p : ptrs) if (p) cudaFree(p);
        if (h_route) cudaFreeHost(h_route);
        if (evRoute) cudaEventDestroy(evRoute);
        if (evWait) cudaEventDestroy(evWait);
        if (stream) cudaStreamDestroy(stream);
    }
    int init() {
        CK(cudaSetDevice(device));
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, device));
        if (orbx::require_sm90(prop.major, prop.minor)) return ORB_ERR_CUDA;
        const size_t B = maxBatch;
        numSMs = prop.multiProcessorCount;
        CK(cudaMalloc(&d_query, sizeof(float4) * mcap * B));
        CK(cudaMalloc(&d_resultIdx, sizeof(int4) * mcap * B));
        CK(cudaMalloc(&d_resultDist, sizeof(int4) * mcap * B));
        CK(cudaMalloc(&d_status, sizeof(int) * B));
        staging.device = device;
        batchBytes = B * ((size_t)kcap * (28 + 32 + 4 + 1) + (size_t)mcap * (1 + 12 + 4 + 4 + 1 + 32) + 28 + 16 + 13 * 256) + 4096;
        CK(cudaMalloc(&d_batch, batchBytes));
        CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        CK(orbx::make_blocking_event(&evWait));
        return ORB_OK;
    }
    // kUse / mUse: the largest keypoint / map-point count any frame of this call can have (the slab capacities when the
    // counts live on the device): they size the kernel's shared memory.  A refused call launches nothing and reports 0 launches.
    int run(MatchParams& P, int kUse, int mUse, cudaStream_t st) {
        launches = 0;
        P.query = d_query; P.resultIdx = d_resultIdx; P.resultDist = d_resultDist; P.status = d_status;
        P.ks = std::max(kUse, 1); P.ms = std::max(mUse, 1);
        if (P.ks > 65535 || P.ms > 65535) { set_error("more than 65535 keypoints or map points per frame"); return ORB_ERR_CAPACITY; }
        // the descriptors are staged only when two CTAs per SM still fit
        const size_t sm = frame_layout(P, 0, 100 * 1024, "frame too large for the matcher's shared-memory grid (keypoints + map points)");
        if (!sm) return ORB_ERR_CAPACITY;
        int rc = ensure_dynamic_smem(match_frame_kernel, sm, device);
        if (rc) return rc;
        ClusterLaunch L(sm, st);
        // cluster size: the largest (up to 8) for which every frame's cluster is resident at once (pass 1 is spread over the
        // cluster; a second wave would double the call's time).  Asked from the occupancy calculator, which counts registers, shared
        // memory and the GPCs clusters cannot straddle; the answer depends only on (batch, shared memory), so it is kept.
        if (P.batch != occBatch || sm != occSmem) {
            occC = 1;
            for (int cand = 8; cand > 1; --cand) {
                if ((long)P.batch * cand > 2L * numSMs) continue;
                int nClusters = 0;
                if (cudaOccupancyMaxActiveClusters(&nClusters, match_frame_kernel, L.shape(P.batch, cand)) == cudaSuccess && nClusters >= P.batch) { occC = cand; break; }
            }
            (void)cudaGetLastError();
            occBatch = P.batch; occSmem = sm;
        }
        const int C = occC;
        CK(cudaLaunchKernelEx(L.shape(P.batch, C), match_frame_kernel, P));
        launches = 1;
        lastCluster = C;
        return ORB_OK;
    }
    int lastCluster = 1;
    int occBatch = -1, occC = 1; size_t occSmem = 0;   // run's cluster size for the last (batch, shared memory) it was asked for

    // The batched tracking calls' scratch, sized for max_batch x max_keypoints / max_mappoints: PoseOptimization's gathered edges
    // ([B][kcap]), the frustum stage's per-point fields and flags ([B][mcap]) and the motion-model step's nInliers ([B]).  The
    // mono-inertial call adds its float edges ([B][kcap]: Xw 3, obs 2, trackDepth; it shares is2, err, outl, edgeKp, N and cam4) and
    // per-slot operands ([B]: route, two preintegrations, fixed / current state, prior, prior and optimised H, return value).  The
    // reference-keyframe call adds the search's group heads ([B][mcap + 1]) and histogram events ([B][kcap]), the streams that passed
    // the match gate and the copy of nmatches the discard loop decrements ([B] each).
    struct TrackScratch {
        double *Xw, *obs, *err; float* is2; uint8_t* outl; int* edgeKp;
        uint8_t *seen, *inView; float *projX, *projY, *depth, *viewCos; int *level, *nInliers;
        int* N; double *poseIn, *poseTmp; float* cam4; int* nInlTmp;
        float *iXw, *iObs, *iTd; int* route; uint8_t* active; float *preint, *preintKF2; double *fixedState, *state, *prior, *priorH, *H15; int* ret;
        int* groupStart; uint8_t *evBin, *poseActive; int* nmCopy;
    } ts;
    int track_scratch() {
        if (d_track) return ORB_OK;
        const size_t BK = (size_t)maxBatch * kcap, BM = (size_t)maxBatch * mcap;
        const size_t B = maxBatch, PS = 4 * IMU_PREINT_FLOATS;
        const size_t sizes[] = {24 * BK, 16 * BK, 16 * BK, 4 * BK, BK, 4 * BK, BM, BM, 4 * BM, 4 * BM, 4 * BM, 4 * BM, 4 * BM, 4 * B, 4 * B, 56 * B, 56 * B, 16 * B, 4 * B,
                                12 * BK, 8 * BK, 4 * BK, 4 * B, B, PS * B, PS * B, 168 * B, 168 * B, 168 * B, 1800 * B, 1800 * B, 4 * B,
                                4 * (BM + B), BK, B, 4 * B};
        constexpr int nSlots = sizeof(sizes) / sizeof(sizes[0]);
        size_t total = 0;
        for (size_t b : sizes) total += (b + 255) & ~(size_t)255;
        CK(cudaMalloc(&d_track, total));
        void** slots[nSlots] = {(void**)&ts.Xw, (void**)&ts.obs, (void**)&ts.err, (void**)&ts.is2, (void**)&ts.outl, (void**)&ts.edgeKp, (void**)&ts.seen,
                          (void**)&ts.inView, (void**)&ts.projX, (void**)&ts.projY, (void**)&ts.depth, (void**)&ts.viewCos, (void**)&ts.level,
                          (void**)&ts.nInliers, (void**)&ts.N, (void**)&ts.poseIn, (void**)&ts.poseTmp, (void**)&ts.cam4, (void**)&ts.nInlTmp,
                          (void**)&ts.iXw, (void**)&ts.iObs, (void**)&ts.iTd, (void**)&ts.route, (void**)&ts.active, (void**)&ts.preint, (void**)&ts.preintKF2,
                          (void**)&ts.fixedState, (void**)&ts.state, (void**)&ts.prior, (void**)&ts.priorH, (void**)&ts.H15, (void**)&ts.ret,
                          (void**)&ts.groupStart, (void**)&ts.evBin, (void**)&ts.poseActive, (void**)&ts.nmCopy};
        size_t off = 0;
        for (int k = 0; k < nSlots; ++k) { *slots[k] = d_track + off; off += (sizes[k] + 255) & ~(size_t)255; }
        return ORB_OK;
    }
    void bind_gather(poseopt::GatherArgs& A) const {
        A.Xw = ts.Xw; A.obs = ts.obs; A.err = ts.err; A.invSigma2 = ts.is2; A.outlier = ts.outl; A.edgeKp = ts.edgeKp;
        A.N = ts.N; A.poseIn = ts.poseIn; A.poseTmp = ts.poseTmp; A.cam4 = ts.cam4; A.nInlTmp = ts.nInlTmp;
    }

    // SearchForInitialization: F2 in shared memory (K2 keypoints), K1 keypoints of F1 as the queries
    int run_init(MatchParams& P, int K2, int K1, cudaStream_t st) {
        P.query = d_query; P.resultIdx = d_resultIdx; P.resultDist = d_resultDist; P.status = d_status;
        P.ks = std::max(K2, 1); P.ms = std::max(K1, 1);
        if (P.ks > 65535 || P.ms > 65535) { set_error("more than 65535 keypoints per frame"); return ORB_ERR_CAPACITY; }
        // vnMatches21 [K2] behind the frame
        const size_t sm = frame_layout(P, al16(sizeof(uint16_t) * (size_t)P.ks), FRAME_SMEM_LIMIT, "frames too large for the matcher's shared-memory grid");
        if (!sm) return ORB_ERR_CAPACITY;
        int rc = ensure_dynamic_smem(init_match_kernel, sm, device);
        if (rc) return rc;
        ClusterLaunch L(sm, st);
        const int C = 8;                                   // one pair of frames: pass 1 spread over a full cluster
        CK(cudaLaunchKernelEx(L.shape(1, C), init_match_kernel, P));
        launches = 1;
        lastCluster = C;
        return ORB_OK;
    }
};

// ---- Frame::isInFrustum + MapPoint::PredictScale, thread per map point (src/Frame.cc:512-574, src/MapPoint.cc:531-546).
//      Every float operation is individually rounded in the order fixed by the oracle; std::log(float) is glibc's logf
//      (exact_math.h: logf_glibc). ----
struct FrustumParams {
    int M;
    const float *P, *N, *minD, *maxD, *maxRaw;
    float R[9], t[3], Ow[3], cam[4], minX, minY, maxX, maxY, mbf, logSF, cosLimit;
    int nLevels;
    uint8_t* inView; float *projX, *projY, *projXR, *depth, *viewCos; int* level;
};
// One map point: the body of frustum_project_kernel and of the batched frustum stage of orbm_track_local_map_batch* (tlm_frustum_kernel).
// Q supplies the pose, camera and image bounds and the point arrays (P, N, minD, maxD, maxRaw); the results go to the references.
__device__ __forceinline__ void frustum_point(const FrustumParams& Q, int i, uint8_t& in, float& px, float& py, float& pxr, float& dep, float& vc, int& lvl) {
    using namespace orbx;
    in = 0; px = -1.f; py = -1.f; pxr = 0.f; dep = 0.f; vc = 0.f; lvl = -1;
    const float X = Q.P[3 * i], Y = Q.P[3 * i + 1], Z = Q.P[3 * i + 2];
    const float xc = fadd(fadd(fadd(fmul(Q.R[0], X), fmul(Q.R[1], Y)), fmul(Q.R[2], Z)), Q.t[0]);
    const float yc = fadd(fadd(fadd(fmul(Q.R[3], X), fmul(Q.R[4], Y)), fmul(Q.R[5], Z)), Q.t[1]);
    const float zc = fadd(fadd(fadd(fmul(Q.R[6], X), fmul(Q.R[7], Y)), fmul(Q.R[8], Z)), Q.t[2]);
    const float pcDist = __fsqrt_rn(fadd(fadd(fmul(xc, xc), fmul(yc, yc)), fmul(zc, zc)));
    const float invz = fdiv(1.0f, zc);
    if (!(zc < 0.0f)) {
        const float u = fadd(fdiv(fmul(Q.cam[0], xc), zc), Q.cam[2]);
        const float v = fadd(fdiv(fmul(Q.cam[1], yc), zc), Q.cam[3]);
        if (!(u < Q.minX || u > Q.maxX) && !(v < Q.minY || v > Q.maxY)) {
            px = u; py = v;
            const float ox = fsub(X, Q.Ow[0]), oy = fsub(Y, Q.Ow[1]), oz = fsub(Z, Q.Ow[2]);
            const float dist = __fsqrt_rn(fadd(fadd(fmul(ox, ox), fmul(oy, oy)), fmul(oz, oz)));
            if (!(dist < Q.minD[i] || dist > Q.maxD[i])) {
                const float c = fdiv(fadd(fadd(fmul(ox, Q.N[3 * i]), fmul(oy, Q.N[3 * i + 1])), fmul(oz, Q.N[3 * i + 2])), dist);
                if (!(c < Q.cosLimit)) {
                    const float ratio = fdiv(Q.maxRaw[i], dist);
                    int n = (int)ceilf(fdiv(logf_glibc(ratio), Q.logSF));
                    if (n < 0) n = 0; else if (n >= Q.nLevels) n = Q.nLevels - 1;
                    in = 1; pxr = __fmaf_rn(-Q.mbf, invz, u) /* one FMA in the reference build, see oracle */; dep = pcDist; lvl = n; vc = c;
                }
            }
        }
    }
}
__global__ void frustum_project_kernel(FrustumParams Q) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Q.M) return;
    uint8_t in; float px, py, pxr, dep, vc; int lvl;
    frustum_point(Q, i, in, px, py, pxr, dep, vc, lvl);
    Q.inView[i] = in; Q.projX[i] = px; Q.projY[i] = py; Q.projXR[i] = pxr; Q.depth[i] = dep; Q.level[i] = lvl; Q.viewCos[i] = vc;
}

// ---- Tracking::SearchLocalPoints (src/Tracking.cc:3346) up to the search, one CTA per stream: the first loop over the frame's matches
//      (a bad point is dropped; the others are counted visible and marked seen -- mnLastFrameSeen), the points TrackWithMotionModel
//      discarded marked seen, Frame::UpdatePoseMatrices, then Frame::isInFrustum (frustum_point) for every local point neither seen
//      nor bad; a point in view is counted visible and becomes a query of the search.  claimed = the kept point has observations. ----
struct TrackLocalParams {
    int batch, kcap, mcap, mcapLast;
    const uint8_t* active; const int *nK, *nM;
    int* match; uint8_t* claimed;                        // [batch][kcap]
    const int* lastToLocal; const uint8_t* discarded;    // [batch][mcapLast] (discarded: [batch][mcap] without lastToLocal)
    const float* Tcw7;                                   // [batch][7]
    FrustumParams F;                                     // camera, bounds, limits; point arrays = the [batch][mcap] slabs
    const uint8_t *bad, *hasObs;
    uint8_t *seen, *inView; float *projX, *projY, *depth, *viewCos; int* level;   // scratch [batch][mcap]
    int *visible, *found, *nToMatch;
};
constexpr int TL_NT = 512;
__global__ void __launch_bounds__(TL_NT) tlm_frustum_kernel(TrackLocalParams T) {
    __shared__ FrustumParams s_Q;
    __shared__ int s_n;
    const int f = blockIdx.x, tid = threadIdx.x;
    if (T.active && !T.active[f]) return;
    const int K = min(T.nK[f], T.kcap), M = min(T.nM[f], T.mcap);
    const size_t kb = (size_t)f * T.kcap, pb = (size_t)f * T.mcap;
    if (tid == 0) {
        s_Q = T.F;
        s_Q.M = M; s_Q.P = T.F.P + 3 * pb; s_Q.N = T.F.N + 3 * pb; s_Q.minD = T.F.minD + pb; s_Q.maxD = T.F.maxD + pb; s_Q.maxRaw = T.F.maxRaw + pb;
        update_pose_matrices(T.Tcw7 + 7 * (size_t)f, s_Q.R, s_Q.t, s_Q.Ow);
        s_n = 0;
    }
    for (int p = tid; p < T.mcap; p += TL_NT) { T.seen[pb + p] = 0; T.inView[pb + p] = 0; T.visible[pb + p] = 0; T.found[pb + p] = 0; }
    for (int i = K + tid; i < T.kcap; i += TL_NT) T.claimed[kb + i] = 0;
    __syncthreads();
    for (int i = tid; i < K; i += TL_NT) {
        const int m = T.match[kb + i];
        if (m < 0) { T.claimed[kb + i] = 0; continue; }
        const int p = T.lastToLocal ? (m < T.mcapLast ? T.lastToLocal[(size_t)f * T.mcapLast + m] : -1) : m;
        if (p < 0 || p >= M || T.bad[pb + p]) { T.match[kb + i] = -1; T.claimed[kb + i] = 0; continue; }
        T.match[kb + i] = p; T.claimed[kb + i] = T.hasObs[pb + p] ? 1 : 0;
        atomicAdd(&T.visible[pb + p], 1);
        T.seen[pb + p] = 1;
    }
    if (T.discarded) {
        const int n = T.lastToLocal ? T.mcapLast : M;
        const size_t db = (size_t)f * (T.lastToLocal ? T.mcapLast : T.mcap);
        for (int j = tid; j < n; j += TL_NT) {
            if (!T.discarded[db + j]) continue;
            const int p = T.lastToLocal ? T.lastToLocal[db + j] : j;
            if (p >= 0 && p < M) T.seen[pb + p] = 1;
        }
    }
    __syncthreads();
    int cnt = 0;
    for (int p = tid; p < M; p += TL_NT) {
        if (T.seen[pb + p] || T.bad[pb + p]) continue;
        uint8_t in; float px, py, pxr, dep, vc; int lvl;
        frustum_point(s_Q, p, in, px, py, pxr, dep, vc, lvl);
        if (!in) continue;
        T.inView[pb + p] = 1; T.projX[pb + p] = px; T.projY[pb + p] = py; T.depth[pb + p] = dep; T.viewCos[pb + p] = vc; T.level[pb + p] = lvl;
        T.visible[pb + p] += 1;
        ++cnt;
    }
    if (cnt) atomicAdd(&s_n, cnt);
    __syncthreads();
    if (tid == 0) T.nToMatch[f] = s_n;
}

}  // namespace orbm

using namespace orbm;

struct orbm_handle { Matcher m; };

MatcherContext orbm::matcher_context(orbm_handle* h) { return {&h->m.staging, h->m.stream, h->m.device, &h->m.launches, &h->m.ulm}; }

// ---- the host forms of the batched tracking calls (below): what they share about the current frame ----
// One stream's current frame: nK in [0, kcap] and every keypoint octave in [0, nlevels).
template <class Batch> static bool stream_frame_ok(const Batch* in, size_t b, const char* who) {
    const int n = in->nK[b];
    if (n < 0 || n > in->kcap) { set_error(std::string(who) + ": nK out of range"); return false; }
    for (int i = 0; i < n; ++i) {
        const int oct = in->kps[b * in->kcap + i].octave;
        if (oct < 0 || oct >= in->nlevels) { set_error(std::string(who) + ": keypoint octave out of range"); return false; }
    }
    return true;
}

// The current frame's pieces: kps, desc and nK, and for TrackReferenceKeyFrame its FeatureVector (fvNode, fvFeature, nEntries).  A
// _resident call reads the frame from device slabs, so its pieces are neither staged nor rebound.
template <class Batch> class BatchFrame {
    static constexpr bool FV = std::is_same<Batch, OrbmRefKeyFrameBatch>::value;
    bool staged;
    int kps = 0, desc = 0, nK = 0, fvNode = 0, fvFeature = 0, nEntries = 0;
public:
    BatchFrame(Staging& S, const Batch* in, bool frameOnDevice) : staged(!frameOnDevice) {
        if (!staged) return;
        const size_t B = in->batch, K = in->kcap;
        kps = S.in(in->kps, 28 * B * K); desc = S.in(in->desc, 32 * B * K); nK = S.in(in->nK, 4 * B);
        if constexpr (FV) { fvNode = S.in(in->fvNode, 4 * B * K); fvFeature = S.in(in->fvFeature, 4 * B * K); nEntries = S.in(in->nEntries, 4 * B); }
    }
    // Points the device copy `d` of the batch at the staged pieces.  The staging is reserved.
    void bind(const Staging& S, Batch& d) const {
        if (!staged) return;
        d.kps = S.dev<OrbKeyPoint>(kps); d.desc = S.dev(desc); d.nK = S.dev<int>(nK);
        if constexpr (FV) { d.fvNode = S.dev<int>(fvNode); d.fvFeature = S.dev<int>(fvFeature); d.nEntries = S.dev<int>(nEntries); }
    }
};

extern "C" {

int orbm_create(orbm_handle** out, int max_batch, int max_keypoints, int max_mappoints, int device) {
    if (!out || max_batch < 1 || max_keypoints < 1 || max_mappoints < 1 || max_keypoints > 65535) { set_error("orbm_create: bad argument"); return ORB_ERR_ARG; }
    if (int rc = check_device(device)) return rc;
    orbm_handle* h = new orbm_handle();
    h->m.device = device; h->m.maxBatch = max_batch; h->m.kcap = max_keypoints; h->m.mcap = max_mappoints;
    int rc = h->m.init();
    if (rc) { delete h; return rc; }
    *out = h;
    return ORB_OK;
}

void orbm_destroy(orbm_handle* h) { delete h; }
int orbm_last_launch_count(const orbm_handle* h) { return h ? h->m.launches : ORB_ERR_ARG; }
int orbm_last_cluster_size(const orbm_handle* h) { return h ? h->m.lastCluster : ORB_ERR_ARG; }
#ifdef MF_PHASES
// out[8]: match_frame_kernel's phase counters (mf_phase) since the last call, which zeroes them; returns the last call's cluster size.
int orbm_match_phases(const orbm_handle* h, unsigned long long* out) {
    if (!h || !out) return ORB_ERR_ARG;
    CK(cudaSetDevice(h->m.device));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpyFromSymbol(out, orbm::mf_phase, sizeof(orbm::mf_phase)));
    const unsigned long long zero[8] = {};
    CK(cudaMemcpyToSymbol(orbm::mf_phase, zero, sizeof(zero)));
    return h->m.lastCluster;
}
#endif

static bool frame_ok(const Matcher& m, const OrbmFrame* fr) {
    if (!fr || fr->K < 0 || fr->K > m.kcap || !fr->scaleFactors || fr->nlevels < 1 || !(fr->maxX > fr->minX) || !(fr->maxY > fr->minY)) {
        set_error("bad OrbmFrame (K > max_keypoints?)"); return false;
    }
    return true;
}

// The current frame of the two single-frame searches: keypoints, descriptors and scale factors, match / claimed in and out, and
// the counts {K, nmatches, M}.
struct FramePieces { int kps, desc, sf, match, claimed, counts; };
static FramePieces stage_frame(Staging& S, const OrbmFrame* fr, int32_t* match, uint8_t* claimed) {
    const size_t K = fr->K;
    return {S.in(fr->keypoints, sizeof(OrbKeyPoint) * K), S.in(fr->descriptors, 32 * K), S.in(fr->scaleFactors, 4 * (size_t)fr->nlevels),
            S.inout(match, 4 * K), S.inout(claimed, K), S.inout(nullptr, 3 * sizeof(int))};
}

// Binds the frame to P, uploads, runs the fused matcher and brings match / claimed / nmatches back.  The staging is reserved.
static int search_frame(Matcher& m, const FramePieces& f, const OrbmFrame* fr, int M, MatchParams& P, int* nmatches) {
    Staging& S = m.staging;
    int* counts = S.host<int>(f.counts);
    counts[0] = fr->K; counts[1] = 0; counts[2] = M;
    P.kps = S.dev<OrbKeyPoint>(f.kps); P.desc = S.dev(f.desc); P.scaleFactors = S.dev<float>(f.sf);
    P.match = S.dev<int>(f.match); P.claimed = S.dev(f.claimed);
    P.nK = S.dev<int>(f.counts); P.nmatches = S.dev<int>(f.counts) + 1; P.nM = P.nK + 2;
    P.batch = 1; P.kcap = m.kcap; P.mcap = m.mcap; P.nlevels = fr->nlevels;
    P.minX = fr->minX; P.minY = fr->minY; P.maxX = fr->maxX; P.maxY = fr->maxY;
    CK(S.upload(m.stream));
    int rc = m.run(P, fr->K, M, m.stream);
    if (rc) return rc;
    CK(S.download(m.stream));
    *nmatches = counts[1];
    return ORB_OK;
}

int orbm_search_local_map(orbm_handle* h, const OrbmFrame* fr, const OrbmLocalPoints* pts, float th, float nnratio, int bFar,
                          float thFar, int32_t* match, uint8_t* claimed, int* nmatches) {
    if (!h || !pts || !match || !claimed || !nmatches || pts->M < 0 || pts->M > h->m.mcap) { set_error("orbm_search_local_map: bad argument"); return ORB_ERR_ARG; }
    Matcher& m = h->m;
    CK(cudaSetDevice(m.device));
    if (!frame_ok(m, fr)) return ORB_ERR_ARG;
    const size_t M = pts->M;
    for (size_t i = 0; i < M; ++i)
        if (pts->inView[i] && !pts->bad[i] && (pts->level[i] < 0 || pts->level[i] >= fr->nlevels)) { set_error("map point level out of range"); return ORB_ERR_ARG; }
    Staging& S = m.staging;
    S.begin();
    const FramePieces f = stage_frame(S, fr, match, claimed);
    const int pIn = S.in(pts->inView, M), pBad = S.in(pts->bad, M), pDepth = S.in(pts->depth, 4 * M), pX = S.in(pts->projX, 4 * M), pY = S.in(pts->projY, 4 * M),
              pLevel = S.in(pts->level, 4 * M), pCos = S.in(pts->viewCos, 4 * M), pObs = S.in(pts->hasObs, M), pDesc = S.in(pts->descriptors, 32 * M);
    int rc = S.reserve();
    if (rc) return rc;
    MatchParams P; memset(&P, 0, sizeof(P));
    P.inView = S.dev(pIn); P.bad = S.dev(pBad); P.depth = S.dev<float>(pDepth); P.projX = S.dev<float>(pX); P.projY = S.dev<float>(pY);
    P.level = S.dev<int>(pLevel); P.viewCos = S.dev<float>(pCos); P.hasObs = S.dev(pObs); P.mpDesc = S.dev(pDesc);
    P.mode = 0; P.th = th; P.nnratio = nnratio; P.bFar = bFar; P.thFar = thFar;
    return search_frame(m, f, fr, pts->M, P, nmatches);
}

int orbm_search_last_frame(orbm_handle* h, const OrbmFrame* fr, const OrbmLastFrame* last, const float* Tcw7, const float* cam4,
                           float th, int checkOri, int32_t* match, uint8_t* claimed, int* nmatches) {
    if (!h || !last || !Tcw7 || !cam4 || !match || !claimed || !nmatches || last->M < 0 || last->M > h->m.mcap) { set_error("orbm_search_last_frame: bad argument"); return ORB_ERR_ARG; }
    Matcher& m = h->m;
    CK(cudaSetDevice(m.device));
    if (!frame_ok(m, fr)) return ORB_ERR_ARG;
    const size_t M = last->M;
    for (size_t i = 0; i < M; ++i)
        if (last->valid[i] && (last->octave[i] < 0 || last->octave[i] >= fr->nlevels)) { set_error("last-frame octave out of range"); return ORB_ERR_ARG; }
    Staging& S = m.staging;
    S.begin();
    const FramePieces f = stage_frame(S, fr, match, claimed);
    const int pValid = S.in(last->valid, M), pXyz = S.in(last->xyz, 12 * M), pOct = S.in(last->octave, 4 * M), pAng = S.in(last->angle, 4 * M),
              pObs = S.in(last->hasObs, M), pDesc = S.in(last->descriptors, 32 * M), pT = S.in(Tcw7, 28);
    int rc = S.reserve();
    if (rc) return rc;
    MatchParams P; memset(&P, 0, sizeof(P));
    P.valid = S.dev(pValid); P.xyz = S.dev<float>(pXyz); P.octave = S.dev<int>(pOct); P.angle = S.dev<float>(pAng); P.hasObs = S.dev(pObs);
    P.mpDesc = S.dev(pDesc); P.Tcw7 = S.dev<float>(pT);
    memcpy(P.cam, cam4, sizeof(float) * 4);
    P.mode = 1; P.th = th; P.checkOri = checkOri;
    return search_frame(m, f, fr, last->M, P, nmatches);
}

int orbm_search_last_frame_batch_device(orbm_handle* h, const OrbmBatchDevice* in, float th, int checkOri, int32_t* d_match,
                                        uint8_t* d_claimed, int32_t* d_nmatches, void* stream) {
    if (!h || !in || !d_match || !d_claimed || !d_nmatches || in->batch < 1 || in->batch > h->m.maxBatch || in->kcap > 65535 ||
        in->kcap > h->m.kcap || in->mcap > h->m.mcap || in->kcap < 1 || in->mcap < 1 || in->nlevels < 1 || !(in->maxX > in->minX) ||
        !(in->maxY > in->minY) || !in->kps || !in->desc || !in->nK || !in->nM || !in->scaleFactors) {
        set_error("orbm_search_last_frame_batch_device: bad argument (sizes, image bounds or null slabs)"); return ORB_ERR_ARG;
    }
    Matcher& m = h->m;
    CK(cudaSetDevice(m.device));
    MatchParams P; memset(&P, 0, sizeof(P));
    P.batch = in->batch; P.kcap = in->kcap; P.mcap = in->mcap; P.nlevels = in->nlevels; P.mode = 1;
    P.kps = in->kps; P.desc = in->desc; P.nK = in->nK;
    P.minX = in->minX; P.minY = in->minY; P.maxX = in->maxX; P.maxY = in->maxY;
    P.scaleFactors = in->scaleFactors; P.nM = in->nM;
    P.valid = in->valid; P.xyz = in->xyz; P.octave = in->octave; P.angle = in->angle; P.hasObs = in->hasObs; P.mpDesc = in->mpDesc;
    P.Tcw7 = in->Tcw7; memcpy(P.cam, in->cam, sizeof(float) * 4);
    P.th = th; P.checkOri = checkOri; P.resetState = in->resetState;
    P.match = d_match; P.claimed = d_claimed; P.nmatches = d_nmatches;
    return m.run(P, in->kcap, in->mcap, (cudaStream_t)stream);
}

static int search_last_frame_batch_host(orbm_handle* h, const OrbmBatchDevice* in, float th, int checkOri, int32_t* match, uint8_t* claimed,
                                       int32_t* nmatches, bool frameOnDevice) {
    if (!h || !in || !match || !claimed || !nmatches || in->batch < 1 || in->batch > h->m.maxBatch || in->kcap > h->m.kcap ||
        in->mcap > h->m.mcap || in->nlevels < 1) { set_error("orbm_search_last_frame_batch: bad argument"); return ORB_ERR_ARG; }
    Matcher& m = h->m;
    CK(cudaSetDevice(m.device));
    cudaStream_t st = m.stream;
    const size_t B = in->batch, K = in->kcap, M = in->mcap;
    size_t off = 0;
    OrbmBatchDevice d = *in;
    auto up = [&](const void* src, size_t bytes, const void** dst) -> int {
        off = (off + 255) & ~(size_t)255;
        if (off + bytes > m.batchBytes) { set_error("orbm_search_last_frame_batch: staging too small"); return ORB_ERR_CAPACITY; }
        if (src) { cudaError_t e = cudaMemcpyAsync(m.d_batch + off, src, bytes, cudaMemcpyHostToDevice, st); if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return ORB_ERR_CUDA; } }
        *dst = m.d_batch + off; off += bytes;
        return ORB_OK;
    };
    int rc;
    const void *dm, *dc, *dn;
#define UP(field, bytes) if ((rc = up(in->field, bytes, (const void**)&d.field))) return rc
    if (!frameOnDevice) { UP(kps, B * K * 28); UP(desc, B * K * 32); UP(nK, B * 4); }
    UP(scaleFactors, (size_t)in->nlevels * 4); UP(nM, B * 4);
    UP(valid, B * M); UP(xyz, B * M * 12); UP(octave, B * M * 4); UP(angle, B * M * 4); UP(hasObs, B * M); UP(mpDesc, B * M * 32); UP(Tcw7, B * 28);
#undef UP
    // with resetState the incoming match / claimed arrays are not read: do not ship them
    if ((rc = up(in->resetState ? nullptr : match, B * K * 4, &dm)) || (rc = up(in->resetState ? nullptr : claimed, B * K, &dc)) ||
        (rc = up(nullptr, B * 4, &dn))) return rc;
    rc = orbm_search_last_frame_batch_device(h, &d, th, checkOri, (int32_t*)dm, (uint8_t*)dc, (int32_t*)dn, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(match, dm, B * K * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(claimed, dc, B * K, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(nmatches, dn, B * 4, cudaMemcpyDeviceToHost, st));
    CK(orbx::wait_stream_blocking(st, m.evWait));
    return ORB_OK;
}

int orbm_search_for_initialization(orbm_handle* h, const OrbmFrame* F1, const OrbmFrame* F2, float* prevMatched, int windowSize, float nnratio,
                                   int checkOrientation, int32_t* matches12, int* nmatches) {
    if (!h || !F1 || !F2 || !prevMatched || !matches12 || !nmatches || F1->K < 0 || F2->K < 0 || F1->K > h->m.mcap || F2->K > h->m.kcap ||
        F2->nlevels < 1 || !(F2->maxX > F2->minX) || !(F2->maxY > F2->minY) || windowSize < 0) {
        set_error("orbm_search_for_initialization: bad argument (F1.K <= max_mappoints, F2.K <= max_keypoints)"); return ORB_ERR_ARG;
    }
    Matcher& m = h->m;
    CK(cudaSetDevice(m.device));
    const size_t K1 = F1->K, K2 = F2->K;
    *nmatches = 0;
    for (size_t i = 0; i < K1; ++i) matches12[i] = -1;              // vnMatches12 = vector<int>(F1.mvKeysUn.size(),-1), :651
    if (K1 == 0) return ORB_OK;
    Staging& S = m.staging;
    S.begin();
    const int pKps = S.in(F2->keypoints, sizeof(OrbKeyPoint) * K2), pDesc = S.in(F2->descriptors, 32 * K2), pMpDesc = S.in(F1->descriptors, 32 * K1),
              pX = S.in(nullptr, 4 * K1), pY = S.in(nullptr, 4 * K1), pAng = S.in(nullptr, 4 * K1), pLvl = S.in(nullptr, 4 * K1), pCounts = S.in(nullptr, 8),
              pMatch = S.out(matches12, 4 * K1), pN = S.out(nmatches, 4), pQ = S.out(nullptr, sizeof(float4) * K1);
    int rc = S.reserve();
    if (rc) return rc;
    float *px = S.host<float>(pX), *py = S.host<float>(pY), *ang = S.host<float>(pAng);
    int* lvl = S.host<int>(pLvl);
    for (size_t i = 0; i < K1; ++i) { px[i] = prevMatched[2 * i]; py[i] = prevMatched[2 * i + 1]; ang[i] = F1->keypoints[i].angle; lvl[i] = F1->keypoints[i].octave; }
    S.host<int>(pCounts)[0] = F2->K; S.host<int>(pCounts)[1] = F1->K;
    MatchParams P; memset(&P, 0, sizeof(P));
    P.kps = S.dev<OrbKeyPoint>(pKps); P.desc = S.dev(pDesc); P.mpDesc = S.dev(pMpDesc);
    P.projX = S.dev<float>(pX); P.projY = S.dev<float>(pY); P.angle = S.dev<float>(pAng); P.level = S.dev<int>(pLvl);
    P.nK = S.dev<int>(pCounts); P.nM = P.nK + 1;
    P.batch = 1; P.kcap = m.kcap; P.mcap = m.mcap; P.nlevels = F2->nlevels; P.mode = 2;
    P.minX = F2->minX; P.minY = F2->minY; P.maxX = F2->maxX; P.maxY = F2->maxY;
    P.th = (float)windowSize; P.nnratio = nnratio; P.checkOri = checkOrientation;
    P.match = S.dev<int>(pMatch); P.nmatches = S.dev<int>(pN);
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    rc = m.run_init(P, F2->K, F1->K, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(S.dev(pQ), m.d_query, sizeof(float4) * K1, cudaMemcpyDeviceToDevice, st));      // the updated window centres
    CK(S.download(st));
    const float4* q = S.host<float4>(pQ);
    for (size_t i = 0; i < K1; ++i) { prevMatched[2 * i] = q[i].x; prevMatched[2 * i + 1] = q[i].y; }
    return ORB_OK;
}

int orbm_search_last_frame_batch(orbm_handle* h, const OrbmBatchDevice* in, float th, int checkOri, int32_t* match, uint8_t* claimed,
                                 int32_t* nmatches) {
    return search_last_frame_batch_host(h, in, th, checkOri, match, claimed, nmatches, false);
}
int orbm_search_last_frame_batch_resident(orbm_handle* h, const OrbmBatchDevice* in, float th, int checkOri, int32_t* match, uint8_t* claimed,
                                          int32_t* nmatches) {
    return search_last_frame_batch_host(h, in, th, checkOri, match, claimed, nmatches, true);
}

// A FeatureVector of n entries over N features: node ids ascending, feature indices in [0, N).
static bool fv_ok(const int32_t* node, const int32_t* feat, int n, int N) {
    for (int e = 0; e < n; ++e) if (feat[e] < 0 || feat[e] >= N || (e && node[e] < node[e - 1])) return false;
    return true;
}

static int search_by_bow_impl(orbm_handle* h, const OrbmBowFrame* KF, const uint8_t* kfPoint, const OrbmBowFrame* F, const uint8_t* fPoint, float nnratio,
                              int checkOrientation, int32_t* match, int32_t* match12, int* nmatches) {
    if (!h || !KF || !F || !kfPoint || (!match && !match12) || !nmatches || KF->N < 0 || F->N < 0 || KF->nEntries < 0 || F->nEntries < 0 || KF->nEntries > KF->N ||
        F->nEntries > F->N || KF->N > h->m.mcap || F->N > h->m.kcap) {
        set_error("orbm_search_by_bow: bad argument (KF.N <= max_mappoints, F.N <= max_keypoints of the handle)"); return ORB_ERR_ARG;
    }
    if (!fv_ok(KF->fvNode, KF->fvFeature, KF->nEntries, KF->N)) { set_error("orbm_search_by_bow: keyframe feature vector not sorted / out of range"); return ORB_ERR_ARG; }
    if (!fv_ok(F->fvNode, F->fvFeature, F->nEntries, F->N)) { set_error("orbm_search_by_bow: frame feature vector not sorted / out of range"); return ORB_ERR_ARG; }
    Matcher& m = h->m;
    CK(cudaSetDevice(m.device));
    *nmatches = 0;
    if (match) for (int i = 0; i < F->N; ++i) match[i] = -1;
    if (match12) for (int i = 0; i < KF->N; ++i) match12[i] = -1;
    if (F->N == 0 || KF->N == 0) return ORB_OK;
    const size_t nKF = KF->N, nF = F->N, eKF = KF->nEntries, eF = F->nEntries;
    Staging& S = m.staging;
    S.begin();
    const int pKpsKF = S.in(KF->keypoints, sizeof(OrbKeyPoint) * nKF), pDescKF = S.in(KF->descriptors, 32 * nKF), pPtKF = S.in(kfPoint, nKF),
              pNodeKF = S.in(KF->fvNode, 4 * eKF), pFeatKF = S.in(KF->fvFeature, 4 * eKF), pKpsF = S.in(F->keypoints, sizeof(OrbKeyPoint) * nF),
              pDescF = S.in(F->descriptors, 32 * nF), pNodeF = S.in(F->fvNode, 4 * eF), pFeatF = S.in(F->fvFeature, 4 * eF), pPtF = S.in(fPoint, fPoint ? nF : 0),
              pMatch = match ? S.out(match, 4 * nF) : S.scratch(4 * nF), pM12 = S.out(match12, match12 ? 4 * nKF : 0), pN = S.out(nmatches, 4),
              pGs = S.scratch(4 * (nKF + 1)), pEv = S.scratch(nF), pCounts = S.in(nullptr, 16);
    int rc = S.reserve();
    if (rc) return rc;
    int* counts = S.host<int>(pCounts);
    counts[0] = KF->N; counts[1] = F->N; counts[2] = KF->nEntries; counts[3] = F->nEntries;
    BowMatchParams Q; memset(&Q, 0, sizeof(Q));
    Q.nKF = S.dev<int>(pCounts); Q.nF = Q.nKF + 1; Q.eKF = Q.nKF + 2; Q.eF = Q.nKF + 3; Q.kfStride = KF->N; Q.fStride = F->N;
    Q.nnratio = nnratio; Q.checkOri = checkOrientation;
    Q.kpsKF = S.dev<OrbKeyPoint>(pKpsKF); Q.descKF = S.dev(pDescKF); Q.kfPoint = S.dev(pPtKF); Q.fvNodeKF = S.dev<int>(pNodeKF); Q.fvFeatKF = S.dev<int>(pFeatKF);
    Q.kpsF = S.dev<OrbKeyPoint>(pKpsF); Q.descF = S.dev(pDescF); Q.fvNodeF = S.dev<int>(pNodeF); Q.fvFeatF = S.dev<int>(pFeatF);
    if (fPoint) Q.fPoint = S.dev(pPtF);
    Q.match12 = match12 ? S.dev<int>(pM12) : nullptr; Q.strictLow = fPoint ? 1 : 0;
    Q.match = S.dev<int>(pMatch); Q.nmatches = S.dev<int>(pN); Q.groupStart = S.dev<int>(pGs); Q.evBin = S.dev(pEv);
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    bow_match_kernel<<<1, BM_NT, 0, st>>>(Q);
    m.launches = 1;
    CK(cudaGetLastError());
    CK(S.download(st));
    return ORB_OK;
}

int orbm_search_by_bow(orbm_handle* h, const OrbmBowFrame* KF, const uint8_t* kfPoint, const OrbmBowFrame* F, float nnratio, int checkOrientation,
                       int32_t* match, int* nmatches) {
    return search_by_bow_impl(h, KF, kfPoint, F, nullptr, nnratio, checkOrientation, match, nullptr, nmatches);
}
int orbm_search_by_bow_kf(orbm_handle* h, const OrbmBowFrame* KF1, const uint8_t* point1, const OrbmBowFrame* KF2, const uint8_t* point2, float nnratio,
                          int checkOrientation, int32_t* match12, int* nmatches) {
    if (!point2 || !match12) { set_error("orbm_search_by_bow_kf: bad argument"); return ORB_ERR_ARG; }
    return search_by_bow_impl(h, KF1, point1, KF2, point2, nnratio, checkOrientation, nullptr, match12, nmatches);
}

// ORB_ERR_ARG with a message naming the query, or ORB_OK.
static int check_common_regions_query(const Matcher& m, const OrbmCommonRegionsQuery& q, int qi) {
    auto bad = [qi](const std::string& what) {
        set_error("orbm_common_regions_bow_batch: query " + std::to_string(qi) + ": " + what); return ORB_ERR_ARG;
    };
    if (q.nKF < 1 || q.nPoints < 0 || q.nCand < 0) return bad("nKF < 1 or a negative count");
    if (!q.kf) return bad("kf is null");
    if (q.nPoints > 0 && !q.pointBad) return bad("pointBad is null");
    if (q.nCand > 0 && (!q.cand || !q.covStart || !q.status || !q.covList || !q.nmatches || !q.numBoWMatches)) return bad("cand / covStart / an output is null");
    if (q.nCand > 0 && q.kf[0].frame.N > 0 && (!q.matchedCov || !q.matchedPoint)) return bad("matchedCov / matchedPoint is null");
    for (int e = 0; e < q.nKF; ++e) {
        const OrbmCommonRegionsKF& K = q.kf[e];
        const OrbmBowFrame& F = K.frame;
        const std::string who = "kf " + std::to_string(e) + ": ";
        if (F.N < 0 || F.nEntries < 0 || F.nEntries > F.N) return bad(who + "N < 0 or nEntries outside [0, N]");
        if (F.N > (e == 0 ? m.mcap : m.kcap)) return bad(who + (e == 0 ? "N > max_mappoints" : "N > max_keypoints"));
        if (F.N > 0 && (!F.keypoints || !F.descriptors || !K.point)) return bad(who + "keypoints / descriptors / point is null");
        if (F.nEntries > 0 && (!F.fvNode || !F.fvFeature)) return bad(who + "fvNode / fvFeature is null");
        if (!fv_ok(F.fvNode, F.fvFeature, F.nEntries, F.N)) return bad(who + "feature vector not sorted / out of range");
        for (int i = 0; i < F.N; ++i) if (K.point[i] < -1 || K.point[i] >= q.nPoints) return bad(who + "point index out of range");
    }
    if (q.nCand > 0) {
        if (!csr_ok(q.nCand, q.covStart)) return bad("covStart must start at 0 and not decrease");
        if (q.covStart[q.nCand] > 0 && !q.cov) return bad("cov is null");
        for (int c = 0; c < q.nCand; ++c) {
            if (q.cand[c] < -1 || q.cand[c] == 0 || q.cand[c] >= q.nKF) return bad("cand outside [-1, nKF) or the current keyframe");
            if (q.covStart[c + 1] - q.covStart[c] > ORBM_CR_MAX_COV - 1) return bad("more than 10 covisibles");
        }
        for (int i = 0; i < q.covStart[q.nCand]; ++i)
            if (q.cov[i] < 1 || q.cov[i] >= q.nKF) return bad("cov outside [1, nKF)");
    }
    return ORB_OK;
}

int orbm_common_regions_bow_batch(orbm_handle* h, int nQueries, const OrbmCommonRegionsQuery* queries) {
    if (!h || nQueries < 0 || (nQueries > 0 && !queries)) { set_error("orbm_common_regions_bow_batch: bad argument"); return ORB_ERR_ARG; }
    Matcher& m = h->m;
    for (int qi = 0; qi < nQueries; ++qi)
        if (int rc = check_common_regions_query(m, queries[qi], qi)) return rc;
    // Steps 1-4 on the host: each candidate's vpCovKFi and status, and the (current keyframe, entry) pairs of the RAN candidates.  Only the
    // keyframes of those pairs are uploaded; `slot` numbers them in the call.
    struct Ran { int q, c, pairBegin, nPairs; };
    std::vector<Ran> ran;
    std::vector<int2> pairEntry;                  // call slots
    std::vector<int> pairJ, slotQ, slotE;         // pair -> j; slot -> (query, table entry)
    std::vector<std::vector<int>> slotOf(nQueries);
    long long nFeat = 0;
    int maxN0 = 0, maxN = 0;
    auto slot = [&](int qi, int e) {
        int& s = slotOf[qi][e];
        if (s < 0) { s = (int)slotQ.size(); slotQ.push_back(qi); slotE.push_back(e); nFeat += queries[qi].kf[e].frame.N; }
        return s;
    };
    for (int qi = 0; qi < nQueries; ++qi) {
        const OrbmCommonRegionsQuery& q = queries[qi];
        slotOf[qi].assign(q.nKF, -1);
        const int N0 = q.kf[0].frame.N;
        for (int c = 0; c < q.nCand; ++c) {
            int32_t* covList = q.covList + (size_t)c * ORBM_CR_MAX_COV;
            int32_t* nm = q.nmatches + (size_t)c * ORBM_CR_MAX_COV;
            for (int j = 0; j < ORBM_CR_MAX_COV; ++j) { covList[j] = -1; nm[j] = -1; }
            q.numBoWMatches[c] = 0;
            for (int k = 0; k < N0; ++k) { q.matchedCov[(size_t)c * N0 + k] = -1; q.matchedPoint[(size_t)c * N0 + k] = -1; }
            const int cand = q.cand[c];
            if (cand < 0 || q.kf[cand].bad) { q.status[c] = ORBM_CR_SKIPPED; continue; }
            const int c0 = q.covStart[c], nc = q.covStart[c + 1] - c0;
            int n = 0;
            covList[n++] = cand;
            for (int i = 1; i < nc; ++i) covList[n++] = q.cov[c0 + i];
            if (nc > 0) covList[n++] = q.cov[c0];
            bool near = false;
            for (int j = 0; j < n; ++j) near = near || q.kf[covList[j]].connected;
            if (near) { q.status[c] = ORBM_CR_ABORTED_NEAR; continue; }
            q.status[c] = ORBM_CR_RAN;
            Ran r{qi, c, (int)pairJ.size(), 0};
            for (int j = 0; j < n; ++j) {
                if (q.kf[covList[j]].bad) continue;
                pairEntry.push_back(make_int2(slot(qi, 0), slot(qi, covList[j])));
                pairJ.push_back(j);
                maxN = std::max(maxN, q.kf[covList[j]].frame.N);
                ++r.nPairs;
            }
            maxN0 = std::max(maxN0, N0);
            ran.push_back(r);
        }
    }
    m.launches = 0;
    if (ran.empty()) return ORB_OK;
    if (nFeat > 0x7fffffffLL) { set_error("orbm_common_regions_bow_batch: more than 2^31 - 1 features to upload"); return ORB_ERR_CAPACITY; }
    CK(cudaSetDevice(m.device));
    const size_t nSlots = slotQ.size(), nPairs = pairJ.size(), F = (size_t)std::max<long long>(nFeat, 1);
    const size_t kfStride = (size_t)std::max(maxN0, 1), fStride = (size_t)std::max(maxN, 1);
    Staging& S = m.staging;
    S.begin();
    const int pKps = S.in(nullptr, sizeof(OrbKeyPoint) * F), pDesc = S.in(nullptr, 32 * F), pFlag = S.in(nullptr, F), pNode = S.in(nullptr, 4 * F),
              pFeat = S.in(nullptr, 4 * F), pPoint = S.in(nullptr, 4 * F), pBase = S.in(nullptr, 4 * nSlots), pN = S.in(nullptr, 4 * nSlots),
              pE = S.in(nullptr, 4 * nSlots), pPair = S.in(pairEntry.data(), sizeof(int2) * nPairs), pJ = S.in(pairJ.data(), 4 * nPairs),
              pItems = S.in(nullptr, sizeof(CrMergeItem) * ran.size()), pNm = S.out(nullptr, 4 * nPairs);
    std::vector<int> pBad(nQueries, -1);
    for (int qi = 0; qi < nQueries; ++qi)
        if (queries[qi].nPoints > 0) pBad[qi] = S.in(queries[qi].pointBad, queries[qi].nPoints);
    std::vector<int> pOut(ran.size()), pHash(ran.size());
    std::vector<size_t> cap(ran.size());
    for (size_t r = 0; r < ran.size(); ++r) {
        const OrbmCommonRegionsQuery& q = queries[ran[r].q];
        const size_t N0 = (size_t)q.kf[0].frame.N, c = (size_t)ran[r].c;
        pOut[r] = S.out(q.matchedCov ? q.matchedCov + c * N0 : nullptr, 4 * N0);
        S.out(q.matchedPoint ? q.matchedPoint + c * N0 : nullptr, 4 * N0);
        S.out(q.numBoWMatches + c, 4);
        size_t hc = 1;
        while (hc < 2 * (size_t)ran[r].nPairs * N0) hc <<= 1;
        cap[r] = hc;
        pHash[r] = S.scratch(8 * hc);
    }
    const int pM12 = S.scratch(4 * nPairs * kfStride), pMatch = S.scratch(4 * nPairs * fStride), pGs = S.scratch(4 * nPairs * (kfStride + 1)),
              pEv = S.scratch(nPairs * fStride);
    if (int rc = S.reserve()) return rc;
    OrbKeyPoint* kps = S.host<OrbKeyPoint>(pKps);
    uint8_t *desc = S.host(pDesc), *flag = S.host(pFlag);
    int *node = S.host<int>(pNode), *feat = S.host<int>(pFeat), *point = S.host<int>(pPoint), *base = S.host<int>(pBase), *cnt = S.host<int>(pN),
        *ent = S.host<int>(pE);
    size_t off = 0;
    for (size_t s = 0; s < nSlots; ++s) {
        const OrbmCommonRegionsQuery& q = queries[slotQ[s]];
        const OrbmCommonRegionsKF& K = q.kf[slotE[s]];
        const size_t N = (size_t)K.frame.N, E = (size_t)K.frame.nEntries;
        base[s] = (int)off; cnt[s] = K.frame.N; ent[s] = K.frame.nEntries;
        if (N) {
            memcpy(kps + off, K.frame.keypoints, sizeof(OrbKeyPoint) * N);
            memcpy(desc + 32 * off, K.frame.descriptors, 32 * N);
            memcpy(point + off, K.point, 4 * N);
        }
        if (E) { memcpy(node + off, K.frame.fvNode, 4 * E); memcpy(feat + off, K.frame.fvFeature, 4 * E); }
        for (size_t i = 0; i < N; ++i) flag[off + i] = K.point[i] < 0 ? 0 : q.pointBad[K.point[i]] ? 2 : 1;
        off += N;
    }
    CrMergeItem* items = S.host<CrMergeItem>(pItems);
    for (size_t r = 0; r < ran.size(); ++r) {
        const OrbmCommonRegionsQuery& q = queries[ran[r].q];
        CrMergeItem& it = items[r];
        it.pairBegin = ran[r].pairBegin; it.nPairs = ran[r].nPairs; it.N0 = q.kf[0].frame.N; it.hashCap = (int)cap[r];
        it.pointBad = pBad[ran[r].q] >= 0 ? S.dev(pBad[ran[r].q]) : nullptr;
        it.matchedCov = S.dev<int>(pOut[r]); it.matchedPoint = S.dev<int>(pOut[r] + 1); it.numBoW = S.dev<int>(pOut[r] + 2);
        it.hashKey = S.dev<int>(pHash[r]); it.hashPos = it.hashKey + cap[r];
    }
    BowMatchParams Q; memset(&Q, 0, sizeof(Q));
    Q.nKF = Q.nF = S.dev<int>(pN); Q.eKF = Q.eF = S.dev<int>(pE); Q.kfStride = (int)kfStride; Q.fStride = (int)fStride;
    Q.kpsKF = Q.kpsF = S.dev<OrbKeyPoint>(pKps); Q.descKF = Q.descF = S.dev(pDesc); Q.kfPoint = Q.fPoint = S.dev(pFlag);
    Q.fvNodeKF = Q.fvNodeF = S.dev<int>(pNode); Q.fvFeatKF = Q.fvFeatF = S.dev<int>(pFeat);
    Q.nnratio = 0.9f; Q.checkOri = 1; Q.strictLow = 1;          // ORBmatcher matcherBoW(0.9, true) (src/LoopClosing.cc)
    Q.match12 = S.dev<int>(pM12); Q.match = S.dev<int>(pMatch); Q.nmatches = S.dev<int>(pNm); Q.groupStart = S.dev<int>(pGs); Q.evBin = S.dev(pEv);
    Q.pairEntry = S.dev<int2>(pPair); Q.entryBase = S.dev<int>(pBase);
    CrMergeParams P;
    P.items = S.dev<CrMergeItem>(pItems); P.match12 = Q.match12; P.kfStride = (int)kfStride;
    P.pairEntry = Q.pairEntry; P.entryBase = Q.entryBase; P.slotPoint = S.dev<int>(pPoint); P.pairJ = S.dev<int>(pJ);
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    bow_match_kernel<<<(unsigned)nPairs, BM_NT, 0, st>>>(Q);
    CK(cudaGetLastError());
    common_regions_merge_kernel<<<(unsigned)ran.size(), CRM_NT, 0, st>>>(P);
    CK(cudaGetLastError());
    m.launches = 2;
    CK(S.download(st));
    const int* nm = S.host<int>(pNm);
    for (const Ran& r : ran)
        for (int t = 0; t < r.nPairs; ++t)
            queries[r.q].nmatches[(size_t)r.c * ORBM_CR_MAX_COV + pairJ[r.pairBegin + t]] = nm[r.pairBegin + t];
    return ORB_OK;
}

// One search of fuse_search_kernel's table, host pointers.  invLevelSigma2 == nullptr: no chi-square gate.
struct FuseJob {
    const OrbmFrame* KF; const float* invLevelSigma2; float logScaleFactor;
    const float *Tcw7, *Ow3, *cam4;      // Tcw7 / Ow3 read in mode 0 only
    const OrbmFusePoints* pts; float th; int mode;
    int32_t *bestIdx, *bestDist;
};

// Runs the jobs (arguments already checked by the entry point) in ONE upload, ONE launch of fuse_search_kernel and ONE download.  Every
// output starts as -1 / 256; jobs with M == 0 or K == 0 stop there and take no CTA.  Keypoint octaves and the shared-memory grid are checked
// for all jobs before anything is staged.
static int fuse_search_run(Matcher& m, int n, const FuseJob* jobs) {
    CK(cudaSetDevice(m.device));
    for (int j = 0; j < n; ++j)
        for (int i = 0; i < jobs[j].pts->M; ++i) { jobs[j].bestIdx[i] = -1; jobs[j].bestDist[i] = 256; }
    std::vector<int> act;
    std::vector<MatchParams> frame;       // the keyframe part of each active job's MatchParams: bounds, grid scale, shared-memory layout
    size_t sm = 0;
    int nCta = 0;
    for (int j = 0; j < n; ++j) {
        const OrbmFrame* KF = jobs[j].KF;
        const int M = jobs[j].pts->M, K = KF->K;
        if (M == 0 || K == 0) continue;
        for (int k = 0; k < K; ++k) if (KF->keypoints[k].octave < 0 || KF->keypoints[k].octave >= KF->nlevels) { set_error("orbm_fuse_search: keypoint octave out of range"); return ORB_ERR_ARG; }
        MatchParams P = {};
        P.minX = KF->minX; P.minY = KF->minY; P.maxX = KF->maxX; P.maxY = KF->maxY;
        P.ks = K; P.ms = 1;
        const size_t b = frame_layout(P, 0, FRAME_SMEM_LIMIT, "keyframe too large for the matcher's shared-memory grid");
        if (!b) return ORB_ERR_CAPACITY;
        sm = std::max(sm, b);
        act.push_back(j);
        frame.push_back(P);
        nCta += std::min(16, (M + 127) / 128);          // every CTA rebuilds its item's grid: a few CTAs per item, ~8 map points per warp
    }
    if (act.empty()) return ORB_OK;
    int rc = ensure_dynamic_smem(fuse_search_kernel, sm, m.device);
    if (rc) return rc;
    struct Pieces { int kp, de, sf, is, st, xy, no, mi, ma, md, bi, bd; };
    std::vector<Pieces> pc(act.size());
    Staging& S = m.staging;
    S.begin();
    for (size_t a = 0; a < act.size(); ++a) {
        const FuseJob& J = jobs[act[a]];
        const OrbmFusePoints* pts = J.pts;
        const size_t M = (size_t)pts->M, K = (size_t)J.KF->K, nl = J.KF->nlevels;
        Pieces& p = pc[a];
        p.kp = S.in(J.KF->keypoints, sizeof(OrbKeyPoint) * K); p.de = S.in(J.KF->descriptors, 32 * K); p.sf = S.in(J.KF->scaleFactors, 4 * nl);
        p.is = S.in(J.invLevelSigma2, J.invLevelSigma2 ? 4 * nl : 0); p.st = S.in(pts->state, M); p.xy = S.in(pts->worldPos, 12 * M);
        p.no = S.in(pts->normal, J.mode == 0 ? 12 * M : 0); p.mi = S.in(pts->minDistance, 4 * M); p.ma = S.in(pts->maxDistance, 4 * M);
        p.md = S.in(pts->descriptors, 32 * M); p.bi = S.out(J.bestIdx, 4 * M); p.bd = S.out(J.bestDist, 4 * M);
    }
    const int pTab = S.in(nullptr, sizeof(FuseParams) * act.size()), pCta = S.in(nullptr, sizeof(int) * nCta);
    if ((rc = S.reserve())) return rc;
    FuseParams* tab = S.host<FuseParams>(pTab);
    int* ctaItem = S.host<int>(pCta);
    for (size_t a = 0, c = 0; a < act.size(); ++a) {
        const FuseJob& J = jobs[act[a]];
        const OrbmFrame* KF = J.KF;
        const Pieces& p = pc[a];
        FuseParams& Q = tab[a];
        memset(&Q, 0, sizeof(Q));
        MatchParams& P = Q.P;
        P = frame[a];
        P.kps = S.dev<OrbKeyPoint>(p.kp); P.desc = S.dev(p.de); P.scaleFactors = S.dev<float>(p.sf); P.kcap = m.kcap; P.nlevels = KF->nlevels; P.batch = 1;
        P.th = J.th; memcpy(P.cam, J.cam4, 16);
        Q.K = KF->K; Q.M = J.pts->M; Q.state = S.dev(p.st); Q.mpDesc = S.dev(p.md); Q.xyz = S.dev<float>(p.xy); Q.normal = S.dev<float>(p.no);
        Q.minD = S.dev<float>(p.mi); Q.maxD = S.dev<float>(p.ma); Q.invSigma2 = S.dev<float>(p.is);
        if (J.mode == 0) { memcpy(Q.Tcw, J.Tcw7, 28); memcpy(Q.Ow, J.Ow3, 12); }
        Q.logSF = J.logScaleFactor; Q.mode = J.mode; Q.gate = J.invLevelSigma2 ? 1 : 0;
        Q.bestIdx = S.dev<int>(p.bi); Q.bestDist = S.dev<int>(p.bd);
        Q.ctaBegin = (int)c; Q.nCta = std::min(16, (Q.M + 127) / 128);
        for (int k = 0; k < Q.nCta; ++k) ctaItem[c++] = (int)a;
    }
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    fuse_search_kernel<<<nCta, MF_NT, sm, st>>>(S.dev<FuseParams>(pTab), S.dev<int>(pCta));
    m.launches = 1;
    CK(cudaGetLastError());
    CK(S.download(st));
    return ORB_OK;
}

static int project_search_impl(orbm_handle* h, const OrbmFrame* KF, const float* invLevelSigma2, float logScaleFactor, const float* Tcw7, const float* Ow3,
                               const float* cam4, const OrbmFusePoints* pts, float th, int mode, int32_t* bestIdx, int32_t* bestDist) {
    if (!h || !KF || (mode == 0 && (!Tcw7 || !Ow3)) || !cam4 || !pts || !bestIdx || !bestDist || pts->M < 0 || KF->K < 0 || KF->K > h->m.kcap ||
        !KF->scaleFactors || KF->nlevels < 1 || KF->nlevels > 256 || !(KF->maxX > KF->minX) || !(KF->maxY > KF->minY)) {
        set_error("orbm_fuse_search: bad argument (KF.K <= max_keypoints of the handle)"); return ORB_ERR_ARG;
    }
    const FuseJob J = {KF, invLevelSigma2, logScaleFactor, Tcw7, Ow3, cam4, pts, th, mode, bestIdx, bestDist};
    return fuse_search_run(h->m, 1, &J);
}

int orbm_fuse_search_batch(orbm_handle* h, int nItems, const OrbmFuseItem* items) {
    if (!h || nItems < 0 || (nItems > 0 && !items)) { set_error("orbm_fuse_search_batch: bad argument"); return ORB_ERR_ARG; }
    std::vector<FuseJob> jobs((size_t)nItems);
    bool any = false;
    for (int j = 0; j < nItems; ++j) {
        const OrbmFuseItem& it = items[j];
        const OrbmFrame& KF = it.KF;
        const OrbmFusePoints& P = it.pts;
        if (KF.K < 0 || P.M < 0 || !it.invLevelSigma2 || !KF.scaleFactors || KF.nlevels < 1 || KF.nlevels > 256 || !(KF.maxX > KF.minX) || !(KF.maxY > KF.minY) ||
            (KF.K > 0 && (!KF.keypoints || !KF.descriptors)) ||
            (P.M > 0 && (!P.state || !P.worldPos || !P.normal || !P.minDistance || !P.maxDistance || !P.descriptors || !it.bestIdx || !it.bestDist))) {
            set_error("orbm_fuse_search_batch: bad argument in item " + std::to_string(j)); return ORB_ERR_ARG;
        }
        if (KF.K > h->m.kcap) { set_error("orbm_fuse_search_batch: item " + std::to_string(j) + " has more keypoints than max_keypoints of the handle"); return ORB_ERR_CAPACITY; }
        jobs[j] = FuseJob{&it.KF, it.invLevelSigma2, it.logScaleFactor, it.Tcw7, it.Ow, it.cam, &it.pts, it.th, 0, it.bestIdx, it.bestDist};
        any = any || (KF.K > 0 && P.M > 0);
    }
    const int rc = fuse_search_run(h->m, nItems, jobs.data());
    if (rc == ORB_OK && !any) h->m.launches = 0;
    return rc;
}

int orbm_fuse_search(orbm_handle* h, const OrbmFrame* KF, const float* invLevelSigma2, float logScaleFactor, const float* Tcw7, const float* Ow3,
                     const float* cam4, const OrbmFusePoints* pts, float th, int32_t* bestIdx, int32_t* bestDist) {
    if (!invLevelSigma2 || !pts || !pts->normal) { set_error("orbm_fuse_search: bad argument"); return ORB_ERR_ARG; }
    return project_search_impl(h, KF, invLevelSigma2, logScaleFactor, Tcw7, Ow3, cam4, pts, th, 0, bestIdx, bestDist);
}
int orbm_fuse_search_sim3(orbm_handle* h, const OrbmFrame* KF, float logScaleFactor, const float* Tcw7, const float* Ow3, const float* cam4, const OrbmFusePoints* pts,
                          float th, int32_t* bestIdx, int32_t* bestDist) {
    if (!pts || !pts->normal) { set_error("orbm_fuse_search_sim3: bad argument"); return ORB_ERR_ARG; }
    return project_search_impl(h, KF, nullptr, logScaleFactor, Tcw7, Ow3, cam4, pts, th, 0, bestIdx, bestDist);
}
int orbm_search_by_sim3(orbm_handle* h, const OrbmFrame* KF1, const OrbmFusePoints* pts1, const OrbmFrame* KF2, const OrbmFusePoints* pts2, float logScaleFactor,
                        const float* cam4, float th, const int32_t* pre12, int32_t* match12, int* nFound) {
    if (!h || !KF1 || !KF2 || !pts1 || !pts2 || !pre12 || !match12 || !nFound || pts1->M != KF1->K || pts2->M != KF2->K) {
        set_error("orbm_search_by_sim3: bad argument (one map-point slot per keyframe feature)"); return ORB_ERR_ARG;
    }
    const int N1 = KF1->K, N2 = KF2->K;
    for (int i = 0; i < N1; ++i) if (pre12[i] >= N2) { set_error("orbm_search_by_sim3: pre12 out of range"); return ORB_ERR_ARG; }
    // vbAlreadyMatched1 / 2 (:1478-1491) folded into the search flags
    std::vector<uint8_t> s1(N1), s2(N2);
    for (int i = 0; i < N1; ++i) s1[i] = pts1->state[i] == 1 && pre12[i] < 0;
    for (int i = 0; i < N2; ++i) s2[i] = pts2->state[i] == 1;
    for (int i = 0; i < N1; ++i) if (pre12[i] >= 0) s2[pre12[i]] = 0;
    std::vector<int32_t> m1(N1), d1(N1), m2(N2), d2(N2);
    OrbmFusePoints a = *pts1, b = *pts2;
    a.state = s1.data(); b.state = s2.data();
    int rc = project_search_impl(h, KF2, nullptr, logScaleFactor, nullptr, nullptr, cam4, &a, th, 2, m1.data(), d1.data());      // KF1's points in KF2 (:1497-1573)
    if (rc) return rc;
    rc = project_search_impl(h, KF1, nullptr, logScaleFactor, nullptr, nullptr, cam4, &b, th, 2, m2.data(), d2.data());          // KF2's points in KF1 (:1576-1652)
    if (rc) return rc;
    h->m.launches = 2;
    int n = 0;
    for (int i1 = 0; i1 < N1; ++i1) {                                                                                               // agreement (:1655-1671)
        match12[i1] = pre12[i1];
        const int idx2 = d1[i1] <= TH_HIGH ? m1[i1] : -1;
        if (idx2 >= 0 && (d2[idx2] <= TH_HIGH ? m2[idx2] : -1) == i1) { match12[i1] = idx2; ++n; }
    }
    *nFound = n;
    return ORB_OK;
}

static bool tri_frame_ok(const OrbmTriFrame* f) {
    if (!f || f->N < 0 || f->nEntries < 0 || f->nEntries > f->N) return false;
    if (f->N && (!f->keypoints || !f->descriptors || !f->hasMapPoint)) return false;
    if (f->nEntries && (!f->fvNode || !f->fvFeature)) return false;
    for (int e = 0; e < f->nEntries; ++e) if (f->fvFeature[e] < 0 || f->fvFeature[e] >= f->N || (e && f->fvNode[e] < f->fvNode[e - 1])) return false;
    return true;
}
// The SearchForTriangulation part (KF1 against nKF2 neighbours) shared by orbm_search_for_triangulation and the CreateNewMapPoints
// calls.  tri_stage declares one item's inputs on the matcher's staging: the level tables, KF1 and every neighbour's arrays.  After the
// caller has declared the item and pair tables and its own pieces and reserved, tri_fill writes the item's TriItem and its nKF2 TriPairs
// into the tables' host mirrors; the caller then uploads everything in ONE copy and runs tri_match_kernel over all pairs.
struct TriPieces {
    int sf, sg, kp1, de1, mp1, fn1, ff1;
    struct Neighbour { int kp, de, mp, fn, ff; };
    std::vector<Neighbour> kf2;
};
static TriPieces tri_stage(Staging& S, const OrbmTriFrame* KF1, int nKF2, const OrbmTriFrame* KF2, const float* scaleFactors, const float* levelSigma2,
                           int nlevels) {
    const size_t N1 = (size_t)KF1->N, E1 = (size_t)KF1->nEntries;
    TriPieces t;
    t.sf = S.in(scaleFactors, 4 * (size_t)nlevels); t.sg = S.in(levelSigma2, 4 * (size_t)nlevels);
    t.kp1 = S.in(KF1->keypoints, sizeof(OrbKeyPoint) * N1); t.de1 = S.in(KF1->descriptors, 32 * N1); t.mp1 = S.in(KF1->hasMapPoint, N1);
    t.fn1 = S.in(KF1->fvNode, 4 * E1); t.ff1 = S.in(KF1->fvFeature, 4 * E1);
    for (int k = 0; k < nKF2; ++k) {
        const size_t N2 = (size_t)KF2[k].N, E2 = (size_t)KF2[k].nEntries;
        t.kf2.push_back({S.in(KF2[k].keypoints, sizeof(OrbKeyPoint) * N2), S.in(KF2[k].descriptors, 32 * N2), S.in(KF2[k].hasMapPoint, N2),
                         S.in(KF2[k].fvNode, 4 * E2), S.in(KF2[k].fvFeature, 4 * E2)});
    }
    return t;
}
// item: the item's row in the item table; m12 / cnt / ev: device addresses of its matches12 [nKF2][N1], nmatches [nKF2] and bins [nKF2][N1].
static void tri_fill(const Staging& S, const TriPieces& t, const OrbmTriFrame* KF1, int nKF2, const OrbmTriFrame* KF2, const float* ep2, const float* F12,
                     int bCoarse, int item, int* m12, int* cnt, uint8_t* ev, TriItem* itemRow, TriPair* pairRows) {
    const size_t N1 = (size_t)KF1->N;
    TriItem Q; memset(&Q, 0, sizeof(Q));
    Q.N1 = (int)N1; Q.E1 = KF1->nEntries; Q.coarse = bCoarse;
    Q.kps1 = S.dev<OrbKeyPoint>(t.kp1); Q.desc1 = S.dev(t.de1); Q.hasMP1 = S.dev(t.mp1); Q.fvNode1 = S.dev<int>(t.fn1); Q.fvFeat1 = S.dev<int>(t.ff1);
    Q.scaleFactors = S.dev<float>(t.sf); Q.levelSigma2 = S.dev<float>(t.sg);
    memcpy(itemRow, &Q, sizeof(Q));
    for (int k = 0; k < nKF2; ++k) {
        const TriPieces::Neighbour& p = t.kf2[k];
        TriPair T; memset(&T, 0, sizeof(T));
        T.item = item; T.N2 = KF2[k].N; T.E2 = KF2[k].nEntries;
        T.kps2 = S.dev<OrbKeyPoint>(p.kp); T.desc2 = S.dev(p.de); T.hasMP2 = S.dev(p.mp); T.fvNode2 = S.dev<int>(p.fn); T.fvFeat2 = S.dev<int>(p.ff);
        memcpy(T.ep, ep2 + 2 * (size_t)k, 8); memcpy(T.F12, F12 + 9 * (size_t)k, 36);
        T.matches12 = m12 + (size_t)k * N1; T.nmatches = cnt + k; T.evBin = ev + (size_t)k * N1;
        memcpy(pairRows + k, &T, sizeof(T));
    }
}

int orbm_search_for_triangulation(orbm_handle* h, const OrbmTriFrame* KF1, int nKF2, const OrbmTriFrame* KF2, const float* scaleFactors, const float* levelSigma2,
                                  int nlevels, const float* ep2, const float* F12, int bCoarse, int checkOrientation, int32_t* matches12, int32_t* nmatches) {
    if (!h || nKF2 < 0 || !tri_frame_ok(KF1) || (nKF2 && (!KF2 || !ep2 || !F12 || !matches12 || !nmatches)) || !scaleFactors || !levelSigma2 || nlevels < 1 || nlevels > 256) {
        set_error("orbm_search_for_triangulation: bad argument (feature vectors must be sorted by node id, indices in range)"); return ORB_ERR_ARG;
    }
    for (int k = 0; k < nKF2; ++k) {
        if (!tri_frame_ok(KF2 + k)) { set_error("orbm_search_for_triangulation: bad KF2 entry"); return ORB_ERR_ARG; }
        for (int i = 0; i < KF2[k].N; ++i) if (KF2[k].keypoints[i].octave < 0 || KF2[k].keypoints[i].octave >= nlevels) { set_error("orbm_search_for_triangulation: keypoint octave out of range"); return ORB_ERR_ARG; }
    }
    if (nKF2 == 0) return ORB_OK;
    Matcher& m = h->m;
    CK(cudaSetDevice(m.device));
    const size_t N1 = (size_t)KF1->N, K = (size_t)nKF2;
    for (size_t i = 0; i < K * N1; ++i) matches12[i] = -1;
    for (int k = 0; k < nKF2; ++k) nmatches[k] = 0;
    if (N1 == 0) return ORB_OK;
    Staging& S = m.staging;
    S.begin();
    const TriPieces t = tri_stage(S, KF1, nKF2, KF2, scaleFactors, levelSigma2, nlevels);
    const int pItem = S.in(nullptr, sizeof(TriItem)), pPairs = S.in(nullptr, sizeof(TriPair) * K), pCnt = S.out(nmatches, 4 * K),
              pM12 = S.out(matches12, 4 * N1 * K), pEv = S.scratch(N1 * K);
    int rc = S.reserve();
    if (rc) return rc;
    tri_fill(S, t, KF1, nKF2, KF2, ep2, F12, bCoarse, 0, S.dev<int>(pM12), S.dev<int>(pCnt), S.dev(pEv), S.host<TriItem>(pItem), S.host<TriPair>(pPairs));
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    TriParams Q;
    Q.checkOri = checkOrientation; Q.items = S.dev<TriItem>(pItem); Q.pairs = S.dev<TriPair>(pPairs);
    tri_match_kernel<<<nKF2, TM_NT, 0, st>>>(Q);
    m.launches = 1;
    CK(cudaGetLastError());
    CK(S.download(st));
    return ORB_OK;
}

// LocalMapping::CreateNewMapPoints for nItems new keyframes, the single call being a batch of one.  Every item is checked before anything
// is staged; then one upload, tri_match_kernel over every (item, neighbour) pair, new_points_kernel over every (pair, idx1), one
// new_points_commit_kernel CTA per item, one download.  An item with nKF2 == 0 or KF1.N == 0 gets zero counts and takes no CTA.
static int new_points_run(orbm_handle* h, int nItems, const OrbmNewPointsItem* items, bool batch) {
    const std::string who = batch ? "orbm_create_new_map_points_batch" : "orbm_create_new_map_points";
    auto fail = [&](int rc, int j, const char* what) {
        set_error(who + (batch ? ": item " + std::to_string(j) + ": " : std::string(": ")) + what);
        return rc;
    };
    constexpr size_t MAX_PAIRS = 65535;       // new_points_kernel's gridDim.y
    size_t nPairs = 0;
    int over = -1;
    for (int j = 0; j < nItems; ++j) {
        const OrbmNewPointsItem& it = items[j];
        const OrbmNewPointsIn& in = it.in;
        if (!it.nNew || in.nKF2 < 0 || !tri_frame_ok(in.KF1) || (in.KF1->N && !it.out) ||
            (in.nKF2 && (!in.KF2 || !in.ep2 || !in.F12 || !it.nmatches || !it.ncreated)) || !in.scaleFactors || !in.levelSigma2 || in.nlevels < 1 ||
            in.nlevels > 256 || !in.Tcw || !in.Ow || !in.cam || !(in.scaleFactor > 0.0f) || !(in.thFarPoints >= 0.0f))
            return fail(ORB_ERR_ARG, j, "bad argument (feature vectors must be sorted by node id, indices in range; Tcw / Ow / cam for 1 + nKF2 keyframes)");
        const OrbmTriFrame* KF1 = in.KF1;
        const int nl = in.nlevels;
        for (int i = 0; i < KF1->N; ++i) if (KF1->keypoints[i].octave < 0 || KF1->keypoints[i].octave >= nl) return fail(ORB_ERR_ARG, j, "keypoint octave out of range");
        for (int k = 0; k < in.nKF2; ++k) {
            if (!tri_frame_ok(in.KF2 + k)) return fail(ORB_ERR_ARG, j, "bad KF2 entry");
            for (int i = 0; i < in.KF2[k].N; ++i) if (in.KF2[k].keypoints[i].octave < 0 || in.KF2[k].keypoints[i].octave >= nl) return fail(ORB_ERR_ARG, j, "keypoint octave out of range");
        }
        if (KF1->N > 0) nPairs += (size_t)in.nKF2;
        if (nPairs > MAX_PAIRS && over < 0) over = j;
    }
    if (over >= 0) return fail(ORB_ERR_CAPACITY, over, "more than 65535 (keyframe, neighbour) pairs in one call");
    std::vector<int> act;
    for (int j = 0; j < nItems; ++j) {
        const OrbmNewPointsItem& it = items[j];
        *it.nNew = 0;
        for (int k = 0; k < it.in.nKF2; ++k) { it.nmatches[k] = 0; it.ncreated[k] = 0; }
        if (it.in.nKF2 > 0 && it.in.KF1->N > 0) act.push_back(j);
    }
    Matcher& m = h->m;
    if (act.empty()) {
        if (batch) m.launches = 0;
        return ORB_OK;
    }
    CK(cudaSetDevice(m.device));
    Staging& S = m.staging;
    S.begin();
    // per item: its search inputs, Tcw / Ow / cam, counts = {nNew, nmatches [K], ncreated [K]} and its records (the first nNew go to `out`)
    struct Pieces { TriPieces t; int tcw, ow, cam, cnt, out; };
    std::vector<Pieces> pc(act.size());
    size_t nSlots = 0, sumN1 = 0;
    int maxN1 = 0;
    for (size_t a = 0; a < act.size(); ++a) {
        const OrbmNewPointsIn& in = items[act[a]].in;
        const size_t N1 = (size_t)in.KF1->N, K = (size_t)in.nKF2;
        Pieces& p = pc[a];
        p.t = tri_stage(S, in.KF1, in.nKF2, in.KF2, in.scaleFactors, in.levelSigma2, in.nlevels);
        p.tcw = S.in(in.Tcw, 48 * (K + 1)); p.ow = S.in(in.Ow, 12 * (K + 1)); p.cam = S.in(in.cam, 16 * (K + 1));
        p.cnt = S.out(nullptr, 4 * (1 + 2 * K)); p.out = S.out(nullptr, sizeof(OrbmNewPoint) * N1);
        nSlots += K * N1; sumN1 += N1; maxN1 = std::max(maxN1, in.KF1->N);
    }
    const int pTri = S.in(nullptr, sizeof(TriItem) * act.size()), pNp = S.in(nullptr, sizeof(NpItem) * act.size()), pPairs = S.in(nullptr, sizeof(TriPair) * nPairs),
              pM12 = S.scratch(4 * nSlots), pEv = S.scratch(nSlots), pNm = S.scratch(4 * nPairs), pReason = S.scratch(nSlots),
              pRecs = S.scratch(sizeof(OrbmNewPoint) * nSlots), pWin = S.scratch(4 * sumN1);
    int rc = S.reserve();
    if (rc) return rc;
    size_t pair = 0, slot = 0, win = 0;
    for (size_t a = 0; a < act.size(); ++a) {
        const OrbmNewPointsIn& in = items[act[a]].in;
        const Pieces& p = pc[a];
        tri_fill(S, p.t, in.KF1, in.nKF2, in.KF2, in.ep2, in.F12, in.bCoarse, (int)a, S.dev<int>(pM12) + slot, S.dev<int>(pNm) + pair, S.dev(pEv) + slot,
                 S.host<TriItem>(pTri) + a, S.host<TriPair>(pPairs) + pair);
        NpItem J; memset(&J, 0, sizeof(J));
        J.pair0 = (int)pair; J.nKF2 = in.nKF2; J.nlevels = in.nlevels; J.bInertial = in.bInertial ? 1 : 0;
        J.ratioFactor = 1.5f * in.scaleFactor; J.thFar = in.thFarPoints; J.slot0 = slot;
        J.Tcw = S.dev<float>(p.tcw); J.Ow = S.dev<float>(p.ow); J.cam = S.dev<float>(p.cam);
        J.winner = S.dev<int>(pWin) + win; J.counts = S.dev<int>(p.cnt); J.out = S.dev<OrbmNewPoint>(p.out);
        memcpy(S.host<NpItem>(pNp) + a, &J, sizeof(J));
        pair += (size_t)in.nKF2; slot += (size_t)in.nKF2 * in.KF1->N; win += (size_t)in.KF1->N;
    }
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    TriParams Q;
    Q.checkOri = 0; Q.items = S.dev<TriItem>(pTri); Q.pairs = S.dev<TriPair>(pPairs);
    tri_match_kernel<<<(unsigned)nPairs, TM_NT, 0, st>>>(Q);
    NewPointsParams P;
    P.tri = Q.items; P.items = S.dev<NpItem>(pNp); P.pairs = Q.pairs;
    P.matches12 = S.dev<int>(pM12); P.reason = S.dev(pReason); P.recs = S.dev<OrbmNewPoint>(pRecs);
    new_points_kernel<<<dim3((unsigned)((maxN1 + NP_NT - 1) / NP_NT), (unsigned)nPairs), NP_NT, 0, st>>>(P);
    new_points_commit_kernel<<<(unsigned)act.size(), NPC_NT, 0, st>>>(P);
    m.launches = 3;
    CK(cudaGetLastError());
    CK(S.download(st));
    for (size_t a = 0; a < act.size(); ++a) {
        const OrbmNewPointsItem& it = items[act[a]];
        const size_t K = (size_t)it.in.nKF2;
        const int* cnt = S.host<int>(pc[a].cnt);
        *it.nNew = cnt[0];
        memcpy(it.nmatches, cnt + 1, 4 * K); memcpy(it.ncreated, cnt + 1 + K, 4 * K);
        memcpy(it.out, S.host(pc[a].out), sizeof(OrbmNewPoint) * (size_t)cnt[0]);
    }
    return ORB_OK;
}

int orbm_create_new_map_points(orbm_handle* h, const OrbmNewPointsIn* in, OrbmNewPoint* out, int* nNew, int32_t* nmatches, int32_t* ncreated) {
    if (!h || !in) { set_error("orbm_create_new_map_points: bad argument"); return ORB_ERR_ARG; }
    const OrbmNewPointsItem it = {*in, out, nNew, nmatches, ncreated};
    return new_points_run(h, 1, &it, false);
}

int orbm_create_new_map_points_batch(orbm_handle* h, int nItems, const OrbmNewPointsItem* items) {
    if (!h || nItems < 0 || (nItems > 0 && !items)) { set_error("orbm_create_new_map_points_batch: bad argument"); return ORB_ERR_ARG; }
    return new_points_run(h, nItems, items, true);
}

int orbm_distinctive_descriptors(orbm_handle* h, int nPoints, const int32_t* obsStart, const uint8_t* descriptors, int32_t* best) {
    if (!h || nPoints < 0 || !obsStart || !best || (nPoints && obsStart[nPoints] > 0 && !descriptors)) { set_error("orbm_distinctive_descriptors: bad argument"); return ORB_ERR_ARG; }
    if (nPoints == 0) return ORB_OK;
    for (int p = 0; p < nPoints; ++p) if (obsStart[p + 1] < obsStart[p] || obsStart[p + 1] - obsStart[p] > 65535) { set_error("orbm_distinctive_descriptors: obsStart must be non-decreasing (<= 65535 observations per point)"); return ORB_ERR_ARG; }
    Matcher& m = h->m;
    CK(cudaSetDevice(m.device));
    const size_t total = (size_t)obsStart[nPoints];
    Staging& S = m.staging;
    S.begin();
    const int pS = S.in(obsStart, 4 * ((size_t)nPoints + 1)), pD = S.in(descriptors, 32 * total), pB = S.out(best, 4 * (size_t)nPoints);
    int rc = S.reserve();
    if (rc) return rc;
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    distinctive_kernel<<<(nPoints + 7) / 8, 256, 0, st>>>(nPoints, S.dev<int>(pS), S.dev(pD), S.dev<int>(pB));
    m.launches = 1;
    CK(cudaGetLastError());
    CK(S.download(st));
    return ORB_OK;
}

int orbm_frustum_project(orbm_handle* h, const OrbmFrustumIn* in, uint8_t* inView, float* projX, float* projY, float* projXR,
                         float* depth, int32_t* level, float* viewCos) {
    if (!h || !in || in->M < 0 || !inView || !projX || !projY || !projXR || !depth || !level || !viewCos ||
        (in->M && (!in->worldPos || !in->normal || !in->minDistInv || !in->maxDistInv || !in->maxDistance)) || in->nScaleLevels < 1) {
        set_error("orbm_frustum_project: bad argument"); return ORB_ERR_ARG;
    }
    Matcher& m = h->m;
    if (in->M > m.mcap) { set_error("orbm_frustum_project: more map points than max_mappoints"); return ORB_ERR_CAPACITY; }
    CK(cudaSetDevice(m.device));
    const size_t M = in->M;
    if (M == 0) return ORB_OK;
    Staging& S = m.staging;
    S.begin();
    const int pP = S.in(in->worldPos, 12 * M), pN = S.in(in->normal, 12 * M), pMin = S.in(in->minDistInv, 4 * M), pMax = S.in(in->maxDistInv, 4 * M),
              pRaw = S.in(in->maxDistance, 4 * M), pX = S.out(projX, 4 * M), pY = S.out(projY, 4 * M), pXR = S.out(projXR, 4 * M),
              pD = S.out(depth, 4 * M), pC = S.out(viewCos, 4 * M), pL = S.out(level, 4 * M), pIn = S.out(inView, M);
    int rc = S.reserve();
    if (rc) return rc;
    FrustumParams Q; memset(&Q, 0, sizeof(Q));
    Q.M = in->M;
    Q.P = S.dev<float>(pP); Q.N = S.dev<float>(pN); Q.minD = S.dev<float>(pMin); Q.maxD = S.dev<float>(pMax); Q.maxRaw = S.dev<float>(pRaw);
    memcpy(Q.R, in->Rcw, sizeof(Q.R)); memcpy(Q.t, in->tcw, sizeof(Q.t)); memcpy(Q.Ow, in->Ow, sizeof(Q.Ow)); memcpy(Q.cam, in->cam, sizeof(Q.cam));
    Q.minX = in->minX; Q.minY = in->minY; Q.maxX = in->maxX; Q.maxY = in->maxY; Q.mbf = in->mbf; Q.logSF = in->logScaleFactor;
    Q.cosLimit = in->viewingCosLimit; Q.nLevels = in->nScaleLevels;
    Q.inView = S.dev(pIn); Q.projX = S.dev<float>(pX); Q.projY = S.dev<float>(pY); Q.projXR = S.dev<float>(pXR);
    Q.depth = S.dev<float>(pD); Q.viewCos = S.dev<float>(pC); Q.level = S.dev<int>(pL);
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    frustum_project_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(Q);
    m.launches = 1;
    CK(cudaGetLastError());
    CK(S.download(st));
    return ORB_OK;
}

int orbm_bf_knn2(orbm_handle* h, const uint8_t* query, int Q, const uint8_t* train, int T, int32_t* idx, int32_t* dist) {
    if (!h || !query || !train || !idx || !dist || Q < 0 || T < 0) { set_error("orbm_bf_knn2: bad argument"); return ORB_ERR_ARG; }
    Matcher& m = h->m;
    CK(cudaSetDevice(m.device));
    if (Q == 0) return ORB_OK;
    Staging& S = m.staging;
    S.begin();
    const int pQ = S.in(query, 32 * (size_t)Q), pT = S.in(train, 32 * (size_t)T), pI = S.out(idx, 8 * (size_t)Q), pD = S.out(dist, 8 * (size_t)Q);
    int rc = S.reserve();
    if (rc) return rc;
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    bf_knn2_kernel<<<(Q + BF_NT / 32 - 1) / (BF_NT / 32), BF_NT, 0, st>>>(S.dev(pQ), Q, S.dev(pT), T, S.dev<int>(pI), S.dev<int>(pD));
    m.launches = 1;
    CK(cudaGetLastError());
    CK(S.download(st));
    return ORB_OK;
}

int orbm_descriptor_distance(orbm_handle* h, const uint8_t* a, const uint8_t* b, int n, int32_t* out) {
    if (!h || !a || !b || !out || n < 0) { set_error("orbm_descriptor_distance: bad argument"); return ORB_ERR_ARG; }
    Matcher& m = h->m;
    CK(cudaSetDevice(m.device));
    if (n == 0) return ORB_OK;
    Staging& S = m.staging;
    S.begin();
    const int pA = S.in(a, 32 * (size_t)n), pB = S.in(b, 32 * (size_t)n), pO = S.out(out, 4 * (size_t)n);
    int rc = S.reserve();
    if (rc) return rc;
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    hamming_pairs_kernel<<<(n + 255) / 256, 256, 0, st>>>(S.dev(pA), S.dev(pB), n, S.dev<int>(pO));
    m.launches = 1;
    CK(cudaGetLastError());
    CK(S.download(st));
    return ORB_OK;
}


// ---- TrackWithMotionModel's pose step and TrackLocalMap for a batch of streams (include/orb_b200.h) ----
static bool batch_shape_ok(const Matcher& m, int batch, int kcap, int mcap, int nlevels) {
    return batch >= 1 && batch <= m.maxBatch && kcap >= 1 && kcap <= m.kcap && mcap >= 1 && nlevels >= 1 && nlevels <= 256;
}
static int motion_model_pose_launch(Matcher& m, const OrbmBatchDevice* in, const float* invLevelSigma2, const uint8_t* active, int32_t* match,
                                    uint8_t* claimed, int32_t* nmatches, double* pose7, float* Tcw7, uint8_t* discarded, int32_t* nmatchesMap,
                                    cudaStream_t st) {
    int rc = m.track_scratch();
    if (rc) return rc;
    poseopt::GatherArgs A; memset(&A, 0, sizeof(A));
    A.batch = in->batch; A.kcap = in->kcap; A.pstride = in->mcap; A.nlevels = in->nlevels; A.mode = poseopt::MOTION_MODEL;
    A.active = active; A.kps = in->kps; A.nK = in->nK; A.match = match; A.claimed = claimed; A.nmatches = nmatches;
    A.xyz = in->xyz; A.hasObs = in->hasObs; A.invLevelSigma2 = invLevelSigma2; memcpy(A.cam, in->cam, 16);
    A.TcwIn = in->Tcw7; A.TcwOut = Tcw7; A.poseOut = pose7; A.nInliers = m.ts.nInliers; A.discarded = discarded; A.nmatchesMap = nmatchesMap;
    m.bind_gather(A);
    CK(poseopt::launch_gathered(A, st));
    m.launches = 3;
    return ORB_OK;
}

// Argument checks shared by both forms of the motion-model step.
static int motion_model_shape(const orbm_handle* h, const OrbmBatchDevice* in, const float* invLevelSigma2, const int32_t* match,
                              const uint8_t* claimed, const int32_t* nmatches, const double* pose7, const float* Tcw7, const uint8_t* discarded,
                              const int32_t* nmatchesMap, const char* who) {
    if (!h || !in || !batch_shape_ok(h->m, in->batch, in->kcap, in->mcap, in->nlevels) || !in->kps || !in->nK || !in->xyz || !in->hasObs ||
        !in->Tcw7 || !invLevelSigma2 || !match || !claimed || !nmatches || !pose7 || !Tcw7 || !discarded || !nmatchesMap) {
        set_error(std::string(who) + ": bad argument (sizes or null arrays)"); return ORB_ERR_ARG;
    }
    return ORB_OK;
}

int orbm_motion_model_pose_batch_device(orbm_handle* h, const OrbmBatchDevice* in, const float* d_invLevelSigma2, const uint8_t* d_active,
                                        int32_t* d_match, uint8_t* d_claimed, int32_t* d_nmatches, double* d_pose7, float* d_Tcw7,
                                        uint8_t* d_discarded, int32_t* d_nmatchesMap, void* stream) {
    if (int rc = motion_model_shape(h, in, d_invLevelSigma2, d_match, d_claimed, d_nmatches, d_pose7, d_Tcw7, d_discarded, d_nmatchesMap,
                                    "orbm_motion_model_pose_batch_device"))
        return rc;
    CK(cudaSetDevice(h->m.device));
    return motion_model_pose_launch(h->m, in, d_invLevelSigma2, d_active, d_match, d_claimed, d_nmatches, d_pose7, d_Tcw7, d_discarded,
                                    d_nmatchesMap, (cudaStream_t)stream);
}

// Copies row b of a downloaded piece to the caller for the active streams only (inactive streams are left untouched).
static void copy_active_rows(const Staging& S, int piece, void* dst, size_t rowBytes, int batch, const uint8_t* active) {
    if (!dst) return;
    const uint8_t* src = S.host(piece);
    for (int b = 0; b < batch; ++b)
        if (!active || active[b]) memcpy((uint8_t*)dst + b * rowBytes, src + b * rowBytes, rowBytes);
}

int orbm_motion_model_pose_batch(orbm_handle* h, const OrbmBatchDevice* in, const float* invLevelSigma2, const uint8_t* active, int32_t* match,
                                 uint8_t* claimed, int32_t* nmatches, double* pose7, float* Tcw7, uint8_t* discarded, int32_t* nmatchesMap) {
    const char* who = "orbm_motion_model_pose_batch";
    if (int rc = motion_model_shape(h, in, invLevelSigma2, match, claimed, nmatches, pose7, Tcw7, discarded, nmatchesMap, who)) return rc;
    Matcher& m = h->m;
    const size_t B = in->batch, K = in->kcap, M = in->mcap;
    for (size_t b = 0; b < B; ++b) {
        if (active && !active[b]) continue;
        if (!stream_frame_ok(in, b, who)) return ORB_ERR_ARG;
        for (int i = 0; i < in->nK[b]; ++i)
            if (match[b * K + i] < -1 || match[b * K + i] >= in->mcap) { set_error(std::string(who) + ": match index out of range"); return ORB_ERR_ARG; }
    }
    CK(cudaSetDevice(m.device));
    Staging& S = m.staging;
    S.begin();
    const int pKps = S.in(in->kps, 28 * B * K), pNK = S.in(in->nK, 4 * B), pXyz = S.in(in->xyz, 12 * B * M), pObs = S.in(in->hasObs, B * M),
              pT = S.in(in->Tcw7, 28 * B), pIs = S.in(invLevelSigma2, 4 * (size_t)in->nlevels), pAct = S.in(active, active ? B : 0),
              pMatch = S.inout(match, 4 * B * K), pCl = S.inout(claimed, B * K), pN = S.inout(nmatches, 4 * B), pPose = S.out(nullptr, 56 * B),
              pTo = S.out(nullptr, 28 * B), pDis = S.out(nullptr, B * M), pMap = S.out(nullptr, 4 * B);
    int rc = S.reserve();
    if (rc) return rc;
    OrbmBatchDevice d = *in;
    d.kps = S.dev<OrbKeyPoint>(pKps); d.nK = S.dev<int>(pNK); d.xyz = S.dev<float>(pXyz); d.hasObs = S.dev(pObs); d.Tcw7 = S.dev<float>(pT);
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    rc = motion_model_pose_launch(m, &d, S.dev<float>(pIs), active ? S.dev(pAct) : nullptr, S.dev<int>(pMatch), S.dev(pCl), S.dev<int>(pN),
                                  S.dev<double>(pPose), S.dev<float>(pTo), S.dev(pDis), S.dev<int>(pMap), st);
    if (rc) return rc;
    CK(S.download(st));
    copy_active_rows(S, pPose, pose7, 56, in->batch, active);
    copy_active_rows(S, pTo, Tcw7, 28, in->batch, active);
    copy_active_rows(S, pDis, discarded, M, in->batch, active);
    copy_active_rows(S, pMap, nmatchesMap, 4, in->batch, active);
    return ORB_OK;
}

// ---- TrackReferenceKeyFrame for a batch of streams (include/orb_b200.h): the batched SearchByBoW, then PoseOptimization and the
//      "discard outliers" loop -- the motion-model step's three launches -- on the streams that passed the match gate ----
constexpr float TRK_REF_NNRATIO = 0.7f;     // TrackReferenceKeyFrame (src/Tracking.cc:2723): ORBmatcher matcher(0.7,true);
constexpr int TRK_REF_MIN_MATCHES = 15;     //   and if(nmatches<15) return false;

static int ref_kf_shape(const Matcher& m, const OrbmRefKeyFrameBatch* in, const OrbmRefKeyFrameResult* out, const char* who) {
    if (!in || !out || in->batch < 1 || in->batch > m.maxBatch || in->kcap < 1 || in->mcap < 1 || in->nlevels < 1 || in->nlevels > 256 || !in->kps ||
        !in->desc || !in->nK || !in->fvNode || !in->fvFeature || !in->nEntries || !in->Tcw7 || !in->kfN || !in->kfKps || !in->kfDesc || !in->kfFvNode ||
        !in->kfFvFeature || !in->kfNEntries || !in->kfPoint || !in->xyz || !in->hasObs || !in->invLevelSigma2 || !out->nmatches || !out->match ||
        !out->pose7 || !out->Tcw7 || !out->discarded || !out->nmatchesMap) {
        set_error(std::string(who) + ": bad argument (sizes or null arrays)"); return ORB_ERR_ARG;
    }
    if (in->kcap > m.kcap || in->mcap > m.mcap) { set_error(std::string(who) + ": slabs wider than max_keypoints / max_mappoints"); return ORB_ERR_CAPACITY; }
    return ORB_OK;
}

// Four launches: bow_match_kernel (one CTA per stream; it also writes the gate mask and the copy of nmatches), then launch_gathered in
// MOTION_MODEL mode over the keyframe slabs with the gate mask as its `active`.  Its `claimed` writes go to the search's histogram
// events, which nothing reads after the search, and its nmatches-- to the copy: TrackReferenceKeyFrame returns before reading it.
static int ref_kf_launch(Matcher& m, const OrbmRefKeyFrameBatch* in, const OrbmRefKeyFrameResult* out, cudaStream_t st) {
    int rc = m.track_scratch();
    if (rc) return rc;
    const Matcher::TrackScratch& ts = m.ts;
    BowMatchParams Q; memset(&Q, 0, sizeof(Q));
    Q.nKF = in->kfN; Q.nF = in->nK; Q.eKF = in->kfNEntries; Q.eF = in->nEntries; Q.kfStride = in->mcap; Q.fStride = in->kcap;
    Q.kpsKF = in->kfKps; Q.descKF = in->kfDesc; Q.kfPoint = in->kfPoint; Q.fvNodeKF = in->kfFvNode; Q.fvFeatKF = in->kfFvFeature;
    Q.kpsF = in->kps; Q.descF = in->desc; Q.fvNodeF = in->fvNode; Q.fvFeatF = in->fvFeature;
    Q.nnratio = TRK_REF_NNRATIO; Q.checkOri = 1;
    Q.match = out->match; Q.nmatches = out->nmatches; Q.groupStart = ts.groupStart; Q.evBin = ts.evBin;
    Q.active = in->active; Q.poseActive = ts.poseActive; Q.nmatchesCopy = ts.nmCopy; Q.gate = TRK_REF_MIN_MATCHES;
    bow_match_kernel<<<in->batch, BM_NT, 0, st>>>(Q);
    CK(cudaGetLastError());
    poseopt::GatherArgs A; memset(&A, 0, sizeof(A));
    A.batch = in->batch; A.kcap = in->kcap; A.pstride = in->mcap; A.nlevels = in->nlevels; A.mode = poseopt::MOTION_MODEL;
    A.active = ts.poseActive; A.kps = in->kps; A.nK = in->nK; A.match = out->match; A.claimed = ts.evBin; A.nmatches = ts.nmCopy;
    A.xyz = in->xyz; A.hasObs = in->hasObs; A.invLevelSigma2 = in->invLevelSigma2; memcpy(A.cam, in->cam, 16);
    A.TcwIn = in->Tcw7; A.TcwOut = out->Tcw7; A.poseOut = out->pose7; A.nInliers = ts.nInliers; A.discarded = out->discarded;
    A.nmatchesMap = out->nmatchesMap;
    m.bind_gather(A);
    CK(poseopt::launch_gathered(A, st));
    m.launches = 4;
    return ORB_OK;
}

int orbm_track_reference_keyframe_batch_device(orbm_handle* h, const OrbmRefKeyFrameBatch* in, const OrbmRefKeyFrameResult* out, void* stream) {
    const char* who = "orbm_track_reference_keyframe_batch_device";
    if (!h) { set_error(std::string(who) + ": bad argument"); return ORB_ERR_ARG; }
    if (int rc = ref_kf_shape(h->m, in, out, who)) return rc;
    CK(cudaSetDevice(h->m.device));
    return ref_kf_launch(h->m, in, out, (cudaStream_t)stream);
}

static int ref_kf_host(orbm_handle* h, const OrbmRefKeyFrameBatch* in, const OrbmRefKeyFrameResult* out, bool frameOnDevice) {
    const char* who = frameOnDevice ? "orbm_track_reference_keyframe_batch_resident" : "orbm_track_reference_keyframe_batch";
    if (!h) { set_error(std::string(who) + ": bad argument"); return ORB_ERR_ARG; }
    if (int rc = ref_kf_shape(h->m, in, out, who)) return rc;
    Matcher& m = h->m;
    const size_t B = in->batch, K = in->kcap, M = in->mcap;
    const uint8_t* active = in->active;
    for (size_t b = 0; b < B; ++b) {
        if (active && !active[b]) continue;
        const int nKF = in->kfN[b], eKF = in->kfNEntries[b];
        if (nKF < 0 || nKF > in->mcap || eKF < 0 || eKF > nKF) { set_error(std::string(who) + ": keyframe N or nEntries out of range"); return ORB_ERR_ARG; }
        if (!fv_ok(in->kfFvNode + b * M, in->kfFvFeature + b * M, eKF, nKF)) { set_error(std::string(who) + ": keyframe feature vector not sorted / out of range"); return ORB_ERR_ARG; }
        if (frameOnDevice) continue;
        if (!stream_frame_ok(in, b, who)) return ORB_ERR_ARG;
        const int nF = in->nK[b], eF = in->nEntries[b];
        if (eF < 0 || eF > nF) { set_error(std::string(who) + ": frame nEntries out of range"); return ORB_ERR_ARG; }
        if (!fv_ok(in->fvNode + b * K, in->fvFeature + b * K, eF, nF)) { set_error(std::string(who) + ": frame feature vector not sorted / out of range"); return ORB_ERR_ARG; }
    }
    CK(cudaSetDevice(m.device));
    Staging& S = m.staging;
    S.begin();
    const BatchFrame<OrbmRefKeyFrameBatch> frame(S, in, frameOnDevice);
    const int pT = S.in(in->Tcw7, 28 * B), pKfN = S.in(in->kfN, 4 * B), pKfKps = S.in(in->kfKps, 28 * B * M), pKfDesc = S.in(in->kfDesc, 32 * B * M),
              pKfNode = S.in(in->kfFvNode, 4 * B * M), pKfFeat = S.in(in->kfFvFeature, 4 * B * M), pKfNE = S.in(in->kfNEntries, 4 * B),
              pPt = S.in(in->kfPoint, B * M), pXyz = S.in(in->xyz, 12 * B * M), pObs = S.in(in->hasObs, B * M),
              pIs = S.in(in->invLevelSigma2, 4 * (size_t)in->nlevels), pAct = S.in(active, active ? B : 0),
              pN = S.out(nullptr, 4 * B), pMatch = S.out(nullptr, 4 * B * K), pPose = S.out(nullptr, 56 * B), pTo = S.out(nullptr, 28 * B),
              pDis = S.out(nullptr, B * M), pMap = S.out(nullptr, 4 * B);
    int rc = S.reserve();
    if (rc) return rc;
    OrbmRefKeyFrameBatch d = *in;
    frame.bind(S, d);
    d.Tcw7 = S.dev<float>(pT); d.kfN = S.dev<int>(pKfN); d.kfKps = S.dev<OrbKeyPoint>(pKfKps); d.kfDesc = S.dev(pKfDesc);
    d.kfFvNode = S.dev<int>(pKfNode); d.kfFvFeature = S.dev<int>(pKfFeat); d.kfNEntries = S.dev<int>(pKfNE); d.kfPoint = S.dev(pPt);
    d.xyz = S.dev<float>(pXyz); d.hasObs = S.dev(pObs); d.invLevelSigma2 = S.dev<float>(pIs); d.active = active ? S.dev(pAct) : nullptr;
    OrbmRefKeyFrameResult o = {S.dev<int>(pN), S.dev<int>(pMatch), S.dev<double>(pPose), S.dev<float>(pTo), S.dev(pDis), S.dev<int>(pMap)};
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    if ((rc = ref_kf_launch(m, &d, &o, st))) return rc;
    CK(S.download(st));
    copy_active_rows(S, pN, out->nmatches, 4, in->batch, active);
    copy_active_rows(S, pMatch, out->match, 4 * K, in->batch, active);
    std::vector<uint8_t> gated(B);               // the streams that ran PoseOptimization
    for (size_t b = 0; b < B; ++b) gated[b] = (!active || active[b]) && S.host<int>(pN)[b] >= TRK_REF_MIN_MATCHES;
    copy_active_rows(S, pPose, out->pose7, 56, in->batch, gated.data());
    copy_active_rows(S, pTo, out->Tcw7, 28, in->batch, gated.data());
    copy_active_rows(S, pDis, out->discarded, M, in->batch, gated.data());
    copy_active_rows(S, pMap, out->nmatchesMap, 4, in->batch, gated.data());
    return ORB_OK;
}

int orbm_track_reference_keyframe_batch(orbm_handle* h, const OrbmRefKeyFrameBatch* in, const OrbmRefKeyFrameResult* out) {
    return ref_kf_host(h, in, out, false);
}
int orbm_track_reference_keyframe_batch_resident(orbm_handle* h, const OrbmRefKeyFrameBatch* in, const OrbmRefKeyFrameResult* out) {
    return ref_kf_host(h, in, out, true);
}

// SearchLocalPoints of both local-map calls: tlm_frustum_kernel, then the local-map search (two launches).  Tcw7: the frame's pose.
static int search_local_points_launch(Matcher& m, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out, const float* Tcw7, const uint8_t* active,
                                      cudaStream_t st) {
    const Matcher::TrackScratch& ts = m.ts;
    TrackLocalParams T; memset(&T, 0, sizeof(T));
    T.batch = in->batch; T.kcap = in->kcap; T.mcap = in->mcap; T.mcapLast = in->lastToLocal ? in->mcapLast : 0;
    T.active = active; T.nK = in->nK; T.nM = in->nM; T.match = out->match; T.claimed = out->claimed;
    T.lastToLocal = in->lastToLocal; T.discarded = in->discarded; T.Tcw7 = Tcw7;
    T.F.P = in->worldPos; T.F.N = in->normal; T.F.minD = in->minDistInv; T.F.maxD = in->maxDistInv; T.F.maxRaw = in->maxDistance;
    memcpy(T.F.cam, in->cam, 16);
    T.F.minX = in->minX; T.F.minY = in->minY; T.F.maxX = in->maxX; T.F.maxY = in->maxY; T.F.mbf = in->mbf; T.F.logSF = in->logScaleFactor;
    T.F.cosLimit = in->viewingCosLimit; T.F.nLevels = in->nlevels;
    T.bad = in->bad; T.hasObs = in->hasObs;
    T.seen = ts.seen; T.inView = ts.inView; T.projX = ts.projX; T.projY = ts.projY; T.depth = ts.depth; T.viewCos = ts.viewCos; T.level = ts.level;
    T.visible = out->visible; T.found = out->found; T.nToMatch = out->nToMatch;
    tlm_frustum_kernel<<<in->batch, TL_NT, 0, st>>>(T);
    CK(cudaGetLastError());
    MatchParams P; memset(&P, 0, sizeof(P));
    P.batch = in->batch; P.kcap = in->kcap; P.mcap = in->mcap; P.nlevels = in->nlevels; P.mode = 0;
    P.kps = in->kps; P.desc = in->desc; P.nK = in->nK;
    P.minX = in->minX; P.minY = in->minY; P.maxX = in->maxX; P.maxY = in->maxY;
    P.scaleFactors = in->scaleFactors; P.nM = in->nM;
    P.inView = ts.inView; P.bad = in->bad; P.depth = ts.depth; P.projX = ts.projX; P.projY = ts.projY; P.level = ts.level; P.viewCos = ts.viewCos;
    P.hasObs = in->hasObs; P.mpDesc = in->mpDesc;
    P.th = 1.0f; P.thBatch = in->th; P.nnratio = in->nnratio; P.bFar = in->bFarPoints; P.thFar = in->thFarPoints; P.active = active;
    P.match = out->match; P.claimed = out->claimed; P.nmatches = out->nmatches;
    return m.run(P, in->kcap, in->mcap, st);
}

static int track_local_map_launch(Matcher& m, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out, cudaStream_t st) {
    int rc = m.track_scratch();
    if (rc) return rc;
    if ((rc = search_local_points_launch(m, in, out, in->Tcw7, in->active, st))) return rc;
    poseopt::GatherArgs A; memset(&A, 0, sizeof(A));
    A.batch = in->batch; A.kcap = in->kcap; A.pstride = in->mcap; A.nlevels = in->nlevels; A.mode = poseopt::LOCAL_MAP;
    A.active = in->active; A.kps = in->kps; A.nK = in->nK; A.match = out->match; A.claimed = out->claimed;
    A.xyz = in->worldPos; A.hasObs = in->hasObs; A.invLevelSigma2 = in->invLevelSigma2; memcpy(A.cam, in->cam, 16);
    A.TcwIn = in->Tcw7; A.TcwOut = out->Tcw7; A.poseOut = out->pose7; A.nInliers = out->nInliers;
    A.outlierKp = out->outlier; A.found = out->found; A.nMatchesInliers = out->nMatchesInliers;
    m.bind_gather(A);
    CK(poseopt::launch_gathered(A, st));
    m.launches = 5;
    return ORB_OK;
}

// Argument checks shared by the three forms that need no host-side data.  ORB_ERR_CAPACITY for a slab wider than the handle's capacities.
// inertial: the mono-inertial call's form, where the pose is predicted and the frame holds nothing (Tcw7, lastToLocal, discarded,
// active and pose7 must be NULL).
static int local_map_shape(const Matcher& m, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out, const char* who, bool inertial = false) {
    if (!in || !out || !batch_shape_ok(m, in->batch, in->kcap, in->mcap, in->nlevels) || (in->lastToLocal && in->mcapLast < 1) || !in->kps ||
        !in->desc || !in->nK || !in->scaleFactors || !in->invLevelSigma2 || (!in->Tcw7 != inertial) || !in->nM || !in->worldPos || !in->normal ||
        !in->minDistInv || !in->maxDistInv || !in->maxDistance || !in->mpDesc || !in->hasObs || !in->bad || !in->th || !(in->maxX > in->minX) ||
        !(in->maxY > in->minY) || !out->match || !out->claimed || !out->outlier || !out->visible || !out->found || !out->nToMatch ||
        !out->nmatches || !out->nInliers || !out->nMatchesInliers || (!out->pose7 != inertial) || !out->Tcw7 ||
        (inertial && (in->lastToLocal || in->discarded || in->active))) {
        set_error(std::string(who) + ": bad argument (sizes or null arrays)"); return ORB_ERR_ARG;
    }
    if (in->mcap > m.mcap) { set_error(std::string(who) + ": more local map points than max_mappoints"); return ORB_ERR_CAPACITY; }
    if (frame_smem_bytes(in->kcap, in->mcap, false) > FRAME_SMEM_LIMIT) { set_error(std::string(who) + ": frame too large for the matcher's shared-memory grid"); return ORB_ERR_CAPACITY; }
    return ORB_OK;
}

int orbm_track_local_map_batch_device(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out, void* stream) {
    if (!h) { set_error("orbm_track_local_map_batch_device: bad argument"); return ORB_ERR_ARG; }
    if (int rc = local_map_shape(h->m, in, out, "orbm_track_local_map_batch_device")) return rc;
    CK(cudaSetDevice(h->m.device));
    return track_local_map_launch(h->m, in, out, (cudaStream_t)stream);
}

// One stream of a host form of either local-map call: nM in [0, mcap], a positive th and, unless the call is resident, the current frame.
static bool local_map_stream_ok(const OrbmLocalMapBatch* in, size_t b, bool frameOnDevice, const char* who) {
    if (in->nM[b] < 0 || in->nM[b] > in->mcap) { set_error(std::string(who) + ": nM out of range"); return false; }
    if (!(in->th[b] > 0.0f)) { set_error(std::string(who) + ": th must be positive"); return false; }
    return frameOnDevice || stream_frame_ok(in, b, who);
}

// The staging of what the host forms of both local-map calls share: the current frame, the local map and the results of
// OrbmLocalMapResult.  Tcw7, lastToLocal, discarded and pose7 are staged when the caller gives them (the mono-inertial call predicts the
// pose and gives none of them); match goes in and out when matchIn (TrackLocalMap remaps it), else only out.
struct LocalMapPieces {
    BatchFrame<OrbmLocalMapBatch> frame;
    bool matchIn;
    int sf, is, T, l2l, dis, nM, wp, no, minD, maxD, raw, md, obs, bad, th, match, cl, outl, vis, found, counts, pose, to;

    LocalMapPieces(Staging& S, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out, bool frameOnDevice, bool matchIn)
        : frame(S, in, frameOnDevice), matchIn(matchIn) {
        const size_t B = in->batch, K = in->kcap, M = in->mcap, ML = in->lastToLocal ? in->mcapLast : 0;
        const size_t DL = in->discarded ? (in->lastToLocal ? ML : M) : 0;
        sf = S.in(in->scaleFactors, 4 * (size_t)in->nlevels); is = S.in(in->invLevelSigma2, 4 * (size_t)in->nlevels);
        T = S.in(in->Tcw7, in->Tcw7 ? 28 * B : 0); l2l = S.in(in->lastToLocal, 4 * B * ML); dis = S.in(in->discarded, B * DL);
        nM = S.in(in->nM, 4 * B); wp = S.in(in->worldPos, 12 * B * M); no = S.in(in->normal, 12 * B * M);
        minD = S.in(in->minDistInv, 4 * B * M); maxD = S.in(in->maxDistInv, 4 * B * M); raw = S.in(in->maxDistance, 4 * B * M);
        md = S.in(in->mpDesc, 32 * B * M); obs = S.in(in->hasObs, B * M); bad = S.in(in->bad, B * M); th = S.in(in->th, 4 * B);
        match = matchIn ? S.inout(out->match, 4 * B * K) : S.out(nullptr, 4 * B * K);
        cl = S.out(nullptr, B * K); outl = S.out(nullptr, B * K); vis = S.out(nullptr, 4 * B * M); found = S.out(nullptr, 4 * B * M);
        counts = S.out(nullptr, 16 * B); pose = S.out(nullptr, out->pose7 ? 56 * B : 0); to = S.out(nullptr, 28 * B);
    }

    // Points `d` and `o`, copies of the caller's batch and result, at the pieces.  The staging is reserved.
    void bind(const Staging& S, OrbmLocalMapBatch& d, OrbmLocalMapResult& o) const {
        frame.bind(S, d);
        d.scaleFactors = S.dev<float>(sf); d.invLevelSigma2 = S.dev<float>(is); d.Tcw7 = d.Tcw7 ? S.dev<float>(T) : nullptr;
        d.lastToLocal = d.lastToLocal ? S.dev<int>(l2l) : nullptr; d.discarded = d.discarded ? S.dev(dis) : nullptr; d.nM = S.dev<int>(nM);
        d.worldPos = S.dev<float>(wp); d.normal = S.dev<float>(no); d.minDistInv = S.dev<float>(minD); d.maxDistInv = S.dev<float>(maxD);
        d.maxDistance = S.dev<float>(raw); d.mpDesc = S.dev(md); d.hasObs = S.dev(obs); d.bad = S.dev(bad); d.th = S.dev<float>(th);
        const size_t B = d.batch;
        int* c = S.dev<int>(counts);      // nToMatch | nmatches | nInliers | nMatchesInliers, [B] each
        o = {S.dev<int>(match), S.dev(cl), S.dev(outl), S.dev<int>(vis), S.dev<int>(found), c, c + B, c + 2 * B, c + 3 * B,
             o.pose7 ? S.dev<double>(pose) : nullptr, S.dev<float>(to)};
    }

    // After the download: the rows of the active streams to the caller's `out` (an in / out match is already back whole).
    void copy_back(const Staging& S, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out, const uint8_t* active) const {
        const size_t B = in->batch, K = in->kcap, M = in->mcap;
        if (!matchIn) copy_active_rows(S, match, out->match, 4 * K, in->batch, active);
        copy_active_rows(S, cl, out->claimed, K, in->batch, active);
        copy_active_rows(S, outl, out->outlier, K, in->batch, active);
        copy_active_rows(S, vis, out->visible, 4 * M, in->batch, active);
        copy_active_rows(S, found, out->found, 4 * M, in->batch, active);
        copy_active_rows(S, pose, out->pose7, 56, in->batch, active);
        copy_active_rows(S, to, out->Tcw7, 28, in->batch, active);
        const int* hc = S.host<int>(counts);
        int32_t* dst[4] = {out->nToMatch, out->nmatches, out->nInliers, out->nMatchesInliers};
        for (size_t b = 0; b < B; ++b)
            if (!active || active[b]) for (int k = 0; k < 4; ++k) dst[k][b] = hc[k * B + b];
    }
};

static int track_local_map_host(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out, bool frameOnDevice) {
    const char* who = frameOnDevice ? "orbm_track_local_map_batch_resident" : "orbm_track_local_map_batch";
    if (!h) { set_error(std::string(who) + ": bad argument"); return ORB_ERR_ARG; }
    if (int rc = local_map_shape(h->m, in, out, who)) return rc;
    Matcher& m = h->m;
    const size_t B = in->batch, K = in->kcap, ML = in->lastToLocal ? in->mcapLast : 0;
    const uint8_t* active = in->active;
    for (size_t b = 0; b < B; ++b) {
        if (active && !active[b]) continue;
        if (!local_map_stream_ok(in, b, frameOnDevice, who)) return ORB_ERR_ARG;
        for (size_t i = 0; i < K; ++i) {
            const int mt = out->match[b * K + i];
            if (mt < -1 || mt >= (in->lastToLocal ? in->mcapLast : in->mcap)) { set_error(std::string(who) + ": match index out of range"); return ORB_ERR_ARG; }
        }
        for (size_t j = 0; j < ML; ++j)
            if (in->lastToLocal[b * ML + j] < -1 || in->lastToLocal[b * ML + j] >= in->nM[b]) { set_error(std::string(who) + ": lastToLocal index out of range"); return ORB_ERR_ARG; }
    }
    CK(cudaSetDevice(m.device));
    Staging& S = m.staging;
    S.begin();
    const LocalMapPieces lm(S, in, out, frameOnDevice, true);
    const int pAct = S.in(active, active ? B : 0);
    int rc = S.reserve();
    if (rc) return rc;
    OrbmLocalMapBatch d = *in;
    OrbmLocalMapResult o = *out;
    lm.bind(S, d, o);
    d.active = active ? S.dev(pAct) : nullptr;
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    if ((rc = track_local_map_launch(m, &d, &o, st))) return rc;
    CK(S.download(st));
    lm.copy_back(S, in, out, active);
    return ORB_OK;
}

int orbm_track_local_map_batch(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out) {
    return track_local_map_host(h, in, out, false);
}
int orbm_track_local_map_batch_resident(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmLocalMapResult* out) {
    return track_local_map_host(h, in, out, true);
}

// ---- TrackLocalMap on the mono-inertial path, after PredictStateIMU, for a batch of streams (include/orb_b200.h) ----
// From the host's mode array: each stream's slot (route; -1 = skipped), the map-updated streams first and the others after them, each
// in stream order, and the device mask of the frustum and search stages.  Also the argument checks of the IMU operands.
struct InertialRoutes {
    std::vector<int> route; std::vector<uint8_t> active; int count[2] = {0, 0};
};
static int inertial_routes(const Matcher& m, const OrbmLocalMapBatch* in, const OrbmImuTrackBatch* imu, const OrbmLocalMapResult* out,
                           const OrbmImuTrackResult* io, InertialRoutes& R, const char* who) {
    if (int rc = local_map_shape(m, in, out, who, true)) return rc;
    if (!imu || !io || !imu->mode || !imu->extrinsics24 || !imu->preintKF || !io->predState21 || !io->predTcw7 || !io->state21 || !io->prior21 || !io->priorH) {
        set_error(std::string(who) + ": bad argument (null IMU arrays)"); return ORB_ERR_ARG;
    }
    R.route.assign(in->batch, -1); R.active.assign(in->batch, 0);
    for (int b = 0; b < in->batch; ++b) {
        if (imu->mode[b] > 2) { set_error(std::string(who) + ": mode must be 0, 1 or 2"); return ORB_ERR_ARG; }
        if (imu->mode[b]) ++R.count[imu->mode[b] - 1];
    }
    if ((R.count[0] && !imu->kfState21) || (R.count[1] && (!imu->preintFrame || !imu->lastState21 || !imu->prior21 || !imu->priorH))) {
        set_error(std::string(who) + ": a stream's mode needs an IMU array that is null"); return ORB_ERR_ARG;
    }
    int next[2] = {0, R.count[0]};
    for (int b = 0; b < in->batch; ++b)
        if (imu->mode[b]) { R.route[b] = next[imu->mode[b] - 1]++; R.active[b] = 1; }
    return ORB_OK;
}

// Predict (1 launch), SearchLocalPoints (2), gather + optimisers + write-back (2 + one per variant with streams).
static int track_inertial_launch(Matcher& m, const OrbmLocalMapBatch* in, const OrbmImuTrackBatch* imu, const OrbmLocalMapResult* out,
                                 const OrbmImuTrackResult* io, const int* d_route, const uint8_t* d_active, const int count[2], cudaStream_t st) {
    const Matcher::TrackScratch& ts = m.ts;
    imu::ImuTrackArgs A; memset(&A, 0, sizeof(A));
    A.batch = in->batch; A.kcap = in->kcap; A.pstride = in->mcap; A.nlevels = in->nlevels; A.count[0] = count[0]; A.count[1] = count[1];
    A.route = d_route; memcpy(A.Tcb7, imu->Tcb7, sizeof(A.Tcb7)); A.extr = imu->extrinsics24;
    A.preintKF = imu->preintKF; A.preintFrame = imu->preintFrame; A.kfState21 = imu->kfState21; A.lastState21 = imu->lastState21;
    A.priorIn = imu->prior21; A.priorHIn = imu->priorH;
    A.predState21 = io->predState21; A.predTcw7 = io->predTcw7; A.match = out->match;
    A.kps = in->kps; A.nK = in->nK; A.xyz = in->worldPos; A.hasObs = in->hasObs; A.depth = ts.depth; A.invLevelSigma2 = in->invLevelSigma2;
    memcpy(A.cam, in->cam, 16);
    A.outlierKp = out->outlier; A.found = out->found; A.nInliers = out->nInliers; A.nMatchesInliers = out->nMatchesInliers;
    A.Tcw7 = out->Tcw7; A.state21 = io->state21; A.priorOut = io->prior21; A.priorHOut = io->priorH;
    A.Xw = ts.iXw; A.obs = ts.iObs; A.invSigma2 = ts.is2; A.trackDepth = ts.iTd; A.edgeKp = ts.edgeKp; A.err = ts.err; A.outlier = ts.outl;
    A.N = ts.N; A.cam4 = ts.cam4; A.preint = ts.preint; A.preintKF2 = ts.preintKF2; A.fixedState = ts.fixedState; A.state = ts.state;
    A.prior = ts.prior; A.priorH = ts.priorH; A.H15 = ts.H15; A.ret = ts.ret;
    m.launches = 0;
    if (!count[0] && !count[1]) return ORB_OK;           // every stream skipped
    CK(imu::launch_predict_imu(A, st));
    if (int rc = search_local_points_launch(m, in, out, io->predTcw7, d_active, st)) return rc;
    int n = 0;
    CK(imu::launch_gathered_inertial(A, st, &n));
    m.launches = 3 + n;
    return ORB_OK;
}

int orbm_track_local_map_inertial_batch_device(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmImuTrackBatch* imu,
                                               const OrbmLocalMapResult* out, const OrbmImuTrackResult* imuOut, void* stream) {
    const char* who = "orbm_track_local_map_inertial_batch_device";
    if (!h) { set_error(std::string(who) + ": bad argument"); return ORB_ERR_ARG; }
    Matcher& m = h->m;
    InertialRoutes R;
    if (int rc = inertial_routes(m, in, imu, out, imuOut, R, who)) return rc;
    CK(cudaSetDevice(m.device));
    if (int rc = m.track_scratch()) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    // the route / active tables go through the handle's pinned mirror, so the copy is asynchronous; before the mirror is rewritten the
    // call waits for the previous call's copy of it (an event, normally long complete), not for the caller's stream
    const size_t B = in->batch, MB = m.maxBatch;
    if (!m.h_route) {
        CK(cudaMallocHost(&m.h_route, 5 * MB));
        CK(cudaEventCreateWithFlags(&m.evRoute, cudaEventDisableTiming));
    } else {
        CK(cudaEventSynchronize(m.evRoute));
    }
    memcpy(m.h_route, R.route.data(), 4 * B);
    memcpy(m.h_route + 4 * MB, R.active.data(), B);
    CK(cudaMemcpyAsync(m.ts.route, m.h_route, 4 * B, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(m.ts.active, m.h_route + 4 * MB, B, cudaMemcpyHostToDevice, st));
    CK(cudaEventRecord(m.evRoute, st));
    return track_inertial_launch(m, in, imu, out, imuOut, m.ts.route, m.ts.active, R.count, st);
}

static int track_inertial_host(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmImuTrackBatch* imu, const OrbmLocalMapResult* out,
                               const OrbmImuTrackResult* io, bool frameOnDevice) {
    const char* who = frameOnDevice ? "orbm_track_local_map_inertial_batch_resident" : "orbm_track_local_map_inertial_batch";
    if (!h) { set_error(std::string(who) + ": bad argument"); return ORB_ERR_ARG; }
    Matcher& m = h->m;
    InertialRoutes R;
    if (int rc = inertial_routes(m, in, imu, out, io, R, who)) return rc;
    const size_t B = in->batch, PS = 4 * IMU_PREINT_FLOATS;
    const uint8_t* active = R.active.data();
    for (size_t b = 0; b < B; ++b)
        if (active[b] && !local_map_stream_ok(in, b, frameOnDevice, who)) return ORB_ERR_ARG;
    CK(cudaSetDevice(m.device));
    if (int rc = m.track_scratch()) return rc;
    Staging& S = m.staging;
    S.begin();
    const bool lf = R.count[1] > 0, kf = R.count[0] > 0;
    const LocalMapPieces lm(S, in, out, frameOnDevice, false);
    const int pRoute = S.in(R.route.data(), 4 * B), pAct = S.in(active, B), pEx = S.in(imu->extrinsics24, 192),
              pPk = S.in(imu->preintKF, PS * B), pPf = S.in(lf ? imu->preintFrame : nullptr, lf ? PS * B : 0),
              pKs = S.in(kf ? imu->kfState21 : nullptr, kf ? 84 * B : 0), pLs = S.in(lf ? imu->lastState21 : nullptr, lf ? 84 * B : 0),
              pPr = S.in(lf ? imu->prior21 : nullptr, lf ? 168 * B : 0), pPh = S.in(lf ? imu->priorH : nullptr, lf ? 1800 * B : 0),
              pPs = S.out(nullptr, 84 * B), pPt = S.out(nullptr, 28 * B), pSt = S.out(nullptr, 84 * B), pPo = S.out(nullptr, 168 * B),
              pHo = S.out(nullptr, 1800 * B);
    int rc = S.reserve();
    if (rc) return rc;
    OrbmLocalMapBatch d = *in;
    OrbmLocalMapResult o = *out;
    lm.bind(S, d, o);
    OrbmImuTrackBatch di = *imu;
    di.extrinsics24 = S.dev<double>(pEx); di.preintKF = S.dev<float>(pPk); di.preintFrame = lf ? S.dev<float>(pPf) : nullptr;
    di.kfState21 = kf ? S.dev<float>(pKs) : nullptr; di.lastState21 = lf ? S.dev<float>(pLs) : nullptr;
    di.prior21 = lf ? S.dev<double>(pPr) : nullptr; di.priorH = lf ? S.dev<double>(pPh) : nullptr;
    OrbmImuTrackResult io2 = {S.dev<float>(pPs), S.dev<float>(pPt), S.dev<float>(pSt), S.dev<double>(pPo), S.dev<double>(pHo)};
    cudaStream_t st = m.stream;
    CK(S.upload(st));
    if ((rc = track_inertial_launch(m, &d, &di, &o, &io2, S.dev<int>(pRoute), S.dev(pAct), R.count, st))) return rc;
    CK(S.download(st));
    lm.copy_back(S, in, out, active);
    copy_active_rows(S, pPs, io->predState21, 84, in->batch, active);
    copy_active_rows(S, pPt, io->predTcw7, 28, in->batch, active);
    copy_active_rows(S, pSt, io->state21, 84, in->batch, active);
    copy_active_rows(S, pPo, io->prior21, 168, in->batch, active);
    copy_active_rows(S, pHo, io->priorH, 1800, in->batch, active);
    return ORB_OK;
}

int orbm_track_local_map_inertial_batch(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmImuTrackBatch* imu, const OrbmLocalMapResult* out,
                                        const OrbmImuTrackResult* imuOut) {
    return track_inertial_host(h, in, imu, out, imuOut, false);
}
int orbm_track_local_map_inertial_batch_resident(orbm_handle* h, const OrbmLocalMapBatch* in, const OrbmImuTrackBatch* imu,
                                                 const OrbmLocalMapResult* out, const OrbmImuTrackResult* imuOut) {
    return track_inertial_host(h, in, imu, out, imuOut, true);
}

}  // extern "C"
