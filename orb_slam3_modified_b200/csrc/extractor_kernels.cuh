// Hand-written sm_90a kernels of the batched ORB extractor.  Every kernel carries a
// batch (frame) dimension in blockIdx.y / blockIdx.z so that one launch covers all streams.
//
// Reference semantics (file:line in the reference checkout) are cited per kernel; the
// bit-exact scalar pieces live in exact_math.h.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "exact_math.h"
#include "device_utils.cuh"
#include "extractor_types.h"

namespace orbx {

__constant__ int8_t c_pattern[1024];      // 256 pairs x (x0,y0,x1,y1), reference src/ORBextractor.cc:149-407
__constant__ int c_umax[HALF_PATCH + 1];  // :453-468

// ------------------------------------------------------------------------------------------
// plane addressing: level 0 may alias the caller's image
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ const uint8_t* plane_ptr(const ExtractParams& P, int f, int l, int& pitch) {
    if (l == 0) { pitch = (int)P.lv0Pitch; return P.lv0 + (size_t)f * P.lv0FrameStride; }
    pitch = P.lv[l].pitch;
    return P.pyr + (size_t)f * P.pyrFrameStride + P.lv[l].planeOff;
}
__device__ __forceinline__ const uint8_t* blur_ptr(const ExtractParams& P, int f, int l, int& pitch) {
    pitch = P.lv[l].pitch;
    return P.blur + (size_t)f * P.pyrFrameStride + P.lv[l].planeOff;
}

// ------------------------------------------------------------------------------------------
// K0: copy the caller's image into the level-0 plane (only when level 0 cannot alias it).
// ------------------------------------------------------------------------------------------
__global__ void copy_level0_kernel(ExtractParams P) {
    const int f = blockIdx.z;
    const int y = blockIdx.y;
    const uint8_t* s = P.src + (size_t)f * P.srcFrameStride + (size_t)y * P.srcStep;
    uint8_t* d = P.pyr + (size_t)f * P.pyrFrameStride + P.lv[0].planeOff + (size_t)y * P.lv[0].pitch;
    for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < P.cols; x += gridDim.x * blockDim.x) d[x] = s[x];
}

// ------------------------------------------------------------------------------------------
// K1: pyramid level l from level l-1.  cv::resize(INTER_LINEAR) restated in integer
// fixed point (SURVEY.md 9C; reference call site src/ORBextractor.cc:1183).  Each thread
// produces 4 horizontally adjacent pixels and stores them as one 32-bit word.
// The 19-px reflected border the reference also writes (:1185-1191) is never read on this
// path (SURVEY.md 8a reach analysis) and is not materialised.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pyr_resize_kernel(ExtractParams P, int l) {
    const LevelGeom& G = P.lv[l];
    const int f = blockIdx.z;
    const int dy = blockIdx.y * blockDim.y + threadIdx.y;
    const int dx0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (dy >= G.h || dx0 >= G.w) return;
    int spitch;
    const uint8_t* src = plane_ptr(P, f, l - 1, spitch);
    uint8_t* dst = P.pyr + (size_t)f * P.pyrFrameStride + G.planeOff + (size_t)dy * G.pitch;
    uint32_t out = 0;
    if (G.area2x) {
        const uint8_t* r0 = src + (size_t)(2 * dy) * spitch;
        const uint8_t* r1 = r0 + spitch;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int dx = dx0 + k;
            if (dx < G.w) {
                int v = (r0[2 * dx] + r0[2 * dx + 1] + r1[2 * dx] + r1[2 * dx + 1] + 2) >> 2;
                out |= (uint32_t)v << (8 * k);
            }
        }
    } else {
        const short4 yt = P.ytab[G.ytabOff + dy];  // {sy0, sy1, b0, b1}
        const uint8_t* r0 = src + (size_t)yt.x * spitch;
        const uint8_t* r1 = src + (size_t)yt.y * spitch;
        const int b0 = yt.z, b1 = yt.w;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int dx = dx0 + k;
            if (dx < G.w) {
                const short4 xt = __ldg(&P.xtab[G.xtabOff + dx]);  // {sx0, sx1, a0, a1}
                const int s0 = r0[xt.x] * xt.z + r0[xt.y] * xt.w;
                const int s1 = r1[xt.x] * xt.z + r1[xt.y] * xt.w;
                const int v = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
                out |= (uint32_t)(v & 0xFF) << (8 * k);
            }
        }
    }
    *reinterpret_cast<uint32_t*>(dst + dx0) = out;   // pitch is a multiple of 32: in-bounds even for the tail
}

// ------------------------------------------------------------------------------------------
// K2: FAST-9/16 per cell with the two-threshold fallback and cell-local NMS.
// Reference: ORBextractor::ComputeKeyPointsOctTree src/ORBextractor.cc:805-873 calling
// cv::FAST(cellROI, th, nonmax=true) (SURVEY.md 9D).  One CTA per (block of up to 2 x 2 cells, frame).
//   score = max over the 16 nine-pixel arcs of max(min(v-p), min(p-v)) - 1; corner at T <=> score >= T;
//   NMS: strict 8-neighbour maximum, neighbours outside the cell's own ROI interior count as 0.
// A strict local maximum of the th=minTh score map with score >= T is exactly what
// cv::FAST(T) keeps, so one score map serves both passes.
// A pixel's score does not depend on the cell that reads it and the cell interiors tile the level, so the quick test and the
// exact score run once over the union of the block's interiors; NMS, the fallback and the emission stay per cell.
// Output: per cell a count and a row-major (y, x) list of packed (x+offX, y+offY, score).
// ------------------------------------------------------------------------------------------
// Threads per (block, frame) CTA: 64 per cell of a 2 x 2 block.  Measured per 240 frames of 640x480 on an H100 80GB HBM3 at 700 W:
// 0.88 ms with the quick test's row runs of 6 (0.92 ms with a thread per quad, 1.05 ms for the former 64-thread CTA per cell).
// ptxas: 64 registers (the launch bound asks for 4 CTAs per SM; unbounded, the row window takes 94), no spills; ~28 KB of dynamic
// shared memory at 640x480, so registers cap an SM at 4 CTAs (32 warps).  Capping the per-quad form at 48 registers for 5 CTAs measured 0.92 ms.
constexpr int FAST_NT = 256;
// Interior rows per thread in the quick test (phase 1): a run's candidates travel as one 32-bit mask, 4 pixels per row.  Measured per
// 240 frames as above: runs of 4 / 6 / 8 rows 0.890 / 0.873 / 0.891 ms (at 6, the 18 quads x 13 runs of a level-0 block fill 234 of
// the 256 threads in one pass).
#ifndef FAST_RUN
#define FAST_RUN 6
#endif
static_assert(FAST_RUN >= 1 && FAST_RUN <= 8, "a run's candidate mask is 4 * FAST_RUN bits of one word");

__device__ __forceinline__ int fast_score_at(const uint8_t* t, const int* off) {
    // d_k = v - p_k (darker ring), e_k = p_k - v (brighter ring) for the 16 ring pixels.
    // NOTE: both polarities are written as min-trees over separately subtracted arrays on purpose.
    // The shorter form max(min9(d), -max9(d)) is miscompiled by ptxas 12.9 for sm_100a (the negation is
    // dropped when it is folded into a VIMNMX3 operand); see DESIGN.md "toolchain findings".
    const int v = t[0];
    int d[16], e[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) { const int p = t[off[k]]; d[k] = v - p; e[k] = p - v; }
    // min over every window of 9 consecutive (cyclic) ring positions via two levels of 3-input minima
    int a3[16], b3[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        a3[k] = min(d[k], min(d[(k + 1) & 15], d[(k + 2) & 15]));
        b3[k] = min(e[k], min(e[(k + 1) & 15], e[(k + 2) & 15]));
    }
    int best = -512;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        const int a9 = min(a3[k], min(a3[(k + 3) & 15], a3[(k + 6) & 15]));
        const int b9 = min(b3[k], min(b3[(k + 3) & 15], b3[(k + 6) & 15]));
        best = max(best, max(a9, b9));
    }
    return best;  // corner at T <=> best > T, score = best - 1
}

// TMA descriptors: one 3-D tensor {x, y, frame} per pyramid level.  Levels >= 1 live in a global-memory table; level 0 (which
// may alias the caller's frames and so changes per call) travels as a __grid_constant__ kernel parameter.
struct alignas(64) TmaMaps { CUtensorMap lv[kMaxLevels]; };

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tWAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// cp.async.bulk.tensor (TMA) 3-D tile load: box {bw, bh, 1} at (x, y, frame) -> shared memory, completion on an mbarrier
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int x, int y, int z, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar)) : "memory");
}

// bits of bitmap word w that lie in columns [x0, x1)
__device__ __forceinline__ uint32_t fast_col_mask(int w, int x0, int x1) {
    const int lo = max(x0 - (w << 5), 0), hi = min(x1 - (w << 5), 32);
    return (hi >= 32 ? 0xFFFFFFFFu : (1u << hi) - 1u) & (0xFFFFFFFFu << lo);
}

__global__ void __launch_bounds__(FAST_NT, 4) fast_cells_kernel(ExtractParams P, const __grid_constant__ CUtensorMap map0, const CUtensorMap* __restrict__ maps) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ int s_nCand, s_warp[33];
    __shared__ int4 s_rect[4];        // per cell: interior [x, z) x [y, w) in union-interior coordinates
    __shared__ int4 s_out[4];         // per cell: listOff, offX, offY
    __shared__ int s_rowBase[5];      // first (cell, row) entry of every cell; [ncell] = number of entries
    __shared__ int s_hasHi[4];        // the cell keeps a corner at iniTh
    const int f = blockIdx.y;
    const FastBlock& bk = P.fastBlocks[blockIdx.x];
    const int ncx = bk.ncx, ncell = ncx * bk.ncy;
    const int iw = bk.iw, ih = bk.ih;
    const int tid = threadIdx.x, lane = tid & 31;
    int* outCount = P.cellCount + (size_t)f * P.cellCountStride;
    if (iw == 0) { if (tid < ncell) outCount[bk.cell[tid]] = 0; return; }
    const LevelGeom& G = P.lv[bk.level];
    const int tp = G.fastBoxW;                  // tile pitch = TMA box width (multiple of 16)
    const FastSmem L = fast_smem_layout(tp, G.fastBoxH, iw, ih);
    const int sp = L.sp, nwp = L.nwp;
    // TMA tile mode needs a 16-byte aligned box start (unaligned inner coordinates fault: measured, see DESIGN.md), so the box
    // starts at x0 & ~15 and the window begins `xoff` bytes into every tile row
    const int xoff = bk.x0 & 15;
    uint8_t* tileBase = smem_raw;                                               // fastBoxH * tp, 128-byte aligned
    const uint8_t* tile = tileBase + xoff;
    uint8_t* score = smem_raw + L.score;
    uint32_t* bitsLo = reinterpret_cast<uint32_t*>(smem_raw + L.bits);         // per-row keep bitmaps at minTh / iniTh
    uint32_t* bitsHi = bitsLo + ih * nwp;
    int* rowOff = reinterpret_cast<int*>(smem_raw + L.rowOff);
    uint16_t* list = reinterpret_cast<uint16_t*>(smem_raw + L.list);

    // ---- tile: one TMA bulk-tensor load of the whole window (image pyramid staged into shared memory) ----
    if (tid == 0) {
        mbar_init(&s_bar, 1);
        mbar_expect_tx(&s_bar, (uint32_t)(tp * G.fastBoxH));
        tma_load_3d(tileBase, bk.level == 0 ? &map0 : maps + bk.level, bk.x0 - xoff, bk.y0, f, &s_bar);
        s_nCand = 0;
    }
    if (tid < ncell) {
        const CellDesc cd = P.cells[bk.cell[tid]];
        const int x = cd.x0 - bk.x0, y = cd.y0 - bk.y0;
        s_rect[tid] = make_int4(x, y, x + max(cd.rw - 6, 0), y + max(cd.rh - 6, 0));
        s_out[tid] = make_int4((int)cd.listOff, cd.offX, cd.offY, 0);
        s_hasHi[tid] = 0;
    }
    for (int i = tid; i < 2 * ih * nwp; i += FAST_NT) bitsLo[i] = 0;
    __syncthreads();                                            // barrier init + cell rects visible, bitmaps cleared
    if (tid == 0) {
        s_rowBase[0] = 0;
        for (int k = 0; k < ncell; ++k) s_rowBase[k + 1] = s_rowBase[k] + s_rect[k].w - s_rect[k].y;
    }
    mbar_wait(&s_bar, 0);

    // phase 1: cheap rejection (any 9-arc contains ring pixel k or k+8 for every k) + compaction of the survivors.
    // One thread owns a run of FAST_RUN interior rows of one quad column (four horizontally adjacent pixels).  It walks the run
    // down a sliding window of tile rows: every tile row of the run (and its 3-row ring margins) is loaded and funnel-shifted once,
    // into the five 4-pixel windows the ring reads from it, instead of once per quad that reads it.  Rows y +- 1 are never read.
    // Pixels travel in pairs as 2 x 16-bit lanes so that one VIADD.16x2 / LOP3 serves two pixels: with NLO = T - v and
    // NHI1 = -(v + T + 1) per lane,
    //   p < v - T  <=>  sign(p + NLO) set,      p > v + T  <=>  sign(p + NHI1) clear.
    const int th = P.minTh;
    {
        const int nq = (iw + 3) >> 2, nI = nq * ((ih + FAST_RUN - 1) / FAST_RUN);
        const unsigned qmagic = 0xFFFFFFFFu / (unsigned)nq + 1u;
        const uint32_t TT = (uint32_t)th * 0x10001u, TT1 = (uint32_t)(th + 1) * 0x10001u;
        const int shC = ((xoff) & 3) * 8;            // byte phase of column (4q + xoff) inside an aligned word
        const int tpw = tp >> 2;
        for (int base = 0; base < nI; base += FAST_NT) {
            // consecutive lanes take consecutive quads of one run, so the lanes of a run read consecutive words of a tile row
            const int it = base + tid;
            uint32_t cand = 0;                       // bit 4k + i: pixel (y0 + k, 4q + i) survives
            int y0 = 0, q = 0;
            if (it < nI) {
                const int j = (int)__umulhi((unsigned)it, qmagic);
                q = it - j * nq; y0 = j * FAST_RUN;
                // aligned word of tile byte (row 0, column 4q + xoff) = first of the 10 bytes c0-3 .. c0+6, c0 = 4q + 3 + xoff
                const uint32_t* col = reinterpret_cast<const uint32_t*>(tileBase + ((4 * q + xoff) & ~3));
                // window byte offsets (relative to c0-3) of tile row y0 + r: x..x+3 = 3..6, x-3 = 0..3, x+3 = 6..9, x-2 = 1..4, x+2 = 5..8
                uint32_t M[FAST_RUN + 6], L0[FAST_RUN + 6], R6[FAST_RUN + 6], L1[FAST_RUN + 6], R5[FAST_RUN + 6];
#define ORBX_LO(w) __byte_perm((w), 0u, 0x4140)   /* bytes 0,1 -> two 16-bit lanes */
#define ORBX_HI(w) __byte_perm((w), 0u, 0x4342)   /* bytes 2,3 */
#pragma unroll
                for (int r = 0; r < FAST_RUN + 6; ++r) {
                    // the last run of a block may stop short: its rows past the window's last tile row (ih + 5) are clamped and
                    // the pixels they feed are dropped below
                    const uint32_t* rw = col + min(y0 + r, ih + 5) * tpw;
                    const uint32_t w0 = rw[0], w1 = rw[1], w2 = rw[2];
                    const uint32_t A = __funnelshift_r(w0, w1, shC), B = __funnelshift_r(w1, w2, shC);
                    M[r] = __funnelshift_r(A, B, 24); L0[r] = A; L1[r] = __funnelshift_r(A, B, 8);
                    if (r > 0 && r < FAST_RUN + 5) {     // the first and last rows only serve as ring rows +-3 (M)
                        const uint32_t C = __funnelshift_r(w2, rw[3], shC);
                        R6[r] = __funnelshift_r(B, C, 16); R5[r] = __funnelshift_r(B, C, 8);
                    }
                    if (r < 6) continue;
                    // interior row y0 + k: centre = tile row k + 3, ring rows k + 1, k + 5 (x +- 2) and k, k + 6 (x)
                    const int k = r - 6;
                    const uint32_t p0 = M[k + 6], p8 = M[k], p4 = R6[k + 3], p12 = L0[k + 3];
                    const uint32_t p2 = R5[k + 5], p14 = L1[k + 5], p6 = R5[k + 1], p10 = L1[k + 1];
                    const uint32_t V01 = ORBX_LO(M[k + 3]), V23 = ORBX_HI(M[k + 3]);
                    const uint32_t NLO01 = __vsub2(TT, V01), NLO23 = __vsub2(TT, V23);                 // T - v
                    const uint32_t NHI01 = __vsub2(0u, __vadd2(V01, TT1)), NHI23 = __vsub2(0u, __vadd2(V23, TT1));   // -(v + T + 1)
                    uint32_t dk01 = 0xFFFFFFFFu, dk23 = 0xFFFFFFFFu, br01 = 0u, br23 = 0u;
#define ORBX_OPP(pa, pb) { \
                    const uint32_t a01 = ORBX_LO(pa), a23 = ORBX_HI(pa), b01 = ORBX_LO(pb), b23 = ORBX_HI(pb); \
                    dk01 &= __vadd2(a01, NLO01) | __vadd2(b01, NLO01); dk23 &= __vadd2(a23, NLO23) | __vadd2(b23, NLO23); \
                    br01 |= __vadd2(a01, NHI01) & __vadd2(b01, NHI01); br23 |= __vadd2(a23, NHI23) & __vadd2(b23, NHI23); }
                    ORBX_OPP(p0, p8); ORBX_OPP(p4, p12); ORBX_OPP(p2, p10); ORBX_OPP(p6, p14);
#undef ORBX_OPP
                    const uint32_t c01 = dk01 | ~br01, c23 = dk23 | ~br23;
                    cand |= (((c01 >> 15) & 1u) | ((c01 >> 30) & 2u) | ((c23 >> 13) & 4u) | ((c23 >> 28) & 8u)) << (4 * k);
                    // the score map needs no clearing pass: every quad writes 0 here and phase 2 overwrites its corners
                    if (y0 + k < ih) *reinterpret_cast<uint32_t*>(score + (y0 + k + 1) * sp + 4 * q + 4) = 0u;
                }
#undef ORBX_LO
#undef ORBX_HI
                const int xr = iw - 4 * q, yr = ih - y0;     // pixels of this quad inside the interior, rows of this run inside it
                if (xr < 4) cand &= ((1u << xr) - 1u) * 0x11111111u;
                if (yr < FAST_RUN) cand &= (1u << (4 * yr)) - 1u;
            }
            // compaction: up to 4 * FAST_RUN candidates per lane, in (y, x) packed form
            const int n = __popc(cand);
            int incl = n;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
            const int wtot = __shfl_sync(0xffffffffu, incl, 31);
            if (wtot) {
                int wbase = 0;
                if (lane == 31) wbase = atomicAdd(&s_nCand, wtot);
                wbase = __shfl_sync(0xffffffffu, wbase, 31);
                int o = wbase + incl - n;
                const int yx = (y0 << 8) | (4 * q);
                for (uint32_t m = cand; m; m &= m - 1) {
                    const int b = __ffs(m) - 1;
                    list[o++] = (uint16_t)(yx + ((b >> 2) << 8) + (b & 3));
                }
            }
        }
    }
    __syncthreads();

    // phase 2: exact score for the survivors
    {
        int off[16];
        const int dxs[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
        const int dys[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
#pragma unroll
        for (int k = 0; k < 16; ++k) off[k] = dys[k] * tp + dxs[k];
        const int nc = s_nCand;
        for (int c = tid; c < nc; c += FAST_NT) {
            const int yx = list[c];
            const int y = yx >> 8, x = yx & 255;
            const int b = fast_score_at(tile + (y + 3) * tp + (x + 3), off);
            if (b > th) score[(y + 1) * sp + x + 4] = (uint8_t)(b - 1);
        }
    }
    __syncthreads();

    // phase 3: strict 8-neighbour maxima among the scored candidates only (corners are sparse) -> per-row keep bitmaps
    // for both thresholds via shared-memory atomicOr.  Neighbours outside the candidate's own cell count as 0 (v > 0 beats them),
    // so the ring and the neighbouring cells' scores are read but never compared.
    {
        const int nc = s_nCand;
        const int splitX = ncx > 1 ? s_rect[1].x : 1 << 30, splitY = ncell > ncx ? s_rect[ncx].y : 1 << 30;
        for (int c = tid; c < nc; c += FAST_NT) {
            const int yx = list[c];
            const int y = yx >> 8, x = yx & 255;
            const uint8_t* sc = score + (y + 1) * sp + x + 4;
            const int v = sc[0];
            if (v == 0) continue;
            const int k = (x >= splitX) + (y >= splitY ? ncx : 0);
            const int4 r = s_rect[k];
            const bool lt = x > r.x, rt = x + 1 < r.z;
            int m = max(lt ? sc[-1] : 0, rt ? sc[1] : 0);
            if (y > r.y) m = max(m, max(sc[-sp], max(lt ? sc[-sp - 1] : 0, rt ? sc[-sp + 1] : 0)));
            if (y + 1 < r.w) m = max(m, max(sc[sp], max(lt ? sc[sp - 1] : 0, rt ? sc[sp + 1] : 0)));
            if (v > m) {                                                      // score >= minTh by construction
                const int w = y * nwp + (x >> 5);
                atomicOr(&bitsLo[w], 1u << (x & 31));
                if (v >= P.iniTh) { atomicOr(&bitsHi[w], 1u << (x & 31)); s_hasHi[k] = 1; }
            }
        }
    }
    __syncthreads();
    // fallback to minTh only if the cell is empty at iniTh (:843-859); ordered (row-major) emission, one thread per (cell, row)
    const int nE = s_rowBase[ncell];
    for (int e = tid; e < nE; e += FAST_NT) {
        int k = 0;
        while (e >= s_rowBase[k + 1]) ++k;
        const int4 r = s_rect[k];
        const uint32_t* row = (s_hasHi[k] ? bitsHi : bitsLo) + (r.y + e - s_rowBase[k]) * nwp;
        int cnt = 0;
        for (int w = r.x >> 5; w << 5 < r.z; ++w) cnt += __popc(row[w] & fast_col_mask(w, r.x, r.z));
        rowOff[e] = cnt;
    }
    __syncthreads();
    const int total = block_prefix<FAST_NT>(nE, rowOff, s_warp, [&](int e) { return rowOff[e]; });
    for (int e = tid; e < nE; e += FAST_NT) {
        int k = 0;
        while (e >= s_rowBase[k + 1]) ++k;
        const int4 r = s_rect[k], od = s_out[k];
        const int y = r.y + e - s_rowBase[k];
        const uint32_t* row = (s_hasHi[k] ? bitsHi : bitsLo) + y * nwp;
        uint32_t* out = P.cellList + (size_t)f * P.cellListStride + od.x;
        int o = rowOff[e] - rowOff[s_rowBase[k]];
        for (int w = r.x >> 5; w << 5 < r.z; ++w)
            for (unsigned m = row[w] & fast_col_mask(w, r.x, r.z); m; m &= m - 1) {
                const int x = (w << 5) + __ffs(m) - 1;
                out[o++] = pack_cand(x - r.x + 3 + od.y, y - r.y + 3 + od.z, score[(y + 1) * sp + x + 4]);
            }
    }
    if (tid < ncell) {
        const int e0 = s_rowBase[tid], e1 = s_rowBase[tid + 1];
        outCount[bk.cell[tid]] = (e1 < nE ? rowOff[e1] : total) - (e0 < nE ? rowOff[e0] : total);
    }
}


// ------------------------------------------------------------------------------------------
// K1 (TMA form): pyramid level l from level l-1 with the source rows of a 128 x PYR_TILE_H destination tile staged into shared memory by
// ONE TMA bulk-tensor load (box pyrBoxW x pyrBoxH of level l-1, start aligned to 16 bytes); the fixed-point bilinear taps then read
// shared memory instead of gathering bytes from global memory.  Same integer arithmetic as pyr_resize_kernel (cv::resize INTER_LINEAR).
// A thread produces 4 columns of PYR_TILE_H / 8 consecutive rows, so one load feeds many output rows and the column taps are read once.
// ------------------------------------------------------------------------------------------
// The 7 levels of 240 frames of 640x480 on an H100 80GB HBM3 at 700 W: 0.44 ms with 128 x 8 tiles; 0.38 / 0.34 / 0.33 ms with
// tiles 16 / 32 / 64 rows tall and strided rows per warp; 0.29 / 0.26 ms at 32 / 64 rows with consecutive rows and the taps reuse.
// At 64 rows a box is at most ~122 rows (256 bytes wide caps the scale below 2), so it stays under 32 KB of shared memory.
constexpr int PYR_TILE_W = 128;
#ifndef PYR_TILE_H
#define PYR_TILE_H 64
#endif
static_assert(PYR_TILE_H % 8 == 0, "a CTA is 32 x 8 threads");
__global__ void __launch_bounds__(256) pyr_resize_tma_kernel(ExtractParams P, int l, const __grid_constant__ CUtensorMap srcMap) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_bar;
    const LevelGeom& G = P.lv[l];
    const int f = blockIdx.z;
    const int tid = threadIdx.y * 32 + threadIdx.x;
    const int dxT = blockIdx.x * PYR_TILE_W, dyT = blockIdx.y * PYR_TILE_H;
    const int cx0 = (int)P.xtab[G.xtabOff + dxT].x & ~15;                 // first source column of the tile, aligned down
    const int ry0 = (int)P.ytab[G.ytabOff + dyT].x;
    if (tid == 0) {
        mbar_init(&s_bar, 1);
        mbar_expect_tx(&s_bar, (uint32_t)(G.pyrBoxW * G.pyrBoxH));
        tma_load_3d(smem_raw, &srcMap, cx0, ry0, f, &s_bar);
    }
    __syncthreads();
    const int dx0 = dxT + threadIdx.x * 4;
    if (dx0 >= G.w) return;
    short4 xt[4];                                                          // {sx0, sx1, a0, a1}, shared by the thread's rows
#pragma unroll
    for (int k = 0; k < 4; ++k) xt[k] = __ldg(&P.xtab[G.xtabOff + min(dx0 + k, G.w - 1)]);
    mbar_wait(&s_bar, 0);
    uint8_t* dst = P.pyr + (size_t)f * P.pyrFrameStride + G.planeOff + dx0;
    // a warp owns PYR_TILE_H / 8 consecutive destination rows: where a row's upper source row is the previous row's lower one, its
    // horizontal taps are taken over instead of gathered again (most rows when downscaling by less than 2)
    int s0[4], s1[4], prevY1 = -1;
#pragma unroll
    for (int i = 0; i < PYR_TILE_H / 8; ++i) {
        const int dy = dyT + threadIdx.y * (PYR_TILE_H / 8) + i;
        if (dy >= G.h) break;
        const short4 yt = P.ytab[G.ytabOff + dy];  // {sy0, sy1, b0, b1}
        const uint8_t* r0 = smem_raw + (yt.x - ry0) * G.pyrBoxW - cx0;
        const uint8_t* r1 = smem_raw + (yt.y - ry0) * G.pyrBoxW - cx0;
        const bool reuse = yt.x == prevY1;
        prevY1 = yt.y;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (reuse) s0[k] = s1[k];
            else s0[k] = r0[xt[k].x] * xt[k].z + r0[xt[k].y] * xt[k].w;
            s1[k] = r1[xt[k].x] * xt[k].z + r1[xt[k].y] * xt[k].w;
        }
        const int b0 = yt.z, b1 = yt.w;
        uint32_t out = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (dx0 + k < G.w) {
                const int v = (((b0 * (s0[k] >> 4)) >> 16) + ((b1 * (s1[k] >> 4)) >> 16) + 2) >> 2;
                out |= (uint32_t)(v & 0xFF) << (8 * k);
            }
        *reinterpret_cast<uint32_t*>(dst + (size_t)dy * G.pitch) = out;   // pitch is a multiple of 32: in-bounds even for the tail
    }
}

// ------------------------------------------------------------------------------------------
// K3: quadtree distribution.  One warp per (level, frame); the warps of a CTA share the level.
// Reference: ORBextractor::DistributeOctTree src/ORBextractor.cc:555-779,
// ExtractorNode::DivideNode :480-536, compareNodes :538-553.
//
// The std::list / push_front choreography of the reference is restated as a rebuild of the
// whole node list per pass ("split a set of nodes in processing order, children blocks go to the
// front in reverse processing order, unsplit nodes keep their relative order"); the only
// sequential piece is the libstdc++ std::sort emulation that decides ties in the final phase.
// A problem's list state and, when they fit, its candidates live in the warp's shared-memory slab
// (qt_layout), so a pass costs warp scans and __syncwarp instead of CTA barriers; counts and best
// keys are shared-memory atomics.  The orientation of the selected keypoints is computed
// by orient_describe_kernel, one warp per keypoint across the batch.
// ------------------------------------------------------------------------------------------
constexpr int QT_MAX_WARPS = 8;

__device__ __forceinline__ int qt_child(const QtNode& n, int px, int py, int& midx, int& midy) {
    const int halfX = (int)ceilf((float)(n.brx - n.ulx) / 2);
    const int halfY = (int)ceilf((float)(n.bry - n.uly) / 2);
    midx = n.ulx + halfX; midy = n.uly + halfY;
    return (px < midx ? 0 : 1) + (py < midy ? 0 : 2);
}

__device__ __forceinline__ unsigned lanemask_lt() { unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }
__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
    return v;
}

// sx_partition_step by one warp.  The unguarded partition's k-th swap exchanges the k-th element from the left (from lo + 1) that is not
// below the pivot with the k-th from the right (from hi - 1) that is not above it, as long as the first lies left of the second: ballots
// list both kinds of stop in order (lpos / rpos, hi - lo entries each), the swaps run at once, and the cut is where the scan from the left
// stops first after the last swap.
template <class Less>
__device__ int warp_partition_step(QtSort* a, int lo, int hi, int16_t* lpos, int16_t* rpos, int lane, Less less) {
    if (lane == 0) sx_median_to_first(a, lo, hi, less);
    __syncwarp();
    const QtSort pivot = a[lo];
    int nL = 0, nR = 0;
    for (int b = lo + 1; b < hi; b += 32) {
        const int p = b + lane;
        const bool stop = p < hi && !less(a[p], pivot);
        const unsigned m = __ballot_sync(0xffffffffu, stop);
        if (stop) lpos[nL + __popc(m & lanemask_lt())] = (int16_t)p;
        nL += __popc(m);
    }
    for (int b = hi - 1; b >= lo; b -= 32) {
        const int p = b - lane;
        const bool stop = p >= lo && !less(pivot, a[p]);
        const unsigned m = __ballot_sync(0xffffffffu, stop);
        if (stop) rpos[nR + __popc(m & lanemask_lt())] = (int16_t)p;
        nR += __popc(m);
    }
    __syncwarp();
    const int nk = min(nL, nR);
    int K = 0;                            // swaps: lpos[k] < rpos[k] holds for a prefix of k
    for (int b = 0; b < nk; b += 32) {
        const unsigned m = __ballot_sync(0xffffffffu, b + lane < nk && lpos[b + lane] < rpos[b + lane]);
        K += __popc(m);
        if (m != 0xffffffffu) break;
    }
    for (int k = lane; k < K; k += 32) { const int pl = lpos[k], pr = rpos[k]; const QtSort x = a[pl]; a[pl] = a[pr]; a[pr] = x; }
    const int rPrev = K > 0 ? rpos[K - 1] : hi;
    const int cut = K < nL ? min((int)lpos[K], rPrev) : rPrev;
    __syncwarp();
    return cut;
}

// std::sort emulation by one warp (see exact_math.h: rounds of independent tasks); the warp runs the partition steps of a round one
// after another (warp_partition_step).  leaf: n / 2 + 1 tasks; qA / qB: n / 17 + 1 each; lpos / rpos: n entries each.  The final insertion
// sort of a leaf (of the whole range when n <= 16) moves an element only past strictly greater ones, so it is the stable sort of the leaf:
// a half-warp per leaf places each element at its stable rank.
__device__ void warp_libstdcxx_sort(QtSort* a, int n, SxTask* leaf, SxTask* qA, SxTask* qB, int16_t* lpos, int16_t* rpos, int lane) {
    const auto less = [](const QtSort& x, const QtSort& y) { return x.size < y.size || (x.size == y.size && x.ulx < y.ulx); };
    if (n < 2) return;
    int nc = 1, nl = 0;
    if (n <= 16) { nc = 0; nl = 1; if (lane == 0) leaf[0] = SxTask{0, n, 0}; }
    int depth = 0;
    for (int t = n; t > 1; t >>= 1) depth++;
    if (lane == 0 && nc) qA[0] = SxTask{0, n, 2 * depth};
    __syncwarp();
    SxTask *cur = qA, *nxt = qB;
    while (nc) {
        int nn = 0;
        for (int i = 0; i < nc; ++i) {
            const SxTask t = cur[i];
            if (t.d == 0) {                   // depth budget spent: heapsort on one lane
                if (lane == 0) sx_heapsort(a + t.lo, t.hi - t.lo, less);
                __syncwarp();
                continue;
            }
            const int cut = warp_partition_step(a, t.lo, t.hi, lpos, rpos, lane, less);
            const SxTask right = {cut, t.hi, t.d - 1}, left = {t.lo, cut, t.d - 1};
            const int rs = right.hi - right.lo, ls = left.hi - left.lo;
            if (lane == 0) {
                if (rs > 16) nxt[nn] = right; else if (rs > 1) leaf[nl] = right;
                if (ls > 16) nxt[nn + (rs > 16)] = left; else if (ls > 1) leaf[nl + (rs > 1 && rs <= 16)] = left;
            }
            nn += (rs > 16) + (ls > 16);
            nl += (rs > 1 && rs <= 16) + (ls > 1 && ls <= 16);
        }
        __syncwarp();
        SxTask* sw = cur; cur = nxt; nxt = sw;
        nc = nn;
    }
    for (int b = 0; b < nl; b += 2) {
        const int li = b + (lane >> 4), e = lane & 15;
        int lo = 0, len = 0;
        if (li < nl) { lo = leaf[li].lo; len = leaf[li].hi - lo; }
        QtSort x = {0, 0, 0};
        unsigned long long key = ~0ull;   // above every real key: (size, ulx) with size < 2^31, ulx >= 0
        if (e < len) { x = a[lo + e]; key = ((unsigned long long)(unsigned)x.size << 16) | (uint16_t)x.ulx; }
        int rank = 0;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const unsigned long long kk = __shfl_sync(0xffffffffu, key, k, 16);
            rank += kk < key || (kk == key && k < e);
        }
        __syncwarp();
        if (e < len) a[lo + rank] = x;
        __syncwarp();
    }
}

// Phase stamps of quadtree_kernel (build with -DQT_PHASES, read by tools/stage_times.py through orbx_qt_phases): lane 0 of every warp
// adds its clock64() spans per level.  [l][0] gather, [1] roots, [2] split passes before the careful phase, [3] careful-phase sorts,
// [4] careful passes without their sort, [5] best key per node + selection, [6] passes, [7] careful passes, [8] problems.
#ifdef QT_PHASES
__device__ unsigned long long qt_phase[kMaxLevels][9];
#define QT_STAMP(t) long long t = 0; if (lane == 0) t = clock64()
#define QT_ADD(k, v) if (lane == 0) atomicAdd(&qt_phase[l][k], (unsigned long long)(v))
#define QT_ONLY(x) x
#else
#define QT_STAMP(t)
#define QT_ADD(k, v)
#define QT_ONLY(x)
#endif

__global__ void __launch_bounds__(QT_MAX_WARPS * 32) quadtree_kernel(ExtractParams P) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const int l = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int f = blockIdx.y * (blockDim.x >> 5) + w;
    if (f >= P.batch) return;
    QT_STAMP(t0);
    const LevelGeom& G = P.lv[l];
    const QtLayout L = qt_layout(G.qtNodes, G.nCells);
    uint8_t* base = smem_raw + (size_t)w * P.qtSlab;
    QtNode* bnd0 = (QtNode*)(base + L.bnd0); QtNode* bnd1 = (QtNode*)(base + L.bnd1);
    int* cnt0 = (int*)(base + L.cnt0); int* cnt1 = (int*)(base + L.cnt1);
    int* childCnt = (int*)(base + L.scratch);
    QtSort* v = (QtSort*)(base + L.v);
    int16_t* proc = (int16_t*)(base + L.proc);          // per list node: processing index or -1
    int16_t* procNode = (int16_t*)(base + L.procNode);  // per processing index: list node
    int16_t* keepPos = (int16_t*)(base + L.keepPos);    // per list node: new position when unsplit
    int16_t* kExcl = (int16_t*)(base + L.kExcl);        // per processing index: children of the earlier ones
    int16_t* childPos = (int16_t*)(base + L.childPos);  // 4 per processing index: new list position (or -1)
    SelKp* sel = P.sel + (size_t)f * P.selStride + G.selOff;

    // ---- gather the per-cell lists into candidate order (cell row-major, then y, x) ----
    int* cellOff = childCnt;
    const int* cellCount = P.cellCount + (size_t)f * P.cellCountStride + G.cellBase;
    int n = 0;
    for (int c0 = 0; c0 < G.nCells; c0 += 32) {
        const int c = c0 + lane;
        const int k = c < G.nCells ? cellCount[c] : 0;
        const int inc = warp_incl_scan(k, lane);
        if (c < G.nCells) cellOff[c] = n + inc - k;
        n += __shfl_sync(0xffffffffu, inc, 31);
    }
    __syncwarp();
    const int capS = (P.qtSlab - L.cand) / 6;
    const bool inSmem = n <= capS;
    uint32_t* cand = inSmem ? (uint32_t*)(base + L.cand) : P.cand + (size_t)f * P.candStride + G.candOff;
    uint16_t* nodeOf = inSmem ? (uint16_t*)(base + L.cand + 4 * capS) : P.nodeOf + (size_t)f * P.candStride + G.candOff;
    if (n > 0) {
        // the lists of a level's cells are consecutive, cellCap apart; candidate i is in the last cell whose offset is <= i
        const uint32_t* lists = P.cellList + (size_t)f * P.cellListStride + P.cells[G.cellBase].listOff;
        int top = 1;
        while (top * 2 < G.nCells) top *= 2;
        for (int i0 = 0; i0 < n; i0 += 128) {
            int c[4] = {0, 0, 0, 0};
            for (int step = top; step; step >>= 1)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int t = c[j] + step;
                    if (t < G.nCells && cellOff[t] <= i0 + 32 * j + lane) c[j] = t;
                }
            uint32_t x[4] = {0, 0, 0, 0};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = i0 + 32 * j + lane;
                if (i < n) x[j] = lists[c[j] * G.cellCap + (i - cellOff[c[j]])];
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) if (i0 + 32 * j + lane < n) cand[i0 + 32 * j + lane] = x[j];
        }
    }
    __syncwarp();
    QT_STAMP(t1);
    QT_ADD(0, t1 - t0);

    // ---- root nodes (:559-598) ----
    for (int i = lane; i < G.nIni; i += 32) {
        QtNode nd;
        nd.ulx = (int16_t)(int)fmul(G.hX, (float)i); nd.uly = 0;
        nd.brx = (int16_t)(int)fmul(G.hX, (float)(i + 1)); nd.bry = (int16_t)(G.maxBY - G.minBY);
        bnd0[i] = nd; cnt0[i] = 0;
    }
    __syncwarp();
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        int r = -1;
        if (i < n) { r = (int)fdiv((float)cand_x(cand[i]), G.hX); nodeOf[i] = (uint16_t)r; }
        if (r >= 0) atomicAdd(&cnt0[r], 1);
    }
    __syncwarp();
    // erase empty roots, keep order
    int m = 0;
    for (int i0 = 0; i0 < G.nIni; i0 += 32) {
        const int i = i0 + lane;
        const bool keep = i < G.nIni && cnt0[i] > 0;
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        const int pos = m + __popc(b & lanemask_lt());
        if (i < G.nIni) keepPos[i] = (int16_t)(keep ? pos : -1);
        if (keep) { bnd1[pos] = bnd0[i]; cnt1[pos] = cnt0[i]; }
        m += __popc(b);
    }
    __syncwarp();
    for (int i = lane; i < n; i += 32) nodeOf[i] = (uint16_t)keepPos[nodeOf[i]];
    __syncwarp();
    QT_STAMP(t2);
    QT_ADD(1, t2 - t1);

    QtNode *bndC = bnd1, *bndN = bnd0;
    int *cntC = cnt1, *cntN = cnt0;
    const int N = G.nDesired;
    bool finish = (n == 0);
    bool careful = false;
    int q = 0;   // size of v
    while (!finish) {
        QT_STAMP(tp);
        QT_ONLY(long long tsort = 0;)
        const int prevSize = m;
        // --- A. processing order of the nodes to split ---
        int P0 = 0;
        if (!careful) {
            for (int s0 = 0; s0 < m; s0 += 32) {
                const int s = s0 + lane;
                const bool split = s < m && cntC[s] > 1;
                const unsigned b = __ballot_sync(0xffffffffu, split);
                const int pi = P0 + __popc(b & lanemask_lt());
                if (s < m) proc[s] = (int16_t)(split ? pi : -1);
                if (split) procNode[pi] = (int16_t)s;
                P0 += __popc(b);
            }
        } else {
            // std::sort(vPrev.begin(), vPrev.end(), compareNodes) (:705): the libstdc++ introsort, whose order among equal keys the result
            // depends on, run as rounds of independent partition steps (a warp per partition step) + independent leaf insertion
            // sorts -- exact_math.h: libstdcxx_sort_rounds_host is the same sequence, checked against std::sort on the host
            SxTask* tasks = reinterpret_cast<SxTask*>(childCnt);   // childPos is dead until step E: the partition's stop lists
            warp_libstdcxx_sort(v, q, tasks, tasks + q / 2 + 1, tasks + q / 2 + 1 + q / 17 + 1, childPos, childPos + G.qtNodes, lane);
            QT_ONLY(if (lane == 0) tsort = clock64() - tp;)
            for (int s = lane; s < m; s += 32) proc[s] = -1;
            __syncwarp();
            P0 = q;
            for (int j = lane; j < q; j += 32) {   // processed from the back (:706)
                const int pi = q - 1 - j;
                proc[v[j].node] = (int16_t)pi; procNode[pi] = v[j].node;
            }
        }
        for (int i = lane; i < 4 * P0; i += 32) childCnt[i] = 0;
        __syncwarp();
        // --- C. distribute the keys of every split node to its four children (:512-526); the child index goes to nodeOf's bits 12-13.
        //        Four keys per lane and sweep, their loads issued before any of them is used ---
        for (int i0 = 0; i0 < n; i0 += 128) {
            int s[4], pi[4];
            uint32_t c[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = i0 + 32 * j + lane;
                s[j] = i < n ? nodeOf[i] : -1; c[j] = i < n ? cand[i] : 0;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) pi[j] = s[j] >= 0 ? proc[s[j]] : -1;
            QtNode nd[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) if (pi[j] >= 0) nd[j] = bndC[s[j]];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (pi[j] >= 0) {
                    int mx, my;
                    const int ch = qt_child(nd[j], cand_x(c[j]), cand_y(c[j]), mx, my);
                    nodeOf[i0 + 32 * j + lane] = (uint16_t)(s[j] | ch << 12);
                    atomicAdd(&childCnt[4 * pi[j] + ch], 1);
                }
        }
        __syncwarp();
        // --- D. children per processed node; in the careful phase stop as soon as the list reaches N nodes (:755-756) ---
        int Pn = P0, totalChildren = 0;
        for (int pi0 = 0; pi0 < P0; pi0 += 32) {
            const int pi = pi0 + lane;
            int k = 0;
            if (pi < P0) { const int* cc = childCnt + 4 * pi; k = (cc[0] > 0) + (cc[1] > 0) + (cc[2] > 0) + (cc[3] > 0); }
            const int inc = warp_incl_scan(k, lane);
            if (pi < P0) kExcl[pi] = (int16_t)(totalChildren + inc - k);
            if (careful) {
                const unsigned hit = __ballot_sync(0xffffffffu, pi < P0 && prevSize + (totalChildren + inc) - (pi + 1) >= N);
                if (hit) {
                    const int h = __ffs(hit) - 1;
                    Pn = pi0 + h + 1;
                    totalChildren += __shfl_sync(0xffffffffu, inc, h);
                    break;
                }
            }
            totalChildren += __shfl_sync(0xffffffffu, inc, 31);
        }
        for (int pi = Pn + lane; pi < P0; pi += 32) proc[procNode[pi]] = -1;
        __syncwarp();
        // --- E/G. positions of the children: blocks in reverse processing order, n4..n1 inside ---
        for (int pi = lane; pi < Pn; pi += 32) {
            const int* cc = childCnt + 4 * pi;
            const int k = (cc[0] > 0) + (cc[1] > 0) + (cc[2] > 0) + (cc[3] > 0);
            const int blockStart = totalChildren - (kExcl[pi] + k);
            int after = 0;
            const QtNode pn = bndC[procNode[pi]];
            int mx, my;
            qt_child(pn, 0, 0, mx, my);
            for (int ch = 3; ch >= 0; --ch) {
                if (cc[ch] > 0) {
                    const int pos = blockStart + after;
                    ++after;
                    childPos[4 * pi + ch] = (int16_t)pos;
                    QtNode c;
                    c.ulx = (ch & 1) ? (int16_t)mx : pn.ulx; c.brx = (ch & 1) ? pn.brx : (int16_t)mx;
                    c.uly = (ch & 2) ? (int16_t)my : pn.uly; c.bry = (ch & 2) ? pn.bry : (int16_t)my;
                    bndN[pos] = c; cntN[pos] = cc[ch];
                } else childPos[4 * pi + ch] = -1;
            }
        }
        // --- F. unsplit nodes keep their order behind the new blocks ---
        int nKeep = 0;
        for (int s0 = 0; s0 < m; s0 += 32) {
            const int s = s0 + lane;
            const bool keep = s < m && proc[s] < 0;
            const unsigned b = __ballot_sync(0xffffffffu, keep);
            if (keep) {
                const int pos = totalChildren + nKeep + __popc(b & lanemask_lt());
                keepPos[s] = (int16_t)pos;
                bndN[pos] = bndC[s]; cntN[pos] = cntC[s];
            }
            nKeep += __popc(b);
        }
        __syncwarp();
        // --- new expandable list in creation order (processing order, n1..n4) (:634-668) ---
        int qNew = 0;
        for (int i0 = 0; i0 < 4 * Pn; i0 += 32) {
            const int i = i0 + lane;
            const bool e = i < 4 * Pn && childCnt[i] > 1;
            const unsigned b = __ballot_sync(0xffffffffu, e);
            if (e) {
                QtSort x; x.size = childCnt[i]; x.node = childPos[i]; x.ulx = bndN[x.node].ulx;
                v[qNew + __popc(b & lanemask_lt())] = x;
            }
            qNew += __popc(b);
        }
        // --- H. re-home the keys ---
        for (int i0 = 0; i0 < n; i0 += 128) {
            int t[4], pi[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) t[j] = i0 + 32 * j + lane < n ? nodeOf[i0 + 32 * j + lane] : 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) pi[j] = proc[t[j] & 0xFFF];
#pragma unroll
            for (int j = 0; j < 4; ++j) t[j] = pi[j] >= 0 ? childPos[4 * pi[j] + (t[j] >> 12)] : keepPos[t[j] & 0xFFF];
#pragma unroll
            for (int j = 0; j < 4; ++j) if (i0 + 32 * j + lane < n) nodeOf[i0 + 32 * j + lane] = (uint16_t)t[j];
        }
        __syncwarp();
        QT_STAMP(te);
        QT_ADD(3, tsort);
        QT_ADD(careful ? 4 : 2, te - tp - tsort);
        QT_ADD(6, 1);
        QT_ADD(7, careful ? 1 : 0);
        m = totalChildren + nKeep;
        q = qNew;
        { QtNode* t = bndC; bndC = bndN; bndN = t; int* c = cntC; cntC = cntN; cntN = c; }
        // --- termination (:684-764) ---
        if (m >= N || m == prevSize) finish = true;
        else if (!careful && m + 3 * q > N) careful = true;
    }
    QT_STAMP(t3);

    // ---- best response per node, first maximum in candidate order (:767-783): key = score << 24 | ~i (i < 2^24, checked on the host) ----
    unsigned* best = reinterpret_cast<unsigned*>(childCnt);
    for (int s = lane; s < m; s += 32) best[s] = 0u;
    __syncwarp();
    for (int i = lane; i < n; i += 32) atomicMax(&best[nodeOf[i]], ((unsigned)cand_s(cand[i]) << 24) | (0xFFFFFFu - (unsigned)i));
    __syncwarp();
    if (lane == 0) {
        P.selCount[f * kMaxLevels + l] = m;
        if (m > G.selCap) atomicOr(&P.status[f], 1);
    }
    const int mOut = min(m, G.selCap);
    for (int s = lane; s < mOut; s += 32) {
        const uint32_t c = cand[0xFFFFFFu - (best[s] & 0xFFFFFFu)];
        SelKp k; k.x = (int16_t)(cand_x(c) + G.minBX); k.y = (int16_t)(cand_y(c) + G.minBY); k.response = cand_s(c);
        sel[s] = k;
    }
    QT_STAMP(t4);
    QT_ADD(5, t4 - t3);
    QT_ADD(8, 1);
}

// ------------------------------------------------------------------------------------------
// K4: 7x7 sigma=2 Gaussian blur of every level (cv::GaussianBlur, fixed-point kernel
// [18,34,48,56,48,34,18]/256, BORDER_REFLECT_101; reference call site src/ORBextractor.cc:1133,
// SURVEY.md 9E).  Tile 64x32 per CTA, all levels in one launch.
// ------------------------------------------------------------------------------------------
constexpr int BL_TW = 128, BL_TH = 64, BL_NT = 256;   // tile per CTA; thread = 4 columns x 8 rows
constexpr int BL_SP = BL_TW + 32;                      // smem row pitch = TMA box width: columns x0-16 .. x0+TW+15 (the box must start 16-byte aligned)
constexpr int BL_C0 = 12;                              // tile byte of column x0-4, the first one the filter reads

__device__ __forceinline__ int reflect101(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = i < 0 ? -i : 2 * n - 2 - i;
    return i;
}

// One thread produces a 4 (columns) x 8 (rows) strip.  Horizontal pass on pairs of pixels packed as 2 x 16 bit
// (k*p <= 56*255 and the 7-tap sum <= 65280 fit 16 bits, so one IMAD serves two pixels), vertical pass in 32 bit,
// result (v + 32768) >> 16 -- bit-identical to cv::GaussianBlur's fixed-point path (SURVEY.md 9E).
__global__ void __launch_bounds__(BL_NT) blur_kernel(ExtractParams P, const __grid_constant__ CUtensorMap map0, const CUtensorMap* __restrict__ maps, int useTma) {
    __shared__ __align__(128) uint8_t tile[(BL_TH + 6) * BL_SP];
    __shared__ __align__(8) uint64_t s_bar;
    const int f = blockIdx.y;
    int l = 0;
    while (l + 1 < P.nlevels && (int)blockIdx.x >= P.lv[l + 1].blurTileBase) ++l;
    const LevelGeom& G = P.lv[l];
    const int t = blockIdx.x - G.blurTileBase;
    const int tyb = t / G.blurTilesX, txb = t - tyb * G.blurTilesX;
    const int x0 = txb * BL_TW, y0 = tyb * BL_TH;
    const int tid = threadIdx.x;
    if (useTma && G.w >= 8 && G.h >= 8) {
        // ---- tile: ONE TMA bulk-tensor load of rows y0-3 .. y0+TH+2, columns x0-16 .. x0+TW+15 of the pyramid plane (out-of-range
        //      elements arrive as 0); tiles on the image border then mirror the 3-px halo in shared memory (BORDER_REFLECT_101) ----
        if (tid == 0) {
            mbar_init(&s_bar, 1);
            mbar_expect_tx(&s_bar, (uint32_t)((BL_TH + 6) * BL_SP));
            tma_load_3d(tile, l == 0 ? &map0 : maps + l, x0 - 16, y0 - 3, f, &s_bar);
        }
        __syncthreads();
        mbar_wait(&s_bar, 0);
        const bool left = x0 == 0, right = x0 + BL_TW + 3 >= G.w, top = y0 == 0, bottom = y0 + BL_TH + 3 >= G.h;
        if (left || right) {
            for (int i = tid; i < (BL_TH + 6) * 8; i += BL_NT) {           // per row: 4 halo columns on either side
                const int r = i >> 3, k = i & 7;
                if (k < 4) { if (left) { const int x = -4 + k; tile[r * BL_SP + 16 + x] = tile[r * BL_SP + 16 - x]; } }
                else if (right) {
                    const int x = G.w + (k - 4);                           // columns w .. w+3
                    if (x - x0 < BL_TW + 4) tile[r * BL_SP + 16 + x - x0] = tile[r * BL_SP + 16 + (2 * G.w - 2 - x) - x0];
                }
            }
            __syncthreads();
        }
        if (top || bottom) {
            for (int i = tid; i < 6 * (BL_SP / 4); i += BL_NT) {           // 3 halo rows above / below, whole rows as words
                const int k = i / (BL_SP / 4), wq = i - k * (BL_SP / 4);
                int y;
                if (k < 3) { if (!top) continue; y = -3 + k; }
                else { if (!bottom) continue; y = G.h + (k - 3); if (y - y0 + 3 >= BL_TH + 6) continue; }
                const int ys = y < 0 ? -y : 2 * G.h - 2 - y;
                reinterpret_cast<uint32_t*>(tile + (y - y0 + 3) * BL_SP)[wq] = reinterpret_cast<const uint32_t*>(tile + (ys - y0 + 3) * BL_SP)[wq];
            }
            __syncthreads();
        }
    } else {
        int pitch;
        const uint8_t* img = plane_ptr(P, f, l, pitch);
        // ---- fallback tile load (level 0 not TMA-addressable, or a plane smaller than the halo logic assumes) ----
        for (int i = tid; i < (BL_TH + 6) * 34; i += BL_NT) {
            const int r = i / 34, wq = i - r * 34;
            const int sy = reflect101(min(y0 + r - 3, G.h + 2), G.h);
            const uint8_t* row = img + (size_t)sy * pitch;
            uint32_t v = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) v |= (uint32_t)row[reflect101(min(x0 - 4 + 4 * wq + k, G.w + 3), G.w)] << (8 * k);
            *reinterpret_cast<uint32_t*>(tile + r * BL_SP + BL_C0 + 4 * wq) = v;
        }
        __syncthreads();
    }
    const int tx = tid & 31, ty = tid >> 5;          // 32 x 8 threads
    const int xo = x0 + 4 * tx, yo = y0 + 8 * ty;
    if (xo >= G.w || yo >= G.h) return;
    // Fused H + V: the 14 input rows of the strip are walked once.  Horizontal pass on pairs of pixels packed as 2 x 16 bit; every
    // horizontal sum is unpacked ONCE and scattered with its tap weight into the (up to 7) output rows it contributes to -- the
    // accumulators of the 8 x 4 outputs stay in registers (the earlier form unpacked every sum once per output row: 7x the work).
    uint32_t acc[8][4];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[r][k] = 0;
#pragma unroll
    for (int r = 0; r < 14; ++r) {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(tile + (8 * ty + r) * BL_SP + BL_C0 + 4 * tx);
        const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];   // bytes b0..b11 = columns xo-4 .. xo+7
        // pair words Ps = b_s | b_{s+1} << 16 (two pixels as 2 x 16 bit), s = 1..9: 32-bit window at byte s, then spread bytes 0,1
#define ORBX_PAIR(lo, hi, sh) __byte_perm(__funnelshift_r(lo, hi, sh), 0u, 0x4140)
        const uint32_t P1 = ORBX_PAIR(w0, w1, 8), P2 = ORBX_PAIR(w0, w1, 16), P3 = ORBX_PAIR(w0, w1, 24);
        const uint32_t P4 = ORBX_PAIR(w1, w2, 0), P5 = ORBX_PAIR(w1, w2, 8), P6 = ORBX_PAIR(w1, w2, 16), P7 = ORBX_PAIR(w1, w2, 24);
        const uint32_t P8 = ORBX_PAIR(w2, 0u, 0), P9 = ORBX_PAIR(w2, 0u, 8);
#undef ORBX_PAIR
        const uint32_t h01 = 18u * (P1 + P7) + 34u * (P2 + P6) + 48u * (P3 + P5) + 56u * P4;
        const uint32_t h23 = 18u * (P3 + P9) + 34u * (P4 + P8) + 48u * (P5 + P7) + 56u * P6;
        const uint32_t h[4] = {h01 & 0xFFFFu, h01 >> 16, h23 & 0xFFFFu, h23 >> 16};
#pragma unroll
        for (int j = 0; j < 7; ++j) {
            const int o = r - j;                         // input row r is tap j of output row r - j
            if (o >= 0 && o < 8) {
                const uint32_t kj = j == 0 || j == 6 ? 18u : (j == 1 || j == 5 ? 34u : (j == 2 || j == 4 ? 48u : 56u));
#pragma unroll
                for (int k = 0; k < 4; ++k) acc[o][k] += kj * h[k];
            }
        }
    }
    int bpitch;
    uint8_t* out = const_cast<uint8_t*>(blur_ptr(P, f, l, bpitch));
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        if (yo + r >= G.h) break;
        uint32_t pk = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) pk |= ((acc[r][k] + 32768u) >> 16) << (8 * k);
        uint8_t* o = out + (size_t)(yo + r) * bpitch + xo;
        if (xo + 3 < G.w) *reinterpret_cast<uint32_t*>(o) = pk;     // bpitch and xo are multiples of 4
        else {
            for (int k = 0; k < 4 && xo + k < G.w; ++k) o[k] = (uint8_t)(pk >> (8 * k));
        }
    }
}

// ------------------------------------------------------------------------------------------
// K5: output assembly.  One CTA per frame: scale coordinates, split lapping / non-lapping
// keypoints (front / back fill), write the cv::KeyPoint-layout slab and the row map.
// Reference: ORBextractor::operator() src/ORBextractor.cc:1120-1164.
// ------------------------------------------------------------------------------------------
constexpr int AS_NT = 256;

__global__ void __launch_bounds__(AS_NT) assemble_kernel(ExtractParams P) {
    extern __shared__ int s_flags[];   // selStride ints
    __shared__ int s_warp[33];
    __shared__ int s_lvOff[kMaxLevels + 1];
    const int f = blockIdx.x, tid = threadIdx.x;
    if (tid == 0) {
        int o = 0;
        for (int l = 0; l < P.nlevels; ++l) { s_lvOff[l] = o; o += min(P.selCount[f * kMaxLevels + l], P.lv[l].selCap); }
        s_lvOff[P.nlevels] = o;
    }
    __syncthreads();
    const int K = s_lvOff[P.nlevels];
    const SelKp* sel = P.sel + (size_t)f * P.selStride;
    // flag = keypoint lies in the lapping area (scaled x within [lap0, lap1])
    for (int e = tid; e < K; e += AS_NT) {
        int l = 0;
        while (e >= s_lvOff[l + 1]) ++l;
        const SelKp k = sel[P.lv[l].selOff + (e - s_lvOff[l])];
        float x = (float)k.x;
        if (l != 0) x = fmul(x, P.lv[l].scale);
        s_flags[e] = (x >= (float)P.lap0 && x <= (float)P.lap1) ? 1 : 0;
    }
    __syncthreads();
    // exclusive scan -> number of lapping keypoints before e
    int* s_scan = s_flags + P.selStride;
    for (int e = tid; e < K; e += AS_NT) s_scan[e] = s_flags[e];
    __syncthreads();
    const int nLap = block_prefix<AS_NT>(K, s_scan, s_warp, [&](int e) { return s_scan[e]; });
    int* dstIndex = P.dstIndex + (size_t)f * P.selStride;
    OrbKeyPoint* out = reinterpret_cast<OrbKeyPoint*>(P.outKp) + (size_t)f * P.outCap;
    const bool fits = K <= P.outCap;
    for (int e = tid; e < K; e += AS_NT) {
        int l = 0;
        while (e >= s_lvOff[l + 1]) ++l;
        const int src = P.lv[l].selOff + (e - s_lvOff[l]);
        const SelKp k = sel[src];
        const int at = s_flags[e] ? (K - 1 - s_scan[e]) : (e - s_scan[e]);
        dstIndex[src] = fits ? at : -1;
        if (fits) {
            OrbKeyPoint o;
            o.x = (float)k.x; o.y = (float)k.y;
            if (l != 0) { o.x = fmul(o.x, P.lv[l].scale); o.y = fmul(o.y, P.lv[l].scale); }
            o.size = P.lv[l].sizeScaled; o.angle = 0.f; o.response = (float)k.response;   // the angle: orient_describe_kernel
            o.octave = l; o.class_id = -1;
            out[at] = o;
        }
    }
    if (tid == 0) {
        P.outN[f] = K;
        P.outMono[f] = K - nLap;
        if (!fits) atomicOr(&P.status[f], 2);
    }
}

// ------------------------------------------------------------------------------------------
// K6: orientation + rotated BRIEF.  One warp per selected keypoint of the batch.
// Reference: IC_Angle src/ORBextractor.cc:76-103 on the pyramid plane, then computeOrbDescriptor
// :107-146 on the blurred plane with lane = descriptor byte.  The angle goes to the output slab,
// where assemble_kernel left it unset.
// ------------------------------------------------------------------------------------------
constexpr int DS_NT = 256;

__global__ void __launch_bounds__(DS_NT) orient_describe_kernel(ExtractParams P) {
    __shared__ char4 s_pat[8][32];   // [pair-in-byte][byte] -> conflict-free across lanes
    const int f = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
    for (int i = tid; i < 256; i += DS_NT) {
        const int byte = i >> 3, k = i & 7;
        s_pat[k][byte] = make_char4(c_pattern[4 * i], c_pattern[4 * i + 1], c_pattern[4 * i + 2], c_pattern[4 * i + 3]);
    }
    __syncthreads();
    const int slot = blockIdx.x * (DS_NT / 32) + (tid >> 5);   // index into the frame's sel array
    if (slot >= (int)P.selStride) return;
    int l = 0;
    while (l + 1 < P.nlevels && slot >= P.lv[l + 1].selOff) ++l;
    const int idx = slot - P.lv[l].selOff;
    if (idx >= min(P.selCount[f * kMaxLevels + l], P.lv[l].selCap)) return;
    const int at = P.dstIndex[(size_t)f * P.selStride + slot];
    if (at < 0) return;
    const SelKp k = P.sel[(size_t)f * P.selStride + slot];
    int pitch;
    // lane = column u of the radius-15 disc, rows walked together: every load instruction of the warp reads one contiguous 31-byte
    // row segment (one or two sectors) instead of 31 different rows
    int m10 = 0, m01 = 0;
    {
        const uint8_t* img = plane_ptr(P, f, l, pitch);
        const int u = lane - HALF_PATCH;
        const int au = u < 0 ? -u : u;
        const uint8_t* centre = img + (size_t)k.y * pitch + k.x + (lane < 31 ? u : 0);
        int colsum = 0;
#pragma unroll
        for (int v = -HALF_PATCH; v <= HALF_PATCH; ++v) {
            const int px = (lane < 31 && au <= c_umax[v < 0 ? -v : v]) ? centre[v * pitch] : 0;
            colsum += px; m01 += v * px;
        }
        m10 = u * colsum;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        m10 += __shfl_xor_sync(0xffffffffu, m10, o);
        m01 += __shfl_xor_sync(0xffffffffu, m01, o);
    }
    const float angle = fast_atan2_deg((float)m01, (float)m10);
    if (lane == 0) reinterpret_cast<OrbKeyPoint*>(P.outKp)[(size_t)f * P.outCap + at].angle = angle;
    const float factorPI = 0.01745329238474369049072265625f;   // (float)(CV_PI/180.f), :106
    float a, b;
    sincosf_glibc(fmul(angle, factorPI), &b, &a);
    const uint8_t* img = blur_ptr(P, f, l, pitch);
    const uint8_t* c = img + (size_t)k.y * pitch + k.x;
    int val = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const char4 q = s_pat[j][lane];
        const float x0 = (float)q.x, y0 = (float)q.y, x1 = (float)q.z, y1 = (float)q.w;
        const int r0 = round_half_even(ffma(x0, b, fmul(y0, a)));
        const int c0 = round_half_even(ffma(x0, a, -fmul(y0, b)));
        const int r1 = round_half_even(ffma(x1, b, fmul(y1, a)));
        const int c1 = round_half_even(ffma(x1, a, -fmul(y1, b)));
        const int t0 = c[r0 * pitch + c0], t1 = c[r1 * pitch + c1];
        val |= (t0 < t1) << j;
    }
    P.outDesc[((size_t)f * P.outCap + at) * 32 + lane] = (uint8_t)val;
}


// ------------------------------------------------------------------------------------------
// K7: Frame::ComputeStereoMatches (reference src/Frame.cc:811-982), the stereo consumer of mvImagePyramid.  One CTA per rectified
// pair; a warp per left keypoint: (1) best right keypoint on the same row band (|dy| <= 2 * scale of the right keypoint, level
// within +-1, disparity window) by Hamming distance, ties to the lower right index (= the reference's row-table order);
// (2) 11 x 11 SAD refinement over 11 shifts on the pyramid planes of the left keypoint's level, parabola fit, disparity / depth;
// then (3) the CTA removes matches whose SAD is >= 1.5 * 1.4 * median.  Float arithmetic is individually rounded like the oracle's.
// The 19-px reflected frame the reference keeps around every plane is not needed: for keypoints the extractor can produce the
// windows stay >= 5 px inside the planes (DESIGN.md); a window that would leave the plane flags status bit 4 instead of reading.
// ------------------------------------------------------------------------------------------
// copyMakeBorder(level, BORDER_REFLECT_101) around one pyramid plane (src/ORBextractor.cc:1185-1191), written on request only
__global__ void border_copy_kernel(ExtractParams P, int f, int l, int border, uint8_t* __restrict__ dst) {
    const LevelGeom& G = P.lv[l];
    const int W = G.w + 2 * border;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    int pitch;
    const uint8_t* img = plane_ptr(P, f, l, pitch);
    dst[(size_t)y * W + x] = img[(size_t)reflect101(y - border, G.h) * pitch + reflect101(x - border, G.w)];
}

constexpr int ST_NT = 256;
struct StereoParams {
    ExtractParams L, R;                    // geometry + pyramid pointers of the two extractors (same image size)
    const OrbKeyPoint *kpsL, *kpsR; const uint8_t *descL, *descR; const int *nL, *nR; int capL, capR;
    float mb, mbf;
    float* uRight; float* depth;           // [batch][capL]
    int* sad;                              // scratch [batch][capL]
    int* status;                           // [batch]
};

__global__ void __launch_bounds__(ST_NT) stereo_matches_kernel(StereoParams Q) {
    __shared__ int s_cnt, s_median;
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int N = min(Q.nL[f], Q.capL), Nr = min(Q.nR[f], Q.capR);
    const OrbKeyPoint* kl = Q.kpsL + (size_t)f * Q.capL; const OrbKeyPoint* kr = Q.kpsR + (size_t)f * Q.capR;
    const uint8_t* dl = Q.descL + (size_t)f * Q.capL * 32; const uint8_t* dr = Q.descR + (size_t)f * Q.capR * 32;
    float* uRight = Q.uRight + (size_t)f * Q.capL; float* depth = Q.depth + (size_t)f * Q.capL;
    int* sad = Q.sad + (size_t)f * Q.capL;
    const float minD = 0.f, maxD = fdiv(Q.mbf, Q.mb);
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    for (int iL = wid; iL < N; iL += ST_NT / 32) {
        const OrbKeyPoint kpL = kl[iL];
        float outU = -1.0f, outD = -1.0f; int outSad = -1;
        const float uL = kpL.x, vL = kpL.y;
        const int rowL = (int)vL;                                    // vRowIndices[vL]: float -> index by truncation
        const float minU = fsub(uL, maxD), maxU = fsub(uL, minD);
        unsigned best = 0xFFFFFFFFu;
        if (!(maxU < 0)) {
            uint32_t da[8];
            load_desc(dl + (size_t)iL * 32, da);
            for (int iR = lane; iR < Nr; iR += 32) {
                const OrbKeyPoint kpR = kr[iR];
                const float r = fmul(2.0f, Q.L.lv[min(max(kpR.octave, 0), Q.L.nlevels - 1)].scale);
                const int maxr = (int)ceilf(fadd(kpR.y, r)), minr = (int)floorf(fsub(kpR.y, r));
                if (rowL < minr || rowL > maxr) continue;
                if (kpR.octave < kpL.octave - 1 || kpR.octave > kpL.octave + 1) continue;
                if (!(kpR.x >= minU && kpR.x <= maxU)) continue;
                uint32_t db[8];
                load_desc(dr + (size_t)iR * 32, db);
                const unsigned dist = (unsigned)hamming256(da, db);
                if (dist < 100u) best = min(best, (dist << 16) | (unsigned)iR);      // bestDist starts at TH_HIGH, strict <
            }
        }
        best = __reduce_min_sync(0xffffffffu, best);
        if (best != 0xFFFFFFFFu && (int)(best >> 16) < (100 + 50) / 2) {             // thOrbDist
            const int bestIdxR = (int)(best & 0xFFFFu);
            const int lvl = min(max(kpL.octave, 0), Q.L.nlevels - 1);
            const float uR0 = kr[bestIdxR].x;
            const float scaleFactor = fdiv(1.0f, Q.L.lv[lvl].scale);                  // mvInvScaleFactors[octave] = 1.0f / mvScaleFactor[octave]
            const float scaleduL = roundf(fmul(kpL.x, scaleFactor)), scaledvL = roundf(fmul(kpL.y, scaleFactor)), scaleduR0 = roundf(fmul(uR0, scaleFactor));
            const int w = 5, Lr = 5;
            const LevelGeom& G = Q.L.lv[lvl];
            const float iniu = fsub(fadd(scaleduR0, (float)Lr), (float)w), endu = fadd(fadd(fadd(scaleduR0, (float)Lr), (float)w), 1.0f);
            if (!(iniu < 0 || endu >= (float)G.w)) {
                const int y0 = (int)fsub(scaledvL, (float)w), xL0 = (int)fsub(scaleduL, (float)w), xR00 = (int)scaleduR0 - Lr - w;
                if (y0 < 0 || y0 + 2 * w + 1 > G.h || xL0 < 0 || xL0 + 2 * w + 1 > G.w || xR00 < 0) { if (lane == 0) atomicOr(&Q.status[f], 4); }
                else {
                    int pitchL, pitchR;
                    const uint8_t* IL = plane_ptr(Q.L, f, lvl, pitchL);
                    const uint8_t* IR = plane_ptr(Q.R, f, lvl, pitchR);
                    // this lane's pixels of the 11 x 11 left window
                    int pa[4], rr[4], cc[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const int p = lane + 32 * k;
                        rr[k] = p / 11; cc[k] = p - rr[k] * 11;
                        pa[k] = p < 121 ? IL[(size_t)(y0 + rr[k]) * pitchL + xL0 + cc[k]] : 0;
                    }
                    int bestSad = 0x7fffffff, bestincR = 0;
                    float vDists[11];
#pragma unroll
                    for (int incR = -5; incR <= 5; ++incR) {
                        const int xR0 = (int)fsub(fadd(scaleduR0, (float)incR), (float)w);
                        int s = 0;
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const int p = lane + 32 * k;
                            if (p < 121) { const int b = IR[(size_t)(y0 + rr[k]) * pitchR + xR0 + cc[k]]; s += abs(pa[k] - b); }
                        }
                        s = __reduce_add_sync(0xffffffffu, s);
                        const float dist = (float)s;
                        if (dist < (float)bestSad) { bestSad = (int)dist; bestincR = incR; }
                        vDists[incR + 5] = dist;
                    }
                    if (!(bestincR == -Lr || bestincR == Lr)) {
                        float dist1 = 0, dist2 = 0, dist3 = 0;
#pragma unroll
                        for (int k = 1; k < 10; ++k) if (k == bestincR + 5) { dist1 = vDists[k - 1]; dist2 = vDists[k]; dist3 = vDists[k + 1]; }
                        const float deltaR = fdiv(fsub(dist1, dist3), fmul(2.0f, fsub(fadd(dist1, dist3), fmul(2.0f, dist2))));
                        if (!(deltaR < -1 || deltaR > 1)) {
                            float bestuR = fmul(G.scale, fadd(fadd(scaleduR0, (float)bestincR), deltaR));
                            float disparity = fsub(uL, bestuR);
                            if (disparity >= minD && disparity < maxD) {
                                if (disparity <= 0) { disparity = 0.01f; bestuR = (float)((double)uL - 0.01); }
                                outD = fdiv(Q.mbf, disparity); outU = bestuR; outSad = bestSad;
                            }
                        }
                    }
                }
            }
        }
        if (lane == 0) { uRight[iL] = outU; depth[iL] = outD; sad[iL] = outSad; if (outSad >= 0) atomicAdd(&s_cnt, 1); }
    }
    __syncthreads();
    // median of the SAD distances of the accepted matches: element size/2 of the (distance, iL)-sorted list (:964-966)
    const int cnt = s_cnt;
    if (cnt == 0) return;
    for (int i = tid; i < N; i += ST_NT) {
        const int di = sad[i];
        if (di < 0) continue;
        int rank = 0;
        for (int j = 0; j < N; ++j) { const int dj = sad[j]; rank += dj >= 0 && (dj < di || (dj == di && j < i)); }
        if (rank == cnt / 2) s_median = di;
    }
    __syncthreads();
    const float thDist = fmul(1.5f * 1.4f, (float)s_median);
    for (int i = tid; i < N; i += ST_NT) {
        const int di = sad[i];
        if (di >= 0 && !((float)di < thDist)) { uRight[i] = -1.0f; depth[i] = -1.0f; }
    }
}

}  // namespace orbx
