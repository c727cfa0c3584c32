// Host side of the batched H100 ORB extractor + its C-ABI (include/orb_b200.h).
// Mirrors ORBextractor (reference include/ORBextractor.h:43-109, src/ORBextractor.cc).
#include <cuda.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/orb_b200.h"
#include "extractor_kernels.cuh"

namespace orbx {

static thread_local std::string g_err;
void set_error(const std::string& s) { g_err = s; }

static const int8_t h_pattern[1024] = {
#include "brief_pattern.inc"
};

static inline int cvRoundF(float v) { return (int)nearbyintf(v); }
static inline int cvFloorD(double v) { int i = (int)v; return i - (i > v); }
static inline int cvCeilD(double v) { int i = (int)v; return i + (i < v); }
static inline size_t alignUp(size_t v, size_t a) { return (v + a - 1) / a * a; }

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link against libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
    }
    return fn;
}
// 3-D u8 tensor {x, y, frame}: x contiguous, row pitch, frame stride; box {bw, bh, 1}; out-of-bounds reads return 0
static bool encode_plane_map(CUtensorMap* m, const void* base, int w, int h, int frames, size_t pitch, size_t frameStride, int bw, int bh) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return false;
    if (((uintptr_t)base & 15) || (pitch & 15) || (frameStride & 15)) return false;
    cuuint64_t dims[3] = {(cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)frames};
    cuuint64_t strides[2] = {(cuuint64_t)pitch, (cuuint64_t)frameStride};
    cuuint32_t box[3] = {(cuuint32_t)bw, (cuuint32_t)bh, 1};
    cuuint32_t es[3] = {1, 1, 1};
    return fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct Extractor {
    // constructor arguments (reference src/ORBextractor.cc:409-413)
    int nfeatures, nlevels, iniTh, minTh;
    double scaleFactor;   // the reference keeps the float argument in a double member (ORBextractor.h:92)
    std::vector<float> scale, invScale, sigma2, invSigma2;
    std::vector<int> featPerLevel;
    int umax[HALF_PATCH + 1];
    int device, maxW, maxH, maxBatch;
    // current geometry
    int rows = 0, cols = 0;
    ExtractParams P;
    std::vector<CellDesc> cells;
    std::vector<FastBlock> fastBlocks;
    // device buffers
    uint8_t *d_pyr = nullptr, *d_blur = nullptr;
    CellDesc* d_cells = nullptr;
    FastBlock* d_fastBlocks = nullptr;
    int* d_cellCount = nullptr;
    uint32_t* d_cellList = nullptr;
    uint32_t* d_cand = nullptr;
    uint16_t* d_nodeOf = nullptr;
    SelKp* d_sel = nullptr;
    int *d_selCount = nullptr, *d_dstIndex = nullptr, *d_status = nullptr;
    short4 *d_xtab = nullptr, *d_ytab = nullptr;
    // staging for the host-pointer entry points
    uint8_t* d_img = nullptr;      // maxBatch frames, tightly packed at level-0 pitch
    OrbKeyPoint* d_outKp = nullptr; uint8_t* d_outDesc = nullptr; int *d_outN = nullptr, *d_outMono = nullptr;
    int* h_counts = nullptr;       // pinned: n[maxBatch], mono[maxBatch], status[maxBatch]
    int outCapInternal = 0;
    cudaStream_t stream = nullptr, stream2 = nullptr;
    cudaEvent_t evWait = nullptr;      // blocking-sync event: batch calls sleep on it instead of spinning (device_utils.cuh)
    cudaEvent_t evFork = nullptr, evJoin = nullptr;
    bool profiling = false; cudaEvent_t evStage[8] = {};   // pyramid | blur | fast | quadtree | assemble | orientation + BRIEF
    float stageMs[6] = {0, 0, 0, 0, 0, 0};
    size_t smemFast = 0, smemQt = 0, smemAs = 0;
    int launches = 0;
    int maxKp = 0;
    ExtractParams lastQ; bool hasLast = false;   // geometry + plane pointers of the last enqueued call (the pyramid the stereo matcher reads)
    int* d_stereoSad = nullptr; float *d_stereoU = nullptr, *d_stereoD = nullptr; int* h_stereoStatus = nullptr;
    OrbKeyPoint* d_outKpUn = nullptr;   // mvKeysUn of the resident slab (orbx_undistort_keypoints), allocated on first use
    TmaMaps maps;            // per-level TMA descriptors of the internal pyramid planes (level 0: internal copy)
    CUtensorMap* d_maps = nullptr;   // device copy of `maps`
    TmaMaps pyrMaps;         // pyrMaps.lv[l]: level l-1 with the source box of level l's resize tiles (host copy: passed by value per launch)
    TmaMaps blurMaps;        // the same planes with the blur tile box (BL_SP x (BL_TH + 6))
    CUtensorMap* d_blurMaps = nullptr;

    ~Extractor() { release(); }
    void release() {
        cudaSetDevice(device);
        void* ptrs[] = {d_pyr, d_blur, d_cells, d_fastBlocks, d_cellCount, d_cellList, d_cand, d_nodeOf, d_sel, d_selCount, d_dstIndex,
                        d_status, d_xtab, d_ytab, d_img, d_outKp, d_outDesc, d_outN, d_outMono, d_maps, d_blurMaps, d_stereoSad, d_stereoU, d_stereoD,
                        d_outKpUn};
        for (void* p : ptrs) if (p) cudaFree(p);
        if (h_counts) cudaFreeHost(h_counts);
        if (h_stereoStatus) cudaFreeHost(h_stereoStatus);
        if (evWait) cudaEventDestroy(evWait);
        if (stream) cudaStreamDestroy(stream);
        if (stream2) cudaStreamDestroy(stream2);
        if (evFork) cudaEventDestroy(evFork);
        if (evJoin) cudaEventDestroy(evJoin);
        for (cudaEvent_t e : evStage) if (e) cudaEventDestroy(e);
    }

    // ORBextractor::ORBextractor, src/ORBextractor.cc:409-469
    void init_tables() {
        scale.resize(nlevels); sigma2.resize(nlevels); invScale.resize(nlevels); invSigma2.resize(nlevels);
        scale[0] = 1.0f; sigma2[0] = 1.0f;
        for (int i = 1; i < nlevels; ++i) {
            scale[i] = (float)(scale[i - 1] * scaleFactor);
            sigma2[i] = scale[i] * scale[i];
        }
        for (int i = 0; i < nlevels; ++i) { invScale[i] = 1.0f / scale[i]; invSigma2[i] = 1.0f / sigma2[i]; }
        featPerLevel.resize(nlevels);
        float factor = (float)(1.0f / scaleFactor);
        float nDesired = nfeatures * (1 - factor) / (1 - (float)pow((double)factor, (double)nlevels));
        int sum = 0;
        for (int l = 0; l < nlevels - 1; ++l) {
            featPerLevel[l] = cvRoundF(nDesired);
            sum += featPerLevel[l];
            nDesired *= factor;
        }
        featPerLevel[nlevels - 1] = std::max(nfeatures - sum, 0);
        int v, v0, vmax = cvFloorD(HALF_PATCH * sqrtf(2.f) / 2 + 1);
        int vmin = cvCeilD(HALF_PATCH * sqrtf(2.f) / 2);
        const double hp2 = HALF_PATCH * HALF_PATCH;
        for (v = 0; v <= vmax; ++v) umax[v] = (int)nearbyint(sqrt(hp2 - v * v));
        for (v = HALF_PATCH, v0 = 0; v >= vmin; --v) {
            while (umax[v0] == umax[v0 + 1]) ++v0;
            umax[v] = v0;
            ++v0;
        }
    }

    // Level geometry for a rows x cols image: pyramid sizes (src/ORBextractor.cc:1174-1175), FAST cell
    // grid (:789-824), quadtree roots (:559-561), resize coefficient tables (SURVEY.md 9C).
    int configure(int r, int c, std::vector<short4>& xtab, std::vector<short4>& ytab) {
        memset(&P, 0, sizeof(P));
        P.nlevels = nlevels; P.iniTh = iniTh; P.minTh = minTh; P.rows = r; P.cols = c;
        cells.clear(); fastBlocks.clear(); xtab.clear(); ytab.clear();
        size_t planeOff = 0, listOff = 0, candOff = 0;
        int selOff = 0, blurTiles = 0, qtEnd = 0;
        maxKp = 0;
        smemFast = 0;
        for (int l = 0; l < nlevels; ++l) {
            LevelGeom& G = P.lv[l];
            G.w = cvRoundF((float)c * invScale[l]);
            G.h = cvRoundF((float)r * invScale[l]);
            if (G.w > 4095 || G.h > 4095) { set_error("image larger than 4095 px is not supported"); return ORB_ERR_ARG; }
            G.pitch = (int)alignUp(G.w, 32);
            G.planeOff = (uint32_t)planeOff;
            planeOff += alignUp((size_t)G.pitch * G.h, 256);
            G.minBX = EDGE_THRESHOLD - 3; G.minBY = G.minBX;
            G.maxBX = G.w - EDGE_THRESHOLD + 3; G.maxBY = G.h - EDGE_THRESHOLD + 3;
            const float width = (float)(G.maxBX - G.minBX), height = (float)(G.maxBY - G.minBY);
            const float W = 35;
            G.nCols = (int)(width / W); G.nRows = (int)(height / W);
            if (G.nCols < 1 || G.nRows < 1) { set_error("image too small for the number of pyramid levels"); return ORB_ERR_ARG; }
            G.wCell = (int)ceil(width / G.nCols); G.hCell = (int)ceil(height / G.nRows);
            G.cellCap = ((G.wCell + 1) / 2) * ((G.hCell + 1) / 2);
            G.cellBase = (int)cells.size();
            for (int i = 0; i < G.nRows; ++i) {
                const float iniY = (float)(G.minBY + i * G.hCell);
                float maxY = iniY + G.hCell + 6;
                if (iniY >= G.maxBY - 3) continue;
                if (maxY > G.maxBY) maxY = (float)G.maxBY;
                for (int j = 0; j < G.nCols; ++j) {
                    const float iniX = (float)(G.minBX + j * G.wCell);
                    float maxX = iniX + G.wCell + 6;
                    if (iniX >= G.maxBX - 6) continue;
                    if (maxX > G.maxBX) maxX = (float)G.maxBX;
                    CellDesc cd;
                    cd.level = (uint16_t)l; cd.x0 = (uint16_t)iniX; cd.y0 = (uint16_t)iniY;
                    cd.rw = (uint16_t)((int)maxX - (int)iniX); cd.rh = (uint16_t)((int)maxY - (int)iniY);
                    cd.offX = (uint16_t)(j * G.wCell); cd.offY = (uint16_t)(i * G.hCell); cd.pad = 0;
                    cd.listOff = (uint32_t)listOff;
                    listOff += G.cellCap;
                    cells.push_back(cd);
                }
            }
            G.nCells = (int)cells.size() - G.cellBase;
            {   // FAST blocks of 2 x 2 cells (partial at the right and bottom edges) and the TMA box covering the largest union window
                // of the level (width rounded up to 16 bytes: the box starts 16-byte aligned).  The skipped cells are trailing rows and
                // columns, so the listed cells form a row-major grid.
                int gx = 0;
                while (gx < G.nCells && cells[G.cellBase + gx].y0 == cells[G.cellBase].y0) ++gx;
                const int gy = gx ? G.nCells / gx : 0;
                int bw = 16, bh = 7, iwm = 0, ihm = 0;
                for (int by = 0; by < gy; by += 2)
                    for (int bx = 0; bx < gx; bx += 2) {
                        FastBlock b = {};
                        b.level = (uint16_t)l; b.ncx = (uint8_t)std::min(2, gx - bx); b.ncy = (uint8_t)std::min(2, gy - by);
                        const CellDesc& c0 = cells[G.cellBase + by * gx + bx];
                        b.x0 = c0.x0; b.y0 = c0.y0;
                        int iw = 0, ih = 0;
                        for (int k = 0; k < b.ncx * b.ncy; ++k) {
                            b.cell[k] = G.cellBase + (by + k / b.ncx) * gx + bx + k % b.ncx;
                            const CellDesc& c = cells[b.cell[k]];
                            if (c.rw < 7 || c.rh < 7) continue;   // no interior: the kernel reports 0 corners
                            iw = std::max(iw, c.x0 + c.rw - 3 - (b.x0 + 3)); ih = std::max(ih, c.y0 + c.rh - 3 - (b.y0 + 3));
                        }
                        b.iw = (uint16_t)iw; b.ih = (uint16_t)ih;
                        if (iw > 0) {
                            bw = std::max(bw, (b.x0 & 15) + iw + 6); bh = std::max(bh, ih + 6);
                            iwm = std::max(iwm, iw); ihm = std::max(ihm, ih);
                        }
                        fastBlocks.push_back(b);
                    }
                G.fastBoxW = (int)alignUp(bw, 16); G.fastBoxH = bh;
                smemFast = std::max(smemFast, (size_t)fast_smem_layout(G.fastBoxW, G.fastBoxH, iwm, ihm).total);
            }
            G.candOff = (uint32_t)candOff; G.candCap = (uint32_t)G.nCells * G.cellCap;
            if (G.candCap >= (1u << 24)) { set_error("too many FAST cells per level for the quadtree's 24-bit candidate index"); return ORB_ERR_ARG; }
            candOff += alignUp(G.candCap, 64);
            G.nDesired = featPerLevel[l];
            G.nIni = (int)roundf((float)(G.maxBX - G.minBX) / (G.maxBY - G.minBY));
            if (G.nIni < 1) { set_error("aspect ratio < 0.5: reference divides by zero (ORBextractor.cc:559-561)"); return ORB_ERR_ASPECT; }
            G.hX = (float)(G.maxBX - G.minBX) / G.nIni;
            G.qtNodes = std::max(G.nDesired + 3, 4 * G.nIni) + 4;
            if (G.qtNodes > QT_MAX_NODES) { set_error("nfeatures too large for the quadtree kernel"); return ORB_ERR_ARG; }
            qtEnd = std::max(qtEnd, qt_layout(G.qtNodes, G.nCells).cand);
            G.selCap = std::max(G.nDesired + 3, 4 * G.nIni);
            G.selOff = selOff; selOff += G.selCap;
            maxKp += G.selCap;
            G.scale = scale[l];
            G.sizeScaled = (float)(int)(PATCH_SIZE * scale[l]);
            G.blurTileBase = blurTiles;
            G.blurTilesX = (G.w + BL_TW - 1) / BL_TW; G.blurTilesY = (G.h + BL_TH - 1) / BL_TH;
            blurTiles += G.blurTilesX * G.blurTilesY;
            G.area2x = 0;
            G.xtabOff = (uint32_t)xtab.size(); G.ytabOff = (uint32_t)ytab.size();
            if (l > 0) {
                const LevelGeom& S = P.lv[l - 1];
                if (S.w == 2 * G.w && S.h == 2 * G.h) G.area2x = 1;
                const double sx_ = (double)S.w / G.w, sy_ = (double)S.h / G.h;
                for (int dx = 0; dx < G.w; ++dx) {
                    float fx = (float)((dx + 0.5) * sx_ - 0.5);
                    int sx = cvFloorD(fx);
                    fx -= sx;
                    if (sx < 0) { fx = 0; sx = 0; }
                    if (sx >= S.w - 1) { fx = 0; sx = S.w - 1; }
                    short4 t;
                    t.x = (short)sx; t.y = (short)std::min(sx + 1, S.w - 1);
                    t.z = (short)cvRoundF((1.f - fx) * 2048); t.w = (short)cvRoundF(fx * 2048);
                    xtab.push_back(t);
                }
                for (int dy = 0; dy < G.h; ++dy) {
                    float fy = (float)((dy + 0.5) * sy_ - 0.5);
                    int sy = cvFloorD(fy);
                    fy -= sy;
                    short4 t;
                    t.x = (short)std::min(std::max(sy, 0), S.h - 1); t.y = (short)std::min(std::max(sy + 1, 0), S.h - 1);
                    t.z = (short)cvRoundF((1.f - fy) * 2048); t.w = (short)cvRoundF(fy * 2048);
                    ytab.push_back(t);
                }
                // TMA box that covers the sources of any PYR_TILE_W x PYR_TILE_H destination tile (start column aligned down to 16 bytes)
                int bw = 16, bh = 2;
                for (int dx0 = 0; dx0 < G.w; dx0 += PYR_TILE_W) {
                    const int first = xtab[G.xtabOff + dx0].x & ~15, last = xtab[G.xtabOff + std::min(dx0 + PYR_TILE_W - 1, G.w - 1)].y;
                    bw = std::max(bw, last - first + 1);
                }
                for (int dy0 = 0; dy0 < G.h; dy0 += PYR_TILE_H)
                    bh = std::max(bh, ytab[G.ytabOff + std::min(dy0 + PYR_TILE_H - 1, G.h - 1)].y - ytab[G.ytabOff + dy0].x + 1);
                G.pyrBoxW = (int)alignUp(bw, 16); G.pyrBoxH = bh;
            }
        }
        P.pyrFrameStride = planeOff;
        P.nCellsTotal = (int)cells.size();
        P.nFastBlocks = (int)fastBlocks.size();
        P.cellCountStride = alignUp(cells.size(), 32);
        P.cellListStride = alignUp(listOff, 64);
        P.candStride = alignUp(candOff, 64);
        P.selStride = (size_t)selOff;
        P.blurTilesTotal = blurTiles;
        smemQt = alignUp((size_t)qtEnd + 6 * QT_SMEM_CANDS, 128);   // one quadtree warp's slab
        P.qtSlab = (int)smemQt;
        smemAs = 2 * P.selStride * sizeof(int);
        rows = r; cols = c;
        return ORB_OK;
    }

    int allocate() {
        // geometry + buffers are sized for the largest image; smaller images reuse them
        std::vector<short4> xtab, ytab;
        int rc = configure(maxH, maxW, xtab, ytab);
        if (rc) return rc;
        CK(cudaSetDevice(device));
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, device));
        if (orbx::require_sm90(prop.major, prop.minor)) return ORB_ERR_CUDA;
        const size_t B = (size_t)maxBatch;
        CK(cudaMalloc(&d_pyr, P.pyrFrameStride * B));
        CK(cudaMalloc(&d_blur, P.pyrFrameStride * B));
        capPyr = P.pyrFrameStride; capCells = cells.size() + cells.size() / 4 + 64; capCellCount = alignUp(capCells, 32);
        capCellList = P.cellListStride + P.cellListStride / 8; capCand = P.candStride + P.candStride / 8;
        capSel = P.selStride + 64; capX = xtab.size() + 64; capY = ytab.size() + 64;
        CK(cudaMalloc(&d_cells, sizeof(CellDesc) * capCells));
        CK(cudaMalloc(&d_fastBlocks, sizeof(FastBlock) * capCells));   // never more blocks than cells
        CK(cudaMalloc(&d_cellCount, sizeof(int) * capCellCount * B));
        CK(cudaMalloc(&d_cellList, sizeof(uint32_t) * capCellList * B));
        CK(cudaMalloc(&d_cand, sizeof(uint32_t) * capCand * B));
        CK(cudaMalloc(&d_nodeOf, sizeof(uint16_t) * capCand * B));
        CK(cudaMalloc(&d_sel, sizeof(SelKp) * capSel * B));
        CK(cudaMalloc(&d_selCount, sizeof(int) * kMaxLevels * B));
        CK(cudaMalloc(&d_dstIndex, sizeof(int) * capSel * B));
        CK(cudaMalloc(&d_status, sizeof(int) * B));
        CK(cudaMalloc(&d_maps, sizeof(TmaMaps)));
        CK(cudaMalloc(&d_blurMaps, sizeof(TmaMaps)));
        CK(cudaMalloc(&d_xtab, sizeof(short4) * capX));
        CK(cudaMalloc(&d_ytab, sizeof(short4) * capY));
        CK(cudaMalloc(&d_img, (size_t)P.lv[0].pitch * maxH * B));
        outCapInternal = (int)capSel;
        CK(cudaMalloc(&d_outKp, sizeof(OrbKeyPoint) * outCapInternal * B));
        CK(cudaMalloc(&d_outDesc, (size_t)32 * outCapInternal * B));
        CK(cudaMalloc(&d_outN, sizeof(int) * B));
        CK(cudaMalloc(&d_outMono, sizeof(int) * B));
        CK(cudaMallocHost(&h_counts, sizeof(int) * 3 * B));
        CK(cudaMallocHost(&h_stereoStatus, sizeof(int) * B));
        CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        CK(cudaStreamCreateWithFlags(&stream2, cudaStreamNonBlocking));
        CK(orbx::make_blocking_event(&evWait));
        CK(cudaEventCreateWithFlags(&evFork, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&evJoin, cudaEventDisableTiming));
        CK(cudaMemcpyToSymbol(c_pattern, h_pattern, sizeof(h_pattern)));
        CK(cudaMemcpyToSymbol(c_umax, umax, sizeof(umax)));
        maxSmemFast = 96 * 1024;   // a cell interior is at most 69 x 69 px, so a 2 x 2 block needs at most ~90 KB
        maxSmemQt = smemQt + 4 * 1024; maxSmemAs = 2 * capSel * sizeof(int);   // per quadtree warp: room for other aspect ratios
        if (maxSmemQt > prop.sharedMemPerBlockOptin) { set_error("nfeatures too large for the quadtree kernel's shared memory"); return ORB_ERR_ARG; }
        // process-wide monotonic maxima (device_utils.cuh): a smaller handle created later must not lower another handle's limit
        if (ensure_dynamic_smem(fast_cells_kernel, maxSmemFast, device) ||
            ensure_dynamic_smem(assemble_kernel, std::max<size_t>(maxSmemAs, 1024), device)) return ORB_ERR_CUDA;
        // quadtree warps per CTA: the most resident warps per SM by the occupancy calculator, the fewest warps per CTA among equals
        qtWarps = 0;
        for (int w = 1, best = 0; w <= QT_MAX_WARPS && w * maxSmemQt <= prop.sharedMemPerBlockOptin; w *= 2) {
            int nb = 0;
            if (ensure_dynamic_smem(quadtree_kernel, w * maxSmemQt, device)) return ORB_ERR_CUDA;
            CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, quadtree_kernel, 32 * w, w * smemQt));
            if (nb * w > best) { best = nb * w; qtWarps = w; }
        }
        if (!qtWarps) { set_error("the quadtree kernel does not fit on the device"); return ORB_ERR_CUDA; }
        maxKpAlloc = (int)capSel;
        rows = cols = 0;   // force set_size on first use
        return set_size(maxH, maxW);
    }
    size_t maxSmemFast = 0, maxSmemQt = 0, maxSmemAs = 0;
    int qtWarps = 0;
    size_t capPyr = 0, capCells = 0, capCellCount = 0, capCellList = 0, capCand = 0, capSel = 0, capX = 0, capY = 0;
    int maxKpAlloc = 0;

    int set_size(int r, int c) {
        if (r == rows && c == cols) return ORB_OK;
        if (r > maxH || c > maxW) { set_error("image larger than max_width x max_height given to orbx_create"); return ORB_ERR_ARG; }
        std::vector<short4> xtab, ytab;
        int rc = configure(r, c, xtab, ytab);
        if (rc) { rows = cols = 0; return rc; }
        if (P.pyrFrameStride > capPyr || cells.size() > capCells || P.cellCountStride > capCellCount || P.cellListStride > capCellList ||
            P.candStride > capCand || P.selStride > capSel || xtab.size() > capX || ytab.size() > capY || smemQt > maxSmemQt ||
            smemFast > maxSmemFast || smemAs > maxSmemAs) {
            rows = cols = 0;
            set_error("image geometry exceeds the buffers sized at orbx_create (aspect ratio very different from max_width x max_height?)");
            return ORB_ERR_ARG;
        }
        CK(cudaSetDevice(device));
        CK(cudaStreamSynchronize(stream));
        if (!cells.empty()) CK(cudaMemcpy(d_cells, cells.data(), sizeof(CellDesc) * cells.size(), cudaMemcpyHostToDevice));
        if (!fastBlocks.empty()) CK(cudaMemcpy(d_fastBlocks, fastBlocks.data(), sizeof(FastBlock) * fastBlocks.size(), cudaMemcpyHostToDevice));
        if (!xtab.empty()) CK(cudaMemcpy(d_xtab, xtab.data(), sizeof(short4) * xtab.size(), cudaMemcpyHostToDevice));
        if (!ytab.empty()) CK(cudaMemcpy(d_ytab, ytab.data(), sizeof(short4) * ytab.size(), cudaMemcpyHostToDevice));
        P.pyr = d_pyr; P.blur = d_blur; P.cells = d_cells; P.fastBlocks = d_fastBlocks; P.cellCount = d_cellCount; P.cellList = d_cellList;
        P.cand = d_cand; P.nodeOf = d_nodeOf; P.sel = d_sel; P.selCount = d_selCount; P.dstIndex = d_dstIndex;
        P.status = d_status; P.xtab = d_xtab; P.ytab = d_ytab;
        for (int l = 0; l < nlevels; ++l) {
            const LevelGeom& G = P.lv[l];
            if (!encode_plane_map(&maps.lv[l], d_pyr + G.planeOff, G.w, G.h, maxBatch, G.pitch, P.pyrFrameStride, G.fastBoxW, G.fastBoxH)) {
                set_error("cuTensorMapEncodeTiled failed for a pyramid level (TMA descriptors are required)");
                rows = cols = 0;
                return ORB_ERR_CUDA;
            }
        }
        CK(cudaMemcpy(d_maps, &maps, sizeof(TmaMaps), cudaMemcpyHostToDevice));
        for (int l = 0; l < nlevels; ++l) {
            const LevelGeom& G = P.lv[l];
            if (!encode_plane_map(&blurMaps.lv[l], d_pyr + G.planeOff, G.w, G.h, maxBatch, G.pitch, P.pyrFrameStride, BL_SP, BL_TH + 6)) {
                set_error("cuTensorMapEncodeTiled failed for a pyramid level (blur tile)");
                rows = cols = 0;
                return ORB_ERR_CUDA;
            }
        }
        CK(cudaMemcpy(d_blurMaps, &blurMaps, sizeof(TmaMaps), cudaMemcpyHostToDevice));
        for (int l = 2; l < nlevels; ++l) {     // level 1 reads level 0, which may alias the caller's frames: encoded per call
            const LevelGeom& S = P.lv[l - 1];
            if (P.lv[l].area2x || P.lv[l].pyrBoxW > 256 || P.lv[l].pyrBoxH > 256 ||
                !encode_plane_map(&pyrMaps.lv[l], d_pyr + S.planeOff, S.w, S.h, maxBatch, S.pitch, P.pyrFrameStride, P.lv[l].pyrBoxW, P.lv[l].pyrBoxH)) P.lv[l].pyrBoxW = 0;
        }
        return ORB_OK;
    }

    // Enqueue the whole pipeline for `batch` frames whose level-0 planes are described by (lv0, pitch, stride).
    int enqueue(const uint8_t* lv0, size_t lv0Pitch, size_t lv0Stride, int batch, int lap0, int lap1,
                OrbKeyPoint* outKp, uint8_t* outDesc, int cap, int* outN, int* outMono, cudaStream_t st) {
        ExtractParams Q = P;
        Q.batch = batch; Q.lap0 = lap0; Q.lap1 = lap1;
        Q.lv0 = lv0; Q.lv0Pitch = lv0Pitch; Q.lv0FrameStride = lv0Stride;
        Q.outKp = outKp; Q.outDesc = outDesc; Q.outCap = cap; Q.outN = outN; Q.outMono = outMono;
        launches = 0;
        CK(cudaMemsetAsync(d_status, 0, sizeof(int) * batch, st));
        // level 0: TMA straight from the caller's frames when base / strides are 16-byte aligned, else from an internal copy
        CUtensorMap map0, mapBlur0;
        if (!encode_plane_map(&map0, lv0, Q.lv[0].w, Q.lv[0].h, batch, lv0Pitch, lv0Stride, Q.lv[0].fastBoxW, Q.lv[0].fastBoxH) ||
            !encode_plane_map(&mapBlur0, lv0, Q.lv[0].w, Q.lv[0].h, batch, lv0Pitch, lv0Stride, BL_SP, BL_TH + 6)) {
            Q.src = lv0; Q.srcStep = lv0Pitch; Q.srcFrameStride = lv0Stride;
            copy_level0_kernel<<<dim3((Q.cols + 255) / 256, Q.rows, batch), 256, 0, st>>>(Q);
            ++launches;
            Q.lv0 = d_pyr + Q.lv[0].planeOff; Q.lv0Pitch = Q.lv[0].pitch; Q.lv0FrameStride = Q.pyrFrameStride;
            map0 = maps.lv[0];
            mapBlur0 = blurMaps.lv[0];
        }
        if (profiling) for (int i = 0; i < 7; ++i) if (!evStage[i]) CK(cudaEventCreate(&evStage[i]));
        if (profiling) CK(cudaEventRecord(evStage[0], st));
        // pyramid: levels depend on each other
        for (int l = 1; l < nlevels; ++l) {
            CUtensorMap srcMap;
            bool tma = Q.lv[l].pyrBoxW > 0 && !Q.lv[l].area2x && Q.lv[l].pyrBoxW <= 256 && Q.lv[l].pyrBoxH <= 256 &&
                       Q.lv[l].pyrBoxW * Q.lv[l].pyrBoxH <= 48 * 1024;   // default dynamic shared-memory limit
            if (tma && l == 1) tma = encode_plane_map(&srcMap, Q.lv0, Q.lv[0].w, Q.lv[0].h, batch, Q.lv0Pitch, Q.lv0FrameStride, Q.lv[1].pyrBoxW, Q.lv[1].pyrBoxH);
            else if (tma) srcMap = pyrMaps.lv[l];
            const int tileH = tma ? PYR_TILE_H : 8;   // pyr_resize_kernel: one destination row per thread
            dim3 blk(32, 8), grd((Q.lv[l].w + PYR_TILE_W - 1) / PYR_TILE_W, (Q.lv[l].h + tileH - 1) / tileH, batch);
            if (tma) pyr_resize_tma_kernel<<<grd, blk, (size_t)Q.lv[l].pyrBoxW * Q.lv[l].pyrBoxH, st>>>(Q, l, srcMap);
            else pyr_resize_kernel<<<grd, blk, 0, st>>>(Q, l);     // exact 2x decimation (INTER_AREA promotion) or a box TMA cannot express
            ++launches;
        }
        if (profiling) CK(cudaEventRecord(evStage[1], st));
        // blur runs on a forked stream, concurrently with detection (in line when profiling, so that events bracket it)
        cudaStream_t sb = profiling ? st : stream2;
        if (!profiling) {
            CK(cudaEventRecord(evFork, st));
            CK(cudaStreamWaitEvent(stream2, evFork, 0));
        }
        blur_kernel<<<dim3(Q.blurTilesTotal, batch), BL_NT, 0, sb>>>(Q, mapBlur0, d_blurMaps, 1);
        ++launches;
        if (!profiling) CK(cudaEventRecord(evJoin, stream2));
        if (profiling) CK(cudaEventRecord(evStage[2], st));
        fast_cells_kernel<<<dim3(Q.nFastBlocks, batch), FAST_NT, smemFast, st>>>(Q, map0, d_maps);
        ++launches;
        if (profiling) CK(cudaEventRecord(evStage[3], st));
        quadtree_kernel<<<dim3(nlevels, (batch + qtWarps - 1) / qtWarps), 32 * qtWarps, qtWarps * smemQt, st>>>(Q);
        ++launches;
        if (profiling) CK(cudaEventRecord(evStage[4], st));
        assemble_kernel<<<batch, AS_NT, smemAs, st>>>(Q);
        ++launches;
        if (profiling) CK(cudaEventRecord(evStage[5], st));
        if (!profiling) CK(cudaStreamWaitEvent(st, evJoin, 0));
        orient_describe_kernel<<<dim3((unsigned)((Q.selStride + DS_NT / 32 - 1) / (DS_NT / 32)), batch), DS_NT, 0, st>>>(Q);
        ++launches;
        if (profiling) CK(cudaEventRecord(evStage[6], st));
        CK(cudaGetLastError());
        lastQ = Q; hasLast = true;
        return ORB_OK;
    }
};

}  // namespace orbx

using namespace orbx;

struct orbx_handle { Extractor e; };

namespace orbx {
int handle_device(const orbx_handle* h) { return h->e.device; }
extern thread_local int g_undistort_launches;
int check_camera(const OrbPinholeCamera* cam, const char* where);
int undistort_enqueue(const OrbPinholeCamera* cam, int batch, const OrbKeyPoint* kps, const int* n, int cap, OrbKeyPoint* out, cudaStream_t st,
                      const char* where);
}  // namespace orbx

extern "C" {

const char* orb_last_error(void) { return g_err.c_str(); }
int orb_abi_version(void) { return 1; }
int orb_compiled_sm(void) { return 100; }

int orbx_create(orbx_handle** out, int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST,
                int max_width, int max_height, int max_batch, int device) {
    if (!out || nfeatures < 1 || nlevels < 1 || nlevels > kMaxLevels || !(scaleFactor > 1.0f) || max_width < 1 || max_height < 1 ||
        max_batch < 1 || iniThFAST < 1 || minThFAST < 1 || minThFAST > iniThFAST) {
        set_error("orbx_create: bad argument");
        return ORB_ERR_ARG;
    }
    if (int rc = check_device(device)) return rc;
    orbx_handle* h = new orbx_handle();
    Extractor& e = h->e;
    e.nfeatures = nfeatures; e.nlevels = nlevels; e.iniTh = iniThFAST; e.minTh = minThFAST; e.scaleFactor = scaleFactor;
    e.device = device; e.maxW = max_width; e.maxH = max_height; e.maxBatch = max_batch;
    e.init_tables();
    int rc = e.allocate();
    if (rc) { delete h; return rc; }
    *out = h;
    return ORB_OK;
}

void orbx_destroy(orbx_handle* h) { delete h; }

int orbx_get_levels(const orbx_handle* h) { return h ? h->e.nlevels : ORB_ERR_ARG; }

int orbx_get_tables(const orbx_handle* h, float* s, float* is, float* g, float* ig, int* fpl) {
    if (!h) return ORB_ERR_ARG;
    const Extractor& e = h->e;
    for (int i = 0; i < e.nlevels; ++i) {
        if (s) s[i] = e.scale[i];
        if (is) is[i] = e.invScale[i];
        if (g) g[i] = e.sigma2[i];
        if (ig) ig[i] = e.invSigma2[i];
        if (fpl) fpl[i] = e.featPerLevel[i];
    }
    return ORB_OK;
}

int orbx_max_keypoints(const orbx_handle* h) { return h ? h->e.maxKpAlloc : ORB_ERR_ARG; }

int orbx_extract_batch_device(orbx_handle* h, const uint8_t* d_images, int batch, int rows, int cols, size_t step,
                              size_t frame_stride, int lap0, int lap1, OrbKeyPoint* d_kps, uint8_t* d_desc, int cap,
                              int* d_n, int* d_mono, void* stream) {
    if (!h || !d_kps || !d_desc || !d_n || !d_mono || cap < 1) { set_error("orbx_extract_batch_device: bad argument"); return ORB_ERR_ARG; }
    if (!d_images || rows <= 0 || cols <= 0 || batch <= 0) return ORB_ERR_EMPTY;
    Extractor& e = h->e;
    if (batch > e.maxBatch) { set_error("batch larger than max_batch"); return ORB_ERR_ARG; }
    if (step < (size_t)cols) { set_error("step < cols"); return ORB_ERR_ARG; }
    CK(cudaSetDevice(e.device));
    int rc = e.set_size(rows, cols);
    if (rc) return rc;
    return e.enqueue(d_images, step, frame_stride, batch, lap0, lap1, d_kps, d_desc, cap, d_n, d_mono, (cudaStream_t)stream);
}

int orbx_extract_batch(orbx_handle* h, const uint8_t* images, int batch, int rows, int cols, size_t step, size_t frame_stride,
                       int lap0, int lap1, OrbKeyPoint* kps, uint8_t* desc, int cap, int* n, int* mono) {
    if (!h || !kps || !desc || !n || !mono || cap < 1) { set_error("orbx_extract_batch: bad argument"); return ORB_ERR_ARG; }
    if (!images || rows <= 0 || cols <= 0 || batch <= 0) return ORB_ERR_EMPTY;
    Extractor& e = h->e;
    if (batch > e.maxBatch) { set_error("batch larger than max_batch"); return ORB_ERR_ARG; }
    if (step < (size_t)cols) { set_error("step < cols"); return ORB_ERR_ARG; }
    CK(cudaSetDevice(e.device));
    int rc = e.set_size(rows, cols);
    if (rc) return rc;
    const size_t pitch = e.P.lv[0].pitch, fstride = pitch * rows;
    cudaStream_t st = e.stream;
    if (batch > 1 && frame_stride == step * rows) {
        CK(cudaMemcpy2DAsync(e.d_img, pitch, images, step, cols, (size_t)rows * batch, cudaMemcpyHostToDevice, st));
    } else {
        for (int f = 0; f < batch; ++f)
            CK(cudaMemcpy2DAsync(e.d_img + f * fstride, pitch, images + f * frame_stride, step, cols, rows, cudaMemcpyHostToDevice, st));
    }
    const int icap = e.outCapInternal;
    rc = e.enqueue(e.d_img, pitch, fstride, batch, lap0, lap1, e.d_outKp, e.d_outDesc, icap, e.d_outN, e.d_outMono, st);
    if (rc) return rc;
    int* hn = e.h_counts; int* hm = hn + e.maxBatch; int* hs = hm + e.maxBatch;
    CK(cudaMemcpyAsync(hn, e.d_outN, sizeof(int) * batch, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(hm, e.d_outMono, sizeof(int) * batch, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(hs, e.d_status, sizeof(int) * batch, cudaMemcpyDeviceToHost, st));
    const bool slabToSlab = cap == icap && batch > 1;
    if (slabToSlab) {
        // the caller's buffers have the internal capacity -> two bulk copies queued behind the kernels, ONE synchronisation per call
        // (rows beyond n[f] are unspecified; on a capacity error the buffers hold whatever the device wrote)
        CK(cudaMemcpyAsync(kps, e.d_outKp, sizeof(OrbKeyPoint) * (size_t)icap * batch, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(desc, e.d_outDesc, (size_t)32 * icap * batch, cudaMemcpyDeviceToHost, st));
    }
    if (batch > 1) CK(orbx::wait_stream_blocking(st, e.evWait)); else CK(cudaStreamSynchronize(st));
    int worst = ORB_OK;
    for (int f = 0; f < batch; ++f) {
        n[f] = hn[f]; mono[f] = hm[f];
        if (hs[f] || hn[f] > cap) { worst = ORB_ERR_CAPACITY; set_error("keypoint capacity exceeded"); }
    }
    if (!slabToSlab) {
        for (int f = 0; f < batch; ++f) {
            if (hs[f] || hn[f] > cap || hn[f] <= 0) continue;
            CK(cudaMemcpyAsync(kps + (size_t)f * cap, e.d_outKp + (size_t)f * icap, sizeof(OrbKeyPoint) * hn[f], cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(desc + (size_t)f * cap * 32, e.d_outDesc + (size_t)f * icap * 32, (size_t)32 * hn[f], cudaMemcpyDeviceToHost, st));
        }
        CK(cudaStreamSynchronize(st));
    }
    return worst;
}

int orbx_extract(orbx_handle* h, const uint8_t* image, int rows, int cols, size_t step, int lap0, int lap1,
                 OrbKeyPoint* kps, uint8_t* desc, int cap, int* n, int* mono) {
    return orbx_extract_batch(h, image, 1, rows, cols, step, step * (size_t)(rows > 0 ? rows : 0), lap0, lap1, kps, desc, cap, n, mono);
}

int orbx_get_level_size(const orbx_handle* h, int level, int* w, int* hh) {
    if (!h || level < 0 || level >= h->e.nlevels || h->e.rows == 0) return ORB_ERR_ARG;
    *w = h->e.P.lv[level].w; *hh = h->e.P.lv[level].h;
    return ORB_OK;
}

int orbx_copy_level(orbx_handle* h, int frame, int level, int blurred, uint8_t* dst) {
    if (!h || !dst || level < 0 || level >= h->e.nlevels || frame < 0 || frame >= h->e.maxBatch || h->e.rows == 0) return ORB_ERR_ARG;
    Extractor& e = h->e;
    CK(cudaSetDevice(e.device));
    const LevelGeom& G = e.P.lv[level];
    const uint8_t* src;
    size_t pitch = G.pitch;
    if (level == 0 && !blurred) {
        // the plane the last call read: the staging copy, the internal copy of unaligned frames, or the caller's own device frames
        if (!e.hasLast || frame >= e.lastQ.batch) { set_error("orbx_copy_level: level 0 of a frame the last call did not process"); return ORB_ERR_ARG; }
        src = e.lastQ.lv0 + (size_t)frame * e.lastQ.lv0FrameStride;
        pitch = e.lastQ.lv0Pitch;
    } else src = (blurred ? e.d_blur : e.d_pyr) + (size_t)frame * e.P.pyrFrameStride + G.planeOff;
    CK(cudaMemcpy2D(dst, G.w, src, pitch, G.w, G.h, cudaMemcpyDeviceToHost));
    return ORB_OK;
}

int orbx_copy_candidates(orbx_handle* h, int frame, int level, int* xys, int cap) {
    if (!h || !xys || level < 0 || level >= h->e.nlevels || frame < 0 || frame >= h->e.maxBatch || h->e.rows == 0) return ORB_ERR_ARG;
    Extractor& e = h->e;
    CK(cudaSetDevice(e.device));
    const LevelGeom& G = e.P.lv[level];
    std::vector<int> counts(G.nCells);
    if (G.nCells == 0) return 0;
    CK(cudaMemcpy(counts.data(), e.d_cellCount + (size_t)frame * e.P.cellCountStride + G.cellBase, sizeof(int) * G.nCells, cudaMemcpyDeviceToHost));
    int total = 0;
    std::vector<uint32_t> buf(G.cellCap);
    for (int c = 0; c < G.nCells; ++c) {
        const int cnt = counts[c];
        if (cnt > G.cellCap) return ORB_ERR_CAPACITY;
        if (cnt) CK(cudaMemcpy(buf.data(), e.d_cellList + (size_t)frame * e.P.cellListStride + e.cells[G.cellBase + c].listOff, sizeof(uint32_t) * cnt, cudaMemcpyDeviceToHost));
        for (int k = 0; k < cnt; ++k) {
            if (total < cap) { xys[3 * total] = cand_x(buf[k]); xys[3 * total + 1] = cand_y(buf[k]); xys[3 * total + 2] = cand_s(buf[k]); }
            ++total;
        }
    }
    return total;
}

int orbx_stereo_matches_device(orbx_handle* left, orbx_handle* right, int batch, const OrbKeyPoint* d_kpsL, const uint8_t* d_descL, const int* d_nL, int capL,
                               const OrbKeyPoint* d_kpsR, const uint8_t* d_descR, const int* d_nR, int capR, float mb, float mbf, float* d_uRight,
                               float* d_depth, void* stream) {
    if (!left || !right || batch < 1 || !d_kpsL || !d_descL || !d_nL || !d_kpsR || !d_descR || !d_nR || capL < 1 || capR < 1 || capR > 65535 || !d_uRight || !d_depth ||
        !(mb > 0) || !(mbf > 0)) { set_error("orbx_stereo_matches_device: bad argument"); return ORB_ERR_ARG; }
    Extractor &L = left->e, &R = right->e;
    if (!L.hasLast || !R.hasLast || L.lastQ.batch < batch || R.lastQ.batch < batch || L.rows != R.rows || L.cols != R.cols || L.nlevels != R.nlevels ||
        L.scaleFactor != R.scaleFactor || L.device != R.device || batch > L.maxBatch) {
        set_error("orbx_stereo_matches: both extractors must have processed the pair's images (same size, levels and scale factor) in their last call");
        return ORB_ERR_ARG;
    }
    CK(cudaSetDevice(L.device));
    cudaStream_t st = (cudaStream_t)stream;
    if (!L.d_stereoSad) CK(cudaMalloc(&L.d_stereoSad, sizeof(int) * L.capSel * (size_t)L.maxBatch));
    if (capL > (int)L.capSel) { set_error("orbx_stereo_matches: capL larger than the left extractor's keypoint capacity"); return ORB_ERR_CAPACITY; }
    StereoParams Q;
    Q.L = L.lastQ; Q.R = R.lastQ;
    Q.kpsL = d_kpsL; Q.kpsR = d_kpsR; Q.descL = d_descL; Q.descR = d_descR; Q.nL = d_nL; Q.nR = d_nR; Q.capL = capL; Q.capR = capR;
    Q.mb = mb; Q.mbf = mbf; Q.uRight = d_uRight; Q.depth = d_depth; Q.sad = L.d_stereoSad; Q.status = L.d_status;
    CK(cudaMemsetAsync(L.d_status, 0, sizeof(int) * batch, st));
    stereo_matches_kernel<<<batch, ST_NT, 0, st>>>(Q);
    CK(cudaGetLastError());
    return ORB_OK;
}

int orbx_stereo_matches(orbx_handle* left, orbx_handle* right, int batch, float mb, float mbf, float* uRight, float* depth, int cap) {
    if (!left || !right || !uRight || !depth || batch < 1) { set_error("orbx_stereo_matches: bad argument"); return ORB_ERR_ARG; }
    Extractor &L = left->e, &R = right->e;
    if (cap != L.outCapInternal) { set_error("orbx_stereo_matches: cap must equal orbx_max_keypoints(left)"); return ORB_ERR_ARG; }
    CK(cudaSetDevice(L.device));
    const size_t n = (size_t)L.outCapInternal * L.maxBatch;
    if (!L.d_stereoU) { CK(cudaMalloc(&L.d_stereoU, sizeof(float) * n)); CK(cudaMalloc(&L.d_stereoD, sizeof(float) * n)); }
    cudaStream_t st = L.stream;
    int rc = orbx_stereo_matches_device(left, right, batch, L.d_outKp, L.d_outDesc, L.d_outN, L.outCapInternal, R.d_outKp, R.d_outDesc, R.d_outN,
                                        R.outCapInternal, mb, mbf, L.d_stereoU, L.d_stereoD, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(uRight, L.d_stereoU, sizeof(float) * (size_t)cap * batch, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(depth, L.d_stereoD, sizeof(float) * (size_t)cap * batch, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(L.h_stereoStatus, L.d_status, sizeof(int) * batch, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int f = 0; f < batch; ++f)
        if (L.h_stereoStatus[f] & 4) { set_error("orbx_stereo_matches: a correlation window left the pyramid plane (keypoints not from this extractor?)"); return ORB_ERR_ARG; }
    return ORB_OK;
}

// mvImagePyramid[level] of the last call WITH the reflected frame ComputePyramid writes around it (src/ORBextractor.cc:1185-1191):
// (w + 2 border) x (h + 2 border), tightly packed.  The mono path never reads that frame (DESIGN.md), so it is materialised on request.
int orbx_copy_level_bordered(orbx_handle* h, int frame, int level, int border, uint8_t* dst) {
    if (!h || !dst || level < 0 || level >= h->e.nlevels || frame < 0 || frame >= h->e.maxBatch || border < 0 || border > 64 || !h->e.hasLast) {
        set_error("orbx_copy_level_bordered: bad argument"); return ORB_ERR_ARG;
    }
    Extractor& e = h->e;
    CK(cudaSetDevice(e.device));
    const LevelGeom& G = e.P.lv[level];
    const int W = G.w + 2 * border, H = G.h + 2 * border;
    uint8_t* d_tmp = nullptr;
    CK(cudaMalloc(&d_tmp, (size_t)W * H));
    border_copy_kernel<<<dim3((W + 255) / 256, H), 256, 0, e.stream>>>(e.lastQ, frame, level, border, d_tmp);
    cudaError_t err = cudaMemcpyAsync(dst, d_tmp, (size_t)W * H, cudaMemcpyDeviceToHost, e.stream);
    if (err == cudaSuccess) err = cudaStreamSynchronize(e.stream);
    cudaFree(d_tmp);
    if (err != cudaSuccess) { set_error(cudaGetErrorString(err)); return ORB_ERR_CUDA; }
    return ORB_OK;
}

int orbx_resident_slabs(const orbx_handle* h, const OrbKeyPoint** d_keypoints, const uint8_t** d_descriptors, const int** d_nkeypoints, int* cap) {
    if (!h || !d_keypoints || !d_descriptors || !d_nkeypoints || !cap) return ORB_ERR_ARG;
    *d_keypoints = h->e.d_outKp; *d_descriptors = h->e.d_outDesc; *d_nkeypoints = h->e.d_outN; *cap = h->e.outCapInternal;
    return ORB_OK;
}

int orbx_last_launch_count(const orbx_handle* h) { return h ? h->e.launches : ORB_ERR_ARG; }

int orbx_undistort_keypoints(orbx_handle* h, const OrbPinholeCamera* cam, int batch, OrbKeyPoint* kpsUn, int cap, const OrbKeyPoint** d_kpsUn) {
    g_undistort_launches = 0;
    if (!h || batch < 0 || (kpsUn && cap != h->e.outCapInternal)) { set_error("orbx_undistort_keypoints: bad argument"); return ORB_ERR_ARG; }
    if (int rc = check_camera(cam, "orbx_undistort_keypoints")) return rc;
    Extractor& e = h->e;
    if (batch > 0 && (!e.hasLast || e.lastQ.outKp != e.d_outKp || e.lastQ.batch < batch)) {
        set_error("orbx_undistort_keypoints: the handle's last call was not orbx_extract[_batch] of at least `batch` frames");
        return ORB_ERR_ARG;
    }
    CK(cudaSetDevice(e.device));
    const size_t slab = sizeof(OrbKeyPoint) * (size_t)e.outCapInternal * e.maxBatch;
    if (!e.d_outKpUn) {
        CK(cudaMalloc(&e.d_outKpUn, slab));
        CK(cudaMemset(e.d_outKpUn, 0, slab));
    }
    cudaStream_t st = e.stream;
    int rc = undistort_enqueue(cam, batch, e.d_outKp, e.d_outN, e.outCapInternal, e.d_outKpUn, st, "orbx_undistort_keypoints");
    if (rc) return rc;
    if (kpsUn && batch > 0) CK(cudaMemcpyAsync(kpsUn, e.d_outKpUn, sizeof(OrbKeyPoint) * (size_t)e.outCapInternal * batch, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (d_kpsUn) *d_kpsUn = e.d_outKpUn;
    return ORB_OK;
}

int orbx_set_profiling(orbx_handle* h, int on) {
    if (!h) return ORB_ERR_ARG;
    h->e.profiling = on != 0;
    return ORB_OK;
}

#ifdef QT_PHASES
// out[kMaxLevels * 9]: quadtree_kernel's phase counters per level (qt_phase) since the last call, which zeroes them.
int orbx_qt_phases(unsigned long long* out) {
    if (!out) return ORB_ERR_ARG;
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpyFromSymbol(out, orbx::qt_phase, sizeof(orbx::qt_phase)));
    static const unsigned long long zero[kMaxLevels * 9] = {};
    CK(cudaMemcpyToSymbol(orbx::qt_phase, zero, sizeof(zero)));
    return ORB_OK;
}
#endif

int orbx_get_stage_ms(orbx_handle* h, float* ms6) {
    if (!h || !ms6 || !h->e.evStage[6]) { set_error("orbx_get_stage_ms: no profiled call yet"); return ORB_ERR_ARG; }
    Extractor& e = h->e;
    CK(cudaSetDevice(e.device));
    CK(cudaEventSynchronize(e.evStage[6]));
    for (int i = 0; i < 6; ++i) CK(cudaEventElapsedTime(&ms6[i], e.evStage[i], e.evStage[i + 1]));
    return ORB_OK;
}

}  // extern "C"
