// Internal layout of the batched extractor (not part of the C-ABI).
#pragma once
#include <stdint.h>

namespace orbx {

constexpr int kMaxLevels = 16;
constexpr int EDGE_THRESHOLD = 19;   // reference src/ORBextractor.cc:73
constexpr int HALF_PATCH = 15;       // :72
constexpr int PATCH_SIZE = 31;       // :71

// Geometry of one pyramid level for the currently configured image size.
struct LevelGeom {
    int w, h, pitch;          // plane size; pitch is a multiple of 32 bytes
    uint32_t planeOff;        // byte offset of the plane inside one frame's pyramid buffer
    int minBX, minBY, maxBX, maxBY;   // detection window (reference :789-792)
    int nCols, nRows, wCell, hCell;   // FAST cell grid (:797-803)
    int cellBase, nCells;     // active cells of this level inside the frame's cell table
    int cellCap;              // list capacity of one cell (max NMS survivors)
    uint32_t candOff, candCap;        // candidate scratch of this level inside one frame
    int nDesired;             // mnFeaturesPerLevel[level]
    int selOff, selCap;       // selected-keypoint slots of this level inside one frame
    int nIni; float hX;       // quadtree roots (:559-561)
    int qtNodes;              // quadtree list capacity: max(nDesired + 3, 4 nIni) + 4
    float scale; float sizeScaled;    // mvScaleFactor[level], (float)(int)(31*scale)
    int area2x;               // level is an exact 2x decimation of the previous (cv::resize -> INTER_AREA)
    uint32_t xtabOff, ytabOff;        // resize coefficient tables (entries, not bytes)
    int blurTileBase, blurTilesX, blurTilesY;   // flattened tile index range of the blur launch
    int fastBoxW, fastBoxH;   // TMA box of the FAST cell ROI: width (multiple of 16 bytes) x height
    int pyrBoxW, pyrBoxH;     // TMA box (in level l-1) that covers the sources of one PYR_TILE_W x PYR_TILE_H destination tile of this level
};

// One active FAST cell (cells skipped by the reference's `continue`s are not listed).
struct CellDesc {
    uint16_t level;
    uint16_t x0, y0;          // ROI origin in level coordinates
    uint16_t rw, rh;          // ROI size (detection interior is [3,rw-3) x [3,rh-3))
    uint16_t offX, offY;      // j*wCell, i*hCell: added to ROI-relative corner coordinates (:866-867)
    uint16_t pad;
    uint32_t listOff;         // offset of this cell's list inside one frame's cell-list buffer
};

// Up to 2 x 2 neighbouring cells of one level that one FAST CTA detects together.  The cells' interiors tile the level, so their
// union is one window: the ROI of the first cell grown to the bottom-right of the others.
struct FastBlock {
    uint16_t level;
    uint16_t x0, y0;          // ROI origin of the first cell = origin of the union window
    uint16_t iw, ih;          // union detection interior [3, 3 + iw) x [3, 3 + ih) of the window (0 x 0: every cell has rw or rh < 7)
    uint8_t ncx, ncy;         // cells across / down
    int cell[4];              // indices into the cell table, row-major inside the block
};

// Shared-memory carve-up of one FAST block CTA (byte offsets; the TMA tile is first, at 0).  Host and device both use it, so
// the launch size is the maximum of exactly what the kernel addresses.
struct FastSmem { int sp, nwp, score, bits, rowOff, list, total; };
__host__ __device__ inline FastSmem fast_smem_layout(int boxW, int boxH, int iw, int ih) {
    FastSmem L;
    L.sp = 4 * ((iw + 3) >> 2) + 8;                    // score-map pitch: whole quads + 4-byte left margin + right ring
    L.nwp = (iw + 31) >> 5;                            // keep-bitmap words per row
    L.score = (boxW * boxH + 127) & ~127;              // (ih + 2) * sp: interior (y, x) at (y + 1) * sp + x + 4
    L.bits = L.score + ((L.sp * (ih + 2) + 15) & ~15); // lo bitmap, then hi bitmap: ih * nwp words each
    L.rowOff = L.bits + 8 * ih * L.nwp;                // one int per (cell, row): at most two cells share a row
    L.list = L.rowOff + 8 * ih;                        // candidates (y << 8 | x), at most iw * ih
    L.total = L.list + 2 * iw * ih;
    return L;
}

// Selected keypoint before output assembly (its angle is computed by orient_describe_kernel).
struct SelKp {
    int16_t x, y;             // level coordinates (border offset already added)
    int32_t response;
};

// Quadtree list nodes and the shared-memory slab of one quadtree warp (one (level, frame) problem).  Host and device both use the
// layout, so the launch size is exactly what the kernel addresses.  A node id shares nodeOf's 16 bits with a 2-bit child index
// (bits 12-13), hence QT_MAX_NODES.
constexpr int QT_MAX_NODES = 4096;
constexpr int QT_SMEM_CANDS = 2048;   // candidates kept in shared memory at the level with the largest node state (more at the others)
struct QtNode { int16_t ulx, uly, brx, bry; };
struct QtSort { int size; int16_t ulx, node; };
struct QtLayout { int bnd0, bnd1, cnt0, cnt1, scratch, v, proc, procNode, keepPos, kExcl, childPos, cand; };
// scratch: 4 child counts per processed node; in turn also the sort's task lists, the cell offsets of the gather and the best keys
__host__ __device__ inline QtLayout qt_layout(int mn, int nCells) {
    QtLayout L;
    int o = 0;
    L.bnd0 = o; o += 8 * mn;
    L.bnd1 = o; o += 8 * mn;
    L.cnt0 = o; o += 4 * mn;
    L.cnt1 = o; o += 4 * mn;
    L.scratch = o; o += 16 * mn > 4 * (nCells + 1) ? 16 * mn : 4 * (nCells + 1);
    L.v = o; o += 8 * mn;
    L.proc = o; o += 2 * mn;
    L.procNode = o; o += 2 * mn;
    L.keepPos = o; o += 2 * mn;
    L.kExcl = o; o += 2 * mn;
    L.childPos = o; o += 8 * mn;
    L.cand = (o + 15) & ~15;          // then uint32 cand[c], uint16 nodeOf[c] for c = (slab - cand) / 6
    return L;
}

struct ExtractParams {
    int nlevels, batch;
    int iniTh, minTh;
    int lap0, lap1;
    LevelGeom lv[kMaxLevels];
    // device pointers (per-frame strides in elements of the pointed type)
    const uint8_t* src; size_t srcStep, srcFrameStride; int rows, cols;
    uint8_t* pyr;  uint8_t* blur; size_t pyrFrameStride;
    // level 0 may alias the caller's device image instead of a copy inside `pyr`
    const uint8_t* lv0; size_t lv0Pitch, lv0FrameStride;
    int blurTilesTotal;
    const CellDesc* cells; int nCellsTotal;
    const FastBlock* fastBlocks; int nFastBlocks;
    int* cellCount;        size_t cellCountStride;
    uint32_t* cellList;    size_t cellListStride;
    uint32_t* cand;        size_t candStride;       // gathered candidates (packed x|y|score)
    uint16_t* nodeOf;                               // same stride as cand
    SelKp* sel;            size_t selStride;
    int* selCount;                                  // [batch][kMaxLevels]
    int* dstIndex;                                  // [batch][selStride] output row of each selected keypoint
    const short4* xtab; const short4* ytab;
    // outputs
    void* outKp; uint8_t* outDesc; int outCap; int* outN; int* outMono;
    int* status;                                    // [batch] sticky error flags
    int qtSlab;                                     // shared-memory bytes per quadtree warp
    int dbg;
};

// candidate packing: x (12 bits) | y (12 bits) << 12 | score << 24
__host__ __device__ inline uint32_t pack_cand(int x, int y, int s) { return (uint32_t)x | ((uint32_t)y << 12) | ((uint32_t)s << 24); }
__host__ __device__ inline int cand_x(uint32_t c) { return c & 0xFFF; }
__host__ __device__ inline int cand_y(uint32_t c) { return (c >> 12) & 0xFFF; }
__host__ __device__ inline int cand_s(uint32_t c) { return c >> 24; }

}  // namespace orbx
