// H100 kernels + C-ABI for the numeric core of Optimizer::LocalBundleAdjustment
// (reference src/Optimizer.cc:1116-1498; g2o BlockSolver_6_3 + Levenberg, see include/orb_b200.h and SURVEY.md 3.2).
//
// Execution model: ONE persistent kernel per batch of problems.  Each problem is owned by one thread-block cluster
// (1..8 CTAs, chosen so that the batch fills the 132 SMs); the whole Levenberg-Marquardt loop -- accept/reject,
// lambda schedule, stop rules, stop-flag polling -- runs on the device, phases are separated by cluster barriers,
// and the host only uploads the flattened graph and downloads the result.  All arithmetic is FP64 (g2o is double).
// SMs the batch's clusters leave idle run helper clusters, which serve chunks of the build, point-record and Schur phases of
// any problem (owner_phase / helper_loop); the results do not depend on which CTA serves a chunk.
// The linearisation is kept FACTORED: an edge stores only (x/z, y/z, 1/z, robust weight) at the linearisation point (32 B);
// its Jacobians are A = -S t (2x3, t = [R0 - xn R2; R1 - yn R2], S = diag(fx, fy)/z) and B = F b (2x6, F = diag(fx, fy),
// b a polynomial in xn, yn, 1/z), so the Hpl block W = w B^T A is rank 2 and is never materialised: every product that
// g2o forms with W (Schur complement, rhs, back-substitution) is evaluated from the factors.  Per LM trial the working
// set is ~1.5 MB per problem (L2 resident for a whole batch) instead of 11.5 MB of W / W Hll^-1 blocks.
// Phases of one LM trial (workers = all threads of the cluster):
//   residual   thread/edge      EdgeSE3ProjectXYZ::computeError + Huber rho, edge factors   (HOT LOOP A)
//   build      8 lanes/point: Hll, bl;  warp/chunk of a pose's edges: Hpp, bp               (HOT LOOP B)
//   schur      thread/point: (Hll + lambda I)^-1;  warp/chunk of the edge pairs of one pose pair:
//              Hschur = Hpp - sum B1^T (w1 w2 A1 Hll^-1 A2^T) B2                            (HOT LOOP C)
//   ldlt       CTA 0, matrix in shared memory: blocked LDL^T with look-ahead, rhs carried as an extra row
//   backsub    8 lanes/point    x_l = Hll^-1 (b_l - W^T x_p)
//   update     thread/vertex    T <- exp(dx) T, p <- p + dx  (+ backup for the LM "pop")
// Every reduction is ordered (no floating-point atomics), so results are reproducible run to run.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>
#include <algorithm>
#include <atomic>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "../../include/orb_b200.h"
#include "host_affinity.h"
#include "device_utils.cuh"
#include "inertial_dev.cuh"
#include "local_ba.h"
#include "staging.h"

using orbx::set_error;

namespace lba {

using namespace g2o;
using orbx::block_prefix;
using orbx::block_sum;

// The open data-parallel phase of one problem, in global memory: CTA 0 of the problem's cluster opens a phase, and the owner CTAs
// and any helper CTA claim its chunks NWARP at a time.  `word` = tag (16 bits) | chunks (24) | next unclaimed chunk (24): one
// atomicAdd claims, and a claim whose next chunk is past the count gets nothing.  A granted chunk pins the phase (its fields and
// the pose-cache mirror) until `done` counts it, so a claimer reads them after the claim.
struct Job {
    unsigned long long word;
    unsigned done;                    // chunks finished this launch, all phases (each phase's join waits for its running total)
    unsigned helped;                  // of those, chunks served by helper CTAs
    unsigned seq;                     // phases opened this launch
    int phase, side;                  // PH_*, which side of the double buffers is current (LoopState::cur)
    double lambda;
};
constexpr int PH_BUILD = 0, PH_PREP = 1, PH_SCHUR = 2;

struct Dev {
    int nP, nL, nE, nF, n;            // n = 6 nF
    Job* job;
    double* pcm;                      // nP x PC: the pose cache of the open phase, for helper CTAs
    double *poses, *posesB, *pts, *ptsB;        // nP x 7, nL x 3: estimate / second buffer (trial state; the two swap when a step is accepted)
    double* outPts;                             // nL x 3: the final point estimates in the caller's point order
    const double *initPoses, *initPts;          // the uploaded initial estimates (a run always restarts from them)
    // the caller's graph as uploaded (caller's edge order); lba_build_structure_kernel derives everything below from it
    const int *rawEdgePoint, *rawEdgePose; const double* rawObs; const float* rawInvSigma2;
    int *bCnt, *bCursor, *bTmp, *bEid, *bTaskLen, *bItemStart;   // build scratch: nL + 1, nL + 1, nE, nF x nL, nTasks, nTasks
    unsigned long long* bKey;         // build scratch: the point sort's keys, nL rounded up to a power of two
    int pairCap, chunkCap;
    const float* cam;                 // nP x 4
    const int* hidx;                  // nP: Hessian block index or -1
    const int* freePose;              // nF: pose index of Hessian block
    // INTERNAL point order: every per-point array of the LM kernel (pts / ptsB, Hll, bl, PT) and every point index below is a
    // rank in it; lba_build_structure_kernel sorts the points by their observing free poses (see there)
    const int* ptOrig;                // nL: caller's index of the point at internal rank r
    // edges in INTERNAL order = sorted by point rank (the edges of a point are contiguous)
    const int *ePt, *ePose;           // nE
    const int* eH;                    // nE: Hessian block of the edge's pose (hidx[ePose]) or -1
    const int* eOrig;                 // nE: caller's edge index
    const double* obs;                // nE x 2
    const float* invSigma2;           // nE
    const int* ptStart;               // nL + 1
    // POSE-MAJOR order: the edge lists of the free poses (ascending point) back to back; position k in them is the pose-major
    // index of the edge.  The Schur phase reads the edge factors in this order, so neighbouring lanes share lines.
    const int* poseEdges;             // internal edge id at pose-major index k
    const int2* pairs;                // (pose-major index of the edge of pose i1, of the edge of pose i2) observing the same point
    const int* pairPt;                // that point
    // Schur work list: tasks 0..nF-1 = diagonal blocks (items = edges of the pose), nF.. = off-diagonal blocks (items = pairs);
    // every task is cut into chunks of SCH items so that all warps of the cluster get the same amount of work
    int nChunks; const int4* chunkHdr; const int* taskChunkStart;   // nChunks x (first item, items, pose A, pose B or -1), nTasks + 1
    const int* poseEdgePt;            // nE: point of the edge at pose-major index k
    double* Spart;                    // nChunks x 42 partial sums (36 block entries + 6 rhs entries for diagonal tasks)
    double* Ppart;                    // (chunks of the diagonal tasks) x 28: partial sums of Hpp (21) and bp (6)
    double* err;                      // nE x 2
    double *E4a, *E4b;                // nE x 4 edge factors (x/z, y/z, 1/z, w): linearisation point / trial state (swapped on accept)
    double2* K;                       // 2 x nE: the factors at the linearisation point at pose-major index k, as two arrays
                                      // (x/z, y/z) | (1/z, w); written by phase_build_poses_partial, read by the Schur phase
    double *Hpp, *bp;                 // nF x 36, nF x 6
    double *Hll, *bl;                 // nL x 6 (00 01 02 11 12 22), nL x 3
    double2* PT;                      // point records as arrays over the points: (d00 d01) | (d02 d11) | (d12 d22) | (db0 db1), nL each,
                                      // then db2 (nL doubles); Dinv = (Hll + lambda I)^-1 (upper triangle), db = Dinv bl
    double *Hs, *bs;                  // n x n (only when it does not fit in shared memory), n
    double* x;                        // n + 3 nL
    double* partial;                  // 4 rotating slots x 16 doubles: per-CTA partial sums + broadcast words
    double* stats;                    // out: [0] iterations [1] trials [2] lambda [3] chi2 [4] initial chi2, [8..17] phase ns (CTA 0)
    double* outChi2; uint8_t* outDepthPos;   // nE, caller's edge order
    double delta, dsqr, userLambdaInit;
    int iterations;
};

namespace cg = cooperative_groups;
__device__ __forceinline__ unsigned long long globaltimer_ns() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#ifndef LBA_NT
#define LBA_NT 512
#endif
#ifndef LBA_MINB
#define LBA_MINB 1     /* __launch_bounds__ min blocks: with LBA_NT=256, 2 caps the kernel at 128 registers = half an SM's file */
#endif
#ifndef LBA_SCH
#define LBA_SCH 128
#endif
#ifndef LBA_UNR
#define LBA_UNR 4
#endif
/* items in flight per lane in the per-edge passes: points per 8-lane group and step (build_points, points_trial), edges per
   lane of a build_poses chunk */
#ifndef LBA_FLY_BP
#define LBA_FLY_BP 2
#endif
#ifndef LBA_FLY_BPP
#define LBA_FLY_BPP 2
#endif
#ifndef LBA_FLY_PT
#define LBA_FLY_PT 1
#endif
constexpr int NT = LBA_NT;
constexpr int NWARP = NT / 32;
constexpr int FLY_BP = LBA_FLY_BP, FLY_BPP = LBA_FLY_BPP, FLY_PT = LBA_FLY_PT;
constexpr int MAXC = 8;            // largest cluster
constexpr int PSLOT = 24;          // doubles per partial slot: A[0..7], flag[8], B[9..16]
constexpr int PC = 20;             // doubles per cached pose: q(4) t(3) R(9) fx fy cx cy

// The thread's place in the cluster is read from the special registers where a phase starts (asm volatile, so that the
// compiler does not merge the reads into one value held in registers across every phase)
__device__ __forceinline__ int sreg_ctarank() { int r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ int sreg_nctarank() { int r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
struct Ctx {
    int slot;              // rotating partial slot
    double* sm;            // NT doubles of scratch
    const double* pc;      // pose cache in shared memory (state at the linearisation point), PC doubles per pose
    __device__ __forceinline__ int crank() const { return sreg_ctarank(); }
    __device__ __forceinline__ int csize() const { return sreg_nctarank(); }
    __device__ __forceinline__ int tid() const { return (int)threadIdx.x; }
    __device__ __forceinline__ int wid() const { return sreg_ctarank() * NT + (int)threadIdx.x; }   // worker id / count over the cluster
    __device__ __forceinline__ int nw() const { return sreg_nctarank() * NT; }
};

// cluster-wide ordered sum (per-CTA partials -> global slot -> cluster barrier -> added in rank order by every thread);
// `flagIn` of CTA 0 / thread 0 is broadcast alongside.
__device__ __forceinline__ double cluster_sum(const Dev& D, Ctx& c, double local, int flagIn, int& flagOut) {
    const double s = block_sum<NT>(local, c.sm);
    double* slot = D.partial + (size_t)(c.slot & 3) * PSLOT;
    if (c.tid() == 0) {
        slot[c.crank()] = s;
        if (c.crank() == 0) slot[MAXC] = (double)flagIn;
    }
    cg::this_cluster().sync();
    double tot = 0;
    for (int r = 0; r < c.csize(); ++r) tot += slot[r];
    flagOut = (int)slot[MAXC];
    ++c.slot;
    return tot;
}
// the same for two sums at once
__device__ __forceinline__ void cluster_sum2(const Dev& D, Ctx& c, double a, double b, int flagIn, int& flagOut, double& totA, double& totB) {
    const int tid = threadIdx.x;
#pragma unroll
    for (int o = 16; o; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
    if ((tid & 31) == 0) { c.sm[tid >> 5] = a; c.sm[NWARP + (tid >> 5)] = b; }
    __syncthreads();
    double* slot = D.partial + (size_t)(c.slot & 3) * PSLOT;
    if (tid == 0) {
        double ra = 0, rb = 0;
        for (int w = 0; w < NWARP; ++w) { ra += c.sm[w]; rb += c.sm[NWARP + w]; }
        slot[c.crank()] = ra; slot[MAXC + 1 + c.crank()] = rb;
        if (c.crank() == 0) slot[MAXC] = (double)flagIn;
    }
    cg::this_cluster().sync();
    totA = 0; totB = 0;
    for (int r = 0; r < c.csize(); ++r) { totA += slot[r]; totB += slot[MAXC + 1 + r]; }
    flagOut = (int)slot[MAXC];
    ++c.slot;
}
__device__ __forceinline__ void csync() { cg::this_cluster().sync(); }

// (re)load every pose into the CTA's shared-memory cache: quaternion, translation, rotation matrix, camera
__device__ void load_pose_cache(const Dev& D, const double* poses, double* pc) {
    for (int i = threadIdx.x; i < D.nP; i += NT) {
        double* o = pc + PC * i;
        const double* T = poses + 7 * (size_t)i;
#pragma unroll
        for (int k = 0; k < 7; ++k) o[k] = T[k];
        qtoR(T, o + 7);
        const float* cm = D.cam + 4 * (size_t)i;
        o[16] = (double)cm[0]; o[17] = (double)cm[1]; o[18] = (double)cm[2]; o[19] = (double)cm[3];   // float params promoted (Pinhole.cpp:35-41)
    }
    __syncthreads();
}

// The graph's index arrays and observations are written by lba_build_structure_kernel and stay fixed for the whole LM kernel:
// they are read through the non-coherent path, which the compiler may also issue ahead of earlier stores
template <typename T>
__device__ __forceinline__ T ro(const T* p) { return __ldg(p); }
__device__ __forceinline__ double2 ro_obs(const Dev& D, int e) { return ro(reinterpret_cast<const double2*>(D.obs) + e); }

// one edge at pose P (cached: q t R cam) and point X with observation ob and 1/sigma^2 is2: residual, robust chi2 and the edge
// factors of this state
__device__ __forceinline__ double edge_error(const Dev& D, const double* P, const double* X, int e, double2 ob, double is2, double* __restrict__ Eout) {
    double r[3]; qrot(P, X, r);                                     // SE3Quat::map: _r * xyz + _t
    const double xc = r[0] + P[4], yc = r[1] + P[5], zc = r[2] + P[6];
    const double u = P[16] * xc / zc + P[18], v = P[17] * yc / zc + P[19];      // Pinhole::project(Vector3d)
    const double e0 = ob.x - u, e1 = ob.y - v;
    *reinterpret_cast<double2*>(D.err + 2 * (size_t)e) = make_double2(e0, e1);
    double r0, r1;
    huber(is2 * (e0 * e0 + e1 * e1), D.delta, D.dsqr, r0, r1);
    const double iz = 1.0 / zc;
    double2* o = reinterpret_cast<double2*>(Eout + 4 * (size_t)e);
    o[0] = make_double2(xc * iz, yc * iz);
    o[1] = make_double2(iz, r1 * is2);
    return r0;
}
// ---- residuals + robust chi2 (SparseOptimizer::computeActiveErrors + activeRobustChi2), thread per edge.
//      Also leaves the edge factors (x/z, y/z, 1/z, rho' / sigma^2) of this state in Eout. ----
__device__ double phase_errors(const Dev& D, const Ctx& c, const double* pts, double* __restrict__ Eout) {
    double acc = 0;
    const int nw = c.nw();
    for (int e = c.wid(); e < D.nE; e += nw)
        acc += edge_error(D, c.pc + PC * ro(D.ePose + e), pts + 3 * (size_t)ro(D.ePt + e), e, ro_obs(D, e), (double)ro(D.invSigma2 + e), Eout);
    return acc;
}

// Edge factors.  With xn = x/z, yn = y/z, iz = 1/z (camera frame) and R the keyframe rotation, the Jacobians of
// EdgeSE3ProjectXYZ::linearizeOplus (-projectJac * R and -projectJac * [-[Xc]x | I], Pinhole.cpp:71-81) are
//   A = -diag(fx iz, fy iz) t,   t = [R0 - xn R2 ; R1 - yn R2]                           (2x3)
//   B =  diag(fx, fy) b,         b = [xn yn, -(1 + xn^2), yn, -iz, 0, xn iz ; 1 + yn^2, -xn yn, -xn, 0, -iz, yn iz]   (2x6)
// A 32-byte record as two 128-bit loads (the widest sm_90 has).  Plain loads, so that the compiler may issue them ahead of
// stores it can tell apart from them
__device__ __forceinline__ void ld256(const double* p, double& a, double& b, double& c, double& d) {
    const double2 u = reinterpret_cast<const double2*>(p)[0], v = reinterpret_cast<const double2*>(p)[1];
    a = u.x; b = u.y; c = v.x; d = v.y;
}
__device__ __forceinline__ void load_e4(const double* __restrict__ E, int e, double& xn, double& yn, double& iz, double& w) {
    ld256(E + 4 * (size_t)e, xn, yn, iz, w);
}
// The same factors from the pose-major arrays (K = (x/z, y/z) of every edge, then (1/z, w)), at pose-major index k.  The Schur
// phase is bound by L1 look-ups per load instruction, and here the lanes of a warp read neighbouring k: a diagonal chunk reads
// 32 consecutive entries (4 lines per LDG.128 instead of 32)
__device__ __forceinline__ void load_k4(const double2* __restrict__ K, int nE, int k, double& xn, double& yn, double& iz, double& w) {
    const double2 a = K[k], b = K[nE + k];
    xn = a.x; yn = a.y; iz = b.x; w = b.y;
}
__device__ __forceinline__ void edge_t(const double* R, double xn, double yn, double* t) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { t[k] = R[k] - xn * R[6 + k]; t[3 + k] = R[3 + k] - yn * R[6 + k]; }
}
__device__ __forceinline__ void edge_b(double xn, double yn, double iz, double* b0, double* b1) {   // b0[4] and b1[3] are zero
    const double xy = xn * yn;
    b0[0] = xy;                 b0[1] = -(1.0 + xn * xn); b0[2] = yn;  b0[3] = -iz; b0[4] = 0.0; b0[5] = xn * iz;
    b1[0] = 1.0 + yn * yn;      b1[1] = -xy;              b1[2] = -xn; b1[3] = 0.0; b1[4] = -iz; b1[5] = yn * iz;
}

// Reduce-scatter of V register values over the 32 lanes of a warp: afterwards lane `lane` holds the totals of entries
// [lo, lo + n) in v[0..n), n <= 2.  Fixed butterfly (halve the vector at every level), ~V shuffles instead of 5 V.
template <int N, int H>
__device__ __forceinline__ void rs_level(double* v, bool up, int o) {
#pragma unroll
    for (int i = 0; i < H; ++i) {
        const double a = v[i];
        const double b = (i + H < N) ? v[i + H] : 0.0;
        const double keep = up ? b : a, send = up ? a : b;
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
}
template <int V>
__device__ __forceinline__ void warp_reduce_scatter(double* v, int lane, int& lo, int& n) {
    constexpr int H1 = (V + 1) / 2, H2 = (H1 + 1) / 2, H3 = (H2 + 1) / 2, H4 = (H3 + 1) / 2, H5 = (H4 + 1) / 2;
    static_assert(H5 <= 2, "vector too long");
    lo = 0; n = V;
    bool up;
    up = lane & 16; rs_level<V, H1>(v, up, 16); if (up) { lo += H1; n -= H1; } else n = min(n, H1);
    up = lane & 8;  rs_level<H1, H2>(v, up, 8); if (up) { lo += H2; n -= H2; } else n = min(n, H2);
    up = lane & 4;  rs_level<H2, H3>(v, up, 4); if (up) { lo += H3; n -= H3; } else n = min(n, H3);
    up = lane & 2;  rs_level<H3, H4>(v, up, 2); if (up) { lo += H4; n -= H4; } else n = min(n, H4);
    up = lane & 1;  rs_level<H4, H5>(v, up, 1); if (up) { lo += H5; n -= H5; } else n = min(n, H5);
}

__device__ __forceinline__ void point_record(const Dev& D, int p, const double* h, const double* bl3, double lambda);
// The per-point passes give every group of 8 lanes the points p, p + G, p + 2G, ... (G groups) and take FLY of them per step:
// a step first issues the loads of the lane's first edge of each of its points, then adds the points one after another,
// each with the same per-lane order (edges sl, sl + 8, ...) and the same shuffle tree as one point per step.  The next step's
// ptStart entries are loaded ahead.
template <int FLY>
__device__ __forceinline__ void step_ranges(const int* ptStart, int nL, int p, int G, int* a, int* b) {
#pragma unroll
    for (int j = 0; j < FLY; ++j) {
        const int q = p + j * G;
        a[j] = q < nL ? ro(ptStart + q) : 0;
        b[j] = q < nL ? ro(ptStart + q + 1) : 0;
    }
}
// operands of one edge in the build pass: its pose, factors and error
struct BuildEdge { int pose; double xn, yn, iz, w; double2 er; };
__device__ __forceinline__ BuildEdge load_build_edge(const Dev& D, const double* __restrict__ E, int e) {
    BuildEdge o;
    o.pose = ro(D.ePose + e);
    load_e4(E, e, o.xn, o.yn, o.iz, o.w);
    o.er = *reinterpret_cast<const double2*>(D.err + 2 * (size_t)e);
    return o;
}
__device__ __forceinline__ void add_build_edge(const double* pcache, const BuildEdge& o, double* h, double* g) {
    const double* P = pcache + PC * o.pose;
    double t[6];
    edge_t(P + 7, o.xn, o.yn, t);
    const double s0 = P[16] * o.iz, s1 = P[17] * o.iz;
    const double c0 = o.w * s0 * s0, c1 = o.w * s1 * s1;          // w A^T A = c0 t0^T t0 + c1 t1^T t1
    const double q0 = s0 * o.w * o.er.x, q1 = s1 * o.w * o.er.y;  // A^T r, r = -w err
    g[0] += t[0] * q0 + t[3] * q1; g[1] += t[1] * q0 + t[4] * q1; g[2] += t[2] * q0 + t[5] * q1;
    h[0] += c0 * t[0] * t[0] + c1 * t[3] * t[3]; h[1] += c0 * t[0] * t[1] + c1 * t[3] * t[4]; h[2] += c0 * t[0] * t[2] + c1 * t[3] * t[5];
    h[3] += c0 * t[1] * t[1] + c1 * t[4] * t[4]; h[4] += c0 * t[1] * t[2] + c1 * t[4] * t[5]; h[5] += c0 * t[2] * t[2] + c1 * t[5] * t[5];
}
constexpr int PCH = 32;            // points per chunk of the per-point phases (build_points, point_prep)
// ---- per point Hll, bl (and, when lambda is already known, the point record of point_prep_chunk); 8 lanes per point
//      (the edges of a point are contiguous); one warp per chunk of PCH points ----
__device__ __forceinline__ void build_points_chunk(const Dev& D, const double* pc, const double* __restrict__ E, double lambda, int ch) {
    constexpr int FLY = FLY_BP, G = 4;
    const int sl = threadIdx.x & 7;
    const unsigned gmask = 0xFFu << (threadIdx.x & 24);
    const int first = ch * PCH + ((threadIdx.x & 31) >> 3), end = min(D.nL, (ch + 1) * PCH);
    int a[FLY], b[FLY];
    step_ranges<FLY>(D.ptStart, end, first, G, a, b);
    for (int p0 = first; p0 < end; p0 += FLY * G) {
        BuildEdge first[FLY] = {};
#pragma unroll
        for (int j = 0; j < FLY; ++j) if (a[j] + sl < b[j]) first[j] = load_build_edge(D, E, a[j] + sl);
        int na[FLY], nb[FLY];
        step_ranges<FLY>(D.ptStart, end, p0 + FLY * G, G, na, nb);
#pragma unroll
        for (int j = 0; j < FLY; ++j) {
            const int p = p0 + j * G;
            if (p >= end) break;
            double h[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
            if (a[j] + sl < b[j]) add_build_edge(pc, first[j], h, g);
            for (int e = a[j] + sl + 8; e < b[j]; e += 8) add_build_edge(pc, load_build_edge(D, E, e), h, g);
#pragma unroll
            for (int o = 4; o; o >>= 1) {
#pragma unroll
                for (int i = 0; i < 6; ++i) h[i] += __shfl_xor_sync(gmask, h[i], o);
#pragma unroll
                for (int i = 0; i < 3; ++i) g[i] += __shfl_xor_sync(gmask, g[i], o);
            }
            if (sl == 0) {
                double2* H = reinterpret_cast<double2*>(D.Hll + 6 * (size_t)p);
                H[0] = make_double2(h[0], h[1]); H[1] = make_double2(h[2], h[3]); H[2] = make_double2(h[4], h[5]);
                D.bl[3 * (size_t)p] = g[0]; D.bl[3 * (size_t)p + 1] = g[1]; D.bl[3 * (size_t)p + 2] = g[2];
                if (lambda >= 0) point_record(D, p, h, g, lambda);
            }
        }
#pragma unroll
        for (int j = 0; j < FLY; ++j) { a[j] = na[j]; b[j] = nb[j]; }
    }
}

constexpr int SCH = LBA_SCH;       // items per chunk of the pose / pose-pair work lists
constexpr int IPL = SCH / 32;      // items per lane
constexpr int UNR = LBA_UNR;       // items in flight per lane in the Schur chunk loops

// ---- per free pose Hpp, bp.  partial: warp per chunk of the pose's edges (the chunks of the diagonal Schur tasks), lane per
//      edge, 21 + 6 sums reduce-scattered to Spart; combine: thread per (pose, entry), chunks added in order.
//      The chunks cover every pose-major index once, so the partial step also writes the pose-major copy K of the factors
//      that the Schur phase reads (coalesced stores; the factors stay fixed for all trials of an iteration).
//      As in the Schur chunks, the chunk's edge ids are loaded into registers up front; then the factors and errors of FLY
//      items per lane are loaded before their K stores and their sums, which keep the item order of the lane. ----
__device__ __forceinline__ void build_poses_chunk(const Dev& D, const double* pc, const double* __restrict__ E, int ch) {
    constexpr int FLY = FLY_BPP;
    const int lane = threadIdx.x & 31;
    {
        const int4 h = D.chunkHdr[ch];
        const double* P = pc + PC * h.z;
        const double fx = P[16], fy = P[17];
        int re[IPL];
#pragma unroll
        for (int j = 0; j < IPL; ++j) { const int i = lane + 32 * j; re[j] = i < h.y ? ro(D.poseEdges + h.x + i) : 0; }
        double acc[27];
#pragma unroll
        for (int i = 0; i < 27; ++i) acc[i] = 0;
#pragma unroll
        for (int j0 = 0; j0 < IPL; j0 += FLY) {
            double f[FLY][4] = {}; double2 er[FLY] = {};
#pragma unroll
            for (int u = 0; u < FLY; ++u) {
                const int j = j0 + u;
                if (j < IPL && lane + 32 * j < h.y) {
                    load_e4(E, re[j], f[u][0], f[u][1], f[u][2], f[u][3]);
                    er[u] = *reinterpret_cast<const double2*>(D.err + 2 * (size_t)re[j]);
                }
            }
#pragma unroll
            for (int u = 0; u < FLY; ++u) {
                const int j = j0 + u, k = h.x + lane + 32 * j;
                if (j < IPL && lane + 32 * j < h.y) { D.K[k] = make_double2(f[u][0], f[u][1]); D.K[D.nE + k] = make_double2(f[u][2], f[u][3]); }
            }
#pragma unroll
            for (int u = 0; u < FLY; ++u) {
                const int j = j0 + u;
                if (j < IPL && lane + 32 * j < h.y) {
                    const double xn = f[u][0], yn = f[u][1], iz = f[u][2], w = f[u][3];
                    double b0[6], b1[6];
                    edge_b(xn, yn, iz, b0, b1);
                    const double c0 = w * fx * fx, c1 = w * fy * fy;          // w B^T B = c0 b0^T b0 + c1 b1^T b1
                    const double q0 = fx * w * er[u].x, q1 = fy * w * er[u].y;  // B^T r = -(b0 q0 + b1 q1)
                    int t = 0;
#pragma unroll
                    for (int a = 0; a < 6; ++a) {
                        const double u0 = c0 * b0[a], u1 = c1 * b1[a];
#pragma unroll
                        for (int i = a; i < 6; ++i) acc[t++] += u0 * b0[i] + u1 * b1[i];
                    }
#pragma unroll
                    for (int a = 0; a < 6; ++a) acc[21 + a] -= b0[a] * q0 + b1[a] * q1;
                }
            }
        }
        int lo, n;
        warp_reduce_scatter<27>(acc, lane, lo, n);
        if (n > 0) D.Ppart[28 * (size_t)ch + lo] = acc[0];
    }
}
__device__ void phase_build_poses_combine(const Dev& D, const Ctx& c) {
    const int nw = c.nw();
    for (int idx = c.wid(); idx < D.nF * 27; idx += nw) {
        const int hI = idx / 27, ent = idx - hI * 27;
        double s = 0;
        for (int ch = D.taskChunkStart[hI]; ch < D.taskChunkStart[hI + 1]; ++ch) s += D.Ppart[28 * (size_t)ch + ent];
        if (ent < 21) {
            int i = 0, t = ent;             // unrank (i, j), i <= j
            while (t >= 6 - i) { t -= 6 - i; ++i; }
            const int j = i + t;
            D.Hpp[36 * (size_t)hI + i * 6 + j] = s; D.Hpp[36 * (size_t)hI + j * 6 + i] = s;
        } else D.bp[6 * (size_t)hI + (ent - 21)] = s;
    }
}

// ---- max |diag| over all Hessian blocks (computeLambdaInit); every CTA computes it redundantly ----
__device__ double phase_maxdiag(const Dev& D, const Ctx& c) {
    double m = 0;
    for (int i = c.tid(); i < D.n; i += NT) m = fmax(m, fabs(D.Hpp[36 * (size_t)(i / 6) + 7 * (i % 6)]));
    for (int i = c.tid(); i < 3 * D.nL; i += NT) { const int k = i % 3; m = fmax(m, fabs(D.Hll[6 * (size_t)(i / 3) + (k == 0 ? 0 : k == 1 ? 3 : 5)])); }
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    __syncthreads();
    if ((c.tid() & 31) == 0) c.sm[c.tid() >> 5] = m;
    __syncthreads();
    double r = 0;
    for (int w = 0; w < NWARP; ++w) r = fmax(r, c.sm[w]);
    __syncthreads();
    return r;
}

// ---- (Hll + lambda I)^-1 and (Hll + lambda I)^-1 bl, thread per point (block_solver.hpp:381-394) ----
__device__ __forceinline__ void point_record(const Dev& D, int p, const double* h, const double* bl3, double lambda) {
    const double m0 = h[0] + lambda, m1 = h[1], m2 = h[2], m4 = h[3] + lambda, m5 = h[4], m8 = h[5] + lambda;
    const double c00 = m4 * m8 - m5 * m5, c10 = m5 * m2 - m1 * m8, c20 = m1 * m5 - m4 * m2;
    const double id = 1.0 / (m0 * c00 + m1 * c10 + m2 * c20);     // Eigen 3x3 inverse: cofactors / determinant
    const double o0 = c00 * id, o1 = c10 * id, o2 = c20 * id;
    const double o4 = (m0 * m8 - m2 * m2) * id, o5 = (m2 * m1 - m0 * m5) * id, o8 = (m0 * m4 - m1 * m1) * id;
    const double b0 = bl3[0], b1 = bl3[1], b2 = bl3[2];
    const size_t nL = D.nL;
    double2* O = D.PT + p;
    O[0] = make_double2(o0, o1); O[nL] = make_double2(o2, o4); O[2 * nL] = make_double2(o5, o8);
    O[3 * nL] = make_double2(o0 * b0 + o1 * b1 + o2 * b2, o1 * b0 + o4 * b1 + o5 * b2);
    reinterpret_cast<double*>(D.PT + 4 * nL)[p] = o2 * b0 + o5 * b1 + o8 * b2;
}
// Dinv of point p (00 01 02 11 12 22) from the point records
__device__ __forceinline__ void load_dinv(const double2* __restrict__ PT, size_t nL, int p, double* dv) {
    const double2 a = PT[p], b = PT[nL + p], c = PT[2 * nL + p];
    dv[0] = a.x; dv[1] = a.y; dv[2] = b.x; dv[3] = b.y; dv[4] = c.x; dv[5] = c.y;
}
__device__ __forceinline__ void point_prep_chunk(const Dev& D, double lambda, int ch) {
    const int p = ch * PCH + (threadIdx.x & 31);
    if (p < D.nL) {
        const double2* H = reinterpret_cast<const double2*>(D.Hll + 6 * (size_t)p);
        const double2 h01 = H[0], h23 = H[1], h45 = H[2];
        const double h[6] = {h01.x, h01.y, h23.x, h23.y, h45.x, h45.y};
        const double b3[3] = {D.bl[3 * (size_t)p], D.bl[3 * (size_t)p + 1], D.bl[3 * (size_t)p + 2]};
        point_record(D, p, h, b3, lambda);
    }
}

// ---- Schur complement (block_solver.hpp:396-431), two steps.
//   partial: the work list (diagonal block i: edges of pose i; off-diagonal block (i1 < i2): the precomputed (k1, k2) pairs)
//            is cut into chunks of SCH items; one warp per chunk, one lane per item.  An item adds
//                b1^T M b2,   M[k][l] = g1_k g2_l (t1_k Hll^-1 t2_l^T),   g_k = w f_k^2 / z
//            (= W1 Hll^-1 W2^T with W = w B^T A) into the lane's 36 accumulators; diagonal items also add
//            W Hll^-1 bl = -sum_k b_k g_k (t_k . db).  The item's operands (two edges, one point) are per-lane loads and
//            the phase is bound by L1 look-ups, one per distinct line of a warp's load instruction (tools/microbench), so
//            they are read from the pose-major edge arrays and the point arrays: the lanes of a chunk hold ascending points
//            and neighbouring pose-major indices and share lines.  The chunk's indices are loaded into registers up front and
//            UNR items are in flight per lane.  The lanes' sums are reduce-scattered into Spart.
//   combine: thread per (task, entry): ordered sum of the task's chunks -> lower triangle of the reduced camera system
//            (diagonal: Hpp_i + lambda I - sum, bs_i = bp_i - sum; off-diagonal: block (i2, i1) = -(sum)^T). ----
__device__ __forceinline__ void schur_item(const double* t1, const double* t2, const double* dv, double g10, double g11, double g20, double g21,
                                           const double* b10, const double* b11, const double* b20, const double* b21, double* acc) {
    // u = t1 Dinv (2x3), dv = 00 01 02 11 12 22
    const double u00 = t1[0] * dv[0] + t1[1] * dv[1] + t1[2] * dv[2], u01 = t1[0] * dv[1] + t1[1] * dv[3] + t1[2] * dv[4], u02 = t1[0] * dv[2] + t1[1] * dv[4] + t1[2] * dv[5];
    const double u10 = t1[3] * dv[0] + t1[4] * dv[1] + t1[5] * dv[2], u11 = t1[3] * dv[1] + t1[4] * dv[3] + t1[5] * dv[4], u12 = t1[3] * dv[2] + t1[4] * dv[4] + t1[5] * dv[5];
    const double m00 = (u00 * t2[0] + u01 * t2[1] + u02 * t2[2]) * (g10 * g20), m01 = (u00 * t2[3] + u01 * t2[4] + u02 * t2[5]) * (g10 * g21);
    const double m10 = (u10 * t2[0] + u11 * t2[1] + u12 * t2[2]) * (g11 * g20), m11 = (u10 * t2[3] + u11 * t2[4] + u12 * t2[5]) * (g11 * g21);
    // T = M b2 (2x6); b20[4] = b21[3] = 0
    double T0[6], T1[6];
#pragma unroll
    for (int q = 0; q < 6; ++q) {
        if (q == 3) { T0[q] = m00 * b20[q]; T1[q] = m10 * b20[q]; }
        else if (q == 4) { T0[q] = m01 * b21[q]; T1[q] = m11 * b21[q]; }
        else { T0[q] = m00 * b20[q] + m01 * b21[q]; T1[q] = m10 * b20[q] + m11 * b21[q]; }
    }
    // acc += b1^T T; b10[4] = b11[3] = 0
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int q = 0; q < 6; ++q) {
            if (a == 3) acc[a * 6 + q] += b10[a] * T0[q];
            else if (a == 4) acc[a * 6 + q] += b11[a] * T1[q];
            else acc[a * 6 + q] += b10[a] * T0[q] + b11[a] * T1[q];
        }
}
struct PairOps { double a[4], b[4], dv[6]; };          // edge 1, edge 2 (x/z, y/z, 1/z, w), Dinv
struct DiagOps { double a[4], dv[6], db[3]; };
__device__ __forceinline__ void schur_chunk_offdiag(const int2* __restrict__ pairs, const int* __restrict__ pairPt, const double2* __restrict__ PT, size_t nL,
                                                  const double2* __restrict__ K, int nE, const double* pcache, double* out42, int4 h) {
    const int lane = threadIdx.x & 31;
    const int cnt = h.y;
    int2 rpr[IPL]; int rpt[IPL];
#pragma unroll
    for (int j = 0; j < IPL; ++j) { const int i = lane + 32 * j; if (i < cnt) { rpr[j] = pairs[h.x + i]; rpt[j] = pairPt[h.x + i]; } else { rpr[j] = make_int2(0, 0); rpt[j] = 0; } }
    const double* P1 = pcache + PC * h.z;
    const double* P2 = pcache + PC * h.w;
    const double f10 = P1[16] * P1[16], f11 = P1[17] * P1[17], f20 = P2[16] * P2[16], f21 = P2[17] * P2[17];
    double acc[36];
#pragma unroll
    for (int i = 0; i < 36; ++i) acc[i] = 0;
#pragma unroll UNR
    for (int j = 0; j < IPL; ++j) {
        const int i = lane + 32 * j;
        if (i < cnt) {
            PairOps o;
            const int k1 = rpr[j].x, k2 = rpr[j].y, ip = rpt[j];
            load_k4(K, nE, k1, o.a[0], o.a[1], o.a[2], o.a[3]);
            load_k4(K, nE, k2, o.b[0], o.b[1], o.b[2], o.b[3]);
            load_dinv(PT, nL, ip, o.dv);
            double t1[6], t2[6], b10[6], b11[6], b20[6], b21[6];
            edge_t(P1 + 7, o.a[0], o.a[1], t1); edge_t(P2 + 7, o.b[0], o.b[1], t2);
            edge_b(o.a[0], o.a[1], o.a[2], b10, b11); edge_b(o.b[0], o.b[1], o.b[2], b20, b21);
            const double q1 = o.a[2] * o.a[3], q2 = o.b[2] * o.b[3];
            schur_item(t1, t2, o.dv, f10 * q1, f11 * q1, f20 * q2, f21 * q2, b10, b11, b20, b21, acc);
        }
    }
    int lo, n;
    warp_reduce_scatter<36>(acc, lane, lo, n);
    double* out = out42 + lo;
    if (n > 0) out[0] = acc[0];
    if (n > 1) out[1] = acc[1];
}
// the items of a diagonal chunk are the edges at pose-major indices h.x .. h.x + cnt - 1: the factors are read coalesced
__device__ __forceinline__ void schur_chunk_diag(const int* __restrict__ poseEdgePt, const double2* __restrict__ PT, size_t nL,
                                               const double2* __restrict__ K, int nE, const double* pcache, double* out42, int4 h) {
    const int lane = threadIdx.x & 31;
    const int cnt = h.y;
    int rpt[IPL];
#pragma unroll
    for (int j = 0; j < IPL; ++j) { const int i = lane + 32 * j; rpt[j] = i < cnt ? poseEdgePt[h.x + i] : 0; }
    const double* P1 = pcache + PC * h.z;
    const double f10 = P1[16] * P1[16], f11 = P1[17] * P1[17];
    const double* db2 = reinterpret_cast<const double*>(PT + 4 * nL);
    double acc[42];
#pragma unroll
    for (int i = 0; i < 42; ++i) acc[i] = 0;
#pragma unroll UNR
    for (int j = 0; j < IPL; ++j) {
        const int i = lane + 32 * j;
        if (i < cnt) {
            DiagOps o;
            const int ip = rpt[j];
            load_k4(K, nE, h.x + i, o.a[0], o.a[1], o.a[2], o.a[3]);
            load_dinv(PT, nL, ip, o.dv);
            const double2 db = PT[3 * nL + ip];
            o.db[0] = db.x; o.db[1] = db.y; o.db[2] = db2[ip];
            double t1[6], b10[6], b11[6];
            edge_t(P1 + 7, o.a[0], o.a[1], t1);
            edge_b(o.a[0], o.a[1], o.a[2], b10, b11);
            const double q1 = o.a[2] * o.a[3], g0 = f10 * q1, g1 = f11 * q1;
            schur_item(t1, t1, o.dv, g0, g1, g0, g1, b10, b11, b10, b11, acc);
            const double y0 = g0 * (t1[0] * o.db[0] + t1[1] * o.db[1] + t1[2] * o.db[2]), y1 = g1 * (t1[3] * o.db[0] + t1[4] * o.db[1] + t1[5] * o.db[2]);
#pragma unroll
            for (int a = 0; a < 6; ++a) acc[36 + a] -= b10[a] * y0 + b11[a] * y1;
        }
    }
    int lo, n;
    warp_reduce_scatter<42>(acc, lane, lo, n);
    double* out = out42 + lo;
    if (n > 0) out[0] = acc[0];
    if (n > 1) out[1] = acc[1];
}
// ---- one chunk of the open phase of a problem, by one warp.  Owner CTAs and helper CTAs both serve chunks through this one
//      function, kept out of line so that there is one compiled copy of every chunk's arithmetic: ptxas contracts products into
//      FMAs depending on the surrounding code, and a chunk must give the same bits whichever CTA serves it.
//      BUILD: chunks [0, nPointChunks) are build_points chunks, the rest the build_poses chunks (the diagonal Schur chunks). ----
__device__ __noinline__ void serve_chunk(const Dev& D, const double* pc, int phase, int side, double lambda, int ch) {
    if (phase == PH_SCHUR) {
        const int4 h = D.chunkHdr[ch];      // first item, items, pose A, pose B (-1: diagonal task)
        if (h.w >= 0) schur_chunk_offdiag(D.pairs, D.pairPt, D.PT, D.nL, D.K, D.nE, pc, D.Spart + 42 * (size_t)ch, h);
        else schur_chunk_diag(D.poseEdgePt, D.PT, D.nL, D.K, D.nE, pc, D.Spart + 42 * (size_t)ch, h);
    } else if (phase == PH_PREP) {
        point_prep_chunk(D, lambda, ch);
    } else {
        const double* E = side ? D.E4b : D.E4a;
        const int nPtCh = (D.nL + PCH - 1) / PCH;
        if (ch < nPtCh) build_points_chunk(D, pc, E, lambda, ch);
        else build_poses_chunk(D, pc, E, ch - nPtCh);
    }
}

__device__ __forceinline__ unsigned long long ld_acquire(const unsigned long long* p) {
    unsigned long long v; asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed(const unsigned long long* p) {
    unsigned long long v; asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ unsigned job_tag(unsigned long long w) { return (unsigned)(w >> 48); }
__device__ __forceinline__ int job_count(unsigned long long w) { return (int)((w >> 24) & 0xFFFFFF); }
__device__ __forceinline__ int job_next(unsigned long long w) { return (int)(w & 0xFFFFFF); }
__device__ void phase_schur_combine(const Dev& D, const Ctx& c, double lambda, double* Hs, int ld) {
    const int nOff = D.nF * (D.nF - 1) / 2, nTasks = D.nF + nOff;
    const int nw = c.nw();
    for (int idx = c.wid(); idx < nTasks * 42; idx += nw) {
        const int task = idx / 42, ent = idx - task * 42;
        if (task >= D.nF && ent >= 36) continue;
        double s = 0;
        for (int ch = D.taskChunkStart[task]; ch < D.taskChunkStart[task + 1]; ++ch) s += D.Spart[42 * (size_t)ch + ent];
        if (task < D.nF) {
            const int i1 = task;
            if (ent < 36) {
                const int r = ent / 6, q = ent % 6;
                if (q <= r) Hs[(size_t)(6 * i1 + r) * ld + 6 * i1 + q] = D.Hpp[36 * (size_t)i1 + ent] + (r == q ? lambda : 0.0) - s;
            } else D.bs[6 * i1 + (ent - 36)] = D.bp[6 * (size_t)i1 + (ent - 36)] - s;
        } else {
            int i1 = 0, rem = task - D.nF;
            while (rem >= D.nF - 1 - i1) { rem -= D.nF - 1 - i1; ++i1; }
            const int i2 = i1 + 1 + rem;
            const int r = ent / 6, q = ent % 6;
            Hs[(size_t)(6 * i2 + q) * ld + 6 * i1 + r] = -s;       // block (i2, i1) = -(sum)^T
        }
    }
}
// ---- dense LDL^T (no pivoting) + solve, one CTA; A = lower triangle, leading dimension ld (shared memory when it fits).
// Right-looking, blocked by the natural 6x6 pose blocks, with look-ahead: while warps 1.. apply the rank-6 trailing update
// of block step k, warp 0 updates the next diagonal block first and factors it (the serial chain of 6 reciprocals),
// so the only barriers are panel | update.  The rhs rides along as row n of the matrix (`brow`): after the last step it
// holds z = D^-1 L^-1 bs, and only the backward substitution L^T x = z remains.
// (LinearSolverEigen::solve: SimplicialLDLT fails only on an exactly zero pivot.)  Returns 1 on success (uniform).
// scratch: 2 x 6 x (n + 1) doubles (unscaled and scaled panel), brow: n doubles, both in shared memory. ----
__device__ __forceinline__ void ldlt_factor6(double* A, int ld, int k0, double* sL, double* sDinv, int* sFail) {   // one thread
    double a[21];            // lower triangle, row-major packed: (i, j) -> i (i + 1) / 2 + j
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j <= i; ++j) a[i * (i + 1) / 2 + j] = A[(size_t)(k0 + i) * ld + k0 + j];
    bool bad = false;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const double dk = a[k * (k + 1) / 2 + k];
        if (dk == 0.0) bad = true;
        const double inv = 1.0 / dk;
        sDinv[k] = inv;
        double l[6];
#pragma unroll
        for (int i = k + 1; i < 6; ++i) l[i] = a[i * (i + 1) / 2 + k] * inv;
#pragma unroll
        for (int i = k + 1; i < 6; ++i)
#pragma unroll
            for (int j = k + 1; j <= i; ++j) a[i * (i + 1) / 2 + j] -= l[i] * a[j * (j + 1) / 2 + k];
#pragma unroll
        for (int i = k + 1; i < 6; ++i) a[i * (i + 1) / 2 + k] = l[i];
    }
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j <= i; ++j) {
            A[(size_t)(k0 + i) * ld + k0 + j] = a[i * (i + 1) / 2 + j];
            if (j < i) sL[i * 6 + j] = a[i * (i + 1) / 2 + j];
        }
    if (bad) *sFail = 1;
}
__device__ int phase_ldlt(const Dev& D, const Ctx& c, double* A, int ld, double* scratch, double* brow) {
    const int n = D.n, tid = c.tid(), lane = tid & 31, warp = tid >> 5;
    const int n1 = n + 1;
    double* Xs = scratch;               // 6 x (n + 1): unscaled panel, column-major by panel column (conflict-free for lanes over rows)
    double* Ls = scratch + 6 * n1;      // 6 x (n + 1): scaled panel (= the final L entries)
    __shared__ double s_L[36], s_dinv[6];
    __shared__ int s_fail;
    for (int i = tid; i < n; i += NT) brow[i] = D.bs[i];
    if (tid == 0) { s_fail = 0; ldlt_factor6(A, ld, 0, s_L, s_dinv, &s_fail); }
    __syncthreads();
    if (s_fail) return 0;
    for (int k0 = 0; k0 < n; k0 += 6) {
        // (1) panel: row i below the block (and the rhs row, i == n): X = A21 L11^-T (unscaled), L21 = X D^-1
        for (int i = k0 + 6 + tid; i <= n; i += NT) {
            double* row = i < n ? A + (size_t)i * ld : brow;
            double xr[6];
#pragma unroll
            for (int cidx = 0; cidx < 6; ++cidx) {
                double v = row[k0 + cidx];
#pragma unroll
                for (int j = 0; j < cidx; ++j) v -= xr[j] * s_L[cidx * 6 + j];
                xr[cidx] = v;
            }
#pragma unroll
            for (int cidx = 0; cidx < 6; ++cidx) {
                const double l = xr[cidx] * s_dinv[cidx];
                Xs[cidx * n1 + i] = xr[cidx]; Ls[cidx * n1 + i] = l; row[k0 + cidx] = l;
            }
        }
        __syncthreads();
        // (2) trailing update A22[i][j] -= sum_c X[i][c] L21[j][c];  warp 0: next diagonal block, then its factorisation
        const int r0 = k0 + 6;
        if (warp == 0) {
            if (r0 < n) {
                if (lane < 21) {
                    int i = 0, t = lane;
                    while (t > i) { t -= i + 1; ++i; }      // lane -> (i, j = t), j <= i
                    double sacc = 0;
#pragma unroll
                    for (int cidx = 0; cidx < 6; ++cidx) sacc += Xs[cidx * n1 + r0 + i] * Ls[cidx * n1 + r0 + t];
                    A[(size_t)(r0 + i) * ld + r0 + t] -= sacc;
                }
                __syncwarp();
                if (lane == 0) ldlt_factor6(A, ld, r0, s_L, s_dinv, &s_fail);
            }
        } else {
            // two rows per warp and pass: the scaled panel entries L21[j][:] are loaded once for both
            for (int ia = r0 + 6 + (warp - 1); ia <= n; ia += 2 * (NWARP - 1)) {
                const int ib = ia + (NWARP - 1);
                const bool hasB = ib <= n;
                double* rowA = ia < n ? A + (size_t)ia * ld : brow;
                double* rowB = !hasB ? rowA : (ib < n ? A + (size_t)ib * ld : brow);
                double xa[6], xb[6];
#pragma unroll
                for (int cidx = 0; cidx < 6; ++cidx) { xa[cidx] = Xs[cidx * n1 + ia]; xb[cidx] = hasB ? Xs[cidx * n1 + ib] : 0.0; }
                const int jendA = ia < n ? ia : n - 1;
                const int jendB = hasB ? (ib < n ? ib : n - 1) : -1;
                const int jmax = jendA > jendB ? jendA : jendB;
                for (int j0 = r0 + lane; j0 <= jmax; j0 += 128) {
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int j = j0 + 32 * u;
                        if (j <= jmax) {
                            double l[6];
#pragma unroll
                            for (int cidx = 0; cidx < 6; ++cidx) l[cidx] = Ls[cidx * n1 + j];
                            if (j <= jendA) {
                                double sacc = 0;
#pragma unroll
                                for (int cidx = 0; cidx < 6; ++cidx) sacc += xa[cidx] * l[cidx];
                                rowA[j] -= sacc;
                            }
                            if (j <= jendB) {
                                double sacc = 0;
#pragma unroll
                                for (int cidx = 0; cidx < 6; ++cidx) sacc += xb[cidx] * l[cidx];
                                rowB[j] -= sacc;
                            }
                        }
                    }
                }
            }
        }
        __syncthreads();
        if (s_fail) return 0;
    }
    // L^T x = z by warp 0 (column-oriented, warp-synchronous)
    if (warp == 0) {
        for (int k = n - 1; k >= 0; --k) {
            const double yk = brow[k];
            const double* Lk = A + (size_t)k * ld;
            for (int j = lane; j < k; j += 32) brow[j] -= Lk[j] * yk;
            __syncwarp();
        }
        for (int i = lane; i < n; i += 32) D.x[i] = brow[i];
    }
    __syncthreads();
    return 1;
}
// ---- the trial state of one LM step, part 1: every CTA applies the pose increments (SparseOptimizer::update,
//      VertexSE3Expmap::oplusImpl) to ALL poses into its own trial pose cache (so that no barrier is needed before the
//      residuals); CTA 0 also writes them to the trial buffer and returns the poses' share of computeScale ----
__device__ double phase_pose_trial(const Dev& D, const Ctx& c, const double* __restrict__ Pcur, double* __restrict__ Ptr, double* pcTr, double lambda) {
    double acc = 0;
    const bool rank0 = c.crank() == 0;
    for (int v = c.tid(); v < D.nP; v += NT) {
        double T[7];
#pragma unroll
        for (int i = 0; i < 7; ++i) T[i] = Pcur[7 * (size_t)v + i];
        const int h = D.hidx[v];
        if (h >= 0) {
            const double* u = D.x + 6 * (size_t)h;
            pose_oplus(T, u);
            if (rank0) {
#pragma unroll
                for (int i = 0; i < 6; ++i) acc += u[i] * (lambda * u[i] + D.bp[6 * (size_t)h + i]);
            }
        }
        if (rank0) {
#pragma unroll
            for (int i = 0; i < 7; ++i) Ptr[7 * (size_t)v + i] = T[i];
        }
        double* o = pcTr + PC * v;
#pragma unroll
        for (int k = 0; k < 7; ++k) o[k] = T[k];
        qtoR(T, o + 7);
        const float* cm = D.cam + 4 * (size_t)v;
        o[16] = (double)cm[0]; o[17] = (double)cm[1]; o[18] = (double)cm[2]; o[19] = (double)cm[3];
    }
    __syncthreads();
    return acc;
}
// ---- part 2, 8 lanes per point, one pass: landmark back-substitution x_l = Hll^-1 (bl - W^T x_p)
//      (block_solver.hpp:461-483; W^T x_p = w A^T (B x_p) = -sum_k t_k g_k (b_k . x_p)), the point update into the trial
//      buffer, its share of computeScale, and the residuals / robust chi2 / edge factors of the point's edges at the
//      trial state (computeActiveErrors + activeRobustChi2).  Returns (scale share, chi2 share).
//      FLY points per step (see phase_build_points): the loads of the lane's first edge of each point (the edge's Hessian block
//      eH, factors, observation) and the point's Dinv, bl and estimate are issued at the top of the step, then the pose
//      increments x_p those edges need; the sums keep the per-lane edge order and the point order of one point per step. ----
struct TrialEdge { int pose, h; double xn, yn, iz, w; double2 ob; double is2; };
__device__ __forceinline__ TrialEdge load_trial_edge(const Dev& D, const double* __restrict__ E, int e) {
    TrialEdge o;
    o.pose = ro(D.ePose + e); o.h = ro(D.eH + e);
    load_e4(E, e, o.xn, o.yn, o.iz, o.w);
    o.ob = ro_obs(D, e); o.is2 = (double)ro(D.invSigma2 + e);
    return o;
}
// the edge's share of W^T x_p, added into cl
__device__ __forceinline__ void add_backsub_edge(const double* pcache, const TrialEdge& o, const double* xp, double* cl) {
    const double* P = pcache + PC * o.pose;
    double t[6], b0[6], b1[6];
    edge_t(P + 7, o.xn, o.yn, t);
    edge_b(o.xn, o.yn, o.iz, b0, b1);
    double be0 = 0, be1 = 0;
#pragma unroll
    for (int k = 0; k < 6; ++k) { const double xa = xp[k]; be0 += b0[k] * xa; be1 += b1[k] * xa; }
    const double q = o.iz * o.w;
    be0 *= P[16] * P[16] * q; be1 *= P[17] * P[17] * q;
#pragma unroll
    for (int k = 0; k < 3; ++k) cl[k] += t[k] * be0 + t[3 + k] * be1;
}
__device__ double2 phase_points_trial(const Dev& D, const Ctx& c, const double* __restrict__ E, double* __restrict__ Eout, const double* Xcur,
                                      double* __restrict__ Xtr, const double* pcTr, double lambda) {
    constexpr int FLY = FLY_PT;
    const int sl = c.tid() & 7;
    const unsigned gmask = 0xFFu << (c.tid() & 24);
    const int G = c.nw() >> 3;
    double accS = 0, accC = 0;
    int a[FLY], b[FLY];
    step_ranges<FLY>(D.ptStart, D.nL, c.wid() >> 3, G, a, b);
    for (int p0 = c.wid() >> 3; p0 < D.nL; p0 += FLY * G) {
        TrialEdge first[FLY] = {};
        double Di[FLY][6] = {}, bl[FLY][3] = {}, X0[FLY][3] = {}, xp[FLY][6] = {};     // Di: 00 01 02 11 12 22
#pragma unroll
        for (int j = 0; j < FLY; ++j) if (a[j] + sl < b[j]) first[j] = load_trial_edge(D, E, a[j] + sl);
#pragma unroll
        for (int j = 0; j < FLY; ++j) {
            const int p = p0 + j * G;
            if (p < D.nL) {
                load_dinv(D.PT, D.nL, p, Di[j]);
#pragma unroll
                for (int k = 0; k < 3; ++k) { bl[j][k] = D.bl[3 * (size_t)p + k]; X0[j][k] = Xcur[3 * (size_t)p + k]; }
            }
        }
#pragma unroll
        for (int j = 0; j < FLY; ++j)
            if (a[j] + sl < b[j] && first[j].h >= 0) {
#pragma unroll
                for (int k = 0; k < 6; ++k) xp[j][k] = D.x[6 * (size_t)first[j].h + k];
            }
        int na[FLY], nb[FLY];
        step_ranges<FLY>(D.ptStart, D.nL, p0 + FLY * G, G, na, nb);
#pragma unroll
        for (int j = 0; j < FLY; ++j) {
            const int p = p0 + j * G;
            if (p >= D.nL) break;
            const bool has = a[j] + sl < b[j];
            double cl[3] = {0, 0, 0};
            if (has && first[j].h >= 0) add_backsub_edge(c.pc, first[j], xp[j], cl);
            for (int e = a[j] + sl + 8; e < b[j]; e += 8) {
                const TrialEdge o = load_trial_edge(D, E, e);
                if (o.h >= 0) add_backsub_edge(c.pc, o, D.x + 6 * (size_t)o.h, cl);
            }
#pragma unroll
            for (int o = 4; o; o >>= 1) {
#pragma unroll
                for (int i = 0; i < 3; ++i) cl[i] += __shfl_xor_sync(gmask, cl[i], o);
            }
            const double* dv = Di[j];
            const double bl0 = bl[j][0], bl1 = bl[j][1], bl2 = bl[j][2];
            const double c0 = cl[0] + bl0, c1 = cl[1] + bl1, c2 = cl[2] + bl2;
            const double u0 = dv[0] * c0 + dv[1] * c1 + dv[2] * c2, u1 = dv[1] * c0 + dv[3] * c1 + dv[4] * c2, u2 = dv[2] * c0 + dv[4] * c1 + dv[5] * c2;
            double X[3] = {X0[j][0] + u0, X0[j][1] + u1, X0[j][2] + u2};
            if (sl == 0) {
                Xtr[3 * (size_t)p] = X[0]; Xtr[3 * (size_t)p + 1] = X[1]; Xtr[3 * (size_t)p + 2] = X[2];
                accS += u0 * (lambda * u0 + bl0) + u1 * (lambda * u1 + bl1) + u2 * (lambda * u2 + bl2);
            }
            if (has) accC += edge_error(D, pcTr + PC * first[j].pose, X, a[j] + sl, first[j].ob, first[j].is2, Eout);
            for (int e = a[j] + sl + 8; e < b[j]; e += 8)
                accC += edge_error(D, pcTr + PC * ro(D.ePose + e), X, e, ro_obs(D, e), (double)ro(D.invSigma2 + e), Eout);
        }
#pragma unroll
        for (int j = 0; j < FLY; ++j) { a[j] = na[j]; b[j] = nb[j]; }
    }
    return make_double2(accS, accC);
}
__device__ void phase_finalize(const Dev& D, const Ctx& c, const double* pts) {
    const int nw = c.nw();
    for (int e = c.wid(); e < D.nE; e += nw) {
        const double e0 = D.err[2 * (size_t)e], e1 = D.err[2 * (size_t)e + 1];
        const int o = D.eOrig[e];
        D.outChi2[o] = (double)D.invSigma2[e] * (e0 * e0 + e1 * e1);   // e->chi2() from the last computed _error (Optimizer.cc:1425)
        const double* P = c.pc + PC * D.ePose[e];
        double r[3]; qrot(P, pts + 3 * (size_t)D.ePt[e], r);
        D.outDepthPos[o] = r[2] + P[6] > 0.0;
    }
    // the estimate ends in whichever buffer was current last; the caller reads D.poses and D.outPts, in its own point order
    for (int i = c.wid(); i < 3 * D.nL; i += nw) {
        const int r = i / 3;
        D.outPts[3 * (size_t)D.ptOrig[r] + (i - 3 * r)] = pts[i];
    }
}

// =============================================================================================
// The persistent kernel: SparseOptimizer::optimize (sparse_optimizer.cpp:354-418) around
// OptimizationAlgorithmLevenberg::solve (optimization_algorithm_levenberg.cpp:61-168), one cluster per problem.
// The LM state is uniform: thread 0 of every CTA runs the policy on the CTA's copy in shared memory, from values every CTA
// reads identically after a cluster barrier, and the other threads read the outcome after the next CTA barrier.  The
// descriptor and that state stay in shared memory so that the registers (128 per thread) go to the phases.
// Dynamic shared memory: 2 pose caches (PC x maxP doubles each, maxP = most poses of any loaded problem, fixed keyframes included) |
// LDLT panel scratch (2 x 6 x (6 maxF + 1), maxF = most FREE poses) | rhs row (6 maxF) | reduced camera system (smemMatrixN^2).
// =============================================================================================
struct LoopState {
    Levenberg lm;
    double currentChi = 0, firstChi = 0, iniChi = 0, rho = 0;
    int cj = 0, trials = 0, qmax = 0, term = 0, ok = 1;
    int cur = 0;                        // the side of the double buffers that holds the current state: 0 = (E4a, poses, pts), 1 = (E4b, posesB, ptsB)
    bool accepted = false, more = false;   // the last trial was accepted / the iteration runs another trial
    unsigned seq = 0, doneTarget = 0;      // phases opened so far (Job::seq) and the chunks they hold (Job::done once they are joined)
};
__shared__ int2 s_grant;                   // the claim group of a helper CTA: chunks [x, y)
__device__ __forceinline__ unsigned long long job_word(unsigned seq, int nCh) {
    return ((unsigned long long)(seq % 65535u + 1u) << 48) | ((unsigned long long)nCh << 24);
}
// ---- a data-parallel phase of nCh chunks in the owner cluster: CTA 0 opens it (pose-cache mirror, phase fields, then the claim
//      word with release semantics), every owner CTA claims and serves chunks until the word is exhausted, then waits with its
//      own acquire until the problem's done count holds every chunk of the phase (helper CTAs may have served some).  The owners
//      never wait for a helper to start, so the result and the progress do not depend on helpers being resident. ----
__device__ void owner_phase(const Dev& D, LoopState& S, const double* pc, int phase, int side, double lambda, int nCh) {
    Job* J = D.job;
    const int tid = threadIdx.x;
    if (sreg_ctarank() == 0) {
        for (int i = tid; i < PC * D.nP; i += NT) D.pcm[i] = pc[i];
        if (tid == 0) { J->phase = phase; J->side = side; J->lambda = lambda; J->seq = S.seq + 1; }
        __syncthreads();
        if (tid == 0) { __threadfence(); atomicExch(&J->word, job_word(S.seq + 1, nCh)); }
    }
    if (tid == 0) {
        ++S.seq; S.doneTarget += nCh;
        const unsigned tag = (unsigned)(job_word(S.seq, 0) >> 48);
        while (job_tag(ld_acquire(&J->word)) != tag) __nanosleep(32);      // ranks > 0 may arrive before CTA 0 has opened it
    }
    __syncthreads();
    // the owner's warps claim one chunk at a time on their own: no CTA barrier inside the loop, and a warp's release of its
    // chunk stalls only that warp.  (Every claim an owner makes is of this phase: CTA 0 opens the next one only after a
    // cluster barrier that every owner thread reaches after leaving this loop.)
    const int lane = tid & 31;
    for (;;) {
        int ch = 0;
        if (lane == 0) {
            const unsigned long long old = atomicAdd(&J->word, 1ull);
            ch = job_next(old) < job_count(old) ? job_next(old) : -1;
        }
        ch = __shfl_sync(0xffffffffu, ch, 0);
        if (ch < 0) break;
        serve_chunk(D, pc, phase, side, lambda, ch);
        __syncwarp();
        if (lane == 0) { __threadfence(); atomicAdd(&J->done, 1u); }
    }
    __syncthreads();
    if (tid == 0) while (ld_acquire(&J->done) < S.doneTarget) __nanosleep(32);
    __syncthreads();
}
// ---- a helper CTA: scans the problems round-robin from its own index (one lane per problem), claims a group of chunks of any
//      open phase, loads that problem's descriptor and pose-cache mirror into its shared memory when the problem or the phase
//      changed, and serves the group.  It leaves once every problem has finished. ----
__device__ void helper_loop(const Dev* __restrict__ probs, int nProb, const unsigned long long* finished, Dev& sD, double* spc, int hIdx) {
    __shared__ int s_q, s_phase, s_side; __shared__ unsigned s_seq; __shared__ double s_lambda;
    const int tid = threadIdx.x, lane = tid & 31;
    int start = hIdx % nProb, cachedQ = -1;
    unsigned cachedSeq = 0;
    for (;;) {
        if (tid < 32) {
            int q = -1;
            if (ld_acquire(finished) >= (unsigned long long)nProb) q = -2;
            for (int b = 0; b < nProb && q == -1; b += 32) {
                const int qi = (start + b + lane) % nProb;
                Job* J = b + lane < nProb ? probs[qi].job : nullptr;
                bool avail = false;
                if (J) { const unsigned long long w = ld_relaxed(&J->word); avail = job_next(w) < job_count(w); }
                unsigned m = __ballot_sync(0xffffffffu, avail);
                while (m && q == -1) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    int got = 0;
                    if (lane == src) {
                        const unsigned long long old = atomicAdd(&J->word, (unsigned long long)NWARP);
                        const int k0 = job_next(old), n = job_count(old);
                        if (k0 < n) {
                            got = 1;
                            __threadfence();
                            s_grant = make_int2(k0, min(k0 + NWARP, n));
                            s_seq = *(volatile unsigned*)&J->seq; s_phase = *(volatile int*)&J->phase; s_side = *(volatile int*)&J->side;
                            s_lambda = *(volatile double*)&J->lambda;
                        }
                    }
                    if (__shfl_sync(0xffffffffu, got, src)) q = __shfl_sync(0xffffffffu, qi, src);
                }
            }
            if (lane == 0) { s_q = q; if (q == -1) __nanosleep(256); }
        }
        __syncthreads();
        const int q = s_q;
        if (q == -2) break;
        if (q >= 0) {
            if (q != cachedQ || s_seq != cachedSeq) {
                static_assert(sizeof(Dev) % 8 == 0, "Dev is copied in 8-byte words");
                for (int i = tid; i < (int)(sizeof(Dev) / 8); i += NT)
                    reinterpret_cast<unsigned long long*>(&sD)[i] = reinterpret_cast<const unsigned long long*>(probs + q)[i];
                __syncthreads();
                for (int i = tid; i < PC * sD.nP; i += NT) spc[i] = sD.pcm[i];
                cachedQ = q; cachedSeq = s_seq;
                __syncthreads();
            }
            // the group: warp w serves chunk g.x + w; then the CTA counts the group (helped, then done, each after a release fence)
            const int2 g = s_grant;
            const int ch = g.x + (tid >> 5);
            if (ch < g.y) serve_chunk(sD, spc, s_phase, s_side, s_lambda, ch);
            __syncthreads();
            if (tid == 0) {
                __threadfence(); atomicAdd(&sD.job->helped, (unsigned)(g.y - g.x));
                __threadfence(); atomicAdd(&sD.job->done, (unsigned)(g.y - g.x));
            }
            start = q;
        }
        __syncthreads();
    }
}
// Grid: nProb owner clusters (problem blockIdx.x / cluster size), then helper clusters of the same size, each of whose CTAs serves
// chunks of any problem on its own (helper_loop) until `finished` counts every problem.
__global__ void __launch_bounds__(NT, LBA_MINB) lba_cluster_kernel(const Dev* __restrict__ probs, const volatile int* stop, int smemMatrixN, int maxP, int maxF,
                                                                   int nProb, unsigned long long* finished) {
    extern __shared__ double s_dyn[];
    __shared__ double s_red[NT];
    __shared__ Dev s_D;
    __shared__ alignas(LoopState) unsigned char s_state[sizeof(LoopState)];   // constructed by thread 0 (a __shared__ variable has no initialiser)
    LoopState& S = *reinterpret_cast<LoopState*>(s_state);
    Ctx c;
    c.slot = 0; c.sm = s_red;
    double* s_pc = s_dyn;                        // pose cache, linearisation state
    double* s_pcT = s_pc + PC * maxP;            // pose cache, trial state
    double* s_col = s_pcT + PC * maxP;           // 2 x 6 x (6 maxF + 1) panel scratch
    double* s_rhs = s_col + 72 * maxF + 12;      // 6 maxF: rhs row of the LDLT
    double* s_mat = s_rhs + 6 * maxF + 2;
    c.pc = s_pc;
    if ((int)blockIdx.x >= nProb * c.csize()) {
        helper_loop(probs, nProb, finished, s_D, s_pc, (int)blockIdx.x - nProb * c.csize());
        return;
    }
    if (c.tid() == 0) {
        s_D = probs[blockIdx.x / c.csize()];
        new (&S) LoopState();
        if (c.crank() == 0) {     // the claim word was left exhausted by the last run (or zeroed by the upload): no claim succeeds before the first phase opens
            Job* J = s_D.job;
            J->done = 0; J->helped = 0; J->seq = 0;
        }
    }
    __syncthreads();
    const Dev& D = s_D;
    // double-buffered state: the trial of an LM step is written next to the current estimate and the two swap when the
    // step is accepted, so a rejected step needs no restore ("pop") pass
    auto cur = [&](double* a, double* b) { return S.cur ? b : a; };
    auto trial = [&](double* a, double* b) { return S.cur ? a : b; };
    auto poll = [&]() { return (c.crank() == 0 && c.tid() == 0 && stop && stop[blockIdx.x / c.csize()]) ? 1 : 0; };

    const int nw = c.nw();
    for (int i = c.wid(); i < D.nP; i += nw) {
        double* T = D.poses + 7 * (size_t)i;
#pragma unroll
        for (int k = 0; k < 7; ++k) T[k] = D.initPoses[7 * (size_t)i + k];
        qnormalize(T);                                              // SE3Quat(q, t) constructor
    }
    for (int i = c.wid(); i < 3 * D.nL; i += nw) {
        const int r = i / 3;
        D.pts[i] = D.initPts[3 * (size_t)D.ptOrig[r] + (i - 3 * r)];
    }
    for (int i = c.wid(); i < 2 * D.nE; i += nw) D.err[i] = 0.0;
    for (int i = c.wid(); i < D.n; i += nw) D.x[i] = 0.0;
    int flag;
    cluster_sum(D, c, 0.0, poll(), flag);        // initial terminate() poll + publishes the poses
    if (c.tid() == 0) S.term = flag;
    load_pose_cache(D, D.poses, s_pc);

    __shared__ unsigned long long s_tph[11];     // per-phase ns of CTA 0 (thread 0), [10] = tick
    if (c.tid() < 11) s_tph[c.tid()] = 0;
    __syncthreads();
#define TICK() do { if (c.wid() == 0) s_tph[10] = globaltimer_ns(); } while (0)
#define TOCK(i) do { if (c.wid() == 0) s_tph[i] += globaltimer_ns() - s_tph[10]; } while (0)
    for (int it = 0; it < D.iterations && !S.term && S.ok; ++it) {
        // the first iteration starts the LM policy: with the user's lambda before the build, else with H's largest diagonal entry after it
        const bool lambdaKnown = it > 0 || D.userLambdaInit > 0;
        // computeActiveErrors at the start of solve(): after an accepted step the state, the errors and the edge factors are
        // exactly those of the accepted trial (same arithmetic), so only the first iteration evaluates them
        if (it == 0) {
            if (lambdaKnown && c.tid() == 0) S.lm.start(D.userLambdaInit, 0.0);
            TICK();
            const double chi = cluster_sum(D, c, phase_errors(D, c, cur(D.pts, D.ptsB), cur(D.E4a, D.E4b)), 0, flag);
            if (c.tid() == 0) S.currentChi = chi;
            TOCK(0);
        }
        if (c.tid() == 0) {
            S.iniChi = S.currentChi;
            if (it == 0) S.firstChi = S.iniChi;
            S.rho = 0; S.qmax = 0;
        }
        const int nPtCh = (D.nL + PCH - 1) / PCH;
        TICK();
        owner_phase(D, S, s_pc, PH_BUILD, S.cur, lambdaKnown ? S.lm.lambda : -1.0, nPtCh + D.taskChunkStart[D.nF]);
        csync();
        TOCK(1); TICK();
        phase_build_poses_combine(D, c);
        TOCK(2);
        if (!lambdaKnown) {
            csync();
            const double maxDiag = phase_maxdiag(D, c);
            if (c.tid() == 0) S.lm.start(0.0, maxDiag);
            __syncthreads();
        }
        bool needPrep = !lambdaKnown;
        do {
            if (needPrep) {
                TICK();
                owner_phase(D, S, s_pc, PH_PREP, S.cur, S.lm.lambda, nPtCh);
                csync();
                TOCK(3);
            }
            int ok2 = 1;
            if (D.nF) {
                // reduced camera system: CTA 0's shared memory; the other CTAs of the cluster reach it as distributed shared memory
                const bool matInSmem = D.n <= smemMatrixN && D.n > 0;
                TICK();
                owner_phase(D, S, s_pc, PH_SCHUR, S.cur, S.lm.lambda, D.nChunks);
                csync();
                TOCK(4); TICK();
                phase_schur_combine(D, c, S.lm.lambda, matInSmem ? cg::this_cluster().map_shared_rank(s_mat, 0) : D.Hs, D.n);   // every CTA writes entries into CTA 0's shared memory through DSMEM
                csync();
                TOCK(6); TICK();
                if (c.crank() == 0) {
                    ok2 = phase_ldlt(D, c, matInSmem ? s_mat : D.Hs, D.n, s_col, s_rhs);
                    if (c.tid() == 0) D.partial[4 * PSLOT] = (double)ok2;
                }
                csync();
                ok2 = (int)D.partial[4 * PSLOT];
                TOCK(5);
            }
            TICK();
            const double sP = phase_pose_trial(D, c, cur(D.poses, D.posesB), trial(D.poses, D.posesB), s_pcT, S.lm.lambda);
            TOCK(7); TICK();
            const double2 sc = phase_points_trial(D, c, cur(D.E4a, D.E4b), trial(D.E4a, D.E4b), cur(D.pts, D.ptsB), trial(D.pts, D.ptsB), s_pcT,
                                                  S.lm.lambda);
            double scale0, tempChi;
            cluster_sum2(D, c, sP + sc.x, sc.y, poll(), flag, scale0, tempChi);
            TOCK(8);
            if (c.tid() == 0) {
                S.term = flag;
                S.accepted = S.lm.trial(S.currentChi, tempChi, scale0, ok2, S.rho);
                if (S.accepted) S.cur ^= 1;                     // a rejected trial's buffers are simply abandoned (pop)
                ++S.qmax; ++S.trials;
                S.more = S.rho < 0 && S.qmax < Levenberg::maxTrials && !S.term;
                if (!S.more) { ++S.cj; S.ok = S.lm.iteration_done(S.qmax, S.rho, S.iniChi, S.currentChi); }
            }
            __syncthreads();
            if (S.accepted) {
                for (int i = c.tid(); i < PC * D.nP; i += NT) s_pc[i] = s_pcT[i];
                __syncthreads();
            }
            needPrep = true;
        } while (S.more);
    }
    phase_finalize(D, c, cur(D.pts, D.ptsB));
    if (S.cur) for (int i = c.wid(); i < 7 * D.nP; i += nw) D.poses[i] = D.posesB[i];
    if (c.wid() == 0) for (int i = 0; i < 9; ++i) D.stats[8 + i] = (double)s_tph[i];
    if (c.wid() == 0) {
        D.stats[0] = S.cj; D.stats[1] = S.trials; D.stats[2] = S.lm.lambda; D.stats[3] = S.currentChi; D.stats[4] = S.firstChi;
        D.stats[17] = (double)*(volatile unsigned*)&D.job->helped;   // complete: every phase has been joined
        __threadfence();
        atomicAdd(finished, 1ull);
    }
}

// =============================================================================================
// BlockSolver::buildStructure (block_solver.hpp:143-295) on the device: one CTA per problem turns the caller's edge list
// into the index structures of the LM kernel -- the internal point order, edges sorted by point (stable), the (free pose, point)
// -> edge table, the per-pose edge lists (the pose-major edge order), the pair list of every off-diagonal Schur block in
// pose-major indices, and the chunked work list.  Only the raw graph (28 B per edge) crosses PCIe; the derived lists (~2.3 MB per
// 40k-edge problem) never exist on the host.
// The internal point order sorts the points by the ascending list of their observing free poses (the first four, points seen
// only by fixed poses last), ties by the caller's index.  Points with the same observers are then neighbours, so the points a
// pose pair shares form a few long runs, and the lanes of a Schur chunk read neighbouring point records and pose-major entries
// instead of lines scattered over the caller's order.  Every list is in a deterministic order (by point rank, ties by the
// caller's edge index).
// status: 0 ok, 1 edge index out of range, 2 duplicate (point, keyframe) observation, 3 pair list larger than sized.
// =============================================================================================
constexpr int BT = 1024;
// Ascending bitonic sort of key[n2] (global memory, n2 a power of two), all threads of the CTA.  The stages whose stride is below
// the tile of 2 BT keys run on that tile in shared memory, so only strides of 2 BT and more cost a pass over global memory.
constexpr int SORT_TILE = 2 * BT;
__device__ __forceinline__ void bitonic_pair(unsigned long long* k, int base, int k2, int j, int pr) {   // pair pr of stage k2, stride j
    const int lo = 2 * pr - (pr & (j - 1)), hi = lo + j;
    const unsigned long long a = k[lo], b = k[hi];
    if ((a > b) == (((base + lo) & k2) == 0)) { k[lo] = b; k[hi] = a; }
}
__device__ void bitonic_sort_keys(unsigned long long* key, int n2, unsigned long long* tile) {
    const int T = min(n2, SORT_TILE), tid = threadIdx.x;
    for (int k2 = T; k2 <= n2; k2 <<= 1) {
        for (int j = k2 >> 1; j >= T; j >>= 1) {
            for (int pr = tid; pr < n2 / 2; pr += BT) bitonic_pair(key, 0, k2, j, pr);
            __syncthreads();
        }
        for (int t0 = 0; t0 < n2; t0 += T) {
            for (int i = tid; i < T; i += BT) tile[i] = key[t0 + i];
            __syncthreads();
            for (int s2 = k2 == T ? 2 : k2; s2 <= k2; s2 <<= 1)      // the first round sorts every tile whole
                for (int j = min(s2, T) >> 1; j > 0; j >>= 1) {
                    if (tid < T / 2) bitonic_pair(tile, t0, s2, j, tid);
                    __syncthreads();
                }
            for (int i = tid; i < T; i += BT) key[t0 + i] = tile[i];
            __syncthreads();
        }
    }
}
__global__ void __launch_bounds__(BT) lba_build_structure_kernel(Dev* probs, int* status) {
    Dev& D = probs[blockIdx.x];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nL = D.nL, nE = D.nE, nF = D.nF, nP = D.nP;
    const int nOff = nF * (nF - 1) / 2, nTasks = nF + nOff;
    __shared__ int s_sm[33];
    __shared__ int s_err;
    __shared__ unsigned long long s_tile[SORT_TILE];
    int* ptStart = const_cast<int*>(D.ptStart); int* ptOrig = const_cast<int*>(D.ptOrig);
    int* ePt = const_cast<int*>(D.ePt); int* ePose = const_cast<int*>(D.ePose); int* eH = const_cast<int*>(D.eH); int* eOrig = const_cast<int*>(D.eOrig);
    double* obs = const_cast<double*>(D.obs); float* is2 = const_cast<float*>(D.invSigma2);
    int* poseEdges = const_cast<int*>(D.poseEdges); int* poseEdgePt = const_cast<int*>(D.poseEdgePt);
    int2* pairs = const_cast<int2*>(D.pairs); int* pairPt = const_cast<int*>(D.pairPt);
    int4* chunkHdr = const_cast<int4*>(D.chunkHdr); int* taskChunkStart = const_cast<int*>(D.taskChunkStart);
    if (tid == 0) { s_err = 0; *D.job = Job{}; }     // an exhausted claim word: no claim succeeds before the LM kernel opens a phase
    for (int i = tid; i <= nL; i += BT) D.bCnt[i] = 0;
    for (size_t i = tid; i < (size_t)nF * nL; i += BT) D.bEid[i] = -1;
    __syncthreads();
    // 1. edges per point (bCnt, by the caller's point index p)
    for (int e = tid; e < nE; e += BT) {
        const int p = D.rawEdgePoint[e], c = D.rawEdgePose[e];
        if (p < 0 || p >= nL || c < 0 || c >= nP) s_err = 1;
        else atomicAdd(&D.bCnt[p], 1);
    }
    __syncthreads();
    if (s_err) { if (tid == 0) status[blockIdx.x] = s_err; return; }
    // 2. where every point's edges start in the caller's point order (exclusive scan, into the cursors of step 3)
    block_prefix<BT>(nL, D.bCursor, s_sm, [&](int i) { return D.bCnt[i]; });
    // 3. group by point (arbitrary order), then order every point's slice by the caller's edge index; afterwards bCursor[p] is the
    //    end of point p's slice of bTmp.  The point's sort key: its four lowest observing free poses (Hessian blocks) in
    //    ascending order, in `sb` bits each, then the caller's index in `ib` bits, so that every key is distinct (the order is
    //    that of 16-bit pose fields with ties broken by the caller's index whenever nF < 2^sb - 1, i.e. for every problem whose
    //    pose caches fit in shared memory; beyond that the poses share the top field value, which still leaves a valid order).
    //    A missing observer is the all-ones field value: fewer free observers sort after more, fixed-only points last.
    for (int e = tid; e < nE; e += BT) D.bTmp[atomicAdd(&D.bCursor[D.rawEdgePoint[e]], 1)] = e;
    __syncthreads();
    const int n2 = nL > 1 ? 1 << (32 - __clz(nL - 1)) : 1;
    {
        const int ib = 32 - __clz(nL), sb = (64 - ib) / 4;        // 2^ib > nL: no real key is all ones, the padding's value
        const unsigned none = (1u << sb) - 1;
        for (int p = tid; p < n2; p += BT) {
            unsigned long long key = ~0ull;
            if (p < nL) {
                const int b = D.bCursor[p], a = b - D.bCnt[p];
                for (int i = a + 1; i < b; ++i) {
                    const int v = D.bTmp[i];
                    int j = i - 1;
                    while (j >= a && D.bTmp[j] > v) { D.bTmp[j + 1] = D.bTmp[j]; --j; }
                    D.bTmp[j + 1] = v;
                }
                unsigned s[4] = {none, none, none, none};
                for (int i = a; i < b; ++i) {
                    const int h = D.hidx[D.rawEdgePose[D.bTmp[i]]];
                    unsigned v = h < 0 ? none : min((unsigned)h, none - 1);
#pragma unroll
                    for (int q = 0; q < 4; ++q) { const unsigned lo = min(s[q], v); v = max(s[q], v); s[q] = lo; }
                }
                key = (unsigned long long)p;
#pragma unroll
                for (int q = 0; q < 4; ++q) key |= (unsigned long long)s[q] << (ib + (3 - q) * sb);
            }
            D.bKey[p] = key;
        }
    }
    __syncthreads();
    if (nL > 0) bitonic_sort_keys(D.bKey, n2, s_tile);
    for (int r = tid; r < nL; r += BT) ptOrig[r] = (int)(D.bKey[r] & ((1ull << (32 - __clz(nL))) - 1));
    __syncthreads();
    // 4. ptStart over the internal order, then every point's edges in their slots: internal edge id = ptStart[rank] + position in
    //    the point's caller-ordered slice (a stable sort of the edges by point rank)
    const int ptEnd = block_prefix<BT>(nL, ptStart, s_sm, [&](int r) { return D.bCnt[ptOrig[r]]; });
    if (tid == 0) ptStart[nL] = ptEnd;
    for (int r = tid; r < nL; r += BT) {
        const int p = ptOrig[r], n = D.bCnt[p], a = D.bCursor[p] - n, k0 = ptStart[r];
        for (int i = 0; i < n; ++i) {
            const int e = D.bTmp[a + i], c = D.rawEdgePose[e], k = k0 + i;
            ePt[k] = r; ePose[k] = c; eOrig[k] = e;
            obs[2 * (size_t)k] = D.rawObs[2 * (size_t)e]; obs[2 * (size_t)k + 1] = D.rawObs[2 * (size_t)e + 1];
            is2[k] = D.rawInvSigma2[e];
            const int h = D.hidx[c];
            eH[k] = h;
            if (h >= 0 && atomicCAS(&D.bEid[(size_t)h * nL + r], -1, k) != -1) s_err = 2;
        }
    }
    __syncthreads();
    if (s_err) { if (tid == 0) status[blockIdx.x] = s_err; return; }
    // 5. items per task: edges of a free pose / points shared by a pair of free poses; warp per task, ballot over points
    auto taskRows = [&](int t, const int*& r1, const int*& r2) {
        if (t < nF) { r1 = D.bEid + (size_t)t * nL; r2 = r1; return; }
        int i1 = 0, rem = t - nF;
        while (rem >= nF - 1 - i1) { rem -= nF - 1 - i1; ++i1; }
        r1 = D.bEid + (size_t)i1 * nL; r2 = D.bEid + (size_t)(i1 + 1 + rem) * nL;
    };
    for (int t = warp; t < nTasks; t += BT / 32) {
        const int *r1, *r2;
        taskRows(t, r1, r2);
        int cnt = 0;
#pragma unroll 4
        for (int p0 = 0; p0 < nL; p0 += 32) {
            const int p = p0 + lane;
            const bool f = p < nL && r1[p] >= 0 && r2[p] >= 0;
            cnt += __popc(__ballot_sync(0xffffffffu, f));
        }
        if (lane == 0) D.bTaskLen[t] = cnt;
    }
    __syncthreads();
    // 6. where every task's items and chunks start (pose lists and pair lists are separate arrays)
    block_prefix<BT>(nF, D.bItemStart, s_sm, [&](int t) { return D.bTaskLen[t]; });
    const int nPairItems = block_prefix<BT>(nOff, D.bItemStart + nF, s_sm, [&](int i) { return D.bTaskLen[nF + i]; });
    if (nPairItems > D.pairCap) s_err = 3;
    const int nChunks = block_prefix<BT>(nTasks, taskChunkStart, s_sm, [&](int t) { return (D.bTaskLen[t] + SCH - 1) / SCH; });
    if (tid == 0) taskChunkStart[nTasks] = nChunks;
    if (nChunks > D.chunkCap) s_err = 3;
    __syncthreads();
    if (s_err) { if (tid == 0) status[blockIdx.x] = s_err; return; }
    // 7. the lists themselves (ascending point rank = ascending internal edge id) and the chunk headers; the pose lists first: the
    //    position of an edge in them is its pose-major index (kept in bTmp, free since step 4), and the pair lists hold those
    for (int pass = 0; pass < 2; ++pass) {
        for (int t = (pass ? nF : 0) + warp; t < (pass ? nTasks : nF); t += BT / 32) {
            const int *r1, *r2;
            taskRows(t, r1, r2);
            int pos = D.bItemStart[t];
            for (int p0 = 0; p0 < nL; p0 += 32) {
                const int p = p0 + lane;
                const int e1 = p < nL ? r1[p] : -1, e2 = p < nL ? r2[p] : -1;
                const bool f = e1 >= 0 && e2 >= 0;
                const unsigned m = __ballot_sync(0xffffffffu, f);
                if (f) {
                    const int k = pos + __popc(m & ((1u << lane) - 1));
                    if (t < nF) { poseEdges[k] = e1; poseEdgePt[k] = p; D.bTmp[e1] = k; }
                    else { pairs[k] = make_int2(D.bTmp[e1], D.bTmp[e2]); pairPt[k] = p; }
                }
                pos += __popc(m);
            }
        }
        __syncthreads();
    }
    for (int t = tid; t < nTasks; t += BT) {
        int poseA, poseB = -1;
        if (t < nF) poseA = D.freePose[t];
        else {
            int i1 = 0, rem = t - nF;
            while (rem >= nF - 1 - i1) { rem -= nF - 1 - i1; ++i1; }
            poseA = D.freePose[i1]; poseB = D.freePose[i1 + 1 + rem];
        }
        const int len = D.bTaskLen[t], first = D.bItemStart[t];
        int ch = taskChunkStart[t];
        for (int f = 0; f < len; f += SCH) chunkHdr[ch++] = make_int4(first + f, min(SCH, len - f), poseA, poseB);
    }
    if (tid == 0) { D.nChunks = nChunks; status[blockIdx.x] = 0; }
}

// A graph built on the device (csrc/local_ba.cu) copied into its slot's uploaded block, as pack() copies a caller's graph: one CTA
// per slot; hidx / freePose from the fixed flags in pose order.
__global__ void __launch_bounds__(BT) lba_fill_kernel(Dev* probs, const FillSrc* src) {
    const Dev& D = probs[blockIdx.x];
    const FillSrc& F = src[blockIdx.x];
    const int tid = threadIdx.x;
    for (int i = tid; i < 7 * D.nP; i += BT) const_cast<double*>(D.initPoses)[i] = F.poses[i];
    for (int i = tid; i < 4 * D.nP; i += BT) const_cast<float*>(D.cam)[i] = F.cam[i];
    for (int i = tid; i < 3 * D.nL; i += BT) const_cast<double*>(D.initPts)[i] = F.points[i];
    for (int e = tid; e < D.nE; e += BT) {
        const_cast<int*>(D.rawEdgePoint)[e] = F.edgePoint[e]; const_cast<int*>(D.rawEdgePose)[e] = F.edgePose[e];
        const_cast<double*>(D.rawObs)[2 * e] = F.obs[2 * e]; const_cast<double*>(D.rawObs)[2 * e + 1] = F.obs[2 * e + 1];
        const_cast<float*>(D.rawInvSigma2)[e] = F.invSigma2[e];
    }
    if (tid == 0) {
        int nF = 0;
        for (int i = 0; i < D.nP; ++i) {
            const int h = F.fixed[i] ? -1 : nF++;
            const_cast<int*>(D.hidx)[i] = h;
            if (h >= 0) const_cast<int*>(D.freePose)[h] = i;
        }
    }
}

// =============================================================================================
// host side
// =============================================================================================
struct Packed {             // one uploaded problem: where its pieces live inside the arena
    int nP, nL, nE, nF;
    size_t posesOff, ptsOff, chi2Off, dposOff, statsOff, initPosesOff, initPtsOff;
};

struct Solver {
    int device, maxP, maxL, maxE, maxBatch;
    cudaStream_t st = nullptr;
    uint8_t* d_arena = nullptr; uint8_t* h_arena = nullptr; size_t arenaBytes = 0, perProblem = 0;
    Dev* d_probs = nullptr; std::vector<Dev> h_probs;
    std::vector<Packed> packed;
    int* h_stop = nullptr; int* d_stop = nullptr;   // mapped pinned stop flags, one per problem
    int* h_status = nullptr; int* d_status = nullptr;   // mapped pinned status words of the structure kernel
    cudaEvent_t evDone = nullptr, evRun = nullptr;   // evRun: end of the last run, on whatever stream the caller launched it
    cudaEvent_t evWait = nullptr;                    // blocking-sync event: upload / download sleep on it instead of spinning (device_utils.cuh)
    bool ranOnce = false;
    int nLoaded = 0, launches = 0, numSMs = 132;
    unsigned long long* d_finished = nullptr;        // problems finished in the running launch (helper CTAs leave when it reaches the batch)
    orbx::Staging stage;                             // lba_local_bundle_adjustment_batch's inputs and outputs (csrc/local_ba.cu)
    int localLaunches = 0;
    ~Solver() {
        cudaSetDevice(device);
        if (d_finished) cudaFree(d_finished);
        if (d_arena) cudaFree(d_arena);
        if (h_arena) cudaFreeHost(h_arena);
        if (d_probs) cudaFree(d_probs);
        if (h_stop) cudaFreeHost(h_stop);
        if (h_status) cudaFreeHost(h_status);
        if (evDone) cudaEventDestroy(evDone);
        if (evRun) cudaEventDestroy(evRun);
        if (evWait) cudaEventDestroy(evWait);
        if (st) cudaStreamDestroy(st);
    }
    static size_t al(size_t b) { return (b + 255) & ~(size_t)255; }
    static size_t outBlock(size_t nP, size_t nL, size_t nE) { return al(56 * nP) + al(24 * nL) + al(8 * nE) + al(nE) + al(512); }
    static size_t pairCapOf(size_t nP, size_t nE) { return nE * (nP > 1 ? nP - 1 : 1) / 2 + 1; }
    static size_t chunkCapOf(size_t nP, size_t nE) { return nP + nP * nP / 2 + 2 + (nE + pairCapOf(nP, nE)) / SCH + 1; }
    static size_t pow2Of(size_t n) { size_t p = 1; while (p < n) p <<= 1; return p; }
    static size_t need(size_t nP, size_t nL, size_t nE) {
        const size_t n = 6 * nP, pc = pairCapOf(nP, nE), cc = chunkCapOf(nP, nE), tasks = nP + nP * nP / 2 + 2;
        size_t b = outBlock(nP, nL, nE);                                          // poses, pts, chi2, depth flags, stats (downloaded in one copy)
        b += al(56 * nP) + al(24 * nL) + al(16 * nP) + 2 * al(4 * nP);            // uploaded: initial estimates, cam, hidx, freePose
        b += 2 * al(4 * nE) + al(16 * nE) + al(4 * nE);                           // uploaded: the caller's edges (point, pose, obs, invSigma2)
        b += al(4 * nL);                                                          // internal point order
        b += 4 * al(4 * nE) + al(16 * nE) + al(4 * nE) + al(4 * (nL + 1));        // edges sorted by point: ePt, ePose, eH, eOrig, obs, invSigma2; ptStart
        b += 2 * al(4 * nE) + al(8 * pc) + al(4 * pc);                            // poseEdges, poseEdgePt, pairs, pairPt
        b += al(16 * cc) + al(4 * (tasks + 1));                                   // chunk headers, task chunk starts
        b += 2 * al(4 * (nL + 1)) + al(4 * nE) + al(4 * nP * nL) + 2 * al(4 * tasks) + al(8 * pow2Of(nL));   // structure-build scratch
        b += al(24 * nL) + al(56 * nP) + al(24 * nL);                             // point state, second state buffers
        b += al(16 * nE) + 3 * al(32 * nE);                                       // err, edge factors x 2, pose-major copy
        b += al(288 * nP) + al(48 * nP) + al(48 * nL) + al(72 * nL) + al(24 * nL);   // Hpp, bp, Hll, PT, bl
        b += al(8 * 42 * cc) + al(8 * 28 * (nP + nE / SCH + 1));                  // Spart, Ppart
        b += al(8 * n * n) + al(8 * n) + al(8 * (n + 3 * nL)) + al(8 * (4 * PSLOT + 8));   // Hs, bs, x, partial
        b += al(sizeof(Job)) + al(8 * PC * nP);                                   // open phase, pose-cache mirror
        return b;
    }
    int init() {
        CK(cudaSetDevice(device));
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, device));
        if (orbx::require_sm90(prop.major, prop.minor)) return ORB_ERR_CUDA;
        numSMs = prop.multiProcessorCount;
        stage.device = device;
        perProblem = need(maxP, maxL, maxE);
        arenaBytes = perProblem * (size_t)maxBatch;
        CK(cudaMalloc(&d_arena, arenaBytes));
        {
            orbx::ScopedGpuAffinity numaLocal(device);     // pinned pages on the GPU's NUMA node (host_affinity.h)
            CK(cudaMallocHost(&h_arena, arenaBytes));
        }
        CK(cudaMalloc(&d_probs, sizeof(Dev) * maxBatch));
        CK(cudaMalloc(&d_finished, sizeof(unsigned long long)));
        CK(cudaHostAlloc(&h_stop, sizeof(int) * maxBatch, cudaHostAllocMapped));
        CK(cudaHostGetDevicePointer(&d_stop, h_stop, 0));
        CK(cudaHostAlloc(&h_status, sizeof(int) * maxBatch, cudaHostAllocMapped));
        CK(cudaHostGetDevicePointer(&d_status, h_status, 0));
        CK(cudaEventCreateWithFlags(&evDone, cudaEventDisableTiming));
        CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&evRun, cudaEventDisableTiming));
        CK(orbx::make_blocking_event(&evWait));
        h_probs.resize(maxBatch); packed.resize(maxBatch);
        return ORB_OK;
    }

    // Where a slot's uploaded block keeps the caller's graph (arena offsets)
    struct UpBlock { size_t poses, pts, cam, hidx, freePose, ePt, ePose, obs, isg; };

    // Lays slot `slot` of the arena out for a problem of the given sizes: the device views of every piece in h_probs[slot], the
    // download layout in packed[slot] and the uploaded block in U.  The problem's scalars are left to the caller.
    int layout(int slot, int nP, int nL, int nE, int nF, UpBlock& U) {
        const int n = 6 * nF;
        const int nOff = nF * (nF - 1) / 2, nTasks = nF + nOff;
        const size_t pc = pairCapOf(nP, nE), cc = chunkCapOf(nP, nE);
        const size_t base = perProblem * (size_t)slot;
        size_t off = base;
        auto carve = [&](size_t bytes) { size_t o = off; off += al(bytes); return o; };
        Dev& D = h_probs[slot]; memset(&D, 0, sizeof(D));
        Packed& K = packed[slot];
        K.nP = nP; K.nL = nL; K.nE = nE; K.nF = nF;
        D.nP = nP; D.nL = nL; D.nE = nE; D.nF = nF; D.n = n; D.pairCap = (int)pc; D.chunkCap = (int)cc;
        // --- output block: fixed layout (sized by the handle's maxima) so that one strided copy downloads every problem ---
        K.posesOff = carve(56 * (size_t)maxP); D.poses = (double*)(d_arena + K.posesOff);
        K.ptsOff = carve(24 * (size_t)maxL); D.outPts = (double*)(d_arena + K.ptsOff);
        K.chi2Off = carve(8 * (size_t)maxE); D.outChi2 = (double*)(d_arena + K.chi2Off);
        K.dposOff = carve((size_t)maxE); D.outDepthPos = (uint8_t*)(d_arena + K.dposOff);
        K.statsOff = carve(512); D.stats = (double*)(d_arena + K.statsOff);
        // --- uploaded block: the caller's graph ---
        const size_t upBase = off;
        U.poses = carve(56 * (size_t)nP); D.initPoses = (const double*)(d_arena + U.poses);
        U.pts = carve(24 * (size_t)nL); D.initPts = (const double*)(d_arena + U.pts);
        U.cam = carve(16 * (size_t)nP); D.cam = (const float*)(d_arena + U.cam);
        U.hidx = carve(4 * (size_t)nP); D.hidx = (const int*)(d_arena + U.hidx);
        U.freePose = carve(4 * (size_t)std::max(nF, 1)); D.freePose = (const int*)(d_arena + U.freePose);
        U.ePt = carve(4 * (size_t)nE); D.rawEdgePoint = (const int*)(d_arena + U.ePt);
        U.ePose = carve(4 * (size_t)nE); D.rawEdgePose = (const int*)(d_arena + U.ePose);
        U.obs = carve(16 * (size_t)nE); D.rawObs = (const double*)(d_arena + U.obs);
        U.isg = carve(4 * (size_t)nE); D.rawInvSigma2 = (const float*)(d_arena + U.isg);
        uploadOff[slot] = upBase; uploadBytes[slot] = off - upBase;
        // --- derived on the device ---
        D.ptOrig = (const int*)(d_arena + carve(4 * (size_t)nL));
        D.ePt = (const int*)(d_arena + carve(4 * (size_t)nE)); D.ePose = (const int*)(d_arena + carve(4 * (size_t)nE));
        D.eH = (const int*)(d_arena + carve(4 * (size_t)nE)); D.eOrig = (const int*)(d_arena + carve(4 * (size_t)nE));
        D.obs = (const double*)(d_arena + carve(16 * (size_t)nE)); D.invSigma2 = (const float*)(d_arena + carve(4 * (size_t)nE));
        D.ptStart = (const int*)(d_arena + carve(4 * (size_t)(nL + 1)));
        D.poseEdges = (const int*)(d_arena + carve(4 * (size_t)nE)); D.poseEdgePt = (const int*)(d_arena + carve(4 * (size_t)nE));
        D.pairs = (const int2*)(d_arena + carve(8 * pc)); D.pairPt = (const int*)(d_arena + carve(4 * pc));
        D.chunkHdr = (const int4*)(d_arena + carve(16 * cc)); D.taskChunkStart = (const int*)(d_arena + carve(4 * (size_t)(nTasks + 1)));
        D.bCnt = (int*)(d_arena + carve(4 * (size_t)(nL + 1))); D.bCursor = (int*)(d_arena + carve(4 * (size_t)(nL + 1)));
        D.bTmp = (int*)(d_arena + carve(4 * (size_t)nE)); D.bEid = (int*)(d_arena + carve(4 * (size_t)std::max(nF, 1) * (size_t)std::max(nL, 1)));
        D.bTaskLen = (int*)(d_arena + carve(4 * (size_t)std::max(nTasks, 1))); D.bItemStart = (int*)(d_arena + carve(4 * (size_t)std::max(nTasks, 1)));
        D.bKey = (unsigned long long*)(d_arena + carve(8 * pow2Of(nL)));
        // --- state / scratch of the LM kernel ---
        D.pts = (double*)(d_arena + carve(24 * (size_t)nL));
        D.posesB = (double*)(d_arena + carve(56 * (size_t)nP));
        D.ptsB = (double*)(d_arena + carve(24 * (size_t)nL));
        D.err = (double*)(d_arena + carve(16 * (size_t)nE));
        D.E4a = (double*)(d_arena + carve(32 * (size_t)nE)); D.E4b = (double*)(d_arena + carve(32 * (size_t)nE));
        D.K = (double2*)(d_arena + carve(32 * (size_t)nE));
        D.Hpp = (double*)(d_arena + carve(288 * (size_t)std::max(nF, 1))); D.bp = (double*)(d_arena + carve(48 * (size_t)std::max(nF, 1)));
        D.Hll = (double*)(d_arena + carve(48 * (size_t)nL)); D.bl = (double*)(d_arena + carve(24 * (size_t)nL));
        D.PT = (double2*)(d_arena + carve(72 * (size_t)nL));
        D.Spart = (double*)(d_arena + carve(8 * 42 * cc));
        D.Ppart = (double*)(d_arena + carve(8 * 28 * ((size_t)nP + (size_t)nE / SCH + 1)));
        D.Hs = (double*)(d_arena + carve(8 * (size_t)n * n)); D.bs = (double*)(d_arena + carve(8 * (size_t)std::max(n, 1)));
        D.x = (double*)(d_arena + carve(8 * ((size_t)n + 3 * (size_t)nL)));
        D.partial = (double*)(d_arena + carve(8 * (4 * PSLOT + 8)));
        D.job = (Job*)(d_arena + carve(sizeof(Job))); D.pcm = (double*)(d_arena + carve(8 * PC * (size_t)nP));
        if (cc + ((size_t)nL + PCH - 1) / PCH >= ((size_t)1 << 23)) { set_error("lba: more chunks in one phase than the claim word counts"); return ORB_ERR_CAPACITY; }
        if (off - base > perProblem) { set_error("lba: arena too small (internal sizing error)"); return ORB_ERR_CAPACITY; }
        return ORB_OK;
    }

    // Lays one problem out in slot `slot` of the arena and copies the caller's graph into the pinned mirror; the index
    // structures are derived on the device (lba_build_structure_kernel).
    int pack(int slot, const LbaProblem* P) {
        const int nP = P->nPoses, nL = P->nPoints, nE = P->nEdges;
        if (nP < 1 || nL < 0 || nE < 0 || nP > maxP || nL > maxL || nE > maxE || !P->poses || !P->poseFixed || !P->cam ||
            (nL && !P->points) || (nE && (!P->edgePoint || !P->edgePose || !P->obs || !P->invSigma2))) {
            set_error("lba: problem larger than the handle or null arrays"); return ORB_ERR_ARG;
        }
        std::vector<int> hidx(nP, -1), freePose;
        for (int i = 0; i < nP; ++i) if (!P->poseFixed[i]) { hidx[i] = (int)freePose.size(); freePose.push_back(i); }
        const int nF = (int)freePose.size();
        if (nF + nL == 0) { set_error("lba: 0 vertices to optimize"); return ORB_ERR_ARG; }
        UpBlock U;
        if (int rc = layout(slot, nP, nL, nE, nF, U)) return rc;
        auto put = [&](size_t o, const void* src, size_t bytes) { if (bytes) memcpy(h_arena + o, src, bytes); };
        put(U.poses, P->poses, 56 * (size_t)nP); put(U.pts, P->points, 24 * (size_t)nL); put(U.cam, P->cam, 16 * (size_t)nP);
        put(U.hidx, hidx.data(), 4 * (size_t)nP); put(U.freePose, freePose.data(), 4 * (size_t)nF);
        put(U.ePt, P->edgePoint, 4 * (size_t)nE); put(U.ePose, P->edgePose, 4 * (size_t)nE); put(U.obs, P->obs, 16 * (size_t)nE);
        put(U.isg, P->invSigma2, 4 * (size_t)nE);
        Dev& D = h_probs[slot];
        D.delta = P->huberDelta; D.dsqr = P->huberDelta * P->huberDelta; D.userLambdaInit = P->userLambdaInit; D.iterations = P->iterations;
        return ORB_OK;
    }
    std::vector<size_t> uploadBytes = std::vector<size_t>(1), uploadOff = std::vector<size_t>(1);

    int upload(int count, const LbaProblem* probs) {
        if (count < 1 || count > maxBatch) { set_error("lba: batch larger than max_batch"); return ORB_ERR_ARG; }
        // from here on the slots' layouts and arena contents change: until this upload succeeds there is nothing to run or download
        nLoaded = 0;
        uploadBytes.assign(maxBatch, 0); uploadOff.assign(maxBatch, 0);
        CK(cudaSetDevice(device));
        if (ranOnce) CK(cudaStreamWaitEvent(st, evRun, 0));   // a run may still be reading the arena on the caller's stream
        {   // stage the callers' graphs in the pinned mirror on a few host threads; every worker queues the host-to-device
            // copy of a problem as soon as it is staged, so the copies overlap the staging of the next problems
            const int nth = std::max(1, std::min<int>({count, (int)std::thread::hardware_concurrency(), 8}));
            std::atomic<int> next(0), firstErr(ORB_OK);
            auto worker = [&]() {
                cudaSetDevice(device);
                for (int i = next.fetch_add(1); i < count; i = next.fetch_add(1)) {
                    int rc = pack(i, probs + i);
                    if (!rc && cudaMemcpyAsync(d_arena + uploadOff[i], h_arena + uploadOff[i], uploadBytes[i], cudaMemcpyHostToDevice, st) != cudaSuccess) rc = ORB_ERR_CUDA;
                    if (rc) { int exp = ORB_OK; firstErr.compare_exchange_strong(exp, rc); }
                }
            };
            std::vector<std::thread> pool;
            for (int t = 1; t < nth; ++t) pool.emplace_back(worker);
            worker();
            for (auto& t : pool) t.join();
            if (firstErr.load()) {
                cudaStreamSynchronize(st);
                // the workers' own messages live in their thread-local error strings: restate it for the calling thread
                set_error(firstErr.load() == ORB_ERR_CUDA ? "lba: host-to-device copy failed"
                                                          : "lba: a problem is larger than the handle, has null arrays or no vertex to optimize");
                return firstErr.load();
            }
        }
        CK(cudaSetDevice(device));
        CK(cudaMemcpyAsync(d_probs, h_probs.data(), sizeof(Dev) * count, cudaMemcpyHostToDevice, st));
        for (int i = 0; i < count; ++i) h_status[i] = -1;
        lba_build_structure_kernel<<<count, BT, 0, st>>>(d_probs, d_status);     // BlockSolver::buildStructure, one CTA per problem
        CK(cudaGetLastError());
        CK(orbx::wait_stream_blocking(st, evWait));   // the resident copy must be complete before a run on any other stream
        if (int rc = check_structure(count)) return rc;
        nLoaded = count;
        return ORB_OK;
    }
    // the status words lba_build_structure_kernel left, once its stream has been synchronised
    int check_structure(int count) {
        for (int i = 0; i < count; ++i) {
            if (h_status[i] == 0) continue;
            nLoaded = 0;
            if (h_status[i] == 1) { set_error("lba: edge index out of range"); return ORB_ERR_ARG; }
            if (h_status[i] == 2) { set_error("lba: duplicate (point, keyframe) observation"); return ORB_ERR_ARG; }
            set_error("lba: pair / chunk list larger than sized"); return ORB_ERR_CAPACITY;
        }
        return ORB_OK;
    }
    // The device form of upload for graphs built on the device (csrc/local_ba.cu): lays every slot out from its sizes, copies the
    // graphs in with lba_fill_kernel and enqueues lba_build_structure_kernel on st.  Its status words are read by check_structure
    // once the caller has synchronised st.
    int load_device(int count, const int4* sizes, const double* userLambdaInit, const FillSrc* dFill) {
        nLoaded = 0;
        uploadBytes.assign(maxBatch, 0); uploadOff.assign(maxBatch, 0);
        CK(cudaSetDevice(device));
        if (ranOnce) CK(cudaStreamWaitEvent(st, evRun, 0));
        for (int i = 0; i < count; ++i) {
            UpBlock U;
            if (int rc = layout(i, sizes[i].x, sizes[i].y, sizes[i].z, sizes[i].w, U)) return rc;
            Dev& D = h_probs[i];
            D.delta = huber_mono(); D.dsqr = D.delta * D.delta; D.userLambdaInit = userLambdaInit[i]; D.iterations = 10;
        }
        CK(cudaMemcpyAsync(d_probs, h_probs.data(), sizeof(Dev) * count, cudaMemcpyHostToDevice, st));
        lba_fill_kernel<<<count, BT, 0, st>>>(d_probs, dFill);
        CK(cudaGetLastError());
        for (int i = 0; i < count; ++i) h_status[i] = -1;
        lba_build_structure_kernel<<<count, BT, 0, st>>>(d_probs, d_status);
        CK(cudaGetLastError());
        nLoaded = count;
        return ORB_OK;
    }
    // run on st, forwarding the callers' stop flags (SparseOptimizer::terminate() polls *pbStopFlag) while the kernel runs
    int run_forwarding(const volatile uint8_t* const* flags) {
        const int count = nLoaded;
        for (int i = 0; i < count; ++i) h_stop[i] = (flags[i] && *flags[i]) ? 1 : 0;
        if (int rc = run(st)) return rc;
        bool anyFlag = false;
        for (int i = 0; i < count; ++i) anyFlag = anyFlag || flags[i];
        if (anyFlag) {
            CK(cudaEventRecord(evDone, st));
            while (cudaEventQuery(evDone) == cudaErrorNotReady) {
                for (int i = 0; i < count; ++i)
                    if (flags[i] && *flags[i]) h_stop[i] = 1;
                std::this_thread::yield();
            }
        }
        CK(cudaGetLastError());
        return ORB_OK;
    }
    // (re)start from the uploaded initial estimates and run the whole LM loop for every loaded problem
    int run(cudaStream_t s) {
        if (nLoaded < 1) { set_error("lba: nothing uploaded"); return ORB_ERR_ARG; }
        CK(cudaSetDevice(device));
        int maxN = 0, mp = 1, mf = 1;
        for (int i = 0; i < nLoaded; ++i) {                             // the kernel itself restarts from the uploaded estimates
            maxN = std::max(maxN, 6 * packed[i].nF); mp = std::max(mp, packed[i].nP); mf = std::max(mf, packed[i].nF);
        }
        // dynamic shared memory: the pose caches hold every pose of the window (fixed keyframes included, the reference puts no
        // bound on lFixedCameras), the LDLT panels and rhs only the free ones; the reduced camera system joins them when it fits
        const size_t fixedSmem = 8 * ((size_t)2 * PC * mp + (size_t)78 * mf + 16);
        const size_t maxDyn = 200 * 1024;                               // of the 227 KB opt-in limit; the kernel has ~5 KB static
        if (fixedSmem > maxDyn) {
            set_error("lba: window too large for the shared-memory pose caches (about 600 keyframes incl. fixed ones)");
            return ORB_ERR_CAPACITY;
        }
        const int smemN = (int)floor(sqrt((double)(maxDyn - fixedSmem) / 8.0));
        const int matN = maxN <= smemN ? maxN : 0;   // matrix in shared memory only when every problem of the batch fits
        const size_t dyn = fixedSmem + 8 * (size_t)matN * matN;
        if (orbx::ensure_dynamic_smem(lba_cluster_kernel, dyn, device)) return ORB_ERR_CUDA;
        cudaLaunchConfig_t cfg; memset(&cfg, 0, sizeof(cfg));
        cfg.blockDim = dim3(NT);
        cfg.dynamicSmemBytes = dyn;
        cfg.stream = s;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        // cluster size: the largest (any size up to 8, not only powers of two) for which every problem's cluster is resident at
        // once -- asked from the occupancy calculator, because clusters cannot straddle GPCs (SM count / size is only an upper bound)
        int csize = 1;
        for (int cand = MAXC; cand >= 1; --cand) {
            if ((long)nLoaded * cand > numSMs) continue;
            attr[0].val.clusterDim.x = cand;
            cfg.gridDim = dim3(nLoaded * cand);
            int nClusters = 0;
            if (cudaOccupancyMaxActiveClusters(&nClusters, lba_cluster_kernel, &cfg) == cudaSuccess && nClusters >= nLoaded) { csize = cand; break; }
        }
        (void)cudaGetLastError();
        if (forcedCluster > 0) csize = forcedCluster;
        attr[0].val.clusterDim.x = csize;
        // helper clusters: as many more clusters of this size as are resident beside the batch's own
        int nHelp = 0;
        if (helpers != 0) {
            cfg.gridDim = dim3(csize);
            int maxActive = 0;
            if (cudaOccupancyMaxActiveClusters(&maxActive, lba_cluster_kernel, &cfg) == cudaSuccess) nHelp = std::max(0, maxActive - nLoaded);
            (void)cudaGetLastError();
            if (helpers > 0) nHelp = std::min(nHelp, helpers);
        }
        cfg.gridDim = dim3((nLoaded + nHelp) * csize);
        CK(cudaMemsetAsync(d_finished, 0, sizeof(unsigned long long), s));
        const Dev* dp = d_probs; const volatile int* ds = d_stop; int mn = matN, np = nLoaded; unsigned long long* fin = d_finished;
        CK(cudaLaunchKernelEx(&cfg, lba_cluster_kernel, dp, ds, mn, mp, mf, np, fin));
        CK(cudaEventRecord(evRun, s));
        ranOnce = true;
        launches = 1;
        lastCluster = csize; lastHelpers = nHelp;
        return ORB_OK;
    }
    int lastCluster = 1, forcedCluster = 0;
    int helpers = -1, lastHelpers = 0;
    int download(int count, LbaResult* res, cudaStream_t s) {
        for (int i = 0; i < count; ++i)
            if (!res[i].poses || !res[i].points || !res[i].edgeChi2 || !res[i].edgeDepthPositive) { set_error("lba: null result arrays"); return ORB_ERR_ARG; }
        // the output blocks sit at the start of every slot with one layout: a single strided copy into the pinned mirror
        const size_t ob = outBlock(maxP, maxL, maxE);
        if (ranOnce) CK(cudaStreamWaitEvent(s, evRun, 0));    // the run may be on another stream than this copy
        CK(cudaMemcpy2DAsync(h_arena, perProblem, d_arena, perProblem, ob, (size_t)count, cudaMemcpyDeviceToHost, s));
        CK(orbx::wait_stream_blocking(s, evWait));
        for (int i = 0; i < count; ++i) {
            const Packed& K = packed[i];
            LbaResult& R = res[i];
            memcpy(R.poses, h_arena + K.posesOff, 56 * (size_t)K.nP);
            if (K.nL) memcpy(R.points, h_arena + K.ptsOff, 24 * (size_t)K.nL);
            if (K.nE) { memcpy(R.edgeChi2, h_arena + K.chi2Off, 8 * (size_t)K.nE); memcpy(R.edgeDepthPositive, h_arena + K.dposOff, (size_t)K.nE); }
            const double* stt = (const double*)(h_arena + K.statsOff);
            R.iterations = (int)stt[0]; R.trials = (int)stt[1]; R.lambda = stt[2]; R.chi2 = stt[3]; R.initialChi2 = stt[4];
            R.gpuLaunches = 1;
        }
        return ORB_OK;
    }
};

}  // namespace lba

using namespace lba;

struct lba_handle { Solver s; };

extern "C" {

int lba_create_batch(lba_handle** out, int max_poses, int max_points, int max_edges, int max_batch, int device) {
    if (!out || max_poses < 1 || max_points < 1 || max_edges < 1 || max_batch < 1) { set_error("lba_create: bad argument"); return ORB_ERR_ARG; }
    if (int rc = orbx::check_device(device)) return rc;
    lba_handle* h = new lba_handle();
    h->s.device = device; h->s.maxP = max_poses; h->s.maxL = max_points; h->s.maxE = max_edges; h->s.maxBatch = max_batch;
    int rc = h->s.init();
    if (rc) { delete h; return rc; }
    *out = h;
    return ORB_OK;
}
int lba_create(lba_handle** out, int max_poses, int max_points, int max_edges, int device) {
    return lba_create_batch(out, max_poses, max_points, max_edges, 1, device);
}
void lba_destroy(lba_handle* h) { delete h; }

int lba_upload_batch(lba_handle* h, int count, const LbaProblem* problems) {
    if (!h || !problems) { set_error("lba_upload_batch: bad argument"); return ORB_ERR_ARG; }
    return h->s.upload(count, problems);
}
int lba_run_batch_device(lba_handle* h, void* stream) {
    if (!h) { set_error("lba_run_batch_device: bad argument"); return ORB_ERR_ARG; }
    for (int i = 0; i < h->s.nLoaded; ++i) h->s.h_stop[i] = 0;
    return h->s.run((cudaStream_t)stream);
}
int lba_download_batch(lba_handle* h, int count, LbaResult* results) {
    if (!h || !results || count < 1 || count > h->s.nLoaded) { set_error("lba_download_batch: bad argument"); return ORB_ERR_ARG; }
    return h->s.download(count, results, h->s.st);
}
int lba_last_cluster_size(const lba_handle* h) { return h ? h->s.lastCluster : ORB_ERR_ARG; }
int lba_set_cluster_size(lba_handle* h, int ctas) {
    if (!h || ctas < 0 || ctas > MAXC) { set_error("lba_set_cluster_size: 0 (auto) or 1..8"); return ORB_ERR_ARG; }
    h->s.forcedCluster = ctas;
    return ORB_OK;
}
int lba_last_helpers(const lba_handle* h) { return h ? h->s.lastHelpers : ORB_ERR_ARG; }
int lba_set_helpers(lba_handle* h, int clusters) {
    if (!h || clusters < -1) { set_error("lba_set_helpers: -1 (fill the GPU), 0 (none) or a maximum"); return ORB_ERR_ARG; }
    h->s.helpers = clusters;
    return ORB_OK;
}
/* ns spent by CTA 0 of problem `i` in each phase of the last downloaded run (include/orb_b200.h), then the chunks helpers served */
int lba_get_phase_ns(const lba_handle* h, int i, double* ns10) {
    if (!h || !ns10 || i < 0 || i >= h->s.nLoaded) return ORB_ERR_ARG;
    const double* stt = (const double*)(h->s.h_arena + h->s.packed[i].statsOff);
    for (int k = 0; k < 10; ++k) ns10[k] = stt[8 + k];
    return ORB_OK;
}

int lba_solve_batch(lba_handle* h, int count, const LbaProblem* problems, LbaResult* results) {
    if (!h || !problems || !results) { set_error("lba_solve_batch: bad argument"); return ORB_ERR_ARG; }
    Solver& S = h->s;
    int rc = S.upload(count, problems);
    if (rc) return rc;
    std::vector<const volatile uint8_t*> flags(count);
    for (int i = 0; i < count; ++i) flags[i] = problems[i].stopFlag;
    if ((rc = S.run_forwarding(flags.data()))) return rc;
    return S.download(count, results, S.st);
}
int lba_solve(lba_handle* h, const LbaProblem* problem, LbaResult* result) { return lba_solve_batch(h, 1, problem, result); }
int lba_local_last_launches(const lba_handle* h) { return h ? h->s.localLaunches : ORB_ERR_ARG; }

}  // extern "C"

namespace lba {
cudaStream_t solver_stream(lba_handle* h) { return h->s.st; }
orbx::Staging& solver_staging(lba_handle* h) { return h->s.stage; }
void solver_limits(const lba_handle* h, int* maxP, int* maxL, int* maxE, int* maxBatch) {
    *maxP = h->s.maxP; *maxL = h->s.maxL; *maxE = h->s.maxE; *maxBatch = h->s.maxBatch;
}
int solver_load_device(lba_handle* h, int count, const int4* sizes, const double* userLambdaInit, const FillSrc* dFill, SlotOut* out) {
    Solver& S = h->s;
    if (int rc = S.load_device(count, sizes, userLambdaInit, dFill)) return rc;
    for (int i = 0; i < count; ++i) {
        const Dev& D = S.h_probs[i];
        out[i] = SlotOut{D.poses, D.outPts, D.outChi2, D.outDepthPos, D.stats};
    }
    return ORB_OK;
}
int solver_run(lba_handle* h, const volatile uint8_t* const* flags) { return h->s.run_forwarding(flags); }
int solver_check_structure(lba_handle* h, int count) {
    Solver& S = h->s;
    CK(orbx::wait_stream_blocking(S.st, S.evWait));
    return S.check_structure(count);
}
void solver_set_local_launches(lba_handle* h, int n) { h->s.localLaunches = n; }
}  // namespace lba
