// Small device-side helpers shared by the kernels of this library, and the host-side error plumbing of its entry points.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <mutex>
#include <string>
#include <utility>

#include "../../include/orb_b200.h"

namespace orbx {

void set_error(const std::string& s);

#define CK(call)                                                                   \
    do {                                                                           \
        cudaError_t e_ = (call);                                                   \
        if (e_ != cudaSuccess) {                                                   \
            orbx::set_error(std::string(#call) + ": " + cudaGetErrorString(e_));   \
            return ORB_ERR_CUDA;                                                   \
        }                                                                          \
    } while (0)

// The device check of every entry point that takes a device index: ORB_ERR_CUDA without a device, ORB_ERR_ARG for an index out of range.
inline int check_device(int device) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { set_error("no CUDA device (this library has no CPU path)"); return ORB_ERR_CUDA; }
    if (device < 0 || device >= n) { set_error("bad device index " + std::to_string(device) + " (" + std::to_string(n) + " CUDA devices)"); return ORB_ERR_ARG; }
    return ORB_OK;
}

// The library is compiled for sm_90a alone (__graft_entry__.py): its cubins load on compute capability 9.0 and on no other device.
inline int require_sm90(int major, int minor) {
    if (major == 9 && minor == 0) return 0;
    set_error("device is not sm_90 (Hopper); this library is built for sm_90a only and has no other code path");
    return ORB_ERR_CUDA;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a property of the (function, device) pair, not of a handle: several handles of
// different sizes share it.  Keep a process-wide monotonic maximum per kernel and device and only ever raise it, so that a
// smaller handle created later can never lower the limit under a larger one (the launch would fail with invalid-value).  Without the
// opt-in, static + dynamic shared memory must stay within 48 KB: the kernel's static shared memory counts towards that bound.
template <class Kernel>
inline int ensure_dynamic_smem(Kernel* kernel, size_t bytes, int device) {
    static std::mutex mu;
    static std::map<std::pair<const void*, int>, size_t> current;
    std::lock_guard<std::mutex> lock(mu);
    size_t& cur = current[std::make_pair((const void*)kernel, device)];
    if (bytes <= cur) return 0;
    cudaFuncAttributes fa;
    if (cudaFuncGetAttributes(&fa, kernel) != cudaSuccess) { set_error("cudaFuncGetAttributes failed"); return ORB_ERR_CUDA; }
    if (bytes + fa.sharedSizeBytes <= 48 * 1024) return 0;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) { set_error(std::string("cudaFuncSetAttribute(MaxDynamicSharedMemorySize): ") + cudaGetErrorString(e)); return ORB_ERR_CUDA; }
    cur = bytes;
    return 0;
}

// Exclusive scan of one int per thread over a CTA of NT threads; `total` gets the CTA's sum.  `sm` needs 33 ints and is free again
// on return.  All threads of the block must call.
template <int NT> __device__ __forceinline__ int block_scan_excl(int v, int* sm, int& total) {
    static_assert(NT % 32 == 0 && NT <= 1024, "NT must be whole warps, at most 1024 threads");
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) sm[w] = inc;
    __syncthreads();
    if (w == 0) {
        const int x = lane < NT / 32 ? sm[lane] : 0;
        int y = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, y, o); if (lane >= o) y += t; }
        sm[lane] = y - x;
        if (lane == 31) sm[32] = y;
    }
    __syncthreads();
    const int r = sm[w] + inc - v;
    total = sm[32];
    __syncthreads();
    return r;
}

// Exclusive prefix of count(i) over i in [0, n), n >= 0, into out[0, n); returns the total and does not write out[n].  count(i) may read out[i]
// (an in-place scan): each thread reads its element before the tile's barriers and writes it after.  `sm` needs 33 ints.  All threads
// of the block must call; on return `out` is visible to all of them.
template <int NT, class Count> __device__ __forceinline__ int block_prefix(int n, int* out, int* sm, Count count) {
    int carry = 0;
    // An unsigned tile base: with a signed one the compiler unrolls this loop
    for (unsigned b = 0; b < (unsigned)n; b += NT) {
        const int i = (int)(b + threadIdx.x);
        int tot;
        const int r = block_scan_excl<NT>(i < n ? count(i) : 0, sm, tot);
        if (i < n) out[i] = carry + r;
        carry += tot;
    }
    __syncthreads();
    return carry;
}
// Ordered sum of one double per thread over a CTA of NT threads: an xor butterfly in each warp, then the warp sums in warp order, so the
// result is run-to-run reproducible and every thread gets the same value.  `sm` needs NT / 32 doubles.  All threads of the block must call.
template <int NT> __device__ __forceinline__ double block_sum(double v, double* sm) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    double r = 0;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) r += sm[w];
    __syncthreads();
    return r;
}

// 256-bit Hamming distance of two 32-byte descriptors held as 8 words (ORBmatcher::DescriptorDistance,
// reference src/ORBmatcher.cc:2058-2074; the SWAR popcount there == __popc).
__device__ __forceinline__ int hamming256(const uint32_t* a, const uint32_t* b) {
    int d = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) d += __popc(a[i] ^ b[i]);
    return d;
}

// One 32-byte descriptor (16-byte aligned, not written by the kernel) as 8 words, through the read-only cache.
__device__ __forceinline__ void load_desc(const uint8_t* p, uint32_t (&d)[8]) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    const uint4 a = __ldg(q), b = __ldg(q + 1);
    d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w; d[4] = b.x; d[5] = b.y; d[6] = b.z; d[7] = b.w;
}

// std::lower_bound / std::upper_bound of key in the ascending a[lo, hi): the first index whose element is >= key / > key, or hi.
__device__ __forceinline__ int lower_bound(const int* a, int lo, int hi, int key) {
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < key) lo = mid + 1; else hi = mid; }
    return lo;
}
__device__ __forceinline__ int upper_bound(const int* a, int lo, int hi, int key) {
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] <= key) lo = mid + 1; else hi = mid; }
    return lo;
}

// MapPoint::ComputeDistinctiveDescriptors' choice (src/MapPoint.cc:329-403) among n <= 65535 rows, for one warp: lane l takes rows
// l, l + 32, ...; row(j) gives the address of row j (32 bytes, 16-byte aligned, not written by the kernel).  Every lane returns the first
// row with the least median distance to the others; the median (element (int)(0.5 (n - 1)) of the sorted row) is found by bisection on the
// distance value.  Used by distinctive_kernel and update_connections_kernel.
template <class Row>
__device__ __forceinline__ int distinctive_best(int n, int lane, Row row) {
    const int k = (int)(0.5 * (double)(n - 1));
    unsigned bestKey = 0xFFFFFFFFu;
    for (int i = lane; i < n; i += 32) {
        uint32_t di[8];
        load_desc(row(i), di);
        int lo = 0, hi = 256;                                    // smallest v with #{j : d(i, j) <= v} >= k + 1
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            int cnt = 0;
            for (int j = 0; j < n; ++j) {
                uint32_t dj[8];
                load_desc(row(j), dj);
                cnt += (i == j ? 0 : hamming256(di, dj)) <= mid;
            }
            if (cnt >= k + 1) hi = mid; else lo = mid + 1;
        }
        bestKey = min(bestKey, ((unsigned)lo << 16) | (unsigned)i);
    }
    return (int)(__reduce_min_sync(0xffffffffu, bestKey) & 0xFFFFu);
}

// Wait for a stream from a host thread that has nothing else to do: through an event created with cudaEventBlockingSync the thread sleeps
// instead of spinning in cudaStreamSynchronize (a server runs several such threads per GPU and several GPUs per host; spinning threads
// take the cores the other ranks' threads need).  Used by the BATCH host entry points; single-frame calls keep the low-latency spin.
inline cudaError_t wait_stream_blocking(cudaStream_t st, cudaEvent_t ev) {
    cudaError_t e = cudaEventRecord(ev, st);
    return e != cudaSuccess ? e : cudaEventSynchronize(ev);
}
inline cudaError_t make_blocking_event(cudaEvent_t* ev) { return cudaEventCreateWithFlags(ev, cudaEventBlockingSync | cudaEventDisableTiming); }
}  // namespace orbx
