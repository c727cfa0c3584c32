// Optimizer::LocalInertialBA (reference src/Optimizer.cc:2383-2958; SURVEY.md 8f rank 1) on the H100: local_inertial_ba_batch.
// One persistent CTA (NT = 512 threads) per local map runs the whole g2o Levenberg-Marquardt loop of liba_core.cuh on the device; a batch
// of maps (one per stream of a multi-stream server) fills the SMs.  The host side flattens the graph (liba_pack.h: layout, CSR lists),
// uploads one packed input buffer, launches ONE kernel and downloads one packed output buffer.
//
// Why one CTA per map: the temporal window is 10 (25 with bLarge) keyframes x 15 unknowns, so the reduced system is a dense 150 (375)
// square; per LM trial the work is ~10^4 EdgeMono evaluations, a Schur complement of ~10^5 6x3 * 3x6 products and a 150^3 / 3 flop
// factorisation -- a dependent chain of small phases whose cost is barrier latency, not throughput.  A CTA barrier is ~20x cheaper than
// a cluster or grid barrier, and the parallel dimension that fills the GPU is the batch of independent maps (the reference runs one
// LocalMapping thread per map).  The working set of a map (~2-8 MB) lives in L2.
#include <cuda_runtime.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "liba_pack.h"
#include "staging.h"

using orbx::set_error;

namespace liba {

// The executor of liba_core.cuh on the device: thread = threadIdx.x, barrier = __syncthreads, ordered CTA reductions.
struct DeviceExec {
    double* red;      // NT / 32 doubles of shared memory
    double* prof;     // 8 doubles of shared memory: nanoseconds per phase group (thread 0 keeps the clock)
    double* pnl;      // MAXN * LW doubles of shared memory: the LDL^T panel
    unsigned long long last; int cur;
    __device__ __forceinline__ double* panel() const { return pnl; }
    __device__ __forceinline__ void tag(int k) {
        if (threadIdx.x == 0) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            prof[cur] += (double)(t - last);
            last = t; cur = k;
        }
    }
    template <class F> __device__ __forceinline__ void par(F f) { f((int)threadIdx.x); __syncthreads(); }
    template <class F> __device__ __forceinline__ double sum(F f) {
        double v = f((int)threadIdx.x);
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
        __syncthreads();
        double total = 0;
#pragma unroll
        for (int w = 0; w < NT / 32; ++w) total += red[w];      // every thread adds the warp sums in the same order
        __syncthreads();
        return total;
    }
    template <class F> __device__ __forceinline__ double max(F f) {
        double v = f((int)threadIdx.x);
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, off));
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
        __syncthreads();
        double m = 0;
#pragma unroll
        for (int w = 0; w < NT / 32; ++w) m = fmax(m, red[w]);
        __syncthreads();
        return m;
    }
};

__global__ void __launch_bounds__(NT) local_inertial_ba_kernel(const Dev* __restrict__ probs) {
    __shared__ double s_red[NT / 32];
    __shared__ Dev s_D;
    if (threadIdx.x == 0) s_D = probs[blockIdx.x];
    __syncthreads();
    __shared__ double s_prof[8];
    __shared__ double s_panel[MAXN * LW];      // 37.5 KB
    if (threadIdx.x < 8) s_prof[threadIdx.x] = 0.0;
    __syncthreads();
    unsigned long long t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    DeviceExec ex{s_red, s_prof, s_panel, t0, 7};
    run(s_D, ex);
    ex.tag(7);
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    if (threadIdx.x == 0) {
        s_D.stats[6] = (double)(t1 - t0);      // nanoseconds this map's CTA spent in the solver
        for (int k = 0; k < 8; ++k) s_D.prof[k] = s_prof[k];
    }
}

// One CTA per problem of the device table probs [count]; local_inertial_ba_map.cu launches it on problems its walk kernel built.
cudaError_t launch_solver(const Dev* probs, int count, cudaStream_t st) {
    local_inertial_ba_kernel<<<count, NT, 0, st>>>(probs);
    return cudaGetLastError();
}

}  // namespace liba

extern "C" int local_inertial_ba_batch(int count, const LocalInertialBAProblem* problems, const LocalInertialBAResult* results, int32_t* iterationsOut, int device) {
    using namespace liba;
    if (count < 1 || !problems || !results) { set_error("local_inertial_ba_batch: bad argument"); return ORB_ERR_ARG; }
    if (int rc = orbx::check_device(device)) return rc;
    CK(cudaSetDevice(device));
    {   // the architecture check is made once per device (cudaGetDeviceProperties costs milliseconds)
        static int s_major[64], s_minor[64];
        static std::mutex s_mu;
        std::lock_guard<std::mutex> lk(s_mu);
        if (device < 64 && s_major[device] == 0) {
            CK(cudaDeviceGetAttribute(&s_major[device], cudaDevAttrComputeCapabilityMajor, device));
            CK(cudaDeviceGetAttribute(&s_minor[device], cudaDevAttrComputeCapabilityMinor, device));
        }
        if (device < 64 && orbx::require_sm90(s_major[device], s_minor[device])) return ORB_ERR_CUDA;
    }
    const bool trace = getenv("ORB_LIBA_TRACE") != nullptr;
    const auto tStart = std::chrono::steady_clock::now();
    auto ms_since = [&](std::chrono::steady_clock::time_point t0) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); };

    std::vector<Layout> lay(count);
    std::vector<size_t> inOff(count), scOff(count), outOff(count);
    size_t inTot = 0, scTot = 0, outTot = 0;
    for (int i = 0; i < count; ++i) {
        const std::string err = check(problems[i]);
        if (!err.empty()) { set_error(err); return ORB_ERR_ARG; }
        lay[i] = make_layout(problems[i]);
        inOff[i] = inTot; scOff[i] = scTot; outOff[i] = outTot;
        inTot += (lay[i].inBytes + 255) & ~(size_t)255; scTot += (lay[i].scBytes + 255) & ~(size_t)255; outTot += (lay[i].outBytes + 255) & ~(size_t)255;
    }
    orbx::ThreadStaging* S;
    int rc = orbx::thread_staging(device, &S);
    if (rc) return rc;
    S->begin();
    const int pIn = S->in(nullptr, inTot), pDev = S->in(nullptr, (size_t)count * sizeof(Dev)), pOut = S->out(nullptr, outTot), pSc = S->scratch(scTot);
    if ((rc = S->reserve())) return rc;
    uint8_t* hIn = S->host(pIn); uint8_t* hOut = S->host(pOut);
    Dev* hDev = S->host<Dev>(pDev);
    {
        const std::string err = pack_batch(count, problems, lay.data(), inOff.data(), hIn);
        if (!err.empty()) { set_error(err); return ORB_ERR_ARG; }
    }
    for (int i = 0; i < count; ++i) bind(hDev[i], problems[i], lay[i], S->dev(pIn) + inOff[i], S->dev(pSc) + scOff[i], S->dev(pOut) + outOff[i]);      // device addresses
    const double msPack = ms_since(tStart);
    const auto tGpu = std::chrono::steady_clock::now();
    CK(S->upload(S->stream));
    CK(launch_solver(S->dev<const Dev>(pDev), count, S->stream));
    CK(S->download(S->stream));
    const double msGpu = ms_since(tGpu);
    for (int i = 0; i < count; ++i) {
        const int it = unpack_outputs(problems[i], results[i], lay[i], hOut + outOff[i]);
        if (iterationsOut) iterationsOut[i] = it;
    }
    if (trace) fprintf(stderr, "local_inertial_ba_batch: %d maps, check + layout + pack %.3f ms (%zu bytes in), copy in + kernel + copy out %.3f ms (%zu bytes out), total %.3f ms\n",
                       count, msPack, inTot + (size_t)count * sizeof(Dev), msGpu, outTot, ms_since(tStart));
    return ORB_OK;
}
