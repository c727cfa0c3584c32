// Microbenchmarks that size the LBA kernel: (1) DFMA issue rate per SM, (2) cost of per-lane gathers of 32-byte records
// (32 distinct 128-byte lines per warp instruction) from an L2-resident array, loaded as lba.cu loads them (2 x LDG.128), next to
// 16-byte records (1 x LDG.128: half the bytes and half the look-ups), (3) cost of one 8-byte field per lane (LDG.64) when a warp
// instruction touches 32, 4 or 2 lines (random gather, half-density and dense structure-of-arrays reads).  Times are SM cycles from clock64(), so they do not depend on
// the clock the card runs at.
#include <cstdio>
#include <cuda_runtime.h>
__global__ void dfma(double* o, long long* cyc, int iters, double a, double b) {
    double x[8];
    for (int i = 0; i < 8; ++i) x[i] = threadIdx.x + i;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it)
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] = fma(x[i], a, b);
    __syncthreads();
    if (threadIdx.x == 0) cyc[blockIdx.x] = clock64() - t0;
    double s = 0; for (int i = 0; i < 8; ++i) s += x[i];
    o[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int MODE>   // 0: 32-byte records as 2 x LDG.128, 1: 16-byte records as 1 x LDG.128
__global__ void gather(const double* __restrict__ E, const int* __restrict__ idx, double* o, long long* cyc, int nPerThread, int stride) {
    double s = 0;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    __syncthreads();
    const long long t0 = clock64();
    for (int k = 0; k < nPerThread; k += 4) {
        int e[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) e[u] = idx[(size_t)(k + u) * stride + t];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const double* p = E + (MODE == 0 ? 4 : 2) * (size_t)e[u];
            double a, b;   // the loads of lba.cu: ld.global.v2.f64 (LDG.E.128)
            asm volatile("ld.global.v2.f64 {%0, %1}, [%2];" : "=d"(a), "=d"(b) : "l"(p));
            s += a + b;
            if (MODE == 0) { asm volatile("ld.global.v2.f64 {%0, %1}, [%2];" : "=d"(a), "=d"(b) : "l"(p + 2)); s += a + b; }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) cyc[blockIdx.x] = clock64() - t0;
    o[t] = s;
}
// one 8-byte field per lane (LDG.64), the load of a structure-of-arrays operand; how many lines an instruction touches is set by
// the index pattern the host writes
__global__ void gather8(const double* __restrict__ A, const int* __restrict__ idx, double* o, long long* cyc, int nPerThread, int stride) {
    double s = 0;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    __syncthreads();
    const long long t0 = clock64();
    for (int k = 0; k < nPerThread; k += 4) {
        int e[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) e[u] = idx[(size_t)(k + u) * stride + t];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            double a;
            asm volatile("ld.global.f64 %0, [%1];" : "=d"(a) : "l"(A + e[u]));
            s += a;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) cyc[blockIdx.x] = clock64() - t0;
    o[t] = s;
}
static double mean_cycles(const long long* d, int n) {
    long long h[1024]; cudaMemcpy(h, d, 8 * n, cudaMemcpyDeviceToHost);
    double s = 0; for (int i = 0; i < n; ++i) s += (double)h[i];
    return s / n;
}
int main() {
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    const int nsm = prop.multiProcessorCount;
    printf("%s, %d SMs\n", prop.name, nsm);
    double* o; cudaMalloc(&o, 8 * (size_t)nsm * 1024);
    long long* cyc; cudaMalloc(&cyc, 8 * 1024);
    for (int nt : {128, 256, 512, 1024}) {
        const int iters = 20000;
        dfma<<<nsm, nt>>>(o, cyc, iters, 1.0000001, 1e-9); dfma<<<nsm, nt>>>(o, cyc, iters, 1.0000001, 1e-9); cudaDeviceSynchronize();
        printf("dfma threads/SM %4d: %.1f DFMA/clk/SM\n", nt, (double)nt * iters * 8 / mean_cycles(cyc, nsm));
    }
    const int nRec = 1 << 16;   // 2 MB of 32-byte records: L2 resident, larger than L1
    double* E; cudaMalloc(&E, 32 * nRec); cudaMemset(E, 0, 32 * nRec);
    const int nt = 512, per = 256, total = nsm * nt;
    int* h = new int[(size_t)per * total]; unsigned r = 12345;
    for (size_t i = 0; i < (size_t)per * total; ++i) { r = r * 1664525u + 1013904223u; h[i] = (r >> 8) % nRec; }
    int* idx; cudaMalloc(&idx, 4 * (size_t)per * total); cudaMemcpy(idx, h, 4 * (size_t)per * total, cudaMemcpyHostToDevice);
    for (int mode = 0; mode < 2; ++mode) for (int blocks : {8, nsm}) {
        auto run = [&]() { if (mode == 0) gather<0><<<blocks, nt>>>(E, idx, o, cyc, per, total); else gather<1><<<blocks, nt>>>(E, idx, o, cyc, per, total); };
        run(); run(); cudaDeviceSynchronize();
        const double clk = mean_cycles(cyc, blocks);
        printf("gather %s, %3d SMs x 512 thr: %.1f clk per warp-record-gather per SM\n", mode ? "16 B records, 1 x LDG.128" : "32 B records, 2 x LDG.128",
               blocks, clk / ((nt / 32) * (double)per));
    }
    // 8-byte fields of the same 2 MB as a double array: every warp instruction reads 32 random lines (each lane its own), the 2 lines
    // of 32 consecutive doubles (dense SoA: lane i reads base + i), or the 4 lines of every other double (half density: base + 2 i)
    const int nDbl = 4 * nRec;
    const char* pat[3] = {"random, 32 lines", "dense SoA, 2 lines", "half density, 4 lines"};
    for (int mode = 0; mode < 3; ++mode) {
        for (size_t k = 0; k < (size_t)per; ++k)
            for (int w = 0; w < total / 32; ++w) {
                r = r * 1664525u + 1013904223u;
                const int base = (int)((r >> 8) % (unsigned)(nDbl / 64)) * 64;   // 512-byte aligned
                for (int l = 0; l < 32; ++l) {
                    int v = base + (mode == 2 ? 2 * l : l);
                    if (mode == 0) { r = r * 1664525u + 1013904223u; v = (int)((r >> 8) % (unsigned)nDbl); }
                    h[k * total + 32 * w + l] = v;
                }
            }
        cudaMemcpy(idx, h, 4 * (size_t)per * total, cudaMemcpyHostToDevice);
        for (int blocks : {8, nsm}) {
            gather8<<<blocks, nt>>>(E, idx, o, cyc, per, total); gather8<<<blocks, nt>>>(E, idx, o, cyc, per, total); cudaDeviceSynchronize();
            const double clk = mean_cycles(cyc, blocks);
            printf("gather 8 B field, 1 x LDG.64, %-22s %3d SMs x 512 thr: %.1f clk per warp-instruction per SM\n", pat[mode], blocks,
                   clk / ((nt / 32) * (double)per));
        }
    }
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
