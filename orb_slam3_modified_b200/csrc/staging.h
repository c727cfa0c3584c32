// Host-side staging of the host-pointer entry points: one device buffer and its pinned host mirror, grown to the high-water mark
// of the calls.  A matcher or vocabulary handle owns one; the stateless batch entry points share one per host thread
// (thread_staging).  A call declares its pieces, reserves, and runs its launches between ONE upload and ONE download:
//
//     S.begin();
//     const int a = S.in(src, bytes), b = S.inout(ptr, bytes), c = S.out(dst, bytes), t = S.scratch(bytes);
//     if ((rc = S.reserve())) return rc;        // layout + growth; pieces without a source are filled through S.host<T>()
//     CK(S.upload(st));                         // every source packed into the mirror, one copy of in + inout
//     kernel<<<..., st>>>(S.dev<T>(a), ...);
//     CK(S.download(st));                       // one copy of inout + out, stream synchronise, every piece to its destination
//
// Pieces are numbered in the order they are declared, from 0 after begin().  They are 256-byte aligned and laid out
// in | inout | out | scratch whatever that order, so each direction is one contiguous copy.  An inout / out piece without a
// destination is read by the caller through S.host<T>() after download.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "host_affinity.h"

namespace orbx {

class Staging {
public:
    int device = -1;     // set by the owner: the device buffer lives there and the pinned pages on its NUMA node

    Staging() = default;
    Staging(const Staging&) = delete;
    Staging& operator=(const Staging&) = delete;
    ~Staging() { release(); }

    void begin() { pieces_.clear(); }
    int in(const void* src, size_t bytes) { return add(IN, bytes, src, nullptr); }
    int inout(void* p, size_t bytes) { return add(INOUT, bytes, p, p); }
    int out(void* dst, size_t bytes) { return add(OUT, bytes, nullptr, dst); }
    int scratch(size_t bytes) { return add(SCRATCH, bytes, nullptr, nullptr); }

    // Lays the declared pieces out and grows the buffers to hold them.  Every user ends its call in a stream synchronise, so the
    // buffers are idle when they are replaced here.
    int reserve() {
        size_t off = 0;
        for (int k = IN; k <= SCRATCH; ++k) {
            if (k == INOUT) downBegin_ = off;
            if (k == OUT) upEnd_ = off;
            if (k == SCRATCH) downEnd_ = off;
            for (Piece& p : pieces_)
                if (p.kind == k) { p.off = off; off += (p.bytes + 255) & ~(size_t)255; }
        }
        if (off > dcap_) {
            const size_t cap = std::max(off, dcap_ + dcap_ / 2);
            if (d_) cudaFree(d_);
            d_ = nullptr; dcap_ = 0;
            CK(cudaMalloc(&d_, cap));
            dcap_ = cap;
        }
        if (downEnd_ > hcap_) {
            const size_t cap = std::max(downEnd_, hcap_ + hcap_ / 2);
            if (h_) cudaFreeHost(h_);
            h_ = nullptr; hcap_ = 0;
            ScopedGpuAffinity numaLocal(device);
            CK(cudaMallocHost(&h_, cap));
            hcap_ = cap;
        }
        return ORB_OK;
    }

    template <class T = uint8_t> T* dev(int piece) const { return reinterpret_cast<T*>(d_ + pieces_[piece].off); }
    template <class T = uint8_t> T* host(int piece) const { return reinterpret_cast<T*>(h_ + pieces_[piece].off); }

    cudaError_t upload(cudaStream_t st) const {
        for (const Piece& p : pieces_)
            if (p.src && p.bytes && p.kind <= INOUT) memcpy(h_ + p.off, p.src, p.bytes);
        return upEnd_ ? cudaMemcpyAsync(d_, h_, upEnd_, cudaMemcpyHostToDevice, st) : cudaSuccess;
    }
    cudaError_t download(cudaStream_t st) const {
        cudaError_t e = downEnd_ > downBegin_ ? cudaMemcpyAsync(h_ + downBegin_, d_ + downBegin_, downEnd_ - downBegin_, cudaMemcpyDeviceToHost, st)
                                              : cudaSuccess;
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return e;
        for (const Piece& p : pieces_)
            if (p.dst && p.bytes) memcpy(p.dst, h_ + p.off, p.bytes);
        return cudaSuccess;
    }

    void release() {
        if (d_ || h_) cudaSetDevice(device);
        if (d_) cudaFree(d_);
        if (h_) cudaFreeHost(h_);
        d_ = h_ = nullptr; dcap_ = hcap_ = 0;
    }

private:
    enum Kind { IN, INOUT, OUT, SCRATCH };
    struct Piece { Kind kind; size_t bytes; const void* src; void* dst; size_t off; };
    int add(Kind k, size_t bytes, const void* src, void* dst) {
        pieces_.push_back({k, bytes, src, dst, 0});
        return (int)pieces_.size() - 1;
    }
    std::vector<Piece> pieces_;
    size_t upEnd_ = 0, downBegin_ = 0, downEnd_ = 0;   // in + inout = [0, upEnd_), inout + out = [downBegin_, downEnd_)
    uint8_t *d_ = nullptr, *h_ = nullptr;
    size_t dcap_ = 0, hcap_ = 0;
};

// Per-row counts of the pose optimisers' [count][cap] slot arrays: N[f] in [0, cap], checked before anything is staged.
inline int check_row_counts(const char* where, const int32_t* N, int count, int cap) {
    for (int f = 0; f < count; ++f)
        if (N[f] < 0 || N[f] > cap) { set_error(std::string(where) + ": N[f] outside [0, cap]"); return ORB_ERR_ARG; }
    return ORB_OK;
}
// CSR offsets start[0, n] that start at 0 and do not decrease.
inline bool csr_ok(int n, const int32_t* start) {
    if (start[0] != 0) return false;
    for (int i = 0; i < n; ++i) if (start[i + 1] < start[i]) return false;
    return true;
}
// No key of keys[0, n) repeats.
inline bool all_distinct(const uint64_t* keys, int n) {
    std::vector<uint64_t> s(keys, keys + n);
    std::sort(s.begin(), s.end());
    return std::adjacent_find(s.begin(), s.end()) == s.end();
}
// The kernels write the slots [0, N[f]) of an output row only and download copies the whole row, so the slots past N[f] would carry
// whatever the staging buffer last held there: they are set to 0 after download.
inline void zero_row_tails(uint8_t* rows, const int32_t* N, int count, int cap) {
    for (int f = 0; f < count; ++f) memset(rows + (size_t)f * cap + N[f], 0, (size_t)(cap - N[f]));
}

// The staging and stream of the stateless batch entry points (inertial.cu, pose_opt.cu, local_inertial_ba.cu; static functions
// in the reference, so no object owns them): one per host thread, moved when a call names another device.
struct ThreadStaging : Staging {
    cudaStream_t stream = nullptr;
    ~ThreadStaging() { if (stream) cudaStreamDestroy(stream); }
};
inline int thread_staging(int device, ThreadStaging** out) {
    thread_local ThreadStaging S;
    if (int rc = check_device(device)) return rc;
    if (S.device != device) {
        S.release();
        if (S.stream) { cudaStreamDestroy(S.stream); S.stream = nullptr; }
        S.device = device;
    }
    CK(cudaSetDevice(device));
    if (!S.stream) CK(cudaStreamCreateWithFlags(&S.stream, cudaStreamNonBlocking));
    *out = &S;
    return ORB_OK;
}

}  // namespace orbx
