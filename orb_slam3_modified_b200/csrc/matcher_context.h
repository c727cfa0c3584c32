// What an entry point compiled outside matcher.cu needs of a matcher handle: its staging, its stream and its launch counter.
#pragma once
#include <cuda_runtime.h>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "staging.h"

namespace orbm {

// A device-form entry point's own scratch: it runs on the caller's stream and returns without a synchronise, so it cannot use the
// staging, which the host forms rewrite on the handle's stream.  Grown to the largest call; cudaFree waits for the kernels still using
// the old buffer.  Like the other device forms' scratch, it is shared by the calls on one handle, which the caller orders on one stream.
struct DeviceScratch {
    uint8_t* ptr = nullptr;
    size_t bytes = 0;
    int reserve(size_t need) {
        if (need <= bytes) return ORB_OK;
        if (ptr) cudaFree(ptr);
        ptr = nullptr; bytes = 0;
        CK(cudaMalloc(&ptr, need));
        bytes = need;
        return ORB_OK;
    }
};

struct MatcherContext {
    orbx::Staging* staging;
    cudaStream_t stream;
    int device;
    int* launches;     // what orbm_last_launch_count() returns
    DeviceScratch* localMapScratch;   // orbm_update_local_map_batch_device's
};
MatcherContext matcher_context(orbm_handle* h);

}  // namespace orbm
