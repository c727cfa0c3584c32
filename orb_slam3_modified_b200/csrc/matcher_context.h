// What an entry point compiled outside matcher.cu needs of a matcher handle: its staging, its stream and its launch counter.
#pragma once
#include <cuda_runtime.h>

#include "../../include/orb_b200.h"
#include "staging.h"

namespace orbm {

struct MatcherContext {
    orbx::Staging* staging;
    cudaStream_t stream;
    int device;
    int* launches;     // what orbm_last_launch_count() returns
};
MatcherContext matcher_context(orbm_handle* h);

}  // namespace orbm
