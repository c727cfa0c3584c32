// What lba.cu's resident solver and local_ba.cu's whole-function path (lba_local_bundle_adjustment_batch) share: the hand-over of a
// graph built on the device into a solver slot, and the solver operations the path drives on the handle's stream.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/orb_b200.h"
#include "staging.h"

namespace lba {

// thHuberMono = (float)sqrt(5.991) (src/Optimizer.cc:1275), as rk->setDelta receives it
inline double huber_mono() { return (double)(float)sqrt(5.991); }

// One problem built on the device, in LbaProblem's layout (device pointers): poses [nP][7], fixed [nP], cam [nP][4], points [nL][3],
// edges [nE] (point, pose, obs [2], invSigma2).  lba_fill_kernel copies it into a slot laid out for its sizes.
struct FillSrc {
    const double* poses; const uint8_t* fixed; const float* cam; const double* points;
    const int* edgePoint; const int* edgePose; const double* obs; const float* invSigma2;
};

// Where a loaded slot's solver writes its results (device pointers; the layout of LbaResult, stats as lba_download_batch reads them).
struct SlotOut { const double* poses; const double* points; const double* chi2; const uint8_t* depthPos; const double* stats; };

// Solver operations on h's stream (lba.cu).
cudaStream_t solver_stream(lba_handle* h);
orbx::Staging& solver_staging(lba_handle* h);
void solver_limits(const lba_handle* h, int* maxP, int* maxL, int* maxE, int* maxBatch);
// Lay out slots 0..count-1 from sizes (nP, nL, nE, nF), fill them from dFill (device table, slot order) and enqueue the structure
// kernel; out[i] receives slot i's result pointers.  Two launches.
int solver_load_device(lba_handle* h, int count, const int4* sizes, const double* userLambdaInit, const FillSrc* dFill, SlotOut* out);
// Run the loaded slots forwarding the stop flags (one per slot, may be NULL); one launch.
int solver_run(lba_handle* h, const volatile uint8_t* const* flags);
// Wait for the structure kernel and return its verdict (ORB_ERR_ARG / ORB_ERR_CAPACITY as lba_upload_batch does); a refused graph
// leaves nothing loaded, so solver_run refuses to run.
int solver_check_structure(lba_handle* h, int count);
void solver_set_local_launches(lba_handle* h, int n);

}  // namespace lba
