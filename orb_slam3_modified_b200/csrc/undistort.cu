// Frame::UndistortKeyPoints and Frame::ComputeImageBounds (reference src/Frame.cc:747, :766, :793) for pinhole cameras with radial /
// tangential distortion: the per-point function is csrc/undistort.h, bit for bit cv::undistortPoints(..., cv::Mat(), K).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <string>

#include "../../include/orb_b200.h"
#include "device_utils.cuh"
#include "undistort.h"

namespace orbx {

thread_local int g_undistort_launches = 0;   // orbx_undistort_last_launch_count(): launches of this thread's last undistortion call

constexpr int UD_NT = 128;

// One thread per keypoint row of a [batch][cap] slab.  Rows [0, n[f]) of frame f are written; a frame with n[f] > cap (the extractor's
// overflow) and the rows past n[f] are not touched.  Only x and y change: the other five fields are copied as raw words.
__global__ void __launch_bounds__(UD_NT) undistort_kernel(OrbPinholeCamera cam, const OrbKeyPoint* __restrict__ kps, const int* __restrict__ n,
                                                          int cap, OrbKeyPoint* __restrict__ out) {
    const int f = blockIdx.y, i = blockIdx.x * UD_NT + threadIdx.x;
    const int nf = n[f];
    if (nf > cap || i >= nf) return;
    const size_t row = (size_t)f * cap + i;
    const uint32_t* src = reinterpret_cast<const uint32_t*>(kps + row);
    uint32_t* dst = reinterpret_cast<uint32_t*>(out + row);
    uint32_t w[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) w[k] = src[k];
    if (cam.k1 != 0.0f) {                                   // mvKeysUn = mvKeys when mDistCoef.at<float>(0) == 0 (src/Frame.cc:749)
        float x, y;
        undistort_point(__uint_as_float(w[0]), __uint_as_float(w[1]), cam.fx, cam.fy, cam.cx, cam.cy, cam.k1, cam.k2, cam.p1, cam.p2, cam.k3, &x, &y);
        w[0] = __float_as_uint(x);
        w[1] = __float_as_uint(y);
    }
#pragma unroll
    for (int k = 0; k < 7; ++k) dst[k] = w[k];
}

__global__ void image_bounds_kernel(OrbPinholeCamera cam, int cols, int rows, float* out) {
    const float c[9] = {cam.fx, cam.fy, cam.cx, cam.cy, cam.k1, cam.k2, cam.p1, cam.p2, cam.k3};
    image_bounds(c, cols, rows, out);
}

// fx, fy non-zero and finite, every other member finite.
int check_camera(const OrbPinholeCamera* cam, const char* where) {
    if (!cam) { set_error(std::string(where) + ": null camera"); return ORB_ERR_ARG; }
    const float v[9] = {cam->fx, cam->fy, cam->cx, cam->cy, cam->k1, cam->k2, cam->p1, cam->p2, cam->k3};
    for (float x : v)
        if (!isfinite(x)) { set_error(std::string(where) + ": non-finite camera parameter"); return ORB_ERR_ARG; }
    if (cam->fx == 0.0f || cam->fy == 0.0f) { set_error(std::string(where) + ": fx or fy is zero"); return ORB_ERR_ARG; }
    return ORB_OK;
}

// The checks and the one launch of orbx_undistort_keypoints_device, shared with the handle's host form (extractor.cu).
int undistort_enqueue(const OrbPinholeCamera* cam, int batch, const OrbKeyPoint* kps, const int* n, int cap, OrbKeyPoint* out, cudaStream_t st,
                      const char* where) {
    g_undistort_launches = 0;
    if (!kps || !n || !out || batch < 0 || cap < 1) { set_error(std::string(where) + ": bad argument"); return ORB_ERR_ARG; }
    if (int rc = check_camera(cam, where)) return rc;
    const uintptr_t a0 = (uintptr_t)kps, b0 = (uintptr_t)out, len = sizeof(OrbKeyPoint) * (uintptr_t)cap * (uintptr_t)(batch > 0 ? batch : 1);
    if (a0 < b0 + len && b0 < a0 + len) {
        set_error(std::string(where) + ": the output slab overlaps the input slab (mvKeys stays in use beside mvKeysUn)");
        return ORB_ERR_ARG;
    }
    if (batch == 0) return ORB_OK;
    if (batch > 65535) { set_error(std::string(where) + ": batch larger than 65535"); return ORB_ERR_ARG; }
    undistort_kernel<<<dim3((cap + UD_NT - 1) / UD_NT, batch), UD_NT, 0, st>>>(*cam, kps, n, cap, out);
    CK(cudaGetLastError());
    g_undistort_launches = 1;
    return ORB_OK;
}

int handle_device(const orbx_handle* h);   // extractor.cu

}  // namespace orbx

using namespace orbx;

extern "C" {

int orbx_undistort_keypoints_device(orbx_handle* h, const OrbPinholeCamera* cam, int batch, const OrbKeyPoint* d_kps, const int* d_n, int cap,
                                    OrbKeyPoint* d_kpsUn, void* stream) {
    g_undistort_launches = 0;
    if (!h) { set_error("orbx_undistort_keypoints_device: null handle"); return ORB_ERR_ARG; }
    CK(cudaSetDevice(handle_device(h)));
    return undistort_enqueue(cam, batch, d_kps, d_n, cap, d_kpsUn, (cudaStream_t)stream, "orbx_undistort_keypoints_device");
}

int orbx_image_bounds(const OrbPinholeCamera* cam, int cols, int rows, float* bounds4, int device) {
    g_undistort_launches = 0;
    if (!bounds4 || cols < 1 || rows < 1) { set_error("orbx_image_bounds: bad argument"); return ORB_ERR_ARG; }
    if (int rc = check_camera(cam, "orbx_image_bounds")) return rc;
    if (int rc = check_device(device)) return rc;
    CK(cudaSetDevice(device));
    float* d_out = nullptr;
    CK(cudaMalloc(&d_out, 4 * sizeof(float)));
    image_bounds_kernel<<<1, 1>>>(*cam, cols, rows, d_out);
    cudaError_t err = cudaGetLastError();
    if (err == cudaSuccess) g_undistort_launches = 1;
    float out[4];
    if (err == cudaSuccess) err = cudaMemcpy(out, d_out, sizeof(out), cudaMemcpyDeviceToHost);
    cudaFree(d_out);
    if (err != cudaSuccess) { set_error(std::string("orbx_image_bounds: ") + cudaGetErrorString(err)); return ORB_ERR_CUDA; }
    for (int i = 0; i < 4; ++i) bounds4[i] = out[i];
    return ORB_OK;
}

int orbx_undistort_last_launch_count(void) { return g_undistort_launches; }

}  // extern "C"
