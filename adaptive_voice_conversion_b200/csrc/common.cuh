// Shared device/host helpers for libavc_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/avc_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libavc_b200 is written for sm_90a (H100) only"
#endif

namespace avc {

#define AVC_LAUNCH(kern, grid, block, smem, st, ...) kern<<<grid, block, smem, st>>>(__VA_ARGS__)

void set_error(const char* fmt, ...);
void count_launch(int n = 1);
// dw += sum over slices of scratch[slice][tap][ci/4][coutp][4], in a fixed order (wgrad_tc.cu; both weight-gradient
// kernels write their per-slice partial sums in this layout)
int wgrad_reduce(const float* scratch, float* dw, int Cout, int Cin, int K, int coutp, int nslices, cudaStream_t stream);

#define AVC_REQUIRE(cond, code, ...) \
  do {                               \
    if (!(cond)) {                   \
      avc::set_error(__VA_ARGS__);   \
      return (code);                 \
    }                                \
  } while (0)

#define AVC_CHECK_LAUNCH(name)                                                  \
  do {                                                                          \
    cudaError_t e__ = cudaGetLastError();                                       \
    if (e__ != cudaSuccess) {                                                   \
      avc::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));   \
      return AVC_ERR_CUDA;                                                      \
    }                                                                           \
    avc::count_launch();                                                        \
  } while (0)

__host__ __device__ inline int cdiv(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Source position of padded/zero-inserted input index p (may be out of range).
// L = logical length (Tin * ups).  Returns -1 for "reads zero".
__device__ __forceinline__ int src_pos(int p, int L, int pad_mode, int ups) {
  if (pad_mode == AVC_PAD_REFLECT) {
    if (p < 0) p = -p;
    if (p >= L) p = 2 * (L - 1) - p;
    if (p < 0 || p >= L) return -1;  // pad wider than the signal: undefined in torch, read 0
  } else {
    if (p < 0 || p >= L) return -1;
  }
  if (ups == 2) {
    if (p & 1) return -1;
    p >>= 1;
  }
  return p;
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace avc
