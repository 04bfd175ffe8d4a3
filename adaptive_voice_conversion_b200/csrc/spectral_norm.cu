// Spectral norm of the decoder weights (torch.nn.utils.spectral_norm, n_power_iterations=1, eps=1e-12, dim=0) and
// its gradient, for a device table of layers in three (iterate), two (fixed) and two (backward) launches.
//
// W = weight_orig viewed as [h][w].  Every matrix is cut into chunks of SN_ROWS rows; one CTA handles one
// (item, chunk) unit, and a grid-stride loop over the units of all items spreads each matrix over several CTAs.
// Quantities a chunk needs from the whole matrix (t = W^T u, ||t||, ||s||, sigma, <g, W_bar>) are partial sums in
// per-item scratch that every CTA of the item adds up again in the same order: no atomics, and an item's bits
// depend neither on the grid size nor on the other items of the launch.
#include "common.cuh"

namespace avc {
namespace {

constexpr int SN_ROWS = 16;      // rows of W per work unit
constexpr int SN_THREADS = 256;
constexpr int SN_MAX_GRID = 4 * 132;
constexpr float SN_EPS = 1e-12f; // F.normalize's eps of torch.nn.utils.spectral_norm

__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
#pragma unroll
  for (int i = 0; i < SN_THREADS / 32; ++i) r += sh[i];   // every thread: the same sum in the same order
  __syncthreads();
  return r;
}

// chunk prefix table of the launch's items (first[i] = first unit of item i); items past the declared maxima get none
struct Units {
  int first[AVC_SN_MAX_ITEMS + 1];
};

__device__ void load_units(const avc_sn_item* items, int n, int max_h, int max_w, Units& u) {
  if (threadIdx.x < n) {   // the item loads in parallel, the prefix sum from shared memory
    const int h = items[threadIdx.x].h, w = items[threadIdx.x].w;
    u.first[threadIdx.x + 1] = (h >= 1 && w >= 1 && h <= max_h && w <= max_w) ? cdiv(h, SN_ROWS) : 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    u.first[0] = 0;
    for (int i = 1; i <= n; ++i) u.first[i] += u.first[i - 1];
  }
  __syncthreads();
}

__device__ __forceinline__ int unit_item(const Units& u, int n, int unit) {
  int i = 0;
  while (u.first[i + 1] <= unit) ++i;
  return i;
}

__device__ __forceinline__ int64_t s_off(const avc_sn_item& it) { return it.scratch_off + (int64_t)cdiv(it.h, SN_ROWS) * it.w; }

// part[c][j] = sum over the rows i of chunk c, in order, of W[i][j] u[i]
__global__ void __launch_bounds__(SN_THREADS) sn_wtu_kernel(const avc_sn_item* __restrict__ items, int n, int max_h, int max_w,
                                                            float* __restrict__ scratch) {
  __shared__ Units U;
  __shared__ float ush[SN_ROWS];
  load_units(items, n, max_h, max_w, U);
  for (int unit = blockIdx.x; unit < U.first[n]; unit += gridDim.x) {
    const int ii = unit_item(U, n, unit);
    const avc_sn_item it = items[ii];
    const int c = unit - U.first[ii], r0 = c * SN_ROWS, r1 = min(it.h, r0 + SN_ROWS);
    if (threadIdx.x < r1 - r0) ush[threadIdx.x] = it.u[r0 + threadIdx.x];
    __syncthreads();
    float* part = scratch + it.scratch_off + (int64_t)c * it.w;
    for (int j = threadIdx.x; j < it.w; j += SN_THREADS) {
      float acc = 0.f;
      for (int i = r0; i < r1; ++i) acc = fmaf(it.weight[(int64_t)i * it.w + j], ush[i - r0], acc);
      part[j] = acc;
    }
    __syncthreads();
  }
}

// v = normalize(sum_c part[c]) (iterate) or the stored v (fixed); s[i] = (W v)[i] for the chunk's rows
__global__ void __launch_bounds__(SN_THREADS) sn_wv_kernel(const avc_sn_item* __restrict__ items, int n, int max_h, int max_w,
                                                           int mode, float* __restrict__ scratch) {
  __shared__ Units U;
  __shared__ float vsh[AVC_SN_MAX_W];
  __shared__ float red[SN_THREADS / 32];
  load_units(items, n, max_h, max_w, U);
  for (int unit = blockIdx.x; unit < U.first[n]; unit += gridDim.x) {
    const int ii = unit_item(U, n, unit);
    const avc_sn_item it = items[ii];
    const int c = unit - U.first[ii], r0 = c * SN_ROWS, r1 = min(it.h, r0 + SN_ROWS);
    if (mode == AVC_SN_ITERATE) {
      const int nc = cdiv(it.h, SN_ROWS);
      const float* part = scratch + it.scratch_off;
      float sq = 0.f;
      for (int j = threadIdx.x; j < it.w; j += SN_THREADS) {
        float t = 0.f;
        for (int k = 0; k < nc; ++k) t += part[(int64_t)k * it.w + j];
        vsh[j] = t;
        sq = fmaf(t, t, sq);
      }
      const float denom = fmaxf(sqrtf(block_sum(sq, red)), SN_EPS);
      for (int j = threadIdx.x; j < it.w; j += SN_THREADS) {
        const float v = vsh[j] / denom;
        vsh[j] = v;
        if (c == 0) it.v[j] = v;
      }
    } else {
      for (int j = threadIdx.x; j < it.w; j += SN_THREADS) vsh[j] = it.v[j];
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* s = scratch + s_off(it);
    for (int i = r0 + warp; i < r1; i += SN_THREADS / 32) {
      const float* row = it.weight + (int64_t)i * it.w;
      float acc = 0.f;
      for (int j = lane; j < it.w; j += 32) acc = fmaf(row[j], vsh[j], acc);
      acc = warp_sum(acc);
      if (lane == 0) s[i] = acc;
    }
    __syncthreads();
  }
}

// iterate: u = normalize(s), sigma = u . s; fixed: sigma = u . s with the stored u.  Then W_bar = W / sigma.
__global__ void __launch_bounds__(SN_THREADS) sn_scale_kernel(const avc_sn_item* __restrict__ items, int n, int max_h, int max_w,
                                                              int mode, const float* __restrict__ scratch) {
  __shared__ Units U;
  __shared__ float red[SN_THREADS / 32];
  load_units(items, n, max_h, max_w, U);
  for (int unit = blockIdx.x; unit < U.first[n]; unit += gridDim.x) {
    const int ii = unit_item(U, n, unit);
    const avc_sn_item it = items[ii];
    const int c = unit - U.first[ii], r0 = c * SN_ROWS, r1 = min(it.h, r0 + SN_ROWS);
    const float* s = scratch + s_off(it);
    float sigma;
    if (mode == AVC_SN_ITERATE) {
      float sq = 0.f;
      for (int i = threadIdx.x; i < it.h; i += SN_THREADS) sq = fmaf(s[i], s[i], sq);
      const float denom = fmaxf(sqrtf(block_sum(sq, red)), SN_EPS);
      float dot = 0.f;
      for (int i = threadIdx.x; i < it.h; i += SN_THREADS) {
        const float u = s[i] / denom;
        if (c == 0) it.u[i] = u;
        dot = fmaf(u, s[i], dot);
      }
      sigma = block_sum(dot, red);
    } else {
      float dot = 0.f;
      for (int i = threadIdx.x; i < it.h; i += SN_THREADS) dot = fmaf(it.u[i], s[i], dot);
      sigma = block_sum(dot, red);
    }
    if (c == 0 && threadIdx.x == 0) it.sigma[0] = sigma;
    const int64_t e0 = (int64_t)r0 * it.w, e1 = (int64_t)r1 * it.w;
    for (int64_t e = e0 + threadIdx.x; e < e1; e += SN_THREADS) it.w_bar[e] = __fdiv_rn(it.weight[e], sigma);
  }
}

// part[c] = sum over the chunk's elements of g * W_bar (thread-strided, then the block's fixed tree)
__global__ void __launch_bounds__(SN_THREADS) sn_bwd_dot_kernel(const avc_sn_item* __restrict__ items, int n, int max_h, int max_w,
                                                                float* __restrict__ scratch) {
  __shared__ Units U;
  __shared__ float red[SN_THREADS / 32];
  load_units(items, n, max_h, max_w, U);
  for (int unit = blockIdx.x; unit < U.first[n]; unit += gridDim.x) {
    const int ii = unit_item(U, n, unit);
    const avc_sn_item it = items[ii];
    const int c = unit - U.first[ii], r0 = c * SN_ROWS, r1 = min(it.h, r0 + SN_ROWS);
    const int64_t e0 = (int64_t)r0 * it.w, e1 = (int64_t)r1 * it.w;
    float acc = 0.f;
    for (int64_t e = e0 + threadIdx.x; e < e1; e += SN_THREADS) acc = fmaf(it.grad[e], it.w_bar[e], acc);
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) scratch[s_off(it) + it.h + c] = acc;
  }
}

// g = (g - <g, W_bar> u v^T) / sigma
__global__ void __launch_bounds__(SN_THREADS) sn_bwd_apply_kernel(const avc_sn_item* __restrict__ items, int n, int max_h, int max_w,
                                                                  const float* __restrict__ scratch) {
  __shared__ Units U;
  load_units(items, n, max_h, max_w, U);
  for (int unit = blockIdx.x; unit < U.first[n]; unit += gridDim.x) {
    const int ii = unit_item(U, n, unit);
    const avc_sn_item it = items[ii];
    const int c = unit - U.first[ii], r0 = c * SN_ROWS, r1 = min(it.h, r0 + SN_ROWS);
    const int nc = cdiv(it.h, SN_ROWS);
    const float* part = scratch + s_off(it) + it.h;
    float dot = 0.f;
    for (int k = 0; k < nc; ++k) dot += part[k];
    const float sigma = it.sigma[0];
    const float* __restrict__ v = it.v;
    const int w = it.w;
    for (int i = r0; i < r1; ++i) {
      const float du = dot * it.u[i];
      float* g = it.grad + (int64_t)i * w;
      for (int j = threadIdx.x; j < w; j += SN_THREADS) g[j] = __fdiv_rn(g[j] - du * v[j], sigma);
    }
  }
}

int sn_check(const avc_sn_item* items, int n, int max_h, int max_w, const float* scratch, const char* who) {
  AVC_REQUIRE(items && scratch && n >= 1 && max_h >= 1 && max_w >= 1, AVC_ERR_INVALID, "%s: bad argument", who);
  AVC_REQUIRE(n <= AVC_SN_MAX_ITEMS && max_h <= AVC_SN_MAX_H && max_w <= AVC_SN_MAX_W, AVC_ERR_UNSUPPORTED,
              "%s: n=%d max_h=%d max_w=%d beyond the limits (%d items, h <= %d, w <= %d)", who, n, max_h, max_w,
              AVC_SN_MAX_ITEMS, AVC_SN_MAX_H, AVC_SN_MAX_W);
  return AVC_OK;
}

int sn_grid(int n, int max_h) {
  const int units = n * cdiv(max_h, SN_ROWS);
  return units < SN_MAX_GRID ? units : SN_MAX_GRID;
}

}  // namespace
}  // namespace avc

using namespace avc;

extern "C" int64_t avc_spectral_norm_scratch_floats(int h, int w) {
  if (h < 1 || w < 1) return 0;
  const int64_t nc = cdiv(h, SN_ROWS);
  return nc * w + h + nc;   // [chunk][w] partials of W^T u, s = W v, [chunk] partials of <g, W_bar>
}

extern "C" int avc_spectral_norm(const avc_sn_item* items, int n, int max_h, int max_w, int mode, float* scratch, void* stream) {
  int rc = sn_check(items, n, max_h, max_w, scratch, "avc_spectral_norm");
  if (rc != AVC_OK) return rc;
  AVC_REQUIRE(mode == AVC_SN_ITERATE || mode == AVC_SN_FIXED, AVC_ERR_INVALID, "avc_spectral_norm: bad mode %d", mode);
  const int grid = sn_grid(n, max_h);
  cudaStream_t st = (cudaStream_t)stream;
  if (mode == AVC_SN_ITERATE) {
    AVC_LAUNCH(sn_wtu_kernel, grid, SN_THREADS, 0, st, items, n, max_h, max_w, scratch);
    AVC_CHECK_LAUNCH("sn_wtu");
  }
  AVC_LAUNCH(sn_wv_kernel, grid, SN_THREADS, 0, st, items, n, max_h, max_w, mode, scratch);
  AVC_CHECK_LAUNCH("sn_wv");
  AVC_LAUNCH(sn_scale_kernel, grid, SN_THREADS, 0, st, items, n, max_h, max_w, mode, scratch);
  AVC_CHECK_LAUNCH("sn_scale");
  return AVC_OK;
}

extern "C" int avc_spectral_norm_bwd(const avc_sn_item* items, int n, int max_h, int max_w, float* scratch, void* stream) {
  int rc = sn_check(items, n, max_h, max_w, scratch, "avc_spectral_norm_bwd");
  if (rc != AVC_OK) return rc;
  const int grid = sn_grid(n, max_h);
  cudaStream_t st = (cudaStream_t)stream;
  AVC_LAUNCH(sn_bwd_dot_kernel, grid, SN_THREADS, 0, st, items, n, max_h, max_w, scratch);
  AVC_CHECK_LAUNCH("sn_bwd_dot");
  AVC_LAUNCH(sn_bwd_apply_kernel, grid, SN_THREADS, 0, st, items, n, max_h, max_w, scratch);
  AVC_CHECK_LAUNCH("sn_bwd_apply");
  return AVC_OK;
}
