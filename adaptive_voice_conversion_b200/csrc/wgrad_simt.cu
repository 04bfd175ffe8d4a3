// Weight gradient of pad_layer + Conv1d (autograd of model.py:21-32 under solver.py:90):
//   dW[co][ci][j] += sum_{b, t} dc[b][co][t] * xpad[b][ci][t*stride + j]
// A [co x ci] GEMM per tap with the reduction over (sample, time).  One CTA: 128 co x
// 128 ci for one tap and one slice of the batch; its partial sums go to a scratch buffer
// [slice][tap][ci/4][coutp][4] (the tensor-core kernel's layout) and wgrad_tc_reduce_kernel adds
// them into the canonical nn.Conv1d-layout gradient in a fixed order: no atomics, so the
// gradient is the same on every run.
#include "common.cuh"

namespace avc {

constexpr int WG_TK = 16;
constexpr int WG_LD = 132;  // 128 + 4: conflict-free float4 staging stores

struct WgradArgs {
  avc_wgrad_desc d;
  float* scratch;
  int nsl, bps, coutp;  // batch slices, samples per slice, Cout rounded up to the 128-row tile
};

__global__ void __launch_bounds__(256, 2) conv_wgrad_kernel(const WgradArgs a) {
  __shared__ __align__(16) float As[WG_TK * WG_LD];  // dc  [t][co]
  __shared__ __align__(16) float Bs[WG_TK * WG_LD];  // x   [t][ci] (tap-shifted, reflect-padded)
  const avc_wgrad_desc& d = a.d;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int ci0 = blockIdx.x * 128, co0 = blockIdx.y * 128;
  const int j = blockIdx.z / a.nsl;
  const int sl = blockIdx.z - j * a.nsl;
  const int bbeg = sl * a.bps;
  const int bend = min(d.B, bbeg + a.bps);

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[i][k] = 0.f;

  for (int b = bbeg; b < bend; ++b) {
    for (int tc0 = 0; tc0 < d.Tout; tc0 += WG_TK) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int idx = tid + r * 256;  // 32 chunks x 16 time steps
        const int q = idx >> 4, tt = idx & 15;
        const int t = tc0 + tt;
        float4 va = zero4(), vb = zero4();
        if (t < d.Tout) {
          const int co = co0 + 4 * q;
          if (co < d.Cout) va = ldg4(d.dc + (int64_t)b * d.dc_bstride + ((int64_t)(co >> 2) * d.Tout + t) * 4);
          const int ci = ci0 + 4 * q;
          if (ci < d.Cin) {
            const int p = src_pos(t * d.stride + j - d.pad_left, d.Tin, AVC_PAD_REFLECT, 1);
            if (p >= 0) vb = ldg4(d.x + (int64_t)b * d.x_bstride + ((int64_t)(ci >> 2) * d.Tin + p) * 4);
          }
        }
        st4(As + tt * WG_LD + 4 * q, va);
        st4(Bs + tt * WG_LD + 4 * q, vb);
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < WG_TK; ++kk) {
        const float4 a0 = *reinterpret_cast<const float4*>(As + kk * WG_LD + ty * 8);
        const float4 a1 = *reinterpret_cast<const float4*>(As + kk * WG_LD + ty * 8 + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(Bs + kk * WG_LD + tx * 8);
        const float4 b1 = *reinterpret_cast<const float4*>(Bs + kk * WG_LD + tx * 8 + 4);
        const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[i][k] = fmaf(av[i], bv[k], acc[i][k]);
      }
      __syncthreads();
    }
  }
  // rows co >= Cout of the last tile hold zeros (their dc was staged as zeros); the reduction skips them
  float* part = a.scratch + ((int64_t)sl * d.K + j) * (int64_t)(d.Cin >> 2) * a.coutp * 4;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int ci = ci0 + tx * 8 + 4 * h;
    if (ci >= d.Cin) continue;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int co = co0 + ty * 8 + i;
      st4(part + ((int64_t)(ci >> 2) * a.coutp + co) * 4,
          make_float4(acc[i][4 * h], acc[i][4 * h + 1], acc[i][4 * h + 2], acc[i][4 * h + 3]));
    }
  }
}

static void wgrad_simt_plan(const avc_wgrad_desc* d, WgradArgs& a) {
  a.d = *d;
  const int tiles = cdiv(d->Cin, 128) * cdiv(d->Cout, 128) * d->K;
  // enough CTAs for ~2 waves of 148 SMs, but keep >= 256 reduction steps per CTA so the
  // partial sums' round trip through the scratch buffer stays a minor cost
  int64_t kdepth = (int64_t)d->B * d->Tout;
  int nsl = (int)cdiv64(2 * 148 * 2, tiles);
  int max_by_depth = (int)(kdepth / 256);
  if (max_by_depth < 1) max_by_depth = 1;
  if (nsl > max_by_depth) nsl = max_by_depth;
  if (nsl > d->B) nsl = d->B;
  if (nsl < 1) nsl = 1;
  a.bps = cdiv(d->B, nsl);
  a.nsl = cdiv(d->B, a.bps);
  a.coutp = cdiv(d->Cout, 128) * 128;
}

static bool wgrad_simt_valid(const avc_wgrad_desc* d) {
  return d->B > 0 && d->Cin > 0 && d->Cout > 0 && d->K >= 1 && d->Tin > 0 && d->Tout > 0 && d->Cin % 4 == 0 && d->Cout % 4 == 0;
}

}  // namespace avc

using namespace avc;

extern "C" int64_t avc_conv_wgrad_scratch_floats(const avc_wgrad_desc* d) {
  if (!d || !wgrad_simt_valid(d)) return -1;
  WgradArgs a;
  wgrad_simt_plan(d, a);
  return (int64_t)a.nsl * d->K * d->Cin * a.coutp;
}

extern "C" int avc_conv_wgrad(const avc_wgrad_desc* d, float* scratch, void* stream) {
  AVC_REQUIRE(d && d->x && d->dc && d->dw && scratch, AVC_ERR_INVALID, "avc_conv_wgrad: null argument");
  AVC_REQUIRE(d->B > 0 && d->Cin > 0 && d->Cout > 0 && d->K >= 1 && d->Tin > 0 && d->Tout > 0, AVC_ERR_INVALID,
              "avc_conv_wgrad: bad shape");
  AVC_REQUIRE(d->Cin % 4 == 0 && d->Cout % 4 == 0, AVC_ERR_INVALID, "avc_conv_wgrad: channels must be multiples of 4");
  WgradArgs a;
  wgrad_simt_plan(d, a);
  a.scratch = scratch;
  dim3 grid(cdiv(d->Cin, 128), cdiv(d->Cout, 128), d->K * a.nsl);
  AVC_LAUNCH(conv_wgrad_kernel, grid, 256, 0, (cudaStream_t)stream, a);
  AVC_CHECK_LAUNCH("conv_wgrad");
  return wgrad_reduce(scratch, d->dw, d->Cout, d->Cin, d->K, a.coutp, a.nsl, (cudaStream_t)stream);
}
