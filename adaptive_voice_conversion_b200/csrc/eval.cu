// Held-out evaluation (evaluate.HeldOut): the per-segment reconstruction and KL sums of one batch of the conversion path,
// in float64.
//
// One CTA per sample.  Each thread accumulates its strided share of the sample in a double, then the block adds the
// 512 partial sums in a fixed tree.  The order depends only on the sample's sizes, so the sums have the same bits on
// every run and in any batch.  dec is read as the engine's A4 [C/4][T][4] (one float4 per 4 channels x 1 step) and x as
// planar [C][T]: the four x reads of a unit are four coalesced warp-wide loads along time.  Each byte is read once.
#include "common.cuh"

namespace avc {

constexpr int EV_THREADS = 512;

__device__ __forceinline__ double block_sum_f64(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x < 32) {
    r = threadIdx.x < EV_THREADS / 32 ? sh[threadIdx.x] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  }
  __syncthreads();
  return r;  // valid on warp 0
}

// exp(ls) + mu^2 - 1 - ls, evaluated left to right in float64 as torch does on float64 tensors
__device__ __forceinline__ double kl_term(float m, float l) {
  const double md = m, ld = l;
  return exp(ld) + md * md - 1.0 - ld;
}

__global__ void __launch_bounds__(EV_THREADS) eval_losses_kernel(const avc_eval_desc d) {
  __shared__ double sh[EV_THREADS / 32];
  const int b = blockIdx.x, T = d.T;
  const int64_t units = (int64_t)(d.C / 4) * T;
  const float* dec = d.dec + (int64_t)b * d.C * T;
  const float* x = d.x + (int64_t)b * d.C * T;
  double rec = 0.0;
#pragma unroll 4
  for (int64_t u = threadIdx.x; u < units; u += EV_THREADS) {
    const int64_t q = u / T, t = u - q * T;
    const float4 v = ldg4(dec + 4 * u);
    const float* xp = x + 4 * q * T + t;
    const float x0 = __ldg(xp), x1 = __ldg(xp + T), x2 = __ldg(xp + 2 * T), x3 = __ldg(xp + 3 * T);
    rec += fabs((double)v.x - (double)x0);
    rec += fabs((double)v.y - (double)x1);
    rec += fabs((double)v.z - (double)x2);
    rec += fabs((double)v.w - (double)x3);
  }
  const int64_t nl4 = (int64_t)(d.C_lat / 4) * d.T_lat;
  const float* mu = d.mu + (int64_t)b * 4 * nl4;
  const float* ls = d.ls + (int64_t)b * 4 * nl4;
  double kl = 0.0;
  for (int64_t i = threadIdx.x; i < nl4; i += EV_THREADS) {
    const float4 m = ldg4(mu + 4 * i), l = ldg4(ls + 4 * i);
    kl += kl_term(m.x, l.x);
    kl += kl_term(m.y, l.y);
    kl += kl_term(m.z, l.z);
    kl += kl_term(m.w, l.w);
  }
  rec = block_sum_f64(rec, sh);
  kl = block_sum_f64(kl, sh);
  if (threadIdx.x == 0) {
    d.out[2 * (d.first + b) + 0] = rec;
    d.out[2 * (d.first + b) + 1] = kl;
  }
}

// Held-out reconstruction of padded batches of different-length utterances (speaker adaptation's check).  One CTA per
// sample; thread i adds the units i, i + 512, ... of the sample's first L_b frames in row-major (c, t) order, then the
// block adds the partial sums in block_sum_f64's fixed tree.  Frames past L_b are never read.
__global__ void __launch_bounds__(EV_THREADS) rec_loss_varlen_kernel(const avc_rec_varlen_desc d) {
  __shared__ double sh[EV_THREADS / 32];
  const int b = blockIdx.x, T = d.T;
  const int Lb = min(max(__ldg(d.lengths + b), 0), T);
  const int64_t units = (int64_t)d.C * Lb;
  const float* dec = d.dec + (int64_t)b * d.C * T;
  const float* x = d.x + (int64_t)b * d.C * T;
  double rec = 0.0;
  for (int64_t u = threadIdx.x; u < units; u += EV_THREADS) {
    const int64_t c = u / Lb, t = u - c * Lb;
    rec += fabs((double)__ldg(dec + c * T + t) - (double)__ldg(x + c * T + t));
  }
  rec = block_sum_f64(rec, sh);
  if (threadIdx.x == 0) d.out[b] = rec;
}

}  // namespace avc

using namespace avc;

extern "C" int avc_eval_losses(const avc_eval_desc* d, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "avc_eval_losses: null descriptor");
  AVC_REQUIRE(d->dec != nullptr && d->x != nullptr && d->mu != nullptr && d->ls != nullptr && d->out != nullptr, AVC_ERR_INVALID,
              "avc_eval_losses: null pointer (dec %p, x %p, mu %p, ls %p, out %p)", (const void*)d->dec, (const void*)d->x,
              (const void*)d->mu, (const void*)d->ls, (const void*)d->out);
  AVC_REQUIRE(d->B > 0 && d->C > 0 && d->T > 0 && d->C_lat > 0 && d->T_lat > 0, AVC_ERR_INVALID,
              "avc_eval_losses: sizes must be positive (B %d, C %d, T %d, C_lat %d, T_lat %d)", d->B, d->C, d->T, d->C_lat,
              d->T_lat);
  AVC_REQUIRE(d->C % 4 == 0 && d->C_lat % 4 == 0, AVC_ERR_INVALID,
              "avc_eval_losses: C and C_lat must be multiples of 4 (C %d, C_lat %d)", d->C, d->C_lat);
  AVC_REQUIRE(d->first >= 0, AVC_ERR_INVALID, "avc_eval_losses: first must be >= 0 (got %lld)", (long long)d->first);
  eval_losses_kernel<<<(unsigned)d->B, EV_THREADS, 0, (cudaStream_t)stream>>>(*d);
  AVC_CHECK_LAUNCH("avc_eval_losses");
  return AVC_OK;
}

extern "C" int avc_rec_loss_varlen(const avc_rec_varlen_desc* d, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "avc_rec_loss_varlen: null descriptor");
  AVC_REQUIRE(d->dec != nullptr && d->x != nullptr && d->lengths != nullptr && d->out != nullptr, AVC_ERR_INVALID,
              "avc_rec_loss_varlen: null pointer (dec %p, x %p, lengths %p, out %p)", (const void*)d->dec,
              (const void*)d->x, (const void*)d->lengths, (const void*)d->out);
  AVC_REQUIRE(d->B > 0 && d->C > 0 && d->T > 0, AVC_ERR_INVALID,
              "avc_rec_loss_varlen: sizes must be positive (B %d, C %d, T %d)", d->B, d->C, d->T);
  rec_loss_varlen_kernel<<<(unsigned)d->B, EV_THREADS, 0, (cudaStream_t)stream>>>(*d);
  AVC_CHECK_LAUNCH("avc_rec_loss_varlen");
  return AVC_OK;
}
