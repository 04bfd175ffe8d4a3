// Speaker-code fitting (fit.CodeFitTrainer): the grouped L1 loss of a batch of several speakers and the per-code
// clip + Adam update.  A batch of B = G * m samples holds G groups of m consecutive samples; nothing here mixes groups.
//
// avc_group_l1 runs two kernels.  group_l1_kernel: one CTA per sample, the sample's sign gradient written straight
// into dec's A4 layout and its float64 sum of |dec - x| reduced as eval_losses_kernel reduces it (each thread its
// strided share of float4 units, then a fixed tree).  group_sums_kernel: one CTA adds each group's m sample sums in
// ascending order, then the groups' sums into the batch total.
//
// avc_code_adam: one CTA of 1024 threads per code.  The code's gradient is the sum of its m demb rows, formed exactly
// as bias_grad_kernel forms a bias gradient at T = 1 (thread j adds rows j, j + 1024, ...; a butterfly within each
// warp; warp partials added in warp order into a zero).  Then the gradient's norm, avc_adam_step's clip coefficient,
// L2 decay and Adam(amsgrad) on the code's C values, and the updated code copied into its m rows of emb.
#include "common.cuh"

namespace avc {

constexpr int GL_THREADS = 512;
constexpr int CA_THREADS = 1024;

__device__ __forceinline__ double fit_block_sum_f64(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x < 32) {
    r = threadIdx.x < GL_THREADS / 32 ? sh[threadIdx.x] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  }
  __syncthreads();
  return r;  // valid on warp 0
}

__device__ __forceinline__ float fit_rna_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// avc_vae_loss's gradient of one element: grec * sign(dec - x), 0 at equality
__device__ __forceinline__ float l1_grad(float dec, float x, float grec, float ngrec, bool rnd) {
  const float df = dec - x;
  const float g = df > 0.f ? grec : (df < 0.f ? ngrec : 0.f);
  return rnd ? fit_rna_tf32(g) : g;
}

__global__ void __launch_bounds__(GL_THREADS) group_l1_kernel(const avc_group_l1_desc d) {
  __shared__ double sh[GL_THREADS / 32];
  const int b = blockIdx.x, T = d.T;
  const float grec = d.hp[0] / (float)((int64_t)d.m * d.C * T);
  const float ngrec = -grec;
  const bool rnd = d.round_tf32 != 0;
  const int64_t units = (int64_t)(d.C / 4) * T;
  const float* dec = d.dec + (int64_t)b * d.C * T;
  const float* x = d.x + (int64_t)b * d.C * T;
  float* ddec = d.ddec + (int64_t)b * d.C * T;
  double rec = 0.0;
#pragma unroll 4
  for (int64_t u = threadIdx.x; u < units; u += GL_THREADS) {
    const int64_t q = u / T, t = u - q * T;
    const float4 v = ldg4(dec + 4 * u);
    const float* xp = x + 4 * q * T + t;
    const float x0 = __ldg(xp), x1 = __ldg(xp + T), x2 = __ldg(xp + 2 * T), x3 = __ldg(xp + 3 * T);
    rec += fabs((double)v.x - (double)x0);
    rec += fabs((double)v.y - (double)x1);
    rec += fabs((double)v.z - (double)x2);
    rec += fabs((double)v.w - (double)x3);
    st4(ddec + 4 * u, make_float4(l1_grad(v.x, x0, grec, ngrec, rnd), l1_grad(v.y, x1, grec, ngrec, rnd),
                                  l1_grad(v.z, x2, grec, ngrec, rnd), l1_grad(v.w, x3, grec, ngrec, rnd)));
  }
  rec = fit_block_sum_f64(rec, sh);
  if (threadIdx.x == 0) d.part[b] = rec;
}

__global__ void __launch_bounds__(256) group_sums_kernel(const avc_group_l1_desc d) {
  const int G = d.B / d.m;
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    double s = 0.0;
    for (int j = 0; j < d.m; ++j) s += d.part[(int64_t)g * d.m + j];
    d.sums[g] = s;
  }
  if (d.total == nullptr) return;
  __syncthreads();  // the block's global writes of sums are visible to the whole block after the barrier
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int g = 0; g < G; ++g) t += d.sums[g];
    d.total[0] = (float)t;
  }
}

__global__ void __launch_bounds__(CA_THREADS) code_adam_kernel(const avc_code_adam_desc d) {
  __shared__ float4 wpart[CA_THREADS / 32][AVC_CODE_MAX_C / 4];
  __shared__ float code_sh[AVC_CODE_MAX_C];
  __shared__ float red[CA_THREADS / 32];
  __shared__ float sq_sh, t_sh;
  const int s = blockIdx.x, C = d.C, m = d.m, nq = d.C / 4;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const float* rows = d.demb + (int64_t)s * m * C;
  if (tid == 0) t_sh = d.steps[s] + 1.f;
  // g_s: bias_grad_kernel's order at T = 1, one 4-channel chunk after the other
  for (int q = 0; q < nq; ++q) {
    float4 v = zero4();
    for (int j = tid; j < m; j += CA_THREADS) {
      const float4 a = ldg4(rows + (int64_t)j * C + 4 * q);
      v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
    }
    v.x = warp_sum(v.x); v.y = warp_sum(v.y); v.z = warp_sum(v.z); v.w = warp_sum(v.w);
    if (lane == 0) wpart[w][q] = v;
  }
  __syncthreads();
  float g = 0.f;
  if (tid < C) {
    const int q = tid >> 2, k = tid & 3;
    float r = 0.f;
    for (int ww = 0; ww < CA_THREADS / 32; ++ww) {
      const float4 p = wpart[ww][q];
      r += k == 0 ? p.x : (k == 1 ? p.y : (k == 2 ? p.z : p.w));
    }
    g += r;   // the zeroed gradient buffer plus the block's sum, as avc_bias_grad adds it
  }
  // sum of squares in a fixed order: each channel's square, the butterfly within a warp, warps in order
  float s2 = warp_sum(tid < C ? g * g : 0.f);
  if (lane == 0) red[w] = s2;
  __syncthreads();
  if (tid == 0) {
    float a = 0.f;
    for (int ww = 0; ww < CA_THREADS / 32; ++ww) a += red[ww];
    sq_sh = a;
  }
  __syncthreads();
  const float* hp = d.hp;
  const float gscale = hp[2], lr = hp[3], b1 = hp[4], b2 = hp[5], eps = hp[6], wd = hp[7], max_norm = hp[8];
  const bool amsgrad = hp[9] != 0.f;
  const float gnorm = gscale * sqrtf(sq_sh);
  if (tid < C) {
    const float coef = fminf(1.f, max_norm / (gnorm + 1e-6f)) * gscale;
    const float t = t_sh;
    const float bc1 = 1.f - powf(b1, t), bc2 = 1.f - powf(b2, t);
    const float step_size = lr / bc1, inv_sqrt_bc2 = rsqrtf(bc2);
    const int64_t i = (int64_t)s * C + tid;
    const float pi = d.codes[i];
    const float gi = fmaf(wd, pi, g * coef);
    const float mi = fmaf(1.f - b1, gi - d.exp_avg[i], d.exp_avg[i]);
    const float vi = fmaf(b2, d.exp_avg_sq[i], (1.f - b2) * gi * gi);
    d.exp_avg[i] = mi;
    d.exp_avg_sq[i] = vi;
    float second = vi;
    if (amsgrad) {
      second = fmaxf(d.max_exp_avg_sq[i], vi);
      d.max_exp_avg_sq[i] = second;
    }
    const float denom = sqrtf(second) * inv_sqrt_bc2 + eps;
    const float pn = pi - step_size * (mi / denom);
    d.codes[i] = pn;
    d.grad[i] = g;
    code_sh[tid] = pn;
  }
  if (tid == 0) {
    d.gnorm[s] = gnorm;
    d.steps[s] = t_sh;
  }
  __syncthreads();
  // the code's m expanded rows for the next step's AdaIN affine layers
  const float4* c4 = reinterpret_cast<const float4*>(code_sh);
  float* emb = d.emb + (int64_t)s * m * C;
  for (int64_t u = tid; u < (int64_t)m * nq; u += CA_THREADS) st4(emb + 4 * u, c4[u % nq]);
}

}  // namespace avc

using namespace avc;

extern "C" int avc_group_l1(const avc_group_l1_desc* d, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "avc_group_l1: null descriptor");
  AVC_REQUIRE(d->dec && d->x && d->hp && d->ddec && d->part && d->sums, AVC_ERR_INVALID,
              "avc_group_l1: null pointer (dec %p, x %p, hp %p, ddec %p, part %p, sums %p)", (const void*)d->dec,
              (const void*)d->x, (const void*)d->hp, (const void*)d->ddec, (const void*)d->part, (const void*)d->sums);
  AVC_REQUIRE(d->B > 0 && d->C > 0 && d->T > 0 && d->m > 0, AVC_ERR_INVALID,
              "avc_group_l1: sizes must be positive (B %d, C %d, T %d, m %d)", d->B, d->C, d->T, d->m);
  AVC_REQUIRE(d->C % 4 == 0 && d->B % d->m == 0, AVC_ERR_INVALID,
              "avc_group_l1: C must be a multiple of 4 and B of m (B %d, C %d, m %d)", d->B, d->C, d->m);
  AVC_LAUNCH(group_l1_kernel, (unsigned)d->B, GL_THREADS, 0, (cudaStream_t)stream, *d);
  AVC_CHECK_LAUNCH("group_l1");
  AVC_LAUNCH(group_sums_kernel, 1, 256, 0, (cudaStream_t)stream, *d);
  AVC_CHECK_LAUNCH("group_sums");
  return AVC_OK;
}

extern "C" int avc_code_adam(const avc_code_adam_desc* d, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "avc_code_adam: null descriptor");
  AVC_REQUIRE(d->demb && d->codes && d->exp_avg && d->exp_avg_sq && d->max_exp_avg_sq && d->steps && d->grad &&
                  d->gnorm && d->emb && d->hp,
              AVC_ERR_INVALID, "avc_code_adam: null pointer");
  AVC_REQUIRE(d->S > 0 && d->m > 0 && d->C > 0 && d->C % 4 == 0 && d->C <= AVC_CODE_MAX_C, AVC_ERR_INVALID,
              "avc_code_adam: need S, m >= 1 and C a multiple of 4 in [4, %d] (S %d, m %d, C %d)", AVC_CODE_MAX_C, d->S,
              d->m, d->C);
  AVC_REQUIRE(((uintptr_t)d->demb | (uintptr_t)d->emb) % 16 == 0, AVC_ERR_INVALID,
              "avc_code_adam: demb and emb must be 16-byte aligned");
  AVC_LAUNCH(code_adam_kernel, (unsigned)d->S, CA_THREADS, 0, (cudaStream_t)stream, *d);
  AVC_CHECK_LAUNCH("code_adam");
  return AVC_OK;
}
