// Layout converters, the small dense layers of the speaker encoder / AdaIN affine heads,
// the VAE reparameterisation, the losses, and the fused clip + Adam(amsgrad) update.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>

#include "common.cuh"

// defaults of the runtime options (avc_set_option).  AVC_TC_ISSUE=legacy / AVC_WGRAD_REDUCE=v1 select the
// round-1 variants.
#ifndef AVC_DEFAULT_TC_UNIFORM_ISSUE
#define AVC_DEFAULT_TC_UNIFORM_ISSUE 1
#endif
#ifndef AVC_DEFAULT_WGRAD_REDUCE_V2
#define AVC_DEFAULT_WGRAD_REDUCE_V2 1
#endif

namespace avc {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// ------------------------------------------------------------------ weight packing
__global__ void pack_weight_kernel(const float* __restrict__ w, float* __restrict__ p, int Cout, int Cin, int K, int mode) {
  const int64_t n = (int64_t)Cout * Cin * K;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    // i indexes the PACKED tensor so that writes are coalesced
    if (mode == AVC_PACK_FWD) {  // P[ci][j][co] = W[co][ci][j]
      const int co = (int)(i % Cout);
      const int64_t r = i / Cout;
      const int j = (int)(r % K), ci = (int)(r / K);
      p[i] = __ldg(w + ((int64_t)co * Cin + ci) * K + j);
    } else {  // P[co][j][ci] = W[co][ci][K-1-j]
      const int ci = (int)(i % Cin);
      const int64_t r = i / Cin;
      const int j = (int)(r % K), co = (int)(r / K);
      p[i] = __ldg(w + ((int64_t)co * Cin + ci) * K + (K - 1 - j));
    }
  }
}

// ------------------------------------------------------------------ planar <-> A4
// 32x32 tile transposes through shared memory would be the classic answer; with only 4
// channels interleaved a direct gather is already coalesced on the wide side: each thread
// builds one float4 (4 channel rows, same t) -- reads are 4 coalesced row segments.
__device__ __forceinline__ float rna_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__global__ void pack_a4_kernel(const float* __restrict__ pl, float* __restrict__ a4, int64_t bstride, int B, int C, int T, int rnd) {
  const int Cq = C >> 2;
  const int64_t n = (int64_t)B * Cq * T;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % T);
    const int64_t bq = i / T;
    const int q = (int)(bq % Cq), b = (int)(bq / Cq);
    const float* src = pl + ((int64_t)b * C + q * 4) * T + t;
    float4 v = make_float4(__ldg(src), __ldg(src + T), __ldg(src + 2 * (int64_t)T), __ldg(src + 3 * (int64_t)T));
    if (rnd) v = make_float4(rna_tf32(v.x), rna_tf32(v.y), rna_tf32(v.z), rna_tf32(v.w));
    st4(a4 + (int64_t)b * bstride + ((int64_t)q * T + t) * 4, v);
  }
}
__global__ void unpack_a4_kernel(const float* __restrict__ a4, int64_t bstride, float* __restrict__ pl, int B, int C, int T) {
  const int Cq = C >> 2;
  const int64_t n = (int64_t)B * Cq * T;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % T);
    const int64_t bq = i / T;
    const int q = (int)(bq % Cq), b = (int)(bq / Cq);
    const float4 v = ldg4(a4 + (int64_t)b * bstride + ((int64_t)q * T + t) * 4);
    float* dst = pl + ((int64_t)b * C + q * 4) * T + t;
    dst[0] = v.x; dst[T] = v.y; dst[2 * (int64_t)T] = v.z; dst[3 * (int64_t)T] = v.w;
  }
}

// ------------------------------------------------------------------ mean over time
__global__ void time_mean_fwd_kernel(const float* __restrict__ a4, int64_t bstride, float* __restrict__ out, int B, int C, int T) {
  const int Cq = C >> 2;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * Cq) return;
  const int b = warp / Cq, q = warp - b * Cq;
  float4 s = zero4();
  for (int t = lane; t < T; t += 32) {
    const float4 v = ldg4(a4 + (int64_t)b * bstride + ((int64_t)q * T + t) * 4);
    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
  }
  s.x = warp_sum(s.x); s.y = warp_sum(s.y); s.z = warp_sum(s.z); s.w = warp_sum(s.w);
  if (lane == 0) {
    const float inv = 1.f / (float)T;
    st4(out + (int64_t)b * C + q * 4, make_float4(s.x * inv, s.y * inv, s.z * inv, s.w * inv));
  }
}
__global__ void time_mean_bwd_kernel(const float* __restrict__ dout, float* __restrict__ da4, int64_t bstride, int B, int C, int T) {
  const int Cq = C >> 2;
  const int64_t n = (int64_t)B * Cq * T;
  const float inv = 1.f / (float)T;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % T);
    const int64_t bq = i / T;
    const int q = (int)(bq % Cq), b = (int)(bq / Cq);
    float4 v = ldg4(dout + (int64_t)b * C + q * 4);
    v.x *= inv; v.y *= inv; v.z *= inv; v.w *= inv;
    st4(da4 + (int64_t)b * bstride + ((int64_t)q * T + t) * 4, v);
  }
}

// ------------------------------------------------------------------ small linear layers
// block = 32 (n or k) x 8 (rows); tiles of 32 along the reduction dim staged in smem.
__global__ void __launch_bounds__(256) linear_fwd_kernel(const avc_linear_desc d) {
  __shared__ float xs[8][33];
  __shared__ float ws[32][33];
  const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
  const int n0 = blockIdx.x * 32, b0 = blockIdx.y * 8;
  float acc = 0.f;
  for (int k0 = 0; k0 < d.K; k0 += 32) {
    {
      const int b = b0 + ly, k = k0 + lx;
      xs[ly][lx] = (b < d.B && k < d.K) ? __ldg(d.x + (int64_t)b * d.x_bstride + k) : 0.f;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int n = n0 + ly + 8 * r, k = k0 + lx;
      ws[ly + 8 * r][lx] = (n < d.N && k < d.K) ? __ldg(d.w + (int64_t)n * d.K + k) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 32; ++kk) acc = fmaf(xs[ly][kk], ws[lx][kk], acc);
    __syncthreads();
  }
  const int b = b0 + ly, n = n0 + lx;
  if (b < d.B && n < d.N) {
    if (d.bias) acc += __ldg(d.bias + n);
    if (d.relu) acc = fmaxf(acc, 0.f);
    if (d.y_act) d.y_act[(int64_t)b * d.N + n] = acc;
    if (d.res) acc += __ldg(d.res + (int64_t)b * d.N + n);
    d.out[(int64_t)b * d.out_bstride + n] = acc;
  }
}

__device__ __forceinline__ float masked_dy(const avc_linear_desc& d, int b, int n) {
  float g = __ldg(d.dy + (int64_t)b * d.dy_bstride + n);
  if (d.relu && !(__ldg(d.y_act + (int64_t)b * d.N + n) > 0.f)) g = 0.f;
  return g;
}

// dx[b][k] = sum_n g[b][n] W[n][k] (+ dx_add)
__global__ void __launch_bounds__(256) linear_bwd_dx_kernel(const avc_linear_desc d) {
  __shared__ float gs[8][33];
  __shared__ float ws[32][33];
  const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
  const int k0 = blockIdx.x * 32, b0 = blockIdx.y * 8;
  float acc = 0.f;
  for (int n0 = 0; n0 < d.N; n0 += 32) {
    {
      const int b = b0 + ly, n = n0 + lx;
      gs[ly][lx] = (b < d.B && n < d.N) ? masked_dy(d, b, n) : 0.f;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int n = n0 + ly + 8 * r, k = k0 + lx;
      ws[ly + 8 * r][lx] = (n < d.N && k < d.K) ? __ldg(d.w + (int64_t)n * d.K + k) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int nn = 0; nn < 32; ++nn) acc = fmaf(gs[ly][nn], ws[nn][lx], acc);
    __syncthreads();
  }
  const int b = b0 + ly, k = k0 + lx;
  if (b < d.B && k < d.K) {
    if (d.dx_add) acc += __ldg(d.dx_add + (int64_t)b * d.K + k);
    d.dx[(int64_t)b * d.K + k] = acc;
  }
}

// dW[n][k] += sum_b g[b][n] x[b][k];  db[n] += sum_b g[b][n]
__global__ void __launch_bounds__(256) linear_bwd_dw_kernel(const avc_linear_desc d) {
  __shared__ float gs[32][9];   // [b][n]
  __shared__ float xs[32][33];  // [b][k]
  const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
  const int k0 = blockIdx.x * 32, n0 = blockIdx.y * 8;
  float acc = 0.f, bacc = 0.f;
  for (int b0 = 0; b0 < d.B; b0 += 32) {
    {
      const int b = b0 + lx, n = n0 + ly;  // lx walks the batch here
      gs[lx][ly] = (b < d.B && n < d.N) ? masked_dy(d, b, n) : 0.f;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int b = b0 + ly + 8 * r, k = k0 + lx;
      xs[ly + 8 * r][lx] = (b < d.B && k < d.K) ? __ldg(d.x + (int64_t)b * d.x_bstride + k) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int bb = 0; bb < 32; ++bb) {
      acc = fmaf(gs[bb][ly], xs[bb][lx], acc);
      bacc += gs[bb][ly];
    }
    __syncthreads();
  }
  const int n = n0 + ly, k = k0 + lx;
  if (n < d.N && k < d.K) d.dw[(int64_t)n * d.K + k] += acc;
  if (d.db && blockIdx.x == 0 && lx == 0 && n < d.N) d.db[n] += bacc;
}

// ------------------------------------------------------------------ reparameterisation
__global__ void reparam_fwd_kernel(const float* __restrict__ mu4, const float* __restrict__ ls4, const float* __restrict__ eps,
                                   float* __restrict__ mu, float* __restrict__ ls, float* __restrict__ z4, int B, int C, int T) {
  const int Cq = C >> 2;
  const int64_t n = (int64_t)B * Cq * T;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % T);
    const int64_t bq = i / T;
    const int q = (int)(bq % Cq), b = (int)(bq / Cq);
    const float4 m = ldg4(mu4 + i * 4);
    const float4 l = ls4 ? ldg4(ls4 + i * 4) : zero4();
    const int64_t p0 = ((int64_t)b * C + q * 4) * T + t;
    float4 z = m;
    if (eps) {
      z.x = fmaf(expf(0.5f * l.x), __ldg(eps + p0), m.x);
      z.y = fmaf(expf(0.5f * l.y), __ldg(eps + p0 + T), m.y);
      z.z = fmaf(expf(0.5f * l.z), __ldg(eps + p0 + 2 * (int64_t)T), m.z);
      z.w = fmaf(expf(0.5f * l.w), __ldg(eps + p0 + 3 * (int64_t)T), m.w);
    }
    st4(z4 + i * 4, z);
    if (mu) { mu[p0] = m.x; mu[p0 + T] = m.y; mu[p0 + 2 * (int64_t)T] = m.z; mu[p0 + 3 * (int64_t)T] = m.w; }
    if (ls) { ls[p0] = l.x; ls[p0 + T] = l.y; ls[p0 + 2 * (int64_t)T] = l.z; ls[p0 + 3 * (int64_t)T] = l.w; }
  }
}
__global__ void reparam_bwd_kernel(const float* __restrict__ dz4, const float* __restrict__ ls4, const float* __restrict__ eps,
                                   const float* __restrict__ dmu_ext, const float* __restrict__ dls_ext,
                                   float* __restrict__ dmu4, float* __restrict__ dls4, int B, int C, int T) {
  const int Cq = C >> 2;
  const int64_t n = (int64_t)B * Cq * T;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % T);
    const int64_t bq = i / T;
    const int q = (int)(bq % Cq), b = (int)(bq / Cq);
    const int64_t p0 = ((int64_t)b * C + q * 4) * T + t;
    const int64_t Ts = T;
    const float4 dz = dz4 ? ldg4(dz4 + i * 4) : zero4();
    float4 dm = dz, dl = zero4();
    if (eps) {
      const float4 l = ldg4(ls4 + i * 4);
      dl.x = dz.x * __ldg(eps + p0) * 0.5f * expf(0.5f * l.x);
      dl.y = dz.y * __ldg(eps + p0 + Ts) * 0.5f * expf(0.5f * l.y);
      dl.z = dz.z * __ldg(eps + p0 + 2 * Ts) * 0.5f * expf(0.5f * l.z);
      dl.w = dz.w * __ldg(eps + p0 + 3 * Ts) * 0.5f * expf(0.5f * l.w);
    }
    if (dmu_ext) { dm.x += __ldg(dmu_ext + p0); dm.y += __ldg(dmu_ext + p0 + Ts); dm.z += __ldg(dmu_ext + p0 + 2 * Ts); dm.w += __ldg(dmu_ext + p0 + 3 * Ts); }
    if (dls_ext) { dl.x += __ldg(dls_ext + p0); dl.y += __ldg(dls_ext + p0 + Ts); dl.z += __ldg(dls_ext + p0 + 2 * Ts); dl.w += __ldg(dls_ext + p0 + 3 * Ts); }
    st4(dmu4 + i * 4, dm);
    st4(dls4 + i * 4, dl);
  }
}

// ------------------------------------------------------------------ losses
__device__ __forceinline__ float block_sum_256(float v, float* sh) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x < 32) {
    r = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
    r = warp_sum(r);
  }
  __syncthreads();
  return r;  // valid on warp 0
}

__global__ void __launch_bounds__(256) vae_loss_kernel(const float* __restrict__ dec, const float* __restrict__ x, int64_t n_rec,
                                                       const float* __restrict__ mu, const float* __restrict__ ls, int64_t n_lat,
                                                       const float* __restrict__ hp, float* __restrict__ part,
                                                       float* __restrict__ ddec, float* __restrict__ dmu, float* __restrict__ dls) {
  __shared__ float sh[8];
  const float lrec = hp[0], lkl = hp[1];
  const float grec = lrec / (float)n_rec, gkl = lkl / (float)n_lat;
  float s_rec = 0.f, s_kl = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rec; i += stride) {
    const float df = dec[i] - x[i];
    s_rec += fabsf(df);
    if (ddec) ddec[i] = df > 0.f ? grec : (df < 0.f ? -grec : 0.f);
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_lat; i += stride) {
    const float m = mu[i], l = ls[i];
    const float e = expf(l);
    s_kl += e + m * m - 1.f - l;
    if (dmu) dmu[i] = gkl * m;
    if (dls) dls[i] = gkl * 0.5f * (e - 1.f);
  }
  const float r = block_sum_256(s_rec, sh);
  const float k = block_sum_256(s_kl, sh);
  if (threadIdx.x == 0) {
    part[2 * blockIdx.x + 0] = r;
    part[2 * blockIdx.x + 1] = k;
  }
}

// sums[j] = the nb block partials part[2 i + j] added in block order
__global__ void vae_sums_kernel(const float* __restrict__ part, int nb, float* __restrict__ sums) {
  if (threadIdx.x >= 2) return;
  float s = 0.f;
  for (int i = 0; i < nb; ++i) s += part[2 * i + threadIdx.x];
  sums[threadIdx.x] = s;
}

// ------------------------------------------------------------------ grad norm + Adam
__global__ void __launch_bounds__(256) sqnorm_stage1(const float* __restrict__ g, int64_t n, float* __restrict__ scratch) {
  __shared__ float sh[8];
  float s = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = g[i];
    s = fmaf(v, v, s);
  }
  const float r = block_sum_256(s, sh);
  if (threadIdx.x == 0) scratch[blockIdx.x] = r;
}
__global__ void __launch_bounds__(256) sqnorm_stage2(const float* __restrict__ scratch, int nb, float* __restrict__ out) {
  __shared__ float sh[8];
  float s = 0.f;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) s += scratch[i];
  const float r = block_sum_256(s, sh);
  if (threadIdx.x == 0) out[0] = r;
}

__global__ void step_inc_kernel(float* step) {
  step[0] += 1.f;
}

__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, float* __restrict__ vmax, int64_t n,
                                                   const float* __restrict__ hp, const float* __restrict__ sqnorm,
                                                   const float* __restrict__ step) {
  const float gscale = hp[2], lr = hp[3], b1 = hp[4], b2 = hp[5], eps = hp[6], wd = hp[7], max_norm = hp[8];
  const bool amsgrad = hp[9] != 0.f;
  const float gnorm = gscale * sqrtf(sqnorm[0]);
  const float coef = fminf(1.f, max_norm / (gnorm + 1e-6f)) * gscale;
  const float t = step[0];
  const float bc1 = 1.f - powf(b1, t), bc2 = 1.f - powf(b2, t);
  const float step_size = lr / bc1, inv_sqrt_bc2 = rsqrtf(bc2);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float pi = p[i];
    const float gi = fmaf(wd, pi, g[i] * coef);
    const float mi = fmaf(1.f - b1, gi - m[i], m[i]);  // lerp, as torch's exp_avg.lerp_(grad, 1-beta1)
    const float vi = fmaf(b2, v[i], (1.f - b2) * gi * gi);
    m[i] = mi;
    v[i] = vi;
    float second = vi;
    if (amsgrad) {
      second = fmaxf(vmax[i], vi);
      vmax[i] = second;
    }
    const float denom = sqrtf(second) * inv_sqrt_bc2 + eps;
    p[i] = pi - step_size * (mi / denom);
  }
}

static int ew_blocks(int64_t n) {
  int64_t b = cdiv64(n, 256);
  if (b > 132 * 8) b = 132 * 8;   // AVC_VAE_PARTIALS = 2 x this
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace avc

namespace avc {
// ---- runtime options: -1 = not read yet (environment default on first use)
struct Option {
  const char* name;
  const char* env;
  const char* on;   // environment value that enables
  const char* off;  // environment value that disables
  int dflt;
  int value;
};
static Option g_opts[] = {
    {"tc_uniform_issue", "AVC_TC_ISSUE", "uniform", "legacy", AVC_DEFAULT_TC_UNIFORM_ISSUE, -1},
    {"wgrad_reduce_v2", "AVC_WGRAD_REDUCE", "v2", "v1", AVC_DEFAULT_WGRAD_REDUCE_V2, -1},
    {"tc_conv_v2", "AVC_TC_CONV", "v2", "v1", 1, -1},   // persistent conv block kernel (conv_tc2.cu); v1 = conv_tc.cu
    {"wgrad_split", "AVC_WGRAD_KERNEL", "split", "r1", 1, -1},   // weight gradient with a dedicated MMA warp (conv_wgrad_split_kernel)
};
static int opt_value(int i) {
  Option& o = g_opts[i];
  if (o.value < 0) {
    const char* e = getenv(o.env);
    o.value = o.dflt;
    if (e && !strcmp(e, o.on)) o.value = 1;
    if (e && !strcmp(e, o.off)) o.value = 0;
  }
  return o.value;
}
int opt_tc_uniform_issue() { return opt_value(0); }
int opt_wgrad_reduce_v2() { return opt_value(1); }
int opt_tc_conv_v2() { return opt_value(2); }
int opt_wgrad_split() { return opt_value(3); }
}  // namespace avc
extern "C" int avc_set_option(const char* name, int value) {
  if (name)
    for (auto& o : avc::g_opts)
      if (!strcmp(o.name, name)) {
        o.value = value ? 1 : 0;
        return AVC_OK;
      }
  avc::set_error("avc_set_option: unknown option '%s'", name ? name : "(null)");
  return AVC_ERR_INVALID;
}
extern "C" int avc_get_option(const char* name) {
  if (name)
    for (int i = 0; i < (int)(sizeof(avc::g_opts) / sizeof(avc::g_opts[0])); ++i)
      if (!strcmp(avc::g_opts[i].name, name)) return avc::opt_value(i);
  return -1;
}

using namespace avc;

extern "C" const char* avc_last_error(void) { return g_err; }
extern "C" const char* avc_build_info(void) {
  return "libavc_b200 sm_90a (compute_90a) fp32-ffma + wgmma paths";
}
extern "C" int64_t avc_launch_count(void) { return (int64_t)g_launches.load(); }

extern "C" int avc_fill_zero(void* ptr, int64_t bytes, void* stream) {
  AVC_REQUIRE(ptr && bytes >= 0, AVC_ERR_INVALID, "avc_fill_zero: bad argument");
  cudaError_t e = cudaMemsetAsync(ptr, 0, (size_t)bytes, (cudaStream_t)stream);
  if (e != cudaSuccess) {
    set_error("avc_fill_zero: %s", cudaGetErrorString(e));
    return AVC_ERR_CUDA;
  }
  return AVC_OK;
}

extern "C" int avc_pack_conv_weight(const float* w, float* packed, int Cout, int Cin, int K, int mode, void* stream) {
  AVC_REQUIRE(w && packed && Cout > 0 && Cin > 0 && K > 0, AVC_ERR_INVALID, "avc_pack_conv_weight: bad argument");
  AVC_REQUIRE(mode == AVC_PACK_FWD || mode == AVC_PACK_DGRAD, AVC_ERR_INVALID, "avc_pack_conv_weight: bad mode");
  AVC_LAUNCH(pack_weight_kernel, ew_blocks((int64_t)Cout * Cin * K), 256, 0, (cudaStream_t)stream, w, packed, Cout, Cin, K, mode);
  AVC_CHECK_LAUNCH("pack_conv_weight");
  return AVC_OK;
}

extern "C" int avc_pack_a4(const float* planar, float* a4, int64_t a4_bstride, int B, int C, int T, int round_tf32, void* stream) {
  AVC_REQUIRE(planar && a4 && B > 0 && C > 0 && C % 4 == 0 && T > 0, AVC_ERR_INVALID, "avc_pack_a4: bad argument (C %% 4 must be 0)");
  AVC_LAUNCH(pack_a4_kernel, ew_blocks((int64_t)B * (C / 4) * T), 256, 0, (cudaStream_t)stream, planar, a4, a4_bstride, B, C, T, round_tf32);
  AVC_CHECK_LAUNCH("pack_a4");
  return AVC_OK;
}
extern "C" int avc_unpack_a4(const float* a4, int64_t a4_bstride, float* planar, int B, int C, int T, void* stream) {
  AVC_REQUIRE(planar && a4 && B > 0 && C > 0 && C % 4 == 0 && T > 0, AVC_ERR_INVALID, "avc_unpack_a4: bad argument (C %% 4 must be 0)");
  AVC_LAUNCH(unpack_a4_kernel, ew_blocks((int64_t)B * (C / 4) * T), 256, 0, (cudaStream_t)stream, a4, a4_bstride, planar, B, C, T);
  AVC_CHECK_LAUNCH("unpack_a4");
  return AVC_OK;
}

extern "C" int avc_time_mean_fwd(const float* a4, int64_t bstride, float* out, int B, int C, int T, void* stream) {
  AVC_REQUIRE(a4 && out && B > 0 && C > 0 && C % 4 == 0 && T > 0, AVC_ERR_INVALID, "avc_time_mean_fwd: bad argument");
  const int64_t warps = (int64_t)B * (C / 4);
  AVC_LAUNCH(time_mean_fwd_kernel, (int)cdiv64(warps * 32, 256), 256, 0, (cudaStream_t)stream, a4, bstride, out, B, C, T);
  AVC_CHECK_LAUNCH("time_mean_fwd");
  return AVC_OK;
}
extern "C" int avc_time_mean_bwd(const float* dout, float* da4, int64_t bstride, int B, int C, int T, void* stream) {
  AVC_REQUIRE(dout && da4 && B > 0 && C > 0 && C % 4 == 0 && T > 0, AVC_ERR_INVALID, "avc_time_mean_bwd: bad argument");
  AVC_LAUNCH(time_mean_bwd_kernel, ew_blocks((int64_t)B * (C / 4) * T), 256, 0, (cudaStream_t)stream, dout, da4, bstride, B, C, T);
  AVC_CHECK_LAUNCH("time_mean_bwd");
  return AVC_OK;
}

extern "C" int avc_linear_fwd(const avc_linear_desc* d, void* stream) {
  AVC_REQUIRE(d && d->x && d->w && d->out && d->B > 0 && d->N > 0 && d->K > 0, AVC_ERR_INVALID, "avc_linear_fwd: bad argument");
  dim3 grid(cdiv(d->N, 32), cdiv(d->B, 8));
  AVC_LAUNCH(linear_fwd_kernel, grid, 256, 0, (cudaStream_t)stream, *d);
  AVC_CHECK_LAUNCH("linear_fwd");
  return AVC_OK;
}
extern "C" int avc_linear_bwd(const avc_linear_desc* d, void* stream) {
  AVC_REQUIRE(d && d->x && d->w && d->dy && d->dw && d->B > 0 && d->N > 0 && d->K > 0, AVC_ERR_INVALID, "avc_linear_bwd: bad argument");
  AVC_REQUIRE(!d->relu || d->y_act, AVC_ERR_INVALID, "avc_linear_bwd: relu needs y_act");
  if (d->dx) {
    dim3 grid(cdiv(d->K, 32), cdiv(d->B, 8));
    AVC_LAUNCH(linear_bwd_dx_kernel, grid, 256, 0, (cudaStream_t)stream, *d);
    AVC_CHECK_LAUNCH("linear_bwd_dx");
  }
  dim3 grid2(cdiv(d->K, 32), cdiv(d->N, 8));
  AVC_LAUNCH(linear_bwd_dw_kernel, grid2, 256, 0, (cudaStream_t)stream, *d);
  AVC_CHECK_LAUNCH("linear_bwd_dw");
  return AVC_OK;
}

extern "C" int avc_reparam_fwd(const float* mu4, const float* ls4, const float* eps, float* mu, float* ls, float* z4,
                               int B, int C, int T, void* stream) {
  AVC_REQUIRE(mu4 && z4 && B > 0 && C > 0 && C % 4 == 0 && T > 0, AVC_ERR_INVALID, "avc_reparam_fwd: bad argument");
  AVC_REQUIRE(!eps || ls4, AVC_ERR_INVALID, "avc_reparam_fwd: eps needs log_sigma");
  AVC_REQUIRE(!ls || ls4, AVC_ERR_INVALID, "avc_reparam_fwd: ls output needs ls4");
  AVC_LAUNCH(reparam_fwd_kernel, ew_blocks((int64_t)B * (C / 4) * T), 256, 0, (cudaStream_t)stream, mu4, ls4, eps, mu, ls, z4, B, C, T);
  AVC_CHECK_LAUNCH("reparam_fwd");
  return AVC_OK;
}
extern "C" int avc_reparam_bwd(const float* dz4, const float* ls4, const float* eps, const float* dmu_ext, const float* dls_ext,
                               float* dmu4, float* dls4, int B, int C, int T, void* stream) {
  AVC_REQUIRE(dmu4 && dls4 && B > 0 && C > 0 && C % 4 == 0 && T > 0, AVC_ERR_INVALID, "avc_reparam_bwd: bad argument");
  AVC_REQUIRE(!eps || ls4, AVC_ERR_INVALID, "avc_reparam_bwd: eps needs log_sigma");
  AVC_LAUNCH(reparam_bwd_kernel, ew_blocks((int64_t)B * (C / 4) * T), 256, 0, (cudaStream_t)stream, dz4, ls4, eps, dmu_ext, dls_ext, dmu4, dls4, B, C, T);
  AVC_CHECK_LAUNCH("reparam_bwd");
  return AVC_OK;
}

extern "C" int avc_vae_loss(const float* dec, const float* x, int64_t n_rec, const float* mu, const float* ls, int64_t n_lat,
                            const float* hp, float* sums, float* part, float* ddec, float* dmu, float* dls, void* stream) {
  AVC_REQUIRE(dec && x && mu && ls && hp && sums && part && n_rec > 0 && n_lat > 0, AVC_ERR_INVALID, "avc_vae_loss: bad argument");
  const int nb = ew_blocks(n_rec);
  AVC_LAUNCH(vae_loss_kernel, nb, 256, 0, (cudaStream_t)stream, dec, x, n_rec, mu, ls, n_lat, hp, part, ddec, dmu, dls);
  AVC_CHECK_LAUNCH("vae_loss");
  AVC_LAUNCH(vae_sums_kernel, 1, 32, 0, (cudaStream_t)stream, part, nb, sums);
  AVC_CHECK_LAUNCH("vae_sums");
  return AVC_OK;
}

extern "C" int avc_sqnorm(const float* g, int64_t n, float* scratch, float* out, void* stream) {
  AVC_REQUIRE(g && scratch && out && n > 0, AVC_ERR_INVALID, "avc_sqnorm: bad argument");
  int nb = ew_blocks(n);
  if (nb > 1024) nb = 1024;
  AVC_LAUNCH(sqnorm_stage1, nb, 256, 0, (cudaStream_t)stream, g, n, scratch);
  AVC_CHECK_LAUNCH("sqnorm_stage1");
  AVC_LAUNCH(sqnorm_stage2, 1, 256, 0, (cudaStream_t)stream, scratch, nb, out);
  AVC_CHECK_LAUNCH("sqnorm_stage2");
  return AVC_OK;
}

extern "C" int avc_adam_step(float* p, const float* g, float* m, float* v, float* vmax, int64_t n, const float* hp,
                             const float* sqnorm, float* step, void* stream) {
  AVC_REQUIRE(p && g && m && v && vmax && hp && sqnorm && step && n > 0, AVC_ERR_INVALID, "avc_adam_step: bad argument");
  AVC_LAUNCH(step_inc_kernel, 1, 1, 0, (cudaStream_t)stream, step);
  AVC_CHECK_LAUNCH("step_inc");
  AVC_LAUNCH(adam_kernel, ew_blocks(n), 256, 0, (cudaStream_t)stream, p, g, m, v, vmax, n, hp, sqnorm, step);
  AVC_CHECK_LAUNCH("adam");
  return AVC_OK;
}
