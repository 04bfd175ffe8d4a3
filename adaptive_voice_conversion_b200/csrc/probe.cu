// Speaker-classifier probes (speaker_probe.py): the valid latent frames of a padded batch as rows, the standardisation
// of a probe's inputs, its softmax cross-entropy with gradient and rank, and the per-utterance vote of a frame probe.
// The probe's linear layers and its Adam update are avc_linear_fwd / avc_linear_bwd and avc_sqnorm / avc_adam_step.
//
// avc_probe_frames: a 32 x 32 (t, c) tile per CTA, transposed through shared memory so that both the planar read and the
// row-major write are coalesced.
// avc_probe_moments: one thread per dimension walks every row twice in ascending order (mean, then squared deviations).
// avc_probe_xent: one warp per row; lane-strided float64 partial sums of exp(z - max) combined by a fixed xor tree, so
// a row's result does not depend on the rest of the launch.  The loss sum is two-stage (per-CTA partials, then one CTA)
// over a grid fixed by the row count, as avc_sqnorm reduces.
// avc_probe_vote: one CTA per utterance; a row's log-sum-exp is two block reductions, the class scores accumulate in
// shared memory in ascending row order.
// Every float64 operation is an explicitly rounded intrinsic (no contraction into an FMA); no atomics anywhere.
#include "common.cuh"

namespace avc {

constexpr int PROBE_THREADS = 256;
constexpr int PROBE_WARPS = PROBE_THREADS / 32;
constexpr int PROBE_SUM_BLOCKS = 1024;   // avc_probe_xent's scratch holds this many partial sums

__device__ __forceinline__ double nan64() { return __longlong_as_double(0x7ff8000000000000ll); }

__device__ __forceinline__ double warp_sum64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max32(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int warp_sum_int(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide reductions over PROBE_THREADS threads (every thread gets the result); `sh` holds PROBE_WARPS entries
__device__ __forceinline__ double block_sum64(double v, double* sh) {
  v = warp_sum64(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int w = 0; w < PROBE_WARPS; ++w) s = __dadd_rn(s, sh[w]);
  return s;
}
__device__ __forceinline__ float block_max32(float v, float* sh) {
  v = warp_max32(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float m = sh[0];
#pragma unroll
  for (int w = 1; w < PROBE_WARPS; ++w) m = fmaxf(m, sh[w]);
  return m;
}
__device__ __forceinline__ int block_sum_int(int v, int* sh) {
  v = warp_sum_int(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  int s = 0;
#pragma unroll
  for (int w = 0; w < PROBE_WARPS; ++w) s += sh[w];
  return s;
}

// ---------------------------------------------------------------- frame rows
__global__ void __launch_bounds__(PROBE_THREADS) probe_frames_kernel(const float* __restrict__ x, int C, int T,
                                                                     const int32_t* __restrict__ lens,
                                                                     const int64_t* __restrict__ row_off,
                                                                     float* __restrict__ out) {
  __shared__ float tile[32][33];   // [c][t]
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int L = __ldg(lens + b);
  if (L < 0 || L > T || t0 >= L) return;   // the whole CTA leaves together: no barrier is skipped by a part of it
  const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
  const float* xb = x + (int64_t)b * C * T;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int c = c0 + ly + 8 * r, t = t0 + lx;
    if (c < C && t < L) tile[ly + 8 * r][lx] = __ldg(xb + (int64_t)c * T + t);
  }
  __syncthreads();
  const int64_t off = __ldg(row_off + b);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int t = t0 + ly + 8 * r, c = c0 + lx;
    if (c < C && t < L) out[(off + t) * C + c] = tile[lx][ly + 8 * r];
  }
}

// ---------------------------------------------------------------- standardisation
__global__ void __launch_bounds__(PROBE_THREADS) probe_moments_kernel(const float* __restrict__ x, int64_t rows, int D,
                                                                      double* __restrict__ mean, double* __restrict__ std) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  const float* p = x + d;
  double s = 0.0;
  for (int64_t r = 0; r < rows; ++r) s = __dadd_rn(s, (double)__ldg(p + r * D));
  const double m = __ddiv_rn(s, (double)rows);
  double v = 0.0;
  for (int64_t r = 0; r < rows; ++r) {
    const double e = __dsub_rn((double)__ldg(p + r * D), m);
    v = __dadd_rn(v, __dmul_rn(e, e));
  }
  const double sd = __dsqrt_rn(__ddiv_rn(v, (double)rows));
  mean[d] = m;
  std[d] = sd == 0.0 ? 1.0 : sd;
}

__global__ void __launch_bounds__(PROBE_THREADS) probe_standardize_kernel(const float* __restrict__ x,
                                                                          const int64_t* __restrict__ index, int64_t rows,
                                                                          int D, const double* __restrict__ mean,
                                                                          const double* __restrict__ std,
                                                                          float* __restrict__ out) {
  const int64_t n = rows * D;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / D;
    const int d = (int)(i - r * D);
    const int64_t src = index ? __ldg(index + r) : r;
    out[i] = (float)__ddiv_rn(__dsub_rn((double)__ldg(x + src * D + d), __ldg(mean + d)), __ldg(std + d));
  }
}

// ---------------------------------------------------------------- cross-entropy
__global__ void __launch_bounds__(PROBE_THREADS) probe_xent_kernel(const float* __restrict__ logits,
                                                                   const int32_t* __restrict__ labels, int R, int S,
                                                                   float scale, double* __restrict__ loss,
                                                                   float* __restrict__ dlogits, int32_t* __restrict__ rank) {
  const int row = blockIdx.x * PROBE_WARPS + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= R) return;   // whole warps leave: the shuffles below see full warps
  const float* z = logits + (int64_t)row * S;
  const int y = __ldg(labels + row);
  if (y < 0 || y >= S) {
    for (int j = lane; j < S; j += 32)
      if (dlogits) dlogits[(int64_t)row * S + j] = 0.f;
    if (lane == 0) {
      loss[row] = nan64();
      rank[row] = -1;
    }
    return;
  }
  const float zy = __ldg(z + y);
  float m = -INFINITY;
  for (int j = lane; j < S; j += 32) m = fmaxf(m, __ldg(z + j));
  m = warp_max32(m);
  const double md = (double)m;
  double s = 0.0;
  int above = 0;
  for (int j = lane; j < S; j += 32) {
    const float zj = __ldg(z + j);
    s = __dadd_rn(s, exp(__dsub_rn((double)zj, md)));
    above += (zj > zy) || (zj == zy && j < y);
  }
  s = warp_sum64(s);
  above = warp_sum_int(above);
  if (dlogits) {
    const double sc = (double)scale;
    for (int j = lane; j < S; j += 32) {
      const double p = __ddiv_rn(exp(__dsub_rn((double)__ldg(z + j), md)), s);
      dlogits[(int64_t)row * S + j] = (float)__dmul_rn(j == y ? __dsub_rn(p, 1.0) : p, sc);
    }
  }
  if (lane == 0) {
    loss[row] = __dsub_rn(__dadd_rn(md, log(s)), (double)zy);
    rank[row] = above;
  }
}

__global__ void __launch_bounds__(PROBE_THREADS) probe_sum_stage1(const double* __restrict__ v, int n,
                                                                  double* __restrict__ part) {
  __shared__ double sh[PROBE_WARPS];
  double s = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) s = __dadd_rn(s, v[i]);
  s = block_sum64(s, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}
__global__ void __launch_bounds__(PROBE_THREADS) probe_sum_stage2(const double* __restrict__ part, int nb,
                                                                  double* __restrict__ out) {
  __shared__ double sh[PROBE_WARPS];
  double s = 0.0;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) s = __dadd_rn(s, part[i]);
  s = block_sum64(s, sh);
  if (threadIdx.x == 0) out[0] = s;
}

// ---------------------------------------------------------------- frame votes
__global__ void __launch_bounds__(PROBE_THREADS) probe_vote_kernel(const float* __restrict__ logits, int S,
                                                                   const int64_t* __restrict__ off,
                                                                   const int32_t* __restrict__ labels,
                                                                   double* __restrict__ scores,
                                                                   int32_t* __restrict__ rank) {
  __shared__ double acc[AVC_PROBE_MAX_CLASSES];
  __shared__ double shd[PROBE_WARPS];
  __shared__ float shf[PROBE_WARPS];
  __shared__ int shi[PROBE_WARPS];
  const int u = blockIdx.x;
  for (int j = threadIdx.x; j < S; j += PROBE_THREADS) acc[j] = 0.0;
  const int64_t r0 = __ldg(off + u), r1 = __ldg(off + u + 1);
  for (int64_t r = r0; r < r1; ++r) {
    const float* z = logits + r * S;
    float m = -INFINITY;
    for (int j = threadIdx.x; j < S; j += PROBE_THREADS) m = fmaxf(m, __ldg(z + j));
    const double md = (double)block_max32(m, shf);
    double s = 0.0;
    for (int j = threadIdx.x; j < S; j += PROBE_THREADS) s = __dadd_rn(s, exp(__dsub_rn((double)__ldg(z + j), md)));
    const double ls = log(block_sum64(s, shd));
    for (int j = threadIdx.x; j < S; j += PROBE_THREADS)
      acc[j] = __dadd_rn(acc[j], __dsub_rn(__dsub_rn((double)__ldg(z + j), md), ls));
  }
  __syncthreads();
  double* o = scores + (int64_t)u * S;
  for (int j = threadIdx.x; j < S; j += PROBE_THREADS) o[j] = acc[j];
  const int y = __ldg(labels + u);
  const bool valid = y >= 0 && y < S;
  const double ay = valid ? acc[y] : 0.0;
  int above = 0;
  if (valid)
    for (int j = threadIdx.x; j < S; j += PROBE_THREADS) above += (acc[j] > ay) || (acc[j] == ay && j < y);
  above = block_sum_int(above, shi);
  if (threadIdx.x == 0) rank[u] = valid ? above : -1;
}

static int probe_blocks(int64_t n) {
  int64_t b = cdiv64(n, PROBE_THREADS);
  if (b > 132 * 16) b = 132 * 16;
  return b < 1 ? 1 : (int)b;
}

}  // namespace avc

using namespace avc;

extern "C" int avc_probe_frames(const float* x, int B, int C, int T, const int32_t* lengths, const int64_t* row_off,
                                float* out, void* stream) {
  AVC_REQUIRE(x && lengths && row_off && out, AVC_ERR_INVALID,
              "avc_probe_frames: null pointer (x %p, lengths %p, row_off %p, out %p)", (const void*)x,
              (const void*)lengths, (const void*)row_off, (const void*)out);
  AVC_REQUIRE(B > 0 && C > 0 && T > 0, AVC_ERR_INVALID, "avc_probe_frames: sizes must be positive (B %d, C %d, T %d)", B,
              C, T);
  AVC_REQUIRE(B <= 65535, AVC_ERR_UNSUPPORTED, "avc_probe_frames: B %d exceeds 65535", B);
  dim3 grid(cdiv(T, 32), cdiv(C, 32), B);
  AVC_LAUNCH(probe_frames_kernel, grid, PROBE_THREADS, 0, (cudaStream_t)stream, x, C, T, lengths, row_off, out);
  AVC_CHECK_LAUNCH("probe_frames");
  return AVC_OK;
}

extern "C" int avc_probe_moments(const float* x, int64_t rows, int D, double* mean, double* std, void* stream) {
  AVC_REQUIRE(x && mean && std, AVC_ERR_INVALID, "avc_probe_moments: null pointer (x %p, mean %p, std %p)",
              (const void*)x, (const void*)mean, (const void*)std);
  AVC_REQUIRE(rows > 0 && D > 0, AVC_ERR_INVALID, "avc_probe_moments: sizes must be positive (rows %lld, D %d)",
              (long long)rows, D);
  AVC_LAUNCH(probe_moments_kernel, cdiv(D, PROBE_THREADS), PROBE_THREADS, 0, (cudaStream_t)stream, x, rows, D, mean, std);
  AVC_CHECK_LAUNCH("probe_moments");
  return AVC_OK;
}

extern "C" int avc_probe_standardize(const float* x, const int64_t* index, int64_t rows, int D, const double* mean,
                                     const double* std, float* out, void* stream) {
  AVC_REQUIRE(x && mean && std && out, AVC_ERR_INVALID,
              "avc_probe_standardize: null pointer (x %p, mean %p, std %p, out %p)", (const void*)x, (const void*)mean,
              (const void*)std, (const void*)out);
  AVC_REQUIRE(rows > 0 && D > 0, AVC_ERR_INVALID, "avc_probe_standardize: sizes must be positive (rows %lld, D %d)",
              (long long)rows, D);
  AVC_LAUNCH(probe_standardize_kernel, probe_blocks(rows * D), PROBE_THREADS, 0, (cudaStream_t)stream, x, index, rows, D,
             mean, std, out);
  AVC_CHECK_LAUNCH("probe_standardize");
  return AVC_OK;
}

extern "C" int avc_probe_xent(const float* logits, const int32_t* labels, int R, int S, float scale, double* loss,
                              float* dlogits, int32_t* rank, double* scratch, double* loss_sum, void* stream) {
  AVC_REQUIRE(logits && labels && loss && rank, AVC_ERR_INVALID,
              "avc_probe_xent: null pointer (logits %p, labels %p, loss %p, rank %p)", (const void*)logits,
              (const void*)labels, (const void*)loss, (const void*)rank);
  AVC_REQUIRE(!scratch == !loss_sum, AVC_ERR_INVALID, "avc_probe_xent: scratch and loss_sum go together (%p, %p)",
              (const void*)scratch, (const void*)loss_sum);
  AVC_REQUIRE(R > 0 && S > 0, AVC_ERR_INVALID, "avc_probe_xent: sizes must be positive (R %d, S %d)", R, S);
  AVC_REQUIRE(S <= AVC_PROBE_MAX_CLASSES, AVC_ERR_UNSUPPORTED, "avc_probe_xent: S %d exceeds %d", S,
              AVC_PROBE_MAX_CLASSES);
  AVC_LAUNCH(probe_xent_kernel, cdiv(R, PROBE_WARPS), PROBE_THREADS, 0, (cudaStream_t)stream, logits, labels, R, S, scale,
             loss, dlogits, rank);
  AVC_CHECK_LAUNCH("probe_xent");
  if (loss_sum) {
    const int nb = cdiv(R, PROBE_THREADS) < PROBE_SUM_BLOCKS ? cdiv(R, PROBE_THREADS) : PROBE_SUM_BLOCKS;
    AVC_LAUNCH(probe_sum_stage1, nb, PROBE_THREADS, 0, (cudaStream_t)stream, loss, R, scratch);
    AVC_CHECK_LAUNCH("probe_sum_stage1");
    AVC_LAUNCH(probe_sum_stage2, 1, PROBE_THREADS, 0, (cudaStream_t)stream, scratch, nb, loss_sum);
    AVC_CHECK_LAUNCH("probe_sum_stage2");
  }
  return AVC_OK;
}

extern "C" int avc_probe_vote(const float* logits, int S, const int64_t* off, int U, const int32_t* labels,
                              double* scores, int32_t* rank, void* stream) {
  AVC_REQUIRE(logits && off && labels && scores && rank, AVC_ERR_INVALID,
              "avc_probe_vote: null pointer (logits %p, off %p, labels %p, scores %p, rank %p)", (const void*)logits,
              (const void*)off, (const void*)labels, (const void*)scores, (const void*)rank);
  AVC_REQUIRE(S > 0 && U > 0, AVC_ERR_INVALID, "avc_probe_vote: sizes must be positive (S %d, U %d)", S, U);
  AVC_REQUIRE(S <= AVC_PROBE_MAX_CLASSES, AVC_ERR_UNSUPPORTED, "avc_probe_vote: S %d exceeds %d", S,
              AVC_PROBE_MAX_CLASSES);
  AVC_LAUNCH(probe_vote_kernel, U, PROBE_THREADS, 0, (cudaStream_t)stream, logits, S, off, labels, scores, rank);
  AVC_CHECK_LAUNCH("probe_vote");
  return AVC_OK;
}
