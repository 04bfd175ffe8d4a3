// Mel-cepstral distortion of converted utterances (mcd.py): the cepstrum of every frame and the DTW of a batch of
// cepstrum pairs.
//
// avc_mel_cepstrum: rows are independent.  A CTA stages the natural-log amplitudes of MC_SMEM / (8 n_mels) rows in
// shared memory as float64, then each thread forms whole coefficients (row, k), adding the n_mels products in
// ascending m.  The order depends only on n_mels, so a row gets the same bits in any batch.
//
// avc_dtw: one CTA per pair walks the anti-diagonals d = i + j of the Tx x Ty grid.  A diagonal's cells are
// independent given the two before it, so its cells are spread over the CTA's threads and one barrier separates two
// diagonals.  Three rotating diagonals of S (float64) and L (int32) live in shared memory, indexed by the position
// along the shorter side (every diagonal has at most min(Tx, Ty) cells).  Both cepstra are staged in shared memory
// with an odd row pitch (conflict-free: the threads of a warp read different rows) when they fit in the launch's
// staging region, and read through L1 otherwise; either way the same values enter the same operations.  Every
// float64 operation is written as an explicitly rounded intrinsic, so nvcc cannot contract a multiply and an add into
// an FMA, and the result equals a float64 restatement that adds in the same order.
#include "common.cuh"

namespace avc {

constexpr int MC_THREADS = 256;
constexpr int MC_SMEM = 32768;            // staged float64 amplitudes per CTA
constexpr int DTW_THREADS = 256;
constexpr int DTW_SMEM_TARGET = 110 * 1024;   // diagonals + staged cepstra: two CTAs per SM
constexpr int DTW_SMEM_LIMIT = 227 * 1024;    // sm_90 opt-in maximum per CTA

__global__ void __launch_bounds__(MC_THREADS) mel_cepstrum_kernel(const avc_cepstrum_desc d, int rows_per_cta) {
  extern __shared__ __align__(16) double ell[];   // [rows_per_cta][n_mels]
  const int N = d.n_mels, D = d.dims;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta;
  const int nr = (int)min((int64_t)rows_per_cta, (int64_t)d.rows - r0);
  const double scale = 2.302585092994045684 / 20.0;   // ln(10) / 20
  const double max_db = d.max_db, ref_db = d.ref_db;
  for (int e = threadIdx.x; e < nr * N; e += MC_THREADS) {
    const int r = e / N, m = e - r * N;
    // the vocoder's MEL_TO_MAG input: denormalised (x std + mean, float32 as numpy computes it), clipped to [0, 1]
    const float a = fminf(fmaxf(__fadd_rn(__fmul_rn(__ldg(d.in + (r0 + r) * N + m), __ldg(d.std + m)), __ldg(d.mean + m)), 0.f), 1.f);
    ell[e] = __dmul_rn(__dadd_rn(__dsub_rn(__dmul_rn((double)a, max_db), max_db), ref_db), scale);
  }
  __syncthreads();
  for (int o = threadIdx.x; o < nr * D; o += MC_THREADS) {
    const int r = o / D, k = o - r * D;
    const double* l = ell + r * N;
    double c = 0.0;
    for (int m = 0; m < N; ++m) c = fma(l[m], __ldg(d.dct + (int64_t)m * D + k), c);
    d.out[(r0 + r) * D + k] = (float)c;
  }
}

// one cell's distance: sqrt of the squared differences added in ascending k, one at a time
__device__ __forceinline__ double cell_dist(const float* x, const float* y, int D) {
  double acc = 0.0;
  for (int k = 0; k < D; ++k) {
    const double t = __dsub_rn((double)x[k], (double)y[k]);
    acc = __dadd_rn(acc, __dmul_rn(t, t));
  }
  return __dsqrt_rn(acc);
}

__global__ void __launch_bounds__(DTW_THREADS) dtw_kernel(const avc_dtw_desc d, int stage_floats) {
  extern __shared__ __align__(16) double sm[];
  const avc_dtw_pair p = d.pairs[blockIdx.x];
  const int Tx = p.tx, Ty = p.ty, D = d.dims, ms = d.max_short;
  if (Tx < 1 || Ty < 1 || min(Tx, Ty) > ms || (int64_t)Tx + Ty > 0x7fffffffll) {   // outside what the launch was sized for: no cell is read or written
    if (threadIdx.x == 0) {
      d.out[2 * blockIdx.x] = __longlong_as_double(0x7ff8000000000000ll);
      d.out[2 * blockIdx.x + 1] = 0.0;
    }
    return;
  }
  double* S = sm;                                  // [3][ms]
  int* Lc = reinterpret_cast<int*>(S + 3 * ms);    // [3][ms]
  float* stage = reinterpret_cast<float*>(Lc + 3 * ms + (3 * ms & 1));
  const float* xs = d.x + p.x_off * D;
  const float* ys = d.y + p.y_off * D;
  int ldx = D, ldy = D;
  const int Dp = D | 1;
  if (((int64_t)Tx + Ty) * Dp <= stage_floats) {
    for (int e = threadIdx.x; e < Tx * D; e += DTW_THREADS) stage[(e / D) * Dp + e % D] = __ldg(xs + e);
    float* sy = stage + Tx * Dp;
    for (int e = threadIdx.x; e < Ty * D; e += DTW_THREADS) sy[(e / D) * Dp + e % D] = __ldg(ys + e);
    xs = stage;
    ys = sy;
    ldx = ldy = Dp;
    __syncthreads();
  }
  const bool by_i = Tx <= Ty;   // cells are indexed by i when X is the shorter side, by j otherwise
  const int nd = Tx + Ty - 1;
  for (int g = 0; g < nd; ++g) {
    double* Sc = S + (g % 3) * ms;
    int* Lcur = Lc + (g % 3) * ms;
    const double* S1 = S + ((g + 2) % 3) * ms;   // diagonal g - 1
    const int* L1 = Lc + ((g + 2) % 3) * ms;
    const double* S2 = S + ((g + 1) % 3) * ms;   // diagonal g - 2
    const int* L2 = Lc + ((g + 1) % 3) * ms;
    const int ilo = max(0, g - (Ty - 1)), ihi = min(g, Tx - 1);
    for (int i = ilo + threadIdx.x; i <= ihi; i += DTW_THREADS) {
      const int j = g - i;
      const double dist = cell_dist(xs + (int64_t)i * ldx, ys + (int64_t)j * ldy, D);
      const int s = by_i ? i : j;
      double best = 0.0;
      int bl = 0;
      bool any = false;
      if (i > 0 && j > 0) {            // (i-1, j-1)
        const int q = s - 1;
        best = S2[q];
        bl = L2[q];
        any = true;
      }
      if (i > 0) {                     // (i-1, j)
        const int q = by_i ? s - 1 : s;
        const double v = S1[q];
        if (!any || v < best) {
          best = v;
          bl = L1[q];
          any = true;
        }
      }
      if (j > 0) {                     // (i, j-1)
        const int q = by_i ? s : s - 1;
        const double v = S1[q];
        if (!any || v < best) {
          best = v;
          bl = L1[q];
          any = true;
        }
      }
      Sc[s] = any ? __dadd_rn(dist, best) : dist;
      Lcur[s] = bl + 1;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int g = nd - 1, s = by_i ? Tx - 1 : Ty - 1;
    d.out[2 * blockIdx.x] = S[(g % 3) * ms + s];
    d.out[2 * blockIdx.x + 1] = (double)Lc[(g % 3) * ms + s];
  }
}

constexpr int64_t dtw_diag_bytes(int max_short) { return 3 * (int64_t)max_short * (8 + 4) + 4; }
static_assert(dtw_diag_bytes(AVC_DTW_MAX_SHORT) <= DTW_SMEM_LIMIT, "the diagonals of the longest supported shorter side must fit");

}  // namespace avc

using namespace avc;

extern "C" int avc_mel_cepstrum(const avc_cepstrum_desc* d, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "avc_mel_cepstrum: null descriptor");
  AVC_REQUIRE(d->in != nullptr && d->mean != nullptr && d->std != nullptr && d->dct != nullptr && d->out != nullptr,
              AVC_ERR_INVALID, "avc_mel_cepstrum: null pointer (in %p, mean %p, std %p, dct %p, out %p)", (const void*)d->in,
              (const void*)d->mean, (const void*)d->std, (const void*)d->dct, (const void*)d->out);
  AVC_REQUIRE(d->rows > 0 && d->n_mels > 0 && d->dims > 0, AVC_ERR_INVALID,
              "avc_mel_cepstrum: sizes must be positive (rows %d, n_mels %d, dims %d)", d->rows, d->n_mels, d->dims);
  AVC_REQUIRE(d->dims <= AVC_CEPSTRUM_MAX_DIMS, AVC_ERR_UNSUPPORTED, "avc_mel_cepstrum: dims %d > %d", d->dims,
              AVC_CEPSTRUM_MAX_DIMS);
  AVC_REQUIRE(d->n_mels <= AVC_CEPSTRUM_MAX_MELS, AVC_ERR_UNSUPPORTED, "avc_mel_cepstrum: n_mels %d > %d", d->n_mels,
              AVC_CEPSTRUM_MAX_MELS);
  const int rows_per_cta = MC_SMEM / (8 * d->n_mels);
  const int64_t ctas = cdiv64(d->rows, rows_per_cta);
  mel_cepstrum_kernel<<<(unsigned)ctas, MC_THREADS, rows_per_cta * d->n_mels * 8, (cudaStream_t)stream>>>(*d, rows_per_cta);
  AVC_CHECK_LAUNCH("avc_mel_cepstrum");
  return AVC_OK;
}

extern "C" int avc_dtw(const avc_dtw_desc* d, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "avc_dtw: null descriptor");
  AVC_REQUIRE(d->pairs != nullptr && d->x != nullptr && d->y != nullptr && d->out != nullptr, AVC_ERR_INVALID,
              "avc_dtw: null pointer (pairs %p, x %p, y %p, out %p)", (const void*)d->pairs, (const void*)d->x,
              (const void*)d->y, (const void*)d->out);
  AVC_REQUIRE(d->n_pairs > 0 && d->dims > 0 && d->max_short > 0, AVC_ERR_INVALID,
              "avc_dtw: sizes must be positive (n_pairs %d, dims %d, max_short %d)", d->n_pairs, d->dims, d->max_short);
  AVC_REQUIRE(d->dims <= AVC_CEPSTRUM_MAX_DIMS, AVC_ERR_UNSUPPORTED, "avc_dtw: dims %d > %d", d->dims,
              AVC_CEPSTRUM_MAX_DIMS);
  AVC_REQUIRE(d->max_short <= AVC_DTW_MAX_SHORT, AVC_ERR_UNSUPPORTED,
              "avc_dtw: a pair's shorter side of %d frames exceeds the supported %d", d->max_short, AVC_DTW_MAX_SHORT);
  const int64_t diag = dtw_diag_bytes(d->max_short);
  const int64_t budget = diag < DTW_SMEM_TARGET ? DTW_SMEM_TARGET : diag;
  const int stage_floats = (int)((budget - diag) / 4);
  const int smem = (int)(diag + 4 * (int64_t)stage_floats);
  const cudaError_t e = cudaFuncSetAttribute(dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DTW_SMEM_LIMIT);
  AVC_REQUIRE(e == cudaSuccess, AVC_ERR_CUDA, "avc_dtw: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  dtw_kernel<<<(unsigned)d->n_pairs, DTW_THREADS, smem, (cudaStream_t)stream>>>(*d, stage_floats);
  AVC_CHECK_LAUNCH("avc_dtw");
  return AVC_OK;
}
