// YIN F0 tracking (de Cheveigne & Kawahara 2002) of a ragged batch of signals: the difference function, its cumulative
// mean normalisation, the lag choice and the parabolic refinement, in float64.  One CTA per frame, no atomics: a
// frame's outputs depend on its own samples only, so a signal gets the same bits alone or in any batch.
#include <climits>
#include <cmath>

#include "common.cuh"

namespace avc {
namespace {

constexpr int YIN_LAGS = 8;       // consecutive lags per thread: a register window of 8 samples slides along j
constexpr int YIN_MAX_THREADS = 256;  // 8 x 192 lags at the span cap
static_assert(YIN_MAX_THREADS * YIN_LAGS >= AVC_YIN_MAX_SPAN / 2, "a CTA must cover tau_max <= AVC_YIN_MAX_SPAN / 2");

// samples staged per frame: the span W + tau_max and a zero tail that the last thread's window reads past tau_max
__host__ __device__ inline int yin_staged(int win, int tau_max) { return win + tau_max + YIN_LAGS + 1; }

// Shared-memory slot of sample i: one pad double after every 16, so that the lanes of a warp, 8 lags apart, read 8
// doubles apart plus one slot per two lanes and hit distinct bank pairs.
__device__ __forceinline__ int skew(int i) { return i + (i >> 4); }

// index of the last table entry whose frame_off <= f (the table is sorted by frame_off)
__device__ __forceinline__ int seg_of_frame_yin(const avc_audio_seg* s, int n, int f) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&s[mid].frame_off) <= f) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// sample i of a signal of length L under numpy 'reflect' padding, one reflection (the STFT's and frame power's);
// clamped so that no index leaves the signal
__device__ __forceinline__ int reflect1(int i, int L) {
  if (i < 0) i = -i;
  if (i >= L) i = 2 * (L - 1) - i;
  return min(max(i, 0), L - 1);
}

// The same for an entry that holds samples [first, first + L) of a longer signal, which starts at 0 and ends with the
// entry: the signal's sample first + p as an index into the entry.  Positions are relative to first, so they stay small
// however long the signal is; the reflection at the signal's sample 0 applies only when first = 0 (at_0), which is
// then reflect1(p, L).
__device__ __forceinline__ int reflect1_window(int p, bool at_0, int L) {
  if (at_0 && p < 0) p = -p;
  if (p >= L) p = 2 * (L - 1) - p;
  return min(max(p, 0), L - 1);
}

// avc_yin_window's first sample of an entry with frame origin o, span = win + tau_max: frame o's reads, reflected at
// the end or not, start at o hop - half with half = floor(span / 2), except for the last frame of a closed signal
// whose length L is a multiple of hop (o hop = L), whose end reflection reaches down to 2 (L - 1) - (L - half + span - 1)
// = o hop - ceil(span / 2) - 1: one sample before its span for an even span, two for an odd one
__host__ __device__ inline int64_t yin_first_sample(int o, int hop, int span) {
  const int64_t v = (int64_t)o * hop - (span - span / 2) - 1;
  return v > 0 ? v : 0;
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Shared memory: the frame's samples x[0, yin_staged) (skewed, float64; zero past W + tau_max), then dp[0, tau_max].
// Thread t owns lags tau0 = 1 + 8t .. tau0 + 7 and sums d(tau) = sum_{j<W} (x[j] - x[j+tau])^2 in ascending j with
// one fma per term; lags past tau_max are computed on the zero tail and dropped.  Warp 0 then computes the energy,
// the prefix sums of d (a lane per chunk of consecutive lags, a fixed shuffle scan of the chunk totals), d', the lag
// choice and the refinement.
// ORIGIN (avc_yin_window): a table entry's reserved field is its frame origin o, and its samples start at the signal's
// sample yin_first_sample(o).  It is its own instance, so that avc_yin's kernel keeps its code.
template <bool ORIGIN>
__global__ void __launch_bounds__(YIN_MAX_THREADS) yin_kernel(avc_audio_desc d, int win, int tau_min, int tau_max,
                                                              double theta, double* __restrict__ tau_out,
                                                              double* __restrict__ ap_out, double* __restrict__ en_out) {
  extern __shared__ double sm[];
  const int f = blockIdx.x, t = threadIdx.x, nt = blockDim.x;
  const int n_stage = yin_staged(win, tau_max);
  double* xs = sm;
  double* dp = sm + skew(n_stage) + 1;
  const avc_audio_seg g = d.segs[seg_of_frame_yin(d.segs, d.n_seg, f)];
  const int span = win + tau_max, half = span / 2, L = g.n_samples;
  const float* y = d.y + g.sample_off;
  if (ORIGIN) {
    // frame F = o + f - frame_off of a signal whose samples [first, first + L) the entry holds: its end is the entry's
    const int o = g.reserved;
    const int64_t first = o >= 0 ? yin_first_sample(o, d.hop, span) : 0;
    const int64_t centre = ((int64_t)o + f - g.frame_off) * d.hop, end = first + L;
    // one reflection on each side, and every read at or after first
    if (o < 0 || L < 1 || half > end - 1 || centre + (span - half - 1) > 2 * (end - 1) - first) {
      if (t == 0) tau_out[f] = ap_out[f] = en_out[f] = __longlong_as_double(0x7ff8000000000000LL);
      return;
    }
    const int base = (int)(centre - half - first);   // relative to first
    for (int i = t; i < n_stage; i += nt)
      xs[skew(i)] = i < span ? (double)__ldg(y + reflect1_window(base + i, first == 0, L)) : 0.0;
  } else {
    const int64_t centre = (int64_t)(f - g.frame_off) * d.hop;
    // one reflection on each side: -half >= -(L-1) and centre + span - half - 1 <= 2 (L-1)
    if (L < 1 || half > L - 1 || centre + (span - half - 1) > 2 * (int64_t)(L - 1)) {
      if (t == 0) tau_out[f] = ap_out[f] = en_out[f] = __longlong_as_double(0x7ff8000000000000LL);
      return;
    }
    const int base = (int)centre - half;
    for (int i = t; i < n_stage; i += nt) xs[skew(i)] = i < span ? (double)__ldg(y + reflect1(base + i, L)) : 0.0;
  }
  __syncthreads();

  const int tau0 = 1 + YIN_LAGS * t;
  if (tau0 <= tau_max) {
    double acc[YIN_LAGS], w[YIN_LAGS];
#pragma unroll
    for (int k = 0; k < YIN_LAGS; ++k) {
      acc[k] = 0.0;
      w[k] = xs[skew(tau0 + k)];
    }
    // w[(jj + k) & 7] holds x[j + jj + tau0 + k]; after step jj the slot of k = 0 takes x[j + jj + tau0 + 8]
    int j = 0;
    for (; j + YIN_LAGS <= win; j += YIN_LAGS) {
#pragma unroll
      for (int jj = 0; jj < YIN_LAGS; ++jj) {
        const double a = xs[skew(j + jj)];
#pragma unroll
        for (int k = 0; k < YIN_LAGS; ++k) {
          const double e = a - w[(jj + k) & (YIN_LAGS - 1)];
          acc[k] = fma(e, e, acc[k]);
        }
        w[jj] = xs[skew(j + jj + tau0 + YIN_LAGS)];
      }
    }
    for (; j < win; ++j) {
      const double a = xs[skew(j)];
#pragma unroll
      for (int k = 0; k < YIN_LAGS; ++k) {
        const double e = a - xs[skew(j + tau0 + k)];
        acc[k] = fma(e, e, acc[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < YIN_LAGS; ++k)
      if (tau0 + k <= tau_max) dp[tau0 + k] = acc[k];
  }
  __syncthreads();
  if (t >= 32) return;

  // energy = (1/W) sum_{j<W} x[j]^2: lane-strided in ascending j, then a fixed shuffle tree
  double e = 0.0;
  for (int i = t; i < win; i += 32) e = fma(xs[skew(i)], xs[skew(i)], e);
  e = warp_sum_d(e) / (double)win;

  // S(tau) = sum_{k<=tau} d(k): lane l sums lags [1 + l c, (l + 1) c] in order, then adds the lanes before it
  const int c = (tau_max + 31) / 32;
  const int lo = 1 + t * c, hi = min(tau_max, (t + 1) * c);
  double part = 0.0;
  for (int i = lo; i <= hi; ++i) part += dp[i];
  double incl = part;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double v = __shfl_up_sync(0xffffffffu, incl, o);
    if (t >= o) incl += v;
  }
  double run = __shfl_up_sync(0xffffffffu, incl, 1);  // the lanes before this one
  if (t == 0) run = 0.0;
  for (int i = lo; i <= hi; ++i) {
    const double di = dp[i];
    run += di;
    dp[i] = run == 0.0 ? 1.0 : di * (double)i / run;
  }
  __syncwarp();

  // the smallest tau in [tau_min, tau_max] with d' < theta, and the argmin (smallest tau on ties)
  int first = INT_MAX, amin = INT_MAX;
  double vmin = INFINITY;
  for (int i = tau_min + t; i <= tau_max; i += 32) {
    const double v = dp[i];
    if (v < theta && i < first) first = i;
    if (v < vmin) { vmin = v; amin = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
    const double v2 = __shfl_xor_sync(0xffffffffu, vmin, o);
    const int a2 = __shfl_xor_sync(0xffffffffu, amin, o);
    if (v2 < vmin || (v2 == vmin && a2 < amin)) { vmin = v2; amin = a2; }
  }
  if (t != 0) return;
  int ts;
  if (first != INT_MAX) {
    ts = first;
    while (ts < tau_max && dp[ts + 1] < dp[ts]) ++ts;
  } else {
    ts = amin;  // every d' is finite (d >= 0, S >= d), so the argmin exists
  }
  double delta = 0.0;
  if (ts - 1 >= 1 && ts + 1 <= tau_max) {
    const double a = dp[ts - 1], b = dp[ts], cc = dp[ts + 1];
    const double den = a - 2.0 * b + cc;
    if (den > 0.0) delta = fmin(0.5, fmax(-0.5, (a - cc) / (2.0 * den)));
  }
  tau_out[f] = (double)ts + delta;
  ap_out[f] = dp[ts];
  en_out[f] = e;
}

// ---------------------------------------------------------------------------------------------- spectral pitch shift
constexpr int PS_BINS = 1025;                  // n_fft 2048
constexpr int PS_N1 = PS_BINS - 1;             // the cosines' period is 2 PS_N1 in q k
constexpr int PS_TAB = 2 * PS_N1;
constexpr int PS_THREADS = 256;
constexpr int PS_PER_THREAD = (PS_BINS + PS_THREADS - 1) / PS_THREADS;
constexpr int PS_MAX_CTAS = 1024;              // CTAs loop over rows, so each builds its cosine table once

// Table slot of cos(pi m / PS_N1): one pad float after every 32, so that lanes whose q k step by a power of two up to
// 32 spread over several banks.
__device__ __forceinline__ int ps_slot(int m) { return m + (m >> 5); }

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One row at a time per CTA.  ls holds l = ln max(S, 1e-5), then F = l - E in place; cs the Q cepstral coefficients.
// Warp w sums c[q] for q = w, w + 8, ...: lane j takes k = 1 + j + 32 i in ascending i, then a fixed shuffle tree.
// Thread t owns bins t + 256 i: E is a sequential sum over q, the interpolation reads F after a barrier.
__global__ void __launch_bounds__(PS_THREADS) pitch_shift_kernel(const float* __restrict__ mag,
                                                                 const float* __restrict__ ratio,
                                                                 float* __restrict__ out, int rows, int lifter) {
  __shared__ float tab[PS_TAB + PS_TAB / 32];
  __shared__ float ls[PS_BINS];
  __shared__ float cs[PS_N1];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int m = t; m < PS_TAB; m += PS_THREADS) tab[ps_slot(m)] = cospif((float)m / (float)PS_N1);
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const float a = __ldg(ratio + row);
    const float* S = mag + (size_t)row * PS_BINS;
    float* o = out + (size_t)row * PS_BINS;
    if (a == 1.0f) {
      for (int k = t; k < PS_BINS; k += PS_THREADS) o[k] = __ldg(S + k);
      continue;
    }
    if (!(a > 0.f) || isinf(a)) {
      for (int k = t; k < PS_BINS; k += PS_THREADS) o[k] = __int_as_float(0x7fc00000);
      continue;
    }
    __syncthreads();  // the previous row's readers of ls and cs are done; the table is written
    for (int k = t; k < PS_BINS; k += PS_THREADS) ls[k] = logf(fmaxf(__ldg(S + k), 1e-5f));
    __syncthreads();
    for (int q = warp; q < lifter; q += PS_THREADS / 32) {
      float s = 0.f;
      for (int k = 1 + lane; k < PS_N1; k += 32) s = fmaf(ls[k], tab[ps_slot((q * k) & (PS_TAB - 1))], s);
      s = warp_sum_f(s);
      if (lane == 0) cs[q] = (ls[0] + ((q & 1) ? -ls[PS_N1] : ls[PS_N1]) + 2.f * s) / (float)PS_TAB;
    }
    __syncthreads();
    float e[PS_PER_THREAD];
#pragma unroll
    for (int i = 0; i < PS_PER_THREAD; ++i) {
      const int k = t + PS_THREADS * i;
      if (k >= PS_BINS) break;
      float acc = 0.f;
      for (int q = 1; q < lifter; ++q) acc = fmaf(cs[q], tab[ps_slot((q * k) & (PS_TAB - 1))], acc);
      e[i] = cs[0] + 2.f * acc;
      ls[k] -= e[i];  // each bin is read and written by its own thread only until the barrier
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < PS_PER_THREAD; ++i) {
      const int k = t + PS_THREADS * i;
      if (k >= PS_BINS) break;
      const float p = fminf((float)k / a, (float)PS_N1);  // correctly rounded: the restatement uses the same position
      const int i0 = (int)p;
      const float fr = p - (float)i0;                       // exact
      const float fl = i0 < PS_N1 ? fmaf(fr, ls[i0 + 1] - ls[i0], ls[i0]) : ls[PS_N1];
      o[k] = expf(e[i] + fl);
    }
  }
}

}  // namespace
}  // namespace avc

using namespace avc;

namespace {
// avc_yin's and avc_yin_window's argument checks and launch; `name` prefixes every message
int yin_launch(const avc_audio_desc* d, int32_t win, int32_t tau_min, int32_t tau_max, float threshold, double* tau,
               double* aperiodicity, double* energy, void* stream, const char* name, bool origin) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "%s: null descriptor", name);
  AVC_REQUIRE(d->segs != nullptr && d->n_seg > 0 && d->n_frames >= 0, AVC_ERR_INVALID,
              "%s: empty or missing utterance table (n_seg %d, n_frames %d)", name, d->n_seg, d->n_frames);
  AVC_REQUIRE(d->y != nullptr, AVC_ERR_INVALID, "%s: null signal y", name);
  AVC_REQUIRE(d->hop > 0, AVC_ERR_INVALID, "%s: hop must be positive (got %d)", name, d->hop);
  AVC_REQUIRE(tau != nullptr && aperiodicity != nullptr && energy != nullptr, AVC_ERR_INVALID,
              "%s: null tau, aperiodicity or energy", name);
  AVC_REQUIRE(tau_min >= 1 && tau_min < tau_max, AVC_ERR_INVALID,
              "%s: tau_min / tau_max must satisfy 1 <= tau_min < tau_max (got %d, %d)", name, tau_min, tau_max);
  AVC_REQUIRE(win >= tau_max, AVC_ERR_INVALID, "%s: win must be >= tau_max (got win %d, tau_max %d)", name, win,
              tau_max);
  AVC_REQUIRE((int64_t)win + tau_max <= AVC_YIN_MAX_SPAN, AVC_ERR_UNSUPPORTED,
              "%s: win + tau_max = %lld exceeds AVC_YIN_MAX_SPAN = %d", name, (long long)win + tau_max,
              AVC_YIN_MAX_SPAN);
  AVC_REQUIRE(std::isfinite(threshold) && threshold > 0.f && threshold <= 1.f, AVC_ERR_INVALID,
              "%s: threshold must be finite and in (0, 1] (got %g)", name, (double)threshold);
  if (d->n_frames == 0) return AVC_OK;
  const int threads = 32 * cdiv(cdiv(tau_max, YIN_LAGS), 32);
  const size_t smem = sizeof(double) * (size_t)((yin_staged(win, tau_max) + (yin_staged(win, tau_max) >> 4) + 1) +
                                                 (tau_max + 1));
  if (origin)
    yin_kernel<true><<<d->n_frames, threads, smem, (cudaStream_t)stream>>>(*d, win, tau_min, tau_max,
                                                                           (double)threshold, tau, aperiodicity, energy);
  else
    yin_kernel<false><<<d->n_frames, threads, smem, (cudaStream_t)stream>>>(*d, win, tau_min, tau_max,
                                                                            (double)threshold, tau, aperiodicity, energy);
  AVC_CHECK_LAUNCH(name);
  return AVC_OK;
}
}  // namespace

extern "C" int avc_yin(const avc_audio_desc* d, int32_t win, int32_t tau_min, int32_t tau_max, float threshold,
                       double* tau, double* aperiodicity, double* energy, void* stream) {
  return yin_launch(d, win, tau_min, tau_max, threshold, tau, aperiodicity, energy, stream, "avc_yin", false);
}

extern "C" int avc_yin_window(const avc_audio_desc* d, int32_t win, int32_t tau_min, int32_t tau_max, float threshold,
                              double* tau, double* aperiodicity, double* energy, void* stream) {
  return yin_launch(d, win, tau_min, tau_max, threshold, tau, aperiodicity, energy, stream, "avc_yin_window", true);
}

extern "C" int avc_pitch_shift(const float* mag, const float* ratio, float* out, int32_t rows, int32_t n_bins,
                               int32_t lifter, void* stream) {
  AVC_REQUIRE(mag != nullptr && ratio != nullptr && out != nullptr, AVC_ERR_INVALID,
              "avc_pitch_shift: null mag, ratio or out");
  AVC_REQUIRE(rows >= 1, AVC_ERR_INVALID, "avc_pitch_shift: rows must be >= 1 (got %d)", rows);
  AVC_REQUIRE(lifter >= 1 && lifter <= n_bins - 1, AVC_ERR_INVALID,
              "avc_pitch_shift: lifter must lie in [1, n_bins - 1] (got %d, n_bins %d)", lifter, n_bins);
  AVC_REQUIRE(n_bins == PS_BINS, AVC_ERR_UNSUPPORTED, "avc_pitch_shift: n_bins must be %d (n_fft 2048), got %d",
              PS_BINS, n_bins);
  const size_t bytes = sizeof(float) * (size_t)rows * PS_BINS;
  const char *m0 = (const char*)mag, *o0 = (const char*)out;
  AVC_REQUIRE(o0 + bytes <= m0 || m0 + bytes <= o0, AVC_ERR_INVALID, "avc_pitch_shift: out overlaps mag");
  pitch_shift_kernel<<<rows < PS_MAX_CTAS ? rows : PS_MAX_CTAS, PS_THREADS, 0, (cudaStream_t)stream>>>(mag, ratio, out,
                                                                                                       rows, lifter);
  AVC_CHECK_LAUNCH("avc_pitch_shift");
  return AVC_OK;
}
