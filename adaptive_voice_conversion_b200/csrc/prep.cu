// Corpus preparation (prepare.py): polyphase resampling straight from the files' PCM, and per-mel corpus statistics.
// No atomics: every output element is computed by one thread in a fixed order, so an utterance gets the same bits in
// any batch and in any chunking.
#include "common.cuh"

namespace avc {
namespace {

constexpr int RS_TILE = AVC_RESAMPLE_TILE;
constexpr int RS_THREADS = 256;
constexpr size_t RS_SMEM = 48 * 1024;   // shared memory of one CTA without an opt-in
constexpr int MOM_THREADS = 128;

// the channel mean of sample k of an utterance
template <int FMT>
__device__ __forceinline__ float pcm_mono(const void* pcm, int64_t off, int ch) {
  if (FMT == AVC_PCM_S16) {
    const int16_t* p = static_cast<const int16_t*>(pcm) + off;
    int s = 0;
    for (int c = 0; c < ch; ++c) s += __ldg(p + c);
    return (float)s * (1.f / (32768.f * (float)ch));   // exact for one or two channels
  } else {
    const float* p = static_cast<const float*>(pcm) + off;
    float s = 0.f;
    for (int c = 0; c < ch; ++c) s += __ldg(p + c);
    return ch == 1 ? s : s / (float)ch;
  }
}

// Window of the tile [m0, m1): input samples kw0 .. kw1, kw0 = (m0 down + half_len) / up - (n_taps - 1), so that every
// tap of every output of the tile reads inside it
__host__ __device__ __forceinline__ int64_t window_first(int64_t m0, const avc_resample_desc& d) {
  return (m0 * d.down + d.half_len) / d.up - (d.n_taps - 1);
}

int window_floats(const avc_resample_desc& d) {
  return (int)(((int64_t)(RS_TILE - 1) * d.down) / d.up) + d.n_taps + 1;
}

// One CTA per tile of RS_TILE outputs of one utterance: the tile's input window (converted to float, channels
// averaged, zero outside the utterance) is staged in shared memory, and so is the tap table when both fit RS_SMEM
// (staged); a larger table is read through L1 instead.  Each output is then one fixed-order dot product of its
// phase's taps with the window, newest sample first: the same sum, in the same order, either way.  `staged` is one
// value for the whole launch, so the branch on it sits outside the tap loop.  Tile bounds are int64: the last tile of
// an utterance of n_out >= 2^31 - RS_TILE + 1 outputs ends past INT_MAX.
template <int FMT>
__global__ void __launch_bounds__(RS_THREADS) resample_poly_kernel(const avc_resample_desc d, const bool staged) {
  extern __shared__ float sm[];
  int lo = 0, hi = d.n_seg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&d.segs[mid].tile0) <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const avc_resample_seg g = d.segs[lo];
  const int64_t m0 = (int64_t)((int)blockIdx.x - g.tile0) * RS_TILE;
  const int64_t m1 = min((int64_t)g.n_out, m0 + RS_TILE);
  const int n = (int)(m1 - m0);   // outputs of this tile, <= RS_TILE
  float* out = d.out + g.out_off + m0;
  if (d.up == 1 && d.down == 1) {
    for (int j = threadIdx.x; j < n; j += RS_THREADS) out[j] = pcm_mono<FMT>(d.pcm, g.in_off + (m0 + j) * g.channels, g.channels);
    return;
  }
  const int ntab = staged ? d.up * d.n_taps : 0;
  float* win = sm + ntab;
  const int64_t kw0 = window_first(m0, d);
  const int nw = (int)(((m1 - 1) * d.down + d.half_len) / d.up - kw0) + 1;
  for (int i = threadIdx.x; i < ntab; i += RS_THREADS) sm[i] = __ldg(d.taps + i);
  for (int w = threadIdx.x; w < nw; w += RS_THREADS) {
    const int64_t k = kw0 + w;
    win[w] = (k >= 0 && k < g.n_in) ? pcm_mono<FMT>(d.pcm, g.in_off + k * g.channels, g.channels) : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < n; j += RS_THREADS) {
    const int64_t p = (m0 + j) * d.down + d.half_len;
    const int r = (int)(p % d.up);
    const int cnt = (2 * d.half_len - r) / d.up + 1;
    const float* x = win + (p / d.up - kw0);
    float acc = 0.f;
    if (staged) {
      const float* t = sm + r * d.n_taps;
      for (int i = 0; i < cnt; ++i) acc = fmaf(x[-i], t[i], acc);
    } else {
      const float* t = d.taps + (int64_t)r * d.n_taps;
      for (int i = 0; i < cnt; ++i) acc = fmaf(x[-i], __ldg(t + i), acc);
    }
    out[j] = acc;
  }
}

// (mean, M2) of one mel of one utterance in float64: one thread, frames in order
__global__ void __launch_bounds__(MOM_THREADS) mel_moments_kernel(const avc_moments_desc d) {
  const int m = blockIdx.y * MOM_THREADS + threadIdx.x;
  if (m >= d.n_mels) return;
  const avc_audio_seg g = d.segs[blockIdx.x];
  const float* x = d.mels + (int64_t)g.frame_off * d.n_mels + m;
  double s = 0.0;
  for (int t = 0; t < g.n_frames; ++t) s += (double)__ldg(x + (int64_t)t * d.n_mels);
  const double mean = g.n_frames > 0 ? s / g.n_frames : 0.0;
  double q = 0.0;
  for (int t = 0; t < g.n_frames; ++t) {
    const double v = (double)__ldg(x + (int64_t)t * d.n_mels) - mean;
    q = fma(v, v, q);
  }
  double* o = d.moments + ((d.first + blockIdx.x) * d.n_mels + m) * 2;
  o[0] = mean;
  o[1] = q;
}

// Chan's pairwise update over the utterances in order: one thread per mel
__global__ void __launch_bounds__(MOM_THREADS)
moments_merge_kernel(const double* mom, const int32_t* counts, int n_utts, int n_mels, float* mean32, float* std32,
                     double* mean64, double* std64) {
  const int m = blockIdx.x * MOM_THREADS + threadIdx.x;
  if (m >= n_mels) return;
  double n = 0.0, mean = 0.0, m2 = 0.0;
  for (int u = 0; u < n_utts; ++u) {
    const double nb = (double)__ldg(counts + u);
    if (nb <= 0.0) continue;
    const double mb = __ldg(mom + ((int64_t)u * n_mels + m) * 2), qb = __ldg(mom + ((int64_t)u * n_mels + m) * 2 + 1);
    const double nn = n + nb, delta = mb - mean;
    mean += delta * (nb / nn);
    m2 += qb + delta * delta * (n * nb / nn);
    n = nn;
  }
  const double sd = sqrt(m2 / n);
  mean64[m] = mean;
  std64[m] = sd;
  mean32[m] = (float)mean;
  std32[m] = (float)sd;
}

}  // namespace
}  // namespace avc

using namespace avc;

extern "C" int avc_resample_poly(const avc_resample_desc* d, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "avc_resample_poly: null descriptor");
  AVC_REQUIRE(d->segs != nullptr && d->pcm != nullptr && d->out != nullptr, AVC_ERR_INVALID,
              "avc_resample_poly: null pointer (segs %p, pcm %p, out %p)", (const void*)d->segs, d->pcm, (const void*)d->out);
  AVC_REQUIRE(d->n_seg >= 1 && d->n_tiles >= 0, AVC_ERR_INVALID, "avc_resample_poly: empty table (n_seg %d, n_tiles %d)",
              d->n_seg, d->n_tiles);
  AVC_REQUIRE(d->format == AVC_PCM_S16 || d->format == AVC_PCM_F32, AVC_ERR_INVALID, "avc_resample_poly: unknown format %d",
              d->format);
  AVC_REQUIRE(d->up >= 1 && d->down >= 1, AVC_ERR_INVALID, "avc_resample_poly: up and down must be >= 1 (got %d, %d)",
              d->up, d->down);
  const bool identity = d->up == 1 && d->down == 1;
  if (!identity) {
    AVC_REQUIRE(d->taps != nullptr, AVC_ERR_INVALID, "avc_resample_poly: null tap table");
    const int64_t mx = d->up > d->down ? d->up : d->down;
    AVC_REQUIRE(d->half_len == 10 * mx && (int64_t)d->n_taps == cdiv64(2 * (int64_t)d->half_len + 1, d->up), AVC_ERR_INVALID,
                "avc_resample_poly: the tap table of up %d / down %d has half_len %lld and %lld taps per phase (got %d, %d)",
                d->up, d->down, (long long)(10 * mx), (long long)cdiv64(20 * mx + 1, d->up), d->half_len, d->n_taps);
    AVC_REQUIRE(d->n_taps <= AVC_RESAMPLE_MAX_PHASE_TAPS && (int64_t)d->up * d->n_taps <= AVC_RESAMPLE_MAX_TAPS,
                AVC_ERR_UNSUPPORTED, "avc_resample_poly: up %d / down %d needs %d taps per phase and %lld in all (at most %d and %d)",
                d->up, d->down, d->n_taps, (long long)d->up * d->n_taps, AVC_RESAMPLE_MAX_PHASE_TAPS, AVC_RESAMPLE_MAX_TAPS);
  }
  if (d->n_tiles == 0) return AVC_OK;
  // the window is at most 511 down/up + n_taps + 1 floats, under 6 800 within the limits above; the table joins it in
  // shared memory when both fit
  const size_t win_bytes = identity ? 0 : sizeof(float) * window_floats(*d);
  const size_t tab_bytes = identity ? 0 : sizeof(float) * d->up * d->n_taps;
  const bool staged = win_bytes + tab_bytes <= RS_SMEM;
  const size_t smem = win_bytes + (staged ? tab_bytes : 0);
  AVC_REQUIRE(smem <= RS_SMEM, AVC_ERR_UNSUPPORTED, "avc_resample_poly: up %d / down %d needs %zu bytes of shared memory",
              d->up, d->down, smem);
  cudaStream_t st = (cudaStream_t)stream;
  if (d->format == AVC_PCM_S16) resample_poly_kernel<AVC_PCM_S16><<<d->n_tiles, RS_THREADS, smem, st>>>(*d, staged);
  else resample_poly_kernel<AVC_PCM_F32><<<d->n_tiles, RS_THREADS, smem, st>>>(*d, staged);
  AVC_CHECK_LAUNCH("avc_resample_poly");
  return AVC_OK;
}

extern "C" int avc_mel_moments(const avc_moments_desc* d, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "avc_mel_moments: null descriptor");
  AVC_REQUIRE(d->segs != nullptr && d->mels != nullptr && d->moments != nullptr, AVC_ERR_INVALID,
              "avc_mel_moments: null pointer (segs %p, mels %p, moments %p)", (const void*)d->segs, (const void*)d->mels,
              (const void*)d->moments);
  AVC_REQUIRE(d->n_seg >= 1 && d->n_mels >= 1 && d->first >= 0, AVC_ERR_INVALID,
              "avc_mel_moments: bad shape (n_seg %d, n_mels %d, first %lld)", d->n_seg, d->n_mels, (long long)d->first);
  AVC_REQUIRE(cdiv(d->n_mels, MOM_THREADS) <= 65535, AVC_ERR_UNSUPPORTED, "avc_mel_moments: %d mels exceed the launch grid",
              d->n_mels);
  const dim3 grid((unsigned)d->n_seg, (unsigned)cdiv(d->n_mels, MOM_THREADS));
  mel_moments_kernel<<<grid, MOM_THREADS, 0, (cudaStream_t)stream>>>(*d);
  AVC_CHECK_LAUNCH("avc_mel_moments");
  return AVC_OK;
}

extern "C" int avc_mel_moments_merge(const double* moments, const int32_t* counts, int32_t n_utts, int32_t n_mels,
                                     float* mean, float* std, double* mean64, double* std64, void* stream) {
  AVC_REQUIRE(moments != nullptr && counts != nullptr && mean != nullptr && std != nullptr && mean64 != nullptr &&
                  std64 != nullptr, AVC_ERR_INVALID, "avc_mel_moments_merge: null pointer");
  AVC_REQUIRE(n_utts >= 1 && n_mels >= 1, AVC_ERR_INVALID, "avc_mel_moments_merge: bad shape (n_utts %d, n_mels %d)",
              n_utts, n_mels);
  moments_merge_kernel<<<cdiv(n_mels, MOM_THREADS), MOM_THREADS, 0, (cudaStream_t)stream>>>(moments, counts, n_utts, n_mels,
                                                                                           mean, std, mean64, std64);
  AVC_CHECK_LAUNCH("avc_mel_moments_merge");
  return AVC_OK;
}
