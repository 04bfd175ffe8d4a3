// The vocoder's DSP: STFT / iSTFT on a shared-memory 2048-point real FFT, Griffin-Lim and its PGHI start phase, the
// mel projections, the de-emphasis recurrence and the per-frame power of the silence trim.  fp32 (PGHI's phases in
// float64), no atomics: every output element is computed by one thread in a fixed order, so a ragged batch gives each
// utterance the bits it gets alone.
#include <float.h>

#include <climits>
#include <cmath>
#include <type_traits>

#include "common.cuh"

namespace avc {
namespace {

constexpr int NFFT = 2048;     // the only supported n_fft
constexpr int NC = NFFT / 2;   // complex points of the half-length FFT
constexpr int NBIN = NC + 1;   // rfft bins
constexpr int FPB = 4;         // frames per CTA
constexpr int TPF = 128;       // threads per frame
constexpr int FFT_THREADS = FPB * TPF;

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// tab[k] = exp(-2 pi i k / 2048), k < 1024; sincospif is exact-argument and accurate to ~1 ulp
__device__ __forceinline__ void fill_twiddles(float2* tab) {
  for (int k = threadIdx.x; k < NC; k += blockDim.x) {
    float s, c;
    sincospif(-(float)k / (float)NC, &s, &c);
    tab[k] = make_float2(c, s);
  }
}
// exp(-2 pi i m / 1024), 0 <= m < 1024
__device__ __forceinline__ float2 tw1024(const float2* tab, int m) {
  const int e = 2 * m;
  if (e < NC) return tab[e];
  const float2 t = tab[e - NC];
  return make_float2(-t.x, -t.y);
}

// Forward 1024-point complex FFT of buf in place (radix-4 Stockham, 5 passes, natural order in and out).  The 128
// threads of a frame own 2 butterflies each; every thread of the CTA calls it (it contains __syncthreads).
__device__ __forceinline__ void fft1024(float2* buf, const float2* tab, int t) {
#pragma unroll 1
  for (int Ns = 1; Ns < NC; Ns *= 4) {
    float2 v[2][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = t + h * TPF, k = j & (Ns - 1);
#pragma unroll
      for (int r = 0; r < 4; ++r) v[h][r] = buf[j + r * (NC / 4)];
      if (Ns > 1) {
        const int step = (NC / 4) / Ns;
        v[h][1] = cmul(v[h][1], tw1024(tab, k * step));
        v[h][2] = cmul(v[h][2], tw1024(tab, 2 * k * step));
        v[h][3] = cmul(v[h][3], tw1024(tab, 3 * k * step));
      }
      const float2 a0 = make_float2(v[h][0].x + v[h][2].x, v[h][0].y + v[h][2].y);
      const float2 a1 = make_float2(v[h][0].x - v[h][2].x, v[h][0].y - v[h][2].y);
      const float2 a2 = make_float2(v[h][1].x + v[h][3].x, v[h][1].y + v[h][3].y);
      const float2 a3 = make_float2(v[h][1].x - v[h][3].x, v[h][1].y - v[h][3].y);
      v[h][0] = make_float2(a0.x + a2.x, a0.y + a2.y);
      v[h][2] = make_float2(a0.x - a2.x, a0.y - a2.y);
      v[h][1] = make_float2(a1.x + a3.y, a1.y - a3.x);  // a1 - i a3
      v[h][3] = make_float2(a1.x - a3.y, a1.y + a3.x);  // a1 + i a3
    }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = t + h * TPF, k = j & (Ns - 1);
      const int d = (j - k) * 4 + k;
#pragma unroll
      for (int r = 0; r < 4; ++r) buf[d + r * Ns] = v[h][r];
    }
    __syncthreads();
  }
}

// periodic Hann of length win at offset q (0 <= q < win)
__device__ __forceinline__ float hann(int q, int win) { return 0.5f - 0.5f * cospif((float)(2 * q) / (float)win); }

// index of the last table entry whose frame_off <= f (the table is sorted by frame_off)
__device__ __forceinline__ int seg_of_frame(const avc_audio_seg* s, int n, int f) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&s[mid].frame_off) <= f) lo = mid; else hi = mid - 1;
  }
  return lo;
}
__device__ __forceinline__ int seg_of_sample(const avc_audio_seg* s, int n, int64_t j) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&s[mid].sample_off) <= j) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// sample i of a signal of length L under numpy 'reflect' padding (one reflection; clamped so that a table entry
// shorter than the documented minimum cannot read outside its utterance)
__device__ __forceinline__ int reflect(int i, int L) {
  if (i < 0) i = -i;
  if (i >= L) i = 2 * (L - 1) - i;
  return min(max(i, 0), L - 1);
}

// The same for a segment that holds samples [first, first + L) of a longer signal, which starts at 0 and ends with
// the segment: the signal's sample first + p as an index into the segment.  Positions are relative to first, so they
// stay small however long the signal is; the reflection at the signal's sample 0 applies only when first = 0 (at_0),
// which is then reflect(p, L).
__device__ __forceinline__ int reflect_window(int p, bool at_0, int L) {
  if (at_0 && p < 0) p = -p;
  if (p >= L) p = 2 * (L - 1) - p;
  return min(max(p, 0), L - 1);
}

// ------------------------------------------------------------------ forward STFT
// One frame per 128 threads: the windowed frame is read straight from the signal (reflect padding and pre-emphasis
// applied on the fly), packed as z[n] = x[2n] + i x[2n+1], transformed, and split into the 1025 rfft bins.
// MOMENTUM: the fast Griffin-Lim projection (X_prev set, mode PROJECT or PROJECT_FIRST).  It is its own instance so
// that the other epilogues keep their 32 registers (4 CTAs per SM).
// ORIGIN (avc_stft_window): a table entry's reserved field is its frame origin.
template <bool MOMENTUM, bool ORIGIN>
__global__ void __launch_bounds__(FFT_THREADS) stft_kernel(avc_audio_desc d) {
  __shared__ float2 tab[NC];
  __shared__ float2 buf[FPB][NC];
  fill_twiddles(tab);
  const int fl = threadIdx.x / TPF, t = threadIdx.x % TPF;
  const int f = blockIdx.x * FPB + fl;
  const bool live = f < d.n_frames;
  avc_audio_seg g = {};
  if (live) g = d.segs[seg_of_frame(d.segs, d.n_seg, f)];
  const float* y = d.y + g.sample_off;
  const int L = g.n_samples, off = (NFFT - d.win) / 2;
  // frame origin o: the entry's frames are frames o, o + 1, ... of a longer signal, and its samples start at that
  // signal's sample first (0 for origin 0, the whole signal).  Every sample a frame reads, reflected at the end or
  // not, is at or after o hop - win/2 - 1, so with first one sample earlier its pre-emphasis neighbour is inside: a
  // read at segment index 0 happens only when first = 0, where index 0 is the signal's sample 0.
  // With an origin, base is relative to first (64-bit products: o hop passes 2^31 after a day of a live stream).
  const int o = ORIGIN ? g.reserved : 0;
  const int64_t first = ORIGIN ? max((int64_t)0, (int64_t)o * d.hop - d.win / 2 - 2) : 0;
  const int base = ORIGIN ? (int)(((int64_t)o + (f - g.frame_off)) * d.hop - NFFT / 2 - first)
                          : (f - g.frame_off) * d.hop - NFFT / 2;
  const float pe = d.preemph;
  float2* z = buf[fl];
  for (int n = t; n < NC; n += TPF) {
    float v[2] = {0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int q = 2 * n + e - off;
      if (live && q >= 0 && q < d.win) {
        const int i = ORIGIN ? reflect_window(base + 2 * n + e, first == 0, L) : reflect(base + 2 * n + e, L);
        float s = __ldg(y + i);
        if (pe != 0.f && i > 0) s -= pe * __ldg(y + i - 1);
        v[e] = hann(q, d.win) * s;
      }
    }
    z[n] = make_float2(v[0], v[1]);
  }
  __syncthreads();
  fft1024(z, tab, t);
  if (!live) return;
  const int64_t row = (int64_t)f * NBIN;
  // fast Griffin-Lim: P, the previous iteration's E, is loaded one bin ahead of its use, so each load is in flight
  // during a bin's shared-memory reads and arithmetic.  P is never read on the first iteration, where it holds
  // whatever the caller's buffer held.
  float2* P = reinterpret_cast<float2*>(d.X_prev) + row;
  const bool read_p = MOMENTUM && d.mode == AVC_STFT_PROJECT;
  const float c = d.momentum / (1.f + d.momentum);
  float2 p = make_float2(0.f, 0.f);
  if (read_p) p = P[t];
  for (int k = t; k <= NC; k += TPF) {
    const float2 zk = z[k & (NC - 1)], zr = z[(NC - k) & (NC - 1)];
    // Xe = (Z[k] + conj Z[N-k]) / 2, Xo = (Z[k] - conj Z[N-k]) / 2i, X[k] = Xe + W^k Xo
    const float2 xe = make_float2(0.5f * (zk.x + zr.x), 0.5f * (zk.y - zr.y));
    const float2 xo = make_float2(0.5f * (zk.y + zr.y), -0.5f * (zk.x - zr.x));
    const float2 w = k < NC ? tab[k] : make_float2(-1.f, 0.f);
    const float2 wx = cmul(w, xo);
    const float2 X = make_float2(xe.x + wx.x, xe.y + wx.y);
    if (MOMENTUM) {  // A = E - c P, P = E, the next spectrum S * A / max(1e-8, |A|)
      const float2 A = read_p ? make_float2(X.x - c * p.x, X.y - c * p.y) : X;
      P[k] = X;
      if (read_p && k + TPF <= NC) p = P[k + TPF];
      const float s = __ldg(d.mag + row + k) / fmaxf(1e-8f, sqrtf(A.x * A.x + A.y * A.y));
      reinterpret_cast<float2*>(d.X)[row + k] = make_float2(A.x * s, A.y * s);
    } else if (d.mode == AVC_STFT_COMPLEX) {
      reinterpret_cast<float2*>(d.X)[row + k] = X;
    } else {
      const float a = sqrtf(X.x * X.x + X.y * X.y);
      if (d.mode == AVC_STFT_MAG) {
        if (d.mag_out) d.mag_out[row + k] = a;
        if (d.mag_db) {
          const float db = 20.f * log10f(fmaxf(1e-5f, a));
          d.mag_db[row + k] = fminf(1.f, fmaxf(1e-8f, (db - d.ref_db + d.max_db) / d.max_db));
        }
      } else {  // AVC_STFT_PROJECT(_FIRST) without momentum: the next Griffin-Lim spectrum S * E / max(1e-8, |E|)
        const float s = __ldg(d.mag + row + k) / fmaxf(1e-8f, a);
        reinterpret_cast<float2*>(d.X)[row + k] = make_float2(X.x * s, X.y * s);
      }
    }
  }
}

// ------------------------------------------------------------------ iSTFT, per frame
// irfft of one frame (imaginary parts of the DC and Nyquist bins ignored) through the same FFT core:
// Z[k] = Xe[k] + i Xo[k], z = conj(FFT(conj Z)) / 1024, x[2n] = Re z[n], x[2n+1] = Im z[n].  Multiplied by the
// window; only the win non-zero samples are stored.  X null: the spectrum is mag with zero phase.
__global__ void __launch_bounds__(FFT_THREADS) istft_frames_kernel(avc_audio_desc d) {
  __shared__ float2 tab[NC];
  __shared__ float2 buf[FPB][NC];
  fill_twiddles(tab);
  __syncthreads();
  const int fl = threadIdx.x / TPF, t = threadIdx.x % TPF;
  const int f = blockIdx.x * FPB + fl;
  const bool live = f < d.n_frames;
  const int64_t row = (int64_t)f * NBIN;
  const float2* X = reinterpret_cast<const float2*>(d.X);
  float2* z = buf[fl];
  for (int k = t; k < NC; k += TPF) {
    float2 a = make_float2(0.f, 0.f), b = a;
    if (live) {
      if (X) {
        a = X[row + k];
        b = X[row + NC - k];
      } else {
        a.x = __ldg(d.mag + row + k);
        b.x = __ldg(d.mag + row + NC - k);
      }
      if (k == 0) a.y = b.y = 0.f;  // DC and Nyquist are real
    }
    b.y = -b.y;  // conj X[N-k]
    const float2 xe = make_float2(0.5f * (a.x + b.x), 0.5f * (a.y + b.y));
    const float2 w = tab[k];
    const float2 xo = cmul(make_float2(0.5f * (a.x - b.x), 0.5f * (a.y - b.y)), make_float2(w.x, -w.y));
    z[k] = make_float2(xe.x - xo.y, -(xe.y + xo.x));  // conj(Xe + i Xo)
  }
  __syncthreads();
  fft1024(z, tab, t);
  if (!live) return;
  const int off = (NFFT - d.win) / 2;
  const float inv = 1.f / (float)NC;
  float* out = d.frames + (int64_t)f * d.win;
  for (int q = t; q < d.win; q += TPF) {
    const int p = off + q;
    const float2 v = z[p >> 1];
    out[q] = ((p & 1) ? -v.y : v.x) * inv * hann(q, d.win);
  }
}

// ------------------------------------------------------------------ iSTFT, overlap-add (gather form)
// Output sample i of an utterance sits at position p = i + n_fft/2 of the padded frame grid; it sums the frames that
// cover it in increasing frame order and divides by their window sum-square where that exceeds FLT_MIN.
__global__ void __launch_bounds__(256) ola_kernel(avc_audio_desc d) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= d.n_samples) return;
  const avc_audio_seg g = d.segs[seg_of_sample(d.segs, d.n_seg, j)];
  const int64_t i = j - g.sample_off;
  if (i < 0 || i >= g.n_samples) return;
  const int hop = d.hop, win = d.win, off = (NFFT - win) / 2;
  const int p = (int)i + NFFT / 2 - off;  // position relative to frame 0's first window sample
  const int f_hi = min(g.n_frames - 1, p / hop);
  const int lo = p - win + 1;
  const int f_lo = lo <= 0 ? 0 : cdiv(lo, hop);
  const float* fr = d.frames + (int64_t)g.frame_off * win;
  float acc = 0.f, wss = 0.f;
  for (int f = f_lo; f <= f_hi; ++f) {
    const int q = p - f * hop;
    acc += __ldg(fr + (int64_t)f * win + q);
    const float w = hann(q, win);
    wss += w * w;
  }
  d.y[j] = wss > FLT_MIN ? acc / wss : acc;
}

// ------------------------------------------------------------------ frame power (silence trim)
// power[f] = mean of y^2 over frame f (n_fft samples, hop apart, reflect-padded by n_fft/2): one warp per frame,
// lane-strided partial sums and a fixed shuffle tree.
__global__ void __launch_bounds__(256) frame_power_kernel(avc_audio_desc d, float* power) {
  const int f = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (f >= d.n_frames) return;
  const avc_audio_seg g = d.segs[seg_of_frame(d.segs, d.n_seg, f)];
  const float* y = d.y + g.sample_off;
  const int base = (f - g.frame_off) * d.hop - d.n_fft / 2;
  float s = 0.f;
  for (int n = lane; n < d.n_fft; n += 32) {
    const float v = __ldg(y + reflect(base + n, g.n_samples));
    s += v * v;
  }
  s = warp_sum(s);
  if (lane == 0) power[f] = s / (float)d.n_fft;
}

// ------------------------------------------------------------------ de-emphasis y[n] = x[n] + a y[n-1], in place
// One CTA per utterance; thread t runs the recurrence over its contiguous chunk from a zero carry.  A chunk maps an
// incoming carry c to its last output B + A c (A = a^len); a block scan of these affine maps gives every chunk its
// exact incoming carry, which a second pass adds as carry * a^k.
__global__ void __launch_bounds__(1024) deemphasis_kernel(avc_audio_desc d, float a) {
  __shared__ float sA[32], sB[32], carry[1024];
  const avc_audio_seg g = d.segs[blockIdx.x];
  float* y = d.y + g.sample_off;
  const int L = g.n_samples, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int per = cdiv(L, blockDim.x);
  const int s0 = min(L, t * per), s1 = min(L, s0 + per);
  float A = 1.f, B = 0.f;
  for (int i = s0; i < s1; ++i) {
    B = y[i] + a * B;
    y[i] = B;
    A *= a;
  }
  // inclusive scan of (A, B) over the threads: earlier map first, (A2, B2) o (A1, B1) = (A2 A1, A2 B1 + B2)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float pa = __shfl_up_sync(0xffffffffu, A, o), pb = __shfl_up_sync(0xffffffffu, B, o);
    if (lane >= o) { B = A * pb + B; A = A * pa; }
  }
  if (lane == 31) { sA[warp] = A; sB[warp] = B; }
  __syncthreads();
  if (warp == 0) {
    float wa = lane < (int)(blockDim.x >> 5) ? sA[lane] : 1.f, wb = lane < (int)(blockDim.x >> 5) ? sB[lane] : 0.f;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float pa = __shfl_up_sync(0xffffffffu, wa, o), pb = __shfl_up_sync(0xffffffffu, wb, o);
      if (lane >= o) { wb = wa * pb + wb; wa = wa * pa; }
    }
    sA[lane] = wa;
    sB[lane] = wb;
  }
  __syncthreads();
  carry[t] = warp > 0 ? A * sB[warp - 1] + B : B;  // last output of chunk t, the utterance starting from rest
  __syncthreads();
  float c = t > 0 ? carry[t - 1] : 0.f;
  for (int i = s0; i < s1; ++i) {
    c *= a;
    y[i] += c;
  }
}

// ------------------------------------------------------------------ mel projections (fp32 SIMT GEMM)
// out[rows][N] = pro(in)[rows][K] x mat[K][N], 64 x 64 tiles, 16-deep k slices, 4 x 4 outputs per thread.
//   MEL_TO_MAG: pro = normalised mel -> amplitude 10^((clip(v,0,1) max_db - max_db + ref_db)/20), K = n_mels, N = bins
//   MAG_TO_MEL: epilogue amplitude -> clip((20 log10(max(1e-5, v)) - ref_db + max_db)/max_db, 1e-8, 1), K = bins
// Column tiles on gridDim.x; row tiles on gridDim.y, which is capped at 65 535, so a CTA takes row tiles blockIdx.y,
// blockIdx.y + gridDim.y, ...: every row count fits, and each output is still one thread's sum in k order.
template <int DIR>
__global__ void __launch_bounds__(256) mel_gemm_kernel(avc_mel_desc d) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64];
  const int M = d.rows;
  const int K = DIR == AVC_MEL_TO_MAG ? d.n_mels : d.n_bins;
  const int N = DIR == AVC_MEL_TO_MAG ? d.n_bins : d.n_mels;
  const int row_tiles = cdiv(M, 64), c0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  for (int rt = blockIdx.y; rt < row_tiles; rt += gridDim.y) {
    const int r0 = rt * 64;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int id = threadIdx.x + 256 * e;
        const int r = id >> 4, kk = id & 15;
        float v = 0.f;
        if (r0 + r < M && k0 + kk < K) {
          v = __ldg(d.in + (int64_t)(r0 + r) * K + k0 + kk);
          if (DIR == AVC_MEL_TO_MAG) v = exp10f((fminf(1.f, fmaxf(0.f, v)) * d.max_db - d.max_db + d.ref_db) / 20.f);
        }
        As[kk][r] = v;
        const int kb = id >> 6, c = id & 63;
        Bs[kb][c] = (k0 + kb < K && c0 + c < N) ? __ldg(d.mat + (int64_t)(k0 + kb) * N + c0 + c) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < 16; ++kk) {
        float av[4], bv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { av[i] = As[kk][ty + 16 * i]; bv[i] = Bs[kk][tx + 16 * i]; }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) acc[i][jj] = fmaf(av[i], bv[jj], acc[i][jj]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = r0 + ty + 16 * i;
      if (r >= M) continue;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int c = c0 + tx + 16 * jj;
        if (c >= N) continue;
        float v = acc[i][jj];
        if (DIR == AVC_MAG_TO_MEL) {
          const float db = 20.f * log10f(fmaxf(1e-5f, v));
          v = fminf(1.f, fmaxf(1e-8f, (db - d.ref_db + d.max_db) / d.max_db));
        }
        d.out[(int64_t)r * N + c] = v;
      }
    }
  }
}

// ------------------------------------------------------------------ PGHI start phase
// One CTA per utterance walks its frames in order.  Thread t owns the PG_PER contiguous bins from PG_PER t, so each
// per-frame block scan folds a thread's bins in order and combines threads with warp shuffles and one shared-memory
// pass over the warp totals: a fixed order, no atomics.  Three rows of ln-magnitude (frames f-1, f, f+1) sit in shared
// memory in float64; each thread keeps its bins' phases of frame f-1 in registers, wrapped, in float64.
//
// A heap key orders the integration's sources: larger magnitude, then frame f-1 before frame f, then the lower bin.
// It is (float bits of s) << 12 | (frame f-1) << 11 | (2047 - k); 0 is "insignificant" (-inf).  With a_k the key of
// (f-1, k) and c_k that of (f, k), the heap assigns (f, k) from the largest of three candidates: the time source a_k,
// the left path min(L_{k-1}, c_{k-1}) and the right path min(R_{k+1}, c_{k+1}), with the directional levels
// L_k = max(a_k, min(L_{k-1}, c_{k-1})) and R_k = max(a_k, min(R_{k+1}, c_{k+1})).  Both are scans of the clamp maps
// x -> max(a, min(x, b)).  A significant bin with no candidate is in a run that no source reaches; the heap seeds
// such a run at its largest key and the run's other bins point toward the seed.  Phases are then segmented sums of
// the trapezoid steps along the left- and right-parented chains, from their time-parented or seed roots.
constexpr int PG_THREADS = 256;
constexpr int PG_WARPS = PG_THREADS / 32;
constexpr int PG_PER = 5;                                      // bins per thread: 205 threads cover the 1025 bins
constexpr int PG_LOADS = (NBIN + PG_THREADS - 1) / PG_THREADS; // coalesced loads of a row per thread
static_assert(PG_THREADS * PG_PER >= NBIN, "every bin needs a thread");

typedef unsigned long long u64;
struct Pair {
  u64 a, b;
};
// clamp map x -> min(max(x, a), b) with a <= b (x -> max(a, min(x, b')) is the clamp to [a, max(a, b')]);
// f(e, l) applies e, then l
struct ClampOp {
  __device__ static Pair id() { return {0ull, ~0ull}; }
  __device__ static Pair f(Pair e, Pair l) {
    return {min(max(e.a, l.a), l.b), min(max(e.b, l.a), l.b)};
  }
};
// segmented max: a = starts a segment, b = key
struct SegMaxOp {
  __device__ static Pair id() { return {0ull, 0ull}; }
  __device__ static Pair f(Pair e, Pair l) { return l.a ? l : Pair{e.a, max(e.b, l.b)}; }
};
// segmented sum: a = starts a segment, b = float64 bits
struct SegSumOp {
  __device__ static Pair id() { return {0ull, 0ull}; }
  __device__ static Pair f(Pair e, Pair l) {
    return l.a ? l : Pair{e.a, (u64)__double_as_longlong(__longlong_as_double((long long)e.b) +
                                                         __longlong_as_double((long long)l.b))};
  }
};

// Exclusive block scan of one element per thread, in thread order (REV: from the last thread down).
template <class Op, bool REV>
__device__ __forceinline__ Pair block_scan_excl(Pair v, Pair* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    Pair u;
    u.a = REV ? __shfl_down_sync(0xffffffffu, v.a, o) : __shfl_up_sync(0xffffffffu, v.a, o);
    u.b = REV ? __shfl_down_sync(0xffffffffu, v.b, o) : __shfl_up_sync(0xffffffffu, v.b, o);
    if (REV ? lane + o < 32 : lane >= o) v = Op::f(u, v);
  }
  Pair ex;
  ex.a = REV ? __shfl_down_sync(0xffffffffu, v.a, 1) : __shfl_up_sync(0xffffffffu, v.a, 1);
  ex.b = REV ? __shfl_down_sync(0xffffffffu, v.b, 1) : __shfl_up_sync(0xffffffffu, v.b, 1);
  if (lane == (REV ? 31 : 0)) ex = Op::id();
  if (lane == (REV ? 0 : 31)) sh[warp] = v;
  __syncthreads();
  Pair p = Op::id();
  if (REV) {
    for (int w = PG_WARPS - 1; w > warp; --w) p = Op::f(p, sh[w]);
  } else {
    for (int w = 0; w < warp; ++w) p = Op::f(p, sh[w]);
  }
  __syncthreads();
  return Op::f(p, ex);
}

__device__ __forceinline__ u64 pghi_key(float s, double thr, int k, bool prev) {
  return (s > 0.f && (double)s >= thr) ? ((u64)__float_as_uint(s) << 12 | (prev ? 2048ull : 0ull) | (u64)(2047 - k))
                                       : 0ull;
}
// centred difference over bins, one-sided at the edges (numpy.gradient)
__device__ __forceinline__ double diff_bins(const double* l, int k) {
  return k == 0 ? l[1] - l[0] : k == NC ? l[NC] - l[NC - 1] : 0.5 * (l[k + 1] - l[k - 1]);
}

// The streaming instance (avc_pghi_stream) runs one stream per CTA, its frames in order across launches.  Frame f is
// integrated once frame f+1 has arrived, or at close, at the threshold tol s_max(f), s_max(f) the largest magnitude of
// frames 0 .. f+1 (0 .. f for the last): the three ln-magnitude rows a frame reads are taken again at its threshold, so
// its bits depend only on the stream's magnitudes, not on how they were split into launches.  The state slot holds
// the magnitudes of the last two frames received (slot frame % 2), the phases of the last frame integrated (float64),
// s_max and the count of frames received.  The CTA's entry is an utterance-table entry: frame_off places the first
// frame the launch completes, f_lo, at the stream's out_off row, and n_frames is the stream's length at close (INT_MAX
// before: no frame the launch completes is the last).
constexpr int PS_PHI = 2 * NBIN;                // float offset of the phases (even: 8-byte aligned)
constexpr int PS_SMAX = PS_PHI + 2 * NBIN;
constexpr int PS_COUNT = PS_SMAX + 1;
constexpr int PS_FLOATS = (PS_COUNT + 1 + 3) / 4 * 4;

__device__ __forceinline__ int32_t ps_count(const avc_pghi_stream_desc& d) {
  return *reinterpret_cast<const int32_t*>(d.state + (int64_t)d.slot[blockIdx.x] * PS_FLOATS + PS_COUNT);
}
// frames f_lo .. f_hi - 1 that a launch completes, of a stream that had n0 frames and has n1
__device__ __forceinline__ int ps_lo(int n0) { return max(0, n0 - 1); }
__device__ __forceinline__ int ps_hi(int n1, bool close) { return close ? n1 : max(0, n1 - 1); }

__device__ __forceinline__ avc_audio_seg pghi_entry(const avc_audio_desc& d) { return d.segs[blockIdx.x]; }
__device__ __forceinline__ avc_audio_seg pghi_entry(const avc_pghi_stream_desc& d) {
  const int s = blockIdx.x, n0 = ps_count(d), n1 = n0 + (d.mag_off[s + 1] - d.mag_off[s]);
  avc_audio_seg g = {};
  g.frame_off = d.out_off[s] - ps_lo(n0);
  g.n_frames = d.close[s] ? n1 : INT_MAX;
  return g;
}

// The streaming instance may use more than 128 registers (at least one CTA per SM); the offline one keeps its bounds.
template <class Desc>
__global__ void __launch_bounds__(PG_THREADS, (std::is_same<Desc, avc_pghi_stream_desc>::value ? 1 : 0))
    pghi_kernel(Desc d, float tol, int8_t* parent) {
  constexpr bool STREAM = std::is_same<Desc, avc_pghi_stream_desc>::value;
  __shared__ double lrow[3][NBIN];  // ln max(s, tol s_max) of frames f-1, f, f+1 (slot = frame % 3)
  __shared__ float srow[3][NBIN];
  __shared__ Pair sh[PG_WARPS];
  __shared__ float red[PG_WARPS];
  const avc_audio_seg g = pghi_entry(d);
  const int nF = g.n_frames, t = threadIdx.x, k0 = t * PG_PER;
  if (nF <= 0) return;
  const float* mag = d.mag + (int64_t)g.frame_off * NBIN;
  float2* X = reinterpret_cast<float2*>(d.X) + (int64_t)g.frame_off * NBIN;
  int8_t* par = parent ? parent + (int64_t)g.frame_off * NBIN : nullptr;

  // streaming: the stream's state, its frames n0 .. n1 - 1 arriving, frames f_lo .. f_hi - 1 completed
  float* st = nullptr;
  int n0 = 0, n1 = 0, f_lo = 0, f_hi = nF, r0 = 0;
  if constexpr (STREAM) {
    st = d.state + (int64_t)d.slot[blockIdx.x] * PS_FLOATS;
    r0 = d.mag_off[blockIdx.x];
    n0 = ps_count(d);
    n1 = n0 + (d.mag_off[blockIdx.x + 1] - r0);
    f_lo = ps_lo(n0);
    f_hi = ps_hi(n1, d.close[blockIdx.x] != 0);
  }

  // s_max of the utterance (fmaxf is exact, so the order does not matter); streaming: of the frames so far
  float m = 0.f;
  if constexpr (STREAM) {
    m = st[PS_SMAX];
  } else {
    for (int64_t i = t; i < (int64_t)nF * NBIN; i += PG_THREADS) m = fmaxf(m, __ldg(mag + i));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((t & 31) == 0) red[t >> 5] = m;
    __syncthreads();
    m = red[0];
    for (int w = 1; w < PG_WARPS; ++w) m = fmaxf(m, red[w]);
  }
  double thr = (double)tol * (double)m;
  const double lambda = 0.25645 * (double)d.win * (double)d.win;
  const double a_t = (double)d.hop * (double)NFFT / lambda, b_t = (double)d.hop * 2.0 * M_PI / (double)NFFT;
  const double a_f = -lambda / ((double)NFFT * (double)d.hop);

  float nxt[PG_LOADS];
  auto fetch = [&](int f) {
#pragma unroll
    for (int i = 0; i < PG_LOADS; ++i) {
      const int k = t + i * PG_THREADS;
      nxt[i] = (f < nF && k < NBIN) ? __ldg(mag + (int64_t)f * NBIN + k) : 0.f;
    }
  };
  auto store = [&](int f) {
    if (f >= nF) return;
#pragma unroll
    for (int i = 0; i < PG_LOADS; ++i) {
      const int k = t + i * PG_THREADS;
      if (k < NBIN) {
        srow[f % 3][k] = nxt[i];
        lrow[f % 3][k] = log(fmax((double)nxt[i], thr));
      }
    }
  };
  // streaming: frames up to `last` (< n1) into srow, s_max updated with the new ones
  int got = n0;
  auto receive = [&](int last) {
    if constexpr (STREAM) {
      for (; got <= last; ++got) {
        float mx = 0.f;
        for (int k = t; k < NBIN; k += PG_THREADS) {
          const float v = __ldg(d.mag + (int64_t)(r0 + got - n0) * NBIN + k);
          srow[got % 3][k] = v;
          mx = fmaxf(mx, v);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if ((t & 31) == 0) red[t >> 5] = mx;
        __syncthreads();
        for (int w = 0; w < PG_WARPS; ++w) m = fmaxf(m, red[w]);
        __syncthreads();
      }
    }
  };
  if constexpr (STREAM) {
    for (int k = t; k < NBIN; k += PG_THREADS) {
      if (n0 >= 1) srow[(n0 - 1) % 3][k] = st[((n0 - 1) & 1) * NBIN + k];
      if (n0 >= 2) srow[(n0 - 2) % 3][k] = st[((n0 - 2) & 1) * NBIN + k];
    }
  } else {
    fetch(0);
    store(0);
    fetch(1);
    store(1);
    fetch(2);
  }
  __syncthreads();

  double phi_prev[PG_PER];
#pragma unroll
  for (int j = 0; j < PG_PER; ++j) phi_prev[j] = 0.0;
  if constexpr (STREAM) {
    const double* st_phi = reinterpret_cast<const double*>(st + PS_PHI);
#pragma unroll
    for (int j = 0; j < PG_PER; ++j) phi_prev[j] = k0 + j < NBIN ? st_phi[k0 + j] : 0.0;
  }

  for (int f = f_lo; f < f_hi; ++f) {
    if constexpr (STREAM) {  // frame f+1 in, then rows f-1 .. f+1 in ln at this frame's threshold
      receive(min(f + 1, n1 - 1));
      thr = (double)tol * (double)m;
      for (int k = t; k < NBIN; k += PG_THREADS) {
        for (int i = max(f - 1, 0); i <= min(f + 1, n1 - 1); ++i) lrow[i % 3][k] = log(fmax((double)srow[i % 3][k], thr));
        d.mag_out[((int64_t)g.frame_off + f) * NBIN + k] = srow[f % 3][k];
      }
      __syncthreads();
    }
    const double* lm = lrow[(f + 2) % 3];
    const double* l0 = lrow[f % 3];
    const double* lp = lrow[(f + 1) % 3];
    const float* sm = srow[(f + 2) % 3];
    const float* s0 = srow[f % 3];
    // step per bin at frame f, bin k: -(lambda / (N hop)) d_f l - pi
    auto dkphi = [&](int k) {
      const double df = nF == 1 ? 0.0 : f == 0 ? lp[k] - l0[k] : f == nF - 1 ? l0[k] - lm[k] : 0.5 * (lp[k] - lm[k]);
      return a_f * df - M_PI;
    };
    float s[PG_PER];
    u64 a[PG_PER], c[PG_PER];
    double troot[PG_PER], dk[PG_PER];
#pragma unroll
    for (int j = 0; j < PG_PER; ++j) {
      const int k = k0 + j;
      s[j] = 0.f; a[j] = c[j] = 0ull; troot[j] = dk[j] = 0.0;
      if (k < NBIN) {
        s[j] = s0[k];
        c[j] = pghi_key(s[j], thr, k, false);
        a[j] = f > 0 ? pghi_key(sm[k], thr, k, true) : 0ull;
        dk[j] = dkphi(k);
        // trapezoid of the advances per frame, hop ((N / lambda) d_k l + 2 pi k / N), at frames f-1 and f
        if (a[j] && c[j]) troot[j] = 0.5 * (a_t * (diff_bins(lm, k) + diff_bins(l0, k)) + 2.0 * b_t * (double)k);
      }
    }
    const bool any = k0 < NBIN;
    const int kl = k0 - 1, kr = k0 + PG_PER;
    const u64 c_left = any && kl >= 0 ? pghi_key(s0[kl], thr, kl, false) : 0ull;
    const u64 c_right = any && kr < NBIN ? pghi_key(s0[kr], thr, kr, false) : 0ull;
    const double dk_left = any && kl >= 0 ? dkphi(kl) : 0.0;
    const double dk_right = any && kr < NBIN ? dkphi(kr) : 0.0;

    // directional levels: left to right, then right to left
    u64 lc[PG_PER], rc[PG_PER];
    Pair M = ClampOp::id();
#pragma unroll
    for (int j = 0; j < PG_PER; ++j) {
      const u64 cb = j == 0 ? c_left : c[j - 1];
      M = ClampOp::f(M, Pair{a[j], max(a[j], cb)});
    }
    u64 x = block_scan_excl<ClampOp, false>(M, sh).a;
#pragma unroll
    for (int j = 0; j < PG_PER; ++j) {
      lc[j] = min(x, j == 0 ? c_left : c[j - 1]);
      x = max(a[j], lc[j]);
    }
    M = ClampOp::id();
#pragma unroll
    for (int j = PG_PER - 1; j >= 0; --j) {
      const u64 cb = j == PG_PER - 1 ? c_right : c[j + 1];
      M = ClampOp::f(M, Pair{a[j], max(a[j], cb)});
    }
    x = block_scan_excl<ClampOp, true>(M, sh).a;
#pragma unroll
    for (int j = PG_PER - 1; j >= 0; --j) {
      rc[j] = min(x, j == PG_PER - 1 ? c_right : c[j + 1]);
      x = max(a[j], rc[j]);
    }

    // parents; ISLAND marks a significant bin no source reaches until the seeds are chosen
    constexpr int ISLAND = 5;
    int pr[PG_PER];
    bool island = false;
#pragma unroll
    for (int j = 0; j < PG_PER; ++j) {
      pr[j] = AVC_PGHI_NONE;
      if (c[j]) {
        if (a[j] && a[j] >= lc[j] && a[j] >= rc[j]) pr[j] = AVC_PGHI_TIME;
        else if (lc[j] > rc[j]) pr[j] = AVC_PGHI_LEFT;
        else if (rc[j] > lc[j]) pr[j] = AVC_PGHI_RIGHT;
        else pr[j] = ISLAND;
      }
      island |= pr[j] == ISLAND;
    }
    if (__syncthreads_or(island)) {  // seed each run of island bins at its largest key (segmented max both ways)
      u64 fw[PG_PER];
      Pair S = SegMaxOp::id();
#pragma unroll
      for (int j = 0; j < PG_PER; ++j) S = SegMaxOp::f(S, pr[j] == ISLAND ? Pair{0ull, c[j]} : Pair{1ull, 0ull});
      u64 run = block_scan_excl<SegMaxOp, false>(S, sh).b;
#pragma unroll
      for (int j = 0; j < PG_PER; ++j) fw[j] = run = pr[j] == ISLAND ? max(run, c[j]) : 0ull;
      S = SegMaxOp::id();
#pragma unroll
      for (int j = PG_PER - 1; j >= 0; --j) S = SegMaxOp::f(S, pr[j] == ISLAND ? Pair{0ull, c[j]} : Pair{1ull, 0ull});
      run = block_scan_excl<SegMaxOp, true>(S, sh).b;
#pragma unroll
      for (int j = PG_PER - 1; j >= 0; --j) {
        run = pr[j] == ISLAND ? max(run, c[j]) : 0ull;
        if (pr[j] == ISLAND) {
          const u64 top = max(fw[j], run);
          pr[j] = c[j] == top ? AVC_PGHI_SEED : run == top ? AVC_PGHI_RIGHT : AVC_PGHI_LEFT;
        }
      }
    }

    // phases: roots (time steps and seeds), then the chains to their right and to their left
    double root[PG_PER];
#pragma unroll
    for (int j = 0; j < PG_PER; ++j) root[j] = pr[j] == AVC_PGHI_TIME ? phi_prev[j] + troot[j] : 0.0;
    Pair S = SegSumOp::id();
#pragma unroll
    for (int j = 0; j < PG_PER; ++j) {
      const double inc = 0.5 * ((j == 0 ? dk_left : dk[j - 1]) + dk[j]);
      S = SegSumOp::f(S, pr[j] == AVC_PGHI_LEFT ? Pair{0ull, (u64)__double_as_longlong(inc)}
                                                : Pair{1ull, (u64)__double_as_longlong(root[j])});
    }
    double run = __longlong_as_double((long long)block_scan_excl<SegSumOp, false>(S, sh).b);
    double phi[PG_PER];
#pragma unroll
    for (int j = 0; j < PG_PER; ++j) {
      run = pr[j] == AVC_PGHI_LEFT ? run + 0.5 * ((j == 0 ? dk_left : dk[j - 1]) + dk[j]) : root[j];
      phi[j] = run;
    }
    S = SegSumOp::id();
#pragma unroll
    for (int j = PG_PER - 1; j >= 0; --j) {
      const double inc = -0.5 * ((j == PG_PER - 1 ? dk_right : dk[j + 1]) + dk[j]);
      S = SegSumOp::f(S, pr[j] == AVC_PGHI_RIGHT ? Pair{0ull, (u64)__double_as_longlong(inc)}
                                                 : Pair{1ull, (u64)__double_as_longlong(root[j])});
    }
    run = __longlong_as_double((long long)block_scan_excl<SegSumOp, true>(S, sh).b);
#pragma unroll
    for (int j = PG_PER - 1; j >= 0; --j) {
      run = pr[j] == AVC_PGHI_RIGHT ? run - 0.5 * ((j == PG_PER - 1 ? dk_right : dk[j + 1]) + dk[j]) : root[j];
      if (pr[j] == AVC_PGHI_RIGHT) phi[j] = run;
    }

    // X = s e^{i phi}, phi wrapped
    const int64_t row = (int64_t)f * NBIN;
#pragma unroll
    for (int j = 0; j < PG_PER; ++j) {
      const int k = k0 + j;
      double p = pr[j] == AVC_PGHI_NONE ? 0.0 : phi[j];
      p -= 2.0 * M_PI * rint(p * (0.5 / M_PI));
      phi_prev[j] = p;
      if (k < NBIN) {
        double sn, cs;
        sincospi(p * M_1_PI, &sn, &cs);  // |p| <= pi: no argument reduction, so no local-memory slow path
        X[row + k] = make_float2((float)((double)s[j] * cs), (float)((double)s[j] * sn));
        if (par) par[row + k] = (int8_t)pr[j];
      }
    }
    // frame f-1's slot takes frame f+2 (every read of it this frame is behind the scans' barriers)
    if constexpr (!STREAM) {
      store(f + 2);
      fetch(f + 3);
    }
    __syncthreads();
  }
  if constexpr (STREAM) {  // the frames that complete none, then the state
    receive(n1 - 1);
    for (int k = t; k < NBIN; k += PG_THREADS) {
      if (n1 >= 1) st[((n1 - 1) & 1) * NBIN + k] = srow[(n1 - 1) % 3][k];
      if (n1 >= 2) st[((n1 - 2) & 1) * NBIN + k] = srow[(n1 - 2) % 3][k];
    }
    double* st_phi = reinterpret_cast<double*>(st + PS_PHI);
#pragma unroll
    for (int j = 0; j < PG_PER; ++j)
      if (k0 + j < NBIN) st_phi[k0 + j] = phi_prev[j];
    if (t == 0) {
      st[PS_SMAX] = m;
      *reinterpret_cast<int32_t*>(st + PS_COUNT) = n1;
    }
  }
}

// ------------------------------------------------------------------ RTISI-LA (streaming phase reconstruction)
// One CTA per stream, RT_TPF = 128 threads per buffer frame (nb = lookahead + 1 groups).  The stream's windowed
// inverse frames and the overlap-add numerator of its committed frames over the open samples live in shared memory
// for the launch and in the state slot between launches.  Sample n is covered by frame F when 0 <= n - F hop + win/2
// < win (mel_to_signal's grid); the numerator holds samples c hop - win/2 ... c hop + win/2 - 1, c the committed count.
// Every sum runs in a fixed order (numerator, then frames in increasing order) with no atomics.
constexpr int RT_MAX_LA = AVC_RTISI_MAX_LOOKAHEAD;

// floats of one stream's state slot: frames [nb][win], magnitudes [nb][n_bins], numerator [win], de-emphasis carry
__host__ __device__ inline int64_t rt_state_floats(int win, int lookahead) {
  const int64_t nb = lookahead + 1;
  return (nb * win + nb * NBIN + win + 1 + 3) / 4 * 4;
}

__host__ __device__ inline int rt_floordiv(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

struct RtSmem {  // dynamic shared-memory layout of one CTA
  int nb, win, hop;
  __host__ __device__ int scratch_floats() const { return max((nb - 1) * hop + win, 2 * win); }
  __host__ __device__ size_t bytes() const {
    return sizeof(float2) * ((size_t)NC + (size_t)nb * NC + nb) + sizeof(float) * ((size_t)nb * win + win + scratch_floats());
  }
};

// est[i] = signal estimate at sample c hop + r0 + i, i < len: (numerator + the buffered frames c .. c + nbuf - 1 that
// cover it) divided by the window sum-square of the frames 0 .. newest (<= c + nbuf - 1) that cover it, where that
// exceeds FLT_MIN.  Sample positions are relative to c hop, so they stay small however long the stream is; frames
// are absolute, and the covering range is capped at c + nbuf so that it stays below 2^31 with the stream's frames.
__device__ void rt_estimate(float* est, int r0, int len, const float* num, const float* fr, int c, int nbuf, int newest,
                            int nb, int win, int hop) {
  const int h = win / 2;
  for (int i = threadIdx.x; i < len; i += blockDim.x) {
    const int r = r0 + i;
    const int lo = c + rt_floordiv(r + h - win, hop) + 1, hi = c + min(rt_floordiv(r + h, hop), nbuf);
    float acc = (r + h >= 0 && r + h < win) ? num[r + h] : 0.f;
    for (int F = max(lo, c); F <= min(hi, c + nbuf - 1); ++F) acc += fr[(F % nb) * win + r - (F - c) * hop + h];
    float wss = 0.f;
    for (int F = max(lo, 0); F <= min(hi, newest); ++F) {
      const float w = hann(r - (F - c) * hop + h, win);
      wss += w * w;
    }
    est[i] = wss > FLT_MIN ? acc / wss : acc;
  }
}

// One frame's projection in the 128 threads of group z: STFT of the windowed estimate e[0 .. win), the magnitudes mag
// with the estimate's phase (phase 0 where |E| = 0), iSTFT times the window into out.  Every thread of the CTA calls it.
// FROM: the spectrum is Xr (n_fft/2 + 1 complex bins) as given, with no STFT (e and mag are not read).
template <bool FROM = false>
__device__ void rt_project(float2* z, float2* nyq, const float2* tab, int t, const float* e, const float* mag, float* out,
                           bool live, int win, const float2* Xr = nullptr) {
  const int off = (NFFT - win) / 2;
  constexpr int PER = NC / TPF + 1;  // bins per thread, the Nyquist bin with thread 0
  float2 X[PER];
  if constexpr (FROM) {
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int k = t + i * TPF;
      X[i] = live && k <= NC ? Xr[k] : make_float2(0.f, 0.f);
    }
  } else {
    for (int n = t; n < NC; n += TPF) {
      float v[2] = {0.f, 0.f};
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int q = 2 * n + k - off;
        if (live && q >= 0 && q < win) v[k] = hann(q, win) * e[q];
      }
      z[n] = make_float2(v[0], v[1]);
    }
    __syncthreads();
    fft1024(z, tab, t);
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int k = t + i * TPF;
      X[i] = make_float2(0.f, 0.f);
      if (k <= NC) {
        const float2 zk = z[k & (NC - 1)], zr = z[(NC - k) & (NC - 1)];
        const float2 xe = make_float2(0.5f * (zk.x + zr.x), 0.5f * (zk.y - zr.y));
        const float2 xo = make_float2(0.5f * (zk.y + zr.y), -0.5f * (zk.x - zr.x));
        const float2 w = k < NC ? tab[k] : make_float2(-1.f, 0.f);
        const float2 wx = cmul(w, xo);
        const float2 E = make_float2(xe.x + wx.x, xe.y + wx.y);
        const float a = sqrtf(E.x * E.x + E.y * E.y);
        const float m = live ? mag[k] : 0.f;
        X[i] = a > 0.f ? make_float2(m * (E.x / a), m * (E.y / a)) : make_float2(m, 0.f);
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int k = t + i * TPF;
    if (k < NC) z[k] = X[i];
    else if (k == NC) *nyq = X[i];
  }
  __syncthreads();
  float2 P[NC / TPF];
#pragma unroll
  for (int i = 0; i < NC / TPF; ++i) {  // istft_frames_kernel's packing
    const int k = t + i * TPF;
    float2 a = z[k], b = k == 0 ? *nyq : z[NC - k];
    if (k == 0) a.y = b.y = 0.f;
    b.y = -b.y;
    const float2 xe = make_float2(0.5f * (a.x + b.x), 0.5f * (a.y + b.y));
    const float2 w = tab[k];
    const float2 xo = cmul(make_float2(0.5f * (a.x - b.x), 0.5f * (a.y - b.y)), make_float2(w.x, -w.y));
    P[i] = make_float2(xe.x - xo.y, -(xe.y + xo.x));
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < NC / TPF; ++i) z[t + i * TPF] = P[i];
  __syncthreads();
  fft1024(z, tab, t);
  if (!live) return;
  const float inv = 1.f / (float)NC;
  for (int q = t; q < win; q += TPF) {
    const int p = off + q;
    const float2 v = z[p >> 1];
    out[q] = ((p & 1) ? -v.y : v.x) * inv * hann(q, win);
  }
}

// FROM (avc_rtisi_la_from): an entering row r starts from the caller's spectrum X row r (n_fft/2 + 1 complex bins)
// instead of the estimate's phase, which skips the entry STFT.
template <bool FROM>
__global__ void __launch_bounds__((RT_MAX_LA + 1) * TPF) rtisi_kernel(avc_rtisi_desc d, RtSmem L, const float2* X) {
  extern __shared__ float4 rt_smem[];
  const int nb = L.nb, win = L.win, hop = L.hop, h = win / 2;
  float2* tab = reinterpret_cast<float2*>(rt_smem);
  float2* zb = tab + NC;
  float2* nyq = zb + (size_t)nb * NC;
  float* fr = reinterpret_cast<float*>(nyq + nb);
  float* num = fr + (size_t)nb * win;
  float* est = num + win;
  const int s = blockIdx.x, g = threadIdx.x / TPF, t = threadIdx.x % TPF;
  const int slot = d.slot[s];
  const int64_t stride = rt_state_floats(win, d.lookahead);
  float* st = d.state + (int64_t)slot * stride;
  float* st_mag = st + (int64_t)nb * win;
  float* st_num = st_mag + (int64_t)nb * NBIN;
  int32_t* cnt = d.count + 2 * (int64_t)slot;
  int c = cnt[0], nbuf = cnt[1];
  float carry = st_num[win];
  fill_twiddles(tab);
  for (int i = threadIdx.x; i < nb * win; i += blockDim.x) fr[i] = st[i];
  for (int i = threadIdx.x; i < win; i += blockDim.x) num[i] = st_num[i];
  float* y = d.y + d.out_off[s];
  int64_t w = 0;  // samples written
  __syncthreads();

  // K Jacobi iterations over the buffered frames c .. c + nbuf - 1, the newest present frame being the last of them
  auto iterate = [&]() {
    for (int it = 0; it < d.n_iter; ++it) {
      rt_estimate(est, -h, (nbuf - 1) * hop + win, num, fr, c, nbuf, c + nbuf - 1, nb, win, hop);
      __syncthreads();
      const int F = c + g;
      const bool live = g < nbuf;
      rt_project(zb + (size_t)g * NC, nyq + g, tab, t, est + g * hop, st_mag + (int64_t)(F % nb) * NBIN,
                 fr + (size_t)(F % nb) * win, live, win);
      __syncthreads();
    }
  };
  // release samples c hop + r0 .. c hop + r0 + len - 1 of the numerator (frames 0 .. last <= c cover them), n >= 0
  // only, de-emphasised; positions relative to c hop as in rt_estimate, only the test n >= 0 forms c hop (in 64 bits)
  auto release = [&](int r0, int len, int last) {
    float* rel = est;
    for (int i = threadIdx.x; i < len; i += blockDim.x) {
      const int r = r0 + i;
      const int lo = c + rt_floordiv(r + h - win, hop) + 1, hi = c + min(rt_floordiv(r + h, hop), 1);
      float wss = 0.f;
      for (int F = max(lo, 0); F <= min(hi, last); ++F) {
        const float wv = hann(r - (F - c) * hop + h, win);
        wss += wv * wv;
      }
      const float acc = num[r + h];
      rel[i] = wss > FLT_MIN ? acc / wss : acc;
    }
    __syncthreads();
    const int64_t n0 = (int64_t)c * hop + r0;
    const int skip = n0 < 0 ? (int)min(-n0, (int64_t)len) : 0, cntw = len - skip;
    if (threadIdx.x == 0) {
      for (int i = skip; i < len; ++i) {
        carry = rel[i] + d.deemph * carry;
        rel[i] = carry;
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < cntw; i += blockDim.x) y[w + i] = rel[skip + i];
    w += cntw;
    __syncthreads();
  };
  // commit frame c: add it to the numerator, release the hop samples it completes, shift the numerator by hop
  auto commit = [&]() {
    const float* f = fr + (size_t)(c % nb) * win;
    for (int i = threadIdx.x; i < win; i += blockDim.x) num[i] += f[i];
    __syncthreads();
    release(-h, hop, c);
    float* tmp = est + win;
    for (int i = threadIdx.x; i < win; i += blockDim.x) tmp[i] = i + hop < win ? num[i + hop] : 0.f;
    __syncthreads();
    for (int i = threadIdx.x; i < win; i += blockDim.x) num[i] = tmp[i];
    __syncthreads();
    ++c;
    --nbuf;
  };

  for (int r = d.mag_off[s]; r < d.mag_off[s + 1]; ++r) {
    const int T = c + nbuf;  // the entering frame
    float* m = st_mag + (int64_t)(T % nb) * NBIN;
    for (int k = threadIdx.x; k < NBIN; k += blockDim.x) m[k] = __ldg(d.mag + (int64_t)r * NBIN + k);
    if (FROM) {  // start: X row r as given
      rt_project<true>(zb + (size_t)g * NC, nyq + g, tab, t, nullptr, nullptr, fr + (size_t)(T % nb) * win, g == 0, win,
                       X + (int64_t)r * NBIN);
    } else {
      // start phase: the estimate of the frames 0 .. T-1 over the entering frame's support
      rt_estimate(est, nbuf * hop - h, win, num, fr, c, nbuf, T - 1, nb, win, hop);
      __syncthreads();
      rt_project(zb + (size_t)g * NC, nyq + g, tab, t, est, m, fr + (size_t)(T % nb) * win, g == 0, win);
    }
    __syncthreads();
    ++nbuf;
    iterate();
    if (nbuf == nb) commit();
  }
  if (d.close[s]) {
    const int T = c + nbuf;
    while (nbuf > 0) {
      iterate();
      commit();
    }
    // the samples after the last commit's, T hop - win/2 .. hop (T - 1) - 1 (c = T now), where the grid ends: there are
    // some when hop < win/2 and T > 1 (for T = 1 they are all before sample 0)
    if (T > 1 && h > hop) release(-h, h - hop, T - 1);
  }
  for (int i = threadIdx.x; i < nb * win; i += blockDim.x) st[i] = fr[i];
  for (int i = threadIdx.x; i < win; i += blockDim.x) st_num[i] = num[i];
  if (threadIdx.x == 0) {
    st_num[win] = carry;
    cnt[0] = c;
    cnt[1] = nbuf;
  }
}

int check_audio(const avc_audio_desc* d, const char* who) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "%s: null descriptor", who);
  AVC_REQUIRE(d->n_fft == NFFT, AVC_ERR_UNSUPPORTED, "%s: only n_fft = %d is supported (got %d)", who, NFFT, d->n_fft);
  AVC_REQUIRE(d->win > 0 && d->win <= d->n_fft && d->win % 2 == 0, AVC_ERR_UNSUPPORTED,
              "%s: win must be even and in (0, n_fft] (got %d)", who, d->win);
  AVC_REQUIRE(d->hop > 0 && d->hop <= d->win, AVC_ERR_UNSUPPORTED, "%s: hop must be in (0, win] (got %d)", who, d->hop);
  AVC_REQUIRE(d->n_seg > 0 && d->segs != nullptr && d->n_frames >= 0 && d->n_samples >= 0, AVC_ERR_INVALID,
              "%s: empty or missing utterance table", who);
  return AVC_OK;
}

// The momentum of a projecting call.  X_prev is cleared when the momentum is 0, so the kernel takes the momentum
// branch exactly when X_prev is set.
int check_momentum(avc_audio_desc& d, const char* who) {
  const float m = d.momentum;
  AVC_REQUIRE(std::isfinite(m) && m >= 0.f && m < 1.f, AVC_ERR_INVALID, "%s: momentum must be in [0, 1) (got %g)", who,
              (double)m);
  if (m == 0.f) {
    d.X_prev = nullptr;
    return AVC_OK;
  }
  AVC_REQUIRE(d.X_prev != nullptr, AVC_ERR_INVALID, "%s: momentum > 0 needs X_prev", who);
  const uintptr_t p = (uintptr_t)d.X_prev, x = (uintptr_t)d.X, bytes = (uintptr_t)d.n_frames * NBIN * sizeof(float2);
  AVC_REQUIRE(p != x && (p + bytes <= x || x + bytes <= p), AVC_ERR_INVALID, "%s: X_prev overlaps X", who);
  return AVC_OK;
}

int check_tol(float tol, const char* who) {
  AVC_REQUIRE(std::isfinite(tol) && tol > 0.f && tol < 1.f, AVC_ERR_INVALID, "%s: tol must be in (0, 1) (got %g)", who,
              (double)tol);
  return AVC_OK;
}

int launch_pghi(const avc_audio_desc& d, float tol, int8_t* parent, cudaStream_t st) {
  if (d.n_frames == 0) return AVC_OK;
  pghi_kernel<<<d.n_seg, PG_THREADS, 0, st>>>(d, tol, parent);
  AVC_CHECK_LAUNCH("avc_pghi");
  return AVC_OK;
}

int launch_stft(const avc_audio_desc& d, cudaStream_t st, bool origin = false) {
  if (d.n_frames == 0) return AVC_OK;
  if (origin) stft_kernel<false, true><<<cdiv(d.n_frames, FPB), FFT_THREADS, 0, st>>>(d);
  else if (d.X_prev != nullptr) stft_kernel<true, false><<<cdiv(d.n_frames, FPB), FFT_THREADS, 0, st>>>(d);
  else stft_kernel<false, false><<<cdiv(d.n_frames, FPB), FFT_THREADS, 0, st>>>(d);
  AVC_CHECK_LAUNCH("avc_stft");
  return AVC_OK;
}

int launch_istft(const avc_audio_desc& d, cudaStream_t st) {
  if (d.n_frames > 0) {
    istft_frames_kernel<<<cdiv(d.n_frames, FPB), FFT_THREADS, 0, st>>>(d);
    AVC_CHECK_LAUNCH("avc_istft: frames");
  }
  if (d.n_samples > 0) {
    ola_kernel<<<(unsigned)cdiv64(d.n_samples, 256), 256, 0, st>>>(d);
    AVC_CHECK_LAUNCH("avc_istft: overlap-add");
  }
  return AVC_OK;
}

}  // namespace
}  // namespace avc

using namespace avc;

extern "C" int avc_stft(const avc_audio_desc* d, void* stream) {
  if (int rc = check_audio(d, "avc_stft")) return rc;
  AVC_REQUIRE(d->y != nullptr, AVC_ERR_INVALID, "avc_stft: null signal");
  const bool project = d->mode == AVC_STFT_PROJECT || d->mode == AVC_STFT_PROJECT_FIRST;
  AVC_REQUIRE(d->mode == AVC_STFT_MAG || d->mode == AVC_STFT_COMPLEX || project, AVC_ERR_INVALID,
              "avc_stft: unknown mode %d", d->mode);
  AVC_REQUIRE(d->mode != AVC_STFT_MAG || d->mag_out != nullptr || d->mag_db != nullptr, AVC_ERR_INVALID,
              "avc_stft: MAG needs mag_out or mag_db");
  AVC_REQUIRE(d->mode == AVC_STFT_MAG || d->X != nullptr, AVC_ERR_INVALID, "avc_stft: null X");
  AVC_REQUIRE(!project || d->mag != nullptr, AVC_ERR_INVALID, "avc_stft: PROJECT needs mag");
  AVC_REQUIRE(d->mode != AVC_STFT_MAG || d->mag_db == nullptr || d->max_db > 0.f, AVC_ERR_INVALID,
              "avc_stft: max_db must be positive");
  avc_audio_desc a = *d;
  if (project) {
    if (int rc = check_momentum(a, "avc_stft")) return rc;
  } else {
    a.X_prev = nullptr;
  }
  return launch_stft(a, (cudaStream_t)stream);
}

extern "C" int avc_stft_window(const avc_audio_desc* d, void* stream) {
  if (int rc = check_audio(d, "avc_stft_window")) return rc;
  AVC_REQUIRE(d->y != nullptr, AVC_ERR_INVALID, "avc_stft_window: null signal");
  AVC_REQUIRE(d->mode == AVC_STFT_MAG || d->mode == AVC_STFT_COMPLEX, AVC_ERR_INVALID,
              "avc_stft_window: mode must be MAG or COMPLEX (got %d)", d->mode);
  AVC_REQUIRE(d->mode != AVC_STFT_MAG || d->mag_out != nullptr || d->mag_db != nullptr, AVC_ERR_INVALID,
              "avc_stft_window: MAG needs mag_out or mag_db");
  AVC_REQUIRE(d->mode == AVC_STFT_MAG || d->X != nullptr, AVC_ERR_INVALID, "avc_stft_window: null X");
  AVC_REQUIRE(d->mode != AVC_STFT_MAG || d->mag_db == nullptr || d->max_db > 0.f, AVC_ERR_INVALID,
              "avc_stft_window: max_db must be positive");
  avc_audio_desc a = *d;
  a.X_prev = nullptr;
  return launch_stft(a, (cudaStream_t)stream, true);
}

extern "C" int avc_istft(const avc_audio_desc* d, void* stream) {
  if (int rc = check_audio(d, "avc_istft")) return rc;
  AVC_REQUIRE((d->X != nullptr || d->mag != nullptr) && d->frames != nullptr && d->y != nullptr, AVC_ERR_INVALID,
              "avc_istft: null X/mag, frames or y");
  return launch_istft(*d, (cudaStream_t)stream);
}

extern "C" int avc_griffin_lim_from(const avc_audio_desc* d, int32_t start, float tol, void* stream) {
  if (int rc = check_audio(d, "avc_griffin_lim")) return rc;
  AVC_REQUIRE(d->mag != nullptr && d->X != nullptr && d->frames != nullptr && d->y != nullptr, AVC_ERR_INVALID,
              "avc_griffin_lim: null mag, X, frames or y");
  AVC_REQUIRE(d->n_iter >= 0, AVC_ERR_INVALID, "avc_griffin_lim: n_iter < 0");
  AVC_REQUIRE(start == AVC_GL_START_ZERO || start == AVC_GL_START_X || start == AVC_GL_START_PGHI, AVC_ERR_INVALID,
              "avc_griffin_lim: unknown start %d", start);
  if (start == AVC_GL_START_PGHI) {
    if (int rc = check_tol(tol, "avc_griffin_lim")) return rc;
  }
  cudaStream_t st = (cudaStream_t)stream;
  avc_audio_desc a = *d;
  if (int rc = check_momentum(a, "avc_griffin_lim")) return rc;
  a.preemph = 0.f;
  // every argument is checked: the PGHI start is the call's first launch
  if (start == AVC_GL_START_PGHI) {
    if (int rc = launch_pghi(a, tol, nullptr, st)) return rc;
  }
  for (int it = 0; it <= a.n_iter; ++it) {
    avc_audio_desc s = a;
    if (it == 0 && start == AVC_GL_START_ZERO) s.X = nullptr;  // X = S with zero phase
    if (int rc = launch_istft(s, st)) return rc;
    if (it == a.n_iter) break;
    a.mode = it == 0 ? AVC_STFT_PROJECT_FIRST : AVC_STFT_PROJECT;  // the same projection when X_prev is null
    if (int rc = launch_stft(a, st)) return rc;
  }
  return AVC_OK;
}

extern "C" int avc_griffin_lim(const avc_audio_desc* d, void* stream) {
  return avc_griffin_lim_from(d, AVC_GL_START_ZERO, 0.f, stream);
}

extern "C" int avc_pghi(const avc_audio_desc* d, float tol, int8_t* parent, void* stream) {
  if (int rc = check_audio(d, "avc_pghi")) return rc;
  AVC_REQUIRE(d->mag != nullptr && d->X != nullptr, AVC_ERR_INVALID, "avc_pghi: null mag or X");
  if (int rc = check_tol(tol, "avc_pghi")) return rc;
  return launch_pghi(*d, tol, parent, (cudaStream_t)stream);
}

extern "C" int avc_frame_power(const avc_audio_desc* d, float* power, void* stream) {
  AVC_REQUIRE(d != nullptr && power != nullptr && d->y != nullptr && d->segs != nullptr && d->n_seg > 0, AVC_ERR_INVALID,
              "avc_frame_power: null argument or empty table");
  AVC_REQUIRE(d->n_fft > 0 && d->n_fft % 2 == 0 && d->hop > 0 && d->n_frames >= 0, AVC_ERR_INVALID,
              "avc_frame_power: bad frame length %d / hop %d", d->n_fft, d->hop);
  if (d->n_frames == 0) return AVC_OK;
  frame_power_kernel<<<(unsigned)cdiv64((int64_t)d->n_frames * 32, 256), 256, 0, (cudaStream_t)stream>>>(*d, power);
  AVC_CHECK_LAUNCH("avc_frame_power");
  return AVC_OK;
}

extern "C" int avc_deemphasis(const avc_audio_desc* d, float coef, void* stream) {
  AVC_REQUIRE(d != nullptr && d->y != nullptr && d->segs != nullptr && d->n_seg > 0, AVC_ERR_INVALID,
              "avc_deemphasis: null argument or empty table");
  deemphasis_kernel<<<d->n_seg, 1024, 0, (cudaStream_t)stream>>>(*d, coef);
  AVC_CHECK_LAUNCH("avc_deemphasis");
  return AVC_OK;
}

extern "C" int avc_mel_project(const avc_mel_desc* d, void* stream) {
  AVC_REQUIRE(d != nullptr && d->in != nullptr && d->mat != nullptr && d->out != nullptr, AVC_ERR_INVALID,
              "avc_mel_project: null argument");
  AVC_REQUIRE(d->rows >= 0 && d->n_mels > 0 && d->n_bins > 0 && d->max_db > 0.f, AVC_ERR_INVALID,
              "avc_mel_project: bad shape rows=%d n_mels=%d n_bins=%d", d->rows, d->n_mels, d->n_bins);
  AVC_REQUIRE(d->dir == AVC_MEL_TO_MAG || d->dir == AVC_MAG_TO_MEL, AVC_ERR_INVALID, "avc_mel_project: unknown dir %d", d->dir);
  if (d->rows == 0) return AVC_OK;
  const int N = d->dir == AVC_MEL_TO_MAG ? d->n_bins : d->n_mels;
  // gridDim.x (column tiles) allows 2^31 - 1, more than any int N needs; gridDim.y is clamped and looped over
  const dim3 grid(cdiv(N, 64), min(cdiv(d->rows, 64), 65535));
  cudaStream_t st = (cudaStream_t)stream;
  if (d->dir == AVC_MEL_TO_MAG) mel_gemm_kernel<AVC_MEL_TO_MAG><<<grid, 256, 0, st>>>(*d);
  else mel_gemm_kernel<AVC_MAG_TO_MEL><<<grid, 256, 0, st>>>(*d);
  AVC_CHECK_LAUNCH("avc_mel_project");
  return AVC_OK;
}

extern "C" int64_t avc_rtisi_state_floats(int win, int lookahead) {
  if (win <= 0 || lookahead < 0) return 0;
  return rt_state_floats(win, lookahead);
}

// avc_rtisi_la's checks (who names the entry point), then the launch of its FROM or estimate instance
static int rtisi_launch(const avc_rtisi_desc* d, const float2* X, const char* who, cudaStream_t stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "%s: null descriptor", who);
  AVC_REQUIRE(d->n_fft == NFFT, AVC_ERR_UNSUPPORTED, "%s: only n_fft = %d is supported (got %d)", who, NFFT, d->n_fft);
  AVC_REQUIRE(d->win > 0 && d->win <= NFFT && d->win % 2 == 0, AVC_ERR_UNSUPPORTED,
              "%s: win must be even and in (0, n_fft] (got %d)", who, d->win);
  AVC_REQUIRE(d->hop > 0 && 2 * d->hop <= d->win, AVC_ERR_UNSUPPORTED, "%s: hop must be in (0, win/2] (got %d)", who,
              d->hop);
  AVC_REQUIRE(d->lookahead >= 0 && d->lookahead <= RT_MAX_LA, AVC_ERR_UNSUPPORTED,
              "%s: lookahead must be in [0, %d] (got %d)", who, RT_MAX_LA, d->lookahead);
  AVC_REQUIRE(d->n_iter >= 0, AVC_ERR_INVALID, "%s: n_iter < 0", who);
  AVC_REQUIRE(d->n_streams >= 0, AVC_ERR_INVALID, "%s: n_streams < 0", who);
  AVC_REQUIRE(std::isfinite(d->deemph), AVC_ERR_INVALID, "%s: de-emphasis coefficient is not finite", who);
  if (d->n_streams == 0) return AVC_OK;
  AVC_REQUIRE(d->mag && d->mag_off && d->slot && d->close && d->out_off && d->y && d->state && d->count, AVC_ERR_INVALID,
              "%s: null pointer", who);
  const bool from = X != nullptr;
  auto kernel = from ? rtisi_kernel<true> : rtisi_kernel<false>;
  RtSmem L{d->lookahead + 1, d->win, d->hop};
  const size_t smem = L.bytes();
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  AVC_REQUIRE(e == cudaSuccess, AVC_ERR_CUDA, "%s: cudaFuncSetAttribute(%zu bytes): %s", who, smem,
              cudaGetErrorString(e));
  kernel<<<d->n_streams, L.nb * TPF, smem, stream>>>(*d, L, X);
  AVC_CHECK_LAUNCH(who);
  return AVC_OK;
}

extern "C" int avc_rtisi_la(const avc_rtisi_desc* d, void* stream) {
  return rtisi_launch(d, nullptr, "avc_rtisi_la", (cudaStream_t)stream);
}

extern "C" int avc_rtisi_la_from(const avc_rtisi_desc* d, const float* X, void* stream) {
  AVC_REQUIRE(X != nullptr, AVC_ERR_INVALID, "avc_rtisi_la_from: null X");
  return rtisi_launch(d, reinterpret_cast<const float2*>(X), "avc_rtisi_la_from", (cudaStream_t)stream);
}

extern "C" int64_t avc_pghi_stream_state_floats(int n_fft) { return n_fft == NFFT ? PS_FLOATS : 0; }

extern "C" int avc_pghi_stream(const avc_pghi_stream_desc* d, float tol, int8_t* parent, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "avc_pghi_stream: null descriptor");
  AVC_REQUIRE(d->n_fft == NFFT, AVC_ERR_UNSUPPORTED, "avc_pghi_stream: only n_fft = %d is supported (got %d)", NFFT,
              d->n_fft);
  AVC_REQUIRE(d->win > 0 && d->win <= NFFT && d->win % 2 == 0, AVC_ERR_UNSUPPORTED,
              "avc_pghi_stream: win must be even and in (0, n_fft] (got %d)", d->win);
  AVC_REQUIRE(d->hop > 0 && 2 * d->hop <= d->win, AVC_ERR_UNSUPPORTED,
              "avc_pghi_stream: hop must be in (0, win/2] (got %d)", d->hop);
  AVC_REQUIRE(d->n_streams >= 0, AVC_ERR_INVALID, "avc_pghi_stream: n_streams < 0");
  if (int rc = check_tol(tol, "avc_pghi_stream")) return rc;
  if (d->n_streams == 0) return AVC_OK;
  AVC_REQUIRE(d->mag && d->mag_off && d->slot && d->close && d->out_off && d->mag_out && d->X && d->state,
              AVC_ERR_INVALID, "avc_pghi_stream: null pointer");
  pghi_kernel<<<d->n_streams, PG_THREADS, 0, (cudaStream_t)stream>>>(*d, tol, parent);
  AVC_CHECK_LAUNCH("avc_pghi_stream");
  return AVC_OK;
}
