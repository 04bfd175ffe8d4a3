// Speaker measures of the held-out sets (speaker_eval.py): statistics pooling of padded batches, the cosine scores of
// every pair of a set with the EER of those trials, and group-mean similarities.
//
// avc_time_stats_varlen: one thread per (sample, channel) walks its own row twice, ascending t: the float64 sum for the
// mean, then the squared deviations.
//
// avc_spk_eer: the trials i < j are cut into 64 x 64 tiles (ti <= tj).  spk_score_kernel computes a tile's dot products
// like a GEMM (both operands staged in shared memory as float64 in chunks of 32 coordinates), each dot added in
// ascending d, and stores the order-preserving 64-bit key of every score in the workspace.  The EER threshold is then
// found by counting, not sorting: three MSD radix searches over the keys (six digits of 11, 11, 11, 11, 11 and 9 bits),
// each pass a histogram of target and non-target trials in the current bucket (spk_hist_kernel: 32-bit shared counts,
// 64-bit integer global counts) and a one-CTA step that picks the next digit (spk_step_kernel).  Every search finds the
// largest key k with F(k) = alpha #{target < k} + beta #{non-target < k} - gamma < 0 for a non-decreasing F:
//   search 0: alpha = n_nontarget, beta = n_target, gamma = n_target n_nontarget: k = m, the largest score with
//             FRR(m) < FAR(m).  Its successor m+ is the first candidate with FRR >= FAR, so the EER is
//             min(FAR(m), FRR(m+)).
//   search 1: when FRR(m+) < FAR(m), the key at rank #{all <= m} (m+ itself); otherwise, when no non-target lies
//             below m, the smallest key; otherwise the non-target key q at rank #{non-target < m} - 1.
//   search 2: (only after q) the key at rank #{all <= q}: the smallest candidate above q, the smallest threshold whose
//             FAR is FAR(m).
// Integer counts are exact and order-free, so the result does not depend on the order of the set or of the launches.
// Every float64 operation of a score is an explicitly rounded intrinsic (no contraction into an FMA), so the scores
// equal a float64 restatement that adds in the same order, and s(a, b) == s(b, a).
#include "common.cuh"

namespace avc {

constexpr int SPK_TILE = 64;       // trials per tile side
constexpr int SPK_KC = 32;         // coordinates per staged chunk
constexpr int SPK_THREADS = 256;
constexpr int SPK_BINS = 2048;     // 11-bit digits
constexpr int SPK_STEP_THREADS = 1024;
constexpr int SPK_PASSES = 6;
constexpr int SPK_SEARCHES = 3;
static_assert(SPK_BINS == 2 * SPK_STEP_THREADS, "each step thread owns two bins");

struct SpkSearch {
  unsigned long long lo;            // bucket start (the key once the search is done)
  long long t_lt, n_lt;             // targets / non-targets below lo
  long long t_eq, n_eq;             // ... at the key (last pass)
  long long alpha, beta, gamma;
  int active, pad;
};

struct SpkState {
  unsigned long long hist[2][SPK_BINS];   // [target, non-target][bin] of the current pass
  long long n_target, n_nontarget;
  int after_q, pad;                       // search 1 found q: search 2 runs
  SpkSearch s[SPK_SEARCHES];
};
static_assert(sizeof(SpkState) <= AVC_SPK_STATE_BYTES, "the state must fit its workspace region");

__device__ __forceinline__ unsigned long long score_key(double s) {
  if (s == 0.0) s = 0.0;   // one key for +0 and -0
  const unsigned long long b = (unsigned long long)__double_as_longlong(s);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

__device__ __forceinline__ double key_score(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// s = dot / (sqrt(na) sqrt(nb)); 0 when either norm is 0
__device__ __forceinline__ double cosine(double dot, double ra, double rb) {
  return (ra == 0.0 || rb == 0.0) ? 0.0 : __ddiv_rn(dot, __dmul_rn(ra, rb));
}

// ---------------------------------------------------------------- statistics pooling
__global__ void __launch_bounds__(256) time_stats_kernel(const float* __restrict__ x, float* __restrict__ out, int B,
                                                         int C, int T, const int32_t* __restrict__ lens) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= (int64_t)B * C) return;
  const int b = (int)(row / C), c = (int)(row - (int64_t)b * C);
  const int L = __ldg(lens + b);
  float* o = out + (int64_t)b * 2 * C;
  if (L < 1 || L > T) {
    o[c] = o[C + c] = __int_as_float(0x7fc00000);
    return;
  }
  const float* p = x + row * T;
  double s = 0.0;
  for (int t = 0; t < L; ++t) s = __dadd_rn(s, (double)__ldg(p + t));
  const double mean = __ddiv_rn(s, (double)L);
  double v = 0.0;
  for (int t = 0; t < L; ++t) {
    const double e = __dsub_rn((double)__ldg(p + t), mean);
    v = __dadd_rn(v, __dmul_rn(e, e));
  }
  o[c] = (float)mean;
  o[C + c] = (float)__dsqrt_rn(__ddiv_rn(v, (double)L));
}

// ---------------------------------------------------------------- norms and scores
// rnorm[i] = sqrt(sum_d v[i][d]^2), ascending d
__global__ void __launch_bounds__(256) spk_norm_kernel(const float* __restrict__ v, int n, int d, double* __restrict__ rnorm,
                                                      SpkState* st) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (int e = i; e < 2 * SPK_BINS; e += gridDim.x * blockDim.x) (&st->hist[0][0])[e] = 0ull;
  if (i == 0) {   // search 0 starts over every key; its F is set from the first pass's totals
    st->s[0].lo = 0;
    st->s[0].t_lt = st->s[0].n_lt = st->s[0].t_eq = st->s[0].n_eq = 0;
    st->s[0].active = 1;
    st->after_q = 0;
  }
  if (i >= n) return;
  const float* p = v + (int64_t)i * d;
  double acc = 0.0;
  for (int k = 0; k < d; ++k) {
    const double a = (double)__ldg(p + k);
    acc = __dadd_rn(acc, __dmul_rn(a, a));
  }
  rnorm[i] = __dsqrt_rn(acc);
}

__device__ __forceinline__ int64_t tile_index(int ti, int tj) { return (int64_t)tj * (tj + 1) / 2 + ti; }

// one 64 x 64 tile (ti <= tj) per CTA; thread (tx, ty) owns rows ty + 16 r and columns tx + 16 c
__global__ void __launch_bounds__(SPK_THREADS) spk_score_kernel(const float* __restrict__ v, int n, int d,
                                                                const double* __restrict__ rnorm,
                                                                unsigned long long* __restrict__ keys) {
  const int tj = blockIdx.x, ti = blockIdx.y;
  if (ti > tj) return;
  __shared__ double As[SPK_KC][SPK_TILE + 1];
  __shared__ double Bs[SPK_KC][SPK_TILE + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
  for (int k0 = 0; k0 < d; k0 += SPK_KC) {
    for (int e = threadIdx.x; e < SPK_TILE * SPK_KC; e += SPK_THREADS) {
      const int r = e / SPK_KC, k = e - r * SPK_KC;
      const int ia = ti * SPK_TILE + r, ib = tj * SPK_TILE + r;
      const bool kin = k0 + k < d;
      As[k][r] = (kin && ia < n) ? (double)__ldg(v + (int64_t)ia * d + k0 + k) : 0.0;
      Bs[k][r] = (kin && ib < n) ? (double)__ldg(v + (int64_t)ib * d + k0 + k) : 0.0;
    }
    __syncthreads();
    // zero-padded coordinates add +0 to a sum that is never -0: the same bits as stopping at d
#pragma unroll 4
    for (int k = 0; k < SPK_KC; ++k) {
      double a[4], b[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) a[r] = As[k][ty + 16 * r];
#pragma unroll
      for (int c = 0; c < 4; ++c) b[c] = Bs[k][tx + 16 * c];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = __dadd_rn(acc[r][c], __dmul_rn(a[r], b[c]));
    }
    __syncthreads();
  }
  unsigned long long* out = keys + tile_index(ti, tj) * (SPK_TILE * SPK_TILE);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = ti * SPK_TILE + ty + 16 * r;
    const double ra = i < n ? rnorm[i] : 0.0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = tj * SPK_TILE + tx + 16 * c;
      const double rb = j < n ? rnorm[j] : 0.0;
      out[(ty + 16 * r) * SPK_TILE + tx + 16 * c] = score_key(cosine(acc[r][c], ra, rb));
    }
  }
}

// ---------------------------------------------------------------- the radix searches
__host__ __device__ constexpr int pass_shift(int p) { return p < SPK_PASSES - 1 ? 64 - 11 * (p + 1) : 0; }
__host__ __device__ constexpr int pass_width(int p) { return p < SPK_PASSES - 1 ? 11 : 64 - 11 * (SPK_PASSES - 1); }

__global__ void __launch_bounds__(SPK_THREADS) spk_hist_kernel(const unsigned long long* __restrict__ keys,
                                                               const int32_t* __restrict__ labels, int n, SpkState* st,
                                                               int q, int pass) {
  const int tj = blockIdx.x, ti = blockIdx.y;
  if (ti > tj || !st->s[q].active) return;
  __shared__ unsigned h[2][SPK_BINS];
  __shared__ int li[SPK_TILE], lj[SPK_TILE];
  for (int e = threadIdx.x; e < 2 * SPK_BINS; e += SPK_THREADS) (&h[0][0])[e] = 0u;
  if (threadIdx.x < SPK_TILE) {
    const int i = ti * SPK_TILE + threadIdx.x, j = tj * SPK_TILE + threadIdx.x;
    li[threadIdx.x] = i < n ? labels[i] : 0;
    lj[threadIdx.x] = j < n ? labels[j] : 0;
  }
  __syncthreads();
  const int shift = pass_shift(pass), top = shift + pass_width(pass);
  const unsigned long long lo = st->s[q].lo, mask = (1ull << pass_width(pass)) - 1;
  const unsigned long long* tk = keys + tile_index(ti, tj) * (SPK_TILE * SPK_TILE);
  for (int e = threadIdx.x; e < SPK_TILE * SPK_TILE; e += SPK_THREADS) {
    const int r = e / SPK_TILE, c = e - r * SPK_TILE;
    const int i = ti * SPK_TILE + r, j = tj * SPK_TILE + c;
    if (i >= j || j >= n) continue;
    const unsigned long long k = tk[e];
    if (top < 64 && (k >> top) != (lo >> top)) continue;
    atomicAdd(&h[li[r] == lj[c] ? 0 : 1][(k >> shift) & mask], 1u);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 2 * SPK_BINS; e += SPK_THREADS) {
    const unsigned c = (&h[0][0])[e];
    if (c) atomicAdd(&st->hist[0][0] + e, (unsigned long long)c);
  }
}

// inclusive block scan of (t, n) pairs over SPK_STEP_THREADS threads
__device__ void scan_pairs(long long& t, long long& nn, long long* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long a = __shfl_up_sync(0xffffffffu, t, o), b = __shfl_up_sync(0xffffffffu, nn, o);
    if (lane >= o) {
      t += a;
      nn += b;
    }
  }
  if (lane == 31) {
    sh[2 * w] = t;
    sh[2 * w + 1] = nn;
  }
  __syncthreads();
  if (w == 0) {
    long long a = sh[2 * lane], b = sh[2 * lane + 1];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long x = __shfl_up_sync(0xffffffffu, a, o), y = __shfl_up_sync(0xffffffffu, b, o);
      if (lane >= o) {
        a += x;
        b += y;
      }
    }
    sh[64 + 2 * lane] = a;
    sh[64 + 2 * lane + 1] = b;
  }
  __syncthreads();
  if (w > 0) {
    t += sh[64 + 2 * (w - 1)];
    nn += sh[64 + 2 * (w - 1) + 1];
  }
}

// the next search's F from the finished ones (before its first histogram pass)
__device__ void setup_search(SpkState* st, int q) {
  SpkSearch& s = st->s[q];
  const SpkSearch& m = st->s[0];
  s.lo = 0;
  s.t_lt = s.n_lt = s.t_eq = s.n_eq = 0;
  if (q == 1) {
    const long long nT = st->n_target, nN = st->n_nontarget;
    const bool succ = (m.t_lt + m.t_eq) * nN < (nN - m.n_lt) * nT;   // FRR(m+) < FAR(m): the threshold is m+
    s.active = m.active;
    st->after_q = m.active && !succ && m.n_lt > 0;
    s.alpha = st->after_q ? 0 : 1;
    s.beta = 1;
    s.gamma = succ ? m.t_lt + m.n_lt + m.t_eq + m.n_eq + 1 : (m.n_lt > 0 ? m.n_lt : 1);
  } else {
    const SpkSearch& p = st->s[1];
    s.active = st->after_q;
    s.alpha = s.beta = 1;
    s.gamma = p.t_lt + p.n_lt + p.t_eq + p.n_eq + 1;
  }
}

// after pass `pass` of search q: pick the digit, clear the histogram, set the next search up after the last pass
__global__ void __launch_bounds__(SPK_STEP_THREADS) spk_step_kernel(SpkState* st, int q, int pass) {
  __shared__ long long sh[128];
  SpkSearch& s = st->s[q];
  const int b0 = 2 * threadIdx.x;
  const long long t0 = (long long)st->hist[0][b0], t1 = (long long)st->hist[0][b0 + 1];
  const long long n0 = (long long)st->hist[1][b0], n1 = (long long)st->hist[1][b0 + 1];
  st->hist[0][b0] = st->hist[0][b0 + 1] = st->hist[1][b0] = st->hist[1][b0 + 1] = 0ull;
  long long ti = t0 + t1, ni = n0 + n1;   // inclusive prefix after the scan
  scan_pairs(ti, ni, sh);
  if (q == 0 && pass == 0 && threadIdx.x == SPK_STEP_THREADS - 1) {   // the first pass counted every trial
    st->n_target = ti;
    st->n_nontarget = ni;
    s.active = ti > 0 && ni > 0;
    s.alpha = ni;
    s.beta = ti;
    s.gamma = ti * ni;
  }
  __syncthreads();
  if (s.active) {
    const long long te0 = ti - t0 - t1, ne0 = ni - n0 - n1;   // exclusive prefix at bin b0
    const long long A = s.alpha, Bt = s.beta, G = s.gamma, tl = s.t_lt, nl = s.n_lt;
    auto F = [&](long long tx, long long nx) { return A * (tl + tx) + Bt * (nl + nx) - G; };
    const long long f0 = F(te0, ne0), f1 = F(te0 + t0, ne0 + n0), f2 = F(ti, ni);
    // F(bucket start) < 0 <= F(bucket end + 1): exactly one bin starts below 0 and ends at or above it
    int win = -1;
    long long wt = 0, wn = 0, et = 0, en = 0;
    if (f0 < 0 && f1 >= 0) {
      win = b0;
      wt = te0, wn = ne0, et = t0, en = n0;
    } else if (f1 < 0 && (f2 >= 0 || b0 + 1 == SPK_BINS - 1)) {
      win = b0 + 1;
      wt = te0 + t0, wn = ne0 + n0, et = t1, en = n1;
    }
    __syncthreads();   // every thread has read the search state
    if (win >= 0) {
      s.lo += (unsigned long long)win << pass_shift(pass);
      s.t_lt = tl + wt;
      s.n_lt = nl + wn;
      s.t_eq = et;
      s.n_eq = en;
    }
  }
  if (pass == SPK_PASSES - 1 && q + 1 < SPK_SEARCHES) {
    __syncthreads();
    if (threadIdx.x == 0) setup_search(st, q + 1);
  }
}

__global__ void spk_result_kernel(const SpkState* st, avc_eer_result* out) {
  const long long nT = st->n_target, nN = st->n_nontarget;
  avc_eer_result r;
  r.n_target = nT;
  r.n_nontarget = nN;
  if (!st->s[0].active) {
    r.eer = r.threshold = r.frr = r.far = __longlong_as_double(0x7ff8000000000000ll);
  } else {
    const SpkSearch& t = st->s[st->after_q ? 2 : 1];
    r.threshold = key_score(t.lo);
    r.frr = __ddiv_rn((double)t.t_lt, (double)nT);
    r.far = __ddiv_rn((double)(nN - t.n_lt), (double)nN);
    r.eer = fmax(r.frr, r.far);
  }
  *out = r;
}

// ---------------------------------------------------------------- query scores
// The block stages query q (float32, promoted) in qv[D]; after a __syncthreads thread 0 writes *rq = sqrt(sum_k q[k]^2),
// ascending k.  The caller syncs again before reading *rq.
__device__ __forceinline__ void stage_query(const float* __restrict__ q, int D, double* qv, double* rq) {
  for (int k = threadIdx.x; k < D; k += blockDim.x) qv[k] = (double)__ldg(q + k);
  __syncthreads();
  if (threadIdx.x == 0) {
    double acc = 0.0;
    for (int k = 0; k < D; ++k) acc = __dadd_rn(acc, __dmul_rn(qv[k], qv[k]));
    *rq = __dsqrt_rn(acc);
  }
}

// s(q, v) of the staged query (qv, rq) and the float32 row p[D]: dot(q, v) and |v|^2 each added in ascending k
__device__ __forceinline__ double staged_score(const double* qv, double rq, const float* __restrict__ p, int D) {
  double dot = 0.0, nv = 0.0;
  for (int k = 0; k < D; ++k) {
    const double b = (double)__ldg(p + k);
    dot = __dadd_rn(dot, __dmul_rn(qv[k], b));
    nv = __dadd_rn(nv, __dmul_rn(b, b));
  }
  return cosine(dot, rq, __dsqrt_rn(nv));
}

// ---------------------------------------------------------------- group means
constexpr int SPK_MAX_EXCLUDE = 64;

// q_exclude read as [m][n_ex]: query m skips every v its list names (n_ex = 1: avc_spk_group_mean)
__global__ void __launch_bounds__(SPK_THREADS) spk_group_mean_kernel(const avc_spk_group_desc d, int n_ex) {
  extern __shared__ double qv[];   // [dims]
  __shared__ double sc[SPK_THREADS];
  __shared__ int ok[SPK_THREADS];
  __shared__ int exl[SPK_MAX_EXCLUDE];
  __shared__ double rq;
  const int m = blockIdx.x, D = d.dims;
  if (threadIdx.x < n_ex) exl[threadIdx.x] = __ldg(d.q_exclude + (int64_t)m * n_ex + threadIdx.x);
  stage_query(d.queries + (int64_t)m * D, D, qv, &rq);
  const int lab = __ldg(d.q_labels + m);
  double sum = 0.0;
  long long cnt = 0;
  for (int base = 0; base < d.n; base += SPK_THREADS) {
    const int v = base + threadIdx.x;
    __syncthreads();   // rq is written; the previous chunk's scores are consumed
    bool excluded = false;
    for (int e = 0; e < n_ex; ++e) excluded |= v == exl[e];
    const bool take = v < d.n && !excluded && __ldg(d.labels + v) == lab;
    ok[threadIdx.x] = take;
    if (take) sc[threadIdx.x] = staged_score(qv, rq, d.set + (int64_t)v * D, D);
    __syncthreads();
    if (threadIdx.x == 0)
      for (int t = 0; t < SPK_THREADS; ++t)
        if (ok[t]) {
          sum = __dadd_rn(sum, sc[t]);
          ++cnt;
        }
  }
  if (threadIdx.x == 0) d.out[m] = cnt ? __ddiv_rn(sum, (double)cnt) : __longlong_as_double(0x7ff8000000000000ll);
}

// ---------------------------------------------------------------- identification against a bank
// (score, index) a beats (score, index) b: a higher score, or the same score at a lower index; index -1 is "none yet"
__device__ __forceinline__ bool beats(double sa, int ia, double sb, int ib) {
  return ia >= 0 && (ib < 0 || sa > sb || (sa == sb && ia < ib));
}

// one CTA per query: the target's score first (thread 0), then every bank row, each thread keeping its best row and
// its count of rows above the target; a warp then a block reduction combines them
__global__ void __launch_bounds__(SPK_THREADS) spk_identify_kernel(const avc_spk_identify_desc d) {
  extern __shared__ double qv[];   // [dims]
  __shared__ double rq, tsc;
  __shared__ double w_best[SPK_THREADS / 32];
  __shared__ int w_idx[SPK_THREADS / 32], w_above[SPK_THREADS / 32];
  const int m = blockIdx.x, D = d.dims;
  stage_query(d.queries + (int64_t)m * D, D, qv, &rq);
  __syncthreads();
  const int t = d.q_target ? __ldg(d.q_target + m) : -1;
  const bool has_t = t >= 0 && t < d.s;
  if (threadIdx.x == 0) tsc = has_t ? staged_score(qv, rq, d.bank + (int64_t)t * D, D) : __longlong_as_double(0x7ff8000000000000ll);
  __syncthreads();
  const double ts = tsc, r = rq;
  double best = 0.0;
  int idx = -1, above = 0;
  for (int v = threadIdx.x; v < d.s; v += SPK_THREADS) {
    const double sc = staged_score(qv, r, d.bank + (int64_t)v * D, D);
    if (beats(sc, v, best, idx)) {
      best = sc;
      idx = v;
    }
    above += sc > ts;   // never with no target: ts is NaN
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ob = __shfl_down_sync(0xffffffffu, best, o);
    const int oi = __shfl_down_sync(0xffffffffu, idx, o);
    above += __shfl_down_sync(0xffffffffu, above, o);
    if (beats(ob, oi, best, idx)) {
      best = ob;
      idx = oi;
    }
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    w_best[w] = best;
    w_idx[w] = idx;
    w_above[w] = above;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < SPK_THREADS / 32; ++k) {
      if (beats(w_best[k], w_idx[k], best, idx)) {
        best = w_best[k];
        idx = w_idx[k];
      }
      above += w_above[k];
    }
    d.best[m] = idx;
    d.best_score[m] = best;
    d.target_score[m] = ts;
    d.target_rank[m] = has_t ? above : -1;
  }
}

int64_t eer_tiles(int n) {
  const int64_t nt = cdiv64(n, SPK_TILE);
  return nt * (nt + 1) / 2;
}

}  // namespace avc

using namespace avc;

extern "C" int avc_time_stats_varlen(const float* x, float* out, int B, int C, int T, const int32_t* lengths, void* stream) {
  AVC_REQUIRE(x != nullptr && out != nullptr && lengths != nullptr, AVC_ERR_INVALID,
              "avc_time_stats_varlen: null pointer (x %p, out %p, lengths %p)", (const void*)x, (const void*)out,
              (const void*)lengths);
  AVC_REQUIRE(B > 0 && C > 0 && T > 0, AVC_ERR_INVALID, "avc_time_stats_varlen: sizes must be positive (B %d, C %d, T %d)",
              B, C, T);
  const int64_t rows = (int64_t)B * C;
  time_stats_kernel<<<(unsigned)cdiv64(rows, 256), 256, 0, (cudaStream_t)stream>>>(x, out, B, C, T, lengths);
  AVC_CHECK_LAUNCH("avc_time_stats_varlen");
  return AVC_OK;
}

extern "C" int64_t avc_spk_eer_workspace_bytes(int n) {
  if (n < 1 || n > AVC_SPK_MAX_N) return -1;
  return AVC_SPK_STATE_BYTES + cdiv64(8 * (int64_t)n, 256) * 256 + eer_tiles(n) * SPK_TILE * SPK_TILE * 8;
}

extern "C" int avc_spk_eer(const float* vecs, const int32_t* labels, int n, int dims, void* workspace,
                           int64_t workspace_bytes, avc_eer_result* out, void* stream) {
  AVC_REQUIRE(vecs != nullptr && labels != nullptr && workspace != nullptr && out != nullptr, AVC_ERR_INVALID,
              "avc_spk_eer: null pointer (vecs %p, labels %p, workspace %p, out %p)", (const void*)vecs,
              (const void*)labels, workspace, (const void*)out);
  AVC_REQUIRE(n > 0 && dims > 0, AVC_ERR_INVALID, "avc_spk_eer: sizes must be positive (n %d, dims %d)", n, dims);
  AVC_REQUIRE(n <= AVC_SPK_MAX_N, AVC_ERR_UNSUPPORTED, "avc_spk_eer: n %d > %d", n, AVC_SPK_MAX_N);
  AVC_REQUIRE(dims <= AVC_SPK_MAX_DIMS, AVC_ERR_UNSUPPORTED, "avc_spk_eer: dims %d > %d", dims, AVC_SPK_MAX_DIMS);
  const int64_t need = avc_spk_eer_workspace_bytes(n);
  AVC_REQUIRE(workspace_bytes >= need, AVC_ERR_INVALID, "avc_spk_eer: workspace of %lld bytes; %lld needed",
              (long long)workspace_bytes, (long long)need);
  AVC_REQUIRE(((uintptr_t)workspace & 255) == 0, AVC_ERR_INVALID, "avc_spk_eer: workspace %p is not 256-byte aligned",
              workspace);
  cudaStream_t st = (cudaStream_t)stream;
  SpkState* state = reinterpret_cast<SpkState*>(workspace);
  double* rnorm = reinterpret_cast<double*>(static_cast<char*>(workspace) + AVC_SPK_STATE_BYTES);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(static_cast<char*>(workspace) + AVC_SPK_STATE_BYTES +
                                                                   cdiv64(8 * (int64_t)n, 256) * 256);
  spk_norm_kernel<<<(unsigned)cdiv64(n > 2 * SPK_BINS ? n : 2 * SPK_BINS, 256), 256, 0, st>>>(vecs, n, dims, rnorm, state);
  AVC_CHECK_LAUNCH("avc_spk_eer: norms");
  const int nt = (int)cdiv64(n, SPK_TILE);
  const dim3 grid(nt, nt);
  spk_score_kernel<<<grid, SPK_THREADS, 0, st>>>(vecs, n, dims, rnorm, keys);
  AVC_CHECK_LAUNCH("avc_spk_eer: scores");
  for (int q = 0; q < SPK_SEARCHES; ++q)
    for (int p = 0; p < SPK_PASSES; ++p) {
      spk_hist_kernel<<<grid, SPK_THREADS, 0, st>>>(keys, labels, n, state, q, p);
      AVC_CHECK_LAUNCH("avc_spk_eer: histogram");
      spk_step_kernel<<<1, SPK_STEP_THREADS, 0, st>>>(state, q, p);
      AVC_CHECK_LAUNCH("avc_spk_eer: step");
    }
  spk_result_kernel<<<1, 1, 0, st>>>(state, out);
  AVC_CHECK_LAUNCH("avc_spk_eer: result");
  return AVC_OK;
}

static int group_mean(const avc_spk_group_desc* d, int n_exclude, const char* what, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "%s: null descriptor", what);
  AVC_REQUIRE(d->queries != nullptr && d->q_labels != nullptr && d->q_exclude != nullptr && d->set != nullptr &&
                  d->labels != nullptr && d->out != nullptr,
              AVC_ERR_INVALID, "%s: null pointer (queries %p, q_labels %p, q_exclude %p, set %p, labels %p, out %p)", what,
              (const void*)d->queries, (const void*)d->q_labels, (const void*)d->q_exclude, (const void*)d->set,
              (const void*)d->labels, (const void*)d->out);
  AVC_REQUIRE(d->m > 0 && d->n > 0 && d->dims > 0, AVC_ERR_INVALID, "%s: sizes must be positive (m %d, n %d, dims %d)",
              what, d->m, d->n, d->dims);
  AVC_REQUIRE(n_exclude >= 1 && n_exclude <= SPK_MAX_EXCLUDE, AVC_ERR_INVALID, "%s: n_exclude %d must lie in [1, %d]",
              what, n_exclude, SPK_MAX_EXCLUDE);
  AVC_REQUIRE(d->n <= AVC_SPK_MAX_N, AVC_ERR_UNSUPPORTED, "%s: n %d > %d", what, d->n, AVC_SPK_MAX_N);
  AVC_REQUIRE(d->dims <= AVC_SPK_MAX_DIMS, AVC_ERR_UNSUPPORTED, "%s: dims %d > %d", what, d->dims, AVC_SPK_MAX_DIMS);
  spk_group_mean_kernel<<<(unsigned)d->m, SPK_THREADS, d->dims * 8, (cudaStream_t)stream>>>(*d, n_exclude);
  AVC_CHECK_LAUNCH(what);
  return AVC_OK;
}

extern "C" int avc_spk_group_mean(const avc_spk_group_desc* d, void* stream) {
  return group_mean(d, 1, "avc_spk_group_mean", stream);
}

extern "C" int avc_spk_group_mean_multi(const avc_spk_group_desc* d, int n_exclude, void* stream) {
  return group_mean(d, n_exclude, "avc_spk_group_mean_multi", stream);
}

extern "C" int avc_spk_identify(const avc_spk_identify_desc* d, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "avc_spk_identify: null descriptor");
  AVC_REQUIRE(d->queries != nullptr && d->bank != nullptr && d->best != nullptr && d->best_score != nullptr &&
                  d->target_score != nullptr && d->target_rank != nullptr,
              AVC_ERR_INVALID,
              "avc_spk_identify: null pointer (queries %p, bank %p, best %p, best_score %p, target_score %p, target_rank %p)",
              (const void*)d->queries, (const void*)d->bank, (const void*)d->best, (const void*)d->best_score,
              (const void*)d->target_score, (const void*)d->target_rank);
  AVC_REQUIRE(d->m > 0 && d->s > 0 && d->dims > 0, AVC_ERR_INVALID, "avc_spk_identify: sizes must be positive (m %d, s %d, dims %d)",
              d->m, d->s, d->dims);
  AVC_REQUIRE(d->s <= AVC_SPK_MAX_N, AVC_ERR_UNSUPPORTED, "avc_spk_identify: s %d > %d", d->s, AVC_SPK_MAX_N);
  AVC_REQUIRE(d->dims <= AVC_SPK_MAX_DIMS, AVC_ERR_UNSUPPORTED, "avc_spk_identify: dims %d > %d", d->dims, AVC_SPK_MAX_DIMS);
  spk_identify_kernel<<<(unsigned)d->m, SPK_THREADS, d->dims * 8, (cudaStream_t)stream>>>(*d);
  AVC_CHECK_LAUNCH("avc_spk_identify");
  return AVC_OK;
}
