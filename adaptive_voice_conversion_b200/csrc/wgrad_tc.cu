// Conv weight gradient on the tensor cores (wgmma m64nNk8, TF32 in, fp32 accumulate in registers):
//   dW[co][ci][j] += sum_{b,t} dc[b][co][t] * xpad[b][ci][t * stride + j]
// (autograd of pad_layer + nn.Conv1d w.r.t. the weight, model.py:21-32 under solver.py:90).
//
// GEMM view: M = co (128 per CTA: two consumer warpgroups of m64), N = taps x ci (K taps x WT_NT = 32 ci per CTA, so
// N = 32 K <= 256 and the accumulator is N / 2 <= 128 registers per consumer thread), reduction = the time rows of a
// batch slice, WG_ROWS rows per pipeline stage.
//
// The A4 activation layout [c/4][t][4] is MN-major for this reduction (K is time), and tf32 wgmma reads shared-memory
// operands K-major only.  The two operands take different routes into a stage:
//   A (dc):  TMA copies the A4 tensor as it is, eight boxes of (4 co, 4 rows, 32 co chunks) per stage:
//            [8 planes][32 co chunks][4 t][4 co], plane p = rows 4p..4p+3 of the chunk.  Every 4-row group lies in one
//            sample (Tout % 8 == 0), so a box never straddles samples; rows past the slice are copied from sample B,
//            past the end of the tensor, and arrive as zeros like co past Cout.  The consumers load their A fragments
//            from there with ld.shared and feed wgmma from registers (wgmma_tf32_rs), which takes A in any layout.
//   B (x, by window): a staging thread loads the 16-byte A4 units (4 channels x 1 time step) of one (4-channel chunk,
//            4-row plane) window once for all K taps, transposes them in registers and stores 4 K 16-byte K-major units
//            into the no-swizzle core-matrix layout of tc_common.cuh: [8 planes][K x 32 rows][4 t], row j * 32 + ci
//            holds xpad[ci][t * stride + j].
// The tap shifts, the reflect padding and the stride-2 gather are all resolved while staging, so ONE wgmma per k-step
// covers every tap.  The fp32 bit patterns are used as they are: the tensor core reads their TF32 part (truncation
// toward zero, the operand model of tests/test_gpu_wgrad_exact.py).
//
// Each CTA owns (ci tile, co tile, batch slice); its partial sums go to a scratch buffer [slice][tap][ci/4][co][4] and
// are reduced into the canonical nn.Conv1d gradient layout by wgrad_tc_reduce_kernel (fixed order, no atomics), or
// added in place (ATOMIC, see below).
#include "common.cuh"
#include "tc_common.cuh"
#include "tmap.cuh"

namespace avc {

constexpr int WT_NT = 32;          // ci columns per CTA per tap
constexpr int WG_ROWS = 32;        // reduction rows (time steps) per pipeline stage: 4 wgmma k-steps, 8 planes
constexpr int WG_A_PLANE = 32 * 4 * 16;                  // one dc box: 32 co chunks x 4 rows x 16 bytes
constexpr int WG_A_BYTES = (WG_ROWS / 4) * WG_A_PLANE;   // dc planes of one stage
constexpr int WG_MAX_STAGES = 8;
constexpr int WG_SMEM_MAX = 224 * 1024;

struct WgTcArgs {
  avc_wgrad_desc d;
  float* scratch;
  int nslices, samp_per_slice, nstage, coutp;
  int* status;
};

// Staging windows.  Window w (0..63) of a chunk is ci chunk c4 = w % 8 and plane pl = w / 8: 4 channels at the plane's
// 4 reduction rows t .. t + 3.  Row t + i, tap j reads input position (t + i) S + j - pad_left = t S + n - pad_left with
// n = i S + j, so the window's K taps read 3 S + K distinct A4 units (K + 3 at stride 1, K + 6 at stride 2), and each is
// loaded once.
__host__ __device__ constexpr int wg_win_units(int K, int S) { return 3 * S + K; }

// Loads the units of window w of chunk `ch` (rows ch * WG_ROWS .. of the CTA's slice) into u[n], n = 0 .. 3 S + K - 1.
// Reflect padding is resolved per unit; rows past the slice and channels past Cin are zeros.
template <int K, int S>
__device__ __forceinline__ void wgrad_win_load(const WgTcArgs& a, float4 (&u)[wg_win_units(K, S)], int w, int ch, int b0, int R) {
  const avc_wgrad_desc& d = a.d;
  const int c4 = w & 7, pl = w >> 3;
  const int r = ch * WG_ROWS + 4 * pl;
  const int g = r / d.Tout, t = r - g * d.Tout;   // Tout % 8 == 0: the 4 rows lie in one sample
  const int ci = blockIdx.x * WT_NT + 4 * c4;
  const bool v = r < R && ci < d.Cin;
  const float* col = d.x + (size_t)(v ? b0 + g : 0) * d.x_bstride + (size_t)((v ? ci : 0) >> 2) * d.Tin * 4;
  const int p0 = t * S - d.pad_left;
  if (v && p0 >= 0 && p0 + wg_win_units(K, S) <= d.Tin) {
    // inside the signal: one base address, the units at fixed offsets
    const float* q = col + (size_t)p0 * 4;
#pragma unroll
    for (int n = 0; n < wg_win_units(K, S); ++n) u[n] = ldg4(q + 4 * n);
  } else {
#pragma unroll
    for (int n = 0; n < wg_win_units(K, S); ++n) {
      const int p = src_pos(p0 + n, d.Tin, AVC_PAD_REFLECT, 1);
      u[n] = (v && p >= 0) ? ldg4(col + (size_t)p * 4) : zero4();
    }
  }
}

__device__ __forceinline__ float comp4(const float4& v, int c) { return c == 0 ? v.x : c == 1 ? v.y : c == 2 ? v.z : v.w; }
// component k of the result = component (k + rot) & 3 of v
__device__ __forceinline__ float4 rot4(float4 v, int rot) {
  if (rot & 1) v = make_float4(v.y, v.z, v.w, v.x);
  if (rot & 2) v = make_float4(v.z, v.w, v.x, v.y);
  return v;
}

// Transposes window w in registers and stores its 4 K K-major units: operand row j * 32 + 4 c4 + c of plane pl (tap j,
// channel c of the chunk) holds component c of u[j], u[S + j], u[2 S + j], u[3 S + j] (rows t .. t + 3).
// Store conflicts: a 16-byte store phase is 8 lanes, and lanes 8 h .. 8 h + 7 of a warp are the chunks c4 = 0..7 of one
// plane at the same tap and store index k.  Store k writes channel c = (k + rot) & 3 with rot = (c4 >> 1) & 3, so its
// 16-byte bank group (4 c4 + c) % 8 = 4 (c4 & 1) + ((k + (c4 >> 1)) & 3) differs for all 8 lanes (a fixed order would
// put 4 of them on one group).  The units are rotated by rot once, so every store reads fixed components.
template <int K, int S>
__device__ __forceinline__ void wgrad_win_store(uint8_t* stage, float4 (&u)[wg_win_units(K, S)], int w) {
  const int c4 = w & 7, pl = w >> 3, rot = (c4 >> 1) & 3;
  uint8_t* row = stage + WG_A_BYTES + pl * (K * WT_NT * 16) + c4 * 64;
#pragma unroll
  for (int n = 0; n < wg_win_units(K, S); ++n) u[n] = rot4(u[n], rot);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    uint8_t* dst = row + ((k + rot) & 3) * 16;
#pragma unroll
    for (int j = 0; j < K; ++j)
      *reinterpret_cast<float4*>(dst + j * WT_NT * 16) = make_float4(comp4(u[j], k), comp4(u[S + j], k), comp4(u[2 * S + j], k), comp4(u[3 * S + j], k));
  }
}

// Staging roles.  A staging warpgroup is two halves of 64 threads, and a half stages one chunk at a time, one window
// per thread, so every staging thread is busy at any K.  Half h of the CTA owns the chunks ch = h (mod wg_halves).  A
// half's loads are its latency: where two window register sets fit (wg_prefetch), a half issues the loads of its next
// chunk before the stores of the current one, so a CTA has up to 2 wg_halves chunks' loads in flight.  K <= 6 runs two
// staging warpgroups and 512 threads; K = 7, 8 one staging warpgroup and 384 threads, because 112-128 accumulators per
// consumer leave too few of 512 threads' 128 registers for a window set.
__host__ __device__ constexpr int wg_stagers(int K) { return K <= 6 ? 2 : 1; }
__host__ __device__ constexpr int wg_halves(int K) { return 2 * wg_stagers(K); }
__host__ __device__ constexpr int wg_threads(int K) { return 128 * (wg_stagers(K) + 2); }
// Registers per thread after the setmaxnreg split of the launch allocation (the __launch_bounds__ cap: 128 at 512
// threads, 168 at 384) between the staging threads and the consumers (N / 2 accumulators and two stages of A
// fragments, 32 registers).  A window set is 4 (3 S + K) registers; "2 x" = the half prefetches its next chunk:
//   K            1..4            5        6        7        8
//   stage / mma  128 / 128       112/144  96/160   120/192  120/192
//   stride 1     2 x 16..28      2 x 32   1 x 36   2 x 40   1 x 44
//   stride 2     2 x 28..40      1 x 44   1 x 48   1 x 52   1 x 56
// Set from -Xptxas -v: K = 8 spills at 104 or 112 staging registers (stride 2) and with a stride-1 prefetch at 120;
// K = 5 serialises its wgmmas at 136 consumer registers.
__host__ __device__ constexpr int wg_regs_stage(int K) { return K <= 4 ? 128 : K == 5 ? 112 : K == 6 ? 96 : 120; }
__host__ __device__ constexpr int wg_regs_mma(int K) { return K <= 4 ? 128 : K == 5 ? 144 : K == 6 ? 160 : 192; }
// two window sets and 40 registers of addresses and loop state
__host__ __device__ constexpr bool wg_prefetch(int K, int S) { return 2 * 4 * wg_win_units(K, S) + 40 <= wg_regs_stage(K); }
__host__ __device__ constexpr bool wg_budget_ok(int K) {
  return K > 8 || (wg_stagers(K) * 128 * wg_regs_stage(K) + 256 * wg_regs_mma(K) <= wg_threads(K) * (wg_stagers(K) == 2 ? 128 : 168) &&
                   wg_budget_ok(K + 1));
}
static_assert(wg_budget_ok(1), "setmaxnreg budget exceeds the launch allocation");
// The ring holds at least as many stages as there are staging halves (the parity argument in the kernel needs it)
__host__ __device__ constexpr bool wg_ring_ok(int K) {
  return K > 8 || ((WG_SMEM_MAX / (WG_A_BYTES + 8 * 16 * WT_NT * K) >= wg_halves(K)) && wg_ring_ok(K + 1));
}
static_assert(wg_ring_ok(1), "a staging half could run a whole ring ahead");

// Stages chunk ch from the window registers u: waits for stage ch % nstage to be free, starts the dc copies (thread 0
// of the half), stores the x windows and arrives on full (one arrival per warp).
template <int K, int S>
__device__ __forceinline__ bool wgrad_win_put(const WgTcArgs& a, const CUtensorMap* tmdc, uint8_t* smem, uint64_t* full, uint64_t* empty,
                                              float4 (&u)[wg_win_units(K, S)], int w, int ch, int b0, int R) {
  const avc_wgrad_desc& d = a.d;
  const int s = ch % a.nstage;
  const uint32_t ph = (uint32_t)(ch / a.nstage) & 1u;
  if (ch >= a.nstage && !__all_sync(0xffffffffu, tc::mbar_wait(&empty[s], ph ^ 1u, a.status, 5))) return false;
  uint8_t* stage = smem + (size_t)s * ((uint32_t)WG_A_BYTES + 8u * (uint32_t)(K * WT_NT * 16));
  if (w == 0) {
    tc::mbar_arrive_expect_tx(&full[s], (uint32_t)WG_A_BYTES);
#pragma unroll
    for (int p = 0; p < WG_ROWS / 4; ++p) {
      const int r = ch * WG_ROWS + 4 * p, g = r / d.Tout;
      tc::tensor_g2s_4d(stage + p * WG_A_PLANE, tmdc, 0, r - g * d.Tout, blockIdx.y * 32, r < R ? b0 + g : d.B, &full[s]);
    }
  }
  wgrad_win_store<K, S>(stage, u, w);
  tc::fence_proxy_async_smem();   // the generic-proxy stores, before the async proxy (wgmma) reads them
  __syncwarp();
  if ((w & 31) == 0) tc::mbar_arrive(&full[s]);
  return true;
}

// The staging loop of half h at stride S.  With prefetch the two register sets alternate by chunk with static indices:
// chunk ch + H's loads are issued before chunk ch's wait and stores.
template <int K, int S>
__device__ __forceinline__ void wgrad_stage_x(const WgTcArgs& a, const CUtensorMap* tmdc, uint8_t* smem, uint64_t* full, uint64_t* empty,
                                              int h, int w, int b0, int R, int nchunk) {
  constexpr int H = wg_halves(K), U = wg_win_units(K, S);
  float4 ua[U];
  if constexpr (wg_prefetch(K, S)) {
    float4 ub[U];
    if (h < nchunk) wgrad_win_load<K, S>(a, ua, w, h, b0, R);
    for (int ch = h; ch < nchunk; ch += 2 * H) {
      if (ch + H < nchunk) wgrad_win_load<K, S>(a, ub, w, ch + H, b0, R);
      if (!wgrad_win_put<K, S>(a, tmdc, smem, full, empty, ua, w, ch, b0, R) || ch + H >= nchunk) return;
      if (ch + 2 * H < nchunk) wgrad_win_load<K, S>(a, ua, w, ch + 2 * H, b0, R);
      if (!wgrad_win_put<K, S>(a, tmdc, smem, full, empty, ub, w, ch + H, b0, R)) return;
    }
  } else {
    for (int ch = h; ch < nchunk; ch += H) {
      wgrad_win_load<K, S>(a, ua, w, ch, b0, R);
      if (!wgrad_win_put<K, S>(a, tmdc, smem, full, empty, ua, w, ch, b0, R)) return;
    }
  }
}

// One stage of a consumer warpgroup: wait for the stage, load this thread's A fragments of its 4 k-steps into `af`
// (a0..a3 of k-step k in af[4k..4k+3]), queue the 4 MMAs, then retire the previous stage's (wait_group 1).  The
// previous stage's fragments `af_prev` were read by those MMAs: they stay live up to the wait.
template <int N>
__device__ __forceinline__ bool wgrad_mma_stage(const WgTcArgs& a, float* acc, uint32_t* af, uint32_t* af_prev, uint64_t* full, int s, uint32_t ph,
                                                const uint8_t* stage, uint32_t a_off, uint32_t b_lo, uint32_t d_hi) {
  constexpr uint32_t B_PLANE = N * 16;
  if (!__all_sync(0xffffffffu, tc::mbar_wait(&full[s], ph, a.status, 6))) {
    tc::wgmma_wait<0>();
    return false;
  }
  // a0 = (row, t), a1 = (row + 8, t): two co chunks further; a2, a3: t + 4, the next plane
#pragma unroll
  for (int k = 0; k < WG_ROWS / 8; ++k)
#pragma unroll
    for (int q = 0; q < 4; ++q)
      af[4 * k + q] = *reinterpret_cast<const uint32_t*>(stage + a_off + (uint32_t)(2 * k + (q >> 1)) * WG_A_PLANE + (uint32_t)(q & 1) * 128u);
  tc::wgmma_fence();
#pragma unroll
  for (int k = 0; k < WG_ROWS / 8; ++k)   // k-step k: planes 2k and 2k + 1
    tc::wgmma_tf32_rs<N>(acc, af + 4 * k, tc::sdesc64(b_lo + (uint32_t)k * ((2u * B_PLANE) >> 4), d_hi), 1u);
  tc::wgmma_commit();
  tc::wgmma_wait<1>();
  tc::acc_fence(acc, N / 2);
  tc::reg_fence(af_prev, 16);
  return true;
}

// Weight gradient of one (ci tile, co tile, batch slice).  mbarrier ring over the slice's row chunks: full[s] = the two
// warps of the staging half that owns the chunk wrote the x planes of stage s, and the dc boxes of its TMA copies
// landed (transaction bytes); empty[s] = both consumer warpgroups' MMAs on stage s retired.  A consumer queues the MMAs
// of stage i, then wait_group 1 retires those of stage i - 1 and releases it; every CTA accumulates its rows in a fixed
// order.  setmaxnreg moves registers from the staging warpgroups to the consumers (wg_regs_*).
template <int K, bool ATOMIC>
__global__ void __launch_bounds__(wg_threads(K), 1) conv_wgrad_wgmma_kernel(const WgTcArgs a, const __grid_constant__ CUtensorMap tmdc) {
  constexpr int STAGERS = wg_stagers(K);
  constexpr int N = K * WT_NT;
  constexpr uint32_t B_PLANE = N * 16;
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ uint64_t bar_full[WG_MAX_STAGES], bar_empty[WG_MAX_STAGES];
  const avc_wgrad_desc& d = a.d;
  const int tid = threadIdx.x, warp = tc::warp_idx_sync();
  const int sl = blockIdx.z, b0 = sl * a.samp_per_slice;
  const int R = max(0, min(a.samp_per_slice, d.B - b0)) * d.Tout;   // reduction rows of the slice
  const int nchunk = cdiv(R, WG_ROWS);
  const uint32_t stage_bytes = (uint32_t)WG_A_BYTES + 8u * B_PLANE;

  if (tid == 0) {
    for (int s = 0; s < a.nstage; ++s) {
      tc::mbar_init(&bar_full[s], 3);   // two staging warps + the arrival that carries the dc copies' bytes
      tc::mbar_init(&bar_empty[s], 2);
    }
    tc::fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4 * STAGERS) {
    // ================================================================ staging warpgroups
    // Staging half h = warp / 2 owns the chunks ch = h (mod H), H = wg_halves(K); thread w = tid % 64 of the half
    // stages window w.  The two warps of a half wait, store and arrive on their own.  The parity wait on empty[s]
    // cannot alias an older phase: before chunk ch, each warp of the half waited for chunk ch - H, that is for the
    // release of chunk ch - H - nstage, and releases come in chunk order.  nstage >= H (wg_ring_ok), so chunk
    // ch - 2 nstage is released and empty[s] is at most one phase behind.  Loads issued ahead (prefetch) touch no
    // barrier; a half's stores never run more than nstage chunks ahead of the consumers.  Once the stage is free,
    // thread 0 of the half starts the TMA copies of its dc planes; they land while the x stores run.
    tc::setmaxnreg_dec<wg_regs_stage(K)>();
    if (d.stride == 1)
      wgrad_stage_x<K, 1>(a, &tmdc, smem, bar_full, bar_empty, warp >> 1, tid & 63, b0, R, nchunk);
    else
      wgrad_stage_x<K, 2>(a, &tmdc, smem, bar_full, bar_empty, warp >> 1, tid & 63, b0, R, nchunk);
    return;
  }

  // ================================================================ MMA warpgroups
  tc::setmaxnreg_inc<wg_regs_mma(K)>();
  const int wg = (warp >> 2) - STAGERS, wt = tid & 127;
  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  // A fragment of this thread: co row m = 64 wg + 16 (wt / 32) + (wt % 32) / 4 (and m + 8), time t = wt % 4 (and t + 4)
  // of each k-step, at [plane][m / 4][t][m % 4].  The 8 row groups of a warp's load sit in two co chunks, 64 bytes
  // apart: with t over 4 x 16 bytes and m % 4 over 4 x 4 bytes, the 32 lanes hit 32 different banks.
  const int m = 64 * wg + tc::wg_acc_row(wt, 0);
  const uint32_t a_off = (uint32_t)(m >> 2) * 64u + (uint32_t)(wt & 3) * 16u + (uint32_t)(m & 3) * 4u;
  uint32_t af[2][16];
  const uint32_t smem0 = tc::smem_u32(smem), d_hi = tc::sdesc_hi(128);
  int s = 0, s_prev = -1;
  uint32_t ph = 0;
  tc::acc_fence(acc, N / 2);
  for (int ch = 0; ch < nchunk; ++ch) {
    const uint32_t b_lo = tc::sdesc_lo(smem0 + (uint32_t)s * stage_bytes + (uint32_t)WG_A_BYTES, B_PLANE);
    const uint8_t* stage = smem + (size_t)s * stage_bytes;
    // the two fragment buffers alternate by chunk (static indices: the registers stay in place under the async MMAs)
    const bool ok = (ch & 1) ? wgrad_mma_stage<N>(a, acc, af[1], af[0], bar_full, s, ph, stage, a_off, b_lo, d_hi)
                             : wgrad_mma_stage<N>(a, acc, af[0], af[1], bar_full, s, ph, stage, a_off, b_lo, d_hi);
    if (!ok) return;
    if (s_prev >= 0 && wt == 0) tc::mbar_arrive(&bar_empty[s_prev]);
    s_prev = s;
    if (++s == a.nstage) { s = 0; ph ^= 1u; }
  }
  tc::wgmma_wait<0>();
  tc::acc_fence(acc, N / 2);
  tc::reg_fence(af[0], 16);
  tc::reg_fence(af[1], 16);
  if (nchunk == 0) return;

  // partial dW of this CTA: scratch[sl][tap][ci/4][co][4] (ATOMIC: added into the layer's accumulation buffer)
  const int co = blockIdx.y * 128 + m;
#pragma unroll
  for (int jj = 0; jj < N / 8; ++jj) {
    const int n = tc::wg_acc_col(wt, 4 * jj), j = n / WT_NT, ci = blockIdx.x * WT_NT + n % WT_NT;
    if (ci < d.Cin) {
      float* sbase = a.scratch + (((size_t)(ATOMIC ? 0 : sl) * K + j) * (size_t)(d.Cin >> 2)) * (size_t)a.coutp * 4;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* p = sbase + ((size_t)(ci >> 2) * a.coutp + co + 8 * h) * 4 + (ci & 3);
        const float v0 = acc[4 * jj + 2 * h], v1 = acc[4 * jj + 2 * h + 1];
        if constexpr (ATOMIC)
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v0), "f"(v1) : "memory");
        else
          *reinterpret_cast<float2*>(p) = make_float2(v0, v1);
      }
    }
  }
}

// dW[co][ci][j] += sum over slices of scratch[sl][j][ci/4][co][ci%4]
// block (32, 8): x = output float4 (coalesced 512 B per warp), y = slice group; four independent 16-byte loads in
// flight per thread (the partials sit in L2)
__global__ void __launch_bounds__(256) wgrad_tc_reduce_kernel(const float* __restrict__ scratch, float* __restrict__ dw, int Cout, int Cin,
                                                              int K, int coutp, int nslices) {
  __shared__ float4 part[8][32];
  const int64_t n = (int64_t)K * (Cin >> 2) * coutp;
  const int64_t slice_stride = n * 4;
  const int64_t i = (int64_t)blockIdx.x * 32 + threadIdx.x;
  float4 s = zero4();
  if (i < n) {
    int sl = threadIdx.y;
    float4 s1 = zero4();
    const float* p = scratch + i * 4;
    for (; sl + 24 < nslices; sl += 32) {
      const float4 v0 = ldg4(p + (sl + 0) * slice_stride), v1 = ldg4(p + (sl + 8) * slice_stride);
      const float4 v2 = ldg4(p + (sl + 16) * slice_stride), v3 = ldg4(p + (sl + 24) * slice_stride);
      s.x += v0.x + v2.x; s.y += v0.y + v2.y; s.z += v0.z + v2.z; s.w += v0.w + v2.w;
      s1.x += v1.x + v3.x; s1.y += v1.y + v3.y; s1.z += v1.z + v3.z; s1.w += v1.w + v3.w;
    }
    s.x += s1.x; s.y += s1.y; s.z += s1.z; s.w += s1.w;
    for (; sl < nslices; sl += 8) {
      const float4 v = ldg4(scratch + sl * slice_stride + i * 4);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
  }
  part[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && i < n) {
#pragma unroll
    for (int y = 1; y < 8; ++y) { const float4 v = part[y][threadIdx.x]; s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
    const int co = (int)(i % coutp);
    if (co < Cout) {
      const int64_t r = i / coutp;
      const int c4 = (int)(r % (Cin >> 2)), j = (int)(r / (Cin >> 2));
      float* o = dw + ((int64_t)co * Cin + c4 * 4) * K + j;
      o[0] += s.x; o[K] += s.y; o[2 * K] += s.z; o[3 * K] += s.w;
    }
  }
}

// dW[co][ci][j] += acc[j][ci/4][co][ci%4]; acc = 0.   grid.y = layer (device item table), grid.x covers the largest
// layer (surplus blocks exit).  A block moves a 32 co x 32 ci x K tile through shared memory so that BOTH sides are
// coalesced: 512-byte runs of the accumulation buffer in, (32 ci x K)-float runs of the nn.Conv1d gradient out.  (Round
// 1 wrote the gradient with a 4-byte scatter at stride K: 209 us per step, now the kernel is copy-bound.)
__global__ void __launch_bounds__(256) wgrad_acc_flush_kernel(const avc_wgrad_acc_item* __restrict__ items) {
  __shared__ float tile[32][32 * 8 + 1];
  const avc_wgrad_acc_item it = items[blockIdx.y];
  const int K = it.K, C4 = it.Cin >> 2;
  const int coutp = cdiv(it.Cout, 128) * 128;
  const int ncg = cdiv(C4, 8);                      // groups of 8 four-channel chunks (32 input channels)
  const int nblk = (coutp >> 5) * ncg;
  if ((int)blockIdx.x >= nblk) return;
  const int cot = blockIdx.x / ncg, cg = blockIdx.x - cot * ncg;
  const int co0 = cot << 5, c40 = cg << 3;
  const int tid = threadIdx.x, col = tid & 31, c4l = tid >> 5;
  if (c40 + c4l < C4) {
    for (int j = 0; j < K; ++j) {
      float4* a4 = reinterpret_cast<float4*>(it.acc) + ((size_t)j * C4 + c40 + c4l) * coutp + co0 + col;
      const float4 s = *a4;
      *a4 = zero4();
      float* t = &tile[col][(c4l * 4) * K + j];
      t[0] = s.x; t[K] = s.y; t[2 * K] = s.z; t[3 * K] = s.w;
    }
  }
  __syncthreads();
  const int nci = min(32, it.Cin - c40 * 4);         // input channels of this tile
  const int run = nci * K;                            // contiguous floats of one output-channel row
  for (int r = tid >> 5; r < 32; r += 8) {
    const int co = co0 + r;
    if (co >= it.Cout) break;
    float* o = it.dw + ((size_t)co * it.Cin + c40 * 4) * K;
    for (int e = tid & 31; e < run; e += 32) o[e] += tile[r][e];
  }
}

// The batch is split into slices of whole G-sample tiles (G * Tout ~ 128 rows, 64 for stride 2) so that the slices and
// the CTAs of one slice fill the 132 SMs; the scratch buffer holds one partial dW per slice.
static int wgrad_tc_plan(const avc_wgrad_desc* d, WgTcArgs& a) {
  const int T = d->Tout;
  a.d = *d;
  int G = T >= 128 ? 1 : 128 / T;
  if (d->stride == 2) G = T >= 64 ? 1 : 64 / T;
  a.coutp = cdiv(d->Cout, 128) * 128;
  const int ntiles = cdiv(d->B, G);
  const int cta_per_slice = cdiv(d->Cin, WT_NT) * cdiv(d->Cout, 128);
  int nsl = 132 / cta_per_slice;
  if (nsl < 1) nsl = 1;
  if (nsl > ntiles) nsl = ntiles;
  const int tiles_per_slice = cdiv(ntiles, nsl);
  a.nslices = cdiv(ntiles, tiles_per_slice);
  a.samp_per_slice = tiles_per_slice * G;
  a.nstage = min(WG_MAX_STAGES, WG_SMEM_MAX / (WG_A_BYTES + 8 * 16 * WT_NT * d->K));
  return AVC_OK;
}

static bool wgrad_tc_supported(const avc_wgrad_desc* d) {
  return (d->stride == 1 || d->stride == 2) && d->Tout % 8 == 0 && d->Tout <= 128 && d->K >= 1 && d->K <= 8 && d->Cin % 4 == 0 &&
         d->Cout % 4 == 0 && d->Tin + d->K - 1 >= (d->Tout - 1) * d->stride + 1 && (d->stride == 1 || d->Tout <= 64);
}

int wgrad_reduce(const float* scratch, float* dw, int Cout, int Cin, int K, int coutp, int nslices, cudaStream_t stream) {
  const int64_t n = (int64_t)K * (Cin / 4) * coutp;
  AVC_LAUNCH(wgrad_tc_reduce_kernel, (int)cdiv64(n, 32), dim3(32, 8), 0, stream, scratch, dw, Cout, Cin, K, coutp, nslices);
  AVC_CHECK_LAUNCH("wgrad_tc_reduce");
  return AVC_OK;
}

// one kernel instance per tap count (N = 32 K accumulator columns) and output mode
template <int K, bool ATOMIC>
static int wgrad_wgmma_launch(const WgTcArgs& a, const CUtensorMap& tmdc, cudaStream_t stream, const char* who) {
  static bool attr_done = false;
  if (!attr_done) {
    const cudaError_t e = cudaFuncSetAttribute(conv_wgrad_wgmma_kernel<K, ATOMIC>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM_MAX);
    if (e != cudaSuccess) {
      set_error("%s: cudaFuncSetAttribute: %s", who, cudaGetErrorString(e));
      return AVC_ERR_CUDA;
    }
    attr_done = true;
  }
  const dim3 grid(cdiv(a.d.Cin, WT_NT), cdiv(a.d.Cout, 128), a.nslices);
  const int smem = a.nstage * (WG_A_BYTES + 8 * 16 * WT_NT * K);
  AVC_LAUNCH((conv_wgrad_wgmma_kernel<K, ATOMIC>), grid, wg_threads(K), smem, stream, a, tmdc);
  AVC_CHECK_LAUNCH(who);
  return AVC_OK;
}

template <bool ATOMIC>
static int wgrad_wgmma_dispatch(const WgTcArgs& a, const CUtensorMap& tmdc, cudaStream_t stream, const char* who) {
  switch (a.d.K) {
    case 1: return wgrad_wgmma_launch<1, ATOMIC>(a, tmdc, stream, who);
    case 2: return wgrad_wgmma_launch<2, ATOMIC>(a, tmdc, stream, who);
    case 3: return wgrad_wgmma_launch<3, ATOMIC>(a, tmdc, stream, who);
    case 4: return wgrad_wgmma_launch<4, ATOMIC>(a, tmdc, stream, who);
    case 5: return wgrad_wgmma_launch<5, ATOMIC>(a, tmdc, stream, who);
    case 6: return wgrad_wgmma_launch<6, ATOMIC>(a, tmdc, stream, who);
    case 7: return wgrad_wgmma_launch<7, ATOMIC>(a, tmdc, stream, who);
    default: return wgrad_wgmma_launch<8, ATOMIC>(a, tmdc, stream, who);
  }
}

}  // namespace avc

using namespace avc;

extern "C" int64_t avc_wgrad_tc_scratch_floats(const avc_wgrad_desc* d) {
  if (!d || !wgrad_tc_supported(d)) return -1;
  WgTcArgs a;
  wgrad_tc_plan(d, a);
  return (int64_t)a.nslices * d->K * d->Cin * a.coutp;
}

static int wgrad_tc_launch(const avc_wgrad_desc* d, float* scratch, int* status, void* stream, bool accumulate, const char* who) {
  AVC_REQUIRE(d && d->x && d->dc && scratch && status && (accumulate || d->dw), AVC_ERR_INVALID, "%s: null argument", who);
  AVC_REQUIRE(d->B > 0 && d->Cin > 0 && d->Cout > 0 && d->Tin > 0 && d->Tout > 0, AVC_ERR_INVALID, "%s: bad shape", who);
  AVC_REQUIRE(wgrad_tc_supported(d), AVC_ERR_UNSUPPORTED, "%s: needs stride 1 (Tout <= 128) or 2 (Tout <= 64), Tout %% 8 == 0, K <= 8", who);
  // dc goes through TMA: its base and sample stride must be 16-byte aligned (the engine's A4 tensors always are)
  AVC_REQUIRE(((uintptr_t)d->dc & 15u) == 0 && d->dc_bstride % 4 == 0, AVC_ERR_UNSUPPORTED,
              "%s: dc and its sample stride (%lld floats) must be 16-byte aligned", who, (long long)d->dc_bstride);
  WgTcArgs a;
  wgrad_tc_plan(d, a);
  a.scratch = scratch;
  a.status = status;
  // dc as (4 co, t, co chunk, sample); box = 4 rows x one co tile (32 chunks), out-of-range elements read as zeros
  CUtensorMap tmdc;
  {
    PFN_tmap_encode enc = tmap_encode_fn();
    AVC_REQUIRE(enc, AVC_ERR_CUDA, "%s: cuTensorMapEncodeTiled is not available from this driver", who);
    const cuuint64_t gdim[4] = {4, (cuuint64_t)d->Tout, (cuuint64_t)(d->Cout / 4), (cuuint64_t)d->B};
    const cuuint64_t gstr[3] = {16, (cuuint64_t)d->Tout * 16u, (cuuint64_t)d->dc_bstride * 4u};
    const cuuint32_t box[4] = {4, 4, 32, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    const CUresult r = enc(&tmdc, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)d->dc, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    AVC_REQUIRE(r == CUDA_SUCCESS, AVC_ERR_CUDA, "%s: cuTensorMapEncodeTiled failed (%d) for dc: B=%d Cout=%d Tout=%d bstride=%lld", who, (int)r,
                d->B, d->Cout, d->Tout, (long long)d->dc_bstride);
  }
  const int rc = accumulate ? wgrad_wgmma_dispatch<true>(a, tmdc, (cudaStream_t)stream, who)
                            : wgrad_wgmma_dispatch<false>(a, tmdc, (cudaStream_t)stream, who);
  if (rc != AVC_OK || accumulate) return rc;
  return wgrad_reduce(scratch, d->dw, d->Cout, d->Cin, d->K, a.coutp, a.nslices, (cudaStream_t)stream);
}

extern "C" int avc_conv_wgrad_tc(const avc_wgrad_desc* d, float* scratch, int* status, void* stream) {
  return wgrad_tc_launch(d, scratch, status, stream, false, "avc_conv_wgrad_tc");
}

// ---- accumulate-in-place variant: every layer owns a zeroed [K][Cin/4][coutp][4] accumulation
// buffer; avc_conv_wgrad_tc_acc adds into it (vector atomics), avc_wgrad_acc_flush folds every
// layer's buffer into its nn.Conv1d gradient and zeroes it again -- ONE launch per backward pass.
extern "C" int64_t avc_wgrad_acc_floats(int Cout, int Cin, int K) {
  if (Cout <= 0 || Cin <= 0 || K <= 0 || Cin % 4 != 0) return -1;
  return (int64_t)K * Cin * (cdiv(Cout, 128) * 128);
}
extern "C" int avc_conv_wgrad_tc_acc(const avc_wgrad_desc* d, float* acc, int* status, void* stream) {
  return wgrad_tc_launch(d, acc, status, stream, true, "avc_conv_wgrad_tc_acc");
}
extern "C" int avc_wgrad_acc_flush(const avc_wgrad_acc_item* items_dev, int n_items, int64_t max_units, void* stream) {
  AVC_REQUIRE(items_dev && n_items > 0 && max_units > 0, AVC_ERR_INVALID, "avc_wgrad_acc_flush: bad argument");
  // a layer needs (coutp / 32) * ceil(Cin / 32) blocks <= units / (256 K) + coutp / 32: max_units / 256 plus a margin
  // covers every layer (surplus blocks exit at once)
  dim3 grid((unsigned)cdiv64(max_units, 256) + 64u, (unsigned)n_items);
  AVC_LAUNCH(wgrad_acc_flush_kernel, grid, 256, 0, (cudaStream_t)stream, items_dev);
  AVC_CHECK_LAUNCH("wgrad_acc_flush");
  return AVC_OK;
}
