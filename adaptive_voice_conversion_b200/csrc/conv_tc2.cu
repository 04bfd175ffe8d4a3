// Fused ConvBlock on the tensor cores, persistent / warp-specialised edition (wgmma m64nNk8 tf32,
// fp32 accumulation in registers).  Same contract as conv_tc.cu / conv_simt.cu:
//   reflect|zero pad -> Conv1d -> [pixel shuffle] -> [InstanceNorm] -> [AdaIN] -> [ReLU] -> [+residual] -> [*mask]
// (model.py:21-32, 52-59, 77-83, 237-250, 309-320, 354-369) and, with the DGRAD weight pack and zero
// padding, autograd's conv data gradient incl. the adjoint of the reflect padding / residual branch
// (AVC_F_FOLD).
//
//   * PERSISTENT CTAs (one per SM) walk a static tile list; a tile = G samples x 128 output channels.
//   * Roles: warp 0 bulk-copy (TMA) producer, warps 1-3 halo patch / TF32 rounding of the staged input,
//     warps 4-11 two consumer warpgroups (output rows 0-63 / 64-127) that issue the wgmma main loop into
//     their register accumulators and then run the epilogue.  mbarrier pipelines per shared-memory stage:
//     full (weights) / fullx (input rows) / ready (patched) / empty (read by both warpgroups' MMAs).
//   * STACKED SAMPLES: the G samples of a tile lie one after another in the staged row space at a
//     pitch of R = (rows one sample needs) and ONE MMA of N <= T2_MAX_N columns per (k-step, tap) covers all
//     of them (columns between two samples are garbage and never read): the small-T layers issue
//     2K MMAs per 16-channel slab instead of 2K*G.
//   * EPILOGUE THROUGH SHARED MEMORY: pass 0 adds the bias and drops the accumulator registers (wgmma
//     fragment layout) into an A4-layout tile in shared memory (chunk pitch == 1 mod 8 sixteen-byte units:
//     conflict-free); the InstanceNorm sums are one sweep over that tile.  A second pass (thread = one
//     16-byte A4 unit, lanes along time) normalises / AdaIN / ReLU / residual / mask / rounds and writes `c`
//     and `out` with fully coalesced 16-byte stores; the reflect-padding adjoint of the data-gradient
//     variant becomes three shared-memory reads.
//   * Halo rows come straight from global memory (no dependence on the bulk copy), so long samples
//     can be TIME-TILED (T > 144 columns: inference) for blocks without InstanceNorm.
//   * STAGE GRANULARITY: a stage is `hs` HALF-SLABS of 8 input channels (one MMA K-step each).  Default hs = 2 (one
//     16-channel slab of the weight pack, one contiguous bulk copy) for K >= 2 and hs = 4 for the 1x1 layers (fewer
//     barrier round trips per tile); hs = 1 (K x 4 KB of weights per stage fetched by ONE 4-D tensor-map copy out of
//     the [slab][tap][chunk] pack) is selectable with AVC_T2_HS=1.  AVC_T2_NSTAGE caps the pipeline depth.
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"
#include "tmap.cuh"

namespace avc {

int validate_conv_desc(const avc_conv_desc* d, const char* who);
int opt_tc_conv_v2();

constexpr int T2_SLAB = 16;          // input channels per weight-pack slab (2 MMA K-steps)
constexpr int T2_WTAP_BYTES = 8192;  // one tap of one slab: 4 chunks x 128 co x 16 B
constexpr int T2_HALF_BYTES = 4096;  // one tap of one half-slab (8 channels): 2 chunks x 128 co x 16 B
constexpr int T2_MAX_STAGES = 8;
constexpr int T2_MAX_G = 8;
constexpr int T2_MAX_N = 160;       // accumulator columns: N / 2 registers per consumer thread
constexpr int T2_SMEM_MAX = 226 * 1024;  // 227 KB per block minus the static shared memory (barriers)

struct Tc2Args {
  avc_conv_desc d;
  int G;        // samples per tile
  int R;        // row pitch between the stacked samples of a tile (= accumulator column pitch)
  int N;        // MMA N: multiple of 16, <= T2_MAX_N
  int srows;    // rows of one 4-channel plane of a stage (>= N + K - 1)
  int nslab, nstage;
  int hs;       // half-slabs (8 input channels = one MMA K-step) per pipeline stage: 1, or an even number
  int nhalf;    // half-slabs per tile (2 * nslab)
  int nst;      // pipeline stages per tile = ceil(nhalf / hs); the last one may hold fewer half-slabs
  int nchunk;   // column chunks of N accumulator columns per tile (> 1 only for a folded sample of more than 144
                // columns: the main loop runs once per chunk over the same staged rows)
  int N_last;   // accumulator columns of the last chunk
  int TT, ntt;  // output time steps per tile, time tiles per sample
  int Ts;       // columns one sample stages for the second pass (TT, or Tout for AVC_F_FOLD)
  int P;        // chunk pitch of the staged tile in 16-byte units (== 1 mod 8)
  int mtiles, ngroups, ntiles;
  uint32_t stage_bytes, w_bytes, x_chunk_bytes;
  uint32_t off_tile, off_par, off_stat;  // byte offsets inside dynamic shared memory
  int patch;    // 1: the patch warps sit between the bulk copy and the MMAs (halo rows and/or TF32 rounding)
  int variant;  // bit 0: `c` rows leave through bulk (TMA) stores; bit 1: `out` rows too (written back in place)
                // ABLATION bits (timing probes only, results are WRONG; tools/diag_ablate.py): 16 weight copies shrunk to
                // 1 KB, 32 no store pass, 64 no MMAs, 128 no accumulator pass, 256 no input-row copies; 2048: one patch warp
                // owns every stage (results stay correct)
  int* status;
  long long* dbg;
};

__device__ __forceinline__ float t2_round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ float4 t2_round4(float4 v) {
  return make_float4(t2_round_tf32(v.x), t2_round_tf32(v.y), t2_round_tf32(v.z), t2_round_tf32(v.w));
}
__device__ __forceinline__ void t2_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// Row hand-out of the store pass: row = (sample, 4-channel chunk) of the staged tile, lanes run along time.  Rows of
// at most 16 time steps share a warp in pairs.  (g, cql) advance incrementally: a runtime division per row was a
// 300-cycle dependent chain in front of every store.
struct RowIter {
  int row, g, cql, step, nq, tl0, tstep;
};
__device__ __forceinline__ RowIter t2_rows(int ewarp, int lane, int extent, int nq) {
  RowIter r;
  const int lpr = extent <= 16 ? 16 : 32, rpp = 32 / lpr;
  r.row = ewarp * rpp + lane / lpr;
  r.step = 8 * rpp;
  r.nq = nq;
  r.g = r.row / nq;
  r.cql = r.row - r.g * nq;
  r.tl0 = lane % lpr;
  r.tstep = lpr;
  return r;
}
__device__ __forceinline__ void t2_next(RowIter& r) {
  r.row += r.step;
  r.cql += r.step;
  while (r.cql >= r.nq) { r.cql -= r.nq; ++r.g; }
}

struct TileCoord {
  int mtile, b0, nsamp, t0, tw;
};
__device__ __forceinline__ TileCoord t2_decode(const Tc2Args& a, int tile) {
  TileCoord c;
  c.mtile = tile % a.mtiles;
  const int r = tile / a.mtiles;
  const int tt = r % a.ntt, grp = r / a.ntt;
  c.b0 = grp * a.G;
  c.nsamp = min(a.G, a.d.B - c.b0);
  c.t0 = tt * a.TT;
  c.tw = min(a.TT, a.d.Tout - c.t0);
  return c;
}

// tmx: 4-D tensor map of the input, dims (4 floats, time, sample, 4-channel chunk): ONE copy-engine instruction
// stages [4 chunks][G samples][R rows] of a 16-channel slab -- exactly the stacked-sample operand layout -- and
// rows / samples outside the tensor arrive as zeros (that IS the zero padding of the data-gradient convs).
// tmw (hs == 1 only): the weight pack as a 4-D tensor (256 floats, 2 halves of a [co][4] row, 4 chunks, slab*K+tap): the box
// (256, 2, 2, K) is one half-slab -- [tap][2 chunks][co][4] -- in one copy-engine instruction.
// Main loop of one tile for one consumer warpgroup (rows 64 wg .. 64 wg + 63 of the 128-row m-tile): every stage is
// K taps x (half-slabs) wgmma m64nNk8 into the register accumulator `acc`; the stage is released to the producer
// once this warpgroup's MMAs have read it (bar_empty counts one arrival per warpgroup).
template <int N>
__device__ __forceinline__ bool t2_mainloop(const Tc2Args& a, uint32_t smem0, uint64_t* bar_full, uint64_t* bar_fullx, uint64_t* bar_ready,
                                            uint64_t* bar_empty, int& s, uint32_t& ph, float* acc, int wg, int wt, int col0) {
  const int K = a.d.K;
  const uint32_t d_hi = tc::sdesc_hi(128);
  const uint32_t ks_b = 2u * (a.x_chunk_bytes >> 4);                       // B operand: next half-slab = 2 chunk planes on
  const uint32_t tap_a = (a.hs == 1 ? T2_HALF_BYTES : T2_WTAP_BYTES) >> 4;   // A operand: next tap
  const uint32_t slab_a = (uint32_t)K * (T2_WTAP_BYTES >> 4);                // A operand: next slab (hs > 1)
  for (int i = 0; i < a.nst; ++i) {
    const bool ok = __all_sync(0xffffffffu, tc::mbar_wait(a.patch ? &bar_ready[s] : &bar_fullx[s], ph, a.status, 3) &&
                                                tc::mbar_wait(&bar_full[s], ph, a.status, 3));
    if (!ok) return false;
    const uint32_t sw = smem0 + (uint32_t)s * a.stage_bytes;
    // rows 64 wg.. of the A operand: 64 rows x 16 B further inside every 4-channel chunk
    // B operand: the chunk's first column = staged row col0 (16 B per row)
    const uint32_t a_lo0 = tc::sdesc_lo(sw + (uint32_t)wg * 1024u, 2048),
                   b_lo0 = tc::sdesc_lo(sw + a.w_bytes, a.x_chunk_bytes) + (uint32_t)col0;
    const int nh = min(a.hs, a.nhalf - i * a.hs);
    tc::wgmma_fence();
    for (int e = 0; e < nh; ++e) {   // half-slab e of the stage: one K-step of 8 input channels per tap
      if (a.variant & 64) break;
      const uint32_t a_off = a.hs == 1 ? 0u : (uint32_t)(e >> 1) * slab_a + (uint32_t)(e & 1) * (T2_HALF_BYTES >> 4);
      uint64_t a_desc = tc::sdesc64(a_lo0 + a_off, d_hi);
      uint64_t b_desc = tc::sdesc64(b_lo0 + (uint32_t)e * ks_b, d_hi);
      if (K == 5) {
#pragma unroll
        for (int j = 0; j < 5; ++j) {
          tc::wgmma_tf32<N>(acc, a_desc, b_desc, ((uint32_t)i | (uint32_t)e | (uint32_t)j) ? 1u : 0u);
          a_desc += (uint64_t)tap_a;
          b_desc += 1u;
        }
      } else {
        for (int j = 0; j < K; ++j) {
          tc::wgmma_tf32<N>(acc, a_desc, b_desc, ((uint32_t)i | (uint32_t)e | (uint32_t)j) ? 1u : 0u);
          a_desc += (uint64_t)tap_a;
          b_desc += 1u;
        }
      }
    }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::acc_fence(acc, N / 2);
    if (wt == 0) tc::mbar_arrive(&bar_empty[s]);
    if (++s == a.nstage) { s = 0; ph ^= 1u; }
  }
  return true;
}

// Pass 0 of the epilogue, straight from the accumulator registers: + bias, raw conv rows of every stacked sample into
// the staged A4 tile (chunk pitch P == 1 mod 8 sixteen-byte units: the four lanes of a quad and the eight row groups of
// a warp hit 32 different banks).
template <int N>
__device__ __forceinline__ void t2_acc_to_tile(const Tc2Args& a, const TileCoord& c, const float* acc, float* stile, int wg, int wt,
                                               int col0) {
  const int sshift = a.d.stride == 2 ? 1 : 0;
  const int ncol = (c.tw - 1) * a.d.stride + 1;  // accumulator columns of one sample that hold outputs
  const int r0 = 64 * wg + tc::wg_acc_row(wt, 0);
  const int co0 = c.mtile * 128 + r0, co1 = co0 + 8;
  const float bias0 = (a.d.bias && co0 < a.d.Cout) ? __ldg(a.d.bias + co0) : 0.f;
  const float bias1 = (a.d.bias && co1 < a.d.Cout) ? __ldg(a.d.bias + co1) : 0.f;
  float* srow0 = stile + ((size_t)(r0 >> 2) * a.P) * 4 + (r0 & 3);
  float* srow1 = stile + ((size_t)((r0 + 8) >> 2) * a.P) * 4 + ((r0 + 8) & 3);
  int g = 0, gbase = 0;   // stacked sample of the column and its first column; columns grow with the register index
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int col = col0 + tc::wg_acc_col(wt, 4 * j + k);
      while (col >= gbase + a.R) { gbase += a.R; ++g; }
      const int tl = col - gbase;
      if (g < c.nsamp && tl < ncol && (tl & sshift) == 0) {
        const size_t off = (size_t)(g * a.Ts + (tl >> sshift)) * 4;
        srow0[off] = acc[4 * j + k] + bias0;
        srow1[off] = acc[4 * j + 2 + k] + bias1;
      }
    }
  }
}

// MMAs and pass 0 of one tile, instantiated for every accumulator width N (a multiple of 16, <= T2_MAX_N)
template <int N>
__device__ __forceinline__ bool t2_tile(const Tc2Args& a, const TileCoord& c, uint32_t smem0, uint64_t* bar_full, uint64_t* bar_fullx,
                                     uint64_t* bar_ready, uint64_t* bar_empty, int& s, uint32_t& ph, float* stile, int wg, int wt, int col0) {
  float acc[N / 2];
  if (!t2_mainloop<N>(a, smem0, bar_full, bar_fullx, bar_ready, bar_empty, s, ph, acc, wg, wt, col0)) return false;
  if (!(a.variant & 128)) t2_acc_to_tile<N>(a, c, acc, stile, wg, wt, col0);
  return true;
}

__global__ void __launch_bounds__(384, 1) conv_block_tc2_kernel(const Tc2Args a, const __grid_constant__ CUtensorMap tmx,
                                                                const __grid_constant__ CUtensorMap tmw) {
  extern __shared__ __align__(1024) uint8_t smem[];
  // per stage: full = weights landed, fullx = input rows landed (they are small and issued first, so the patch step
  // runs while the 5x larger weight copy is still in flight), ready = patched, empty = consumed by the MMAs
  __shared__ uint64_t bar_full[T2_MAX_STAGES], bar_fullx[T2_MAX_STAGES], bar_ready[T2_MAX_STAGES], bar_empty[T2_MAX_STAGES];
  const avc_conv_desc& d = a.d;
  const int tid = threadIdx.x, warp = tc::warp_idx_sync(), lane = tid & 31;
  const int K = d.K, S = d.stride;

  if (tid == 0) {
    for (int s = 0; s < a.nstage; ++s) {
      tc::mbar_init(&bar_full[s], 1);
      tc::mbar_init(&bar_fullx[s], 1);
      tc::mbar_init(&bar_ready[s], 1);
      tc::mbar_init(&bar_empty[s], 2);
    }
    tc::fence_mbar_init();
  }
  __syncthreads();
  long long tm0 = 0;
  if (a.dbg && tid == 0) tm0 = clock64();

  if (warp == 0) {
    // ================================================================ bulk-copy producer
    int s = 0;
    uint32_t ph = 0;
    bool ok = true;
    bool first_round = true;
    long long dbg0 = 0;
    for (int tile = blockIdx.x; tile < a.ntiles && ok; tile += gridDim.x) {
      const TileCoord c = t2_decode(a, tile);
      const float* wsrc = d.w_tc + (size_t)c.mtile * a.nslab * ((size_t)K * (T2_WTAP_BYTES / 4));
      const int tstart = c.t0 * S - d.pad_left;   // first input position of the staged rows (may be negative)
      // warm L2 with the NEXT tile's input rows (they usually come from HBM: a saved activation, or an input the L2
      // no longer holds), so that the latency-sensitive stage copies of that tile hit L2 like the weights do
      if (tile + (int)gridDim.x < a.ntiles && (a.variant & 8)) {   // opt-in: measured slower (the prefetches occupy the copy engine), AVC_T2_VARIANT bit 3
        const TileCoord cn = t2_decode(a, tile + gridDim.x);
        if (cn.b0 != c.b0 || cn.t0 != c.t0) {   // (another m-tile of the same samples reads the same rows)
          const int tsn = cn.t0 * S - d.pad_left;
          for (int i = lane; i < a.nst; i += 32) tc::tensor_prefetch_l2_4d(&tmx, 0, tsn, cn.b0, i * 2 * a.hs);
        }
      }
      __syncwarp();
      for (int ii = 0; ii < a.nst * a.nchunk; ++ii) {   // every column chunk streams the same stages again
        const int i = ii % a.nst;
        const long long w0 = a.dbg ? clock64() : 0;
        if (!first_round) ok = __all_sync(0xffffffffu, tc::mbar_wait(&bar_empty[s], ph ^ 1u, a.status, 2));
        if (a.dbg) dbg0 += clock64() - w0;
        if (!ok) break;
        uint8_t* sw = smem + (size_t)s * a.stage_bytes;
        const int h0 = i * a.hs, nh = min(a.hs, a.nhalf - h0);   // half-slabs [h0, h0 + nh) of the tile
        if (tc::elect_one()) {
          if (a.variant & 256) tc::mbar_arrive(&bar_fullx[s]);
          else {
            // the box always has 2*hs chunk planes; planes past Cin/4 (short last stage) arrive as zeros and are not used
            tc::mbar_arrive_expect_tx(&bar_fullx[s], 2u * (uint32_t)a.hs * a.x_chunk_bytes);
            tc::tensor_g2s_4d(sw + a.w_bytes, &tmx, 0, tstart, c.b0, h0 * 2, &bar_fullx[s]);
          }
          if (a.hs == 1) {
            const uint32_t wb = (uint32_t)K * T2_HALF_BYTES;
            if (a.variant & 16) {
              tc::mbar_arrive_expect_tx(&bar_full[s], 1024u);
              tc::bulk_g2s(sw, wsrc, 1024u, &bar_full[s]);
            } else {
              tc::mbar_arrive_expect_tx(&bar_full[s], wb);
              tc::tensor_g2s_4d(sw, &tmw, 0, 0, (h0 & 1) * 2, (c.mtile * a.nslab + (h0 >> 1)) * K, &bar_full[s]);
            }
          } else {
            const uint32_t wfull = (uint32_t)(nh >> 1) * (uint32_t)K * T2_WTAP_BYTES;   // whole slabs, contiguous in the pack
            const uint32_t wb = (a.variant & 16) ? 1024u : wfull;
            tc::mbar_arrive_expect_tx(&bar_full[s], wb);
            tc::bulk_g2s(sw, wsrc + (size_t)(h0 >> 1) * ((size_t)K * (T2_WTAP_BYTES / 4)), wb, &bar_full[s]);
          }
        }
        __syncwarp();
        if (++s == a.nstage) { s = 0; ph ^= 1u; first_round = false; }
      }
    }
    if (a.dbg && lane == 0) a.dbg[(size_t)blockIdx.x * 16 + 2] = dbg0;
  } else if (warp < 4) {
    // ================================================================ patch warps (3 warps, ROUND ROBIN over the stages)
    // (a) reflect padding: the copy engine delivered zeros for the rows outside the sample; they are overwritten
    //     with their mirror rows, taken from the staged rows of the same sample (from global memory only when a
    //     time-tiled sample's mirror row lies outside the tile);
    // (b) TF32 rounding, when the producer of the input did not round it (AVC_F_IN_TF32 unset: the residual
    //     stream stays full fp32 like the reference's activations): every row is rounded to nearest in place, so
    //     that the tensor core's truncation is exact.
    // a.patch == 0 (zero padding or K = 1, pre-rounded input): these warps idle, the MMAs wait on the copies directly.
    // One patch step is a dependent chain (barrier wake-up, shared-memory load, store, proxy fence, arrive) of
    // ~400-1000 cycles whatever the stage holds, and with ONE owner of all stages it is the serial resource of the
    // whole pipeline.  Warp w therefore owns the shared-memory STAGES s % npw == w outright (wait, round, mirror, fence, ONE
    // arrive): up to three patch steps are in flight and none of them synchronises with another warp.  Ownership goes
    // by stage, not by iteration: every phase of a stage's barrier is then seen by the same warp in order (a warp
    // that skipped a phase could run a whole ring revolution ahead, and a parity wait on a barrier that is still one
    // phase behind returns immediately -- the false positive every mbarrier pipeline has to exclude).
    const int pw = warp - 1;
    const bool rnd = !(d.flags & AVC_F_IN_TF32);
    const bool refl = d.pad_mode == AVC_PAD_REFLECT;
    const int npw = (a.variant & 2048) ? 1 : min(3, a.nstage);   // probe bit 2048: a single patch warp owns every stage (the previous structure)
    int s = 0;
    uint32_t ph = 0;
    bool ok = true;
    long long dbg0 = 0, dbg1 = 0;
    for (int tile = blockIdx.x; a.patch && pw < npw && tile < a.ntiles && ok; tile += gridDim.x) {
      const TileCoord c = t2_decode(a, tile);
      const int pbeg = c.t0 * S - d.pad_left;
      const int nr = (c.tw - 1) * S + K;  // rows one sample needs
      const int p_lo = max(0, pbeg), p_hi = min(d.Tin, pbeg + a.R);   // input positions present in the staged rows
      const int ncopy = max(0, min(p_hi, pbeg + nr) - p_lo), r_lo = p_lo - pbeg;
      const int nh = refl ? nr - ncopy : 0;
      // The halo assignment of a lane is the same for every stage of the tile: resolve it ONCE (the index arithmetic
      // -- runtime divisions and the mirror position -- was a ~600-cycle dependent chain in front of every stage).
      // Entry e = lane + 32 j (j < 4) is (sample g, halo row h, plane q); more than 128 entries use the generic loop.
      const int npl = 2 * a.hs;                  // 4-channel planes of a stage
      const int nent = c.nsamp * nh * npl;
      int h_dst[4], h_src[4], h_glob[4], h_q[4], h_g[4];   // float4 offsets inside the stage's x region; global source
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int e = lane + 32 * j;
        h_dst[j] = h_src[j] = h_glob[j] = -1;
        h_q[j] = h_g[j] = 0;
        if (e < nent) {
          const int q = e % npl, r = e / npl;
          const int g = r / nh, h = r - g * nh;
          const int u = h < r_lo ? h : h + ncopy;
          const int p = src_pos(pbeg + u, d.Tin, AVC_PAD_REFLECT, 1);
          h_dst[j] = q * a.srows + g * a.R + u;
          h_q[j] = q;
          h_g[j] = g;
          if (p >= p_lo && p < p_hi) h_src[j] = q * a.srows + g * a.R + (p - pbeg);
          else if (p >= 0) h_glob[j] = p;
        }
      }
      for (int ii = 0; ii < a.nst * a.nchunk && ok; ++ii) {
        const int i = ii % a.nst;
        if (s % npw == pw) {
          const long long w0 = a.dbg ? clock64() : 0;
          ok = tc::mbar_wait(&bar_fullx[s], ph, a.status, 4);
          const long long w1 = a.dbg ? clock64() : 0;
          dbg0 += w1 - w0;
          if (!ok) break;
          float4* sx = reinterpret_cast<float4*>(smem + (size_t)s * a.stage_bytes + a.w_bytes);
          bool wrote = false;
          if (rnd) {
            // every row of every plane (halo / gap rows included: rounding them again is harmless): the planes are
            // contiguous, so the sweep is a linear, conflict-free walk with no index arithmetic; 4 loads in flight
            const int nf4 = npl * a.srows;
            int e = lane;
            for (; e + 96 < nf4; e += 128) {
              const float4 v0 = sx[e], v1 = sx[e + 32], v2 = sx[e + 64], v3 = sx[e + 96];
              sx[e] = t2_round4(v0); sx[e + 32] = t2_round4(v1); sx[e + 64] = t2_round4(v2); sx[e + 96] = t2_round4(v3);
            }
            for (; e < nf4; e += 32) sx[e] = t2_round4(sx[e]);
            wrote = true;
            if (nh > 0) __syncwarp();   // the reflect rows below copy ROUNDED rows
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (h_dst[j] >= 0) {
              float4 v = zero4();
              if (h_src[j] >= 0) v = sx[h_src[j]];
              else if (h_glob[j] >= 0 && (i * npl + h_q[j]) * 4 < d.Cin) {
                v = ldg4(d.in + (size_t)(c.b0 + h_g[j]) * d.in_bstride + ((size_t)(i * npl + h_q[j]) * d.Tin + h_glob[j]) * 4);
                if (rnd) v = t2_round4(v);
              }
              sx[h_dst[j]] = v;
              wrote = true;
            }
          }
          for (int e = lane + 128; e < nent; e += 32) {   // more than 128 halo entries (large K x G): generic path
            const int q = e % npl, r = e / npl;
            const int g = r / nh, h = r - g * nh;
            const int u = h < r_lo ? h : h + ncopy;
            const int p = src_pos(pbeg + u, d.Tin, AVC_PAD_REFLECT, 1);
            float4 v = zero4();
            if (p >= p_lo && p < p_hi) v = sx[(size_t)q * a.srows + g * a.R + (p - pbeg)];
            else if (p >= 0 && (i * npl + q) * 4 < d.Cin) {
              v = ldg4(d.in + (size_t)(c.b0 + g) * d.in_bstride + ((size_t)(i * npl + q) * d.Tin + p) * 4);
              if (rnd) v = t2_round4(v);
            }
            sx[(size_t)q * a.srows + g * a.R + u] = v;
            wrote = true;
          }
          if (wrote) tc::fence_proxy_async_smem();   // only writers pay for the proxy fence
          __syncwarp();
          if (lane == 0) tc::mbar_arrive(&bar_ready[s]);
          if (a.dbg) dbg1 += clock64() - w1;
        }
        if (++s == a.nstage) { s = 0; ph ^= 1u; }
      }
    }
    if (a.dbg && tid == 32) {
      long long* o = a.dbg + (size_t)blockIdx.x * 16;
      o[3] = dbg0; o[4] = dbg1;
    }
  } else {
    // ================================================================ MMA + epilogue (two warpgroups, 256 threads)
    const int etid = tid - 128, ewarp = warp - 4;
    const int wg = ewarp >> 2, wt = etid & 127;      // warpgroup: accumulator rows 64 wg .. 64 wg + 63
    const int quarter = ewarp & 3, half = ewarp >> 2;
    const int col_l = quarter * 32 + lane;            // conv output row of the per-channel parameter pass
    const uint32_t smem0 = tc::smem_u32(smem);
    int s = 0;
    uint32_t ph = 0;
    float* stile = reinterpret_cast<float*>(smem + a.off_tile);
    float* par = reinterpret_cast<float*>(smem + a.off_par);          // [3][G][128]: mean, scale, shift
    float2* stat = reinterpret_cast<float2*>(smem + a.off_stat);      // [2][G][128] partial (sum, sum sq)
    const int P = a.P, Ts = a.Ts;
    const int shuf = d.shuffle;
    const int Cn = shuf ? d.Cout / 2 : d.Cout;
    const int Tn = shuf ? d.Tout * 2 : d.Tout;                        // normalised length of a whole sample
    const int out_T = d.out_T > 0 ? d.out_T : Tn;
    const int ots = d.out_tstride > 0 ? d.out_tstride : 1, oto = d.out_toff;
    const bool fold = (d.flags & AVC_F_FOLD) != 0;
    // AVC_F_NORMBWD (with AVC_F_FOLD): norm / relu / eps / cond / save_c / stats / dc / dcond / dbias describe the UPSTREAM
    // block whose output gradient this data-gradient conv produces; its InstanceNorm/AdaIN/ReLU backward runs here
    const bool nbw = fold && (d.flags & AVC_F_NORMBWD) != 0;
    const bool fwd_norm = d.norm && !nbw;
    float* dbacc = par;   // [128] per-CTA bias-gradient partial sums of the upstream block (nbw, upstream without norm)
    if (nbw && d.dbias && etid < 128) par[etid] = 0.f;   // ordered before the first use by the barriers of the first tile
    const int fpl = (d.flags >> 8) & 0xff, fpr = (d.flags >> 16) & 0xff;
    const bool rnd_out = (d.flags & AVC_F_ROUND_OUT) != 0;
    bool ok = true;
    int tl = 0;
    long long dbg0 = 0, dbg1 = 0, dbg2 = 0, dbg3 = 0, dbg4 = 0, dbg5 = 0;
    for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x, ++tl) {
      const TileCoord c = t2_decode(a, tile);
      long long e3b = 0;
      const long long e0 = a.dbg ? clock64() : 0;
      // ---------------- main loop, then pass 0: accumulators (+bias) -> staged A4 tile
      for (int ch = 0; ch < a.nchunk; ++ch) {
        bool mok = false;
        const int col0 = ch * a.N;
        switch (ch + 1 == a.nchunk ? a.N_last : a.N) {
#define T2_CASE(n) \
  case n: mok = t2_tile<n>(a, c, smem0, bar_full, bar_fullx, bar_ready, bar_empty, s, ph, stile, wg, wt, col0); break;
          T2_CASE(16) T2_CASE(32) T2_CASE(48) T2_CASE(64) T2_CASE(80) T2_CASE(96) T2_CASE(112) T2_CASE(128) T2_CASE(144) T2_CASE(160)
#undef T2_CASE
        }
        ok = ok && mok;
      }
      const long long e1 = a.dbg ? clock64() : 0;
      const int co = c.mtile * 128 + col_l;
      const bool co_ok = co < d.Cout;
      t2_bar_sync(2, 256);
      // ---------------- InstanceNorm sums of every (sample, row) over the staged tile
      if (ok && fwd_norm) {
        for (int e = etid; e < c.nsamp * 128; e += 256) {
          const int g = e >> 7, r = e & 127;
          const float* src = stile + ((size_t)(r >> 2) * P + g * Ts) * 4 + (r & 3);
          float s1 = 0.f, s2 = 0.f;
          for (int t = 0; t < c.tw; ++t) {
            const float x = src[(size_t)t * 4];
            s1 += x;
            s2 = fmaf(x, x, s2);
          }
          stat[(0 * a.G + g) * 128 + r] = make_float2(s1, s2);
          stat[(1 * a.G + g) * 128 + r] = make_float2(0.f, 0.f);
        }
      }
      if (a.variant & 3) tc::fence_proxy_async_smem();   // the staged rows will be read by bulk (async-proxy) stores
      const long long e2 = a.dbg ? clock64() : 0;
      t2_bar_sync(2, 256);
      // ---------------- per (sample, channel) parameters: mean, scale = rstd*gamma, shift = beta
      for (int g = half; g < c.nsamp && !fold; g += 2) {
        const int b = c.b0 + g;
        float mean = 0.f, rstd = 1.f;
        const int cn = shuf ? co >> 1 : co;
        if (d.norm) {
          const float2 p0 = stat[(0 * a.G + g) * 128 + col_l], p1 = stat[(1 * a.G + g) * 128 + col_l];
          float s1 = p0.x + p1.x, s2 = p0.y + p1.y;
          if (shuf) {  // conv rows (2c, 2c+1) pool into normalised channel c
            s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
            s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
          }
          const float inv = 1.f / (float)Tn;
          mean = s1 * inv;
          const float var = fmaxf(s2 * inv - mean * mean, 0.f);
          rstd = rsqrtf(var + d.eps);
          if (d.stats && co_ok && (!shuf || (co & 1) == 0)) {
            d.stats[((size_t)b * Cn + cn) * 2 + 0] = mean;
            d.stats[((size_t)b * Cn + cn) * 2 + 1] = rstd;
          }
        }
        float beta = 0.f, gamma = 1.f;
        if (d.cond && co_ok) {
          beta = __ldg(d.cond + (size_t)b * d.cond_bstride + cn);
          gamma = __ldg(d.cond + (size_t)b * d.cond_bstride + Cn + cn);
        }
        par[(0 * a.G + g) * 128 + col_l] = mean;
        par[(1 * a.G + g) * 128 + col_l] = rstd * gamma;
        par[(2 * a.G + g) * 128 + col_l] = beta;
      }
      t2_bar_sync(2, 256);
      const long long e3 = a.dbg ? clock64() : 0;
      // ---------------- pass B: staged tile -> c / out, thread = one 16-byte A4 unit, lanes along time
      if (ok && !(a.variant & 32)) {
        const int nq = min(32, (d.Cout - c.mtile * 128) >> 2);  // valid 4-row chunks of this tile
        const float4* st4p = reinterpret_cast<const float4*>(stile);
        const float4* par4 = reinterpret_cast<const float4*>(par);
        if (fold) {
          // D holds Tout = T + pl + pr columns of the zero-padded transposed conv; dx[t] = D[t+pl]
          // + D[pl-t] (1 <= t <= pl) + D[2(T-1)-t+pl] (t >= T-1-pr, t <= T-2) + residual adjoint
          const int Tf = d.Tout - fpl - fpr;
          RowIter ri;   // (g, cql) walk: per-sample base pointers, per-row pointer = base + row * stride
          ri.tstep = Tf <= 16 ? 16 : 32;
          ri.tl0 = lane % ri.tstep;
          const int frpp = 32 / ri.tstep, fsub = lane / ri.tstep;
          for (int g = 0; g < c.nsamp; ++g)
          for (int cql = ewarp * frpp + fsub; cql < nq; cql += 8 * frpp) {
            const int b = c.b0 + g, cq = c.mtile * 32 + cql;
            const float4* sr = st4p + (size_t)cql * P + g * Ts;
            float* ob = d.out ? d.out + (size_t)b * d.out_bstride + ((size_t)cq * Tf) * 4 : nullptr;
            const float* rb = d.res ? d.res + (size_t)b * d.res_bstride + ((size_t)cq * d.res_T) * 4 : nullptr;
            // upstream block (nbw): its raw conv output c, statistics and AdaIN row for these 4 channels
            const float* ucb = nbw ? d.save_c + (((size_t)b * (d.Cout >> 2) + cq) * Tf) * 4 : nullptr;
            float4 um = zero4(), ur = make_float4(1.f, 1.f, 1.f, 1.f), ub = zero4(), ug = make_float4(1.f, 1.f, 1.f, 1.f);
            if (nbw && d.norm) {
              const float4 s01 = ldg4(d.stats + ((size_t)b * d.Cout + cq * 4) * 2), s23 = ldg4(d.stats + ((size_t)b * d.Cout + cq * 4) * 2 + 4);
              um = make_float4(s01.x, s01.z, s23.x, s23.z);
              ur = make_float4(s01.y, s01.w, s23.y, s23.w);
              if (d.cond) {
                ub = ldg4(d.cond + (size_t)b * d.cond_bstride + cq * 4);
                ug = ldg4(d.cond + (size_t)b * d.cond_bstride + d.Cout + cq * 4);
              }
            }
            float4 a0 = zero4(), a1 = zero4();   // sum of g, sum of g * xhat over the row (this lane's share)
            for (int t = ri.tl0; t < Tf; t += ri.tstep) {
              float4 o = sr[t + fpl];
              if (t >= 1 && t <= fpl) {
                const float4 m = sr[fpl - t];
                o.x += m.x; o.y += m.y; o.z += m.z; o.w += m.w;
              }
              if (t <= Tf - 2 && t >= Tf - 1 - fpr) {
                const float4 m = sr[2 * (Tf - 1) - t + fpl];
                o.x += m.x; o.y += m.y; o.z += m.z; o.w += m.w;
              }
              if (rb) {  // adjoint of the forward residual branch (same cases as fold_add_kernel)
                float4 r;
                if (d.res_mode == AVC_RES_SAME) {
                  r = ldg4(rb + (size_t)t * 4);
                } else if (d.res_mode == AVC_RES_POOL) {
                  r = ldg4(rb + (size_t)(t >> 1) * 4);
                  const float wgt = ((Tf & 1) && t == Tf - 1) ? 1.f : 0.5f;
                  r.x *= wgt; r.y *= wgt; r.z *= wgt; r.w *= wgt;
                } else {
                  r = ldg4(rb + (size_t)(2 * t) * 4);
                  const float4 r2 = ldg4(rb + (size_t)(2 * t + 1) * 4);
                  r.x += r2.x; r.y += r2.y; r.z += r2.z; r.w += r2.w;
                }
                o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
              }
              if (ob) st4(ob + (size_t)t * 4, o);
              if (nbw) {
                // first half of the upstream norm backward: ReLU mask, row sums; the masked gradient goes back into
                // the staged tile (column t + fpl is read by this lane only)
                const float4 c4 = ldg4(ucb + (size_t)t * 4);
                float4 xh = c4, pre = c4;
                if (d.norm) {
                  xh = make_float4((c4.x - um.x) * ur.x, (c4.y - um.y) * ur.y, (c4.z - um.z) * ur.z, (c4.w - um.w) * ur.w);
                  pre = make_float4(fmaf(xh.x, ug.x, ub.x), fmaf(xh.y, ug.y, ub.y), fmaf(xh.z, ug.z, ub.z), fmaf(xh.w, ug.w, ub.w));
                }
                if (d.relu) {
                  o.x = pre.x > 0.f ? o.x : 0.f; o.y = pre.y > 0.f ? o.y : 0.f; o.z = pre.z > 0.f ? o.z : 0.f; o.w = pre.w > 0.f ? o.w : 0.f;
                }
                a0.x += o.x; a0.y += o.y; a0.z += o.z; a0.w += o.w;
                a1.x = fmaf(o.x, xh.x, a1.x); a1.y = fmaf(o.y, xh.y, a1.y); a1.z = fmaf(o.z, xh.z, a1.z); a1.w = fmaf(o.w, xh.w, a1.w);
                const_cast<float4*>(sr)[t + fpl] = o;
              }
            }
            if (nbw) {
              // row sums across the lanes of this row (16 or 32 lanes)
#pragma unroll
              for (int off = 16; off > 0; off >>= 1) {
                if (off < ri.tstep) {
                  a0.x += __shfl_xor_sync(0xffffffffu, a0.x, off); a0.y += __shfl_xor_sync(0xffffffffu, a0.y, off);
                  a0.z += __shfl_xor_sync(0xffffffffu, a0.z, off); a0.w += __shfl_xor_sync(0xffffffffu, a0.w, off);
                  a1.x += __shfl_xor_sync(0xffffffffu, a1.x, off); a1.y += __shfl_xor_sync(0xffffffffu, a1.y, off);
                  a1.z += __shfl_xor_sync(0xffffffffu, a1.z, off); a1.w += __shfl_xor_sync(0xffffffffu, a1.w, off);
                }
              }
              if (d.norm && d.dcond && ri.tl0 == 0) {   // AdaIN row gradients: d beta = sum g, d gamma = sum g * xhat
                st4(d.dcond + (size_t)b * d.dcond_bstride + cq * 4, a0);
                st4(d.dcond + (size_t)b * d.dcond_bstride + d.Cout + cq * 4, a1);
              }
              const float invT = 1.f / (float)Tf;
              const float4 m0 = make_float4(a0.x * invT, a0.y * invT, a0.z * invT, a0.w * invT);
              const float4 m1 = make_float4(a1.x * invT, a1.y * invT, a1.z * invT, a1.w * invT);
              const float4 k = make_float4(ur.x * ug.x, ur.y * ug.y, ur.z * ug.z, ur.w * ug.w);
              float* dcb = d.dc + (((size_t)b * (d.Cout >> 2) + cq) * Tf) * 4;
              float4 db = zero4();
              __syncwarp();
              for (int t = ri.tl0; t < Tf; t += ri.tstep) {
                float4 gq = sr[t + fpl];
                if (d.norm) {
                  const float4 c4 = ldg4(ucb + (size_t)t * 4);
                  const float4 xh = make_float4((c4.x - um.x) * ur.x, (c4.y - um.y) * ur.y, (c4.z - um.z) * ur.z, (c4.w - um.w) * ur.w);
                  gq = make_float4(k.x * (gq.x - m0.x - xh.x * m1.x), k.y * (gq.y - m0.y - xh.y * m1.y), k.z * (gq.z - m0.z - xh.z * m1.z),
                                   k.w * (gq.w - m0.w - xh.w * m1.w));
                }
                db.x += gq.x; db.y += gq.y; db.z += gq.z; db.w += gq.w;
                if (rnd_out) gq = t2_round4(gq);
                st4(dcb + (size_t)t * 4, gq);
              }
              if (d.dbias) {   // upstream bias gradient: per-CTA partial sums in shared memory, flushed once at the end
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) {
                  if (off < ri.tstep) {
                    db.x += __shfl_xor_sync(0xffffffffu, db.x, off); db.y += __shfl_xor_sync(0xffffffffu, db.y, off);
                    db.z += __shfl_xor_sync(0xffffffffu, db.z, off); db.w += __shfl_xor_sync(0xffffffffu, db.w, off);
                  }
                }
                if (ri.tl0 == 0) {
                  atomicAdd(dbacc + cql * 4 + 0, db.x); atomicAdd(dbacc + cql * 4 + 1, db.y);
                  atomicAdd(dbacc + cql * 4 + 2, db.z); atomicAdd(dbacc + cql * 4 + 3, db.w);
                }
              }
            }
          }
        } else if (!shuf && !d.mask && ots == 1 && (a.variant & 3) == 0) {
          // Common case (every block without pixel shuffle / mask): `c` and `out` in ONE sweep over the staged tile.
          // Per-sample base pointers, per-row pointer = base + row * stride, four time steps per lane in flight:
          // the per-row 64-bit address arithmetic of the generic loops below was a ~300-cycle dependent chain in
          // front of every store with only two epilogue warps per scheduler to hide it.
          const int lpr = c.tw <= 16 ? 16 : 32, rpp = 32 / lpr, sub = lane / lpr, tl0 = lane - sub * lpr;
          for (int g = 0; g < c.nsamp; ++g) {
            const int b = c.b0 + g;
            float* ob_g = d.out + (size_t)b * d.out_bstride + ((size_t)(c.mtile * 32) * out_T + c.t0 + oto) * 4;
            float* cb_g = d.save_c ? d.save_c + (((size_t)b * (d.Cout >> 2) + c.mtile * 32) * d.Tout + c.t0) * 4 : nullptr;
            const float* rb_g = d.res ? d.res + (size_t)b * d.res_bstride + ((size_t)(c.mtile * 32) * d.res_T) * 4 : nullptr;
            const float4* sr_g = st4p + g * Ts;
            for (int cql = ewarp * rpp + sub; cql < nq; cql += 8 * rpp) {
              const float4 mean4 = par4[(0 * a.G + g) * 32 + cql], sc4 = par4[(1 * a.G + g) * 32 + cql], sh4 = par4[(2 * a.G + g) * 32 + cql];
              const float4* sr = sr_g + (size_t)cql * P;
              float* ob = ob_g + (size_t)cql * out_T * 4;
              float* cb = cb_g ? cb_g + (size_t)cql * d.Tout * 4 : nullptr;
              const float* rb = rb_g ? rb_g + (size_t)cql * d.res_T * 4 : nullptr;
              for (int tb = tl0; tb < c.tw; tb += 4 * lpr) {
                float4 x[4], r[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                  const int tl_ = tb + k * lpr;
                  x[k] = tl_ < c.tw ? sr[tl_] : zero4();
                  r[k] = zero4();
                }
                if (rb) {
#pragma unroll
                  for (int k = 0; k < 4; ++k) {
                    const int tl_ = tb + k * lpr, t = c.t0 + tl_;
                    if (tl_ < c.tw) {
                      if (d.res_mode == AVC_RES_SAME) r[k] = ldg4(rb + (size_t)t * 4);
                      else if (d.res_mode == AVC_RES_UP) r[k] = ldg4(rb + (size_t)(t >> 1) * 4);
                      else {
                        r[k] = ldg4(rb + (size_t)(2 * t) * 4);
                        if (2 * t + 1 < d.res_T) {
                          const float4 r2 = ldg4(rb + (size_t)(2 * t + 1) * 4);
                          r[k] = make_float4(0.5f * (r[k].x + r2.x), 0.5f * (r[k].y + r2.y), 0.5f * (r[k].z + r2.z), 0.5f * (r[k].w + r2.w));
                        }
                      }
                    }
                  }
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                  const int tl_ = tb + k * lpr;
                  if (tl_ < c.tw) {
                    if (cb) st4(cb + (size_t)tl_ * 4, x[k]);
                    float4 o;
                    o.x = fmaf(x[k].x - mean4.x, sc4.x, sh4.x); o.y = fmaf(x[k].y - mean4.y, sc4.y, sh4.y);
                    o.z = fmaf(x[k].z - mean4.z, sc4.z, sh4.z); o.w = fmaf(x[k].w - mean4.w, sc4.w, sh4.w);
                    if (d.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
                    o.x += r[k].x; o.y += r[k].y; o.z += r[k].z; o.w += r[k].w;
                    if (rnd_out) o = t2_round4(o);
                    st4(ob + (size_t)tl_ * 4, o);
                  }
                }
              }
            }
          }
          if (a.dbg) e3b = clock64();
        } else {
          const bool bulk_c = (a.variant & 1) != 0;
          const bool bulk_y = (a.variant & 2) != 0 && !shuf && ots == 1;
          if (d.save_c) {  // raw conv (+bias) rows in conv layout, kept for the backward pass
            for (RowIter ri = t2_rows(ewarp, lane, c.tw, nq); ri.row < c.nsamp * nq; t2_next(ri)) {
              const int g = ri.g, cql = ri.cql;
              const float4* sr = st4p + (size_t)cql * P + g * Ts;
              float* cb = d.save_c + (((size_t)(c.b0 + g) * (d.Cout >> 2) + (c.mtile * 32 + cql)) * d.Tout + c.t0) * 4;
              if (bulk_c) {   // one bulk (TMA) store per row: the copy engine moves it, no LSU traffic
                if (ri.tl0 == 0) tc::bulk_s2g(cb, sr, (uint32_t)c.tw * 16u);
              } else {
                for (int t = ri.tl0; t < c.tw; t += ri.tstep) st4(cb + (size_t)t * 4, sr[t]);
              }
            }
            if (bulk_c) {
              tc::bulk_commit();
              if (bulk_y) tc::bulk_wait_read_all();   // the rows are about to be overwritten in place
            }
            __syncwarp();
          }
          if (a.dbg) e3b = clock64();
          const int nqo = shuf ? nq >> 1 : nq;       // output chunks of this tile
          const int two = shuf ? c.tw * 2 : c.tw;    // output time steps of this tile
          const int to0 = shuf ? c.t0 * 2 : c.t0;    // first output time step of this tile
          for (RowIter ri = t2_rows(ewarp, lane, two, nqo); ri.row < c.nsamp * nqo; t2_next(ri)) {
            const int g = ri.g, cql = ri.cql;
            const int b = c.b0 + g;
            const int cqo = c.mtile * (shuf ? 16 : 32) + cql;
            float* ob = d.out + (size_t)b * d.out_bstride + ((size_t)cqo * out_T) * 4;
            const float* rb = d.res ? d.res + (size_t)b * d.res_bstride + ((size_t)cqo * d.res_T) * 4 : nullptr;
            const float* mb = d.mask ? d.mask + (size_t)b * d.mask_bstride + ((size_t)cqo * Tn) * 4 : nullptr;
            float4 mean4, sc4, sh4;
            const float4 *srA, *srB = nullptr;
            if (!shuf) {
              mean4 = par4[(0 * a.G + g) * 32 + cql];
              sc4 = par4[(1 * a.G + g) * 32 + cql];
              sh4 = par4[(2 * a.G + g) * 32 + cql];
              srA = st4p + (size_t)cql * P + g * Ts;
            } else {
              // output channel 4*cql+j <- conv row 8*cql + 2j + s (s = output time parity): rows of the
              // conv chunks 2*cql (j = 0, 1) and 2*cql+1 (j = 2, 3); the parameters of a row pair are equal
              const float4 mA = par4[(0 * a.G + g) * 32 + 2 * cql], mB = par4[(0 * a.G + g) * 32 + 2 * cql + 1];
              const float4 cA = par4[(1 * a.G + g) * 32 + 2 * cql], cB = par4[(1 * a.G + g) * 32 + 2 * cql + 1];
              const float4 hA = par4[(2 * a.G + g) * 32 + 2 * cql], hB = par4[(2 * a.G + g) * 32 + 2 * cql + 1];
              mean4 = make_float4(mA.x, mA.z, mB.x, mB.z);
              sc4 = make_float4(cA.x, cA.z, cB.x, cB.z);
              sh4 = make_float4(hA.x, hA.z, hB.x, hB.z);
              srA = st4p + (size_t)(2 * cql) * P + g * Ts;
              srB = st4p + (size_t)(2 * cql + 1) * P + g * Ts;
            }
            for (int tl_ = ri.tl0; tl_ < two; tl_ += ri.tstep) {
              float4 x;
              if (!shuf) {
                x = srA[tl_];
              } else {
                const float4 va = srA[tl_ >> 1], vb = srB[tl_ >> 1];
                x = (tl_ & 1) ? make_float4(va.y, va.w, vb.y, vb.w) : make_float4(va.x, va.z, vb.x, vb.z);
              }
              const int t = to0 + tl_;  // output time step inside the sample
              float4 o;
              o.x = fmaf(x.x - mean4.x, sc4.x, sh4.x); o.y = fmaf(x.y - mean4.y, sc4.y, sh4.y);
              o.z = fmaf(x.z - mean4.z, sc4.z, sh4.z); o.w = fmaf(x.w - mean4.w, sc4.w, sh4.w);
              if (d.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
              if (rb) {
                float4 r;
                if (d.res_mode == AVC_RES_SAME) r = ldg4(rb + (size_t)t * 4);
                else if (d.res_mode == AVC_RES_UP) r = ldg4(rb + (size_t)(t >> 1) * 4);
                else {
                  r = ldg4(rb + (size_t)(2 * t) * 4);
                  if (2 * t + 1 < d.res_T) {
                    const float4 r2 = ldg4(rb + (size_t)(2 * t + 1) * 4);
                    r.x = 0.5f * (r.x + r2.x); r.y = 0.5f * (r.y + r2.y); r.z = 0.5f * (r.z + r2.z); r.w = 0.5f * (r.w + r2.w);
                  }
                }
                o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
              }
              if (mb) {
                const float4 m = ldg4(mb + (size_t)t * 4);
                o.x = m.x > 0.f ? o.x : 0.f; o.y = m.y > 0.f ? o.y : 0.f; o.z = m.z > 0.f ? o.z : 0.f; o.w = m.w > 0.f ? o.w : 0.f;
              }
              if (rnd_out) o = t2_round4(o);
              if (bulk_y) const_cast<float4*>(srA)[tl_] = o;   // in place: this warp owns the row
              else st4(ob + (size_t)(t * ots + oto) * 4, o);
            }
            if (bulk_y) {
              tc::fence_proxy_async_smem();
              __syncwarp();
              if (ri.tl0 == 0) tc::bulk_s2g(ob + (size_t)(to0 + oto) * 4, srA, (uint32_t)two * 16u);
            }
          }
          if (bulk_c || bulk_y) {
            tc::bulk_commit();
            tc::bulk_wait_read_all();   // the staged tile is rewritten by the next tile's accumulator pass
          }
        }
      }
      const long long e3c = a.dbg ? clock64() : 0;
      t2_bar_sync(2, 256);  // the staged tile and the parameter arrays are reused by the next tile
      if (a.dbg) {
        const long long e4 = clock64();
        if (e3b == 0) e3b = e3;
        dbg0 += e1 - e0; dbg1 += e2 - e1; dbg2 += e3 - e2; dbg3 += e3b - e3; dbg4 += e3c - e3b; dbg5 += e4 - e3c;
      }
    }
    if (nbw && d.dbias && etid < 128 && etid < d.Cout && tl > 0) atomicAdd(d.dbias + etid, dbacc[etid]);   // mtiles == 1 (plan)
    if (a.dbg && etid == 0) {
      long long* o = a.dbg + (size_t)blockIdx.x * 16;
      o[8] = dbg0; o[9] = dbg1; o[10] = dbg2; o[11] = dbg3; o[12] = tl; o[13] = dbg4; o[14] = dbg5;
    }
  }
  __syncthreads();
  if (a.dbg && tid == 0) {
    long long* o = a.dbg + (size_t)blockIdx.x * 16;
    o[0] = tm0; o[1] = clock64();
  }
}

// ------------------------------------------------------------------ host side: tile plan
static int t2_num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaDeviceProp p;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaGetDeviceProperties(&p, dev) == cudaSuccess) n = p.multiProcessorCount;
    if (n <= 0) n = 132;
  }
  return n;
}

// returns AVC_OK and fills a, or AVC_ERR_UNSUPPORTED (caller falls back to the round-1 kernel / FFMA path)
int t2_plan(const avc_conv_desc* d, Tc2Args& a) {
  const int K = d->K, S = d->stride;
  const bool fold = (d->flags & AVC_F_FOLD) != 0;
  a.d = *d;
  if (!a.d.res) a.d.res_mode = AVC_RES_NONE;
  a.nslab = d->Cin / T2_SLAB;
  a.nhalf = 2 * a.nslab;
  a.mtiles = cdiv(d->Cout, 128);
  const int ncol_full = (d->Tout - 1) * S + 1;
  if (d->pad_mode == AVC_PAD_REFLECT && d->Tin <= d->pad_left) return AVC_ERR_UNSUPPORTED;   // no mirror row to copy
  if ((d->flags & AVC_F_NORMBWD) && (!fold || d->Cout > 128 || !d->save_c || !d->dc || (d->norm && !d->stats))) return AVC_ERR_UNSUPPORTED;
  if (d->in_bstride % 4 != 0 || ((uintptr_t)d->in & 15u)) return AVC_ERR_UNSUPPORTED;        // tensor-map strides are multiples of 16 bytes
  // a folded data-gradient sample of up to 256 staged rows (one tensor-map box) stays one tile: its columns are
  // accumulated in chunks of 128
  const bool chunked = ncol_full > 144 && fold && ncol_full + K - 1 <= 256;
  if (ncol_full <= 144 || chunked) {
    a.TT = d->Tout;
    a.ntt = 1;
  } else {
    if (d->norm || fold || d->shuffle) return AVC_ERR_UNSUPPORTED;  // whole-sample statistics / fold need one tile per sample
    a.TT = S == 2 ? 64 : 128;
    a.ntt = cdiv(d->Tout, a.TT);
  }
  a.Ts = a.TT;  // fold: TT == Tout (all columns incl. the halo ones are staged)
  const int ncol = (a.TT - 1) * S + 1;
  a.R = ncol + K - 1;
  // samples per tile: minimise rounds x (fixed + MMA time); an N-column MMA costs ~max(40, N/2) cycles
  const int sms = t2_num_sms();
  int bestG = 0;
  double best = 1e30;
  const int gmax = a.ntt > 1 ? 1 : T2_MAX_G;
  for (int G = 1; G <= gmax && G <= d->B; ++G) {
    if (chunked) { bestG = 1; break; }
    if (G * a.Ts > 144) break;
    const int span = (G - 1) * a.R;
    if (span + (ncol + 15) / 16 * 16 > T2_MAX_N) break;
    const int N = (span + ncol + 15) / 16 * 16;
    const int ntiles = cdiv(d->B, G) * a.ntt * a.mtiles;
    const double mma = (double)a.nhalf * K * (N / 2 > 40 ? N / 2 : 40);
    const double cost = (double)cdiv(ntiles, sms) * (3000.0 + mma);
    if (cost <= best) { best = cost; bestG = G; }
  }
  if (bestG == 0) return AVC_ERR_UNSUPPORTED;
  a.G = bestG;
  a.N = ((a.G - 1) * a.R + ncol + 15) / 16 * 16;
  a.nchunk = 1;
  a.N_last = a.N;
  if (chunked) {
    a.N = 128;
    a.nchunk = cdiv(ncol, 128);
    a.N_last = (ncol - (a.nchunk - 1) * 128 + 15) / 16 * 16;
  }
  a.srows = a.G * a.R;   // one plane of the tensor-copy box: [G samples][R rows] of 16 bytes
  a.x_chunk_bytes = (uint32_t)a.srows * 16u;
  a.ngroups = cdiv(d->B, a.G);
  a.ntiles = a.ngroups * a.ntt * a.mtiles;
  // staged tile: 32 chunks, pitch == 1 mod 8 sixteen-byte units
  const int cols = a.G * a.Ts;
  a.P = (cols + 7) / 8 * 8 + 1;
  const uint32_t tile_bytes = 32u * (uint32_t)a.P * 16u;
  const uint32_t par_bytes = 3u * (uint32_t)a.G * 128u * 4u, stat_bytes = 2u * (uint32_t)a.G * 128u * 8u;
  const uint32_t tail = tile_bytes + par_bytes + stat_bytes;
  // Half-slabs per stage (see the header): one slab for K >= 2; the 1x1 layers have tiny half-slabs and want fewer
  // barrier round trips (hs = 4, falling back to one slab per stage when the tile leaves no room for three such stages).
  static int hs_env = -1;
  if (hs_env < 0) {
    const char* e = getenv("AVC_T2_HS");
    hs_env = e ? atoi(e) : 0;
  }
  int hs = K >= 2 ? 2 : 4;
  if (hs_env > 0) hs = hs_env == 1 ? 1 : (hs_env + 1) / 2 * 2;
  if (hs > a.nhalf) hs = a.nhalf;
  int nstage = 0;
  for (;; hs = hs > 2 ? hs - 2 : 1) {
    a.hs = hs;
    a.w_bytes = hs == 1 ? (uint32_t)K * T2_HALF_BYTES : (uint32_t)(hs / 2) * (uint32_t)K * T2_WTAP_BYTES;
    // an N-column MMA reads up to N + K - 1 rows of the last plane, at most 15 + K rows past its end (garbage columns):
    // keep that inside the stage
    a.stage_bytes = (a.w_bytes + 2u * (uint32_t)hs * a.x_chunk_bytes + 32u * 16u + 1023u) / 1024u * 1024u;
    nstage = (int)((T2_SMEM_MAX - (int)tail) / (int)a.stage_bytes);
    if (nstage >= 3 || hs == 1) break;
  }
  if (nstage > T2_MAX_STAGES) nstage = T2_MAX_STAGES;
  {
    static int cap = -1;   // probe: AVC_T2_NSTAGE caps the pipeline depth (how does the main loop scale with stages in flight?)
    if (cap < 0) {
      const char* e = getenv("AVC_T2_NSTAGE");
      cap = e ? atoi(e) : 0;
    }
    if (cap >= 2 && nstage > cap) nstage = cap;
  }
  if (nstage < 2) return AVC_ERR_UNSUPPORTED;
  a.nst = cdiv(a.nhalf, a.hs);
  a.nstage = nstage;
  a.off_tile = (uint32_t)nstage * a.stage_bytes;
  a.off_par = a.off_tile + tile_bytes;
  a.off_stat = a.off_par + par_bytes;
  return AVC_OK;
}

static long long* g_tc2_dbg = nullptr;
static int g_tc2_variant = -1;
static int t2_variant() {
  if (g_tc2_variant < 0) {
    const char* e = getenv("AVC_T2_VARIANT");
    g_tc2_variant = e ? atoi(e) : 0;
  }
  return g_tc2_variant;
}

int conv_block_tc2_launch(const avc_conv_desc* d, int* status, void* stream) {
  Tc2Args a;
  const int rc = t2_plan(d, a);
  if (rc != AVC_OK) return rc;
  a.status = status;
  a.dbg = g_tc2_dbg;
  a.patch = (!(d->flags & AVC_F_IN_TF32) || (d->pad_mode == AVC_PAD_REFLECT && d->K > 1)) ? 1 : 0;
  a.variant = t2_variant();
  CUtensorMap tmx, tmw;
  {
    PFN_tmap_encode enc = tmap_encode_fn();
    if (!enc) {
      set_error("avc_conv_block_tc: cuTensorMapEncodeTiled is not available from this driver");
      return AVC_ERR_CUDA;
    }
    const cuuint64_t gdim[4] = {4, (cuuint64_t)d->Tin, (cuuint64_t)d->B, (cuuint64_t)(d->Cin / 4)};
    const cuuint64_t gstr[3] = {16, (cuuint64_t)d->in_bstride * 4u, (cuuint64_t)d->Tin * 16u};
    const cuuint32_t box[4] = {4, (cuuint32_t)a.R, (cuuint32_t)a.G, (cuuint32_t)(2 * a.hs)};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    const CUresult r = enc(&tmx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)d->in, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("avc_conv_block_tc: cuTensorMapEncodeTiled failed (%d) for Tin=%d B=%d Cin=%d bstride=%lld box R=%d G=%d", (int)r, d->Tin, d->B,
                d->Cin, (long long)d->in_bstride, a.R, a.G);
      return AVC_ERR_CUDA;
    }
    tmw = tmx;   // unused unless hs == 1
    if (a.hs == 1) {
      if ((uintptr_t)d->w_tc & 15u) return AVC_ERR_UNSUPPORTED;
      // the weight pack [mtile][slab][tap][chunk 4][co 128][4] as rows of 2 KB, each split into two 1 KB halves (a box
      // dimension holds at most 256 elements): (256 floats, half, chunk, slab*K + tap)
      const cuuint64_t wdim[4] = {256, 2, 4, (cuuint64_t)a.mtiles * (cuuint64_t)a.nslab * (cuuint64_t)d->K};
      const cuuint64_t wstr[3] = {1024, 2048, 8192};
      const cuuint32_t wbox[4] = {256, 2, 2, (cuuint32_t)d->K};
      const CUresult rw = enc(&tmw, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)d->w_tc, wdim, wstr, wbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (rw != CUDA_SUCCESS) {
        set_error("avc_conv_block_tc: cuTensorMapEncodeTiled failed (%d) for the weight pack K=%d Cin=%d Cout=%d", (int)rw, d->K, d->Cin, d->Cout);
        return AVC_ERR_CUDA;
      }
    }
  }
  const int smem = (int)(a.off_stat + 2u * (uint32_t)a.G * 128u * 8u);
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(conv_block_tc2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, T2_SMEM_MAX);
    if (e != cudaSuccess) {
      set_error("avc_conv_block_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return AVC_ERR_CUDA;
    }
    attr_done = true;
  }
  const int grid = a.ntiles < t2_num_sms() ? a.ntiles : t2_num_sms();
  AVC_LAUNCH(conv_block_tc2_kernel, grid, 384, smem, (cudaStream_t)stream, a, tmx, tmw);
  AVC_CHECK_LAUNCH("conv_block_tc2");
  return AVC_OK;
}

}  // namespace avc

extern "C" void avc_tc2_set_debug(void* dev_buffer) { avc::g_tc2_dbg = (long long*)dev_buffer; }
extern "C" void avc_tc2_set_variant(int v) { avc::g_tc2_variant = v; }
