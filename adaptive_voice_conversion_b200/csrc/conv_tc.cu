// Fused ConvBlock forward on the tensor cores (wgmma m64nNk8 tf32, fp32 accumulate), one tile per CTA.
//
// Same contract as conv_simt.cu (reflect/zero pad -> Conv1d -> [pixel shuffle] ->
// [InstanceNorm] -> [AdaIN] -> [ReLU] -> [+residual] -> [*mask]); replaces the same reference
// ops (model.py:21-32, 52-59, 77-83, 237-250, 309-320, 354-369) and, with the DGRAD pack and
// zero padding, autograd's conv data gradient.  The persistent kernel (conv_tc2.cu) runs every
// shape it plans; this one takes the rest up to TC_MAX_COLS columns per CTA.
//
// Formulation (no im2col): per sample, D[co][t] = sum_tap sum_ci W_tap[co][ci] * X[ci][t+tap].
//   * A operand = weights of one tap, K-major [ci/4][co][4] (no swizzle): 128 co rows x 16 ci.
//   * B operand = the input tile in its HBM layout [ci/4][row][4] staged ONCE per 16-channel
//     slab; the taps are the same tile at descriptor start + tap*16 bytes (row shift), so one
//     staged tile feeds all K taps.  Reflect / zero halos are patched in shared memory.
//   * D = 128 rows (co) x npad columns (time) per sample, in the registers of two consumer
//     warpgroups (64 rows each); after the main loop they are written to a shared-memory image
//     over the stage ring, and the epilogue reads it with thread <-> row <-> output channel, so the
//     InstanceNorm statistics of a (sample, channel) are a per-thread reduction over its row.
// Pipeline: warp 0 = bulk-copy (TMA) producer, warps 1+3 = halo patch + round-to-nearest TF32
// of the staged inputs (the tensor core truncates; rounding here keeps the path unbiased),
// warps 4-11 = the two wgmma warpgroups; all 16 warps run the epilogue.
#include "common.cuh"
#include "tc_common.cuh"

namespace avc {

int validate_conv_desc(const avc_conv_desc* d, const char* who);
int opt_tc_conv_v2();
int conv_block_tc2_launch(const avc_conv_desc* d, int* status, void* stream);  // conv_tc2.cu

constexpr int TC_SLAB = 16;          // input channels per pipeline stage (2 MMA K-steps)
constexpr int TC_WTAP_BYTES = 8192;  // one tap of one slab: 4 chunks x 128 co x 16 B
constexpr int TC_MAX_STAGES = 4;
constexpr int TC_MAX_COLS = 128;   // accumulator columns of a CTA (G samples x npad): 64 registers per consumer thread

struct TcArgs {
  avc_conv_desc d;
  int G, npad, rows, nslab, nstage;  // samples/CTA, padded cols/sample, smem rows/sample, Cin/16, ring depth
  uint32_t stage_bytes, w_bytes;
  int* status;
  long long* dbg;  // optional: per-CTA phase timestamps (tools/diag_phases.py)
};

__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// 4x4 transpose across the 4 lanes of a quad: in: lane r holds (a0..a3) = 4 consecutive time
// steps of ITS channel; out: lane r holds the 4 channels of the quad at time step r.
__device__ __forceinline__ void quad_transpose(float& a0, float& a1, float& a2, float& a3, int r) {
  {
    const bool odd = r & 1;
    const float s0 = odd ? a0 : a1, s1 = odd ? a2 : a3;
    const float g0 = __shfl_xor_sync(0xffffffffu, s0, 1), g1 = __shfl_xor_sync(0xffffffffu, s1, 1);
    if (odd) { a0 = g0; a2 = g1; } else { a1 = g0; a3 = g1; }
  }
  {
    const bool hi = r & 2;
    const float s0 = hi ? a0 : a2, s1 = hi ? a1 : a3;
    const float g0 = __shfl_xor_sync(0xffffffffu, s0, 2), g1 = __shfl_xor_sync(0xffffffffu, s1, 2);
    if (hi) { a0 = g0; a1 = g1; } else { a2 = g0; a3 = g1; }
  }
}

// Main loop of one consumer warpgroup (accumulator rows 64 wg .. 64 wg + 63): per 16-channel slab, 2 k-steps x nsamp
// samples x K taps of wgmma m64nNk8 (N = npad), taps j = 0..K-1 of one (k-step, sample) accumulating into the same
// registers; sample g owns acc[g * N / 2, (g + 1) * N / 2).  Then the accumulators go to the shared-memory image
// img[row][col] (row pitch `pitch` floats, col = g * npad + time column) that the epilogue reads.
template <int N>
__device__ __forceinline__ bool tc_mainloop(const TcArgs& a, uint32_t smem0, uint64_t* bar_ready, uint64_t* bar_empty, int nsamp, int wg,
                                            int wt, float* img, int pitch) {
  constexpr int GMAX = TC_MAX_COLS / N;
  float acc[GMAX * N / 2];
  const int K = a.d.K;
  const uint32_t x_chunk_bytes = (uint32_t)(a.G * a.rows) * 16u;
  const uint32_t ks_b = 2u * (x_chunk_bytes >> 4);
  const uint32_t d_hi = tc::sdesc_hi(128);
  for (int i = 0; i < a.nslab; ++i) {
    const int s = i % a.nstage;
    const uint32_t ph = (uint32_t)(i / a.nstage) & 1u;
    if (!__all_sync(0xffffffffu, tc::mbar_wait(&bar_ready[s], ph, a.status, 3))) return false;
    const uint32_t sw = smem0 + (uint32_t)s * a.stage_bytes;
    const uint32_t a_lo0 = tc::sdesc_lo(sw + (uint32_t)wg * 1024u, 2048), b_lo0 = tc::sdesc_lo(sw + a.w_bytes, x_chunk_bytes);
    tc::wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
#pragma unroll
      for (int g = 0; g < GMAX; ++g) {
        if (g >= nsamp) break;
        uint64_t a_desc = tc::sdesc64(a_lo0 + (uint32_t)ks * (4096 >> 4), d_hi);
        uint64_t b_desc = tc::sdesc64(b_lo0 + (uint32_t)ks * ks_b + (uint32_t)(g * a.rows), d_hi);
        for (int j = 0; j < K; ++j) {
          tc::wgmma_tf32<N>(acc + g * (N / 2), a_desc, b_desc, ((uint32_t)i | (uint32_t)ks | (uint32_t)j) ? 1u : 0u);
          a_desc += (uint64_t)(TC_WTAP_BYTES >> 4);
          b_desc += 1u;
        }
      }
    }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::acc_fence(acc, GMAX * N / 2);
    if (wt == 0) tc::mbar_arrive(&bar_empty[s]);
  }
  // the image overwrites the stage ring: both warpgroups must be done reading it
  asm volatile("bar.sync 2, 256;" ::: "memory");
#pragma unroll
  for (int g = 0; g < GMAX; ++g) {
    if (g >= nsamp) break;
#pragma unroll
    for (int r = 0; r < N / 2; ++r)
      img[(size_t)(64 * wg + tc::wg_acc_row(wt, r)) * pitch + g * a.npad + tc::wg_acc_col(wt, r)] = acc[g * (N / 2) + r];
  }
  return true;
}

// 16 consecutive accumulator columns of one row of the shared-memory image
__device__ __forceinline__ void img_ld16(const float* p, float (&v)[16]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = p[i];
}

// UI: warp index via lane-0 broadcast (AVC_TC_ISSUE=legacy: plain tid >> 5).
// FOLD (AVC_F_FOLD, plain stride-1 data-gradient convs): the epilogue applies the adjoint of the forward
// conv's reflect padding and of its residual branch itself (what avc_fold_add_fwd does in a second pass).
template <bool UI, bool FOLD>
__global__ void __launch_bounds__(512, 1) conv_block_tc_kernel(const TcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ uint64_t bar_full[TC_MAX_STAGES], bar_ready[TC_MAX_STAGES], bar_empty[TC_MAX_STAGES];
  __shared__ float2 ep_stat[4][128];  // partial InstanceNorm sums of the 4 epilogue warp groups
  const avc_conv_desc& d = a.d;
  const int tid = threadIdx.x, warp = UI ? tc::warp_idx_sync() : (tid >> 5), lane = tid & 31;
  const int b0 = blockIdx.x * a.G;
  const int mtile = blockIdx.y;
  const int nsamp = min(a.G, d.B - b0);
  const int xrows = a.G * a.rows;                 // rows of one chunk plane in a stage
  const uint32_t x_chunk_bytes = (uint32_t)xrows * 16u;

  if (tid == 0) {
    for (int s = 0; s < a.nstage; ++s) {
      tc::mbar_init(&bar_full[s], 1);
      tc::mbar_init(&bar_ready[s], 64);
      tc::mbar_init(&bar_empty[s], 2);
    }
    tc::fence_mbar_init();
  }
  __syncthreads();
  float* img = reinterpret_cast<float*>(smem);   // accumulator image, written over the stage ring after the main loop
  const int pitch = a.G * a.npad + 1;
  bool ok = true;
  long long tm0 = 0, tm1 = 0, tm2 = 0, dbg_acc0 = 0, dbg_acc1 = 0;
  if (a.dbg && tid == 64) tm0 = clock64();

  // ------------------------------------------------------------------ main loop (warp roles)
  if (warp == 0) {
    // TMA producer: warp-converged loop, one elected lane per bulk copy (uniform operands)
    const float* wsrc = d.w_tc + (size_t)mtile * a.nslab * (a.w_bytes / 4);
    for (int i = 0; i < a.nslab; ++i) {
      const int s = i % a.nstage;
      const uint32_t ph = (uint32_t)(i / a.nstage) & 1u;
      const long long w0 = a.dbg ? clock64() : 0;
      if (i >= a.nstage) ok = __all_sync(0xffffffffu, tc::mbar_wait(&bar_empty[s], ph ^ 1u, a.status, 2));
      if (a.dbg) dbg_acc0 += clock64() - w0;
      if (!ok) break;
      uint8_t* sw = smem + (size_t)s * a.stage_bytes;
      uint8_t* sx = sw + a.w_bytes;
      if (tc::elect_one()) {
        tc::mbar_arrive_expect_tx(&bar_full[s], a.w_bytes + (uint32_t)nsamp * 4u * (uint32_t)d.Tin * 16u);
        tc::bulk_g2s(sw, wsrc + (size_t)i * (a.w_bytes / 4), a.w_bytes, &bar_full[s]);
      }
      __syncwarp();
      for (int g = 0; g < nsamp; ++g)
        for (int q = 0; q < 4; ++q)
          if (tc::elect_one())
            tc::bulk_g2s(sx + (size_t)q * x_chunk_bytes + ((size_t)g * a.rows + d.pad_left) * 16,
                         d.in + (size_t)(b0 + g) * d.in_bstride + ((size_t)(i * 4 + q) * d.Tin) * 4, (uint32_t)d.Tin * 16u, &bar_full[s]);
    }
  } else if (warp >= 4 && warp < 12) {
    // two consumer warpgroups: wgmma main loop, accumulators -> shared-memory image
    const int wg = (warp - 4) >> 2, wt = tid & 127;
    const uint32_t smem0 = tc::smem_u32(smem);
    switch (a.npad) {
#define TC_CASE(n) \
  case n: ok = tc_mainloop<n>(a, smem0, bar_ready, bar_empty, nsamp, wg, wt, img, pitch); break;
      TC_CASE(16) TC_CASE(32) TC_CASE(48) TC_CASE(64) TC_CASE(80) TC_CASE(96) TC_CASE(112) TC_CASE(128)
#undef TC_CASE
      default: ok = false;
    }
  } else if (warp == 1 || warp == 3) {
    // warps 1 and 3: round staged inputs to TF32 (RN) and patch the halo rows
    const int ptid = (warp == 1 ? 0 : 32) + lane;  // 0..63
    for (int i = 0; i < a.nslab && ok; ++i) {
      const int s = i % a.nstage;
      const uint32_t ph = (uint32_t)(i / a.nstage) & 1u;
      const long long w0 = a.dbg ? clock64() : 0;
      ok = tc::mbar_wait(&bar_full[s], ph, a.status, 4);
      const long long w1 = a.dbg ? clock64() : 0;
      dbg_acc0 += w1 - w0;
      if (!ok) break;
      float4* sx = reinterpret_cast<float4*>(smem + (size_t)s * a.stage_bytes + a.w_bytes);
      // data rows: round in place.  One (g, t) decomposition per row, reused for the 4 chunks --
      // the runtime integer divisions were the kernel's bottleneck when done per element.
      const int per = (d.flags & AVC_F_IN_TF32) ? 0 : nsamp * d.Tin;
      for (int r = ptid; r < per; r += 64) {
        const int g = r / d.Tin, t = r - g * d.Tin;
        float4* p = sx + g * a.rows + d.pad_left + t;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float4 v = p[(size_t)q * xrows];
          v.x = round_tf32(v.x); v.y = round_tf32(v.y); v.z = round_tf32(v.z); v.w = round_tf32(v.w);
          p[(size_t)q * xrows] = v;
        }
      }
      __syncwarp();
      // the halo rows are copies of rounded data rows: both patch warps must be done rounding
      asm volatile("bar.sync 1, 64;" ::: "memory");
      const int halo = a.rows - d.Tin;  // rows that are not data (left pad + right pad + slack)
      for (int r = ptid; r < nsamp * halo; r += 64) {
        const int g = r / halo, h = r - g * halo;
        const int u = h < d.pad_left ? h : d.Tin + h;  // row index within the sample's segment
        const int p = src_pos(u - d.pad_left, d.Tin, d.pad_mode, 1);
        float4* base = sx + g * a.rows;
#pragma unroll
        for (int q = 0; q < 4; ++q) base[(size_t)q * xrows + u] = (p >= 0) ? base[(size_t)q * xrows + d.pad_left + p] : zero4();
      }
      tc::fence_proxy_async_smem();
      tc::mbar_arrive(&bar_ready[s]);
      if (a.dbg) dbg_acc1 += clock64() - w1;
    }
  }
  if (a.dbg && (tid == 0 || tid == 32 || tid == 64)) {  // producer / patcher / MMA thread: wait, work cycles
    long long* o = a.dbg + (size_t)(blockIdx.y * gridDim.x + blockIdx.x) * 12 + 4 + (tid >> 5) * 2;
    o[0] = dbg_acc0; o[1] = dbg_acc1;
  }

  // ------------------------------------------------------------------ epilogue (all warps)
  __syncwarp();
  ok = __syncthreads_and(ok) != 0;  // the accumulator image is complete
  if (a.dbg && tid == 64) tm1 = clock64();
  // 16 epilogue warps = 4 groups x 4 row quarters.  A group takes one (sample, column part):
  // with fewer than 4 samples per CTA the columns of a sample are split between groups and the
  // InstanceNorm partial sums are merged through shared memory.
  const int etid = tid & 127, egrp = warp >> 2;
  const int co = mtile * 128 + etid;  // conv output row of this thread
  const bool co_ok = co < d.Cout;
  if (ok) {
    const float bias = (d.bias && co_ok) ? __ldg(d.bias + co) : 0.f;
    const int shuf = d.shuffle;
    const int Cn = shuf ? d.Cout / 2 : d.Cout;
    const int Tn = shuf ? d.Tout * 2 : d.Tout;
    const int cn = shuf ? co >> 1 : co;  // normalized channel
    const int sx_ = shuf ? (co & 1) : 0;
    const int r4 = lane & 3;             // position inside the 4-lane quad (= channel within an A4 chunk)
    const int cq = (mtile * 128 + (etid & ~3)) >> 2;  // A4 chunk of the quad's 4 conv rows
    const bool q_ok = (mtile * 128 + (etid & ~3)) < d.Cout;
    const float* lane_addr = img + (size_t)etid * pitch;   // this thread's accumulator row
    // stride 2: the MMAs compute every input position; only even columns are conv outputs
    const int sshift = d.stride == 2 ? 1 : 0, smask = sshift;
    const int ots = d.out_tstride > 0 ? d.out_tstride : 1, oto = d.out_toff;  // out time index = t*ots + oto
    const int ncol = d.stride == 2 ? min(a.npad, 2 * d.Tout) : d.Tout;  // accumulator columns that matter
    const int nsplit = nsamp >= 3 ? 1 : (nsamp == 2 ? 2 : 4);
    const int items = nsamp * nsplit, nchunk = a.npad >> 4;
    for (int it0 = 0; it0 < items; it0 += 4) {
      const int item = it0 + egrp;
      const bool active = item < items;
      const int g = active ? item / nsplit : 0, part = active ? item - g * nsplit : 0;
      const int cbeg = active ? (part * nchunk / nsplit) << 4 : 0, cend = active ? ((part + 1) * nchunk / nsplit) << 4 : 0;
      const int b = b0 + g;
      float mean = 0.f, rstd = 1.f;
      if (d.norm) {
        float s1 = 0.f, s2 = 0.f;
        for (int c0 = cbeg; c0 < cend; c0 += 16) {
          float v[16];
          img_ld16(lane_addr + (uint32_t)(g * a.npad + c0), v);
#pragma unroll
          for (int i = 0; i < 16; ++i)
            if (c0 + i < ncol && ((c0 + i) & smask) == 0) {
              const float x = v[i] + bias;
              s1 += x;
              s2 = fmaf(x, x, s2);
            }
        }
        ep_stat[egrp][etid] = make_float2(s1, s2);
        __syncthreads();
        s1 = 0.f; s2 = 0.f;
        const int grp0 = egrp - part;  // first group working on this sample
        for (int p2 = 0; p2 < nsplit; ++p2) {
          const float2 ps = ep_stat[(grp0 + p2) & 3][etid];
          s1 += ps.x; s2 += ps.y;
        }
        __syncthreads();   // ep_stat is reused by the next batch of items
        if (shuf) {  // rows (2c, 2c+1) pool into normalized channel c
          s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
          s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
        }
        const float inv = 1.f / (float)Tn;
        mean = s1 * inv;
        const float var = fmaxf(s2 * inv - mean * mean, 0.f);
        rstd = rsqrtf(var + d.eps);
        if (d.stats && co_ok && sx_ == 0 && active && part == 0) {
          d.stats[((size_t)b * Cn + cn) * 2 + 0] = mean;
          d.stats[((size_t)b * Cn + cn) * 2 + 1] = rstd;
        }
      }
      if (!active) continue;
      if constexpr (FOLD) {
        // D holds Tout = T + pl + pr columns of the zero-padded transposed conv (dxp); the input gradient
        // is dx[t] = D[t+pl] + D[pl-t] (1 <= t <= pl) + D[2(T-1)-t+pl] (that column >= pl+T) + residual
        // adjoint.  All mirrored columns belong to this thread's own row.
        const int fpl = (d.flags >> 8) & 0xff, fpr = (d.flags >> 16) & 0xff;
        const int Tf = d.Tout - fpl - fpr;
        const float* col0 = lane_addr + g * a.npad;
        float Le[4], Re[4];
        {
          float v0[16], v1[16], v2[16];
          img_ld16(col0, v0);
          Le[0] = v0[0]; Le[1] = v0[1]; Le[2] = v0[2]; Le[3] = v0[3];
          const int rc0 = ((fpl + Tf) >> 4) << 4, ro = fpl + Tf - rc0;   // chunk and offset of column pl+T
          img_ld16(col0 + (uint32_t)rc0, v1);
          if (rc0 + 16 < a.npad) {
            img_ld16(col0 + (uint32_t)(rc0 + 16), v2);
          } else {
#pragma unroll
            for (int i = 0; i < 16; ++i) v2[i] = 0.f;
          }
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float r = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              r = (i == ro + e) ? v1[i] : r;
              r = (i + 16 == ro + e) ? v2[i] : r;
            }
            Re[e] = e < fpr ? r : 0.f;
          }
        }
        float* fobase = d.out + (size_t)b * d.out_bstride + ((size_t)cq * Tf) * 4;
        const float* frb = d.res ? d.res + (size_t)b * d.res_bstride + ((size_t)cq * d.res_T) * 4 : nullptr;
        const int ur = Tf - 2 + fpl;   // column that receives Re[0]; Re[e] goes to column ur - e
        for (int c0 = cbeg; c0 < cend; c0 += 16) {
          float v[16];
          img_ld16(col0 + (uint32_t)c0, v);
          if (c0 == 0) {   // left halo: source column e -> target column 2*pl - e (2*pl <= 8 < 16)
#pragma unroll
            for (int i = 0; i < 16; ++i)
#pragma unroll
              for (int e = 0; e < 4; ++e)
                if (e < fpl && i == 2 * fpl - e) v[i] += Le[e];
          }
          if (c0 + 16 > ur - 3 && c0 <= ur) {   // right halo
#pragma unroll
            for (int i = 0; i < 16; ++i)
#pragma unroll
              for (int e = 0; e < 4; ++e)
                if (e < fpr && c0 + i == ur - e) v[i] += Re[e];
          }
#pragma unroll
          for (int i4 = 0; i4 < 16; i4 += 4) {
            float x0 = v[i4], x1 = v[i4 + 1], x2 = v[i4 + 2], x3 = v[i4 + 3];
            quad_transpose(x0, x1, x2, x3, r4);
            const int t = c0 + i4 + r4 - fpl;   // this lane now owns one time step of the quad's 4 channels
            if (q_ok && t >= 0 && t < Tf) {
              float4 o = make_float4(x0, x1, x2, x3);
              if (frb) {   // adjoint of the forward residual branch (same cases as fold_add_kernel)
                float4 r;
                if (d.res_mode == AVC_RES_SAME) {
                  r = ldg4(frb + (size_t)t * 4);
                } else if (d.res_mode == AVC_RES_POOL) {
                  r = ldg4(frb + (size_t)(t >> 1) * 4);
                  const float wgt = ((Tf & 1) && t == Tf - 1) ? 1.f : 0.5f;
                  r.x *= wgt; r.y *= wgt; r.z *= wgt; r.w *= wgt;
                } else {
                  r = ldg4(frb + (size_t)(2 * t) * 4);
                  const float4 r2 = ldg4(frb + (size_t)(2 * t + 1) * 4);
                  r.x += r2.x; r.y += r2.y; r.z += r2.z; r.w += r2.w;
                }
                o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
              }
              st4(fobase + (size_t)t * 4, o);
            }
          }
        }
        continue;
      }
      float beta = 0.f, gamma = 1.f;
      if (d.cond && co_ok) {
        beta = __ldg(d.cond + (size_t)b * d.cond_bstride + cn);
        gamma = __ldg(d.cond + (size_t)b * d.cond_bstride + Cn + cn);
      }
      // raw conv (+bias) rows for backward: conv layout, always vectorizable
      float* cbase = d.save_c ? d.save_c + (((size_t)b * (d.Cout >> 2) + cq) * d.Tout) * 4 : nullptr;
      // non-shuffle output: the quad's 4 lanes are the 4 channels of A4 chunk cq
      float* obase = d.out + (size_t)b * d.out_bstride + ((size_t)cq * (d.out_T > 0 ? d.out_T : Tn)) * 4;
      const float* rbase = d.res ? d.res + (size_t)b * d.res_bstride + ((size_t)cq * d.res_T) * 4 : nullptr;
      const float* mbase = d.mask ? d.mask + (size_t)b * d.mask_bstride + ((size_t)cq * Tn) * 4 : nullptr;
      // shuffle output (scalar path): channel cn, time 2t+s
      float* outp = d.out + (size_t)b * d.out_bstride + ((size_t)(cn >> 2) * Tn) * 4 + (cn & 3);
      const float* resp = d.res ? d.res + (size_t)b * d.res_bstride + ((size_t)(cn >> 2) * d.res_T) * 4 + (cn & 3) : nullptr;
      const float* maskp = d.mask ? d.mask + (size_t)b * d.mask_bstride + ((size_t)(cn >> 2) * Tn) * 4 + (cn & 3) : nullptr;
      for (int c0 = cbeg; c0 < cend; c0 += 16) {
        float v[16];
        img_ld16(lane_addr + (uint32_t)(g * a.npad + c0), v);
#pragma unroll
        for (int i4 = 0; i4 < 16; i4 += 4) {
          float x0 = v[i4] + bias, x1 = v[i4 + 1] + bias, x2 = v[i4 + 2] + bias, x3 = v[i4 + 3] + bias;
          const int tc_ = c0 + i4 + r4;  // after the quad transpose this lane owns column tc_ for 4 channels
          const bool t_ok = tc_ < ncol && (tc_ & smask) == 0;
          const int t = tc_ >> sshift;   // conv output time step
          if (cbase) {
            float y0 = x0, y1 = x1, y2 = x2, y3 = x3;
            quad_transpose(y0, y1, y2, y3, r4);
            if (q_ok && t_ok) st4(cbase + (size_t)t * 4, make_float4(y0, y1, y2, y3));
          }
          if (d.norm) {
            x0 = (x0 - mean) * rstd; x1 = (x1 - mean) * rstd; x2 = (x2 - mean) * rstd; x3 = (x3 - mean) * rstd;
          }
          x0 = fmaf(x0, gamma, beta); x1 = fmaf(x1, gamma, beta); x2 = fmaf(x2, gamma, beta); x3 = fmaf(x3, gamma, beta);
          if (d.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); x2 = fmaxf(x2, 0.f); x3 = fmaxf(x3, 0.f); }
          if (!shuf) {
            quad_transpose(x0, x1, x2, x3, r4);
            if (q_ok && t_ok) {
              float4 o = make_float4(x0, x1, x2, x3);
              if (rbase) {
                float4 r;
                if (d.res_mode == AVC_RES_SAME) r = ldg4(rbase + (size_t)t * 4);
                else if (d.res_mode == AVC_RES_UP) r = ldg4(rbase + (size_t)(t >> 1) * 4);
                else {
                  r = ldg4(rbase + (size_t)(2 * t) * 4);
                  if (2 * t + 1 < d.res_T) {
                    const float4 r2 = ldg4(rbase + (size_t)(2 * t + 1) * 4);
                    r.x = 0.5f * (r.x + r2.x); r.y = 0.5f * (r.y + r2.y); r.z = 0.5f * (r.z + r2.z); r.w = 0.5f * (r.w + r2.w);
                  }
                }
                o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
              }
              if (mbase) {
                const float4 m = ldg4(mbase + (size_t)t * 4);
                o.x = m.x > 0.f ? o.x : 0.f; o.y = m.y > 0.f ? o.y : 0.f; o.z = m.z > 0.f ? o.z : 0.f; o.w = m.w > 0.f ? o.w : 0.f;
              }
              if (d.flags & AVC_F_ROUND_OUT) o = make_float4(round_tf32(o.x), round_tf32(o.y), round_tf32(o.z), round_tf32(o.w));
              st4(obase + (size_t)(t * ots + oto) * 4, o);
            }
          } else if (co_ok) {
            const float xs[4] = {x0, x1, x2, x3};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int tcc = c0 + i4 + i;
              if (tcc >= ncol || (tcc & smask)) continue;
              const int tt = tcc >> sshift;
              const int tn = 2 * tt + sx_;
              float x = xs[i];
              if (resp) {
                float r;
                if (d.res_mode == AVC_RES_SAME) r = __ldg(resp + (size_t)tn * 4);
                else if (d.res_mode == AVC_RES_UP) r = __ldg(resp + (size_t)(tn >> 1) * 4);
                else {
                  r = __ldg(resp + (size_t)(2 * tn) * 4);
                  if (2 * tn + 1 < d.res_T) r = 0.5f * (r + __ldg(resp + (size_t)(2 * tn + 1) * 4));
                }
                x += r;
              }
              if (maskp && !(__ldg(maskp + (size_t)tn * 4) > 0.f)) x = 0.f;
              outp[(size_t)tn * 4] = (d.flags & AVC_F_ROUND_OUT) ? round_tf32(x) : x;
            }
          }
        }
      }
    }
  }
  if (a.dbg && tid == 64) {
    tm2 = clock64();
    long long* o = a.dbg + (size_t)(blockIdx.y * gridDim.x + blockIdx.x) * 12;
    o[0] = tm0; o[1] = tm1; o[2] = tm2; o[3] = 0;
  }
}

// nn.Conv1d weight [Cout][Cin][K] -> per (m-tile, 16-channel slab) blocks
// [tap][chunk 4][co 128][4 floats], TF32-rounded, zero padded: one contiguous bulk copy per stage.
__global__ void pack_weight_tc_kernel(const float* __restrict__ w, float* __restrict__ p, int Cout, int Cin, int K, int mode,
                                      int co_total, int ci_total) {
  // mode FWD: conv(co', ci', j) = W[co'][ci'][j];  DGRAD: conv(co', ci', j) = W[ci'][co'][K-1-j]
  // co_total / ci_total: channel counts of the conv being packed (FWD: Cout/Cin, DGRAD: Cin/Cout)
  const int mt = (co_total + 127) / 128, nslab = (ci_total + TC_SLAB - 1) / TC_SLAB;
  const int64_t n = (int64_t)mt * nslab * K * 4 * 128 * 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int e = (int)(r % 4); r /= 4;
    const int col = (int)(r % 128); r /= 128;
    const int q = (int)(r % 4); r /= 4;
    const int j = (int)(r % K); r /= K;
    const int sl = (int)(r % nslab); r /= nslab;
    const int m = (int)r;
    const int co = m * 128 + col, ci = sl * TC_SLAB + q * 4 + e;
    float v = 0.f;
    if (co < co_total && ci < ci_total)
      v = (mode == AVC_PACK_FWD) ? __ldg(w + ((int64_t)co * Cin + ci) * K + j) : __ldg(w + ((int64_t)ci * Cin + co) * K + (K - 1 - j));
    p[i] = round_tf32(v);
  }
}

// All weight re-packs of a model in ONE launch: blockIdx.y walks a device-resident item table.
__global__ void __launch_bounds__(256) pack_weights_batch_kernel(const avc_pack_item* __restrict__ items) {
  const avc_pack_item it = items[blockIdx.y];
  const int Cout = it.Cout, Cin = it.Cin, K = it.K;
  const int64_t nw = (int64_t)Cout * Cin * K;
  const int64_t n_tf = it.tc_fwd ? (int64_t)((Cout + 127) / 128) * ((Cin + TC_SLAB - 1) / TC_SLAB) * K * 2048 : 0;
  const int64_t n_td = it.tc_dgrad ? (int64_t)((Cin + 127) / 128) * ((Cout + TC_SLAB - 1) / TC_SLAB) * K * 2048 : 0;
  int64_t nmax = nw;
  if (n_tf > nmax) nmax = n_tf;
  if (n_td > nmax) nmax = n_td;
  const float* w = it.w;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nmax; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < nw) {
      if (it.simt_fwd) {  // P[ci][j][co] = W[co][ci][j]
        const int co = (int)(i % Cout);
        const int64_t r = i / Cout;
        it.simt_fwd[i] = __ldg(w + ((int64_t)co * Cin + (int)(r / K)) * K + (int)(r % K));
      }
      if (it.simt_dgrad) {  // P[co][j][ci] = W[co][ci][K-1-j]
        const int ci = (int)(i % Cin);
        const int64_t r = i / Cin;
        it.simt_dgrad[i] = __ldg(w + ((int64_t)(r / K) * Cin + ci) * K + (K - 1 - (int)(r % K)));
      }
    }
#pragma unroll
    for (int mode = 0; mode < 4; ++mode) {  // 0 fwd, 1 dgrad, 2 dgrad even taps, 3 dgrad odd taps
      float* dst = mode == 0 ? it.tc_fwd : mode == 1 ? it.tc_dgrad : mode == 2 ? it.tc_dgrad_even : it.tc_dgrad_odd;
      if (!dst) continue;
      const int co_total = mode == 0 ? Cout : Cin, ci_total = mode == 0 ? Cin : Cout;
      const int nslab = (ci_total + TC_SLAB - 1) / TC_SLAB;
      const int Ks = mode < 2 ? K : mode == 2 ? (K + 1) / 2 : K / 2;  // taps in this pack
      const int64_t n = (int64_t)((co_total + 127) / 128) * nslab * Ks * 2048;
      if (i >= n) continue;
      int64_t r = i;
      const int e = (int)(r % 4); r /= 4;
      const int col = (int)(r % 128); r /= 128;
      const int q = (int)(r % 4); r /= 4;
      const int jj = (int)(r % Ks); r /= Ks;
      const int sl = (int)(r % nslab); r /= nslab;
      const int co = (int)r * 128 + col, ci = sl * TC_SLAB + q * 4 + e;
      const int j = mode < 2 ? jj : mode == 2 ? 2 * jj : 2 * jj + 1;  // tap of the full (flipped) dgrad conv
      float v = 0.f;
      if (co < co_total && ci < ci_total)
        v = (mode == 0) ? __ldg(w + ((int64_t)co * Cin + ci) * K + j) : __ldg(w + ((int64_t)ci * Cin + co) * K + (K - 1 - j));
      dst[i] = round_tf32(v);
    }
  }
}

}  // namespace avc

using namespace avc;

extern "C" int avc_pack_conv_weights_batch(const avc_pack_item* items_dev, int n_items, int64_t max_elems, void* stream) {
  AVC_REQUIRE(items_dev && n_items > 0 && max_elems > 0, AVC_ERR_INVALID, "avc_pack_conv_weights_batch: bad argument");
  int bx = (int)cdiv64(max_elems, 256 * 4);
  if (bx > 64) bx = 64;
  if (bx < 1) bx = 1;
  dim3 grid(bx, n_items);
  AVC_LAUNCH(pack_weights_batch_kernel, grid, 256, 0, (cudaStream_t)stream, items_dev);
  AVC_CHECK_LAUNCH("pack_weights_batch");
  return AVC_OK;
}

extern "C" int64_t avc_tc_packed_floats(int co_total, int ci_total, int K) {
  return (int64_t)((co_total + 127) / 128) * ((ci_total + TC_SLAB - 1) / TC_SLAB) * K * 4 * 128 * 4;
}

extern "C" int avc_pack_conv_weight_tc(const float* w, float* packed, int Cout, int Cin, int K, int mode, void* stream) {
  AVC_REQUIRE(w && packed && Cout > 0 && Cin > 0 && K > 0, AVC_ERR_INVALID, "avc_pack_conv_weight_tc: bad argument");
  AVC_REQUIRE(mode == AVC_PACK_FWD || mode == AVC_PACK_DGRAD, AVC_ERR_INVALID, "avc_pack_conv_weight_tc: bad mode");
  const int co_total = mode == AVC_PACK_FWD ? Cout : Cin, ci_total = mode == AVC_PACK_FWD ? Cin : Cout;
  const int64_t n = avc_tc_packed_floats(co_total, ci_total, K);
  int blocks = (int)cdiv64(n, 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  AVC_LAUNCH(pack_weight_tc_kernel, blocks, 256, 0, (cudaStream_t)stream, w, packed, Cout, Cin, K, mode, co_total, ci_total);
  AVC_CHECK_LAUNCH("pack_conv_weight_tc");
  return AVC_OK;
}

static long long* g_tc_dbg = nullptr;
extern "C" void avc_tc_set_debug(void* dev_buffer) { g_tc_dbg = (long long*)dev_buffer; }

extern "C" int avc_conv_block_tc(const avc_conv_desc* d, int* status, void* stream) {
  int rc = validate_conv_desc(d, "avc_conv_block_tc");
  if (rc != AVC_OK) return rc;
  const bool normbwd = (d->flags & AVC_F_NORMBWD) != 0;
  AVC_REQUIRE(d->in && d->w_tc && (d->out || normbwd) && status, AVC_ERR_INVALID, "avc_conv_block_tc: null in/w_tc/out/status");
  AVC_REQUIRE(!normbwd || ((d->flags & AVC_F_FOLD) && d->save_c && d->dc && (!d->norm || d->stats) && (!d->cond || d->dcond) && !d->shuffle),
              AVC_ERR_INVALID, "avc_conv_block_tc: AVC_F_NORMBWD needs AVC_F_FOLD and the upstream block's save_c / stats / dc (dcond with cond)");
  AVC_REQUIRE((d->stride == 1 || d->stride == 2) && d->in_ups == 1, AVC_ERR_UNSUPPORTED, "avc_conv_block_tc: stride must be 1 or 2, in_ups 1");
  AVC_REQUIRE(d->stride == 1 || !d->shuffle, AVC_ERR_UNSUPPORTED, "avc_conv_block_tc: stride 2 with pixel shuffle");
  AVC_REQUIRE(d->out_tstride <= 1 || (!d->shuffle && !d->res && !d->mask && !d->norm), AVC_ERR_UNSUPPORTED,
              "avc_conv_block_tc: out_tstride only for plain (data-gradient) convs");
  AVC_REQUIRE(d->K >= 1 && d->K <= 8, AVC_ERR_UNSUPPORTED, "avc_conv_block_tc: K=%d not in 1..8", d->K);
  if (d->flags & AVC_F_FOLD) {
    const int fpl = (d->flags >> 8) & 0xff, fpr = (d->flags >> 16) & 0xff;
    AVC_REQUIRE(d->stride == 1 && !d->shuffle && !d->mask && !d->bias && d->out_tstride <= 1 && (normbwd || (!d->norm && !d->relu && !d->cond && !d->save_c)),
                AVC_ERR_UNSUPPORTED, "avc_conv_block_tc: AVC_F_FOLD is for plain stride-1 (data-gradient) convs");
    AVC_REQUIRE(fpl <= 4 && fpr <= 4 && d->Tout - fpl - fpr >= 2 * fpl + 1 && d->Tout - fpl - fpr >= fpr + 2, AVC_ERR_UNSUPPORTED,
                "avc_conv_block_tc: AVC_F_FOLD pads (%d,%d) do not fit %d columns", fpl, fpr, d->Tout);
  }
  AVC_REQUIRE(d->Cin % TC_SLAB == 0, AVC_ERR_UNSUPPORTED, "avc_conv_block_tc: Cin %% 16 != 0");
  AVC_REQUIRE(!d->res || d->res_mode != AVC_RES_NONE, AVC_ERR_INVALID, "avc_conv_block_tc: res without res_mode");
  if (opt_tc_conv_v2()) {   // persistent kernel (conv_tc2.cu); shapes it does not plan fall through to the round-1 kernel
    const int rc2 = conv_block_tc2_launch(d, status, stream);
    if (rc2 != AVC_ERR_UNSUPPORTED) return rc2;
  }
  AVC_REQUIRE(!normbwd, AVC_ERR_UNSUPPORTED, "avc_conv_block_tc: AVC_F_NORMBWD needs the persistent kernel and a one-tile shape (Tout <= 144, Cout <= 128)");
  const int ncols_full = d->stride == 2 ? 2 * d->Tout - 1 : d->Tout;  // stride 2: full-resolution columns 0 .. 2(Tout-1)
  AVC_REQUIRE(ncols_full <= TC_MAX_COLS, AVC_ERR_UNSUPPORTED, "avc_conv_block_tc: more than %d columns per sample", TC_MAX_COLS);
  AVC_REQUIRE(!d->res || d->res_mode != AVC_RES_NONE, AVC_ERR_INVALID, "avc_conv_block_tc: res without res_mode");
  TcArgs a;
  a.d = *d;
  if (!a.d.res) a.d.res_mode = AVC_RES_NONE;
  a.status = status;
  a.dbg = g_tc_dbg;
  a.npad = (ncols_full + 15) / 16 * 16;
  a.rows = a.npad + d->K - 1;
  if (a.rows < d->Tin + d->pad_left) a.rows = d->Tin + d->pad_left;  // all data rows must fit
  a.nslab = d->Cin / TC_SLAB;
  a.w_bytes = (uint32_t)d->K * TC_WTAP_BYTES;
  const int mtiles = cdiv(d->Cout, 128);
  int G = cdiv(d->B * mtiles, 132);
  const int gmax_acc = TC_MAX_COLS / a.npad;
  if (G > gmax_acc) G = gmax_acc;
  if (G < 1) G = 1;
  const int smem_max = 220 * 1024;
  auto stage_bytes = [&](int g) { return (uint32_t)(a.w_bytes + 4 * g * a.rows * 16); };
  while (G > 1 && 2 * stage_bytes(G) > (uint32_t)smem_max) --G;
  AVC_REQUIRE(2 * stage_bytes(G) <= (uint32_t)smem_max, AVC_ERR_UNSUPPORTED, "avc_conv_block_tc: tile does not fit shared memory");
  a.G = G;
  a.stage_bytes = (stage_bytes(G) + 1023) / 1024 * 1024;
  a.nstage = smem_max / (int)a.stage_bytes;
  if (a.nstage > TC_MAX_STAGES) a.nstage = TC_MAX_STAGES;
  if (a.nstage > a.nslab) a.nstage = a.nslab;
  const int img_bytes = 128 * (G * a.npad + 1) * 4;
  const int smem = a.nstage * (int)a.stage_bytes > img_bytes ? a.nstage * (int)a.stage_bytes : img_bytes;
  static int attr_smem = 0;
  if (smem > attr_smem) {
    cudaError_t e = cudaFuncSetAttribute(conv_block_tc_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_block_tc_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_block_tc_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    if (e != cudaSuccess) {
      set_error("avc_conv_block_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return AVC_ERR_CUDA;
    }
    attr_smem = smem_max;
  }
  dim3 grid(cdiv(d->B, G), mtiles);
  void (*kern)(const TcArgs) = opt_tc_uniform_issue() ? conv_block_tc_kernel<true, false> : conv_block_tc_kernel<false, false>;
  if (d->flags & AVC_F_FOLD) kern = conv_block_tc_kernel<true, true>;
  AVC_LAUNCH(kern, grid, 512, smem, (cudaStream_t)stream, a);
  AVC_CHECK_LAUNCH("conv_block_tc");
  return AVC_OK;
}
