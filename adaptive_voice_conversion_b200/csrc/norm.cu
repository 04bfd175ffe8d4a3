// HBM-bound epilogue kernels on A4 tensors:
//  * avc_norm_apply_fwd : two-pass InstanceNorm/AdaIN/ReLU/residual for sequences too long
//                         for the fused conv tile (nn.InstanceNorm1d, append_cond; model.py:296,341,77-83)
//  * avc_norm_apply_varlen : the same over each sample's valid frames of a padded batch
//  * avc_norm_apply_morph : avc_norm_apply_varlen with a per-frame AdaIN mix of K anchor rows (time-varying morphs)
//  * avc_morph_weights    : the per-layer-frame anchor weights avc_norm_apply_morph reads
//  * avc_varlen_tail    : rewrites the frames just past each sample's length of a padded batch
//  * avc_norm_bwd       : backward of that epilogue (autograd under solver.py:90)
//  * avc_fold_add_fwd   : adjoint of F.pad(mode='reflect') (model.py:28-30) + residual adjoint
//  * avc_bias_grad      : bias gradient of a conv without epilogue
// One warp owns one (sample, 4-normalized-channel chunk) row: lanes stride over time with
// 16-byte vectors (coalesced along the time axis), statistics reduce with warp shuffles.
#include "common.cuh"

namespace avc {

int validate_conv_desc(const avc_conv_desc* d, const char* who);

__device__ __forceinline__ float rna_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__device__ __forceinline__ float4 warp_sum4(float4 v) {
  v.x = warp_sum(v.x);
  v.y = warp_sum(v.y);
  v.z = warp_sum(v.z);
  v.w = warp_sum(v.w);
  return v;
}

// Values of the 4 normalized channels of chunk qn at normalized time tn, read from the raw
// conv output c (dense A4 [Cout/4][Tout][4]).  SHUF: channel ch, time 2t+s <- conv row 2ch+s, time t.
template <bool SHUF>
__device__ __forceinline__ void load_rows(const float* cb /*sample base*/, int qn, int Tout, int t, float (&v)[2][4]) {
  if (!SHUF) {
    const float4 a = ldg4(cb + ((int64_t)qn * Tout + t) * 4);
    v[0][0] = a.x; v[0][1] = a.y; v[0][2] = a.z; v[0][3] = a.w;
    v[1][0] = v[1][1] = v[1][2] = v[1][3] = 0.f;
  } else {
    const float4 a = ldg4(cb + ((int64_t)(2 * qn) * Tout + t) * 4);      // ch0s0 ch0s1 ch1s0 ch1s1
    const float4 c = ldg4(cb + ((int64_t)(2 * qn + 1) * Tout + t) * 4);  // ch2s0 ch2s1 ch3s0 ch3s1
    v[0][0] = a.x; v[1][0] = a.y; v[0][1] = a.z; v[1][1] = a.w;
    v[0][2] = c.x; v[1][2] = c.y; v[0][3] = c.z; v[1][3] = c.w;
  }
}

// Valid frames of sample b of a padded batch: ceil(lengths[b] / div) * mul (avc_b200.h).
__device__ __forceinline__ int varlen_len(const int32_t* lengths, int b, int div, int mul) {
  return ((__ldg(lengths + b) + div - 1) / div) * mul;
}

// avc_norm_apply_morph: the layer's weight table [B][Tn][K] and the stride between a sample's K anchor rows in d.cond
struct MorphArgs {
  const float* wtab;
  int64_t kstride;
  int K;
};

// lengths null: every sample has Tout conv outputs; otherwise sample b has L_b = varlen_len(...) and only its first
// L_b (2 L_b after the shuffle) frames enter the statistics and are written.
// MORPH: frame tn's AdaIN row is sum_k wtab[b][tn][k] * (anchor k's row), formed with fmaf in k order from 0; each warp
// stages its sample's K anchor rows of its 4 channels in shared memory (blockDim / 32 * K * 2 float4)
template <bool SHUF, bool MORPH = false>
__global__ void __launch_bounds__(256) norm_apply_fwd_kernel(const avc_conv_desc d, const int32_t* __restrict__ lengths,
                                                             int div, int mul, MorphArgs m = {}) {
  constexpr int NS = SHUF ? 2 : 1;
  const int Cn = SHUF ? d.Cout / 2 : d.Cout;
  const int Tn = SHUF ? d.Tout * 2 : d.Tout;
  const int Cnq = Cn >> 2;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= d.B * Cnq) return;
  const int b = warp / Cnq, qn = warp - b * Cnq;
  const int Lc = lengths ? min(varlen_len(lengths, b, div, mul), d.Tout) : d.Tout;   // conv outputs used
  const float* cb = d.save_c + (int64_t)b * d.Cout * d.Tout;
  float mean[4] = {0, 0, 0, 0}, rstd[4] = {1, 1, 1, 1};
  if (d.norm) {
    float4 s = zero4();
    for (int t = lane; t < Lc; t += 32) {
      float v[2][4];
      load_rows<SHUF>(cb, qn, d.Tout, t, v);
#pragma unroll
      for (int sx = 0; sx < NS; ++sx) { s.x += v[sx][0]; s.y += v[sx][1]; s.z += v[sx][2]; s.w += v[sx][3]; }
    }
    s = warp_sum4(s);
    const float inv = 1.f / (float)(SHUF ? 2 * Lc : Lc);
    mean[0] = s.x * inv; mean[1] = s.y * inv; mean[2] = s.z * inv; mean[3] = s.w * inv;
    // corrected two-pass: the deviations also sum to the rounding error of the first pass's mean, which is removed
    // from the mean and the variance.  Without it a channel that is constant over time (rstd = eps^-1/2) normalises
    // to (c - mean) * 316 instead of 0.
    float4 m1 = zero4(), m2 = zero4();
    for (int t = lane; t < Lc; t += 32) {
      float v[2][4];
      load_rows<SHUF>(cb, qn, d.Tout, t, v);
#pragma unroll
      for (int sx = 0; sx < NS; ++sx) {
        float e;
        e = v[sx][0] - mean[0]; m1.x += e; m2.x += e * e;
        e = v[sx][1] - mean[1]; m1.y += e; m2.y += e * e;
        e = v[sx][2] - mean[2]; m1.z += e; m2.z += e * e;
        e = v[sx][3] - mean[3]; m1.w += e; m2.w += e * e;
      }
    }
    m1 = warp_sum4(m1);
    m2 = warp_sum4(m2);
    const float s1[4] = {m1.x, m1.y, m1.z, m1.w}, s2[4] = {m2.x, m2.y, m2.z, m2.w};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float dm = s1[c] * inv;
      mean[c] += dm;
      rstd[c] = rsqrtf(fmaxf(s2[c] * inv - dm * dm, 0.f) + d.eps);
    }
    if (d.stats && lane == 0) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        d.stats[((int64_t)b * Cn + qn * 4 + c) * 2 + 0] = mean[c];
        d.stats[((int64_t)b * Cn + qn * 4 + c) * 2 + 1] = rstd[c];
      }
    }
  }
  float beta[4] = {0, 0, 0, 0}, gamma[4] = {1, 1, 1, 1};
  float4* sh_beta = nullptr;   // MORPH: [K] anchor rows of this warp's 4 channels, then [K] gamma rows
  if constexpr (MORPH) {
    extern __shared__ float4 morph_sh[];
    sh_beta = morph_sh + (int64_t)(threadIdx.x >> 5) * 2 * m.K;
    for (int k = lane; k < m.K; k += 32) {
      const float* row = d.cond + (int64_t)b * d.cond_bstride + k * m.kstride + qn * 4;
      sh_beta[k] = make_float4(__ldg(row), __ldg(row + 1), __ldg(row + 2), __ldg(row + 3));
      sh_beta[m.K + k] = make_float4(__ldg(row + Cn), __ldg(row + Cn + 1), __ldg(row + Cn + 2), __ldg(row + Cn + 3));
    }
    __syncwarp();
  } else if (d.cond) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      beta[c] = __ldg(d.cond + (int64_t)b * d.cond_bstride + qn * 4 + c);
      gamma[c] = __ldg(d.cond + (int64_t)b * d.cond_bstride + Cn + qn * 4 + c);
    }
  }
  // a POOL residual's input holds ceil(lengths[b] / (div / 2)) * mul valid frames; an odd last one is averaged alone
  const int res_L = (lengths && d.res_mode == AVC_RES_POOL) ? min(varlen_len(lengths, b, div / 2, mul), d.res_T) : d.res_T;
  for (int t = lane; t < Lc; t += 32) {
    float v[2][4];
    load_rows<SHUF>(cb, qn, d.Tout, t, v);
#pragma unroll
    for (int sx = 0; sx < NS; ++sx) {
      const int tn = SHUF ? 2 * t + sx : t;
      if constexpr (MORPH) {
        const float* wr = m.wtab + ((int64_t)b * Tn + tn) * m.K;
        float4 bs = zero4(), gs = zero4();
#pragma unroll 1
        for (int k = 0; k < m.K; ++k) {
          const float w = __ldg(wr + k);
          const float4 bk = sh_beta[k], gk = sh_beta[m.K + k];
          bs.x = fmaf(w, bk.x, bs.x); bs.y = fmaf(w, bk.y, bs.y); bs.z = fmaf(w, bk.z, bs.z); bs.w = fmaf(w, bk.w, bs.w);
          gs.x = fmaf(w, gk.x, gs.x); gs.y = fmaf(w, gk.y, gs.y); gs.z = fmaf(w, gk.z, gs.z); gs.w = fmaf(w, gk.w, gs.w);
        }
        beta[0] = bs.x; beta[1] = bs.y; beta[2] = bs.z; beta[3] = bs.w;
        gamma[0] = gs.x; gamma[1] = gs.y; gamma[2] = gs.z; gamma[3] = gs.w;
      }
      float o[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float x = (v[sx][c] - mean[c]) * rstd[c];
        x = fmaf(x, gamma[c], beta[c]);
        o[c] = d.relu ? fmaxf(x, 0.f) : x;
      }
      float4 ov = make_float4(o[0], o[1], o[2], o[3]);
      if (d.res) {
        const float* rb = d.res + (int64_t)b * d.res_bstride + (int64_t)qn * d.res_T * 4;
        float4 r;
        if (d.res_mode == AVC_RES_SAME) r = ldg4(rb + (int64_t)tn * 4);
        else if (d.res_mode == AVC_RES_UP) r = ldg4(rb + (int64_t)(tn >> 1) * 4);
        else {
          r = ldg4(rb + (int64_t)(2 * tn) * 4);
          if (2 * tn + 1 < res_L) {
            const float4 r2 = ldg4(rb + (int64_t)(2 * tn + 1) * 4);
            r.x = 0.5f * (r.x + r2.x); r.y = 0.5f * (r.y + r2.y); r.z = 0.5f * (r.z + r2.z); r.w = 0.5f * (r.w + r2.w);
          }
        }
        ov.x += r.x; ov.y += r.y; ov.z += r.z; ov.w += r.w;
      }
      if (d.mask) {
        const float4 m = ldg4(d.mask + (int64_t)b * d.mask_bstride + ((int64_t)qn * Tn + tn) * 4);
        ov.x = m.x > 0.f ? ov.x : 0.f; ov.y = m.y > 0.f ? ov.y : 0.f;
        ov.z = m.z > 0.f ? ov.z : 0.f; ov.w = m.w > 0.f ? ov.w : 0.f;
      }
      if (d.flags & AVC_F_ROUND_OUT) ov = make_float4(rna_tf32(ov.x), rna_tf32(ov.y), rna_tf32(ov.z), rna_tf32(ov.w));
      st4(d.out + (int64_t)b * d.out_bstride + ((int64_t)qn * Tn + tn) * 4, ov);
    }
  }
}

template <bool SHUF>
__global__ void __launch_bounds__(256) norm_bwd_kernel(const avc_conv_desc d) {
  constexpr int NS = SHUF ? 2 : 1;
  const int Cn = SHUF ? d.Cout / 2 : d.Cout;
  const int Tn = SHUF ? d.Tout * 2 : d.Tout;
  const int Cnq = Cn >> 2;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= d.B * Cnq) return;
  const int b = warp / Cnq, qn = warp - b * Cnq;
  const float* cb = d.save_c + (int64_t)b * d.Cout * d.Tout;
  const float* dyb = d.dy + (int64_t)b * d.dy_bstride + (int64_t)qn * Tn * 4;
  float mean[4] = {0, 0, 0, 0}, rstd[4] = {1, 1, 1, 1}, beta[4] = {0, 0, 0, 0}, gamma[4] = {1, 1, 1, 1};
  if (d.norm) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      mean[c] = __ldg(d.stats + ((int64_t)b * Cn + qn * 4 + c) * 2 + 0);
      rstd[c] = __ldg(d.stats + ((int64_t)b * Cn + qn * 4 + c) * 2 + 1);
    }
  }
  if (d.cond) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      beta[c] = __ldg(d.cond + (int64_t)b * d.cond_bstride + qn * 4 + c);
      gamma[c] = __ldg(d.cond + (int64_t)b * d.cond_bstride + Cn + qn * 4 + c);
    }
  }
  // pass 1: s0 = sum g, s1 = sum g*xhat  (g = dy masked by the ReLU)
  float s0[4] = {0, 0, 0, 0}, s1[4] = {0, 0, 0, 0};
  if (d.norm) {
    for (int t = lane; t < d.Tout; t += 32) {
      float v[2][4];
      load_rows<SHUF>(cb, qn, d.Tout, t, v);
#pragma unroll
      for (int sx = 0; sx < NS; ++sx) {
        const int tn = SHUF ? 2 * t + sx : t;
        const float4 g4 = ldg4(dyb + (int64_t)tn * 4);
        const float g[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float xh = (v[sx][c] - mean[c]) * rstd[c];
          const float pre = fmaf(xh, gamma[c], beta[c]);
          const float gg = (d.relu && !(pre > 0.f)) ? 0.f : g[c];
          s0[c] += gg;
          s1[c] += gg * xh;
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      s0[c] = warp_sum(s0[c]);
      s1[c] = warp_sum(s1[c]);
    }
    if (d.dcond && lane == 0) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        d.dcond[(int64_t)b * d.dcond_bstride + qn * 4 + c] = s0[c];
        d.dcond[(int64_t)b * d.dcond_bstride + Cn + qn * 4 + c] = s1[c];
      }
    }
  }
  // pass 2: dc, bias gradient
  const float invT = 1.f / (float)Tn;
  float db[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
  float* dcb = d.dc + (int64_t)b * d.Cout * d.Tout;
  for (int t = lane; t < d.Tout; t += 32) {
    float v[2][4], o[2][4];
    load_rows<SHUF>(cb, qn, d.Tout, t, v);
#pragma unroll
    for (int sx = 0; sx < NS; ++sx) {
      const int tn = SHUF ? 2 * t + sx : t;
      const float4 g4 = ldg4(dyb + (int64_t)tn * 4);
      const float g[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float dv;
        if (d.norm) {
          const float xh = (v[sx][c] - mean[c]) * rstd[c];
          const float pre = fmaf(xh, gamma[c], beta[c]);
          const float gg = (d.relu && !(pre > 0.f)) ? 0.f : g[c];
          dv = rstd[c] * gamma[c] * (gg - invT * s0[c] - xh * invT * s1[c]);
        } else {
          dv = (d.relu && !(v[sx][c] > 0.f)) ? 0.f : g[c];
        }
        db[sx][c] += dv;
        o[sx][c] = (d.flags & AVC_F_ROUND_OUT) ? rna_tf32(dv) : dv;
      }
    }
    if (!SHUF) {
      st4(dcb + ((int64_t)qn * d.Tout + t) * 4, make_float4(o[0][0], o[0][1], o[0][2], o[0][3]));
    } else {
      st4(dcb + ((int64_t)(2 * qn) * d.Tout + t) * 4, make_float4(o[0][0], o[1][0], o[0][1], o[1][1]));
      st4(dcb + ((int64_t)(2 * qn + 1) * d.Tout + t) * 4, make_float4(o[0][2], o[1][2], o[0][3], o[1][3]));
    }
  }
  if (d.dbias) {
#pragma unroll
    for (int sx = 0; sx < NS; ++sx)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float s = warp_sum(db[sx][c]);
        if (lane == 0) {
          const int co = SHUF ? 2 * (qn * 4 + c) + sx : qn * 4 + c;
          if (d.dbias_part) d.dbias_part[(int64_t)b * d.Cout + co] = s;   // partial of sample b
          else atomicAdd(d.dbias + co, s);
        }
      }
  }
}

// norm_bwd for the common training shape (no pixel shuffle, Tout <= 128): the row of `c` and of
// `dy` is read ONCE into registers (4 float4 each per lane) and reused by both passes.
// Warps are numbered chunk-major (the 8 warps of a block work on the SAME 4-channel chunk of 8 consecutive
// samples), so the bias gradient is reduced inside the block first: one atomic per channel per block instead of
// one per warp (32 768 atomics on 128 addresses at B=256 were a measurable part of this kernel).
__global__ void __launch_bounds__(256) norm_bwd_cached_kernel(const avc_conv_desc d) {
  __shared__ float db_sh[8][4];
  const int Cn = d.Cout, Tn = d.Tout;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int bgroups = (d.B + 7) >> 3;                  // blocks per chunk
  const int qn = blockIdx.x / bgroups, b = (blockIdx.x - qn * bgroups) * 8 + wib;
  const bool live = b < d.B;                           // dead warps still join the block reduction below
  if (!live && !d.dbias) return;
  if (!live) {
    if (lane < 4) db_sh[wib][lane] = 0.f;
    __syncthreads();
    return;
  }
  const float* cb = d.save_c + (int64_t)b * d.Cout * d.Tout + (int64_t)qn * d.Tout * 4;
  const float* dyb = d.dy + (int64_t)b * d.dy_bstride + (int64_t)qn * Tn * 4;
  float mean[4] = {0, 0, 0, 0}, rstd[4] = {1, 1, 1, 1}, beta[4] = {0, 0, 0, 0}, gamma[4] = {1, 1, 1, 1};
  if (d.norm) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      mean[c] = __ldg(d.stats + ((int64_t)b * Cn + qn * 4 + c) * 2 + 0);
      rstd[c] = __ldg(d.stats + ((int64_t)b * Cn + qn * 4 + c) * 2 + 1);
    }
  }
  if (d.cond) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      beta[c] = __ldg(d.cond + (int64_t)b * d.cond_bstride + qn * 4 + c);
      gamma[c] = __ldg(d.cond + (int64_t)b * d.cond_bstride + Cn + qn * 4 + c);
    }
  }
  float xv[4][4], gv[4][4];   // [iteration][channel]: xhat (or c when !norm) and the ReLU-masked dy
  float s0[4] = {0, 0, 0, 0}, s1[4] = {0, 0, 0, 0};
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int t = lane + 32 * it;
    float4 c4 = zero4(), g4 = zero4();
    if (t < d.Tout) {
      c4 = ldg4(cb + (int64_t)t * 4);
      g4 = ldg4(dyb + (int64_t)t * 4);
    }
    const float cc[4] = {c4.x, c4.y, c4.z, c4.w}, gg[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float xh = d.norm ? (cc[c] - mean[c]) * rstd[c] : cc[c];
      const float pre = d.norm ? fmaf(xh, gamma[c], beta[c]) : cc[c];
      const float g = (t < d.Tout && !(d.relu && !(pre > 0.f))) ? gg[c] : 0.f;
      xv[it][c] = xh;
      gv[it][c] = g;
      s0[c] += g;
      s1[c] += g * xh;
    }
  }
  if (d.norm) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      s0[c] = warp_sum(s0[c]);
      s1[c] = warp_sum(s1[c]);
    }
    if (d.dcond && lane == 0) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        d.dcond[(int64_t)b * d.dcond_bstride + qn * 4 + c] = s0[c];
        d.dcond[(int64_t)b * d.dcond_bstride + Cn + qn * 4 + c] = s1[c];
      }
    }
  }
  const float invT = 1.f / (float)Tn;
  float db[4] = {0, 0, 0, 0};
  float* dcb = d.dc + (int64_t)b * d.Cout * d.Tout + (int64_t)qn * d.Tout * 4;
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int t = lane + 32 * it;
    float o[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float dv = d.norm ? rstd[c] * gamma[c] * (gv[it][c] - invT * s0[c] - xv[it][c] * invT * s1[c]) : gv[it][c];
      db[c] += (t < d.Tout) ? dv : 0.f;
      o[c] = (d.flags & AVC_F_ROUND_OUT) ? rna_tf32(dv) : dv;
    }
    if (t < d.Tout) st4(dcb + (int64_t)t * 4, make_float4(o[0], o[1], o[2], o[3]));
  }
  if (d.dbias) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float s = warp_sum(db[c]);
      if (lane == 0) db_sh[wib][c] = s;
    }
    __syncthreads();
    if (threadIdx.x < 4) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) s += db_sh[w][threadIdx.x];
      if (d.dbias_part) d.dbias_part[(int64_t)(blockIdx.x - qn * bgroups) * d.Cout + qn * 4 + threadIdx.x] = s;   // partial of the sample group
      else atomicAdd(d.dbias + qn * 4 + threadIdx.x, s);
    }
  }
}

// thread = (sample b, layer frame j, anchor k): out[b][j][k] = mean over the f output frames t = j f + i of
// w[b][k][s] / sum_k' w[b][k'][s], s = min(t, L_b - 1); frames j >= 8 ceil(L_b / 8) / f are 0
__global__ void __launch_bounds__(256) morph_weights_kernel(const float* __restrict__ w, const int32_t* __restrict__ lengths,
                                                            int B, int K, int T, int f, float* __restrict__ out, int T_l) {
  const int64_t total = (int64_t)B * T_l * K;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % K);
    const int64_t bj = i / K;
    const int j = (int)(bj % T_l), b = (int)(bj / T_l);
    const int L = __ldg(lengths + b);
    const int n = ((L + 7) / 8) * 8 / f;
    float acc = 0.f;
    if (j < n) {
      const float* wb = w + (int64_t)b * K * T;
      for (int u = 0; u < f; ++u) {
        const int s = min(j * f + u, L - 1);
        float sum = 0.f;
        for (int kk = 0; kk < K; ++kk) sum += __ldg(wb + (int64_t)kk * T + s);
        acc += __ldg(wb + (int64_t)k * T + s) / sum;
      }
      acc *= 1.f / (float)f;   // f is a power of two: exact
    }
    out[i] = acc;
  }
}

// thread = (sample, 4-channel chunk, frame j past the sample's L_b); the modes of avc_varlen_tail (avc_b200.h)
__global__ void __launch_bounds__(256) varlen_tail_kernel(float* __restrict__ a4, int64_t bstride, int B, int C, int T,
                                                          const int32_t* __restrict__ lengths, int div, int mul, int mode, int n) {
  const int Cq = C >> 2;
  const int64_t total = (int64_t)B * Cq * n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(i % n);
    const int64_t bq = i / n;
    const int q = (int)(bq % Cq), b = (int)(bq / Cq);
    const int Lb = varlen_len(lengths, b, div, mul), t = Lb + j;
    if (t >= T) continue;
    float* row = a4 + (int64_t)b * bstride + (int64_t)q * T * 4;
    if (mode == AVC_TAIL_ZERO) st4(row + (int64_t)t * 4, zero4());
    else if (mode == AVC_TAIL_REFLECT) st4(row + (int64_t)t * 4, *reinterpret_cast<const float4*>(row + (int64_t)abs(Lb - 2 - j) * 4));
    else if (Lb & 1) st4(row + (int64_t)t * 4, *reinterpret_cast<const float4*>(row + (int64_t)(Lb - 1) * 4));   // REPLICATE
  }
}

__global__ void __launch_bounds__(256) fold_add_kernel(const avc_fold_desc d) {
  const int Cq = d.C >> 2;
  const int64_t total = (int64_t)d.B * Cq * d.Tin;
  const int Lp = d.Tin + d.pad_left + d.pad_right;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(idx % d.Tin);
    const int64_t bq = idx / d.Tin;
    const int q = (int)(bq % Cq);
    const int b = (int)(bq / Cq);
    const float* row = d.dxp + bq * Lp * 4;
    float4 v = ldg4(row + (int64_t)(t + d.pad_left) * 4);
    if (t >= 1 && t <= d.pad_left) {
      const float4 r = ldg4(row + (int64_t)(d.pad_left - t) * 4);
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    const int u2 = 2 * (d.Tin - 1) - t + d.pad_left;
    if (t <= d.Tin - 2 && u2 >= d.pad_left + d.Tin && u2 < Lp) {
      const float4 r = ldg4(row + (int64_t)u2 * 4);
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    if (d.dres) {
      const float* rb = d.dres + (int64_t)b * d.dres_bstride + (int64_t)q * d.res_T * 4;
      float4 r;
      if (d.res_mode == AVC_RES_SAME) {
        r = ldg4(rb + (int64_t)t * 4);
      } else if (d.res_mode == AVC_RES_POOL) {
        r = ldg4(rb + (int64_t)(t >> 1) * 4);
        const bool lone = (d.Tin & 1) && (t == d.Tin - 1);
        const float w = lone ? 1.f : 0.5f;
        r.x *= w; r.y *= w; r.z *= w; r.w *= w;
      } else {
        r = ldg4(rb + (int64_t)(2 * t) * 4);
        const float4 r2 = ldg4(rb + (int64_t)(2 * t + 1) * 4);
        r.x += r2.x; r.y += r2.y; r.z += r2.z; r.w += r2.w;
      }
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    st4(d.dx + (int64_t)b * d.dx_bstride + ((int64_t)q * d.Tin + t) * 4, v);
  }
}

// dbias[c] += sum over the nslices rows of part[slice][C], in slice order
__global__ void __launch_bounds__(256) partial_sum_kernel(const float* __restrict__ part, int nslices, int C, float* __restrict__ dbias) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int i = 0; i < nslices; ++i) s += part[(int64_t)i * C + c];
  dbias[c] += s;
}

// grid (C/4 chunks): one block reduces all (b, t) of its 4 channels in a fixed order and adds the result to dbias --
// no atomics, so the bias gradient is the same on every run
// dbias_tab != null: channel group g = c / group_c accumulates into dbias_tab[g][c % group_c] (several layers whose dc
// rows lie side by side in one tensor: the conv bank)
__global__ void __launch_bounds__(1024) bias_grad_kernel(const float* __restrict__ dc, int64_t bstride, float* __restrict__ dbias,
                                                         int B, int C, int T, float* const* __restrict__ dbias_tab, int group_c) {
  const int q = blockIdx.x;
  if (dbias_tab) dbias = dbias_tab[(q * 4) / group_c] - ((q * 4) / group_c) * group_c;
  float4 s = zero4();
  const int rows = blockDim.x / T;   // thread = (sample row, time step); the threads past rows * T idle
  if ((int)threadIdx.x < rows * T) {
    for (int b = threadIdx.x / T; b < B; b += rows) {
      const float4 v = ldg4(dc + (int64_t)b * bstride + ((int64_t)q * T + threadIdx.x % T) * 4);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
  }
  s = warp_sum4(s);
  __shared__ float4 part[32];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float4 r = zero4();
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { r.x += part[w].x; r.y += part[w].y; r.z += part[w].z; r.w += part[w].w; }
    dbias[q * 4 + 0] += r.x; dbias[q * 4 + 1] += r.y;
    dbias[q * 4 + 2] += r.z; dbias[q * 4 + 3] += r.w;
  }
}

}  // namespace avc

using namespace avc;

extern "C" int avc_norm_apply_fwd(const avc_conv_desc* d, void* stream) {
  int rc = validate_conv_desc(d, "avc_norm_apply_fwd");
  if (rc != AVC_OK) return rc;
  AVC_REQUIRE(d->save_c && d->out, AVC_ERR_INVALID, "avc_norm_apply_fwd: null save_c/out");
  AVC_REQUIRE(!d->res || d->res_mode != AVC_RES_NONE, AVC_ERR_INVALID, "avc_norm_apply_fwd: res without res_mode");
  const int Cn = d->shuffle ? d->Cout / 2 : d->Cout;
  const int64_t warps = (int64_t)d->B * (Cn / 4);
  const int blocks = (int)cdiv64(warps * 32, 256);
  if (d->shuffle) AVC_LAUNCH(norm_apply_fwd_kernel<true>, blocks, 256, 0, (cudaStream_t)stream, *d, nullptr, 1, 1);
  else AVC_LAUNCH(norm_apply_fwd_kernel<false>, blocks, 256, 0, (cudaStream_t)stream, *d, nullptr, 1, 1);
  AVC_CHECK_LAUNCH("norm_apply_fwd");
  return AVC_OK;
}

extern "C" int avc_norm_apply_varlen(const avc_conv_desc* d, const int32_t* lengths, int len_div, int len_mul, void* stream) {
  int rc = validate_conv_desc(d, "avc_norm_apply_varlen");
  if (rc != AVC_OK) return rc;
  AVC_REQUIRE(lengths && len_div >= 1 && len_mul >= 1, AVC_ERR_INVALID, "avc_norm_apply_varlen: lengths null or len_div/len_mul < 1");
  AVC_REQUIRE(d->save_c && d->out, AVC_ERR_INVALID, "avc_norm_apply_varlen: null save_c/out");
  AVC_REQUIRE(!d->res || d->res_mode != AVC_RES_NONE, AVC_ERR_INVALID, "avc_norm_apply_varlen: res without res_mode");
  AVC_REQUIRE(!d->res || d->res_mode != AVC_RES_POOL || len_div % 2 == 0, AVC_ERR_INVALID,
              "avc_norm_apply_varlen: a POOL residual needs an even len_div");
  AVC_REQUIRE(!d->mask, AVC_ERR_UNSUPPORTED, "avc_norm_apply_varlen: mask is not supported");
  const int Cn = d->shuffle ? d->Cout / 2 : d->Cout;
  const int blocks = (int)cdiv64((int64_t)d->B * (Cn / 4) * 32, 256);
  if (d->shuffle) AVC_LAUNCH(norm_apply_fwd_kernel<true>, blocks, 256, 0, (cudaStream_t)stream, *d, lengths, len_div, len_mul);
  else AVC_LAUNCH(norm_apply_fwd_kernel<false>, blocks, 256, 0, (cudaStream_t)stream, *d, lengths, len_div, len_mul);
  AVC_CHECK_LAUNCH("norm_apply_varlen");
  return AVC_OK;
}

extern "C" int avc_norm_apply_morph(const avc_conv_desc* d, const int32_t* lengths, int len_div, int len_mul, const float* wtab,
                                    int K, int64_t cond_kstride, void* stream) {
  int rc = validate_conv_desc(d, "avc_norm_apply_morph");
  if (rc != AVC_OK) return rc;
  AVC_REQUIRE(lengths && len_div >= 1 && len_mul >= 1, AVC_ERR_INVALID, "avc_norm_apply_morph: lengths null or len_div/len_mul < 1");
  AVC_REQUIRE(d->save_c && d->out, AVC_ERR_INVALID, "avc_norm_apply_morph: null save_c/out");
  AVC_REQUIRE(d->cond && wtab, AVC_ERR_INVALID, "avc_norm_apply_morph: null cond (anchor rows) or weight table");
  AVC_REQUIRE(K >= 1 && K <= AVC_MORPH_MAX_K, AVC_ERR_INVALID, "avc_norm_apply_morph: K=%d outside [1, %d]", K, AVC_MORPH_MAX_K);
  AVC_REQUIRE(!d->res || d->res_mode == AVC_RES_SAME || d->res_mode == AVC_RES_UP, AVC_ERR_INVALID,
              "avc_norm_apply_morph: the residual must be SAME or UP");
  AVC_REQUIRE(!d->mask, AVC_ERR_UNSUPPORTED, "avc_norm_apply_morph: mask is not supported");
  const int Cn = d->shuffle ? d->Cout / 2 : d->Cout;
  const int blocks = (int)cdiv64((int64_t)d->B * (Cn / 4) * 32, 256);
  const size_t smem = (size_t)(256 / 32) * 2 * K * sizeof(float4);
  const MorphArgs m{wtab, cond_kstride, K};
  const auto kern = d->shuffle ? norm_apply_fwd_kernel<true, true> : norm_apply_fwd_kernel<false, true>;
  AVC_LAUNCH(kern, blocks, 256, smem, (cudaStream_t)stream, *d, lengths, len_div, len_mul, m);
  AVC_CHECK_LAUNCH("norm_apply_morph");
  return AVC_OK;
}

extern "C" int avc_morph_weights(const float* w, const int32_t* lengths, int B, int K, int T, int f, float* out, int T_l,
                                 void* stream) {
  AVC_REQUIRE(w && lengths && out && B > 0 && T > 0 && T_l > 0, AVC_ERR_INVALID, "avc_morph_weights: bad argument");
  AVC_REQUIRE(K >= 1 && K <= AVC_MORPH_MAX_K, AVC_ERR_INVALID, "avc_morph_weights: K=%d outside [1, %d]", K, AVC_MORPH_MAX_K);
  AVC_REQUIRE(f >= 1 && f <= 8 && (f & (f - 1)) == 0, AVC_ERR_INVALID, "avc_morph_weights: f=%d is not 1, 2, 4 or 8", f);
  int blocks = (int)cdiv64((int64_t)B * T_l * K, 256);
  if (blocks > 148 * 16) blocks = 148 * 16;
  AVC_LAUNCH(morph_weights_kernel, blocks, 256, 0, (cudaStream_t)stream, w, lengths, B, K, T, f, out, T_l);
  AVC_CHECK_LAUNCH("morph_weights");
  return AVC_OK;
}

extern "C" int avc_varlen_tail(float* a4, int64_t bstride, int B, int C, int T, const int32_t* lengths, int len_div, int len_mul,
                               int mode, int n, void* stream) {
  AVC_REQUIRE(a4 && B > 0 && C > 0 && C % 4 == 0 && T > 0, AVC_ERR_INVALID, "avc_varlen_tail: bad argument");
  AVC_REQUIRE(lengths && len_div >= 1 && len_mul >= 1, AVC_ERR_INVALID, "avc_varlen_tail: lengths null or len_div/len_mul < 1");
  AVC_REQUIRE(mode == AVC_TAIL_REFLECT || mode == AVC_TAIL_REPLICATE || mode == AVC_TAIL_ZERO, AVC_ERR_INVALID,
              "avc_varlen_tail: bad mode %d", mode);
  if (mode == AVC_TAIL_REPLICATE) n = 1;
  else if (mode == AVC_TAIL_ZERO) n = T;
  AVC_REQUIRE(n >= 1 && n <= T, AVC_ERR_INVALID, "avc_varlen_tail: n=%d outside [1, T=%d]", n, T);
  int blocks = (int)cdiv64((int64_t)B * (C / 4) * n, 256);
  if (blocks > 148 * 16) blocks = 148 * 16;
  AVC_LAUNCH(varlen_tail_kernel, blocks, 256, 0, (cudaStream_t)stream, a4, bstride, B, C, T, lengths, len_div, len_mul, mode, n);
  AVC_CHECK_LAUNCH("varlen_tail");
  return AVC_OK;
}

extern "C" int avc_norm_bwd(const avc_conv_desc* d, void* stream) {
  int rc = validate_conv_desc(d, "avc_norm_bwd");
  if (rc != AVC_OK) return rc;
  AVC_REQUIRE(d->save_c && d->dy && d->dc, AVC_ERR_INVALID, "avc_norm_bwd: null save_c/dy/dc");
  AVC_REQUIRE(!d->norm || d->stats, AVC_ERR_INVALID, "avc_norm_bwd: norm without stats");
  AVC_REQUIRE(d->norm || !d->cond, AVC_ERR_UNSUPPORTED, "avc_norm_bwd: AdaIN without norm");
  const int Cn = d->shuffle ? d->Cout / 2 : d->Cout;
  const int64_t warps = (int64_t)d->B * (Cn / 4);
  const int blocks = (int)cdiv64(warps * 32, 256);
  const bool cached = !d->shuffle && d->Tout <= 128;
  if (d->shuffle) AVC_LAUNCH(norm_bwd_kernel<true>, blocks, 256, 0, (cudaStream_t)stream, *d);
  else if (cached) AVC_LAUNCH(norm_bwd_cached_kernel, (Cn / 4) * ((d->B + 7) / 8), 256, 0, (cudaStream_t)stream, *d);
  else AVC_LAUNCH(norm_bwd_kernel<false>, blocks, 256, 0, (cudaStream_t)stream, *d);
  AVC_CHECK_LAUNCH("norm_bwd");
  if (d->dbias && d->dbias_part) {   // partials: one row per sample, or per group of 8 samples (cached kernel)
    const int nslices = cached ? (d->B + 7) / 8 : d->B;
    AVC_LAUNCH(partial_sum_kernel, cdiv(d->Cout, 256), 256, 0, (cudaStream_t)stream, d->dbias_part, nslices, d->Cout, d->dbias);
    AVC_CHECK_LAUNCH("norm_bwd_dbias");
  }
  return AVC_OK;
}

extern "C" int avc_fold_add_fwd(const avc_fold_desc* d, void* stream) {
  AVC_REQUIRE(d && d->dxp && d->dx, AVC_ERR_INVALID, "avc_fold_add_fwd: null argument");
  AVC_REQUIRE(d->B > 0 && d->C > 0 && d->C % 4 == 0 && d->Tin > 0 && d->pad_left >= 0 && d->pad_right >= 0,
              AVC_ERR_INVALID, "avc_fold_add_fwd: bad shape");
  AVC_REQUIRE(!d->dres || (d->res_mode >= AVC_RES_SAME && d->res_mode <= AVC_RES_UP), AVC_ERR_INVALID,
              "avc_fold_add_fwd: bad res_mode");
  const int64_t total = (int64_t)d->B * (d->C / 4) * d->Tin;
  int blocks = (int)cdiv64(total, 256);
  if (blocks > 148 * 16) blocks = 148 * 16;
  AVC_LAUNCH(fold_add_kernel, blocks, 256, 0, (cudaStream_t)stream, *d);
  AVC_CHECK_LAUNCH("fold_add");
  return AVC_OK;
}

extern "C" int avc_bias_grad(const float* dc, int64_t bstride, float* dbias, int B, int C, int T, void* stream) {
  AVC_REQUIRE(dc && dbias && B > 0 && C > 0 && C % 4 == 0 && T > 0, AVC_ERR_INVALID, "avc_bias_grad: bad argument");
  AVC_REQUIRE(T <= 1024, AVC_ERR_UNSUPPORTED, "avc_bias_grad: T=%d > 1024", T);
  AVC_LAUNCH(bias_grad_kernel, C / 4, 1024, 0, (cudaStream_t)stream, dc, bstride, dbias, B, C, T, (float* const*)nullptr, 0);
  AVC_CHECK_LAUNCH("bias_grad");
  return AVC_OK;
}

extern "C" int avc_bias_grad_groups(const float* dc, int64_t bstride, float* const* dbias_tab_dev, int group_c, int B, int C, int T, void* stream) {
  AVC_REQUIRE(dc && dbias_tab_dev && B > 0 && C > 0 && C % 4 == 0 && T > 0 && group_c > 0 && group_c % 4 == 0 && C % group_c == 0, AVC_ERR_INVALID,
              "avc_bias_grad_groups: bad argument");
  AVC_REQUIRE(T <= 1024, AVC_ERR_UNSUPPORTED, "avc_bias_grad_groups: T=%d > 1024", T);
  AVC_LAUNCH(bias_grad_kernel, C / 4, 1024, 0, (cudaStream_t)stream, dc, bstride, (float*)nullptr, B, C, T, dbias_tab_dev, group_c);
  AVC_CHECK_LAUNCH("bias_grad_groups");
  return AVC_OK;
}
