// Fused ConvBlock forward, fp32 FFMA path (exact-fp32 twin of the tensor-core path).
//
//   reflect/zero pad -> Conv1d(K, stride) -> [pixel shuffle] -> [InstanceNorm over T]
//   -> [AdaIN gamma/beta] -> [ReLU] -> [+ residual (same | avg-pool2 | nearest-up2)] -> [* mask]
//
// replaces pad_layer + nn.Conv1d + pixel_shuffle_1d + nn.InstanceNorm1d + append_cond +
// ReLU + residual add of one reference ConvBlock (model.py:21-32, 52-59, 77-83, 237-250,
// 309-320, 354-369).
//
// Tiling: one CTA owns TCO output channels x TT output time steps; every thread an 8x8
// register tile (8 channels x 8 consecutive time steps).  A tile is cut into `nseg`
// power-of-two segments of `seg_out` columns, one sample per segment, so that the whole
// time axis of a sample sits inside the CTA and the InstanceNorm statistics are a
// shuffle reduction over the `seg_out/8` lanes of a segment (Chan/Welford merge).
// Input channels stream through shared memory 8 at a time: A4 global vectors are
// de-interleaved into planar rows [ci][time] (padding resolved at staging time), weights
// arrive pre-packed [ci][tap][co] so a tap's 8 channels are two broadcast LDS.128.
#include "common.cuh"

namespace avc {

constexpr int CK = 8;  // input channels per shared-memory stage

template <int K, int S, int TCO, int TT>
struct ConvCfg {
  static constexpr int NTX = TT / 8;
  static constexpr int NTY = TCO / 8;
  static_assert(NTX * NTY == 256, "256 threads per CTA");
  static constexpr int NX = 7 * S + K;  // input values one thread needs per channel
  static constexpr int NX4 = (NX + 3) / 4;
  static constexpr int SEG8 = ((8 * S + K - 1) + 3) / 4 * 4;
  static constexpr int XROW_A = (TT / 8) * SEG8;
  static constexpr int XROW_B = ((TT * S + K - 1) + 3) / 4 * 4;
  static constexpr int XROW = (XROW_A > XROW_B ? XROW_A : XROW_B) + 4;
  static constexpr int WROW = K * TCO;
  static constexpr int SMEM_BYTES = (CK * XROW + CK * WROW) * 4;
};

struct ConvArgs {
  avc_conv_desc d;
  int seg_out, nseg, segp, tiled, ntt;
};

__device__ __forceinline__ float rna_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

struct Wf {
  float n, mean, m2;
};
__device__ __forceinline__ Wf wf_merge(const Wf& a, const Wf& b) {
  Wf r;
  r.n = a.n + b.n;
  if (r.n <= 0.f) {
    r.mean = 0.f;
    r.m2 = 0.f;
    return r;
  }
  const float dlt = b.mean - a.mean;
  r.mean = (a.n * a.mean + b.n * b.mean) / r.n;
  r.m2 = a.m2 + b.m2 + dlt * dlt * (a.n * b.n / r.n);
  return r;
}

// Residual value for normalized-layout position (chunk q, time tn) of sample b.
__device__ __forceinline__ float4 res_fetch(const avc_conv_desc& d, int b, int q, int tn) {
  const float* base = d.res + (int64_t)b * d.res_bstride + (int64_t)q * d.res_T * 4;
  if (d.res_mode == AVC_RES_SAME) return ldg4(base + (int64_t)tn * 4);
  if (d.res_mode == AVC_RES_UP) return ldg4(base + (int64_t)(tn >> 1) * 4);
  // POOL: mean of (2tn, 2tn+1), a lone last element divides by one (ceil_mode=True)
  const int t1 = 2 * tn, t2 = 2 * tn + 1;
  float4 a = ldg4(base + (int64_t)t1 * 4);
  if (t2 < d.res_T) {
    float4 c = ldg4(base + (int64_t)t2 * 4);
    a.x = 0.5f * (a.x + c.x);
    a.y = 0.5f * (a.y + c.y);
    a.z = 0.5f * (a.z + c.z);
    a.w = 0.5f * (a.w + c.w);
  }
  return a;
}

// Epilogue on the thread's 8x8 tile.  SHUF: rows (2c, 2c+1) interleave in time into
// normalized channel c; NC normalized channels x NK time steps per thread.
template <bool SHUF>
__device__ __forceinline__ void conv_epilogue(float (&acc)[8][8], const ConvArgs& a, int b, int tq0,
                                              int cobase, int nvalid, int nlanes) {
  const avc_conv_desc& d = a.d;
  constexpr int NC = SHUF ? 4 : 8;
  constexpr int NK = SHUF ? 16 : 8;
#define VAL(ic, k) acc[SHUF ? (2 * (ic) + ((k)&1)) : (ic)][SHUF ? ((k) >> 1) : (k)]
  const int Cn = SHUF ? d.Cout / 2 : d.Cout;
  const int Tn = SHUF ? d.Tout * 2 : d.Tout;
  const int cnbase = SHUF ? cobase / 2 : cobase;
  const int nk = SHUF ? nvalid * 2 : nvalid;  // valid normalized time steps of this thread
  const int tn0 = SHUF ? tq0 * 2 : tq0;
  const bool bvalid = b < d.B;

  if (d.norm) {
#pragma unroll
    for (int ic = 0; ic < NC; ++ic) {
      Wf w;
      w.n = bvalid ? (float)nk : 0.f;
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < NK; ++k) s += (k < nk) ? VAL(ic, k) : 0.f;
      w.mean = w.n > 0.f ? s / w.n : 0.f;
      float m2 = 0.f;
#pragma unroll
      for (int k = 0; k < NK; ++k) {
        const float dv = VAL(ic, k) - w.mean;
        m2 += (k < nk) ? dv * dv : 0.f;
      }
      w.m2 = w.n > 0.f ? m2 : 0.f;
      for (int o = 1; o < nlanes; o <<= 1) {
        Wf other;
        other.n = __shfl_xor_sync(0xffffffffu, w.n, o);
        other.mean = __shfl_xor_sync(0xffffffffu, w.mean, o);
        other.m2 = __shfl_xor_sync(0xffffffffu, w.m2, o);
        w = wf_merge(w, other);
      }
      const float rstd = rsqrtf(w.m2 / fmaxf(w.n, 1.f) + d.eps);
#pragma unroll
      for (int k = 0; k < NK; ++k) VAL(ic, k) = (VAL(ic, k) - w.mean) * rstd;
      if (d.stats && bvalid && tq0 == 0 && cnbase + ic < Cn) {
        float* st = d.stats + ((int64_t)b * Cn + cnbase + ic) * 2;
        st[0] = w.mean;
        st[1] = rstd;
      }
    }
  }
  if (!bvalid) return;
  if (d.cond) {
#pragma unroll
    for (int ic = 0; ic < NC; ++ic) {
      if (cnbase + ic < Cn) {
        const float beta = __ldg(d.cond + (int64_t)b * d.cond_bstride + cnbase + ic);
        const float gamma = __ldg(d.cond + (int64_t)b * d.cond_bstride + Cn + cnbase + ic);
#pragma unroll
        for (int k = 0; k < NK; ++k) VAL(ic, k) = fmaf(VAL(ic, k), gamma, beta);
      }
    }
  }
  if (d.relu) {
#pragma unroll
    for (int ic = 0; ic < NC; ++ic)
#pragma unroll
      for (int k = 0; k < NK; ++k) VAL(ic, k) = fmaxf(VAL(ic, k), 0.f);
  }
#pragma unroll
  for (int g = 0; g < NC / 4; ++g) {
    if (cnbase + 4 * g >= Cn) continue;
    const int q = (cnbase >> 2) + g;
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      if (k >= nk) continue;
      const int tn = tn0 + k;
      float4 v = make_float4(VAL(4 * g + 0, k), VAL(4 * g + 1, k), VAL(4 * g + 2, k), VAL(4 * g + 3, k));
      if (d.res) {
        const float4 r = res_fetch(d, b, q, tn);
        v.x += r.x;
        v.y += r.y;
        v.z += r.z;
        v.w += r.w;
      }
      if (d.mask) {
        const float4 m = ldg4(d.mask + (int64_t)b * d.mask_bstride + ((int64_t)q * Tn + tn) * 4);
        v.x = m.x > 0.f ? v.x : 0.f;
        v.y = m.y > 0.f ? v.y : 0.f;
        v.z = m.z > 0.f ? v.z : 0.f;
        v.w = m.w > 0.f ? v.w : 0.f;
      }
      if (d.flags & AVC_F_ROUND_OUT) {
        v = make_float4(rna_tf32(v.x), rna_tf32(v.y), rna_tf32(v.z), rna_tf32(v.w));
      }
      st4(d.out + (int64_t)b * d.out_bstride + ((int64_t)q * Tn + tn) * 4, v);
    }
  }
#undef VAL
}

template <int K, int S, int TCO, int TT>
__global__ void __launch_bounds__(256, 2) conv_block_fwd_kernel(const ConvArgs a) {
  using C = ConvCfg<K, S, TCO, TT>;
  extern __shared__ __align__(16) float smem[];
  float* Xs = smem;                 // [CK][XROW] planar input rows (padding resolved)
  float* Ws = smem + CK * C::XROW;  // [CK][K][TCO]
  const avc_conv_desc& d = a.d;
  const int tid = threadIdx.x;
  const int tx = tid % C::NTX, ty = tid / C::NTX;
  const int co0 = blockIdx.y * TCO;
  int b0, t0;
  if (a.tiled) {
    b0 = blockIdx.x / a.ntt;
    t0 = (blockIdx.x - b0 * a.ntt) * TT;
  } else {
    b0 = blockIdx.x * a.nseg;
    t0 = 0;
  }
  const int seg = (tx * 8) / a.seg_out;
  const int tl = (tx * 8) - seg * a.seg_out;
  const int L = d.Tin * d.in_ups;
  const int ncols = a.nseg * a.segp;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[i][k] = 0.f;

  for (int ci0 = 0; ci0 < d.Cin; ci0 += CK) {
    // ---- stage the input rows: A4 vectors -> 4 planar rows each
    for (int idx = tid; idx < 2 * ncols; idx += 256) {
      const int qq = idx / ncols;
      const int col = idx - qq * ncols;
      const int sg = col / a.segp;
      const int u = col - sg * a.segp;
      const int b = b0 + sg;
      const int ci = ci0 + qq * 4;
      float4 v = zero4();
      if (b < d.B && ci < d.Cin) {
        const int p = src_pos(t0 * S + u - d.pad_left, L, d.pad_mode, d.in_ups);
        if (p >= 0) v = ldg4(d.in + (int64_t)b * d.in_bstride + ((int64_t)(ci >> 2) * d.Tin + p) * 4);
      }
      float* xr = Xs + (qq * 4) * C::XROW + col;
      xr[0] = v.x;
      xr[C::XROW] = v.y;
      xr[2 * C::XROW] = v.z;
      xr[3 * C::XROW] = v.w;
    }
    // ---- stage the weights of these CK channels: rows (ci, tap) of TCO contiguous floats
    constexpr int W4 = TCO / 4;
    for (int idx = tid; idx < CK * K * W4; idx += 256) {
      const int row = idx / W4;
      const int c4 = idx - row * W4;
      const int cil = row / K;
      const int j = row - cil * K;
      const int ci = ci0 + cil;
      const int co = co0 + c4 * 4;
      float4 v = zero4();
      if (ci < d.Cin && co < d.Cout) v = ldg4(d.w_packed + ((int64_t)ci * K + j) * d.w_ld + co);
      st4(Ws + row * TCO + c4 * 4, v);
    }
    __syncthreads();

    const float* xb = Xs + seg * a.segp + tl * S;
#pragma unroll 1
    for (int c = 0; c < CK; ++c) {
      float x[C::NX4 * 4];
#pragma unroll
      for (int i = 0; i < C::NX4; ++i) {
        const float4 v = *reinterpret_cast<const float4*>(xb + c * C::XROW + 4 * i);
        x[4 * i + 0] = v.x;
        x[4 * i + 1] = v.y;
        x[4 * i + 2] = v.z;
        x[4 * i + 3] = v.w;
      }
#pragma unroll
      for (int j = 0; j < K; ++j) {
        const float4 w0 = *reinterpret_cast<const float4*>(Ws + (c * K + j) * TCO + ty * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(Ws + (c * K + j) * TCO + ty * 8 + 4);
        const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[i][k] = fmaf(w[i], x[k * S + j], acc[i][k]);
      }
    }
    __syncthreads();
  }

  // ---- epilogue
  const int cobase = co0 + ty * 8;
  const int b = b0 + seg;
  const int tq0 = t0 + tl;
  int nvalid = d.Tout - tq0;
  nvalid = nvalid < 0 ? 0 : (nvalid > 8 ? 8 : nvalid);
  if (d.bias) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float bv = (cobase + i < d.Cout) ? __ldg(d.bias + cobase + i) : 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[i][k] += bv;
    }
  }
  if (d.save_c && b < d.B) {
#pragma unroll
    for (int g = 0; g < 2; ++g) {
      if (cobase + 4 * g >= d.Cout) continue;
      float* base = d.save_c + (((int64_t)b * (d.Cout >> 2) + (cobase >> 2) + g) * d.Tout + tq0) * 4;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (k < nvalid) st4(base + k * 4, make_float4(acc[4 * g][k], acc[4 * g + 1][k], acc[4 * g + 2][k], acc[4 * g + 3][k]));
    }
  }
  const int nlanes = a.seg_out / 8;
  if (d.shuffle)
    conv_epilogue<true>(acc, a, b, tq0, cobase, nvalid, nlanes);
  else
    conv_epilogue<false>(acc, a, b, tq0, cobase, nvalid, nlanes);
}

template <int K, int S, int TCO, int TT>
static int launch_conv(const ConvArgs& a, dim3 grid, cudaStream_t st) {
  using C = ConvCfg<K, S, TCO, TT>;
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(conv_block_fwd_kernel<K, S, TCO, TT>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) {
      set_error("conv_block_fwd: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return AVC_ERR_CUDA;
    }
    attr_done = true;
  }
  void (*kern)(const ConvArgs) = conv_block_fwd_kernel<K, S, TCO, TT>;  // a macro-safe name
  AVC_LAUNCH(kern, grid, 256, C::SMEM_BYTES, st, a);
  AVC_CHECK_LAUNCH("conv_block_fwd");
  return AVC_OK;
}

static int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

int validate_conv_desc(const avc_conv_desc* d, const char* who) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "%s: null descriptor", who);
  AVC_REQUIRE(d->B > 0 && d->Cin > 0 && d->Cout > 0 && d->Tin > 0 && d->Tout > 0, AVC_ERR_INVALID,
              "%s: non-positive shape", who);
  AVC_REQUIRE(d->Cin % 4 == 0 && d->Cout % 4 == 0, AVC_ERR_INVALID, "%s: channel counts must be multiples of 4 (A4 layout), got %d/%d", who, d->Cin, d->Cout);
  AVC_REQUIRE(!d->shuffle || d->Cout % 8 == 0, AVC_ERR_INVALID, "%s: pixel shuffle needs Cout %% 8 == 0", who);
  AVC_REQUIRE(d->in_ups == 1 || d->in_ups == 2, AVC_ERR_INVALID, "%s: in_ups must be 1 or 2", who);
  return AVC_OK;
}

}  // namespace avc

using namespace avc;

extern "C" int avc_conv_block_fwd(const avc_conv_desc* d, void* stream) {
  int rc = validate_conv_desc(d, "avc_conv_block_fwd");
  if (rc != AVC_OK) return rc;
  AVC_REQUIRE(d->in && d->w_packed && d->out, AVC_ERR_INVALID, "avc_conv_block_fwd: null in/w/out");
  AVC_REQUIRE(d->K >= 1 && d->K <= 8, AVC_ERR_UNSUPPORTED, "avc_conv_block_fwd: K=%d not in 1..8", d->K);
  AVC_REQUIRE(d->stride == 1 || (d->stride == 2 && d->K == 5), AVC_ERR_UNSUPPORTED,
              "avc_conv_block_fwd: stride %d with K=%d unsupported", d->stride, d->K);
  AVC_REQUIRE(d->w_ld % 4 == 0 && d->w_ld >= d->Cout, AVC_ERR_INVALID, "avc_conv_block_fwd: bad w_ld");
  AVC_REQUIRE(!d->res || d->res_mode != AVC_RES_NONE, AVC_ERR_INVALID, "avc_conv_block_fwd: res without res_mode");
  cudaStream_t st = (cudaStream_t)stream;
  ConvArgs a;
  a.d = *d;
  if (!a.d.res) a.d.res_mode = AVC_RES_NONE;
  const int S = d->stride, K = d->K;
  int TT, TCO;
  if (d->Tout <= 128) {
    TT = 128;
    TCO = 128;
    a.tiled = 0;
    a.seg_out = next_pow2(d->Tout < 8 ? 8 : d->Tout);
    a.nseg = TT / a.seg_out;
    a.ntt = 1;
  } else if (d->norm && d->Tout <= 256 && (K == 1 || K == 5)) {
    TT = 256;
    TCO = 64;
    a.tiled = 0;
    a.seg_out = 256;
    a.nseg = 1;
    a.ntt = 1;
  } else if (!d->norm) {
    TT = 128;
    TCO = 128;
    a.tiled = 1;
    a.seg_out = 128;
    a.nseg = 1;
    a.ntt = cdiv(d->Tout, TT);
  } else {
    set_error("avc_conv_block_fwd: fused InstanceNorm needs Tout <= 256 (got %d); use avc_norm_apply_fwd", d->Tout);
    return AVC_ERR_UNSUPPORTED;
  }
  a.segp = ((a.seg_out * S + K - 1) + 3) / 4 * 4;
  dim3 grid(a.tiled ? d->B * a.ntt : cdiv(d->B, a.nseg), cdiv(d->Cout, TCO));
#define CASE(KK, SS)                                                          \
  if (K == KK && S == SS) {                                                   \
    if (TT == 128) return launch_conv<KK, SS, 128, 128>(a, grid, st);         \
  }
#define CASE256(KK, SS)                                                       \
  if (K == KK && S == SS && TT == 256) return launch_conv<KK, SS, 64, 256>(a, grid, st);
  CASE(1, 1) CASE(2, 1) CASE(3, 1) CASE(4, 1) CASE(5, 1) CASE(6, 1) CASE(7, 1) CASE(8, 1) CASE(5, 2)
  CASE256(1, 1) CASE256(5, 1) CASE256(5, 2)
#undef CASE
#undef CASE256
  set_error("avc_conv_block_fwd: no kernel for K=%d stride=%d tile=%d", K, S, TT);
  return AVC_ERR_UNSUPPORTED;
}
