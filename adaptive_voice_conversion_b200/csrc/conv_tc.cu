// Tensor-core (wgmma TF32) fused ConvBlock: the C entry point avc_conv_block_tc and the weight packs it reads.
//
// avc_conv_block_tc validates the descriptor and runs the persistent kernel (conv_tc2.cu), which implements the
// contract of conv_simt.cu (reflect/zero pad -> Conv1d -> [pixel shuffle] -> [InstanceNorm] -> [AdaIN] -> [ReLU] ->
// [+residual] -> [*mask]) and, with the DGRAD pack and zero padding, autograd's conv data gradient.  A shape its
// tile planner cannot take returns AVC_ERR_UNSUPPORTED; the exact-fp32 path is avc_conv_block_fwd.
#include "common.cuh"

namespace avc {

int validate_conv_desc(const avc_conv_desc* d, const char* who);
int conv_block_tc2_launch(const avc_conv_desc* d, int* status, void* stream);  // conv_tc2.cu
int conv_block_tc2_plan(const avc_conv_desc* d, int num_sms, avc_tc_plan* out);

constexpr int TC_SLAB = 16;  // input channels per weight-pack slab (2 MMA K-steps)

__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
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

// the argument checks of avc_conv_block_tc (all but the status pointer), shared with the plan query
static int check_conv_tc(const avc_conv_desc* d) {
  int rc = validate_conv_desc(d, "avc_conv_block_tc");
  if (rc != AVC_OK) return rc;
  const bool normbwd = (d->flags & AVC_F_NORMBWD) != 0;
  AVC_REQUIRE(d->in && d->w_tc && (d->out || normbwd), AVC_ERR_INVALID, "avc_conv_block_tc: null in/w_tc/out");
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
  return AVC_OK;
}

extern "C" int avc_conv_block_tc(const avc_conv_desc* d, int* status, void* stream) {
  const int rc = check_conv_tc(d);
  if (rc != AVC_OK) return rc;
  AVC_REQUIRE(status, AVC_ERR_INVALID, "avc_conv_block_tc: null status");
  return conv_block_tc2_launch(d, status, stream);
}

extern "C" int avc_conv_block_tc_plan(const avc_conv_desc* d, int num_sms, avc_tc_plan* out) {
  AVC_REQUIRE(out, AVC_ERR_INVALID, "avc_conv_block_tc_plan: null out");
  const int rc = check_conv_tc(d);
  if (rc != AVC_OK) return rc;
  return conv_block_tc2_plan(d, num_sms, out);
}
