/*
 * avc_b200.h -- C ABI of libavc_b200.so: the sm_90a (H100) kernels behind the AdaIN-VC hot path.
 *
 * The reference (jjery2243542/adaptive_voice_conversion) has no FFI: its hot path is the
 * Python class surface model.AE / solver.Solver / inference.Inferencer on top of stock
 * torch.nn modules.  Each entry point below therefore cites the reference lines (relative
 * to the reference repo root) whose torch ops it replaces; the Python side
 * (adaptive_voice_conversion_b200/model.py ...) re-exposes the reference's own class API
 * on top of these calls through ctypes.  See INTEGRATION.md for the binding.
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is a DEVICE pointer owned by the caller
 *    (PyTorch allocates; the library never allocates or frees device memory);
 *  - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing
 *    synchronises, so every call is CUDA-graph capturable;
 *  - every function returns AVC_OK (0) or a negative AVC_ERR_* code and never throws;
 *    avc_last_error() returns a static message for the most recent failure on the calling
 *    thread;
 *  - activations use the "A4" layout: a logical [B][C][T] fp32 tensor is stored as
 *    [B][C/4][T][4] (four channels interleaved per time step, C % 4 == 0), so one
 *    (sample, 4-channel chunk) is a contiguous run of T 16-byte vectors.  The reference's
 *    boundary tensors (x, dec, mu, log_sigma, eps) stay planar [B][C][T]; avc_pack_a4 /
 *    avc_unpack_a4 convert.  `*_bstride` is the distance in floats between samples, which
 *    lets a tensor be a channel sub-range of a wider one (the conv-bank concat).
 */
#ifndef AVC_B200_H_
#define AVC_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AVC_OK 0
#define AVC_ERR_INVALID (-1)     /* bad argument (null pointer, C % 4 != 0, ...) */
#define AVC_ERR_UNSUPPORTED (-2) /* valid request this kernel family does not cover */
#define AVC_ERR_CUDA (-3)        /* a CUDA runtime call failed; see avc_last_error() */

#define AVC_PAD_REFLECT 0
#define AVC_PAD_ZERO 1

#define AVC_RES_NONE 0
#define AVC_RES_SAME 1 /* out += res[t]                                   (model.py:249,368) */
#define AVC_RES_POOL 2 /* out += avg_pool1d(res, 2, ceil_mode=True)[t]    (model.py:248,319) */
#define AVC_RES_UP 3   /* out += nearest-upsample-x2(res)[t]              (model.py:61-63,367) */

/* avc_conv_desc.flags: the tensor core truncates fp32 operands to TF32; to stay unbiased the
 * TF32 path rounds to nearest -- once, where an activation is produced. */
#define AVC_F_ROUND_OUT 1 /* round out (conv block / norm_apply) or dc (norm_bwd) to TF32 */
#define AVC_F_IN_TF32 2   /* `in` is already TF32-exact: avc_conv_block_tc skips its rounding pass */
/* avc_conv_block_tc, plain stride-1 conv used as a data gradient: the epilogue also applies the
 * adjoint of the forward conv's reflect padding (pl = (flags>>8)&255, pr = (flags>>16)&255) and of
 * its residual branch (res / res_mode / res_T read as in avc_fold_desc): Tout = T+pl+pr columns are
 * computed, `out` receives the T folded time steps (what avc_fold_add_fwd produces in a second pass). */
#define AVC_F_FOLD 4
/* with AVC_F_FOLD on the persistent kernel: the epilogue also runs the backward of the UPSTREAM block's InstanceNorm /
 * AdaIN / ReLU on the folded gradient (what avc_norm_bwd does in a second pass).  The descriptor's norm, relu, eps, cond,
 * save_c, stats (inputs) and dc, dcond, dbias (outputs) then describe that upstream block -- same [B][Cout][T] shape as
 * this conv's folded output, no pixel shuffle, Cout <= 128 -- and `out` may be null when nobody else needs the folded
 * gradient itself.  dc is rounded to TF32 when AVC_F_ROUND_OUT is set. */
#define AVC_F_NORMBWD 8
#define AVC_FOLD_FLAGS(pl, pr) (AVC_F_FOLD | ((pl) << 8) | ((pr) << 16))

#define AVC_PACK_FWD 0   /* P[ci][j][co]  = W[co][ci][j]                                   */
#define AVC_PACK_DGRAD 1 /* P[co][j][ci]  = W[co][ci][K-1-j]  (transposed, tap-flipped)     */

/* One fused conv block: reflect-pad -> Conv1d -> [pixel shuffle] -> [InstanceNorm] ->
 * [AdaIN affine] -> [ReLU] -> [+ residual] -> [* mask].
 * Replaces pad_layer (model.py:21-32) + nn.Conv1d + pixel_shuffle_1d (:52-59) +
 * nn.InstanceNorm1d (:296,341) + append_cond (:77-83) + ReLU + the residual adds with
 * F.avg_pool1d / upsample (:248-249, :319-320, :366-369) of one ConvBlock.
 * With pad_mode = ZERO / in_ups = 2 the same kernel computes the data gradient of a conv
 * (see avc_fold_add_fwd).  The struct is also the argument of avc_norm_apply_fwd,
 * avc_norm_bwd. */
typedef struct avc_conv_desc {
  int32_t B, Cin, Cout, K, stride, pad_left, pad_mode, in_ups;
  int32_t Tin;  /* stored input length; logical length is Tin * in_ups (zero insertion) */
  int32_t Tout; /* conv output length */
  const float* in; /* A4 [B][Cin/4][Tin][4] */
  int64_t in_bstride;
  const float* w_packed; /* [Cin][K][w_ld] (avc_pack_conv_weight) */
  int32_t w_ld;
  const float* bias; /* [Cout] or null */
  float* out;        /* A4 [B][Cn/4][Tn][4]; Cn = Cout/(1+shuffle), Tn = Tout*(1+shuffle) */
  int64_t out_bstride;
  int32_t shuffle; /* 1: out[b][c][2t+s] = conv[b][2c+s][t] before the norm (model.py:52-59) */
  int32_t norm;    /* 1: InstanceNorm over Tn per (b, c), biased variance */
  float eps;
  int32_t relu;
  const float* cond; /* AdaIN rows: beta = cond[b*cond_bstride + c], gamma = cond[... + Cn + c]; or null */
  int64_t cond_bstride;
  const float* res; /* A4 [B][Cn/4][res_T][4] or null */
  int64_t res_bstride;
  int32_t res_mode, res_T;
  const float* mask; /* A4 like out; out *= (mask > 0); or null */
  int64_t mask_bstride;
  float* save_c; /* dense A4 [B][Cout/4][Tout][4] raw conv (+bias) kept for backward; or null */
  float* stats;  /* [B][Cn][2] = (mean, rstd) when norm; or null */
  /* ---- backward-only fields (avc_norm_bwd) ---- */
  const float* dy; /* A4 [B][Cn/4][Tn][4], grad w.r.t. the block output */
  int64_t dy_bstride;
  float* dc;    /* dense A4 [B][Cout/4][Tout][4], grad w.r.t. the raw conv output */
  float* dcond; /* [B][2*Cn] (dbeta | dgamma) rows, dcond_bstride apart; or null */
  int64_t dcond_bstride;
  float* dbias; /* [Cout] (+=); or null */
  /* ---- tensor-core path (avc_conv_block_tc) ---- */
  const float* w_tc; /* weights packed by avc_pack_conv_weight_tc; or null */
  int32_t flags;     /* AVC_F_* */
  int32_t out_tstride, out_toff, out_T; /* avc_conv_block_tc: out time index = t*out_tstride + out_toff inside an out
                                          tensor of out_T time steps (0, 0, 0 = dense: index t of Tn) */
  float* dbias_part; /* avc_norm_bwd with dbias: scratch of B x Cout floats for per-block partial sums, reduced into
                        dbias in a fixed order (the same result on every run); null = per-block atomics */
} avc_conv_desc;

/* Fused block forward.  norm=1 needs the whole Tn of a sample inside one CTA tile:
 * supported for Tout <= 128, and Tout <= 256 at K = 1 or 5; otherwise AVC_ERR_UNSUPPORTED -- run it with norm=0,
 * relu=0, res=null, save_c=out-of-conv and follow with avc_norm_apply_fwd.  AVC_F_FOLD, AVC_F_NORMBWD and a non-zero
 * out_tstride / out_toff / out_T (avc_conv_block_tc only) are AVC_ERR_UNSUPPORTED; AVC_F_IN_TF32 is ignored. */
int avc_conv_block_fwd(const avc_conv_desc* d, void* stream);
/* The tile plan avc_conv_block_fwd runs a descriptor with.  Host only: launches nothing, reads no pointer; runs the same
 * argument checks and returns the same code (and avc_last_error() message) as the launch.  A CTA of 256 threads owns TCO
 * output channels x TT output steps; untiled, the tile holds nseg = TT / seg_out samples of seg_out >= Tout columns
 * (staged input segments segp floats apart); tiled (no InstanceNorm), one sample's output is cut into ntt tiles of TT. */
typedef struct avc_simt_plan {
  int32_t TT, TCO, tiled, seg_out, nseg, segp, ntt, grid_x, grid_y;
  int32_t xrow;       /* floats per staged input row (one channel) in shared memory */
  int32_t smem_bytes; /* dynamic shared memory of the launch */
  int32_t instance;   /* index into the fixed table of kernel instances (K, stride, TCO, TT): (K, 1, 128, 128) for
                         K = 1..8, (5, 2, 128, 128), (1, 1, 64, 256), (5, 1, 64, 256), (5, 2, 64, 256); or -1 */
} avc_simt_plan;
int avc_conv_block_fwd_plan(const avc_conv_desc* d, avc_simt_plan* out);
/* The same fused block on the tensor cores (wgmma, TF32 inputs rounded to nearest, fp32
 * accumulation).  Covers stride 1|2, in_ups 1, Cin % 16 == 0; whole samples up to 144 columns, folded
 * (AVC_F_FOLD) ones up to 256 staged rows (longer ones time-tiled without InstanceNorm / fold / pixel shuffle); otherwise
 * AVC_ERR_UNSUPPORTED (use avc_conv_block_fwd).  Reads d->w_tc instead of d->w_packed.
 * status: device int, set non-zero if an internal pipeline barrier timed out. */
int avc_conv_block_tc(const avc_conv_desc* d, int* status, void* stream);
/* The tile plan avc_conv_block_tc runs a descriptor with.  Host only: launches nothing, reads no pointer; runs the same
 * argument checks and returns AVC_ERR_UNSUPPORTED (with the message of avc_last_error()) where the launch would; `out` is
 * filled when the plan exists, also when no kernel instance has its widths (instance = -1, AVC_ERR_UNSUPPORTED).
 * num_sms: SMs of the device the kernel would run on; <= 0 = the current device. */
typedef struct avc_tc_plan {
  int32_t G;          /* samples per tile (stacked along the accumulator columns R rows apart) */
  int32_t N, N_last;  /* accumulator columns of a column chunk, of the last chunk */
  int32_t nchunk;     /* column chunks per tile (> 1: folded sample of more than 144 columns) */
  int32_t R, srows;   /* staged rows per sample, per 4-channel plane of a stage (G * R) */
  int32_t hs;         /* half-slabs (8 input channels) per pipeline stage */
  int32_t nstage;     /* shared-memory stages of the ring */
  int32_t nst;        /* pipeline stages per tile (and column chunk) */
  int32_t ntt, TT;    /* time tiles per sample, output steps per time tile */
  int32_t Ts, P;      /* columns one sample stages for the epilogue; chunk pitch of that tile in 16-byte units */
  int32_t mtiles, ntiles;  /* 128-channel output tiles; tiles in all */
  int32_t patch;      /* 1: the patch warps round / mirror the staged input */
  int32_t stage_bytes, smem_bytes, smem_max;  /* one stage, dynamic shared memory of the launch, its limit */
  int32_t instance;   /* index of the kernel instance for (N, N_last), or -1 */
} avc_tc_plan;
int avc_conv_block_tc_plan(const avc_conv_desc* d, int num_sms, avc_tc_plan* out);
/* nn.Conv1d weight [Cout][Cin][K] -> tensor-core operand blocks (TF32-rounded), AVC_PACK_FWD or
 * AVC_PACK_DGRAD; avc_tc_packed_floats gives the buffer size for a conv with co_total output
 * and ci_total input channels (FWD: Cout, Cin; DGRAD: Cin, Cout). */
int avc_pack_conv_weight_tc(const float* w, float* packed, int Cout, int Cin, int K, int mode, void* stream);
int64_t avc_tc_packed_floats(int co_total, int ci_total, int K);
/* Diagnostics: device buffer of 16 int64 per CTA receiving phase counters of subsequent avc_conv_block_tc launches
 * (null disables): [0] start [1] end clock; wait / work cycle sums of the roles:
 * [2] producer wait-empty, [3] patch wait-full [4] patch work, [5] MMA wait-ready [6] wait-accumulator [7] issue,
 * [8] epilogue wait-accumulator [9] accumulator pass [10] parameters [11] c rows [13] out rows [14] end barrier, [12] tiles done. */
void avc_tc2_set_debug(void* dev_buffer);
/* Every re-pack of a model in one launch: a DEVICE-resident table of items (null destinations
 * are skipped); max_elems = the largest destination element count in the table. */
typedef struct avc_pack_item {
  const float* w;     /* nn.Conv1d weight [Cout][Cin][K] */
  float* simt_fwd;    /* AVC_PACK_FWD   layout for avc_conv_block_fwd, or null */
  float* simt_dgrad;  /* AVC_PACK_DGRAD layout for avc_conv_block_fwd, or null */
  float* tc_fwd;      /* avc_pack_conv_weight_tc FWD layout, or null */
  float* tc_dgrad;    /* avc_pack_conv_weight_tc DGRAD layout, or null */
  float* tc_dgrad_even; /* DGRAD layout restricted to taps 0,2,4,.. (stride-2 transposed conv, even outputs), or null */
  float* tc_dgrad_odd;  /* ... taps 1,3,.. (odd outputs), or null */
  int32_t Cout, Cin, K, reserved;
} avc_pack_item;
int avc_pack_conv_weights_batch(const avc_pack_item* items_dev, int n_items, int64_t max_elems, void* stream);
/* Two-pass epilogue for long sequences: reads d->save_c, applies shuffle/norm/AdaIN/ReLU/
 * residual/mask, writes d->out and d->stats. */
int avc_norm_apply_fwd(const avc_conv_desc* d, void* stream);
/* Backward of the epilogue: dy, save_c, stats, cond -> dc, dcond, dbias.
 * (autograd of InstanceNorm1d + append_cond + ReLU, solver.py:90) */
int avc_norm_bwd(const avc_conv_desc* d, void* stream);

/* Weight gradient of pad_layer+Conv1d: dW[co][ci][j] += sum_{b,t} dc[b][co][t] *
 * xpad[b][ci][t*stride + j]  (canonical nn.Conv1d layout, added to dw's content).  x is the conv
 * input A4, dc the dense grad of the raw conv output.  Exact fp32 on the FMA pipe, any shape with
 * Cin % 4 == Cout % 4 == 0; deterministic: per-slice partial sums go to `scratch`, of
 * avc_conv_wgrad_scratch_floats(d) floats (-1: invalid shape), and are reduced in a fixed order. */
typedef struct avc_wgrad_desc {
  int32_t B, Cin, Cout, K, stride, pad_left, Tin, Tout;
  const float* x;
  int64_t x_bstride;
  const float* dc; /* A4 [B][Cout/4][Tout][4], samples dc_bstride apart */
  int64_t dc_bstride;
  float* dw; /* [Cout][Cin][K] */
} avc_wgrad_desc;
int64_t avc_conv_wgrad_scratch_floats(const avc_wgrad_desc* d);
int avc_conv_wgrad(const avc_wgrad_desc* d, float* scratch, void* stream);
/* The same gradient on the tensor cores (mma.sync TF32, fp32
 * accumulate; deterministic two-stage reduction through `scratch`).  Supported for Tout % 8 == 0 with
 * stride 1 and Tout <= 128 or stride 2 and Tout <= 64: avc_wgrad_tc_scratch_floats returns the scratch size in floats,
 * or -1 when the shape must use avc_conv_wgrad.  status as in avc_conv_block_tc. */
int64_t avc_wgrad_tc_scratch_floats(const avc_wgrad_desc* d);
int avc_conv_wgrad_tc(const avc_wgrad_desc* d, float* scratch, int* status, void* stream);
/* Accumulate-in-place variant (opt-in, non-deterministic summation order): every conv layer owns a
 * ZEROED buffer of avc_wgrad_acc_floats(Cout, Cin, K) floats; avc_conv_wgrad_tc_acc adds the
 * layer's weight gradient into it with vector atomics (no scratch round trip, no per-layer
 * reduction launch; d->dw is ignored) and avc_wgrad_acc_flush folds EVERY layer's buffer into its
 * nn.Conv1d gradient (dw += ...) and zeroes it again, in one launch over a DEVICE item table;
 * max_units = the largest avc_wgrad_acc_floats()/4 of the table. */
typedef struct avc_wgrad_acc_item {
  float* acc;
  float* dw; /* [Cout][Cin][K] accumulated (+=) */
  int32_t Cout, Cin, K, reserved;
} avc_wgrad_acc_item;
int64_t avc_wgrad_acc_floats(int Cout, int Cin, int K);
int avc_conv_wgrad_tc_acc(const avc_wgrad_desc* d, float* acc, int* status, void* stream);
int avc_wgrad_acc_flush(const avc_wgrad_acc_item* items_dev, int n_items, int64_t max_units, void* stream);

/* Adjoint of the reflect padding + residual adjoint.  dxp is the zero-padded "full"
 * transposed conv output (length Tin + pad_left + pad_right) produced by
 * avc_conv_block_fwd with the DGRAD weight pack; this folds the mirrored halo back
 * (adjoint of F.pad(mode='reflect'), model.py:28-30) and adds the gradient arriving
 * through the block's residual branch. */
typedef struct avc_fold_desc {
  int32_t B, C, Tin, pad_left, pad_right;
  const float* dxp; /* dense A4 [B][C/4][Tin+pad_left+pad_right][4] */
  const float* dres; /* A4 grad of the block output the residual fed; or null */
  int64_t dres_bstride;
  int32_t res_mode, res_T; /* adjoint of AVC_RES_*: SAME (res_T=Tin), POOL (res_T=ceil(Tin/2)), UP (res_T=2*Tin) */
  float* dx; /* A4 [B][C/4][Tin][4] */
  int64_t dx_bstride;
} avc_fold_desc;
int avc_fold_add_fwd(const avc_fold_desc* d, void* stream);

/* nn.Conv1d weight [Cout][Cin][K] -> kernel operand layout (AVC_PACK_*). */
int avc_pack_conv_weight(const float* w, float* packed, int Cout, int Cin, int K, int mode, void* stream);

/* planar [B][C][T] <-> A4.  round_tf32 != 0 rounds every packed value to TF32 (cvt.rna: to nearest, ties away from
 * zero), so each stored value has its low 13 bits clear. */
int avc_pack_a4(const float* planar, float* a4, int64_t a4_bstride, int B, int C, int T, int round_tf32, void* stream);
int avc_unpack_a4(const float* a4, int64_t a4_bstride, float* planar, int B, int C, int T, void* stream);

/* sum over (b, t) of an A4 tensor -> out[C] (+=): bias gradient of a conv.  Fixed summation order (no atomics):
 * the same result on every run; T <= 1024. */
int avc_bias_grad(const float* dc, int64_t bstride, float* dbias, int B, int C, int T, void* stream);
/* The same for a tensor whose C channels are `C / group_c` layers side by side (the conv-bank gradient): channel c adds
 * into dbias_tab_dev[c / group_c][c % group_c]; dbias_tab_dev is a DEVICE array of C / group_c pointers.  One launch
 * instead of one per layer. */
int avc_bias_grad_groups(const float* dc, int64_t bstride, float* const* dbias_tab_dev, int group_c, int B, int C, int T, void* stream);

/* AdaptiveAvgPool1d(1) (model.py:231,273) and its adjoint. */
int avc_time_mean_fwd(const float* a4, int64_t bstride, float* out /*[B][C]*/, int B, int C, int T, void* stream);
int avc_time_mean_bwd(const float* dout /*[B][C]*/, float* da4, int64_t bstride, int B, int C, int T, void* stream);

/* Padded batches of different-length utterances (AE.inference with lengths; norm.cu, small_ops.cu).  `lengths` is a DEVICE
 * int32 [B] array; at a layer, sample b holds L_b = ceil(lengths[b] / len_div) * len_mul valid frames (len_div: the
 * product of the strides above the layer, len_mul: of the upsamplings) and every later frame is padding, whatever it
 * holds.  The caller keeps L_b <= T.
 *
 * avc_norm_apply_varlen: avc_norm_apply_fwd with the statistics over each sample's L_b conv outputs (2 L_b normalized
 * frames after a pixel shuffle), corrected two-pass form; writes out's first L_b (2 L_b) frames of each sample and
 * nothing past them.  L_b counts d->save_c's frames (before the shuffle).  AdaIN, ReLU, AVC_F_ROUND_OUT and the SAME /
 * UP / POOL residuals as in avc_norm_apply_fwd; a POOL residual's input holds ceil(lengths[b] / (len_div / 2)) *
 * len_mul valid frames (len_div even) and its odd last frame is divided by 1.  mask must be null. */
int avc_norm_apply_varlen(const avc_conv_desc* d, const int32_t* lengths, int len_div, int len_mul, void* stream);
/* avc_time_mean_fwd over each sample's L_b frames. */
int avc_time_mean_varlen_fwd(const float* a4, int64_t bstride, float* out /*[B][C]*/, int B, int C, int T,
                             const int32_t* lengths, int len_div, int len_mul, void* stream);
/* Frame-weighted pooling over groups of samples (few-shot speaker codes): group g is the rows group_offsets[g] ..
 * group_offsets[g+1] - 1 of the padded batch (DEVICE int32 [G+1], 0 = offsets[0] < offsets[1] < ... < offsets[G] = B,
 * validated by the caller).  With S_m[c] member m's float32 sum over its L_m frames, added as avc_time_mean_varlen_fwd
 * adds it: out[g][c] = (S_first + S_next + ..., in ascending row) * (1.f / (float)N_g), N_g = sum of the members' L_m
 * -- the mean over the union of the members' valid frames.  A one-member group gives avc_time_mean_varlen_fwd's row
 * bit for bit; frames past L_m are never read.  AVC_ERR_INVALID for null pointers, non-positive sizes, C % 4 != 0,
 * len_div or len_mul < 1, G < 1 or G > B.  No allocation, no synchronisation, no atomics: graph-capturable. */
int avc_time_mean_grouped_fwd(const float* a4, int64_t bstride, float* out /*[G][C]*/, int B, int C, int T,
                              const int32_t* lengths, int len_div, int len_mul, const int32_t* group_offsets, int G,
                              void* stream);
/* The two halves of avc_time_mean_grouped_fwd, for groups spread over several batches (speaker banks).
 * avc_time_sum_varlen: sums[b][c] = sample b's float32 sum over its L_b = min(ceil(lengths[b] / len_div) * len_mul, T)
 * frames, formed exactly as avc_time_mean_grouped_fwd forms a member's sum, and counts[b] = L_b (DEVICE int32 [B]).
 * sums[b] * (1.f / L_b) is avc_time_mean_varlen_fwd's row bit for bit; frames past L_b are never read.
 * avc_pooled_group_mean: group g is the rows group_offsets[g] .. group_offsets[g+1] - 1 of a table sums[n_rows][C],
 * counts[n_rows] (DEVICE int64 [G+1] offsets, 0 = offsets[0] < ... < offsets[G] <= n_rows, validated by the caller):
 * out[g][c] = (S_first + S_next + ..., in ascending row) * (1.f / (float)N_g), N_g = the sum of the rows' counts, the
 * first row assigned, not added to zero, with avc_time_mean_grouped_fwd's add step.  So the same members in the same
 * order give avc_time_mean_grouped_fwd's row bit for bit, however they were spread over batches.  The counts are
 * device values the host does not read: a group with N_g outside [1, 2^31) gets NaN, and callers reject such a group
 * before the launch (AE.speaker_codes_from_sums does).
 * Both: AVC_ERR_INVALID for null pointers, non-positive sizes, C % 4 != 0, len_div or len_mul < 1, G outside
 * [1, n_rows], a4, sums, out or the sample stride not 16-byte aligned.  No allocation, no synchronisation, no atomics:
 * graph-capturable. */
int avc_time_sum_varlen(const float* a4, int64_t bstride, float* sums /*[B][C]*/, int32_t* counts /*[B]*/, int B, int C,
                        int T, const int32_t* lengths, int len_div, int len_mul, void* stream);
int avc_pooled_group_mean(const float* sums /*[n_rows][C]*/, const int32_t* counts /*[n_rows]*/, int64_t n_rows, int C,
                          const int64_t* group_offsets /*[G+1]*/, int G, float* out /*[G][C]*/, void* stream);
/* Rewrites, in place, frames of an A4 tensor (or a channel range of one: C channels of T frames, samples bstride floats
 * apart) just past each sample's L_b:
 *   AVC_TAIL_REFLECT   x[L_b + j] = x[L_b - 2 - j] for j < n (and L_b + j < T): the reflect padding F.pad applies to the
 *                      sample alone, for a conv that reads n = pad_right frames past its input (needs L_b > n);
 *   AVC_TAIL_REPLICATE x[L_b] = x[L_b - 1] when L_b is odd (and < T), so that a POOL residual's 0.5 (a + b) at the
 *                      sample's last output gives a, as avg_pool1d(ceil_mode=True) does; n is ignored;
 *   AVC_TAIL_ZERO      x[t] = 0 for L_b <= t < T; n is ignored. */
#define AVC_TAIL_REFLECT 0
#define AVC_TAIL_REPLICATE 1
#define AVC_TAIL_ZERO 2
int avc_varlen_tail(float* a4, int64_t bstride, int B, int C, int T, const int32_t* lengths, int len_div, int len_mul,
                    int mode, int n, void* stream);

/* nn.Linear (+ReLU, + residual): y_act = act(x W^T + b); out = y_act + res.
 * (model.py:252-263 dense blocks, :276 output layer, :342-343 AdaIN affine layers) */
typedef struct avc_linear_desc {
  int32_t B, N, K, relu;
  const float* x; /* [B][K] */
  int64_t x_bstride;
  const float* w;    /* [N][K] (nn.Linear layout) */
  const float* bias; /* [N] or null */
  const float* res;  /* [B][N] dense or null */
  float* y_act;      /* [B][N] dense: activation output kept for the ReLU mask; or null */
  float* out;        /* [B][N] rows out_bstride apart */
  int64_t out_bstride;
  /* backward */
  const float* dy; /* [B][N] rows dy_bstride apart */
  int64_t dy_bstride;
  const float* dx_add; /* [B][K] dense added to dx; or null */
  float* dx;           /* [B][K] dense or null */
  float* dw;           /* [N][K] accumulated (+=) */
  float* db;           /* [N] accumulated (+=) or null */
} avc_linear_desc;
int avc_linear_fwd(const avc_linear_desc* d, void* stream);
int avc_linear_bwd(const avc_linear_desc* d, void* stream); /* mask = (y_act > 0) when relu */

/* The SpeakerEncoder tail as one kernel per direction (model.py:252-263 dense_blocks, :273-276
 * output_layer): n_blocks x { y = relu(W1 h + b1); a = relu(W2 y + b2); h = a + h }, out = Wo h + bo.
 * Built for C = c_out = 128 (AVC_ERR_UNSUPPORTED otherwise: use avc_linear_fwd/bwd per layer).
 * params: DEVICE table of 4*n_blocks+2 pointers [W1_l, b1_l]* [W2_l, b2_l]* Wo bo (nn.Linear layouts).
 * save  : [3*n_blocks+1][B][C] planes h_0..h_n | y_0.. | a_0.. (null at inference).
 * gsave : [2*n_blocks+1][B][C] planes g1_0.. | g2_0.. | dout: the ReLU-masked upstream gradient of
 *         every linear layer = left operand of its weight gradient (avc_linear_batch_dw). */
typedef struct avc_dense_stack_desc {
  int32_t B, C, c_out, n_blocks;
  const float* const* params;
  const float* x; /* [B][C] */
  float* save;
  float* out;        /* [B][c_out] */
  const float* dout; /* [B][c_out] (backward) */
  float* gsave;
  float* dx; /* [B][C] */
} avc_dense_stack_desc;
int avc_dense_stack_fwd(const avc_dense_stack_desc* d, void* stream);
int avc_dense_stack_bwd(const avc_dense_stack_desc* d, void* stream);

/* L same-shape nn.Linear layers per launch (the 12 AdaIN affine layers model.py:342-343; the weight
 * gradients of the dense stack).  Layer l reads x + x_off[l] ([B][K], rows x_bstride apart) and
 * reads/writes the [B][N] tensor at y_off[l] (rows y_bstride apart): `out` in _fwd, the upstream
 * gradient `y` in _dx/_dw.  params / grads: DEVICE tables [W_l, b_l]* / [dW_l, db_l]* (accumulated).
 * _dx: dx[B][K] = sum_l y_l W_l (+ dx_add) through the scratch part[L][B][K]. */
#define AVC_LINEAR_BATCH_MAX 16
typedef struct avc_linear_batch_desc {
  int32_t L, B, N, K;
  const float* const* params;
  float* const* grads;
  const float* x;
  int64_t x_off[AVC_LINEAR_BATCH_MAX];
  int64_t x_bstride;
  const float* y;
  float* out;
  int64_t y_off[AVC_LINEAR_BATCH_MAX];
  int64_t y_bstride;
  float* part;
  const float* dx_add;
  float* dx;
} avc_linear_batch_desc;
int avc_linear_batch_fwd(const avc_linear_batch_desc* d, void* stream);
int avc_linear_batch_dx(const avc_linear_batch_desc* d, void* stream);
int avc_linear_batch_dw(const avc_linear_batch_desc* d, void* stream);

/* VAE reparameterisation (model.py:383-384) fused with the A4->planar conversion of the
 * two heads: z = mu + exp(log_sigma/2)*eps (eps null: z = mu, the inference path :389-390). */
int avc_reparam_fwd(const float* mu4, const float* ls4, const float* eps /*planar or null*/,
                    float* mu /*planar or null*/, float* ls /*planar or null*/, float* z4,
                    int B, int C, int T, void* stream);
/* dmu4 = dz4 + dmu_ext ; dls4 = dz4 * eps * 0.5*exp(ls/2) + dls_ext  (ext planar or null) */
int avc_reparam_bwd(const float* dz4, const float* ls4, const float* eps, const float* dmu_ext,
                    const float* dls_ext, float* dmu4, float* dls4, int B, int C, int T, void* stream);

/* Losses of Solver.ae_step (solver.py:84-88) with their gradients in one pass.
 * hp (device): [0]=lambda_rec [1]=lambda_kl.  sums (device, overwritten by the call):
 * [0]=sum|dec-x| [1]=sum(exp(ls)+mu^2-1-ls).  d* receive d(lambda_rec*L1 + lambda_kl*KL).
 * part (device, AVC_VAE_PARTIALS floats): per-block partial sums, added in a fixed order (the same sums on every run). */
#define AVC_VAE_PARTIALS 2112
int avc_vae_loss(const float* dec, const float* x, int64_t n_rec, const float* mu, const float* ls,
                 int64_t n_lat, const float* hp, float* sums, float* part, float* ddec, float* dmu, float* dls,
                 void* stream);

/* clip_grad_norm_ + Adam(amsgrad, L2 weight decay) over flat fp32 buffers
 * (solver.py:91-93, :75-77).  avc_sqnorm writes sum(g^2) to out[0] (deterministic
 * two-stage reduction; scratch >= 1024 floats).
 * hp (device): [2]=grad_scale (1/world for DP) [3]=lr [4]=beta1 [5]=beta2 [6]=eps
 * [7]=weight_decay [8]=max_norm [9]=amsgrad(0/1).  step (device, float) is incremented by
 * the kernel.  The clip coefficient is min(1, max_norm / (grad_scale*sqrt(sqnorm) + 1e-6)). */
int avc_sqnorm(const float* g, int64_t n, float* scratch, float* out, void* stream);
int avc_adam_step(float* p, const float* g, float* m, float* v, float* vmax, int64_t n,
                  const float* hp, const float* sqnorm, float* step, void* stream);

int avc_fill_zero(void* ptr, int64_t bytes, void* stream);

/* ---- Device-resident training corpus (csrc/corpus.cu, data_utils.DeviceSegments).
 * One training batch cut out of the corpus in the layout CollateFn (data_utils.py:10-22) gives, bit for bit:
 *   x[b][j*n_mels + m][tau] = corpus[(starts[order[first + b]] + tau*frame + j) * n_mels + m],
 *   tau < seg/frame, j < frame, b < batch.
 * A plain copy (no atomics, one thread per output element).  The kernel trusts `starts` and `order`: every crop must lie
 * inside the corpus and first + batch must not exceed the table (the host validates them once, at load).
 * AVC_ERR_INVALID for null pointers, n_mels % 4 != 0, seg % frame != 0 or batch < 1. */
typedef struct avc_gather_desc {
  const float* corpus;   /* [total_frames][n_mels]: every utterance's [T][n_mels] frames, end to end */
  const int64_t* starts; /* [entries] absolute start frame of each index entry (utterance offset + t) */
  const int32_t* order;  /* a permutation of the index entries (the epoch order) */
  float* x;              /* [batch][frame*n_mels][seg/frame] */
  int64_t first;         /* position in `order` of the batch's first entry */
  int32_t batch, seg, frame, n_mels; /* seg = segment_size in frames, frame = frame_size */
} avc_gather_desc;
int avc_segment_gather(const avc_gather_desc* d, void* stream);

/* ---- Held-out evaluation (csrc/eval.cu, evaluate.HeldOut): the per-segment sums of the conversion path's losses.
 * For every sample b < B, in float64 (each term and each sum):
 *   out[first + b][0] = sum_{c < C, t < T} |dec[b][c][t] - x[b][c][t]|
 *   out[first + b][1] = sum_{c < C_lat, t < T_lat} (exp(ls) + mu^2 - 1 - ls)[b][c][t]
 * dec, mu and ls are whole A4 tensors ([B][C/4][T][4], batch stride C*T), x is planar [B][C][T].  One CTA per sample
 * adds in a fixed order without atomics: a sample's two sums have the same bits on every run and in any batch.
 * AVC_ERR_INVALID for null pointers, non-positive sizes, C or C_lat not a multiple of 4, or first < 0. */
typedef struct avc_eval_desc {
  int32_t B, C, T, C_lat, T_lat, reserved;
  const float* dec; /* A4 [B][C/4][T][4] */
  const float* x;   /* planar [B][C][T] */
  const float* mu;  /* A4 [B][C_lat/4][T_lat][4] */
  const float* ls;  /* A4 [B][C_lat/4][T_lat][4] */
  double* out;      /* [n_entries][2] */
  int64_t first;    /* row of sample 0 in out */
} avc_eval_desc;
int avc_eval_losses(const avc_eval_desc* d, void* stream);
/* Per-utterance reconstruction sums of a padded batch (speaker adaptation's held-out check).  For every sample b < B,
 * with L_b = min(max(lengths[b], 0), T) (lengths: DEVICE int32 [B]; callers keep 1 <= lengths[b] <= T):
 *   out[b] = sum_{c < C, t < L_b} |dec[b][c][t] - x[b][c][t]|    in float64 (each term and each sum)
 * dec and x are planar [B][C][T]; frames t >= L_b are never read, whatever they hold.  One CTA per sample adds in a fixed
 * order without atomics (avc_eval_losses' tree): a sample's sum has the same bits on every run and in any batch.
 * AVC_ERR_INVALID, before any launch, for a null descriptor or pointer or non-positive sizes. */
typedef struct avc_rec_varlen_desc {
  int32_t B, C, T, reserved;
  const float* dec;       /* planar [B][C][T] */
  const float* x;         /* planar [B][C][T] */
  const int32_t* lengths; /* DEVICE [B] */
  double* out;            /* [B] */
} avc_rec_varlen_desc;
int avc_rec_loss_varlen(const avc_rec_varlen_desc* d, void* stream);

/* ---- Speaker-code fitting (csrc/fit.cu, fit.CodeFitTrainer).  A batch of B = G * m samples holds G groups (speakers)
 * of m consecutive samples each: sample b belongs to group b / m.
 *
 * avc_group_l1: the grouped L1 loss and its gradient in one pass.  With grec = hp[0] / (float)(m * C * T):
 *   ddec = grec * sign(dec - x), 0 where dec == x (avc_vae_loss's convention), written in dec's A4 layout; with
 *          round_tf32 != 0 each value is rounded to TF32 (cvt.rna) as avc_pack_a4 rounds, so the result is what
 *          avc_vae_loss + avc_pack_a4 give for one group of m = B;
 *   part[b] = sum_{c, t} |dec - x| of sample b in float64, in avc_eval_losses' fixed order;
 *   sums[g] = part[g m] + part[g m + 1] + ... in ascending sample order (float64);
 *   total (or null) = (float)(sums[0] + sums[1] + ...), the batch's L1 sum.
 * dec and ddec are whole A4 tensors [B][C/4][T][4] (batch stride C*T), x is planar [B][C][T].  Two launches, no
 * atomics: every sum has the same bits on every run and whatever the other groups hold.
 * AVC_ERR_INVALID for null pointers (but total), non-positive sizes, C % 4 != 0 or B % m != 0. */
typedef struct avc_group_l1_desc {
  int32_t B, C, T, m;
  int32_t round_tf32, reserved;
  const float* dec; /* A4 [B][C/4][T][4] */
  const float* x;   /* planar [B][C][T] */
  const float* hp;  /* DEVICE: hp[0] = lambda (the trainers' hyper-parameter vector) */
  float* ddec;      /* A4, dec's layout */
  double* part;     /* [B] */
  double* sums;     /* [G] */
  float* total;     /* [1] or null */
} avc_group_l1_desc;
int avc_group_l1(const avc_group_l1_desc* d, void* stream);

/* avc_code_adam: clip_grad_norm_ + Adam(amsgrad, L2 weight decay) of every code on its own.  One CTA per code s < S:
 *   g_s[c]   = sum_{j < m} demb[s m + j][c], added in avc_bias_grad's order at T = 1 (so avc_bias_grad over the same
 *              m rows gives g_s bit for bit); written to grad[s][c];
 *   gnorm[s] = hp[2] * sqrt(sum_c g_s[c]^2) (sum in a fixed order);
 *   steps[s] += 1, then avc_adam_step's clip coefficient min(1, hp[8] / (gnorm + 1e-6)) * hp[2], L2 decay and Adam
 *              (hp layout of avc_adam_step) on codes[s], exp_avg[s], exp_avg_sq[s], max_exp_avg_sq[s];
 *   emb[s m + j] = the updated codes[s] for j < m: the expanded rows the next step's AdaIN affine layers read.
 * A code's bits depend on its own rows only.  No atomics.  AVC_ERR_INVALID for null pointers, S, m or C < 1,
 * C % 4 != 0 or C > AVC_CODE_MAX_C. */
#define AVC_CODE_MAX_C 256
typedef struct avc_code_adam_desc {
  int32_t S, m, C, reserved;
  const float* demb;     /* [S*m][C] dense */
  float* codes;          /* [S][C] */
  float* exp_avg;        /* [S][C] */
  float* exp_avg_sq;     /* [S][C] */
  float* max_exp_avg_sq; /* [S][C] */
  float* steps;          /* [S] */
  float* grad;           /* [S][C] */
  float* gnorm;          /* [S] */
  float* emb;            /* [S*m][C] */
  const float* hp;       /* DEVICE, avc_adam_step's layout */
} avc_code_adam_desc;
int avc_code_adam(const avc_code_adam_desc* d, void* stream);

/* ---- Vocoder DSP (csrc/audio.cu): the reference's librosa STFT / Griffin-Lim path
 * (preprocess/tacotron/utils.py get_spectrograms, melspectrogram2wav), fp32.
 *
 * Every call takes a ragged batch: a DEVICE table of utterances, sorted by both frame_off and sample_off.  Frame f
 * of utterance u lives in row segs[u].frame_off + f of the frame-major buffers; its signal is the n_samples floats
 * at y + sample_off.  An STFT of a signal of n_samples gives 1 + n_samples / hop frames and needs
 * n_samples >= n_fft/2 + 1 (one reflection); an iSTFT of n_frames gives hop * (n_frames - 1) samples.  No call uses
 * atomics: an utterance gets the same bits in any batch.  Supported: n_fft = 2048, even win <= n_fft, 0 < hop <= win
 * (AVC_ERR_UNSUPPORTED otherwise).  The window is the periodic Hann of length win centred in n_fft. */
typedef struct avc_audio_seg {
  int64_t sample_off;          /* first sample of the utterance in y */
  int32_t n_samples;
  int32_t frame_off, n_frames; /* first row and row count in the frame-major buffers */
  int32_t reserved;
} avc_audio_seg;

#define AVC_STFT_MAG 0     /* mag_out = |X| and / or mag_db = clip((20 log10(max(1e-5,|X|)) - ref_db + max_db) / max_db, 1e-8, 1) */
#define AVC_STFT_COMPLEX 1 /* X = the half spectrum */
#define AVC_STFT_PROJECT 2 /* X = mag * A / max(1e-8, |A|), E the half spectrum: one Griffin-Lim projection.
                              momentum 0: A = E.  momentum m > 0 (fast Griffin-Lim): A = E - m/(1+m) * X_prev,
                              then X_prev = E */
#define AVC_STFT_PROJECT_FIRST 3 /* as PROJECT for the first iteration: A = E, X_prev is written but not read */

typedef struct avc_audio_desc {
  int32_t n_fft, hop, win;
  int32_t n_seg;     /* entries of segs */
  int32_t n_frames;  /* rows of the frame-major buffers (sum of segs[].n_frames) */
  int32_t n_samples; /* floats of y the table spans (iSTFT output grid) */
  int32_t mode;      /* avc_stft: AVC_STFT_* */
  int32_t n_iter;    /* avc_griffin_lim */
  float preemph;     /* avc_stft: y'[n] = y[n] - preemph * y[n-1] applied on the fly (0: none) */
  float max_db, ref_db; /* avc_stft MAG with mag_db */
  float momentum;    /* avc_griffin_lim / avc_stft PROJECT: fast Griffin-Lim momentum m in [0, 1) (0: plain) */
  const avc_audio_seg* segs; /* DEVICE table */
  float* y;          /* signal: avc_stft / avc_frame_power input, avc_istft / avc_griffin_lim output, avc_deemphasis in place */
  const float* mag;  /* [n_frames][n_fft/2+1]: target magnitude S of PROJECT / avc_griffin_lim; avc_istft input when X is null */
  float* X;          /* [n_frames][n_fft/2+1] complex (re, im): avc_stft COMPLEX / PROJECT output, avc_istft input,
                        avc_griffin_lim workspace */
  float* frames;     /* [n_frames][win] workspace of avc_istft / avc_griffin_lim: windowed inverse frames */
  float* mag_out;    /* avc_stft MAG: [n_frames][n_fft/2+1] or null */
  float* mag_db;     /* avc_stft MAG: [n_frames][n_fft/2+1] or null */
  float* X_prev;     /* [n_frames][n_fft/2+1] complex: the previous iteration's spectrum E when momentum > 0 (must not
                        overlap X); ignored when momentum is 0 */
} avc_audio_desc;

/* STFT (center, reflect padding) of every utterance: one launch. */
int avc_stft(const avc_audio_desc* d, void* stream);
/* iSTFT: irfft x window per frame into `frames`, then a gather overlap-add divided by the exact window sum-square
 * (where it exceeds FLT_MIN) with n_fft/2 cut from each end, into y.  X null: the spectrum is mag with zero phase.
 * Two launches. */
int avc_istft(const avc_audio_desc* d, void* stream);
/* Griffin-Lim: X = mag (zero phase); n_iter x { X = mag * E / max(1e-8, |E|), E = stft(istft(X)) }; y = istft(X).
 * 3 n_iter + 2 launches (iSTFT frames, overlap-add, projecting STFT per iteration).
 * momentum m > 0: fast Griffin-Lim (Perraudin, Balazs & Sondergaard 2013, librosa's form), c = m / (1 + m):
 * n_iter x { E = stft(istft(X)); A = E - c P (A = E the first time); P = E; X = mag * A / max(1e-8, |A|) }, with P in
 * X_prev; same launches.  AVC_ERR_INVALID before any launch when m is not finite or outside [0, 1), or when m > 0 and
 * X_prev is null or overlaps X.  m = 0 ignores X_prev. */
int avc_griffin_lim(const avc_audio_desc* d, void* stream);
/* avc_griffin_lim with a choice of start.  AVC_GL_START_ZERO is avc_griffin_lim itself.  AVC_GL_START_X starts the first
 * iSTFT from X as the caller left it instead of mag with zero phase.  AVC_GL_START_PGHI first writes avc_pghi's start
 * spectrum (threshold tol) into X and starts from it: one more launch, 3 n_iter + 3.  tol is read only with
 * AVC_GL_START_PGHI.  Every argument of the call (the start, tol, and all of avc_griffin_lim's) is checked before its
 * first launch; AVC_ERR_INVALID otherwise.
 * The start is an argument rather than a descriptor field on purpose: avc_griffin_lim would have to read such a field
 * on every call, past the end of a descriptor built against the previous header, and the descriptor's size is part
 * of the ABI.  (X_prev could be appended because it is read only when the in-struct momentum is non-zero.) */
#define AVC_GL_START_ZERO 0
#define AVC_GL_START_X 1
#define AVC_GL_START_PGHI 2
int avc_griffin_lim_from(const avc_audio_desc* d, int32_t start, float tol, void* stream);
/* Phase Gradient Heap Integration (Prusa, Balazs & Sondergaard 2017; RTPGHI per frame, Prusa & Holighaus 2017): a
 * start spectrum X = mag * e^{i phi} for avc_griffin_lim_from (AVC_GL_START_X, or AVC_GL_START_PGHI in one call).  Per utterance, s_max = its largest
 * magnitude; bins with s = 0 or s < tol * s_max are insignificant (phi = 0).  l = ln max(s, tol * s_max) and, with
 * lambda = 0.25645 win^2 and d_k, d_f centred differences over bins and frames (one-sided at the edges),
 *   phase advance per frame  dt(f,k) = hop ((n_fft / lambda) d_k l + 2 pi k / n_fft),
 *   phase step per bin       dk(f,k) = -(lambda / (n_fft hop)) d_f l - pi.
 * Frame by frame, phi is what the literal heap integration gives: sources are the significant bins of frame f-1,
 * larger magnitude first (then frame f-1 first, then the lower bin), a time step adds (dt(f-1,k) + dt(f,k)) / 2, a
 * bin step to k+-1 adds +-(dk(f,k) + dk(f,k+-1)) / 2, and each run of bins with no source is seeded at its largest
 * bin with phi = 0.  The kernel computes it with block scans (one CTA per utterance, float64 phases, no atomics).
 * parent (nullable, [n_frames][n_fft/2+1]) receives each bin's AVC_PGHI_* choice.  Reads mag, writes X.
 * AVC_ERR_INVALID before any launch when tol is not finite or not in (0, 1), or mag or X is null. */
#define AVC_PGHI_NONE 0  /* insignificant */
#define AVC_PGHI_TIME 1  /* from (f-1, k) */
#define AVC_PGHI_LEFT 2  /* from (f, k-1) */
#define AVC_PGHI_RIGHT 3 /* from (f, k+1) */
#define AVC_PGHI_SEED 4  /* largest bin of a run with no source: phi = 0 */
int avc_pghi(const avc_audio_desc* d, float tol, int8_t* parent, void* stream);
/* power[frame] = mean of y^2 over frames of n_fft samples hop apart, reflect-padded by n_fft/2 (librosa's trim
 * statistic): segs frame_off / n_frames count these frames, 1 + n_samples / hop per utterance.  Any even n_fft. */
int avc_frame_power(const avc_audio_desc* d, float* power, void* stream);
/* y[n] = y[n] + coef * y[n-1] over each utterance in place (scipy.signal.lfilter([1], [1, -coef])): an exact chunked
 * scan, one CTA per utterance.  Reads segs, n_seg, y. */
int avc_deemphasis(const avc_audio_desc* d, float coef, void* stream);

/* Mel projections of the concatenated frames of a ragged batch (rows are independent).
 *   AVC_MEL_TO_MAG: out[rows][n_bins] = A x mat, A = 10^((clip(in,0,1) max_db - max_db + ref_db) / 20),
 *                   in [rows][n_mels], mat [n_mels][n_bins] (the transposed mel-to-linear matrix)
 *   AVC_MAG_TO_MEL: out[rows][n_mels] = clip((20 log10(max(1e-5, in x mat)) - ref_db + max_db) / max_db, 1e-8, 1),
 *                   in [rows][n_bins], mat [n_bins][n_mels] (the transposed filterbank) */
#define AVC_MEL_TO_MAG 0
#define AVC_MAG_TO_MEL 1
typedef struct avc_mel_desc {
  int32_t rows, n_mels, n_bins, dir;
  float max_db, ref_db;
  const float* in;
  const float* mat;
  float* out;
} avc_mel_desc;
int avc_mel_project(const avc_mel_desc* d, void* stream);

/* ---- Corpus preparation (csrc/prep.cu, prepare.py): resampling from raw PCM and per-mel corpus statistics.
 * No allocation, no synchronisation, no atomics: every output element is written by one thread in a fixed order, so
 * an utterance gets the same bits in any batch and in any chunking.
 *
 * avc_resample_poly: per utterance, its channels averaged, then exactly the sum scipy.signal.resample_poly(x, up, down)
 * computes (zero padding), in fp32 with a fixed accumulation order:
 *   y[m] = sum_i x[k_m - i] * taps[r_m][i],  p_m = m*down + half_len, k_m = p_m / up, r_m = p_m % up,
 *   i < (2*half_len - r_m) / up + 1, x[k] = 0 outside [0, n_in);  n_out = ceil(n_in * up / down)
 * taps[r][i] = h[r + i*up] (zero past h's end), h = firwin(2*half_len + 1, 1/max(up, down), ('kaiser', 5.0)) * up,
 * half_len = 10*max(up, down): the polyphase table [up][n_taps], n_taps = ceil((2*half_len + 1) / up).
 * up = down = 1: y = x (conversion and channel mix only; taps may be null).
 * AVC_ERR_INVALID for null pointers, n_seg < 1, n_tiles < 0, up/down < 1, an unknown format, or a tap table whose shape
 * is not the one above; AVC_ERR_UNSUPPORTED for tables of more than AVC_RESAMPLE_MAX_TAPS floats or
 * AVC_RESAMPLE_MAX_PHASE_TAPS taps per phase.  The kernel trusts the utterance table (offsets inside the buffers). */
#define AVC_PCM_S16 0 /* int16, scaled by 1/32768 */
#define AVC_PCM_F32 1 /* float32 as is */
#define AVC_RESAMPLE_TILE 512          /* output samples per CTA */
#define AVC_RESAMPLE_MAX_TAPS 8192     /* up * n_taps */
#define AVC_RESAMPLE_MAX_PHASE_TAPS 96 /* n_taps */
typedef struct avc_resample_seg {
  int64_t in_off;    /* first PCM element of the utterance (element = one channel's sample) */
  int64_t out_off;   /* first output sample */
  int32_t n_in;      /* samples per channel */
  int32_t n_out;     /* ceil(n_in * up / down) */
  int32_t channels;  /* interleaved channels, >= 1 */
  int32_t tile0;     /* first CTA of the utterance: sum of ceil(n_out / AVC_RESAMPLE_TILE) over the ones before it */
} avc_resample_seg;
typedef struct avc_resample_desc {
  int32_t format;    /* AVC_PCM_* */
  int32_t up, down, half_len, n_taps;
  int32_t n_seg;     /* entries of segs */
  int32_t n_tiles;   /* CTAs: tile0 + ceil(n_out / AVC_RESAMPLE_TILE) of the last utterance */
  int32_t reserved;
  const avc_resample_seg* segs; /* DEVICE table, sorted by tile0 */
  const void* pcm;   /* interleaved PCM of every utterance */
  const float* taps; /* [up][n_taps] */
  float* out;        /* mono float32 at the new rate */
} avc_resample_desc;
int avc_resample_poly(const avc_resample_desc* d, void* stream);

/* avc_mel_moments: for every utterance u of a ragged batch of [frames][n_mels] fp32 mels (segs frame_off / n_frames as in
 * avc_audio_seg), in float64, two fixed-order passes over its own frames:
 *   moments[first + u][m] = (mean_u[m], M2_u[m] = sum_t (x[t][m] - mean_u[m])^2).
 * avc_mel_moments_merge: Chan's pairwise update over utterances 0 .. n_utts-1 in order (counts = their frame counts),
 *   mean64[m], std64[m] = sqrt(M2[m] / N) (ddof 0) and their float32 roundings mean[m], std[m].
 * AVC_ERR_INVALID for null pointers, n_seg < 1, n_mels < 1, first < 0 or n_utts < 1. */
typedef struct avc_moments_desc {
  int32_t n_mels, n_seg;
  int64_t first;                /* global index of the batch's first utterance */
  const avc_audio_seg* segs;    /* DEVICE table */
  const float* mels;            /* [frames][n_mels] */
  double* moments;              /* [n_utts][n_mels][2] */
} avc_moments_desc;
int avc_mel_moments(const avc_moments_desc* d, void* stream);
int avc_mel_moments_merge(const double* moments, const int32_t* counts, int32_t n_utts, int32_t n_mels, float* mean,
                          float* std, double* mean64, double* std64, void* stream);

/* ---- Mel-cepstral distortion (csrc/mcd.cu, mcd.py).  No allocation, no synchronisation, no atomics.
 *
 * avc_mel_cepstrum: for every row r of a ragged batch of attr-normalised mel frames in[rows][n_mels], and k < dims:
 *   a_m = clip(in[r][m] * std[m] + mean[m], 0, 1)           (float32, as the vocoder's AVC_MEL_TO_MAG input)
 *   l_m = (a_m max_db - max_db + ref_db) ln(10) / 20         (float64: the natural-log amplitude)
 *   out[r][k] = sum_m l_m dct[m][k]  (float64, ascending m; stored as float32)
 * dct[n_mels][dims] is the orthonormal DCT-II without c_0, built by the caller: dct[m][k] =
 * sqrt(2 / n_mels) cos(pi (k + 1) (2m + 1) / (2 n_mels)).  A row gets the same bits in any batch.
 * AVC_ERR_INVALID for null pointers or non-positive sizes; AVC_ERR_UNSUPPORTED for dims > AVC_CEPSTRUM_MAX_DIMS or
 * n_mels > AVC_CEPSTRUM_MAX_MELS.
 *
 * avc_dtw: for every pair p of a DEVICE table, X = x rows [x_off, x_off + tx), Y = y rows [y_off, y_off + ty) of two
 * [rows][dims] float32 cepstrum buffers, in float64 with every operation rounded on its own (no fused multiply-add):
 *   d(i,j) = sqrt(sum_k (X[i][k] - Y[j][k])^2)   (terms added in ascending k)
 *   S(i,j) = d(i,j) + min(S(i-1,j-1), S(i-1,j), S(i,j-1)) over the predecessors that exist, ties preferring them in
 *            that order;  L(i,j) = L(pred) + 1;  S(0,0) = d(0,0), L(0,0) = 1
 *   out[p] = (S(tx-1, ty-1), L(tx-1, ty-1)).
 * max_short must be at least min(tx, ty) of every pair: the launch sizes its shared memory by it.  A pair that breaks
 * this, or has tx or ty < 1, is not computed: its out row is (NaN, 0).  A pair gets the same bits in any batch.
 * AVC_ERR_INVALID for null pointers or non-positive sizes; AVC_ERR_UNSUPPORTED for dims > AVC_CEPSTRUM_MAX_DIMS or
 * max_short > AVC_DTW_MAX_SHORT.  The kernel trusts the offsets (rows inside the buffers). */
#define AVC_CEPSTRUM_MAX_DIMS 64
#define AVC_CEPSTRUM_MAX_MELS 4096
#define AVC_DTW_MAX_SHORT 4096
typedef struct avc_cepstrum_desc {
  int32_t rows, n_mels, dims, reserved;
  float max_db, ref_db;
  const float* in;     /* [rows][n_mels] */
  const float* mean;   /* [n_mels] */
  const float* std;    /* [n_mels] */
  const double* dct;   /* [n_mels][dims] */
  float* out;          /* [rows][dims] */
} avc_cepstrum_desc;
int avc_mel_cepstrum(const avc_cepstrum_desc* d, void* stream);
typedef struct avc_dtw_pair {
  int64_t x_off, y_off; /* first row of each sequence */
  int32_t tx, ty;       /* rows of each sequence */
} avc_dtw_pair;
typedef struct avc_dtw_desc {
  int32_t n_pairs, dims, max_short, reserved;
  const avc_dtw_pair* pairs; /* DEVICE table [n_pairs] */
  const float* x;            /* [rows][dims] */
  const float* y;            /* [rows][dims] */
  double* out;               /* [n_pairs][2] */
} avc_dtw_desc;
int avc_dtw(const avc_dtw_desc* d, void* stream);

/* ---- Speaker measures (csrc/spk.cu, speaker_eval.py).  No allocation, no synchronisation, no atomics on floats;
 * every float64 operation below is rounded on its own (no fused multiply-add).
 *
 * avc_time_stats_varlen: statistics pooling of a padded batch x[B][C][T] (planar fp32) over each sample's L_b =
 * lengths[b] frames (DEVICE int32 [B]); frames past L_b are never read.  In float64, ascending t:
 *   mean = (sum_t x) / L_b,   var = (sum_t (x - mean)^2) / L_b,   std = sqrt(var)
 *   out[b][c] = (float)mean,  out[b][C + c] = (float)std     (out [B][2C])
 * A sample with L_b < 1 or L_b > T gets NaN.  AVC_ERR_INVALID for null pointers or non-positive sizes.
 *
 * avc_spk_eer: every unordered pair i < j of the n vectors vecs[n][dims] is a trial, a target trial when labels[i] ==
 * labels[j] (DEVICE int32 [n]).  Its score, from the float32 values promoted to float64 and sums in ascending d:
 *   s(a, b) = dot(a, b) / (sqrt(|a|^2) sqrt(|b|^2)),  s = 0 when either norm is 0;  s(a, b) == s(b, a) bit for bit.
 * With FRR(t) = #{target < t} / n_target and FAR(t) = #{non-target >= t} / n_nontarget over the candidate thresholds
 * t in {every score} U {+inf}: threshold = the smallest t minimising max(FRR, FAR); frr, far at it (float64
 * quotients of the exact counts), eer = max(frr, far).  n_target / n_nontarget count the trials; when either is 0,
 * eer, threshold, frr and far are NaN.  The result is written to the DEVICE struct `out` and does not depend on the
 * order of the vectors.  Vectors must be finite.  workspace (DEVICE, 256-byte aligned) holds at least
 * avc_spk_eer_workspace_bytes(n) bytes: AVC_SPK_STATE_BYTES of search state, then rnorm[n] = sqrt(|v_i|^2) (float64,
 * padded to 256 bytes), then the scores of the 64 x 64 tiles (ti <= tj) of the trial matrix: tile (ti, tj) at index
 * tj (tj + 1) / 2 + ti holds key(s(64 ti + r, 64 tj + c)) at [r][c] (uint64), key(s) = bits(s) | 2^63 for s >= +0
 * and ~bits(s) for s < 0 (order-preserving; entries outside i < j < n are unspecified).  A fixed sequence of 40
 * launches, no host synchronisation: the call can be captured in a CUDA graph.  avc_spk_eer_workspace_bytes returns
 * -1 outside 1 <= n <= AVC_SPK_MAX_N.
 * AVC_ERR_INVALID for null pointers, non-positive sizes, a short or misaligned workspace; AVC_ERR_UNSUPPORTED for
 * n > AVC_SPK_MAX_N or dims > AVC_SPK_MAX_DIMS.
 *
 * avc_spk_group_mean: for every query m < m_count (queries[m][dims], q_labels[m], q_exclude[m]): out[m] = the float64
 * mean of s(queries[m], set[v]) over the v < n with labels[v] == q_labels[m] and v != q_exclude[m], the scores added
 * in ascending v, NaN when there is no such v.  All arrays on the DEVICE.  AVC_ERR_INVALID for null pointers or
 * non-positive sizes; AVC_ERR_UNSUPPORTED for n > AVC_SPK_MAX_N or dims > AVC_SPK_MAX_DIMS. */
#define AVC_SPK_MAX_N 32768
#define AVC_SPK_MAX_DIMS 2048
#define AVC_SPK_STATE_BYTES 65536
typedef struct avc_eer_result {
  double eer, threshold, frr, far;
  int64_t n_target, n_nontarget;
} avc_eer_result;
int avc_time_stats_varlen(const float* x, float* out, int B, int C, int T, const int32_t* lengths, void* stream);
int64_t avc_spk_eer_workspace_bytes(int n);
int avc_spk_eer(const float* vecs, const int32_t* labels, int n, int dims, void* workspace, int64_t workspace_bytes,
                avc_eer_result* out, void* stream);
typedef struct avc_spk_group_desc {
  int32_t m, n, dims, reserved;
  const float* queries;     /* [m][dims] */
  const int32_t* q_labels;  /* [m] */
  const int32_t* q_exclude; /* [m]: an index into the set, or any value outside [0, n) for none */
  const float* set;         /* [n][dims] */
  const int32_t* labels;    /* [n] */
  double* out;              /* [m] */
} avc_spk_group_desc;
int avc_spk_group_mean(const avc_spk_group_desc* d, void* stream);
/* avc_spk_group_mean with q_exclude read as [m][n_exclude]: query m skips every v its list names.  Entries outside
 * [0, n) mean "none" and duplicates are allowed; n_exclude = 1 gives avc_spk_group_mean's bits.  AVC_ERR_INVALID also
 * for n_exclude outside [1, 64]. */
int avc_spk_group_mean_multi(const avc_spk_group_desc* d, int n_exclude, void* stream);
/* avc_spk_identify: closed-set identification of m queries against a bank of s codes (speaker banks).  For query i,
 * with s(q, v) scored exactly as avc_spk_group_mean scores it (so s(queries[i], bank[v]) is avc_spk_group_mean of the
 * one-member group {v} bit for bit):
 *   best[i]         = the v maximising s(queries[i], bank[v]), the lowest such v among equal scores;
 *   best_score[i]   = that score;
 *   target_score[i] = s(queries[i], bank[t]) for t = q_target[i] in [0, s); NaN when q_target is NULL or t is outside;
 *   target_rank[i]  = #{v : s(queries[i], bank[v]) > target_score[i]} (0: the target is nearest); -1 with no target.
 * One CTA per query, every bank row scored once.  All arrays on the DEVICE; no allocation, no synchronisation, no
 * atomics: graph-capturable, and a second launch gives the same bits.  AVC_ERR_INVALID for a null descriptor or
 * pointer (q_target may be NULL) or non-positive sizes; AVC_ERR_UNSUPPORTED for s > AVC_SPK_MAX_N or
 * dims > AVC_SPK_MAX_DIMS. */
typedef struct avc_spk_identify_desc {
  int32_t m, s, dims, reserved;
  const float* queries;     /* [m][dims] */
  const float* bank;        /* [s][dims] */
  const int32_t* q_target;  /* [m] bank rows, -1 = none; or NULL */
  int32_t* best;            /* [m] */
  double* best_score;       /* [m] */
  double* target_score;     /* [m] */
  int32_t* target_rank;     /* [m] */
} avc_spk_identify_desc;
int avc_spk_identify(const avc_spk_identify_desc* d, void* stream);

/* ---- Spectral norm of the decoder weights (csrc/spectral_norm.cu): torch.nn.utils.spectral_norm with
 * n_power_iterations=1, eps=1e-12, dim=0, for a DEVICE-resident table of n layers.  W = weight viewed as [h][w]
 * (nn.Conv1d: h = Cout, w = Cin*K; nn.Linear: [out][in]); normalize(x) = x / max(||x||, eps).
 *   AVC_SN_ITERATE (training mode): v = normalize(W^T u), u = normalize(W v) (both written back),
 *                                   sigma = u . (W v), w_bar = W / sigma.
 *   AVC_SN_FIXED   (eval mode):     sigma = u . (W v) with the stored u and v, w_bar = W / sigma.
 * avc_spectral_norm_bwd: grad <- (grad - <grad, w_bar> u v^T) / sigma, in place, with the u, v, sigma and w_bar of
 * the forward (the gradient of weight_orig when grad held the gradient of w_bar).
 * Every reduction runs in a fixed order without atomics: repeated calls give the same bits, and an item's result does
 * not depend on the other items of the launch.  scratch: each item owns avc_spectral_norm_scratch_floats(h, w) floats
 * from scratch + scratch_off; the regions must not overlap.  Every item must have 1 <= h <= max_h and 1 <= w <= max_w
 * (an item outside them is left untouched).  AVC_ERR_INVALID for null pointers, n < 1 or an unknown mode;
 * AVC_ERR_UNSUPPORTED for n > AVC_SN_MAX_ITEMS, max_h > AVC_SN_MAX_H or max_w > AVC_SN_MAX_W. */
#define AVC_SN_ITERATE 0
#define AVC_SN_FIXED 1
#define AVC_SN_MAX_ITEMS 64
#define AVC_SN_MAX_H 4096
#define AVC_SN_MAX_W 4096
typedef struct avc_sn_item {
  const float* weight;  /* weight_orig [h][w] */
  float* w_bar;         /* weight_orig / sigma, same layout */
  float* u;             /* [h] (weight_u) */
  float* v;             /* [w] (weight_v) */
  float* sigma;         /* [1] */
  float* grad;          /* [h][w], avc_spectral_norm_bwd only */
  int64_t scratch_off;  /* floats */
  int32_t h, w;
} avc_sn_item;
int64_t avc_spectral_norm_scratch_floats(int h, int w);
int avc_spectral_norm(const avc_sn_item* items, int n, int max_h, int max_w, int mode, float* scratch, void* stream);
int avc_spectral_norm_bwd(const avc_sn_item* items, int n, int max_h, int max_w, float* scratch, void* stream);

/* wgmma self-test (one CTA): D[128][N] = sum_k A_k * B_k^T over nk K=8 tf32 steps, the
 * operands given as raw shared-memory images; strides[10] = {a_lbo, a_sbo, b_lbo, b_sbo,
 * a_kstep, b_kstep, a_off, b_off (bytes), a_layout, b_layout (must be 0: no swizzle)}; a_mn/b_mn must be 0
 * (tf32 wgmma reads K-major operands only: AVC_ERR_UNSUPPORTED otherwise); the nk steps
 * are issued `reps` times (accumulating) for timing.  status (device int[2]): [0] 0,
 * [1] SM cycles from first MMA issue to completion.  Used by the tests to
 * pin the descriptor conventions the conv kernels rely on. */
int avc_tc_probe_gemm(const float* a_img, int a_bytes, const float* b_img, int b_bytes, const uint32_t* strides,
                      int nk, int N, int a_mn, int b_mn, int reps, float* D, int* status, void* stream);
/* Read-back variant of the self-test: only columns >= `shift` are written (columns below `shift` are left
 * untouched in D). */
void avc_tc_probe_set_ld_shift(int shift);
/* Store-path probe (diagnostic): `ctas` CTAs of 256 threads each write bytes_per_cta (multiple of 4096) to their own
 * region of dst; mode 0 = STG.128, 1 = 2 KB bulk (TMA) stores from shared memory, 2 = half each; cycles[cta] = span. */
int avc_probe_store(float* dst, long long bytes_per_cta, int ctas, int mode, long long* cycles, void* stream);

const char* avc_last_error(void);
/* "sm_90a" build tag, number of kernels launched so far by this process (for bench.py's
 * gpu_launches claim). */
const char* avc_build_info(void);
int64_t avc_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* AVC_B200_H_ */
