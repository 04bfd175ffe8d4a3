"""ctypes binding of libavc_b200.so (the C ABI declared in include/avc_b200.h).

There is no CPU fallback: if the shared library is missing and cannot be built, importing
a symbol raises.  ``AVC_LIB`` can point at an explicit .so.
"""
from __future__ import annotations

import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
# engine.py: fused speaker dense stack / batched AdaIN affine layers (csrc/dense_fused.cu);
# AVC_FUSED_DENSE=0 = one launch per nn.Linear
DEFAULT_FUSED_DENSE = True
# engine.py: AVC_WGRAD_ACC=1 accumulates conv weight gradients in place with vector atomics + ONE flush launch per
# backward pass (csrc/wgrad_tc.cu, ATOMIC); off by default: the atomics' summation order varies from run to run, and
# Adam turns that rounding noise into different trajectories.  Default = per-slice partials + deterministic reduction
DEFAULT_WGRAD_ACC = False
# engine.py: reflect-padding / residual adjoint inside the data-gradient conv's epilogue (AVC_F_FOLD, 30
# avc_fold_add_fwd launches fewer per step)
DEFAULT_FOLD_FUSED = True
# engine.py: the data-gradient conv of a block also runs the UPSTREAM block's InstanceNorm / AdaIN / ReLU backward in
# its epilogue (AVC_F_NORMBWD, persistent kernel): 27 avc_norm_bwd launches and their dy/dc round trips fewer per step.
# Correct (tests/test_gpu_normbwd_fused.py) but it lengthens the conv kernel's epilogue while the stand-alone
# avc_norm_bwd runs at full occupancy -> opt-in
DEFAULT_NORM_BWD_FUSED = False
LIB_PATH = os.environ.get("AVC_LIB", os.path.join(_PKG, "libavc_b200.so"))

PAD_REFLECT, PAD_ZERO = 0, 1
RES_NONE, RES_SAME, RES_POOL, RES_UP = 0, 1, 2, 3
PACK_FWD, PACK_DGRAD = 0, 1
F_ROUND_OUT, F_IN_TF32, F_FOLD, F_NORMBWD = 1, 2, 4, 8
TAIL_REFLECT, TAIL_REPLICATE, TAIL_ZERO = 0, 1, 2
OK, ERR_INVALID, ERR_UNSUPPORTED, ERR_CUDA = 0, -1, -2, -3

_fp = C.c_void_p  # device pointers travel as integers


class ConvDesc(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("Cin", C.c_int32), ("Cout", C.c_int32), ("K", C.c_int32),
        ("stride", C.c_int32), ("pad_left", C.c_int32), ("pad_mode", C.c_int32), ("in_ups", C.c_int32),
        ("Tin", C.c_int32), ("Tout", C.c_int32),
        ("in_", _fp), ("in_bstride", C.c_int64),
        ("w_packed", _fp), ("w_ld", C.c_int32),
        ("bias", _fp),
        ("out", _fp), ("out_bstride", C.c_int64),
        ("shuffle", C.c_int32), ("norm", C.c_int32), ("eps", C.c_float), ("relu", C.c_int32),
        ("cond", _fp), ("cond_bstride", C.c_int64),
        ("res", _fp), ("res_bstride", C.c_int64), ("res_mode", C.c_int32), ("res_T", C.c_int32),
        ("mask", _fp), ("mask_bstride", C.c_int64),
        ("save_c", _fp), ("stats", _fp),
        ("dy", _fp), ("dy_bstride", C.c_int64),
        ("dc", _fp), ("dcond", _fp), ("dcond_bstride", C.c_int64), ("dbias", _fp),
        ("w_tc", _fp), ("flags", C.c_int32), ("out_tstride", C.c_int32), ("out_toff", C.c_int32), ("out_T", C.c_int32),
        ("dbias_part", _fp),
    ]


class TcPlan(C.Structure):
    """avc_tc_plan: the tile plan of avc_conv_block_tc for one descriptor (avc_conv_block_tc_plan)."""
    _fields_ = [(n, C.c_int32) for n in (
        "G", "N", "N_last", "nchunk", "R", "srows", "hs", "nstage", "nst", "ntt", "TT", "Ts", "P", "mtiles", "ntiles", "patch",
        "stage_bytes", "smem_bytes", "smem_max", "instance")]


class SimtPlan(C.Structure):
    """avc_simt_plan: the tile plan of avc_conv_block_fwd for one descriptor (avc_conv_block_fwd_plan)."""
    _fields_ = [(n, C.c_int32) for n in (
        "TT", "TCO", "tiled", "seg_out", "nseg", "segp", "ntt", "grid_x", "grid_y", "xrow", "smem_bytes", "instance")]


# avc_simt_plan.instance -> (K, stride, TCO, TT) of the conv_block_fwd_kernel instance
SIMT_INSTANCES = [(k, 1, 128, 128) for k in range(1, 9)] + [(5, 2, 128, 128), (1, 1, 64, 256), (5, 1, 64, 256), (5, 2, 64, 256)]


class WgradDesc(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("Cin", C.c_int32), ("Cout", C.c_int32), ("K", C.c_int32),
        ("stride", C.c_int32), ("pad_left", C.c_int32), ("Tin", C.c_int32), ("Tout", C.c_int32),
        ("x", _fp), ("x_bstride", C.c_int64),
        ("dc", _fp), ("dc_bstride", C.c_int64),
        ("dw", _fp),
    ]


class FoldDesc(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("C", C.c_int32), ("Tin", C.c_int32), ("pad_left", C.c_int32), ("pad_right", C.c_int32),
        ("dxp", _fp), ("dres", _fp), ("dres_bstride", C.c_int64),
        ("res_mode", C.c_int32), ("res_T", C.c_int32),
        ("dx", _fp), ("dx_bstride", C.c_int64),
    ]


class PackItem(C.Structure):
    _fields_ = [("w", _fp), ("simt_fwd", _fp), ("simt_dgrad", _fp), ("tc_fwd", _fp), ("tc_dgrad", _fp),
                ("tc_dgrad_even", _fp), ("tc_dgrad_odd", _fp),
                ("Cout", C.c_int32), ("Cin", C.c_int32), ("K", C.c_int32), ("reserved", C.c_int32)]


class LinearDesc(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("relu", C.c_int32),
        ("x", _fp), ("x_bstride", C.c_int64),
        ("w", _fp), ("bias", _fp), ("res", _fp), ("y_act", _fp),
        ("out", _fp), ("out_bstride", C.c_int64),
        ("dy", _fp), ("dy_bstride", C.c_int64),
        ("dx_add", _fp), ("dx", _fp), ("dw", _fp), ("db", _fp),
    ]


class WgradAccItem(C.Structure):
    _fields_ = [("acc", _fp), ("dw", _fp), ("Cout", C.c_int32), ("Cin", C.c_int32), ("K", C.c_int32), ("reserved", C.c_int32)]


class DenseStackDesc(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("C", C.c_int32), ("c_out", C.c_int32), ("n_blocks", C.c_int32),
        ("params", _fp), ("x", _fp), ("save", _fp), ("out", _fp), ("dout", _fp), ("gsave", _fp), ("dx", _fp),
    ]


LINEAR_BATCH_MAX = 16
VAE_PARTIALS = 2112   # AVC_VAE_PARTIALS


class LinearBatchDesc(C.Structure):
    _fields_ = [
        ("L", C.c_int32), ("B", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("params", _fp), ("grads", _fp),
        ("x", _fp), ("x_off", C.c_int64 * LINEAR_BATCH_MAX), ("x_bstride", C.c_int64),
        ("y", _fp), ("out", _fp), ("y_off", C.c_int64 * LINEAR_BATCH_MAX), ("y_bstride", C.c_int64),
        ("part", _fp), ("dx_add", _fp), ("dx", _fp),
    ]


STFT_MAG, STFT_COMPLEX, STFT_PROJECT, STFT_PROJECT_FIRST = 0, 1, 2, 3
MEL_TO_MAG, MAG_TO_MEL = 0, 1
GL_START_ZERO, GL_START_X, GL_START_PGHI = 0, 1, 2
PGHI_NONE, PGHI_TIME, PGHI_LEFT, PGHI_RIGHT, PGHI_SEED = 0, 1, 2, 3, 4


class AudioSeg(C.Structure):
    _fields_ = [("sample_off", C.c_int64), ("n_samples", C.c_int32), ("frame_off", C.c_int32), ("n_frames", C.c_int32),
                ("reserved", C.c_int32)]


class AudioDesc(C.Structure):
    _fields_ = [
        ("n_fft", C.c_int32), ("hop", C.c_int32), ("win", C.c_int32), ("n_seg", C.c_int32),
        ("n_frames", C.c_int32), ("n_samples", C.c_int32), ("mode", C.c_int32), ("n_iter", C.c_int32),
        ("preemph", C.c_float), ("max_db", C.c_float), ("ref_db", C.c_float), ("momentum", C.c_float),
        ("segs", _fp), ("y", _fp), ("mag", _fp), ("X", _fp), ("frames", _fp), ("mag_out", _fp), ("mag_db", _fp),
        ("X_prev", _fp),
    ]


class MelDesc(C.Structure):
    _fields_ = [("rows", C.c_int32), ("n_mels", C.c_int32), ("n_bins", C.c_int32), ("dir", C.c_int32),
                ("max_db", C.c_float), ("ref_db", C.c_float), ("in_", _fp), ("mat", _fp), ("out", _fp)]


class GatherDesc(C.Structure):
    _fields_ = [("corpus", _fp), ("starts", _fp), ("order", _fp), ("x", _fp), ("first", C.c_int64),
                ("batch", C.c_int32), ("seg", C.c_int32), ("frame", C.c_int32), ("n_mels", C.c_int32)]


class EvalDesc(C.Structure):
    _fields_ = [("B", C.c_int32), ("C", C.c_int32), ("T", C.c_int32), ("C_lat", C.c_int32), ("T_lat", C.c_int32),
                ("reserved", C.c_int32), ("dec", _fp), ("x", _fp), ("mu", _fp), ("ls", _fp), ("out", _fp), ("first", C.c_int64)]


class RecVarlenDesc(C.Structure):
    _fields_ = [("B", C.c_int32), ("C", C.c_int32), ("T", C.c_int32), ("reserved", C.c_int32), ("dec", _fp), ("x", _fp),
                ("lengths", _fp), ("out", _fp)]


class GroupL1Desc(C.Structure):
    _fields_ = [("B", C.c_int32), ("C", C.c_int32), ("T", C.c_int32), ("m", C.c_int32), ("round_tf32", C.c_int32),
                ("reserved", C.c_int32), ("dec", _fp), ("x", _fp), ("hp", _fp), ("ddec", _fp), ("part", _fp), ("sums", _fp),
                ("total", _fp)]


CODE_MAX_C = 256


class CodeAdamDesc(C.Structure):
    _fields_ = [("S", C.c_int32), ("m", C.c_int32), ("C", C.c_int32), ("reserved", C.c_int32), ("demb", _fp),
                ("codes", _fp), ("exp_avg", _fp), ("exp_avg_sq", _fp), ("max_exp_avg_sq", _fp), ("steps", _fp),
                ("grad", _fp), ("gnorm", _fp), ("emb", _fp), ("hp", _fp)]


PCM_S16, PCM_F32 = 0, 1
RESAMPLE_TILE, RESAMPLE_MAX_TAPS, RESAMPLE_MAX_PHASE_TAPS = 512, 8192, 96


class ResampleSeg(C.Structure):
    _fields_ = [("in_off", C.c_int64), ("out_off", C.c_int64), ("n_in", C.c_int32), ("n_out", C.c_int32),
                ("channels", C.c_int32), ("tile0", C.c_int32)]


class ResampleDesc(C.Structure):
    _fields_ = [("format", C.c_int32), ("up", C.c_int32), ("down", C.c_int32), ("half_len", C.c_int32),
                ("n_taps", C.c_int32), ("n_seg", C.c_int32), ("n_tiles", C.c_int32), ("reserved", C.c_int32),
                ("segs", _fp), ("pcm", _fp), ("taps", _fp), ("out", _fp)]


class MomentsDesc(C.Structure):
    _fields_ = [("n_mels", C.c_int32), ("n_seg", C.c_int32), ("first", C.c_int64), ("segs", _fp), ("mels", _fp),
                ("moments", _fp)]


CEPSTRUM_MAX_DIMS, CEPSTRUM_MAX_MELS, DTW_MAX_SHORT = 64, 4096, 4096


class CepstrumDesc(C.Structure):
    _fields_ = [("rows", C.c_int32), ("n_mels", C.c_int32), ("dims", C.c_int32), ("reserved", C.c_int32),
                ("max_db", C.c_float), ("ref_db", C.c_float),
                ("in_", _fp), ("mean", _fp), ("std", _fp), ("dct", _fp), ("out", _fp)]


class DtwPair(C.Structure):
    _fields_ = [("x_off", C.c_int64), ("y_off", C.c_int64), ("tx", C.c_int32), ("ty", C.c_int32)]


class DtwDesc(C.Structure):
    _fields_ = [("n_pairs", C.c_int32), ("dims", C.c_int32), ("max_short", C.c_int32), ("reserved", C.c_int32),
                ("pairs", _fp), ("x", _fp), ("y", _fp), ("out", _fp)]


SPK_MAX_N, SPK_MAX_DIMS, SPK_STATE_BYTES = 32768, 2048, 65536


class EerResult(C.Structure):
    _fields_ = [("eer", C.c_double), ("threshold", C.c_double), ("frr", C.c_double), ("far", C.c_double),
                ("n_target", C.c_int64), ("n_nontarget", C.c_int64)]


class SpkGroupDesc(C.Structure):
    _fields_ = [("m", C.c_int32), ("n", C.c_int32), ("dims", C.c_int32), ("reserved", C.c_int32),
                ("queries", _fp), ("q_labels", _fp), ("q_exclude", _fp), ("set", _fp), ("labels", _fp), ("out", _fp)]


class SpkIdentifyDesc(C.Structure):
    _fields_ = [("m", C.c_int32), ("s", C.c_int32), ("dims", C.c_int32), ("reserved", C.c_int32),
                ("queries", _fp), ("bank", _fp), ("q_target", _fp), ("best", _fp), ("best_score", _fp),
                ("target_score", _fp), ("target_rank", _fp)]


SN_ITERATE, SN_FIXED = 0, 1
SN_MAX_ITEMS, SN_MAX_H, SN_MAX_W = 64, 4096, 4096


class SnItem(C.Structure):
    _fields_ = [("weight", _fp), ("w_bar", _fp), ("u", _fp), ("v", _fp), ("sigma", _fp), ("grad", _fp),
                ("scratch_off", C.c_int64), ("h", C.c_int32), ("w", C.c_int32)]


# name -> (restype, argtypes); the single source of truth for tests/test_cabi_symbols.py
_i, _i64, _p = C.c_int, C.c_int64, C.c_void_p
PROTOTYPES = {
    "avc_conv_block_fwd": (_i, [C.POINTER(ConvDesc), _p]),
    "avc_conv_block_fwd_plan": (_i, [C.POINTER(ConvDesc), C.POINTER(SimtPlan)]),
    "avc_conv_block_tc": (_i, [C.POINTER(ConvDesc), _p, _p]),
    "avc_conv_block_tc_plan": (_i, [C.POINTER(ConvDesc), _i, C.POINTER(TcPlan)]),
    "avc_pack_conv_weight_tc": (_i, [_p, _p, _i, _i, _i, _i, _p]),
    "avc_tc_packed_floats": (_i64, [_i, _i, _i]),
    "avc_tc2_set_debug": (None, [_p]),
    "avc_pack_conv_weights_batch": (_i, [_p, _i, _i64, _p]),
    "avc_norm_apply_fwd": (_i, [C.POINTER(ConvDesc), _p]),
    "avc_norm_bwd": (_i, [C.POINTER(ConvDesc), _p]),
    "avc_conv_wgrad_scratch_floats": (_i64, [C.POINTER(WgradDesc)]),
    "avc_conv_wgrad": (_i, [C.POINTER(WgradDesc), _p, _p]),
    "avc_wgrad_tc_scratch_floats": (_i64, [C.POINTER(WgradDesc)]),
    "avc_conv_wgrad_tc": (_i, [C.POINTER(WgradDesc), _p, _p, _p]),
    "avc_wgrad_acc_floats": (_i64, [_i, _i, _i]),
    "avc_conv_wgrad_tc_acc": (_i, [C.POINTER(WgradDesc), _p, _p, _p]),
    "avc_wgrad_acc_flush": (_i, [_p, _i, _i64, _p]),
    "avc_fold_add_fwd": (_i, [C.POINTER(FoldDesc), _p]),
    "avc_pack_conv_weight": (_i, [_p, _p, _i, _i, _i, _i, _p]),
    "avc_pack_a4": (_i, [_p, _p, _i64, _i, _i, _i, _i, _p]),
    "avc_unpack_a4": (_i, [_p, _i64, _p, _i, _i, _i, _p]),
    "avc_bias_grad": (_i, [_p, _i64, _p, _i, _i, _i, _p]),
    "avc_bias_grad_groups": (_i, [_p, _i64, _p, _i, _i, _i, _i, _p]),
    "avc_time_mean_fwd": (_i, [_p, _i64, _p, _i, _i, _i, _p]),
    "avc_time_mean_bwd": (_i, [_p, _p, _i64, _i, _i, _i, _p]),
    "avc_norm_apply_varlen": (_i, [C.POINTER(ConvDesc), _p, _i, _i, _p]),
    "avc_time_mean_varlen_fwd": (_i, [_p, _i64, _p, _i, _i, _i, _p, _i, _i, _p]),
    "avc_time_mean_grouped_fwd": (_i, [_p, _i64, _p, _i, _i, _i, _p, _i, _i, _p, _i, _p]),
    "avc_time_sum_varlen": (_i, [_p, _i64, _p, _p, _i, _i, _i, _p, _i, _i, _p]),
    "avc_pooled_group_mean": (_i, [_p, _p, _i64, _i, _p, _i, _p, _p]),
    "avc_varlen_tail": (_i, [_p, _i64, _i, _i, _i, _p, _i, _i, _i, _i, _p]),
    "avc_linear_fwd": (_i, [C.POINTER(LinearDesc), _p]),
    "avc_linear_bwd": (_i, [C.POINTER(LinearDesc), _p]),
    "avc_dense_stack_fwd": (_i, [C.POINTER(DenseStackDesc), _p]),
    "avc_dense_stack_bwd": (_i, [C.POINTER(DenseStackDesc), _p]),
    "avc_linear_batch_fwd": (_i, [C.POINTER(LinearBatchDesc), _p]),
    "avc_linear_batch_dx": (_i, [C.POINTER(LinearBatchDesc), _p]),
    "avc_linear_batch_dw": (_i, [C.POINTER(LinearBatchDesc), _p]),
    "avc_reparam_fwd": (_i, [_p, _p, _p, _p, _p, _p, _i, _i, _i, _p]),
    "avc_reparam_bwd": (_i, [_p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _p]),
    "avc_vae_loss": (_i, [_p, _p, _i64, _p, _p, _i64, _p, _p, _p, _p, _p, _p, _p]),
    "avc_sqnorm": (_i, [_p, _i64, _p, _p, _p]),
    "avc_adam_step": (_i, [_p, _p, _p, _p, _p, _i64, _p, _p, _p, _p]),
    "avc_fill_zero": (_i, [_p, _i64, _p]),
    "avc_segment_gather": (_i, [C.POINTER(GatherDesc), _p]),
    "avc_eval_losses": (_i, [C.POINTER(EvalDesc), _p]),
    "avc_rec_loss_varlen": (_i, [C.POINTER(RecVarlenDesc), _p]),
    "avc_group_l1": (_i, [C.POINTER(GroupL1Desc), _p]),
    "avc_code_adam": (_i, [C.POINTER(CodeAdamDesc), _p]),
    "avc_stft": (_i, [C.POINTER(AudioDesc), _p]),
    "avc_istft": (_i, [C.POINTER(AudioDesc), _p]),
    "avc_griffin_lim": (_i, [C.POINTER(AudioDesc), _p]),
    "avc_griffin_lim_from": (_i, [C.POINTER(AudioDesc), C.c_int32, C.c_float, _p]),
    "avc_pghi": (_i, [C.POINTER(AudioDesc), C.c_float, _p, _p]),
    "avc_frame_power": (_i, [C.POINTER(AudioDesc), _p, _p]),
    "avc_deemphasis": (_i, [C.POINTER(AudioDesc), C.c_float, _p]),
    "avc_mel_project": (_i, [C.POINTER(MelDesc), _p]),
    "avc_resample_poly": (_i, [C.POINTER(ResampleDesc), _p]),
    "avc_mel_moments": (_i, [C.POINTER(MomentsDesc), _p]),
    "avc_mel_moments_merge": (_i, [_p, _p, C.c_int32, C.c_int32, _p, _p, _p, _p, _p]),
    "avc_mel_cepstrum": (_i, [C.POINTER(CepstrumDesc), _p]),
    "avc_dtw": (_i, [C.POINTER(DtwDesc), _p]),
    "avc_time_stats_varlen": (_i, [_p, _p, _i, _i, _i, _p, _p]),
    "avc_spk_eer_workspace_bytes": (_i64, [_i]),
    "avc_spk_eer": (_i, [_p, _p, _i, _i, _p, _i64, _p, _p]),
    "avc_spk_group_mean": (_i, [C.POINTER(SpkGroupDesc), _p]),
    "avc_spk_group_mean_multi": (_i, [C.POINTER(SpkGroupDesc), _i, _p]),
    "avc_spk_identify": (_i, [C.POINTER(SpkIdentifyDesc), _p]),
    "avc_spectral_norm_scratch_floats": (_i64, [_i, _i]),
    "avc_spectral_norm": (_i, [_p, _i, _i, _i, _i, _p, _p]),
    "avc_spectral_norm_bwd": (_i, [_p, _i, _i, _i, _p, _p]),
    "avc_tc_probe_gemm": (_i, [_p, _i, _p, _i, C.POINTER(C.c_uint32), _i, _i, _i, _i, _i, _p, _p, _p]),
    "avc_tc_probe_set_ld_shift": (None, [_i]),
    "avc_probe_store": (_i, [_p, C.c_longlong, _i, _i, _p, _p]),
    "avc_last_error": (C.c_char_p, []),
    "avc_build_info": (C.c_char_p, []),
    "avc_launch_count": (_i64, []),
}

_lib = None


class AvcError(RuntimeError):
    pass


def load(build_if_missing: bool = True):
    """Load (building first if necessary) the shared library; raises if impossible."""
    global _lib
    if _lib is not None:
        return _lib
    if "AVC_LIB" not in os.environ:
        # stamp-checked: a no-op when libavc_b200.so matches the sources, a rebuild when a
        # .cu/.cuh/.h changed, an error when it is stale and nvcc is unavailable
        from . import build as _build
        if build_if_missing or os.path.exists(LIB_PATH):
            _build.build(allow_build=build_if_missing)
    if not os.path.exists(LIB_PATH):
        raise AvcError(f"{LIB_PATH} is missing (run `python -m adaptive_voice_conversion_b200.build`); there is no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().avc_last_error().decode()


def check(rc: int, what: str = ""):
    if rc != OK:
        raise AvcError(f"{what}: rc={rc}: {last_error()}")


def launch_count() -> int:
    return int(load().avc_launch_count())
