"""ctypes binding of libb200gen.so (the C-ABI declared in include/b200gen.h).

The library is the product: if it is missing, cannot be loaded or the device is not an sm_90 (Hopper) GPU, every op
raises — there is no CPU or PyTorch fallback anywhere in this package.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
# 16-bit storage type ("h16") of activations and packed weights: IEEE fp16 by default, bfloat16 with
# B200_ACT_DTYPE=bf16 (the same sources built with -DB200_H16_IS_BF16; for models whose activations exceed fp16's
# range — fp16 stores saturate at +-65504).  Read once at import; the loaded library must agree (b200_act_dtype()).
ACT_DTYPE = os.environ.get("B200_ACT_DTYPE", "fp16").lower()
if ACT_DTYPE in ("float16", "half", "f16"):
    ACT_DTYPE = "fp16"
if ACT_DTYPE in ("bfloat16",):
    ACT_DTYPE = "bf16"
if ACT_DTYPE not in ("fp16", "bf16"):
    raise ValueError(f"B200_ACT_DTYPE must be fp16 or bf16, got {ACT_DTYPE!r}")
LIB_PATH = _HERE / "lib" / ("libb200gen.so" if ACT_DTYPE == "fp16" else "libb200gen_bf16.so")

B200_OK, B200_EINVAL, B200_ENOTSUP, B200_ECUDA, B200_ENODEV = 0, -1, -2, -3, -4
DT_H16, DT_F32 = 0, 1
DT_F64, DT_FP16, DT_BF16 = 2, 3, 4      # inputs only (b200_interpolate's x, b200_ssim, b200_mmd, b200_fid_moments)
SSIM_MAX_K, SSIM_MAX_SCALES = 128, 32
FID_MAX_F = 32768
H16_FP16, H16_BF16 = 0, 1
ACT_NONE, ACT_RELU, ACT_SILU, ACT_LEAKYRELU, ACT_GELU, ACT_TANH, ACT_SIGMOID = 0, 1, 2, 3, 4, 5, 6
ACT_GEGLU = 7        # b200_igemm act1 only: [32 a | 32 gate] column groups -> a * gelu(gate), half as many output channels
ACT_LEAKYRELU02 = 8  # nn.LeakyReLU(0.2)
INTERP_BILINEAR, INTERP_BICUBIC = 0, 1
POOL_AVG, POOL_MAX = 0, 1
(INTERPOLATE_NEAREST, INTERPOLATE_LINEAR, INTERPOLATE_BILINEAR, INTERPOLATE_BICUBIC, INTERPOLATE_TRILINEAR,
 INTERPOLATE_AREA) = 0, 1, 2, 3, 4, 5
PRED_EPSILON, PRED_SAMPLE, PRED_V = 0, 1, 2
IGEMM_MAX_SEG = 128


class B200Error(RuntimeError):
    pass


class IgemmSeg(C.Structure):
    _fields_ = [("src", C.c_int8), ("dw", C.c_int8), ("dh", C.c_int8), ("dd", C.c_int8),
                ("c0", C.c_uint16), ("nchunks", C.c_uint16)]


class IgemmParams(C.Structure):
    _fields_ = [
        ("a_ptr", C.c_void_p * 2), ("a_C", C.c_int32 * 2), ("a_pitch", C.c_int32 * 2),
        ("in_N", C.c_int32), ("in_D", C.c_int32), ("in_H", C.c_int32), ("in_W", C.c_int32),
        ("stride_d", C.c_int32), ("stride_h", C.c_int32), ("stride_w", C.c_int32),
        ("w_ptr", C.c_void_p), ("w_rows", C.c_int32), ("w_pitch", C.c_int32), ("w_K", C.c_int32),
        ("w_bstride", C.c_int64), ("w_batched", C.c_int32), ("n_seg", C.c_int32),
        ("seg", IgemmSeg * IGEMM_MAX_SEG),
        ("out_ptr", C.c_void_p), ("out_dtype", C.c_int32),
        ("out_N", C.c_int32), ("out_D", C.c_int32), ("out_H", C.c_int32), ("out_W", C.c_int32),
        ("cout", C.c_int32), ("out_cols", C.c_int32),
        ("out_sN", C.c_int64), ("out_sD", C.c_int64), ("out_sH", C.c_int64), ("out_sW", C.c_int64),
        ("bias", C.c_void_p), ("rowvec", C.c_void_p), ("rowvec_bstride", C.c_int64), ("row_bias", C.c_void_p),
        ("act1", C.c_int32), ("scale", C.c_float),
        ("res_ptr", C.c_void_p), ("res_dtype", C.c_int32),
        ("res_sN", C.c_int64), ("res_sD", C.c_int64), ("res_sH", C.c_int64), ("res_sW", C.c_int64),
        ("act2", C.c_int32), ("stat_ptr", C.c_void_p), ("impl", C.c_int32),
        ("gn_partial", C.c_void_p), ("gn_slots", C.c_int32), ("gn_slot0", C.c_int32),
        ("split_ws", C.c_void_p), ("split_ws_bytes", C.c_int64),
        ("a_broadcast", C.c_int32), ("gn_group", C.c_int32),
    ]


class GnStatsParams(C.Structure):
    _fields_ = [("x_ptr", C.c_void_p * 2), ("x_C", C.c_int32 * 2), ("x_pitch", C.c_int32 * 2),
                ("N", C.c_int32), ("spatial", C.c_int64), ("groups", C.c_int32), ("eps", C.c_float),
                ("gamma", C.c_void_p), ("beta", C.c_void_p), ("partial", C.c_void_p), ("affine", C.c_void_p)]


class GnApplyParams(C.Structure):
    _fields_ = [("x_ptr", C.c_void_p * 2), ("x_C", C.c_int32 * 2), ("x_pitch", C.c_int32 * 2),
                ("N", C.c_int32), ("spatial", C.c_int64), ("affine", C.c_void_p), ("act", C.c_int32),
                ("y_ptr", C.c_void_p), ("y_pitch", C.c_int32)]


class FlashParams(C.Structure):
    _fields_ = [("q", C.c_void_p), ("k", C.c_void_p), ("vt", C.c_void_p), ("out", C.c_void_p), ("res", C.c_void_p),
                ("B", C.c_int32), ("T", C.c_int32), ("S", C.c_int32), ("heads", C.c_int32), ("dh", C.c_int32),
                ("q_pitch", C.c_int32), ("k_pitch", C.c_int32), ("vt_pitch", C.c_int32), ("out_pitch", C.c_int32),
                ("res_pitch", C.c_int32), ("scale", C.c_float),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64)]


class DdimCoef(C.Structure):
    _fields_ = [("sqrt_alpha_prod_t", C.c_float), ("sqrt_beta_prod_t", C.c_float),
                ("sqrt_alpha_prod_prev", C.c_float), ("dir_coef", C.c_float), ("sigma", C.c_float),
                ("clip_min", C.c_float), ("clip_max", C.c_float),
                ("prediction_type", C.c_int32), ("clip", C.c_int32)]


class DdpmCoef(C.Structure):
    _fields_ = [("sqrt_alpha_prod_t", C.c_float), ("sqrt_beta_prod_t", C.c_float),
                ("coef_x0", C.c_float), ("coef_xt", C.c_float), ("sigma", C.c_float),
                ("clip_min", C.c_float), ("clip_max", C.c_float), ("min_log", C.c_float), ("max_log", C.c_float),
                ("var_mode", C.c_int32), ("prediction_type", C.c_int32), ("clip", C.c_int32)]


class KlCoef(C.Structure):
    _fields_ = [("sqrt_alpha_prod_t", C.c_float), ("sqrt_beta_prod_t", C.c_float), ("coef_x0", C.c_float),
                ("coef_xt", C.c_float), ("log_pred_var", C.c_float), ("log_post_var", C.c_float),
                ("bin_width", C.c_float), ("prediction_type", C.c_int32), ("clip", C.c_int32), ("is_t0", C.c_int32)]


class PndmCoef(C.Structure):
    _fields_ = [("w", C.c_float * 4), ("n_hist", C.c_int32), ("sample_coeff", C.c_float), ("eps_coeff", C.c_float),
                ("v_alpha", C.c_float), ("v_beta", C.c_float), ("prediction_type", C.c_int32)]


class RepackBlock(C.Structure):
    _fields_ = [("col0", C.c_int32), ("cin0", C.c_int32), ("cs", C.c_int32), ("ntaps", C.c_int32),
                ("tap", C.c_int16 * 8)]


class SsimParams(C.Structure):
    _fields_ = [("x", C.c_void_p), ("y", C.c_void_p), ("x_dtype", C.c_int32), ("y_dtype", C.c_int32),
                ("x_strides", C.c_int64 * 5), ("y_strides", C.c_int64 * 5),
                ("N", C.c_int32), ("C", C.c_int32), ("D", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
                ("kd", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
                ("taps_d", C.c_float * SSIM_MAX_K), ("taps_h", C.c_float * SSIM_MAX_K),
                ("taps_w", C.c_float * SSIM_MAX_K), ("scale", C.c_float), ("c1", C.c_float), ("c2", C.c_float),
                ("ssim_map", C.c_void_p), ("cs_map", C.c_void_p), ("partials", C.c_void_p)]


class SsimCombineParams(C.Structure):
    _fields_ = [("partials", C.c_void_p * SSIM_MAX_SCALES), ("slots", C.c_int32 * SSIM_MAX_SCALES),
                ("count", C.c_int64 * SSIM_MAX_SCALES), ("weights", C.c_float * SSIM_MAX_SCALES),
                ("N", C.c_int32), ("n_scales", C.c_int32),
                ("ssim_mean", C.c_void_p), ("cs_mean", C.c_void_p), ("ms_ssim", C.c_void_p)]


class FidMomentsParams(C.Structure):
    _fields_ = [("x", C.c_void_p), ("x_dtype", C.c_int32), ("F", C.c_int32), ("n", C.c_int64),
                ("x_strides", C.c_int64 * 2), ("mu", C.c_void_p), ("sigma", C.c_void_p)]


class FrechetParams(C.Structure):
    _fields_ = [("mu_x", C.c_void_p), ("sigma_x", C.c_void_p), ("mu_y", C.c_void_p), ("sigma_y", C.c_void_p),
                ("F", C.c_int32), ("reserved", C.c_int32), ("workspace", C.c_void_p), ("out", C.c_void_p),
                ("eigvals", C.c_void_p), ("rank", C.c_void_p)]


REPACK_BLOCKS, REPACK_TAP_IN, REPACK_TAP_OUT = 0, 1, 2

_P, _I32, _I64, _F = C.c_void_p, C.c_int32, C.c_int64, C.c_float

# name -> argtypes (restype is int unless listed in _RESTYPES); mirrors include/b200gen.h exactly
SIGNATURES = {
    "b200_last_error_string": [],
    "b200_version": [],
    "b200_act_dtype": [],
    "b200_device_check": [],
    "b200_sm_count": [],
    "b200_abi_sizeof": [C.c_int],
    "b200_igemm": [C.POINTER(IgemmParams), _P],
    "b200_groupnorm_workspace_bytes": [_I32, _I64, _I32],
    "b200_groupnorm_stats": [C.POINTER(GnStatsParams), _P],
    "b200_groupnorm_from_partials_ex": [C.POINTER(GnStatsParams), _P, _P, _P, _P],
    "b200_spade_apply": [C.POINTER(GnApplyParams), _P, _I32, _P, _P],
    "b200_groupnorm_apply": [C.POINTER(GnApplyParams), _P],
    "b200_groupnorm_fused": [C.POINTER(GnStatsParams), C.POINTER(GnApplyParams), _P],
    "b200_layernorm": [_P, _I64, _I32, _I32, _P, _P, _F, _P, _I32, _P],
    "b200_nchw_to_nhwc": [_P, _I32, _I32, _I64, _P, _I32, _P],
    "b200_nhwc_to_nchw": [_P, _I32, _I32, _I32, _I64, _I32, _P, _P],
    "b200_upsample2x_interp": [_P, _I32, _I32, _I32, _I32, _I32, _P, _P],
    "b200_pool_s2": [_P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P],
    "b200_interpolate": [_P, _I32, _P, _P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _F, _F,
                         _F, _P],
    "b200_axpy_h16": [_P, _P, _F, _P, _I64, _P],
    "b200_copy_channels": [_P, _I32, _I32, _P, _I32, _I32, _I64, _P],
    "b200_geglu": [_P, _I64, _I32, _I32, _P, _I32, _P],
    "b200_softmax_rows_partials": [_P, _I64, _I32, _I64, _P, _I32, _P, _I64, _P],
    "b200_attention_small_ex": [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, C.c_float, _I32,
                                _I32, _I32, _P, _P],
    "b200_embed_tokens": [_P, _I64, _I32, _I32, _P, _P, _I32, _P, _I32, _P, _P],
    "b200_rows_linear": [_P, _I32, _I32, _I32, _P, _P, C.c_float, _P, _I32, _I32, _P, _I32, _P, _I32, _P, _I32, _I32, _P],
    "b200_attention_decode": [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, C.c_float, _I32, _P, _P],
    "b200_cache_append": [_P, _P, _I32, _I32, _I32, _I32, _P, _P],
    "b200_advance_i32": [_P, _I32, _P],
    "b200_tap_gather": [_P, _I32, _I32, _P, _P, _I32, _P],
    "b200_tap_sum": [_P, _I32, _P, _I32, _P, _P, _I32, _I32, _P],
    "b200_attention_flash": [C.POINTER(FlashParams), _P],
    "b200_attention_flash_workspace_bytes": [C.POINTER(FlashParams)],
    "b200_igemm_split_workspace_bytes": [C.POINTER(IgemmParams)],
    "b200_igemm_plan": [C.POINTER(IgemmParams), _I32, _I32, _P],
    "b200_attention_small": [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _F, _P],
    "b200_timestep_embedding": [_P, _I32, _I32, _F, _P, _P],
    "b200_small_linear": [_P, _I32, _I32, _P, _P, _I32, _I32, _I32, _P, _P],
    "b200_ddim_step": [_P, _P, _P, C.POINTER(DdimCoef), _P, _P, _I64, _P],
    "b200_ddpm_step": [_P, _P, _P, _P, C.POINTER(DdpmCoef), _P, _P, _I64, _P],
    "b200_ddpm_kl": [_P, _P, _P, C.POINTER(KlCoef), _P, _P, _I32, _I64, _P],
    "b200_pndm_step": [C.POINTER(_P), _P, C.POINTER(PndmCoef), _P, _P, _I64, _P],
    "b200_exp_half_clamped": [_P, _F, _F, _P, _I64, _P],
    "b200_vae_reparam_kld": [_P, _P, _P, _P, _P, _I64, _P],
    "b200_scale_f32": [_P, _F, _F, _P, _I64, _P],
    "b200_fma_f32": [_P, _P, _P, _P, _I64, _P],
    "b200_add_noise": [_P, _P, _P, _P, _F, _I32, _I64, _P, _P],
    "b200_vq_argmin_gather": [_P, _I64, _I32, _I32, _P, _I32, _P, _P, _I32, _P, _I32, _P, _P, _P],
    "b200_vq_gather": [_P, _I64, _P, _I32, _I32, _P, _I32, _P],
    "b200_repack_weight": [_P, _I32, _I32, _I32, _I32, _I32, C.POINTER(RepackBlock), _I32, _P, _I32, _I32, _P],
    "b200_batchnorm_fold": [_P, _P, _P, _P, _P, _P, _F, _I32, _I64, _P, _P, _P],
}
# the sample-quality metrics' entry points; mirrors include/b200gen_metrics.h exactly
METRIC_SIGNATURES = {
    "b200_ssim_workspace_bytes": [C.POINTER(SsimParams)],
    "b200_ssim": [C.POINTER(SsimParams), _P],
    "b200_ssim_combine": [C.POINTER(SsimCombineParams), _P],
    "b200_mmd_workspace_bytes": [_P],
    "b200_mmd": [_P, _I32, _P, _P, _I32, _P, _P, _P, _P, _P],
}
# FID's entry points; mirrors include/b200gen_fid.h exactly
FID_SIGNATURES = {
    "b200_fid_moments": [C.POINTER(FidMomentsParams), _P],
    "b200_frechet_workspace_bytes": [_I32],
    "b200_frechet": [C.POINTER(FrechetParams), _P],
}
# the perceptual distance's entry points; mirrors include/b200gen_perceptual.h exactly
PERCEPTUAL_SIGNATURES = {
    "b200_perceptual_prep": [_P, _I32, _P, _P, _I32, _P, _I32, _I32, _I32, _I32, _P, _I32, _P, _P, _P],
    "b200_perceptual_distance": [_P, _P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P],
    "b200_perceptual_mean": [_P, _I32, _P, _P, _P, _P],
}
_RESTYPES = {"b200_last_error_string": C.c_char_p, "b200_groupnorm_workspace_bytes": C.c_int64,
             "b200_attention_flash_workspace_bytes": C.c_int64, "b200_igemm_split_workspace_bytes": C.c_int64,
             "b200_ssim_workspace_bytes": C.c_int64, "b200_mmd_workspace_bytes": C.c_int64,
             "b200_frechet_workspace_bytes": C.c_int64}

_lib = None
_device_ok = False


def load():
    """Load the shared library (no GPU needed) and bind every symbol the header declares."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise B200Error(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(generativemodels_b200/csrc/build.sh). There is no fallback path.")
    lib = C.CDLL(str(LIB_PATH))
    for name, argtypes in {**SIGNATURES, **METRIC_SIGNATURES, **FID_SIGNATURES, **PERCEPTUAL_SIGNATURES}.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export it
        fn.argtypes = argtypes
        fn.restype = _RESTYPES.get(name, C.c_int)
    for which, struct in enumerate((IgemmParams, GnStatsParams, GnApplyParams, DdimCoef, DdpmCoef, PndmCoef, IgemmSeg,
                                    FlashParams, KlCoef, RepackBlock, SsimParams, SsimCombineParams,
                                    FidMomentsParams, FrechetParams)):
        c_size = lib.b200_abi_sizeof(which)
        if c_size != C.sizeof(struct):
            raise B200Error(f"ABI mismatch: {struct.__name__} is {C.sizeof(struct)} bytes in Python but {c_size} in "
                            f"{LIB_PATH.name}; rebuild the library (generativemodels_b200/csrc/build.sh)")
    want = H16_FP16 if ACT_DTYPE == "fp16" else H16_BF16
    if lib.b200_act_dtype() != want:
        raise B200Error(f"{LIB_PATH.name} stores 16-bit data as format {lib.b200_act_dtype()} but B200_ACT_DTYPE="
                        f"{ACT_DTYPE} was requested; rebuild the library (generativemodels_b200/csrc/build.sh)")
    _lib = lib
    return lib


def last_error() -> str:
    return load().b200_last_error_string().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise B200Error(f"{what} failed with code {rc}: {last_error()}")


def require_device():
    """Fail loudly unless the current CUDA device is sm_90 (H100)."""
    global _device_ok
    lib = load()
    if not _device_ok:
        import torch

        if not torch.cuda.is_available():
            raise B200Error("generativemodels_b200 needs a CUDA device (sm_90a); none is visible and there is no CPU path")
        check(lib.b200_device_check(), "b200_device_check")
        _device_ok = True
    return lib
