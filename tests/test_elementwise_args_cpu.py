"""Argument checks of the elementwise, scheduler and vector-quantiser entry points, without a GPU.

The library loads without a device (_lib.load()) and every check runs before anything touches one, so each call
below passes fake pointer values: a call outside the contract must return B200_EINVAL, and the same call with the one
argument put right must get past every check and fail only at the launch (B200_ECUDA, no device).  That second half
shows each rejection is the check under test and not some other one.  Skipped where a CUDA device is visible: there
the fake pointers would reach a kernel.
"""
import ctypes as C

import pytest
import torch

from generativemodels_b200 import _lib
from generativemodels_b200._lib import B200_ECUDA, B200_EINVAL, DdimCoef, DdpmCoef, KlCoef, PndmCoef

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers must not reach a device")

P = 0x100000                       # a 16-byte aligned fake address
Q = 0x200000
R = 0x300000


def geom(**kw):
    g = dict(N=1, D=4, H=5, W=6, OD=4, OH=5, OW=6, kd=3, kh=3, kw=3, sd=1, sh=1, sw=1, pd=1, ph=1, pw=1)
    g.update(kw)
    return (C.c_int32 * 16)(*g.values())


def pndm(n_hist=2):
    c = PndmCoef()
    c.n_hist = n_hist
    return c


def ddpm(var_mode=0):
    c = DdpmCoef()
    c.var_mode = var_mode
    return c


HIST = (C.c_void_p * 4)(P, Q, R, P)
HIST_NULL = (C.c_void_p * 4)(P, None, R, P)
ST = (C.c_int64 * 5)(64, 16, 16, 16, 1)                      # planar strides: the one-element-per-thread path
INTERP = (1, 1, 1, 1, 8, 1, 1, 4, 1, _lib.INTERPOLATE_LINEAR, 1.0, 1.0, 2.0, None)

# entry point, arguments outside the contract, the same call inside it
CASES = {
    "nchw_to_nhwc_pitch_below_C": ("b200_nchw_to_nhwc", (P, 1, 8, 64, Q, 7, None), (P, 1, 8, 64, Q, 8, None)),
    "nchw_to_nhwc_N_above_65535": ("b200_nchw_to_nhwc", (P, 65536, 8, 64, Q, 8, None), (P, 65535, 8, 64, Q, 8, None)),
    "nhwc_to_nchw_spatial_0": ("b200_nhwc_to_nchw", (P, 0, 1, 8, 0, 8, Q, None), (P, 0, 1, 8, 1, 8, Q, None)),
    "interpolate_y_dtype_f64": ("b200_interpolate", (P, 2, ST, Q, 2, ST, *INTERP), (P, 2, ST, Q, 1, ST, *INTERP)),
    "interpolate_x_dtype_5": ("b200_interpolate", (P, 5, ST, Q, 1, ST, *INTERP), (P, 4, ST, Q, 1, ST, *INTERP)),
    "axpy_a_misaligned": ("b200_axpy_h16", (P + 2, Q, 1.0, R, 64, None), (P, Q, 1.0, R, 64, None)),
    "axpy_b_misaligned": ("b200_axpy_h16", (P, Q + 8, 1.0, R, 64, None), (P, Q, 1.0, R, 64, None)),
    "axpy_y_misaligned": ("b200_axpy_h16", (P, Q, 1.0, R + 4, 64, None), (P, Q, 1.0, R, 64, None)),
    "axpy_n_not_multiple_of_8": ("b200_axpy_h16", (P, Q, 1.0, R, 60, None), (P, Q, 1.0, R, 64, None)),
    "axpy_n_negative": ("b200_axpy_h16", (P, Q, 1.0, R, -8, None), (P, Q, 1.0, R, 8, None)),
    "copy_channels_dst_too_narrow": ("b200_copy_channels", (P, 8, 8, Q, 15, 8, 10, None), (P, 8, 8, Q, 16, 8, 10, None)),
    "copy_channels_src_pitch_below_C": ("b200_copy_channels", (P, 8, 7, Q, 16, 8, 10, None),
                                        (P, 8, 8, Q, 16, 8, 10, None)),
    "geglu_x_misaligned": ("b200_geglu", (P + 2, 4, 8, 16, Q, 8, None), (P, 4, 8, 16, Q, 8, None)),
    "geglu_y_misaligned": ("b200_geglu", (P, 4, 8, 16, Q + 4, 8, None), (P, 4, 8, 16, Q, 8, None)),
    "geglu_H_0": ("b200_geglu", (P, 4, 0, 16, Q, 8, None), (P, 4, 8, 16, Q, 8, None)),
    "geglu_M_0": ("b200_geglu", (P, 0, 8, 16, Q, 8, None), (P, 1, 8, 16, Q, 8, None)),
    "geglu_x_pitch_below_2H": ("b200_geglu", (P, 4, 16, 24, Q, 16, None), (P, 4, 16, 32, Q, 16, None)),
    "tap_gather_out_pitch_not_multiple_of_8": ("b200_tap_gather", (P, 1, 1, geom(), Q, 28, None),
                                               (P, 1, 1, geom(), Q, 32, None)),
    "tap_gather_out_misaligned": ("b200_tap_gather", (P, 1, 1, geom(), Q + 2, 32, None),
                                  (P, 1, 1, geom(), Q, 32, None)),
    "tap_gather_out_pitch_below_taps_C": ("b200_tap_gather", (P, 2, 2, geom(), Q, 48, None),
                                          (P, 2, 2, geom(), Q, 56, None)),
    "tap_gather_negative_padding": ("b200_tap_gather", (P, 1, 1, geom(pw=-1), Q, 32, None),
                                    (P, 1, 1, geom(pw=0), Q, 32, None)),
    "tap_sum_cout_5": ("b200_tap_sum", (P, 135, geom(), 5, None, Q, 8, 0, None), (P, 135, geom(), 4, None, Q, 8, 0, None)),
    "tap_sum_stride_2": ("b200_tap_sum", (P, 27, geom(sh=2), 1, None, Q, 8, 0, None),
                         (P, 27, geom(), 1, None, Q, 8, 0, None)),
    "tap_sum_y_pitch_below_taps_cout": ("b200_tap_sum", (P, 53, geom(), 2, None, Q, 8, 0, None),
                                        (P, 54, geom(), 2, None, Q, 8, 0, None)),
    "tap_sum_out_pitch_below_cout": ("b200_tap_sum", (P, 81, geom(), 3, None, Q, 2, 0, None),
                                     (P, 81, geom(), 3, None, Q, 3, 0, None)),
    "embed_tokens_pitch_below_C": ("b200_embed_tokens", (P, 4, 4, 0, Q, R, 8, P, 7, None, None),
                                   (P, 4, 4, 0, Q, R, 8, P, 8, None, None)),
    "embed_tokens_negative_pos0": ("b200_embed_tokens", (P, 4, 4, -1, Q, R, 8, P, 8, None, None),
                                   (P, 4, 4, 0, Q, R, 8, P, 8, None, None)),
    "cache_append_L_below_T": ("b200_cache_append", (P, Q, 1, 4, 3, 8, R, None), (P, Q, 1, 4, 4, 8, R, None)),
    "cache_append_pos_null": ("b200_cache_append", (P, Q, 1, 4, 8, 8, None, None), (P, Q, 1, 4, 8, 8, R, None)),
    "advance_i32_null": ("b200_advance_i32", (None, 1, None), (P, 1, None)),
    "timestep_embedding_N_dim_2pow31": ("b200_timestep_embedding", (P, 1 << 16, 1 << 15, 10000.0, Q, None),
                                        (P, (1 << 16) - 1, 1 << 15, 10000.0, Q, None)),
    "timestep_embedding_dim_0": ("b200_timestep_embedding", (P, 4, 0, 10000.0, Q, None), (P, 4, 1, 10000.0, Q, None)),
    "small_linear_M_4097": ("b200_small_linear", (P, 4097, 64, Q, None, 8, 0, 0, R, None),
                            (P, 4096, 64, Q, None, 8, 0, 0, R, None)),
    "small_linear_M_0": ("b200_small_linear", (P, 0, 64, Q, None, 8, 0, 0, R, None),
                         (P, 1, 64, Q, None, 8, 0, 0, R, None)),
    "ddim_n_0": ("b200_ddim_step", (P, Q, None, C.byref(DdimCoef()), R, None, 0, None),
                 (P, Q, None, C.byref(DdimCoef()), R, None, 1, None)),
    "ddim_prev_null": ("b200_ddim_step", (P, Q, None, C.byref(DdimCoef()), None, None, 8, None),
                       (P, Q, None, C.byref(DdimCoef()), R, None, 8, None)),
    "ddpm_learned_without_pred_var": ("b200_ddpm_step", (P, Q, R, None, C.byref(ddpm(1)), P, None, 8, None),
                                      (P, Q, R, R, C.byref(ddpm(1)), P, None, 8, None)),
    "ddpm_learned_range_without_pred_var": ("b200_ddpm_step", (P, Q, R, None, C.byref(ddpm(2)), P, None, 8, None),
                                            (P, Q, R, R, C.byref(ddpm(2)), P, None, 8, None)),
    "pndm_n_hist_0": ("b200_pndm_step", (HIST, Q, C.byref(pndm(0)), R, None, 8, None),
                      (HIST, Q, C.byref(pndm(1)), R, None, 8, None)),
    "pndm_n_hist_5": ("b200_pndm_step", (HIST, Q, C.byref(pndm(5)), R, None, 8, None),
                      (HIST, Q, C.byref(pndm(4)), R, None, 8, None)),
    "pndm_null_history": ("b200_pndm_step", (HIST_NULL, Q, C.byref(pndm(2)), R, None, 8, None),
                          (HIST_NULL, Q, C.byref(pndm(1)), R, None, 8, None)),
    "pndm_prev_without_sample": ("b200_pndm_step", (HIST, None, C.byref(pndm(2)), R, None, 8, None),
                                 (HIST, None, C.byref(pndm(2)), None, R, 8, None)),
    "add_noise_N_65536": ("b200_add_noise", (P, Q, R, P, 1.0, 65536, 8, Q, None), (P, Q, R, P, 1.0, 65535, 8, Q, None)),
    "add_noise_per_sample_0": ("b200_add_noise", (P, Q, R, P, 1.0, 2, 0, Q, None), (P, Q, R, P, 1.0, 2, 1, Q, None)),
    "exp_half_clamped_n_0": ("b200_exp_half_clamped", (P, -1.0, 1.0, Q, 0, None), (P, -1.0, 1.0, Q, 1, None)),
    "fma_f32_out_null": ("b200_fma_f32", (P, Q, R, None, 8, None), (P, Q, R, P, 8, None)),
    "scale_f32_div_0": ("b200_scale_f32", (P, 1.0, 0.0, Q, 8, None), (P, 1.0, 1.0, Q, 8, None)),
    "vae_reparam_kld_n_0": ("b200_vae_reparam_kld", (P, Q, R, P, Q, 0, None), (P, Q, R, P, Q, 1, None)),
    "ddpm_kl_N_0": ("b200_ddpm_kl", (P, Q, R, C.byref(KlCoef()), None, P, 0, 8, None),
                    (P, Q, R, C.byref(KlCoef()), None, P, 1, 8, None)),
    "ddpm_kl_sample_sum_null": ("b200_ddpm_kl", (P, Q, R, C.byref(KlCoef()), None, None, 1, 8, None),
                                (P, Q, R, C.byref(KlCoef()), None, P, 1, 8, None)),
    "vq_argmin_x_pitch_below_D": ("b200_vq_argmin_gather", (P, 8, 32, 31, Q, 16, R, None, 0, None, 0, None, None, None),
                                  (P, 8, 32, 32, Q, 16, R, None, 0, None, 0, None, None, None)),
    "vq_argmin_q_pitch_below_D": ("b200_vq_argmin_gather", (P, 8, 3, 3, Q, 16, R, P, 2, None, 0, None, None, None),
                                  (P, 8, 3, 3, Q, 16, R, P, 3, None, 0, None, None, None)),
    "vq_gather_q_pitch_below_D": ("b200_vq_gather", (P, 8, Q, 16, 8, R, 7, None), (P, 8, Q, 16, 8, R, 8, None)),
}


def interp(N=1, C=1, D=1, H=1, W=8, OD=1, OH=1, OW=4, dims=1, mode=_lib.INTERPOLATE_LINEAR, rd=1.0, rh=1.0, rw=2.0,
           xs=ST):
    return (P, 1, xs, Q, 1, ST, N, C, D, H, W, OD, OH, OW, dims, mode, rd, rh, rw, None)


def rows_linear(x_pitch=64, M=2, K=64, g=None, b=None, w=Q, w_pitch=64, O=16, res=None, r_pitch=0, o_pitch=16):
    return (P, x_pitch, M, K, g, b, 1e-5, w, w_pitch, O, None, 0, res, r_pitch, R, o_pitch, 0, None)


def pool(pitch=8, x=P, dims=2, k=3, pad=1, mode=_lib.POOL_AVG, H=8):
    return (x, 1, 1, H, 8, pitch, dims, k, pad, mode, Q, None)


def up2(pitch=8, y=Q, mode=_lib.INTERP_BILINEAR, H=4):
    return (P, 1, H, 4, pitch, mode, y, None)


def bnf(gamma=Q, eps=1e-5, cout=4, per=9):
    return (P, None, gamma, R, P, Q, eps, cout, per, R, P, None)


NEG = (C.c_int64 * 5)(64, 16, 16, -16, 1)
CASES.update({
    "interpolate_W_2pow24_plus_1": ("b200_interpolate", interp(W=(1 << 24) + 1), interp(W=1 << 24)),
    "interpolate_OW_2pow24_plus_1": ("b200_interpolate", interp(OW=(1 << 24) + 1), interp(OW=1 << 24)),
    "interpolate_area_in_out_plus_out_2pow32_plus_1": (
        "b200_interpolate", interp(W=640, OW=6700417, mode=_lib.INTERPOLATE_AREA),
        interp(W=65535, OW=65536, mode=_lib.INTERPOLATE_AREA)),
    "interpolate_bilinear_dims_1": ("b200_interpolate", interp(mode=_lib.INTERPOLATE_BILINEAR),
                                    interp(mode=_lib.INTERPOLATE_BILINEAR, dims=2)),
    "interpolate_ratio_0": ("b200_interpolate", interp(rw=0.0), interp(rw=0.5)),
    "interpolate_ratio_inf": ("b200_interpolate", interp(rw=float("inf")), interp(rw=3.0e38)),
    "interpolate_negative_stride": ("b200_interpolate", interp(xs=NEG), interp()),
    "interpolate_D_2_with_dims_2": ("b200_interpolate", interp(D=2, OD=2, dims=2, mode=_lib.INTERPOLATE_NEAREST),
                                    interp(dims=2, mode=_lib.INTERPOLATE_NEAREST)),
    "rows_linear_M_9": ("b200_rows_linear", rows_linear(M=9), rows_linear(M=8)),
    "rows_linear_M_0": ("b200_rows_linear", rows_linear(M=0), rows_linear(M=1)),
    "rows_linear_w_pitch_below_Kp": ("b200_rows_linear", rows_linear(x_pitch=72, K=65, w_pitch=64),
                                     rows_linear(x_pitch=72, K=65, w_pitch=72)),
    "rows_linear_w_pitch_not_multiple_of_8": ("b200_rows_linear", rows_linear(w_pitch=68), rows_linear(w_pitch=72)),
    "rows_linear_w_misaligned": ("b200_rows_linear", rows_linear(w=Q + 8), rows_linear()),
    "rows_linear_x_pitch_below_K": ("b200_rows_linear", rows_linear(x_pitch=63), rows_linear(x_pitch=64)),
    "rows_linear_o_pitch_below_O": ("b200_rows_linear", rows_linear(o_pitch=15), rows_linear(o_pitch=16)),
    "rows_linear_r_pitch_below_O": ("b200_rows_linear", rows_linear(res=P, r_pitch=15), rows_linear(res=P, r_pitch=16)),
    "rows_linear_gamma_without_beta": ("b200_rows_linear", rows_linear(g=Q), rows_linear(g=Q, b=R)),
    "rows_linear_rows_past_48KB": ("b200_rows_linear", rows_linear(x_pitch=3080, M=8, K=3073, w_pitch=3080),
                                   rows_linear(x_pitch=3080, M=8, K=3072, w_pitch=3080)),
    "pool_s2_pitch_12": ("b200_pool_s2", pool(pitch=12), pool(pitch=16)),
    "pool_s2_x_misaligned": ("b200_pool_s2", pool(x=P + 8), pool()),
    "pool_s2_dims_1": ("b200_pool_s2", pool(dims=1), pool(dims=2)),
    "pool_s2_mode_2": ("b200_pool_s2", pool(mode=2), pool(mode=_lib.POOL_MAX)),
    "pool_s2_padding_above_half_kernel": ("b200_pool_s2", pool(k=3, pad=2), pool(k=4, pad=2)),
    "pool_s2_kernel_0": ("b200_pool_s2", pool(k=0, pad=0), pool(k=1, pad=0)),
    "pool_s2_input_below_kernel": ("b200_pool_s2", pool(k=4, pad=1, H=1), pool(k=4, pad=1, H=2)),
    "upsample2x_pitch_4": ("b200_upsample2x_interp", up2(pitch=4), up2(pitch=8)),
    "upsample2x_y_misaligned": ("b200_upsample2x_interp", up2(y=Q + 2), up2()),
    "upsample2x_mode_2": ("b200_upsample2x_interp", up2(mode=2), up2(mode=_lib.INTERP_BICUBIC)),
    "upsample2x_H_0": ("b200_upsample2x_interp", up2(H=0), up2(H=1)),
    "batchnorm_fold_gamma_null": ("b200_batchnorm_fold", bnf(gamma=None), bnf()),
    "batchnorm_fold_eps_negative": ("b200_batchnorm_fold", bnf(eps=-1e-5), bnf(eps=0.0)),
    "batchnorm_fold_cout_0": ("b200_batchnorm_fold", bnf(cout=0), bnf(cout=1)),
    "batchnorm_fold_per_out_0": ("b200_batchnorm_fold", bnf(per=0), bnf(per=1)),
})


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.mark.parametrize("name", list(CASES))
def test_rejected_before_launch(lib, name):
    entry, bad, good = CASES[name]
    fn = getattr(lib, entry)
    assert fn(*bad) == B200_EINVAL, (name, _lib.last_error())
    rc = fn(*good)
    assert rc == B200_ECUDA, (name, rc, _lib.last_error())


def test_vq_codebook_too_large_for_shared_memory(lib):
    rc = lib.b200_vq_argmin_gather(P, 8, 64, 64, Q, 1 << 14, R, None, 0, None, 0, None, None, None)
    assert rc == _lib.B200_ENOTSUP
