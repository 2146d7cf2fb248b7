"""No-GPU checks of the boundary: the C-ABI library loads and exports every symbol include/b200gen.h declares, the
ctypes structs match the C structs, and the reference-facing API surface (constructor validation, scheduler
bookkeeping, error conventions; SURVEY.md §4 / §8b) behaves like the reference's."""
import re
from pathlib import Path

import pytest
import torch

from generativemodels_b200 import _lib

ROOT = Path(__file__).resolve().parents[1]


def test_library_exports_every_declared_symbol():
    header = (ROOT / "include" / "b200gen.h").read_text()
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", header))
    declared -= {"b200_igemm_seg", "b200_igemm_params", "b200_flash_params"}
    lib = _lib.load()
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in b200gen.h but not exported by libb200gen.so"
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    assert lib.b200_version() >= 100


def test_struct_sizes_match():
    lib = _lib.load()
    import ctypes as C
    for which, struct in enumerate((_lib.IgemmParams, _lib.GnStatsParams, _lib.GnApplyParams, _lib.DdimCoef,
                                    _lib.DdpmCoef, _lib.PndmCoef, _lib.IgemmSeg, _lib.FlashParams, _lib.KlCoef)):
        assert lib.b200_abi_sizeof(which) == C.sizeof(struct)


def test_product_fails_loudly_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from generativemodels_b200.networks.nets import DiffusionModelUNet
    m = DiffusionModelUNet(2, 1, 1, num_res_blocks=1, num_channels=(8, 8), attention_levels=(False, False),
                           norm_num_groups=4)
    with pytest.raises(RuntimeError):
        m(torch.randn(1, 1, 8, 8), torch.tensor([1]))
    with pytest.raises(_lib.B200Error):
        _lib.require_device()


def test_unet_constructor_validation():
    """Error cases of tests/test_diffusion_model_unet.py:326-361, 385-398, 457-469 in the reference."""
    from generativemodels_b200.networks.nets import DiffusionModelUNet as U
    with pytest.raises(ValueError):
        U(2, 1, 1, num_res_blocks=1, num_channels=(8, 8, 12), attention_levels=(False, False, False), norm_num_groups=8)
    with pytest.raises(ValueError):
        U(2, 1, 1, num_res_blocks=1, num_channels=(8, 8, 8), attention_levels=(False, False), norm_num_groups=8)
    with pytest.raises(ValueError):
        U(2, 1, 1, num_res_blocks=1, num_channels=(8, 8, 8), attention_levels=(False, False, False),
          num_head_channels=(0, 2), norm_num_groups=8)
    with pytest.raises(ValueError):
        U(2, 1, 1, num_res_blocks=(1, 1), num_channels=(8, 8, 8), attention_levels=(False, False, False),
          norm_num_groups=8)
    with pytest.raises(ValueError):
        U(2, 1, 1, num_res_blocks=1, num_channels=(8, 8), attention_levels=(False, True), norm_num_groups=8,
          with_conditioning=True, cross_attention_dim=None)
    with pytest.raises(ValueError):
        U(2, 1, 1, num_res_blocks=1, num_channels=(8, 8), attention_levels=(False, True), norm_num_groups=8,
          with_conditioning=False, cross_attention_dim=3)
    with pytest.raises(ValueError):
        U(2, 1, 1, num_res_blocks=1, num_channels=(8, 8), attention_levels=(False, True), norm_num_groups=8,
          with_conditioning=True, cross_attention_dim=3, dropout_cattn=3.0)


def test_other_constructor_validation():
    from generativemodels_b200.networks.nets import VQVAE, AutoencoderKL, ControlNet
    with pytest.raises(ValueError):
        AutoencoderKL(2, 1, 1, num_channels=(8, 12), attention_levels=(False, False), num_res_blocks=1, norm_num_groups=8)
    with pytest.raises(ValueError):
        AutoencoderKL(2, 1, 1, num_channels=(8, 8), attention_levels=(False,), num_res_blocks=1, norm_num_groups=8)
    with pytest.raises(ValueError):
        AutoencoderKL(2, 1, 1, num_channels=(8, 8), attention_levels=(False, False), num_res_blocks=(1, 1, 1),
                      norm_num_groups=8)
    with pytest.raises(ValueError):
        VQVAE(2, 1, 1, num_channels=(8, 8), num_res_channels=(8, 8, 8))
    with pytest.raises(ValueError):
        VQVAE(2, 1, 1, num_channels=(8, 8), num_res_channels=8, downsample_parameters=((2, 4, 1),) * 2)
    with pytest.raises(ValueError):
        VQVAE(2, 1, 1, num_channels=(8, 8), num_res_channels=8, upsample_parameters=((2, 4, 1, 1, 0),) * 3)
    with pytest.raises(ValueError):
        ControlNet(2, 1, num_channels=(8, 8), attention_levels=(False, True), norm_num_groups=8,
                   with_conditioning=True, cross_attention_dim=None)


def test_scheduler_bookkeeping():
    """set_timesteps lengths and errors: tests/test_scheduler_{ddpm,ddim,pndm}.py of the reference (PNDM with PRK
    steps: 100 -> 109, test_scheduler_pndm.py:58-62)."""
    from generativemodels_b200.networks.schedulers import DDIMScheduler, DDPMScheduler, NoiseSchedules, PNDMScheduler
    for cls in (DDPMScheduler, DDIMScheduler):
        s = cls(num_train_timesteps=1000)
        s.set_timesteps(100)
        assert s.num_inference_steps == 100 and len(s.timesteps) == 100
        with pytest.raises(ValueError):
            s.set_timesteps(2000)
    p = PNDMScheduler(num_train_timesteps=1000, skip_prk_steps=True)
    p.set_timesteps(100)
    assert len(p.timesteps) == 100
    p = PNDMScheduler(num_train_timesteps=1000, skip_prk_steps=False)
    p.set_timesteps(100)
    assert p.num_inference_steps == 109 and len(p.timesteps) == 109
    with pytest.raises(ValueError):
        DDIMScheduler(prediction_type="nope")
    with pytest.raises(ValueError):
        DDPMScheduler(variance_type="nope")
    with pytest.raises(ValueError):
        DDIMScheduler(clip_sample_min=1, clip_sample_max=-1)
    assert set(NoiseSchedules) >= {"linear_beta", "scaled_linear_beta", "sigmoid_beta", "cosine"}
    d = DDIMScheduler(num_train_timesteps=1000, steps_offset=1)
    d.set_timesteps(10)
    assert d.timesteps[-1] == 1          # steps_offset is added after the ratio (ddim.py:144)


def test_inferer_error_conventions():
    from generativemodels_b200.inferers import DiffusionInferer, LatentDiffusionInferer
    from generativemodels_b200.networks.schedulers import DDIMScheduler
    s = DDIMScheduler(num_train_timesteps=10)
    with pytest.raises(NotImplementedError):
        DiffusionInferer(s).sample(torch.zeros(1, 1, 4, 4), lambda *a, **k: None, s, mode="foo", verbose=False)
    with pytest.raises(ValueError):
        LatentDiffusionInferer(s, ldm_latent_shape=[8, 8], autoencoder_latent_shape=None)


def test_igemm_planner_rules():
    """b200_igemm_plan (host-only, no CUDA call): the planner's column-tile / split-K decisions for a 132-SM part (H100
    SXM), pinned on shapes of the UNets DESIGN.md section 2 quotes.  Column tiles are at most 128 wide; out[3] is reserved
    and always 0."""
    import ctypes as C
    lib = _lib.load()

    def plan(rows, cout, K, workspace=True, n=1):
        p = _lib.IgemmParams()
        p.in_N = p.out_N = n
        p.in_D = p.in_H = p.out_D = p.out_H = 1
        p.in_W = p.out_W = rows // n
        p.stride_d = p.stride_h = p.stride_w = 1
        p.cout, p.out_cols = cout, cout
        p.n_seg = 1
        p.seg[0].nchunks = K // 64
        out = (C.c_int32 * 4)()
        assert lib.b200_igemm_plan(C.byref(p), 132, int(workspace), out) == 0
        return tuple(out)          # (column tile, splits, tiles, pair kernel)

    # machine-filling convolution-sized calls: widest tile, no split
    assert plan(5734400, 256, 6912) == (128, 1, 89600, 0)
    assert plan(131072, 128, 1152) == (128, 1, 1024, 0)
    # under-filled grids narrow the column tile only while the tiles still fit ONE wave
    assert plan(8192, 256, 2304)[:2] == (128, 1)          # 64 M tiles x 2 = 128 <= 132; x 4 would be a second wave
    assert plan(8192, 512, 4608)[:2] == (128, 1)          # 256 tiles already
    assert plan(1024, 256, 2304)[:2] == (64, 1)
    # short reductions (K = 256: the transformer linears) follow the same one-wave rule
    assert plan(8192, 256, 256)[:2] == (128, 1)
    assert plan(4096, 256, 256)[:2] == (64, 1)            # 32 M tiles x 4 = 128 <= 132
    # a reduction is split only into >= 3 ranges of >= 32 chunks (and only with a workspace)
    assert plan(8192, 256, 4608)[1] == 1                  # 128 wide tiles: no room for a second range
    assert plan(1024, 256, 2304)[1] == 1                  # 36 chunks: never
    assert plan(1400, 512, 13824)[:2] == (128, 3)         # brain-LDM level 1: 44 wide tiles x 3 ranges of 72 chunks
    assert plan(1400, 512, 13824, workspace=False)[1] == 1
    assert plan(175, 768, 20736)[1] == 10                 # 12 wide tiles, 324 chunks -> 10 ranges of >= 32
    bad = (C.c_int32 * 4)()
    assert lib.b200_igemm_plan(None, 132, 1, bad) != 0
