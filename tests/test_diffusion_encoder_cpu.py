"""DiffusionModelEncoder without a GPU: constructor, attributes, exceptions and state_dict layout against the unmodified
reference (where a checkout is readable) and against the committed fixture (tests/golden/g_diffusion_encoder.pt,
everywhere); the reference's quirks; the import path under the ``generative`` alias; the forward-only and CUDA-only
refusals; and the module's host code end to end on the CPU stand-in of the library."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from generativemodels_b200.networks.nets.diffusion_model_unet import (Downsample, DiffusionModelEncoder,
                                                                       ResnetBlock)
from oracle import ref_import
from tests import cpu_backend
from tests.golden import configs as G
from tests.golden import load

ROOT = Path(__file__).resolve().parents[1]
GOLD = load("g_diffusion_encoder")
CASES = [k for k in GOLD if k != "ddim_encode"]
TUTORIAL = GOLD["tutorial"]["kwargs"]

BAD_KWARGS = [
    dict(with_conditioning=True),                                       # no cross_attention_dim
    dict(cross_attention_dim=8),                                        # without with_conditioning
    dict(num_channels=(32, 48, 64)),                                    # 48 % 32
    dict(attention_levels=(False, True)),                               # length mismatch
    dict(num_head_channels=(64, 64)),                                   # length mismatch
    dict(num_res_blocks=1),                                             # an int is indexed, not expanded
]


def _kw(**over):
    kw = dict(TUTORIAL)
    kw.update(over)
    return kw


def _reference_modules():
    return {k: v for k, v in sys.modules.items() if k.split(".")[0] in ("generative", "monai")}


@pytest.fixture(scope="module")
def ref():
    """The reference's module.  Importing it puts the reference checkout (which has a ``tests`` package of its own)
    at the front of ``sys.path``; both that and ``sys.modules`` are restored afterwards, so that later test files (and
    the processes they spawn, which inherit ``sys.path``) still resolve ``tests`` and ``generative`` here."""
    if not ref_import.available():
        pytest.skip("reference checkout not present")
    saved_path, saved_modules = list(sys.path), _reference_modules()
    ref_import.import_reference()
    import generative.networks.nets.diffusion_model_unet as R
    yield R
    sys.path[:] = saved_path
    for k in _reference_modules():
        del sys.modules[k]
    sys.modules.update(saved_modules)


# ---- constructor ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("over", BAD_KWARGS, ids=["cond_no_dim", "dim_no_cond", "groups", "attn_len", "heads_len",
                                                  "int_res_blocks"])
def test_constructor_errors(over):
    with pytest.raises(TypeError if "num_res_blocks" in over else ValueError):
        DiffusionModelEncoder(**_kw(**over))


@pytest.mark.parametrize("over", BAD_KWARGS, ids=["cond_no_dim", "dim_no_cond", "groups", "attn_len", "heads_len",
                                                  "int_res_blocks"])
def test_constructor_errors_match_reference(ref, over):
    with pytest.raises(Exception) as want:
        ref.DiffusionModelEncoder(**_kw(**over))
    with pytest.raises(Exception) as got:
        DiffusionModelEncoder(**_kw(**over))
    assert type(got.value) is type(want.value)
    if isinstance(want.value, ValueError):
        assert str(got.value) == str(want.value)


ATTRS = ("in_channels", "block_out_channels", "out_channels", "num_res_blocks", "attention_levels",
         "num_head_channels", "with_conditioning", "num_class_embeds")


def test_attributes():
    m = DiffusionModelEncoder(**TUTORIAL)
    assert m.num_head_channels == (64, 64, 64) and m.block_out_channels == (32, 64, 64)
    assert m.num_res_blocks == (1, 1, 1) and m.num_class_embeds is None and m.with_conditioning is False
    assert m.out[0].in_features == 4096 and m.out[0].out_features == 512 and m.out[3].out_features == 2
    assert isinstance(m.out[1], torch.nn.ReLU) and m.out[2].p == 0.1


@pytest.mark.parametrize("name", CASES)
def test_attributes_match_reference(ref, name):
    kw = GOLD[name]["kwargs"]
    a, b = DiffusionModelEncoder(**kw), ref.DiffusionModelEncoder(**kw)
    for attr in ATTRS:
        assert getattr(a, attr) == getattr(b, attr), attr
    assert set(dict(a.named_modules())) <= set(dict(b.named_modules()))     # monai's Convolution children aside
    a.load_state_dict(b.state_dict(), strict=True)


# ---- state_dict layout ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_state_dict_matches_fixture(name):
    g = GOLD[name]
    m = DiffusionModelEncoder(**g["kwargs"])
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, tuple(s)) for k, s in g["keys"]]
    gen = torch.Generator().manual_seed(0)
    sd = {k: torch.randn(s, generator=gen) for k, s in g["keys"]}      # a checkpoint with the reference's layout
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.out[0].weight, sd["out.0.weight"])


def test_no_middle_block_and_every_level_downsamples():
    for updown, kind in ((False, Downsample), (True, ResnetBlock)):
        m = DiffusionModelEncoder(**_kw(resblock_updown=updown))
        assert not hasattr(m, "middle_block") and not hasattr(m, "up_blocks")
        assert all(isinstance(b.downsampler, kind) for b in m.down_blocks)
        if updown:
            assert all(b.downsampler.down for b in m.down_blocks)


def test_no_flash_attention_or_dropout_cattn_arguments():
    for extra in (dict(use_flash_attention=True), dict(dropout_cattn=0.1)):
        with pytest.raises(TypeError):
            DiffusionModelEncoder(**_kw(**extra))


# ---- import path -------------------------------------------------------------------------------------------------
def test_import_through_alias_module_only():
    code = f'''
import sys
sys.path.insert(0, {str(ROOT)!r})
from generative.networks.nets.diffusion_model_unet import DiffusionModelEncoder, DiffusionModelUNet
from generativemodels_b200.networks.nets.diffusion_model_unet import DiffusionModelEncoder as E
import generative.networks.nets as nets
import generativemodels_b200.networks.nets.diffusion_model_unet as M
assert DiffusionModelEncoder is E and DiffusionModelUNet is nets.DiffusionModelUNet
assert not hasattr(nets, "DiffusionModelEncoder"), "generative.networks.nets must not export the encoder"
assert M.__all__ == ["DiffusionModelUNet"]
'''
    env = {k: v for k, v in os.environ.items() if k != "PYTHONPATH"}
    subprocess.run([sys.executable, "-c", code], check=True, cwd="/tmp", env=env)


# ---- refusals ----------------------------------------------------------------------------------------------------
def test_cpu_input_raises():
    m = DiffusionModelEncoder(**TUTORIAL)
    with pytest.raises(RuntimeError, match="CUDA devices only"):
        m(torch.randn(1, 1, 64, 64), torch.Tensor((10,)))


def test_grad_enabled_call_raises_forward_only():
    m = DiffusionModelEncoder(**TUTORIAL)
    x = torch.randn(1, 1, 64, 64).requires_grad_(True)
    with torch.enable_grad():
        with pytest.raises(RuntimeError, match="forward only"):
            m(x, timesteps=torch.Tensor((10,)))
    with torch.no_grad():                      # not a gradient request: reaches the (CPU) device check instead
        with pytest.raises(RuntimeError, match="CUDA devices only"):
            m(x, timesteps=torch.Tensor((10,)))


# ---- the host code on the CPU stand-in -------------------------------------------------------------------------
@pytest.fixture
def cpu_lib(monkeypatch):
    return cpu_backend.install(monkeypatch)


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("name", CASES)
def test_host_path_vs_fixture(cpu_lib, name):
    g = GOLD[name]
    m = DiffusionModelEncoder(**g["kwargs"])
    G.recipe_state_dict(m, g["seed"])
    for r in g["runs"]:
        got = m(g["x"], r["t"], context=g["context"], class_labels=g["class_labels"])
        assert got.shape == r["logits"].shape and got.dtype == torch.float32
        assert _rel(got, r["logits"]) < 2e-2


SMALL_HEAD = dict(spatial_dims=2, in_channels=1, out_channels=2, num_channels=(32,), attention_levels=(False,),
                  num_res_blocks=(1,))


def test_head_width_other_than_4096_raises(cpu_lib):
    with torch.no_grad():
        with pytest.raises(RuntimeError, match=r"mat1 and mat2 shapes cannot be multiplied \(2x512 and 4096x512\)"):
            DiffusionModelEncoder(**SMALL_HEAD)(torch.randn(2, 1, 8, 8), torch.Tensor((5,)))


def test_head_width_error_matches_reference(ref):
    with torch.no_grad():
        with pytest.raises(RuntimeError) as want:
            ref.DiffusionModelEncoder(**SMALL_HEAD)(torch.randn(2, 1, 8, 8), torch.Tensor((5,)))
    assert str(want.value) == "mat1 and mat2 shapes cannot be multiplied (2x512 and 4096x512)"
