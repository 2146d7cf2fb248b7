"""SpatialRescaler and b200_interpolate without a GPU: the header's coordinate rules (tests/rescaler_oracle.py) and the
host-side size / ratio rules against F.interpolate on a grid of extents and multipliers; the module's host code end to
end on the CPU stand-in against the committed fixture; the reference test's shape and exception cases; state_dict keys
and seeded initialisation against the fixture and, where a checkout is readable, the unmodified reference."""
import itertools

import pytest
import torch
import torch.nn.functional as F

from tests import rescaler_oracle as RO
from tests.golden import load
from oracle import ref_import
from generativemodels_b200 import ops
from generativemodels_b200.networks._holders import Convolution
from generativemodels_b200.networks.blocks import SpatialRescaler

GOLD = load("g_spatial_rescaler")
_MODE_DIMS = [("nearest", 1), ("nearest", 2), ("nearest", 3), ("linear", 1), ("bilinear", 2), ("bicubic", 2),
              ("trilinear", 3), ("area", 1), ("area", 2), ("area", 3)]
_EXTENTS = (1, 2, 5, 7, 16, 17, 33)
_SCALES = (0.25, 0.5, 0.6, 1.0, 1.1, 1.3, 1.5, 1.7, 2.0, 2.1, 3.0)


@pytest.fixture(scope="module")
def ref():
    if not ref_import.available():
        pytest.skip("reference checkout not present")
    ref_import.import_reference()
    import generative.networks.blocks.encoder_modules as em
    return em


@pytest.fixture
def cpu_lib(monkeypatch):
    return RO.install(monkeypatch)


def _rescaler(kw, seed=0):
    return RO.seeded_weights(SpatialRescaler(**kw), seed).eval()


def _cpu_nearest2d_shortcut(ext, out, ratios):
    """ATen's CPU 2-D nearest kernel alone copies an axis whose extent does not change and halves the index of an axis
    that exactly doubles (nearest_idx), whatever the ratio; its CUDA kernels and the 1-D / 3-D CPU kernels apply
    min(floor(dst * ratio), in - 1) throughout, and so does b200_interpolate.  The two differ only there with a ratio
    other than 1 or 1/2."""
    return any((o == i and r != 1.0) or (o == 2 * i and r != 0.5) for i, o, r in zip(ext, out, ratios))


# ---- host-side size and ratio rules, and the header's coordinate rules, against F.interpolate ----------------------
@pytest.mark.parametrize("mode,dims", _MODE_DIMS)
def test_plan_and_header_rules_vs_interpolate(mode, dims):
    g = torch.Generator().manual_seed(dims)
    for n, s in itertools.product(_EXTENTS, _SCALES):
        ext = (n, 5, 4)[:dims][::-1]
        x = torch.randn((1, 2, *ext), generator=g)
        for arg in (dict(scale_factor=s), dict(size=max(1, int(n * s)))):
            if arg.get("scale_factor") is not None and min(int(e * s) for e in ext) < 1:
                continue
            want = F.interpolate(x, mode=mode, **arg)
            out, ratios = ops.interpolate_plan(ext, mode=mode, **arg)
            assert tuple(want.shape[2:]) == tuple(out), (mode, ext, arg)
            got = RO.header_interpolate(x, out, ratios, RO.MODES[mode])
            if mode == "nearest" and dims == 2 and _cpu_nearest2d_shortcut(ext, out, ratios):
                continue
            if mode == "nearest":
                assert torch.equal(got, want), (ext, arg)
            else:
                assert (got - want).abs().max() <= RO.ulps_of(x, 8), (mode, ext, arg)


def test_ratio_rule_odd_extent():
    # scale_factor=0.5 on 17 samples 0.5, 2.5, ...; size=8 samples 0.5625, 2.6875, ...
    assert ops.interpolate_plan((17,), scale_factor=0.5, mode="linear") == ([8], [2.0])
    assert ops.interpolate_plan((17,), size=8, mode="linear") == ([8], [2.125])
    x = torch.arange(17.0).view(1, 1, 17)
    for arg, first in ((dict(scale_factor=0.5), [0.5, 2.5]), (dict(size=8), [0.5625, 2.6875])):
        out, r = ops.interpolate_plan((17,), mode="linear", **arg)
        assert RO.header_interpolate(x, out, r, RO.LINEAR)[0, 0, :2].tolist() == first
    # scale_factor=1.1 on 5: nearest indices 0, 0, 1, 2, 3 (not the identity); linear copies the unchanged axis
    x = torch.arange(5.0).view(1, 1, 5)
    out, r = ops.interpolate_plan((5,), scale_factor=1.1, mode="nearest")
    assert RO.header_interpolate(x, out, r, RO.NEAREST)[0, 0].tolist() == [0, 0, 1, 2, 3]
    assert RO.header_interpolate(x, out, r, RO.LINEAR)[0, 0].tolist() == [0, 1, 2, 3, 4]


_BAD_ARGS = [dict(), dict(size=4, scale_factor=0.5), dict(size=(4, 4, 4)), dict(scale_factor=(0.5, 0.5, 0.5)),
             dict(size=(4.0, 4.0)), dict(size=4.5)]


@pytest.mark.parametrize("arg", _BAD_ARGS)
def test_plan_exceptions_match_interpolate(arg):
    with pytest.raises(Exception) as want:
        F.interpolate(torch.zeros(1, 1, 8, 8), mode="bilinear", **arg)
    with pytest.raises(want.type):
        ops.interpolate_plan((8, 8), mode="bilinear", **arg)


@pytest.mark.parametrize("mode,rank", [(m, r) for m in RO.MODES for r in (3, 4, 5)
                                       if (m, r - 2) not in _MODE_DIMS] + [("nearest", 6)])
def test_plan_mode_rank_mismatch_matches_interpolate(mode, rank):
    x = torch.zeros((1, 1) + (4,) * (rank - 2))
    with pytest.raises(NotImplementedError) as want:
        F.interpolate(x, scale_factor=2.0, mode=mode)
    with pytest.raises(NotImplementedError) as got:
        ops.interpolate_plan((4,) * (rank - 2), scale_factor=2.0, mode=mode)
    if rank != 6:
        assert str(got.value) == str(want.value)


# ---- the module's host code on the CPU stand-in -----------------------------------------------------------------
@pytest.mark.parametrize("name", [n for n in GOLD if not n.startswith("brain")])
def test_host_path_vs_fixture(cpu_lib, name):
    g = GOLD[name]
    m = _rescaler(g["kwargs"])
    with torch.no_grad():
        got = m(RO.input_of(g))
    want = g["out"]
    assert got.shape == want.shape and got.dtype == torch.float32
    if m.remap_output:
        assert ((got - want).norm() / want.norm()) < 2e-2
    elif g["kwargs"].get("method") == "nearest":
        assert torch.equal(got, want)
    else:
        assert (got - want).abs().max() <= RO.ulps_of(want, 8)


_REF_CASES = [(GOLD[f"ref_{i}"]["kwargs"], GOLD[f"ref_{i}"]["shape"], tuple(GOLD[f"ref_{i}"]["out"].shape))
              for i in range(7)]


@pytest.mark.parametrize("kw,shape,expected", _REF_CASES)
def test_reference_shape_cases(cpu_lib, kw, shape, expected):
    with torch.no_grad():
        assert SpatialRescaler(**kw)(torch.randn(shape)).shape == expected


def test_reference_exception_cases():
    with pytest.raises(AssertionError):
        SpatialRescaler(method="none")
    with pytest.raises(AssertionError):
        SpatialRescaler(n_stages=-1)
    with pytest.raises(ValueError):
        SpatialRescaler(n_stages=2, size=[8, 8, 8])
    with pytest.raises(ValueError):
        SpatialRescaler(size=[1, 2, 3], multiplier=0.5)


def test_forward_errors(cpu_lib):
    x = torch.randn(1, 3, 8, 8)
    with torch.no_grad():
        with pytest.raises(ValueError):                    # neither size nor multiplier: F.interpolate's error
            SpatialRescaler()(x)
        with pytest.raises(ValueError):
            SpatialRescaler(in_channels=3, out_channels=2)(x)
        with pytest.raises(NotImplementedError):           # bilinear on a 5-D input
            SpatialRescaler(multiplier=0.5)(torch.randn(1, 1, 4, 4, 4))
        with pytest.raises(ValueError):                    # multiplier of the wrong length
            SpatialRescaler(multiplier=(0.5, 0.5, 0.5))(x)
        assert SpatialRescaler(n_stages=0)(x) is x         # no stage, no error
        y = _rescaler(dict(n_stages=0, in_channels=3, out_channels=5))(x)
        assert y.shape == (1, 5, 8, 8)


def test_forward_errors_match_reference(ref):
    x = torch.randn(1, 3, 8, 8)
    with pytest.raises(ValueError):
        ref.SpatialRescaler()(x)
    with pytest.raises(NotImplementedError):
        ref.SpatialRescaler(multiplier=0.5)(torch.randn(1, 1, 4, 4, 4))
    with pytest.raises(ValueError):
        ref.SpatialRescaler(multiplier=(0.5, 0.5, 0.5))(x)
    assert ref.SpatialRescaler(n_stages=0)(x) is x


def test_caller_dtype_and_encode(cpu_lib):
    x = torch.randn(1, 3, 8, 12)
    m = _rescaler(dict(multiplier=0.5, in_channels=3, out_channels=4))
    with torch.no_grad():
        assert m(x.double()).dtype == torch.float64
        assert SpatialRescaler(multiplier=0.5, method="nearest")(x.half()).dtype == torch.float16
        assert torch.equal(m.encode(x), m(x))
        assert m.interpolator(x, scale_factor=2.0).shape == (1, 3, 16, 24)


def test_cpu_tensor_refused():
    with pytest.raises(RuntimeError, match="CPU"):
        SpatialRescaler(multiplier=0.5)(torch.randn(1, 3, 8, 8))


def test_no_gradients(cpu_lib):
    x = torch.randn(1, 3, 8, 8, requires_grad=True)
    assert not SpatialRescaler(multiplier=0.5)(x).requires_grad


def test_print_when_remapping(capsys):
    SpatialRescaler(in_channels=3, out_channels=2)
    assert capsys.readouterr().out == "Spatial Rescaler mapping from 3 to 2 channels before resizing.\n"
    SpatialRescaler()
    assert capsys.readouterr().out == ""


# ---- keys, seeded initialisation, the 1-D holder ----------------------------------------------------------------
@pytest.mark.parametrize("name", list(GOLD))
def test_keys_and_init_vs_fixture(name):
    g = GOLD[name]
    torch.manual_seed(0)
    m = SpatialRescaler(**g["kwargs"])
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == g["keys"]
    for k, v in m.state_dict().items():
        assert torch.allclose(torch.stack([v.double().sum(), (v.double() ** 2).sum()]), g["init_sums"][k], rtol=1e-12)
    assert m.n_stages == g["kwargs"].get("n_stages", 1) and m.multiplier == g["kwargs"].get("multiplier")
    assert m.remap_output == (g["kwargs"].get("out_channels") is not None)


@pytest.mark.parametrize("spatial_dims", [1, 2, 3])
@pytest.mark.parametrize("bias", [False, True])
def test_keys_and_init_vs_reference(ref, spatial_dims, bias):
    kw = dict(spatial_dims=spatial_dims, multiplier=0.5, in_channels=3, out_channels=5, bias=bias)
    torch.manual_seed(0)
    r = ref.SpatialRescaler(**kw)
    torch.manual_seed(0)
    mine = SpatialRescaler(**kw)
    assert list(mine.state_dict()) == list(r.state_dict())
    for k, v in r.state_dict().items():
        assert torch.equal(mine.state_dict()[k], v)
    mine.load_state_dict(r.state_dict(), strict=True)
    assert type(mine.channel_mapper.conv) is type(r.channel_mapper.conv)


def test_holder_builds_conv1d_for_one_spatial_dim():
    for sd, cls in ((1, torch.nn.Conv1d), (2, torch.nn.Conv2d), (3, torch.nn.Conv3d)):
        c = Convolution(spatial_dims=sd, in_channels=3, out_channels=4, kernel_size=1, conv_only=True)
        assert type(c.conv) is cls and tuple(c.conv.weight.shape) == (4, 3) + (1,) * sd


def test_import_through_alias():
    import subprocess
    import sys
    from pathlib import Path
    code = ("from generative.networks.blocks import SpatialRescaler as A; "
            "from generative.networks.blocks.encoder_modules import SpatialRescaler as B; "
            "from generativemodels_b200.networks.blocks import SpatialRescaler as C; assert A is B is C")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=Path(__file__).resolve().parents[1])


# ---- the fixture against the reference ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(GOLD))
def test_fixture_vs_reference(ref, name):
    g = GOLD[name]
    m = RO.seeded_weights(ref.SpatialRescaler(**g["kwargs"])).eval()
    x = RO.input_of(g)
    with torch.no_grad():
        assert torch.equal(m(x), g["out"])
        sd = m.state_dict()
        kw = {k: v for k, v in g["kwargs"].items() if k in ("n_stages", "size", "method", "multiplier")}
        assert torch.allclose(RO.rescaler(sd, x, **kw), g["out"], rtol=0, atol=RO.ulps_of(g["out"], 4))
