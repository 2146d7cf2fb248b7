"""PatchDiscriminator / MultiScalePatchDiscriminator without a GPU: the plain-PyTorch restatement
(tests/patchgan_oracle.py) against the unmodified reference where a checkout is readable and against the committed
fixture everywhere; state_dict keys and the seeded initialisation against both; the reference's quirks and exceptions;
the mode rule; the BatchNorm fold and its pack cache and the module's host code end to end on the CPU stand-in of the
library."""
import subprocess
import sys
import warnings
from pathlib import Path

import pytest
import torch
import torch.nn as nn

from tests.golden import load
from tests import patchgan_oracle as PO
from oracle import ref_import
from generativemodels_b200 import ops
from generativemodels_b200.networks._holders import Convolution
from generativemodels_b200.networks.nets.patchgan_discriminator import MultiScalePatchDiscriminator, PatchDiscriminator

GOLD = load("g_patchgan")
CLASSES = {"PatchDiscriminator": PatchDiscriminator, "MultiScalePatchDiscriminator": MultiScalePatchDiscriminator}
FEATURE_CASES = [n for n, g in GOLD.items() if "features" in g]


def _net(g, seed=0):
    return PO.seeded_weights(CLASSES[g["cls"]](**g["kwargs"]), seed).eval()


def _oracle(g, sd, x):
    """(scores, features) as the fixture stores them."""
    if g["cls"] == "PatchDiscriminator":
        o = PO.patch_discriminator(sd, x, **g["kwargs"])
        return o[-1], o[:-1]
    return PO.multiscale(sd, x, **g["kwargs"])


def _flat(t):
    return [u for v in t for u in _flat(v)] if isinstance(t, (list, tuple)) else [t]


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


@pytest.fixture(scope="module")
def ref():
    if not ref_import.available():
        pytest.skip("reference checkout not present")
    ref_import.import_reference()
    import generative.networks.nets.patchgan_discriminator as nets
    return nets


# ---- the oracle ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(GOLD))
def test_oracle_vs_fixture(name):
    g = GOLD[name]
    with torch.no_grad():
        scores, feats = _oracle(g, _net(g).state_dict(), PO.input_of(g))
    for got, want in zip(_flat(scores), _flat(g["scores"]), strict=True):
        assert got.shape == want.shape and _rel(got, want) < 1e-5
    if "features" in g:
        for got, want in zip(_flat(feats), _flat(g["features"]), strict=True):
            assert got.shape == want.shape and _rel(got, want) < 1e-3       # stored as fp16


ORACLE_CONFIGS = [
    ("PatchDiscriminator", dict(spatial_dims=2, num_channels=8, in_channels=2, num_layers_d=3), (2, 2, 32, 40)),
    ("PatchDiscriminator", dict(spatial_dims=3, num_channels=4, in_channels=1, num_layers_d=2, kernel_size=3,
                                activation="SILU", bias=True), (1, 1, 16, 12, 20)),
    ("PatchDiscriminator", dict(spatial_dims=2, num_channels=8, in_channels=3, num_layers_d=2, activation="GELU",
                                last_conv_kernel_size=1, padding=2, kernel_size=5), (1, 3, 24, 24)),
    ("MultiScalePatchDiscriminator", dict(num_d=3, num_layers_d=2, spatial_dims=2, num_channels=4, in_channels=2,
                                          pooling_method="avg", kernel_size=4, minimum_size_im=64), (1, 2, 48, 64)),
    ("MultiScalePatchDiscriminator", dict(num_d=2, num_layers_d=2, spatial_dims=3, num_channels=4, in_channels=1,
                                          pooling_method="max", norm="Instance", kernel_size=3, minimum_size_im=64,
                                          dropout=("dropout", {"p": 0.3})), (1, 1, 24, 32, 16)),
]


@pytest.mark.parametrize("cls,kw,shape", ORACLE_CONFIGS)
def test_oracle_vs_reference(ref, cls, kw, shape):
    m = PO.seeded_weights(getattr(ref, cls)(**kw), seed=3).eval()
    x = torch.randn(shape, generator=torch.Generator().manual_seed(4))
    g = dict(cls=cls, kwargs=kw)
    with torch.no_grad():
        want = m(x)
        scores, feats = _oracle(g, m.state_dict(), x)
    want_scores, want_feats = (want[-1], want[:-1]) if cls == "PatchDiscriminator" else want
    for got, w in zip(_flat([scores, feats]), _flat([want_scores, want_feats]), strict=True):
        assert got.shape == w.shape and _rel(got, w) < 1e-5


# ---- module tree, keys and initialisation -------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(GOLD))
def test_state_dict_keys_vs_fixture(name):
    g = GOLD[name]
    m = CLASSES[g["cls"]](**g["kwargs"])
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [tuple(kv) for kv in g["keys"]]


@pytest.mark.parametrize("name", list(GOLD))
def test_seeded_initialisation_vs_fixture(name):
    g = GOLD[name]
    torch.manual_seed(0)
    sd = CLASSES[g["cls"]](**g["kwargs"]).state_dict()
    for k, want in g["init_sums"].items():
        v = sd[k].double()
        # float64 sums of float32 values: any different draw shows far above the summation-order noise
        assert torch.allclose(torch.stack([v.sum(), (v ** 2).sum()]), want, rtol=1e-12, atol=1e-12), k


@pytest.mark.parametrize("name", list(GOLD))
def test_state_dict_and_initialisation_match_reference(ref, name):
    g = GOLD[name]
    torch.manual_seed(0)
    r = getattr(ref, g["cls"])(**g["kwargs"])
    torch.manual_seed(0)
    mine = CLASSES[g["cls"]](**g["kwargs"])
    rs, ms = r.state_dict(), mine.state_dict()
    assert list(ms) == list(rs)
    for k in rs:
        assert torch.equal(ms[k], rs[k]), k                        # bit-identical parameters and buffers
    assert set(dict(mine.named_modules())) <= set(dict(r.named_modules()))   # monai's ADN act / dropout aside
    assert [n for n, _ in mine.named_children()] == [n for n, _ in r.named_children()]
    mine.load_state_dict(PO.seeded_weights(r).state_dict(), strict=True)


def test_pooled_subnetworks_repeat_one_pool():
    m = MultiScalePatchDiscriminator(3, 2, 2, 4, 1, pooling_method="max", kernel_size=3, minimum_size_im=64)
    d2 = m.discriminator_2
    assert isinstance(d2, nn.Sequential) and len(d2) == 3 and d2[0] is d2[1] and isinstance(d2[0], nn.MaxPool2d)
    assert isinstance(d2[2], PatchDiscriminator) and "discriminator_2.2.initial_conv.conv.weight" in m.state_dict()
    assert d2[0].kernel_size == 3 and d2[0].stride == 2 and d2[0].padding == (1, 1)


# ---- quirks and exceptions ---------------------------------------------------------------------------------------
def test_num_layers_multiplied_without_pooling():
    assert MultiScalePatchDiscriminator(3, 2, 2, 4, 1, minimum_size_im=256).num_layers_d == [2, 4, 6]
    assert MultiScalePatchDiscriminator(3, 2, 2, 4, 1, pooling_method="avg").num_layers_d == [2, 2, 2]
    assert MultiScalePatchDiscriminator(2, [1, 3], 2, 4, 1).num_layers_d == [1, 3]


def test_assertions(ref):
    for cls in (MultiScalePatchDiscriminator, ref.MultiScalePatchDiscriminator):
        with pytest.raises(AssertionError):                       # reference test: TEST_TOO_SMALL_SIZE
            cls(num_d=2, num_layers_d=6, spatial_dims=2, num_channels=8, in_channels=3, kernel_size=3, norm="instance")
        with pytest.raises(AssertionError):                       # reference test: TEST_MISMATCHED_NUM_LAYERS
            cls(num_d=5, num_layers_d=[3, 4, 5], spatial_dims=2, num_channels=8, in_channels=3, norm="instance")


def test_assertions_without_reference():
    with pytest.raises(AssertionError):
        MultiScalePatchDiscriminator(2, 6, 2, 8, 3, kernel_size=3, norm="instance")
    with pytest.raises(AssertionError):
        MultiScalePatchDiscriminator(5, [3, 4, 5], 2, 8, 3)
    with pytest.raises(AssertionError):
        MultiScalePatchDiscriminator(1, 9, 2, 8, 3, minimum_size_im=256)


@pytest.mark.parametrize("norm", [("BATCH", {}), None, 3])
def test_non_string_norm_raises_attributeerror(norm):
    with pytest.raises(AttributeError):
        PatchDiscriminator(2, 8, 1, norm=norm)
    with pytest.raises(AttributeError):
        MultiScalePatchDiscriminator(2, 2, 2, 8, 1, norm=norm)


def test_non_string_norm_matches_reference(ref):
    with pytest.raises(AttributeError):
        ref.PatchDiscriminator(2, 8, 1, norm=("BATCH", {}))


def test_ddp_batchnorm_warning(monkeypatch):
    monkeypatch.setattr(torch.distributed, "is_initialized", lambda: True)
    with pytest.warns(UserWarning, match="SyncBatchNorm"):
        PatchDiscriminator(2, 8, 1, norm="batch")
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        PatchDiscriminator(2, 8, 1, norm="INSTANCE")


@pytest.mark.parametrize("kw", [dict(spatial_dims=1), dict(norm="GROUP"), dict(norm="layer"),
                                dict(activation="PRELU"), dict(activation=("LEAKYRELU", {"negative_slope": 0.3})),
                                dict(norm="INSTANCE", activation="RELU"), dict(norm="instance", activation="TANH"),
                                dict(dropout=("GAUSSIAN", {"p": 0.1})), dict(dropout="0.1")])
def test_unsupported_raise_notimplemented(kw):
    args = dict(spatial_dims=2, num_channels=8, in_channels=1)
    args.update(kw)
    with pytest.raises(NotImplementedError, match="support"):
        PatchDiscriminator(**args)


@pytest.mark.parametrize("pooling", ["adaptiveavg", "lp"])
def test_unsupported_pooling(pooling):
    with pytest.raises(NotImplementedError, match="'avg' or 'max'"):
        MultiScalePatchDiscriminator(2, 2, 2, 8, 1, pooling_method=pooling)


def test_supported_variants_construct():
    for kw in (dict(norm="batch"), dict(norm="Instance", activation="SWISH"), dict(activation="LEAKYRELU"),
               dict(activation=("LEAKYRELU", {})), dict(activation=None, norm="instance"), dict(activation="SIGMOID"),
               dict(dropout=0.5), dict(dropout=("alphadropout", {"p": 0.2})), dict(spatial_dims=3, kernel_size=3)):
        args = dict(spatial_dims=2, num_channels=8, in_channels=1)
        args.update(kw)
        PatchDiscriminator(**args)


def test_import_through_alias():
    code = ("from generative.networks.nets import PatchDiscriminator as A, MultiScalePatchDiscriminator as B; "
            "from generativemodels_b200.networks.nets import PatchDiscriminator as C, MultiScalePatchDiscriminator as D; "
            "import generative.networks.nets.patchgan_discriminator as M; "
            "assert A is C and B is D and M.PatchDiscriminator is A")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=Path(__file__).resolve().parents[1])


# ---- the host code on the CPU stand-in ---------------------------------------------------------------------------
@pytest.fixture
def cpu_lib(monkeypatch):
    return PO.install(monkeypatch)


def _run(net, x):
    with torch.no_grad():
        out = net(x)
    return (out[-1], out[:-1]) if isinstance(net, PatchDiscriminator) else out


@pytest.mark.parametrize("name", ["ldm2d", "spade_vae", "test_2d_pool", "test_3d_pool"])
def test_host_path_vs_fixture(cpu_lib, name):
    g = GOLD[name]
    scores, feats = _run(_net(g), PO.input_of(g))
    for got, want in zip(_flat(scores), _flat(g["scores"]), strict=True):
        assert got.dtype == torch.float32 and got.shape == want.shape and _rel(got, want) < 2e-2
    for got, want in zip(_flat(feats), _flat(g["features"]), strict=True):
        assert got.shape == want.shape and _rel(got, want) < 2e-2


def test_mode_rule(cpu_lib):
    x = torch.randn(1, 1, 32, 32)
    for kw in (dict(norm="BATCH"), dict(norm="INSTANCE", dropout=0.1), dict(norm="INSTANCE", dropout=("DROPOUT", {}))):
        net = PatchDiscriminator(2, 4, 1, num_layers_d=2, **kw)
        with pytest.raises(RuntimeError, match=r"\.eval\(\)"):
            net(x)
        ms = MultiScalePatchDiscriminator(2, 1, 2, 4, 1, minimum_size_im=32, **kw)
        with pytest.raises(RuntimeError, match=r"\.eval\(\)"):
            ms(x)
        assert len(net.eval()(x)) == 4 and len(ms.eval()(x)[0]) == 2
    # the 2d_spade_vae discriminator (INSTANCE, p = 0) runs as constructed, in train mode, with the eval-mode result
    ms = MultiScalePatchDiscriminator(2, 1, 2, 4, 1, minimum_size_im=32, norm="INSTANCE", kernel_size=3)
    assert ms.training
    a = ms(x)
    b = ms.eval()(x)
    assert all(torch.equal(u, v) for u, v in zip(_flat(list(a)), _flat(list(b))))


def test_features_in_caller_dtype(cpu_lib):
    net = PO.seeded_weights(PatchDiscriminator(2, 8, 1, num_layers_d=2)).eval()
    out = _run(net, torch.randn(1, 1, 24, 24).double())
    assert all(t.dtype == torch.float64 for t in [out[0], *out[1]])


def _holder(seed=0):
    h = Convolution(2, 5, 12, strides=2, kernel_size=4, padding=1, bias=False, conv_only=False,
                    act=PO.LEAKY02, norm="BATCH")
    return PO.seeded_weights(h, seed).eval()


def test_holder_batchnorm_fold_and_cache(cpu_lib):
    h = _holder()
    assert isinstance(h.adn.N, nn.BatchNorm2d) and h.conv.bias is None
    bn = h.adn.N
    pc = h.packed([5])
    assert h.packed([5]) is pc                                     # cached
    s = bn.weight.double() / (bn.running_var.double() + bn.eps).sqrt()
    w_want = (h.conv.weight.double() * s[:, None, None, None]).float()
    assert torch.equal(pc.bias, (bn.bias.double() - bn.running_mean.double() * s).float())
    assert torch.equal(pc.w, ops.PackedConv(w_want, None, 2, 1).w)  # one rounding to h16 of the folded weight
    x = torch.randn(2, 5, 16, 16)
    with torch.no_grad():
        got = ops.from_cl(h(ops.to_cl(x)))
        want = PO.act_fn(PO.LEAKY02)(bn(h.conv(ops.from_cl(ops.to_cl(x)))))
    assert _rel(got, want) < 1e-2
    # new statistics / affine parameters through load_state_dict: the next call repacks
    for key in ("adn.N.running_var", "adn.N.running_mean", "adn.N.weight", "adn.N.bias"):
        sd = h.state_dict()
        sd[key] = sd[key] * 1.5 + 0.25
        h.load_state_dict(sd)
        pc2 = h.packed([5])
        assert pc2 is not pc, key
        pc = pc2
    with torch.no_grad():
        got = ops.from_cl(h(ops.to_cl(x)))
        want = PO.act_fn(PO.LEAKY02)(bn(h.conv(ops.from_cl(ops.to_cl(x)))))
    assert _rel(got, want) < 1e-2


def test_holder_batchnorm_train_mode_raises(cpu_lib):
    h = _holder().train()
    with pytest.raises(RuntimeError, match=r"\.eval\(\)"):
        h(ops.to_cl(torch.randn(1, 5, 8, 8)))


def test_holder_other_norms_unchanged():
    h = Convolution(3, 4, 8, conv_only=False, norm="instance", act="LEAKYRELU")
    assert isinstance(h.adn.N, nn.InstanceNorm3d) and h.instance_norm and not list(h.adn.parameters())
    assert not hasattr(Convolution(2, 4, 8, conv_only=True, norm="BATCH"), "adn")
    with pytest.raises(NotImplementedError, match="INSTANCE or BATCH"):
        Convolution(2, 4, 8, conv_only=False, norm="GROUP")
    with pytest.raises(NotImplementedError):
        Convolution(2, 4, 8, conv_only=False, norm="BATCH", is_transposed=True)


def test_load_state_dict_statistics_reach_forward(cpu_lib):
    g = GOLD["ldm2d"]
    net = _net(g)
    x = PO.input_of(g)
    a = _run(net, x)[0]
    sd = net.state_dict()
    sd["1.adn.N.running_var"] = sd["1.adn.N.running_var"] * 4
    sd["2.adn.N.running_mean"] = sd["2.adn.N.running_mean"] + 0.5
    net.load_state_dict(sd)
    b = _run(net, x)[0]
    with torch.no_grad():
        want = PO.patch_discriminator(net.state_dict(), x, **g["kwargs"])[-1]
    assert _rel(b, want) < 2e-2 and _rel(a, want) > 5e-2
