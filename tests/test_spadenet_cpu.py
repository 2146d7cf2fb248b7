"""SPADENet without a GPU: the plain-PyTorch restatement (tests/spadenet_oracle.py) against the unmodified reference
where a checkout is readable and against the committed fixture everywhere; the module's host code end to end on the
CPU stand-in of the library; state_dict keys, constructor quirks, exceptions and the activation / norm mapping rules."""
import pytest
import torch

from tests.golden import load
from tests import spadenet_oracle as SO
from oracle import ref_import
from generativemodels_b200 import ops
from generativemodels_b200.networks._holders import act_code
from generativemodels_b200.networks.blocks.spade_norm import SPADE
from generativemodels_b200.networks.nets.spade_network import SPADENet

GOLD = load("g_spadenet")


def _net(kw):
    kw = dict(kw)
    kw["num_channels"] = list(kw["num_channels"])
    return SO.seeded_weights(SPADENet(**kw)).eval()


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.fixture(scope="module")
def ref():
    if not ref_import.available():
        pytest.skip("reference checkout not present")
    ref_import.import_reference()
    import generative.networks.nets.spade_network as nets
    return nets


# ---- the oracle ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tutorial", "bilinear", "bicubic"])
def test_oracle_vs_fixture(name):
    g = GOLD[name]
    kw = g["kwargs"]
    sd = _net(kw).state_dict()
    seg = SO.labels_to_onehot(g["labels"], kw["label_nc"])
    with torch.no_grad():
        img, kld, mu, logvar, z = SO.spadenet_vae(sd, seg, g["x"], g["eps"], len(kw["num_channels"]),
                                                  kw.get("upsampling_mode", "nearest"),
                                                  None if "last_act" in kw else 0.2)
    for got, want in ((mu, g["mu"]), (logvar, g["logvar"]), (z, g["z"]), (img, g["out"])):
        assert _rel(got, want) < 1e-5
    assert abs(kld.item() - g["kld"].item()) <= 1e-5 * abs(g["kld"].item())


def test_oracle_gan_vs_fixture():
    g = GOLD["gan"]
    kw = g["kwargs"]
    sd = _net(kw).state_dict()
    seg = SO.labels_to_onehot(g["labels"], kw["label_nc"])
    with torch.no_grad():
        out = SO.decoder(sd, seg, None, 8, [8, 8], 2, True)
    assert out.shape == (1, 1, 32, 2048)
    assert _rel(out, g["out"]) < 1e-5


@pytest.mark.parametrize("mode", ["nearest", "bilinear", "bicubic"])
def test_oracle_vs_reference(ref, mode):
    kw = dict(spatial_dims=2, in_channels=2, out_channels=3, label_nc=4, input_shape=[16, 24], num_channels=[8, 12],
              z_dim=5, upsampling_mode=mode, spade_intermediate_channels=16)
    m = SO.seeded_weights(ref.SPADENet(**kw), seed=3).eval()
    seg = SO.one_hot_seg(2, 4, (16, 24), seed=5)
    x = torch.randn(2, 2, 16, 24)
    eps = torch.randn(2, 5)
    with torch.no_grad():
        mu, logvar = m.encoder(x)
        img, kld, mu2, logvar2, z = SO.spadenet_vae(m.state_dict(), seg, x, eps, 2, mode)
        want = m.decode(seg, eps * torch.exp(0.5 * logvar) + mu)
        want_kld = m.kld_loss(mu, logvar)
    assert _rel(mu2, mu) < 1e-6 and _rel(logvar2, logvar) < 1e-6
    assert _rel(img, want) < 1e-5
    assert abs(kld.item() - want_kld.item()) <= 1e-5 * abs(want_kld.item())


def test_oracle_vs_reference_3d_and_gan(ref):
    kw = dict(spatial_dims=3, in_channels=1, out_channels=2, label_nc=3, input_shape=[8, 8, 16], num_channels=[8, 16],
              z_dim=4, spade_intermediate_channels=8)
    m = SO.seeded_weights(ref.SPADENet(**kw)).eval()
    seg = SO.one_hot_seg(1, 3, (8, 8, 16))
    z = torch.randn(1, 4)
    with torch.no_grad():
        assert _rel(SO.decoder(m.state_dict(), seg, z, 16, [2, 2, 4], 2, False), m.decode(seg, z)) < 1e-5
    g = SO.seeded_weights(ref.SPADENet(2, 1, 1, 8, [32, 32], [8, 8], None, False)).eval()
    seg = SO.one_hot_seg(1, 8, (32, 32))
    with torch.no_grad():
        assert _rel(SO.decoder(g.state_dict(), seg, None, 8, [8, 8], 2, True), g(seg)[0]) < 1e-5


# ---- module tree, keys and quirks -------------------------------------------------------------------------------
def test_state_dict_matches_reference(ref):
    for args in ([2, 1, 1, 3, [64, 64], [16, 32, 64, 128], 16, True], [3, 1, 1, 3, [64, 64, 64], [16, 32, 64, 128], 16, True],
                 [2, 1, 1, 8, [32, 32], [8, 8], None, False]):
        a, b = list(args), list(args)
        a[5], b[5] = list(args[5]), list(args[5])
        r = ref.SPADENet(*a)
        mine = SPADENet(*b)
        assert list(mine.state_dict()) == list(r.state_dict())
        assert set(dict(mine.named_modules())) <= set(dict(r.named_modules()))   # monai's ADN act children aside
        mine.load_state_dict(r.state_dict(), strict=True)
        assert a[5] == b[5]                     # the same in-place reversal and append


def test_state_dict_keys_2d_count():
    assert len(SPADENet(2, 1, 1, 3, [64, 64], [16, 32, 64, 128], 16, True).state_dict()) == 112


def test_num_channels_reversed_in_place_and_appended():
    ch = [16, 32]
    net = SPADENet(2, 1, 1, 3, [16, 16], ch, 4, True)
    assert ch == [32, 16, 1]
    assert net.num_channels is ch and net.decoder.num_channels is ch and net.encoder.num_channels is ch


def test_vae_without_z_dim_fails_in_linear_not_valueerror():
    # the reference builds the ValueError without raising it; nn.Linear(.., None) then fails
    with pytest.raises(TypeError):
        SPADENet(2, 1, 1, 3, [16, 16], [8, 8], None, True)


def test_vae_without_z_dim_matches_reference(ref):
    with pytest.raises(TypeError):
        ref.SPADENet(2, 1, 1, 3, [16, 16], [8, 8], None, True)


def test_input_shape_errors():
    with pytest.raises(ValueError):
        SPADENet(2, 1, 1, 3, [16, 16, 16], [8, 8], 4, True)
    with pytest.raises(ValueError):
        SPADENet(2, 1, 1, 3, [18, 16], [8, 8], 4, True)


# ---- the host code on the CPU stand-in ---------------------------------------------------------------------------
@pytest.fixture
def cpu_lib(monkeypatch):
    return SO.install(monkeypatch)


@pytest.mark.parametrize("name", ["tutorial", "bilinear", "bicubic"])
def test_host_path_vs_fixture(cpu_lib, name):
    g = GOLD[name]
    kw = g["kwargs"]
    net = _net(kw)
    seg = SO.labels_to_onehot(g["labels"], kw["label_nc"])
    with torch.no_grad():
        mu, logvar = net.encoder(g["x"])
        z, kld = ops.vae_reparam_kld(g["mu"], g["logvar"], g["eps"])
        out = net.decode(seg, g["z"])
    assert _rel(mu, g["mu"]) < 2e-2 and _rel(logvar, g["logvar"]) < 2e-2
    assert _rel(z, g["z"]) < 1e-6 and abs(kld.item() - g["kld"].item()) <= 1e-5 * abs(g["kld"].item())
    assert _rel(out, g["out"]) < 2e-2


def test_host_path_gan(cpu_lib):
    g = GOLD["gan"]
    net = _net(g["kwargs"])
    seg = SO.labels_to_onehot(g["labels"], 8)
    with torch.no_grad():
        (out,) = net(seg)
    assert out.shape == (1, 1, 32, 2048)
    assert _rel(out, g["out"]) < 2e-2


def test_forward_returns_tuple_and_kld(cpu_lib):
    net = SO.seeded_weights(SPADENet(2, 1, 1, 3, [16, 16], [8, 8], 4, True)).eval()
    seg = SO.one_hot_seg(2, 3, (16, 16))
    with torch.no_grad():
        out = net(seg, torch.randn(2, 1, 16, 16))
        assert isinstance(out, tuple) and len(out) == 2 and out[0].shape == (2, 1, 16, 16) and out[1].dim() == 0
        assert net.encode(torch.randn(2, 1, 16, 16)).shape == (2, 4)


def test_gan_mode_errors(cpu_lib):
    with torch.no_grad():
        net = SPADENet(2, 1, 1, 8, [32, 32], [8, 8], None, False)      # latent 8x8 == label_nc: runs
        assert net(SO.one_hot_seg(1, 8, (32, 32)))[0].shape == (1, 1, 32, 2048)
        with pytest.raises(RuntimeError):                              # last latent axis 8 != label_nc 3
            SPADENet(2, 1, 1, 3, [32, 32], [8, 8], None, False)(SO.one_hot_seg(1, 3, (32, 32)))
        with pytest.raises(RuntimeError):                              # label_nc 8 != the first block's 16 channels
            SPADENet(2, 1, 1, 8, [32, 32], [8, 16], None, False)(SO.one_hot_seg(1, 8, (32, 32)))


def test_gan_mode_errors_match_reference(ref):
    with torch.no_grad():
        with pytest.raises(RuntimeError):
            ref.SPADENet(2, 1, 1, 3, [32, 32], [8, 8], None, False)(SO.one_hot_seg(1, 3, (32, 32)))
        with pytest.raises(RuntimeError):
            ref.SPADENet(2, 1, 1, 8, [32, 32], [8, 16], None, False)(SO.one_hot_seg(1, 8, (32, 32)))


def test_decode_without_z_raises_attributeerror(cpu_lib, ref):
    seg = SO.one_hot_seg(1, 3, (16, 16))
    with pytest.raises(AttributeError):
        SPADENet(2, 1, 1, 3, [16, 16], [8, 8], 4, True).decode(seg)
    with pytest.raises(AttributeError):
        ref.SPADENet(2, 1, 1, 3, [16, 16], [8, 8], 4, True).decode(seg)


@pytest.mark.parametrize("mode", ["bilinear", "bicubic"])
def test_3d_interpolating_upsample_not_implemented(cpu_lib, ref, mode):
    seg = SO.one_hot_seg(1, 3, (8, 8, 8))
    z = torch.randn(1, 4)
    with torch.no_grad():
        with pytest.raises(NotImplementedError):
            SPADENet(3, 1, 1, 3, [8, 8, 8], [8, 8], 4, True, upsampling_mode=mode).decode(seg, z)
        with pytest.raises(NotImplementedError):
            ref.SPADENet(3, 1, 1, 3, [8, 8, 8], [8, 8], 4, True, upsampling_mode=mode).decode(seg, z)


def test_import_through_alias():
    import subprocess
    import sys
    from pathlib import Path
    code = ("from generative.networks.nets import SPADENet as A; "
            "from generativemodels_b200.networks.nets import SPADENet as B; assert A is B")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=Path(__file__).resolve().parents[1])


# ---- activation and norm mapping rules ---------------------------------------------------------------------------
def test_act_code_leakyrelu_slopes():
    assert act_code("LEAKYRELU") == ops.ACT_LEAKYRELU
    assert act_code(("LEAKYRELU", {})) == ops.ACT_LEAKYRELU
    assert act_code(("LEAKYRELU", {"negative_slope": 0.2})) == ops.ACT_LEAKYRELU02 == 8
    assert act_code(("leakyrelu", {"negative_slope": 0.2})) == ops.ACT_LEAKYRELU02


@pytest.mark.parametrize("act", [("LEAKYRELU", {"negative_slope": 0.1}), ("LEAKYRELU", {"negative_slope": 0.2,
                                 "inplace": True}), ("RELU", {"inplace": True}), ("PRELU", {}), "ELU"])
def test_act_code_refusals(act):
    with pytest.raises(NotImplementedError):
        act_code(act)


def test_spade_norm_rules():
    s = SPADE(3, 16, norm="INSTANCE")
    assert isinstance(s.param_free_norm.N, torch.nn.InstanceNorm2d) and not list(s.param_free_norm.parameters())
    assert isinstance(SPADE(3, 16, spatial_dims=3).param_free_norm.N, torch.nn.InstanceNorm3d)
    g = SPADE(3, 16, norm="GROUP", norm_params={"num_groups": 4, "affine": False})
    assert isinstance(g.param_free_norm.N, torch.nn.GroupNorm) and g.param_free_norm.N.num_groups == 4
    for bad in (dict(norm="BATCH"), dict(norm="INSTANCE", norm_params={"affine": True}), dict(norm="LAYER")):
        with pytest.raises(NotImplementedError, match="GROUP|INSTANCE"):
            SPADE(3, 16, **bad)
