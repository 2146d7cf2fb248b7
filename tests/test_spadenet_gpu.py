"""SPADENet on the H100 kernels: the CUDA path against every case of the reference fixture (tests/golden/g_spadenet.pt),
b200_upsample2x_interp against F.interpolate, LeakyReLU(0.2) (B200_ACT_LEAKYRELU02) on every igemm store path against
the emulator and in the SPADE / GroupNorm apply passes, repeat calls and CUDA-graph replays bit for bit."""
from dataclasses import replace

import pytest
import torch
import torch.nn.functional as F

from generativemodels_b200 import ops
from generativemodels_b200._lib import ACT_GEGLU, ACT_LEAKYRELU02, ACT_NONE
from generativemodels_b200.cuda_graph import graphed
from generativemodels_b200.networks.nets.spade_network import SPADENet
from tests import spadenet_oracle as SO
from tests.golden import load
from tests.test_igemm_contract_gpu import CASES, lib, run_case  # noqa: F401  (lib is a fixture)

pytestmark = pytest.mark.gpu

GOLD = load("g_spadenet")
FP16 = ops.H16 is torch.float16


def _net(kw):
    kw = dict(kw)
    kw["num_channels"] = list(kw["num_channels"])
    return SO.seeded_weights(SPADENet(**kw)).eval().cuda()


def _close(got, want, what):
    got, want = got.float().cpu(), want.float().cpu()
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(want.shape)}"
    rel = ((got - want).norm() / want.norm()).item()
    mx = ((got - want).abs().max() / want.abs().max()).item()
    assert rel < 2e-2 and mx < 4e-2, f"{what}: rel L2 {rel:.3e}, normalised max-abs {mx:.3e}"


def _seg(g):
    return SO.labels_to_onehot(g["labels"], g["kwargs"]["label_nc"]).cuda()


# ---- the network against the reference fixture ------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tutorial", "ref3d"])
def test_vae_pieces_vs_fixture(cuda_device, name):
    g = GOLD[name]
    net = _net(g["kwargs"])
    with torch.no_grad():
        mu, logvar = net.encoder(g["x"].cuda())
        _close(mu, g["mu"], f"{name} mu")
        _close(logvar, g["logvar"], f"{name} logvar")
        z, kld = ops.vae_reparam_kld(g["mu"].cuda(), g["logvar"].cuda(), g["eps"].cuda())
        assert ((z.cpu() - g["z"]).abs().max() / g["z"].abs().max()).item() < 1e-5
        assert abs(kld.item() - g["kld"].item()) <= 2e-2 * abs(g["kld"].item())
        _close(net.decode(_seg(g), g["z"].cuda()), g["out"], f"{name} decode")


@pytest.mark.parametrize("name", ["bilinear", "bicubic"])
def test_interpolating_decoder_vs_fixture(cuda_device, name):
    g = GOLD[name]
    net = _net(g["kwargs"])
    with torch.no_grad():
        _close(net.decode(_seg(g), g["z"].cuda()), g["out"], name)


def test_gan_mode_vs_fixture(cuda_device):
    g = GOLD["gan"]
    net = _net(g["kwargs"])
    with torch.no_grad():
        out = net(_seg(g))
    assert isinstance(out, tuple) and len(out) == 1
    _close(out[0], g["out"], "gan")


def test_forward_vae_kld_matches_pieces(cuda_device):
    g = GOLD["tutorial"]
    net = _net(g["kwargs"])
    x, seg = g["x"].cuda(), _seg(g)
    with torch.no_grad():
        torch.manual_seed(7)
        img, kld = net(seg, x)
        mu, logvar = net.encoder(x)
        torch.manual_seed(7)
        eps = torch.randn_like(mu)
        want_kld = SO.kld(mu.double(), logvar.double())
        z = eps * torch.exp(0.5 * logvar) + mu
        want = net.decode(seg, z)
    assert abs(kld.item() - want_kld.item()) <= 1e-5 * abs(want_kld.item())
    _close(img, want, "forward vs decode(encode)")


def test_repeat_calls_bit_identical(cuda_device):
    g = GOLD["tutorial"]
    net = _net(g["kwargs"])
    seg, z, x = _seg(g), g["z"].cuda(), g["x"].cuda()
    with torch.no_grad():
        a, b = net.decode(seg, z), net.decode(seg, z)
        m1, m2 = net.encoder(x), net.encoder(x)
        k1 = ops.vae_reparam_kld(m1[0], m1[1], z)[1]
        k2 = ops.vae_reparam_kld(m2[0], m2[1], z)[1]
    assert torch.equal(a, b) and torch.equal(m1[0], m2[0]) and torch.equal(m1[1], m2[1]) and torch.equal(k1, k2)


@pytest.mark.parametrize("name", ["tutorial", "bicubic", "gan"])
def test_graph_replay_equals_eager(cuda_device, name):
    g = GOLD[name]
    net = _net(g["kwargs"])
    seg = _seg(g)
    args = (seg,) if name == "gan" else (seg, g["z"].cuda())
    with torch.no_grad():
        eager = net.decoder(*args)
        gd = graphed(net.decoder)
        first = gd(*args)
        second = gd(*args)
    assert torch.equal(first, eager) and torch.equal(second, eager)


# ---- b200_upsample2x_interp ---------------------------------------------------------------------------------------
def _ulp16(x):
    mant = 10 if FP16 else 7
    tiny = 2.0 ** -24 if FP16 else 2.0 ** -133
    e = torch.floor(torch.log2(x.abs().clamp_min(tiny)))
    return torch.maximum(torch.exp2(e - mant), torch.full_like(x, tiny))


@pytest.mark.parametrize("mode", ["bilinear", "bicubic"])
@pytest.mark.parametrize("shape", [(2, 13, 1, 1), (1, 24, 5, 7), (3, 64, 32, 48), (1, 8, 1, 9)])
def test_upsample2x_interp_vs_interpolate(cuda_device, mode, shape):
    torch.manual_seed(0)
    x = torch.randn(shape, device="cuda") * 3
    a = ops.to_cl(x)
    want = F.interpolate(ops.from_cl(a), scale_factor=2, mode=mode, align_corners=False)   # same h16 input, fp32
    out = ops.upsample2x_interp(a, mode)
    got = ops.from_cl(out)
    # one h16 ulp, plus the fp32 rounding of a different summation order: where the (partly negative) bicubic taps
    # cancel, that exceeds the ulp of a near-zero result (about 2^-23 * max |x| measured against torch's CPU kernel)
    tol = _ulp16(want) + 2.0 ** -21 * x.abs().max()
    assert (got - want).abs().le(tol).all(), f"{mode} {shape}: max err {(got - want).abs().max():.3g}"
    assert out.t[..., a.C:].eq(0).all(), "pad channels must stay zero"


def test_upsample2x_interp_rejects(cuda_device):
    a = ops.to_cl(torch.randn(1, 8, 2, 4, 4, device="cuda"))
    with pytest.raises(NotImplementedError):
        ops.upsample2x_interp(a, "bilinear")
    with pytest.raises(ValueError):
        ops.upsample2x_interp(ops.to_cl(torch.randn(1, 8, 4, 4, device="cuda")), "trilinear")


# ---- LeakyReLU(0.2) on every igemm store path ------------------------------------------------------------------
def _leaky02(c):
    swap = lambda a: ACT_LEAKYRELU02 if a not in (ACT_NONE, ACT_GEGLU) else a
    return replace(c, name=c.name + "_leaky02", act1=swap(c.act1), act2=swap(c.act2))


LEAKY_CASES = [_leaky02(c) for c in CASES if {c.act1, c.act2} - {ACT_NONE, ACT_GEGLU}]


@pytest.mark.parametrize("case", LEAKY_CASES, ids=[c.name for c in LEAKY_CASES])
def test_igemm_leakyrelu02_matches_emulator(cuda_device, lib, case, monkeypatch):  # noqa: F811
    SO.patch_emulator(monkeypatch)
    run_case(lib, case)


# ---- SPADE modulation and GroupNorm apply with the new activation ----------------------------------------------
@pytest.mark.parametrize("C_", [16, 12])              # 16: the 8-channel vector kernels, 12: the scalar ones
def test_spade_apply_and_groupnorm_leakyrelu02(cuda_device, C_):
    torch.manual_seed(1)
    x = torch.randn(2, C_, 9, 11, device="cuda") * 2 + 0.5
    gb = torch.randn(2, 2 * C_, 9, 11, device="cuda")
    a, gbc = ops.to_cl(x), ops.to_cl(gb)
    xr, gr = ops.from_cl(a), ops.from_cl(gbc)
    aff = ops.groupnorm_affine(a, C_, 1e-5, None, None)
    gaff = ops.groupnorm_affine(gbc, 2 * C_, 1e-5, None, None)
    got = ops.from_cl(ops.spade_modulate(a, aff, gbc, gaff, act=ACT_LEAKYRELU02))
    want = F.leaky_relu(F.instance_norm(xr) * (1 + F.instance_norm(gr[:, :C_])) + F.instance_norm(gr[:, C_:]), 0.2)
    tol = 4 * _ulp16(want) + 1e-3
    assert (got - want).abs().le(tol).all(), f"spade_apply: max err {(got - want).abs().max():.3g}"

    one, zero = torch.ones(C_, device="cuda"), torch.zeros(C_, device="cuda")
    want = F.leaky_relu(F.group_norm(xr, 4 if C_ == 16 else 3, eps=1e-5), 0.2)
    for small in (True, False):                        # b200_groupnorm_fused and stats + b200_groupnorm_apply
        old = ops._GN_SMALL
        ops._GN_SMALL = small
        try:
            got = ops.from_cl(ops.groupnorm(a, 4 if C_ == 16 else 3, 1e-5, one, zero, act=ACT_LEAKYRELU02))
        finally:
            ops._GN_SMALL = old
        assert (got - want).abs().le(4 * _ulp16(want) + 1e-3).all(), f"groupnorm small={small}"
