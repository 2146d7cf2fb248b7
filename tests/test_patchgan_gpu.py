"""PatchDiscriminator / MultiScalePatchDiscriminator on the H100 kernels: every case of the reference fixture
(tests/golden/g_patchgan.pt), scores and every intermediate feature; b200_pool_s2 against F.avg_pool / F.max_pool;
b200_batchnorm_fold against a float64 evaluation of its formula; new running statistics after load_state_dict; repeat
calls and CUDA-graph replays bit for bit; random small configurations against tests/patchgan_oracle.py."""
import random

import pytest
import torch
import torch.nn.functional as F

from generativemodels_b200 import ops
from generativemodels_b200.cuda_graph import graphed
from generativemodels_b200.networks.nets.patchgan_discriminator import MultiScalePatchDiscriminator, PatchDiscriminator
from tests import patchgan_oracle as PO
from tests.golden import load

pytestmark = pytest.mark.gpu

GOLD = load("g_patchgan")
CLASSES = {"PatchDiscriminator": PatchDiscriminator, "MultiScalePatchDiscriminator": MultiScalePatchDiscriminator}
FP16 = ops.H16 is torch.float16


def _flat(t):
    return [u for v in t for u in _flat(v)] if isinstance(t, (list, tuple)) else [t]


def _close(got, want, what, tol=(2e-2, 4e-2)):
    got, want = got.double().cpu(), want.double().cpu()
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(want.shape)}"
    rel = ((got - want).norm() / want.norm()).item()
    mx = ((got - want).abs().max() / want.abs().max()).item()
    assert rel < tol[0] and mx < tol[1], f"{what}: rel L2 {rel:.3e}, normalised max-abs {mx:.3e}"


def _tol(feats):
    """The project's bound, except in the bf16 flavour for a discriminator whose deepest layers normalise 4 voxels or
    fewer (the 2d_spade_vae tutorial's second one: 2 x 2): bf16 keeps 8 significant bits, and InstanceNorm over so few
    voxels amplifies their rounding (measured up to 3e-2 rel L2 / 1e-1 normalised max-abs on an H100)."""
    few = min(f[0, 0].numel() for f in feats) <= 4
    return (6e-2, 2e-1) if few and not FP16 else (2e-2, 4e-2)


def _check_case(name, g, scores, feats, want_feats):
    """Scores against the fixture, features against ``want_feats``, one discriminator at a time."""
    if g["cls"] == "PatchDiscriminator":
        scores, feats, want_scores, want_feats = [scores], [feats], [g["scores"]], [want_feats]
    else:
        want_scores = g["scores"]
    for d, (s, f, ws, wf) in enumerate(zip(scores, feats, want_scores, want_feats, strict=True)):
        tol = _tol(wf)
        assert s.dtype == torch.float32
        _close(s, ws, f"{name} discriminator {d} scores", tol)
        for i, (got, want) in enumerate(zip(f, wf, strict=True)):
            _close(got, want, f"{name} discriminator {d} feature {i}", tol)


def _split(cls_name, out):
    """(scores, features) of either class's forward."""
    return (out[-1], out[:-1]) if cls_name == "PatchDiscriminator" else out


def _oracle64(cls_name, kw, sd, x):
    sd = {k: v.double().cuda() for k, v in sd.items() if v.is_floating_point()}
    with torch.no_grad():
        if cls_name == "PatchDiscriminator":
            o = PO.patch_discriminator(sd, x.double().cuda(), **kw)
            return o[-1], o[:-1]
        return PO.multiscale(sd, x.double().cuda(), **kw)


def _net(g, seed=0):
    return PO.seeded_weights(CLASSES[g["cls"]](**g["kwargs"]), seed).eval().cuda()


# ---- the networks against the reference fixture -----------------------------------------------------------------
@pytest.mark.parametrize("name", list(GOLD))
def test_fixture_case(cuda_device, name):
    g = GOLD[name]
    net = _net(g)
    x = PO.input_of(g).cuda()
    with torch.no_grad():
        scores, feats = _split(g["cls"], net(x))
    want_feats = g.get("features")
    if want_feats is None:            # features of the large inputs are not stored: the float64 oracle on the GPU
        want_feats = _oracle64(g["cls"], g["kwargs"], net.state_dict(), PO.input_of(g))[1]
    _check_case(name, g, scores, feats, want_feats)


def test_spade_vae_discriminator_runs_in_train_mode(cuda_device):
    g = GOLD["spade_vae"]
    net = PO.seeded_weights(MultiScalePatchDiscriminator(**g["kwargs"])).cuda()
    assert net.training
    with torch.no_grad():
        scores, feats = net(PO.input_of(g).cuda())
    _check_case("spade_vae (train mode)", g, scores, feats, g["features"])


# ---- b200_pool_s2 --------------------------------------------------------------------------------------------------
def _ulp16(x):
    mant = 10 if FP16 else 7
    tiny = 2.0 ** -24 if FP16 else 2.0 ** -133
    e = torch.floor(torch.log2(x.abs().clamp_min(tiny)))
    return torch.maximum(torch.exp2(e - mant), torch.full_like(x, tiny))


POOL_CASES = [(k, p, mode, shape) for k in (2, 3, 4) for p in range(k // 2 + 1) for mode in ("avg", "max")
              for shape in ((2, 13, 17, 22), (1, 16, 9, 10, 7), (1, 5, 8, 8))]


@pytest.mark.parametrize("k,p,mode,shape", POOL_CASES)
def test_pool_s2_vs_torch(cuda_device, k, p, mode, shape):
    torch.manual_seed(k * 10 + p)
    x = torch.randn(shape, device="cuda") * 3
    a = ops.to_cl(x)
    xr = ops.from_cl(a)                                          # the same h16 input, fp32
    nd = x.dim() - 2
    fn = {"avg": (F.avg_pool2d, F.avg_pool3d), "max": (F.max_pool2d, F.max_pool3d)}[mode][nd == 3]
    want = fn(xr, k, 2, p)
    out = ops.pool_s2(a, k, p, mode)
    got = ops.from_cl(out)
    assert got.shape == want.shape
    if mode == "max":
        assert torch.equal(got, want)
    else:
        # one h16 ulp, plus the fp32 rounding of a different summation order where the taps cancel to near zero
        err = (got - want).abs()
        assert err.le(_ulp16(want) + 2.0 ** -21 * x.abs().max()).all(), f"avg k{k} p{p} {shape}: max err {err.max():.3g}"
    assert out.t[..., a.C:].eq(0).all(), "pad channels must stay zero"


@pytest.mark.parametrize("nd", [2, 3])
def test_pool_s2_max_nan_and_inf(cuda_device, nd):
    shape = (1, 8, 9, 11) if nd == 2 else (1, 8, 5, 9, 11)
    x = torch.randn(shape, device="cuda")
    x.view(-1)[::37] = float("nan")
    x.view(-1)[5::41] = float("inf")
    x.view(-1)[7::43] = float("-inf")
    a = ops.to_cl(x)
    want = (F.max_pool2d if nd == 2 else F.max_pool3d)(ops.from_cl(a), 3, 2, 1)
    got = ops.from_cl(ops.pool_s2(a, 3, 1, "max"))
    assert torch.equal(got.isnan(), want.isnan()) and want.isnan().any()
    fin = ~want.isnan()
    assert torch.equal(got[fin], want[fin])


def test_pool_s2_rejects(cuda_device):
    a = ops.to_cl(torch.randn(1, 8, 4, 4, device="cuda"))
    with pytest.raises(ValueError):
        ops.pool_s2(a, 3, 2, "avg")                              # padding above half the kernel
    with pytest.raises(ValueError):
        ops.pool_s2(a, 3, 1, "lp")


# ---- b200_batchnorm_fold -------------------------------------------------------------------------------------------
def _ulp32(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 23)


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("shape", [(64, 32, 4, 4), (7, 3, 3, 3, 3), (256, 128, 4, 4, 4)])
def test_batchnorm_fold_vs_float64(cuda_device, shape, bias):
    g = torch.Generator().manual_seed(sum(shape))
    co = shape[0]
    w = torch.randn(shape, generator=g)
    b = torch.randn(co, generator=g) if bias else None
    gamma, beta, mean = 1 + 0.3 * torch.randn(co, generator=g), torch.randn(co, generator=g), torch.randn(co, generator=g)
    var = torch.rand(co, generator=g) * 2 + 1e-3
    eps = 1e-5
    w_out, b_out = ops.batchnorm_fold(*(None if t is None else t.cuda() for t in (w, b, gamma, beta, mean, var)), eps)
    s = gamma.double() / (var.double() + float(torch.tensor(eps, dtype=torch.float32))).sqrt()
    w_want = w.double() * s.view(-1, *[1] * (w.dim() - 1))
    b_want = beta.double() + ((b.double() if bias else 0.0) - mean.double()) * s
    for got, want in ((w_out.cpu(), w_want), (b_out.cpu(), b_want)):
        assert got.dtype == torch.float32 and got.shape == want.shape
        assert ((got.double() - want).abs() <= _ulp32(want.float()).double()).all()


# ---- load_state_dict, determinism, graphs ---------------------------------------------------------------------------
def test_load_state_dict_new_statistics_used(cuda_device):
    g = GOLD["ldm2d"]
    net = _net(g)
    x = PO.input_of(g).cuda()
    with torch.no_grad():
        before = net(x)[-1]
        sd = net.state_dict()
        sd["0.adn.N.running_var"] = sd["0.adn.N.running_var"] * 3
        sd["1.adn.N.running_mean"] = sd["1.adn.N.running_mean"] - 0.4
        sd["2.adn.N.weight"] = sd["2.adn.N.weight"] * 0.5
        net.load_state_dict(sd)
        after = net(x)[-1]
    want = _oracle64(g["cls"], g["kwargs"], net.state_dict(), x)[0]
    _close(after, want, "after load_state_dict")
    assert ((before - after).norm() / want.norm()).item() > 5e-2


@pytest.mark.parametrize("name", ["ldm2d", "spade_vae", "test_3d_pool"])
def test_repeat_and_graph_replay_bit_identical(cuda_device, name):
    g = GOLD[name]
    net = _net(g)
    x = PO.input_of(g).cuda()
    with torch.no_grad():
        a, b = _flat(net(x)), _flat(net(x))
        gd = graphed(net)
        first, second = _flat(gd(x)), _flat(gd(x))
    assert all(torch.equal(u, v) for u, v in zip(a, b, strict=True))
    assert all(torch.equal(u, v) for u, v in zip(a, first, strict=True))
    assert all(torch.equal(u, v) for u, v in zip(a, second, strict=True))


def _random_config(rng):
    sd = rng.choice([2, 3])
    k = rng.choice([2, 3, 4, 5]) if sd == 2 else rng.choice([3, 4])
    norm = rng.choice(["BATCH", "instance"])
    acts = ["LEAKYRELU", PO.LEAKY02, "SILU", None] + (["RELU", "GELU", "TANH", "SIGMOID"] if norm == "BATCH" else [])
    kw = dict(spatial_dims=sd, num_channels=rng.choice([4, 8, 12, 16]), in_channels=rng.choice([1, 3, 9]),
              out_channels=rng.choice([1, 2, 5]), kernel_size=k, activation=rng.choice(acts), norm=norm,
              bias=rng.choice([True, False]), dropout=rng.choice([0.0, 0.2]))
    if rng.random() < 0.5:
        kw.update(num_layers_d=rng.choice([1, 2]), padding=rng.choice([0, 1, (k - 1) // 2]),
                  last_conv_kernel_size=rng.choice([None, 1, 3]))
        return "PatchDiscriminator", kw
    kw.update(num_d=rng.choice([2, 3]), num_layers_d=1, pooling_method=rng.choice([None, "avg", "max"]),
              last_conv_kernel_size=rng.choice([1, 3]), minimum_size_im=32)
    return "MultiScalePatchDiscriminator", kw


@pytest.mark.parametrize("seed", range(12))
def test_random_configs_vs_oracle(cuda_device, seed):
    rng = random.Random(seed)
    while True:                       # draw until the reference would accept the shapes (no empty layer, no 1-voxel
        cls_name, kw = _random_config(rng)      # InstanceNorm)
        n = rng.choice([1, 2])
        lo, hi = (40, 64) if kw["spatial_dims"] == 2 else (24, 40)
        x = torch.randn((n, kw["in_channels"], *[rng.randrange(lo, hi) for _ in range(kw["spatial_dims"])]),
                        generator=torch.Generator().manual_seed(seed))
        net = PO.seeded_weights(CLASSES[cls_name](**kw), seed).eval().cuda()
        try:
            want_scores, want_feats = _oracle64(cls_name, kw, net.state_dict(), x)
            break
        except (RuntimeError, ValueError):
            continue
    with torch.no_grad():
        scores, feats = _split(cls_name, net(x.cuda()))
    for i, (got, want) in enumerate(zip(_flat([scores, feats]), _flat([want_scores, want_feats]), strict=True)):
        _close(got, want, f"{cls_name} {kw} output {i}")
