"""CPU checks of PerceptualLoss(network_type="resnet50"): the torch oracle against the reference's outputs in
tests/golden/g_perceptual.pt; the float64 reading of include/b200gen_perceptual.h (tests/perceptual_emulator.py)
against float64 torch and against mutants of the contract; the host code (argument rules, the reference's exceptions,
the slice draws, the ResNet-50 wiring) end to end on the CPU stand-in of the C ABI (tests/perceptual_backend.py); and
agreement between the perceptual header, its bindings and the stand-in."""
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from generativemodels_b200 import _lib
from generativemodels_b200.losses import PerceptualLoss, TorchvisionModelPerceptualSimilarity
from generativemodels_b200.losses import perceptual as P
from oracle import perceptual_oracle as O
from tests import golden, perceptual_backend
from tests import perceptual_checks as K
from tests import perceptual_emulator as E
from tests.golden import make_golden_perceptual as G

ROOT = Path(__file__).resolve().parents[1]
FIX = golden.load("g_perceptual")
CASES_2D = ["2d_1ch", "2d_3ch", "odd"]


@pytest.fixture
def cpu(monkeypatch):
    perceptual_backend.install(monkeypatch)


@pytest.fixture(scope="module")
def nets():
    return K.networks(FIX), K.networks(FIX, spatial_dims=3, is_fake_3d=True, fake_3d_ratio=0.5)


def oracle_loss(net, name, order=(2, 3, 4)):
    rec = FIX[name]
    with torch.no_grad():
        if name != "fake3d":
            return float(O.loss(net, rec["x"], rec["y"], 2))
        torch.manual_seed(G.SLICE_SEED)
        means = {}
        for axis in order:
            xs, ys = O.slices(rec["x"], axis), O.slices(rec["y"], axis)
            idx = torch.randperm(xs.shape[0])[: int(xs.shape[0] * 0.5)]
            means[axis] = torch.mean(O.similarity(net, xs[idx], ys[idx]))
        return float(torch.mean(means[2] + means[4] + means[3]))


@pytest.mark.parametrize("name", [*CASES_2D, "fake3d"])
def test_oracle_matches_fixture(nets, name):
    net = nets[0][1]
    want = float(FIX[name]["loss"])
    assert abs(oracle_loss(net, name) - want) <= 1e-5 * want
    if name != "fake3d":
        with torch.no_grad():
            got = O.similarity(net, FIX[name]["x"], FIX[name]["y"])
        torch.testing.assert_close(got, FIX[name]["per_image"], rtol=1e-5, atol=0)


def test_mutant_randperm_axis_order(nets):
    """Drawing the slices in another axis order selects other slices: far outside the oracle's 1e-5."""
    want = float(FIX["fake3d"]["loss"])
    assert abs(oracle_loss(nets[0][1], "fake3d", order=(2, 4, 3)) - want) > 100 * 1e-5 * want


def test_fixture_features(nets):
    net = nets[0][1]
    with torch.no_grad():
        f = O.features(net, O.zscore(FIX["2d_1ch"]["x"].repeat(1, 3, 1, 1)))
    torch.testing.assert_close(f, FIX["2d_1ch"]["features"], rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------
# the float64 reading of the contract
# ---------------------------------------------------------------------------------------------------------------
def test_prep_reading_matches_float64_torch():
    torch.manual_seed(0)
    for C in (1, 3):
        x = torch.rand(2, C, 7, 5)
        exact = O.zscore(x.double().repeat(1, 3 // C, 1, 1))
        # the contract's constants are the fp32 values of the reference's Python floats
        torch.testing.assert_close(E.prep(x, torch.float64), exact, rtol=0, atol=8 * E.U)
        torch.testing.assert_close(E.prep(x).double(), exact, rtol=0, atol=16 * E.U)


def test_prep_gather_matches_reference_slices():
    """The 2.5-D gather of the reading is the reference's batchify_axis; swapping the two remaining axes is not."""
    torch.manual_seed(1)
    v = torch.rand(2, 1, 6, 5, 4)
    idx = torch.tensor([7, 0, 3])
    for axis in (2, 3, 4):
        rest = [a for a in (2, 3, 4) if a != axis]
        src = v.permute(0, 1, axis, *rest)
        got = E.gather(src, v.shape[axis], idx)
        assert torch.equal(got, O.slices(v, axis)[idx])
        swapped = E.gather(v.permute(0, 1, axis, rest[1], rest[0]), v.shape[axis], idx)
        assert swapped.shape != got.shape          # extents 6, 5, 4: H and W never match
    # equal remaining extents: the swap keeps the shape, and the values differ
    c = torch.rand(1, 1, 3, 5, 5)
    pick = torch.tensor([2, 0])
    got = E.gather(c, 3, pick)
    assert torch.equal(got, O.slices(c, 2)[pick])
    swapped = E.gather(c.permute(0, 1, 2, 4, 3), 3, pick)
    assert swapped.shape == got.shape and not torch.equal(swapped, got)


def _features(B=2, HW=12, C=2048, noise=0.01, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(B, HW, C, generator=g)) * torch.rand(B, HW, 1, generator=g) * 3
    return x, x + noise * x.abs() * torch.randn(B, HW, C, generator=g)


def test_distance_reading_matches_float64_torch():
    x, y = _features()
    want = ((O.normalize(x.double().transpose(1, 2)) - O.normalize(y.double().transpose(1, 2))) ** 2).sum(1).mean(1)
    torch.testing.assert_close(E.distance(x, y), want, rtol=1e-12, atol=0)
    assert torch.equal(E.distance(x, x), torch.zeros(2, dtype=torch.float64))


def _direct32(x, y, eps_inside=False):
    x, y = x.float(), y.float()
    if eps_inside:
        nx, ny = (t.pow(2).sum(-1, keepdim=True).add(E.EPS32).sqrt() for t in (x, y))
        return (x / nx - y / ny).pow(2).sum(-1).double().mean(1)
    nx, ny = (t.pow(2).sum(-1, keepdim=True).sqrt() + E.EPS32 for t in (x, y))
    return (x / nx - y / ny).pow(2).sum(-1).double().mean(1)


def _expanded32(x, y):
    x, y = x.float(), y.float()
    nx, ny = (t.pow(2).sum(-1, keepdim=True).sqrt() + E.EPS32 for t in (x, y))
    a, b = x / nx, y / ny
    return (a.pow(2).sum(-1) + b.pow(2).sum(-1) - 2 * (a * b).sum(-1)).double().mean(1)


def test_distance_bound_holds_for_fp32_and_rejects_mutants():
    for noise in (0.0, 0.01, 0.2):
        x, y = _features(noise=noise)
        tol = E.distance_bound(x, y)
        assert bool(((_direct32(x, y) - E.distance(x, y)).abs() <= tol).all())
    x, y = _features(noise=0.01)
    err = (_expanded32(x, y) - E.distance(x, y)).abs() / E.distance_bound(x, y)
    assert float(err.max()) > 10, float(err.max())
    # features of a norm near the epsilon: eps inside the square root changes every normalised vector
    x, y = _features(noise=0.5)
    x, y = x * 1e-12, y * 1e-12
    err = (_direct32(x, y, eps_inside=True) - E.distance(x, y)).abs() / E.distance_bound(x, y)
    assert float(err.min()) > 1e3, float(err.min())


def test_mean_reading():
    img = torch.tensor([1.0, 2.0, 3.0, 4.0, 5.0, 6.0], dtype=torch.float64)
    assert E.mean(img, [2, 3, 1]).tolist() == [1.5, 4.0, 6.0, 11.5]


# ---------------------------------------------------------------------------------------------------------------
# the host code on the stand-in
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["2d_1ch", "odd", "fake3d"])
def test_stand_in_within_bound(cpu, nets, name):
    (m2, net), (m3, _) = nets
    rec = FIX[name]
    m = m3 if name == "fake3d" else m2
    with torch.no_grad():
        torch.manual_seed(G.SLICE_SEED)
        got = float(m(rec["x"], rec["y"]))
        if name == "fake3d":
            torch.manual_seed(G.SLICE_SEED)
            xs, ys = [], []
            for axis in (2, 3, 4):
                n = rec["x"].shape[0] * rec["x"].shape[axis]
                idx = torch.randperm(n)[: int(n * 0.5)]
                xs.append(O.slices(rec["x"], axis)[idx])
                ys.append(O.slices(rec["y"], axis)[idx])
            d = max(K.delta(K.product_features(m), K.oracle_features(net), a, b) for a, b in zip(xs, ys))
        else:
            d = K.delta(K.product_features(m), K.oracle_features(net), rec["x"], rec["y"])
    want = float(rec["loss"])
    assert d <= K.DELTA_MAX, d
    assert abs(got - want) <= K.loss_bound(want), (got, want, d)
    if K.LOSS_REL_TOL is not None:
        assert abs(got - want) <= K.LOSS_REL_TOL * want, (got, want)


def test_wiring_mutants_fall_outside_every_tolerance(nets):
    """The fixture network tells a mis-wired ResNet-50 from the right one: each wiring mutant's features, delta and
    loss against the reference's lie outside the tolerances the product is held to (by 3x at least)."""
    net = nets[0][1]
    rec = FIX["2d_1ch"]
    z = O.zscore(rec["x"].repeat(1, 3, 1, 1))
    f0 = rec["features"]
    for name, mut in G.wiring_mutants(net):
        with torch.no_grad():
            f = O.features(mut, z)
            d = K.delta(K.oracle_features(mut), K.oracle_features(net), rec["x"], rec["y"])
            loss = float(O.loss(mut, rec["x"], rec["y"], 2))
        rel = float((f - f0).norm() / f0.norm())
        assert rel > 3 * K.FEATURE_TOL[0], (name, rel)
        assert d > 3 * K.DELTA_MAX, (name, d)
        if K.LOSS_REL_TOL is not None:
            assert abs(loss - float(rec["loss"])) > 3 * K.LOSS_REL_TOL * float(rec["loss"]), (name, loss)


def test_identical_inputs_and_no_mutation(cpu, nets):
    m = nets[0][0]
    x = FIX["2d_3ch"]["x"].clone()
    x0 = x.clone()
    with torch.no_grad():
        assert float(m(x, x)) == 0.0
        m(x, FIX["2d_3ch"]["y"])
        out = m.perceptual_function(x, FIX["2d_3ch"]["y"])
    assert torch.equal(x, x0)
    assert out.shape == (2, 1, 1, 1) and out.dtype == torch.float32


def test_chunking_does_not_change_the_result(cpu, nets, monkeypatch):
    m = nets[1][0]
    rec = FIX["fake3d"]
    with torch.no_grad():
        torch.manual_seed(3)
        a = m(rec["x"], rec["y"])
        monkeypatch.setattr(P, "_CHUNK_PIXELS", 2 * 48 * 36 * 3)
        torch.manual_seed(3)
        b = m(rec["x"], rec["y"])
    assert torch.equal(a, b)


def test_forward_only_and_mode_rules(cpu, nets):
    m = nets[0][0]
    x = FIX["2d_1ch"]["x"].clone().requires_grad_(True)
    with pytest.raises(RuntimeError, match="forward only"):
        m(x, FIX["2d_1ch"]["y"])
    with torch.no_grad():
        m(x, FIX["2d_1ch"]["y"])
    m.train()
    try:
        with pytest.raises(RuntimeError, match="eval"):
            with torch.no_grad():
                m(FIX["2d_1ch"]["x"], FIX["2d_1ch"]["y"])
    finally:
        m.eval()


def test_shape_and_channel_errors(cpu, nets):
    m = nets[0][0]
    with pytest.raises(ValueError, match="differing shape"):
        m(torch.rand(1, 1, 32, 32), torch.rand(1, 1, 32, 33))
    with torch.no_grad(), pytest.raises(ValueError):
        m.perceptual_function(torch.rand(1, 1, 32, 32), torch.rand(1, 3, 32, 32))   # the reference: IndexError
    with torch.no_grad(), pytest.raises(ValueError):
        m(torch.rand(1, 2, 32, 32), torch.rand(1, 2, 32, 32))


def test_load_state_dict_repacks(cpu, nets):
    m = K.networks(FIX)[0]
    rec = FIX["odd"]
    with torch.no_grad():
        a = float(m(rec["x"], rec["y"]))
        sd = m.state_dict()
        sd["perceptual_function.model.layer4.2.bn3.weight"] = sd["perceptual_function.model.layer4.2.bn3.weight"] * 3
        m.load_state_dict(sd)
        b = float(m(rec["x"], rec["y"]))
    assert a != b


def test_constructor_errors():
    with pytest.raises(NotImplementedError, match="only in 2D and 3D"):
        PerceptualLoss(1, "resnet50", pretrained=False)
    with pytest.raises(ValueError, match="MedicalNet"):
        PerceptualLoss(2, "medicalnet_resnet10_23datasets")
    with pytest.raises(ValueError, match="MedicalNet"):
        PerceptualLoss(3, "medicalnet_resnet10_23datasets", is_fake_3d=True)
    for args, kw in (((2,), {}), ((2, "vgg"), {}), ((2, "squeeze"), {}), ((2, "radimagenet_resnet50"), {}),
                     ((3, "medicalnet_resnet10_23datasets"), {"is_fake_3d": False}),
                     ((3, "resnet50"), {"is_fake_3d": False})):
        with pytest.raises(NotImplementedError, match="resnet50"):
            PerceptualLoss(*args, **kw)
    with pytest.raises(NotImplementedError, match="resnet50"):
        TorchvisionModelPerceptualSimilarity(net="vgg")


def test_pretrained_path(tmp_path):
    net = G.network(FIX)
    sd = {k: v for k, v in net.state_dict().items()}
    torch.save(sd, tmp_path / "plain.pt")
    torch.save({"state": sd}, tmp_path / "keyed.pt")
    for path, key in ((tmp_path / "plain.pt", None), (tmp_path / "keyed.pt", "state")):
        m = PerceptualLoss(2, "resnet50", pretrained=True, pretrained_path=str(path), pretrained_state_dict_key=key)
        for k, v in G.loss_state_dict(net).items():
            assert torch.equal(m.state_dict()[k], v), k


def test_state_dict_keys():
    m = PerceptualLoss(2, "resnet50", pretrained=False)
    keys = list(m.state_dict())
    assert len(keys) == 318
    assert keys[0] == "perceptual_function.model.conv1.weight"
    assert keys[-1] == "perceptual_function.model.layer4.2.bn3.num_batches_tracked"
    assert not any(p.requires_grad for p in m.parameters())


def test_header_bindings_and_stand_in_agree():
    header = (ROOT / "include" / "b200gen_perceptual.h").read_text()
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_lib.PERCEPTUAL_SIGNATURES)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name)
        assert callable(getattr(perceptual_backend.PerceptualFakeLib, name, None)), name
