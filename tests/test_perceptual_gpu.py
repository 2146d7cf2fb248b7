"""GPU checks of PerceptualLoss(network_type="resnet50") on the H100 kernels: b200_perceptual_prep bit-exact against
the float64 reading of include/b200gen_perceptual.h (tests/perceptual_emulator.py), b200_perceptual_distance within
its bound on the device's own features, the ResNet-50 features within the network tolerance of the reference's fp32
features, the loss within 2 sqrt(L_ref) delta + delta^2 of the reference (delta measured against the torchvision
oracle in fp32 on the same card), and the determinism the module promises: loss(x, x) == 0, repeated calls and slice
chunk sizes bit-identical.  Prints the measured delta and err / tol per case."""
import pytest
import torch

from generativemodels_b200 import ops
from generativemodels_b200.losses import perceptual as P
from oracle import perceptual_oracle as O
from tests import golden
from tests import perceptual_checks as K
from tests import perceptual_emulator as E
from tests.fixture_checks import close
from tests.golden import make_golden_perceptual as G

pytestmark = pytest.mark.gpu
FIX = golden.load("g_perceptual")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device in this container")
    torch.backends.cudnn.allow_tf32 = False          # the oracle in fp32, as the reference computes
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def nets(dev):
    return K.networks(FIX, dev), K.networks(FIX, dev, spatial_dims=3, is_fake_3d=True, fake_3d_ratio=0.5)


def _prep_case(x, y, S, OH, OW, idx, n, strides):
    out = torch.empty((2 * n, 1, OH, OW, 8), dtype=ops.H16, device=x.device)
    ops.perceptual_prep(x, y, strides, S, OH, OW, idx, n, out)
    return out.cpu()


def _expect(t5, S, idx):
    z = E.prep(E.gather(t5.cpu(), S, None if idx is None else idx.cpu()))
    o = torch.zeros(z.shape[0], 1, *z.shape[2:], 8, dtype=ops.H16)
    o[..., :3] = z.permute(0, 2, 3, 1).unsqueeze(1).to(ops.H16)
    return o


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.float64])
def test_prep_bit_exact(dev, dtype):
    g = torch.Generator().manual_seed(0)
    # 2-D: one channel (repeated), three channels as a non-contiguous view
    for C in (1, 3):
        base = torch.rand(3, 4, C, 21, 17, generator=g).to(dtype).to(dev)
        x, y = base[:, 1].transpose(-1, -2), base[:, 2].transpose(-1, -2)       # [3, C, 17, 21], strided
        st = [(s[0], s[1], 0, s[2], s[3]) for s in (x.stride(), y.stride())]
        got = _prep_case(x, y, 1, 17, 21, None, 3, st)
        for k, t in enumerate((x, y)):
            assert torch.equal(got[3 * k:3 * k + 3].view(torch.int16), _expect(t.unsqueeze(2), 1, None).view(torch.int16))
    # 2.5-D: a slice set along every axis, picked by a permutation
    v = torch.rand(2, 1, 11, 9, 7, generator=g).to(dtype).to(dev)
    w = torch.rand(2, 1, 11, 9, 7, generator=g).to(dtype).to(dev)
    for axis in (2, 3, 4):
        rest = [a for a in (2, 3, 4) if a != axis]
        n = 2 * v.shape[axis]
        idx = torch.randperm(n, generator=g)[: n // 2].to(dev)
        st = [(s[0], s[1], s[axis], s[rest[0]], s[rest[1]]) for s in (v.stride(), w.stride())]
        got = _prep_case(v, w, v.shape[axis], v.shape[rest[0]], v.shape[rest[1]], idx, n // 2, st)
        for k, t in enumerate((v, w)):
            want = _expect(t.permute(0, 1, axis, *rest), t.shape[axis], idx)
            assert torch.equal(got[k * (n // 2):(k + 1) * (n // 2)].view(torch.int16), want.view(torch.int16))
            assert torch.equal(want[..., :3].float().permute(0, 4, 2, 3, 1)[..., 0],
                               E.prep(O.slices(t.cpu(), axis)[idx.cpu()]).to(ops.H16).float())


@pytest.mark.parametrize("storage", ["f32", "h16"])
def test_distance_within_bound(dev, nets, storage):
    m = nets[0][0]
    rec = FIX["2d_1ch"]
    with torch.no_grad():
        z = O.zscore(torch.cat([rec["x"], rec["y"]]).repeat(1, 3, 1, 1)).to(dev)
        f = m.perceptual_function.model.forward_cl(ops.to_cl(z))
    if storage == "h16":
        f = f.to(ops.H16)
    B = rec["x"].shape[0]
    image = torch.empty(B, dtype=torch.float64, device=dev)
    ops.perceptual_distance(f[:B], f[B:], 2048, image)
    fx, fy = (t.reshape(B, -1, 2048).cpu() for t in (f[:B], f[B:]))
    want, tol = E.distance(fx, fy), E.distance_bound(fx, fy)
    err = (image.cpu() - want).abs()
    print(f"\n[perceptual] distance ({storage}): max err/tol {float((err / tol).max()):.3e}")
    assert bool((err <= tol).all()), (err, tol)
    ops.perceptual_distance(f[:B], f[:B], 2048, image)
    assert bool((image == 0).all())


def test_features_match_reference(dev, nets):
    m = nets[0][0]
    x = FIX["2d_1ch"]["x"]
    with torch.no_grad():
        f = m.perceptual_function.model(O.zscore(x.repeat(1, 3, 1, 1)).to(dev))["layer4.2.relu_2"]
    r, mx = close(f, FIX["2d_1ch"]["features"], "layer4.2.relu_2", *K.FEATURE_TOL)
    print(f"\n[perceptual] features: rel-L2 {r:.3e}, normalised max-abs {mx:.3e} (tol {K.FEATURE_TOL})")


@pytest.mark.parametrize("name", ["2d_1ch", "2d_3ch", "odd", "fake3d"])
def test_loss_within_bound(dev, nets, name):
    (m2, net), (m3, _) = nets
    rec = FIX[name]
    x, y = rec["x"].to(dev), rec["y"].to(dev)
    with torch.no_grad():
        if name == "fake3d":
            torch.manual_seed(G.SLICE_SEED)
            got = float(m3(x, y))
            torch.manual_seed(G.SLICE_SEED)
            d = 0.0
            for axis in (2, 3, 4):
                n = x.shape[0] * x.shape[axis]
                idx = torch.randperm(n)[: int(n * 0.5)].to(dev)
                d = max(d, K.delta(K.product_features(m2), K.oracle_features(net), O.slices(x, axis)[idx],
                                   O.slices(y, axis)[idx]))
        else:
            got = float(m2(x, y))
            d = K.delta(K.product_features(m2), K.oracle_features(net), x, y)
            per = m2.perceptual_function(x, y)
            assert per.shape == rec["per_image"].shape and per.dtype == torch.float32
    want = float(rec["loss"])
    tol = K.loss_bound(want)
    print(f"\n[perceptual] {name}: loss {got:.6e} ref {want:.6e} rel err {abs(got - want) / want:.3e} delta {d:.3e} "
          f"(max {K.DELTA_MAX:g}) err/tol {abs(got - want) / tol:.3e}")
    assert d <= K.DELTA_MAX
    assert abs(got - want) <= tol
    if K.LOSS_REL_TOL is not None:
        assert abs(got - want) <= K.LOSS_REL_TOL * want


def test_identity_repeats_and_chunks(dev, nets, monkeypatch):
    m2, m3 = nets[0][0], nets[1][0]
    x, y = FIX["2d_3ch"]["x"].to(dev), FIX["2d_3ch"]["y"].to(dev)
    x0 = x.clone()
    with torch.no_grad():
        assert float(m2(x, x)) == 0.0
        a, b = m2(x, y), m2(x, y)
        assert torch.equal(a, b) and torch.equal(x, x0)
        v, w = FIX["fake3d"]["x"].to(dev), FIX["fake3d"]["y"].to(dev)
        torch.manual_seed(5)
        assert float(m3(v, v)) == 0.0
        outs = []
        for pixels in (P._CHUNK_PIXELS, 2 * 48 * 36 * 3, 2 * 48 * 36 * 7):
            monkeypatch.setattr(P, "_CHUNK_PIXELS", pixels)
            torch.manual_seed(5)
            outs.append(m3(v, w))
        assert all(torch.equal(outs[0], o) for o in outs[1:]), [float(o) for o in outs]


def test_chunks_across_tile_choices(dev, nets, monkeypatch):
    """A volume whose slice sets are large enough that, left to the planner, layer3 / layer4's 3x3 convolutions would
    take the 128 x 256 kernel for one chunk and the 128-column one for another (and the 128-column kernel its 128- or
    64-column tile): the network pins the 128-column kernel, and chunks of 3 slices give the bits of one chunk per axis."""
    m3 = nets[1][0]
    g = torch.Generator(device=dev).manual_seed(1)
    v = torch.rand(2, 1, 96, 112, 80, device=dev, generator=g)
    w = (v + 0.05 * torch.randn(v.shape, device=dev, generator=g)).clamp(0, 1)
    outs = []
    with torch.no_grad():
        for pixels in (P._CHUNK_PIXELS, 2 * 112 * 96 * 3):
            monkeypatch.setattr(P, "_CHUNK_PIXELS", pixels)
            torch.manual_seed(9)
            outs.append(m3(v, w))
    assert torch.equal(outs[0], outs[1]), [float(o) for o in outs]
