"""Pin oracle/perceptual_oracle.py against the UNMODIFIED reference PerceptualLoss(network_type="resnet50") beyond
the fixture's cases (other ratios, weights from a file with and without a state-dict key, non-contiguous inputs), and
check the reference's module tree and errors that the package mirrors.  The reference imports offline through the stub
`lpips` of oracle/monai_shim.  Runs only where the reference tree exists."""
import sys

import pytest
import torch

from generativemodels_b200.losses import PerceptualLoss
from oracle import perceptual_oracle as O
from oracle import ref_import
from tests import golden
from tests.golden import make_golden_perceptual as G

pytestmark = pytest.mark.skipif(not ref_import.available(), reason="the reference checkout is not present")
FIX = golden.load("g_perceptual") if ref_import.available() else None


@pytest.fixture(scope="module")
def ref():
    """The reference's `generative.losses` for this module only (see tests/test_metrics_oracle_vs_reference.py)."""
    saved = {k: v for k, v in sys.modules.items() if k == "generative" or k.startswith("generative.")}
    for k in saved:
        del sys.modules[k]
    path, meta = list(sys.path), list(sys.meta_path)
    sys.meta_path[:] = [f for f in meta if type(f).__name__ != "_AliasFinder"]
    ref_import.import_reference()
    if str(ref_import._SHIM) not in sys.path:
        sys.path.insert(0, str(ref_import._SHIM))
    import generative.losses as gl
    yield gl
    for k in [k for k in sys.modules if k == "generative" or k.startswith("generative.")]:
        del sys.modules[k]
    sys.modules.update(saved)
    sys.path[:] = path
    sys.meta_path[:] = meta


@pytest.fixture(scope="module")
def net():
    return G.network(FIX)


def _ref(gl, net, dims, **kw):
    m = gl.PerceptualLoss(spatial_dims=dims, network_type="resnet50", pretrained=False, **kw)
    m.load_state_dict(G.loss_state_dict(net))
    return m.eval()


@pytest.mark.parametrize("ratio", [0.25, 1.0])
def test_fake3d_ratios(ref, net, ratio):
    x, y = G.inputs("fake3d")
    m = _ref(ref, net, 3, is_fake_3d=True, fake_3d_ratio=ratio)
    with torch.no_grad():
        torch.manual_seed(11)
        want = float(m(x.clone(), y.clone()))
        torch.manual_seed(11)
        got = float(O.loss(net, x, y, 3, ratio))
    assert abs(got - want) <= 1e-5 * abs(want)


def test_non_contiguous_and_three_channels(ref, net):
    torch.manual_seed(2)
    base = torch.rand(2, 3, 40, 56)
    x = base.transpose(2, 3)                      # [2, 3, 56, 40], strided
    y = (base + 0.05 * torch.randn_like(base)).transpose(2, 3)
    m = _ref(ref, net, 2)
    x0 = x.clone()
    with torch.no_grad():
        got = float(O.loss(net, x, y, 2))
        assert torch.equal(x, x0)                 # the oracle works on copies
        want = float(m(x, y))
    assert abs(got - want) <= 1e-5 * abs(want)
    assert not torch.equal(x, x0)                 # the reference's z-score wrote into its argument


def test_pretrained_path(ref, net, tmp_path):
    sd = net.state_dict()
    torch.save(sd, tmp_path / "plain.pt")
    torch.save({"model": sd}, tmp_path / "keyed.pt")
    x, y = G.inputs("odd")
    for path, key in ((tmp_path / "plain.pt", None), (tmp_path / "keyed.pt", "model")):
        kw = dict(pretrained=True, pretrained_path=str(path), pretrained_state_dict_key=key)
        m = ref.PerceptualLoss(spatial_dims=2, network_type="resnet50", **kw).eval()
        ours = PerceptualLoss(2, "resnet50", **kw)
        assert list(m.state_dict()) == list(ours.state_dict())
        for k, v in m.state_dict().items():
            assert torch.equal(ours.state_dict()[k], v), k
        with torch.no_grad():
            want = float(m(x.clone(), y.clone()))
            assert abs(float(O.loss(net, x, y, 2)) - want) <= 1e-5 * abs(want)
    ours.load_state_dict(m.state_dict(), strict=True)


def test_reference_errors(ref):
    with pytest.raises(NotImplementedError):
        ref.PerceptualLoss(spatial_dims=1, network_type="resnet50", pretrained=False)
    with pytest.raises(ValueError):
        ref.PerceptualLoss(spatial_dims=2, network_type="medicalnet_resnet10_23datasets")
    m = ref.PerceptualLoss(spatial_dims=2, network_type="resnet50", pretrained=False).eval()
    with pytest.raises(ValueError):
        m(torch.rand(1, 1, 32, 32), torch.rand(1, 1, 32, 33))
    with pytest.raises(IndexError):            # one input with one channel, the other with three: no repeat
        m.perceptual_function(torch.rand(1, 1, 32, 32), torch.rand(1, 3, 32, 32))
    with pytest.raises(RuntimeError, match="lpips"):
        ref.PerceptualLoss(spatial_dims=2, network_type="alex", pretrained=False)
