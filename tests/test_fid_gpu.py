"""FID on the GPU: every case of tests/golden/g_fid.pt against its exact value and the reference's output, a sweep
against the float64 reading of b200_fid_moments / b200_frechet (tests/fid_emulator.py) over feature counts, row
counts, dtypes and strided views, the optional outputs, the analytic identities, bit-identical repeats, CUDA-graph
capture and NaN features.  Observed errors are printed relative to S = tr Sigma_p + tr Sigma_y + |mu_p - mu_y|^2."""
import numpy as np
import pytest
import torch

from generativemodels_b200 import metrics as GM
from generativemodels_b200 import ops
from tests import fid_emulator as M
from tests.golden import load
from tests.golden.make_golden_fid import CASES, checksum, features, inputs

pytestmark = pytest.mark.gpu
FIX = load("g_fid")
DEV = "cuda"
F64 = torch.float64
EPS = 2.0 ** -52


def scale(p, y):
    (mp, sp), (my, sy) = M.fid_moments(p.cpu()), M.fid_moments(y.cpu())
    return float(torch.trace(sp) + torch.trace(sy) + (mp - my) @ (mp - my))


# exact value: 1e-10 S everywhere; the reference: 1e-10 S where both covariances have full rank, 1e-7 S where its
# sqrtm of a singular product carries noise (2.0e-8 S observed at 1000 x 2048); the x 1e4 case, where the reference
# raises, against the exact value only
@pytest.mark.parametrize("name", list(CASES))
def test_fixture_case(cuda_device, name):
    case, rec = CASES[name], FIX[name]
    p, y = inputs(case)
    assert all(torch.equal(checksum(t), c) for t, c in zip((p, y), rec["checksum"]))
    got = GM.FIDMetric()(p.to(DEV), y.to(DEV))
    assert got.dim() == 0 and got.dtype == F64 and got.is_cuda
    e_exact = abs(float(got) - rec["exact"]) / rec["S"]
    e_ref = None if rec["error"] else abs(float(got) - float(rec["out"])) / rec["S"]
    print(f"{name}: |fid - exact| = {e_exact:.2e} S, |fid - reference| = "
          f"{'(reference raised)' if e_ref is None else f'{e_ref:.2e} S'}, S = {rec['S']:.4e}")
    assert e_exact <= 1e-10
    if e_ref is not None:
        assert e_ref <= (1e-7 if case["singular"] else 1e-10)


DTYPES = [torch.float32, torch.float64, torch.float16, torch.bfloat16]
SWEEP = [  # (F, n_pred, n_y, layout)
    (1, 5, 7, "dense"),
    (2, 2, 3, "dense"),
    (63, 40, 100, "transposed"),
    (1000, 300, 1200, "sliced"),
    (2047, 2, 500, "dense"),
    (2048, 10000, 2500, "dense"),
    (4096, 600, 200, "sliced"),
]


def _layout(x, layout):
    if layout == "transposed":      # feature stride 1 along rows: a [F, n] tensor seen as [n, F]
        return x.t().contiguous().t()
    if layout == "sliced":          # every other column of a wider buffer
        big = torch.zeros(x.shape[0], 2 * x.shape[1], dtype=x.dtype, device=x.device)
        big[:, 1::2] = x
        return big[:, 1::2]
    return x


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("i", range(len(SWEEP)))
def test_sweep_matches_the_contract(cuda_device, i, dtype):
    F, n_p, n_y, layout = SWEEP[i]
    if F >= 2047 and dtype != DTYPES[i % 4]:
        pytest.skip("the large feature counts run in one dtype each")
    p = features(n_p, F, 50 + i, shift=0.1).to(dtype)
    y = features(n_y, F, 60 + i).to(dtype)
    pd, yd = (_layout(t.to(DEV), layout) for t in (p, y))
    got, eig, rank = ops.frechet(*ops.fid_moments(pd), *ops.fid_moments(yd), details=True)
    (mp, sp), (my, sy) = M.fid_moments(p), M.fid_moments(y)
    want, weig, wrank = M.frechet(mp, sp, my, sy)
    S = scale(p, y)
    err = abs(float(got) - want) / S
    eig = eig.cpu().numpy()
    e_eig = np.abs(eig - weig).max()
    print(f"F={F} n={n_p}/{n_y} {dtype} {layout}: |fid - reading| = {err:.2e} S, rank {int(rank)} / {wrank}, "
          f"max |eig - eigvalsh| = {e_eig / max(weig[-1], 1e-300):.2e} mu_max")
    assert err <= 1e-8
    assert int(rank) == wrank
    assert np.all(np.diff(eig) >= 0)
    # F eps mu_max, and at least the few roundings of the two GEMMs that form a 1 x 1 or 2 x 2 M
    assert e_eig <= max(F, 4) * EPS * max(weig[-1], 0.0) + 1e-300


@pytest.mark.parametrize("layout", ["dense", "transposed", "sliced"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_moments_match_torch_cov(cuda_device, dtype, layout):
    x = features(700, 300, 5).to(dtype)
    mu, sigma = ops.fid_moments(_layout(x.to(DEV), layout))
    want = torch.cov(x.to(DEV, F64).T)
    err = (sigma - want).abs().max().item() / want.abs().max().item()
    assert err <= 1e-13, err
    assert torch.equal(sigma, sigma.T)
    assert (mu - x.to(DEV, F64).mean(0)).abs().max().item() <= 1e-13 * x.double().abs().max().item()


@pytest.mark.parametrize("n,F", [(60, 16), (12, 40), (3000, 2048)])
def test_analytic_identities(cuda_device, n, F):
    y = features(n, F, 7 + F).double().to(DEV)
    c, b = 0.5, torch.linspace(-1.0, 1.0, F, dtype=F64, device=DEV)
    p = c * y + b
    mu_y, s_y = M.fid_moments(y.cpu())
    d = (c - 1) * mu_y + b.cpu()
    want = float(d @ d + (1 - c) ** 2 * torch.trace(s_y))
    e_aff = abs(float(GM.FIDMetric()(p, y)) - want) / scale(p, y)
    e_id = abs(float(GM.FIDMetric()(y, y))) / scale(y, y)
    print(f"n={n} F={F}: affine copy {e_aff:.2e} S, identical sets {e_id:.2e} S")
    assert e_aff <= 1e-12 and e_id <= 1e-12


def test_repeat_calls_are_bit_identical(cuda_device):
    p, y = (t.to(DEV) for t in inputs(CASES["tutorial_1000x2048"]))
    assert torch.equal(GM.FIDMetric()(p, y), GM.FIDMetric()(p, y))


def test_cuda_graph_capture(cuda_device):
    p, y = (t.to(DEV) for t in inputs(CASES["singular_30x256_vs_40x256"]))
    m = GM.FIDMetric()
    eager = m(p, y)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m(p, y)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = m(p, y)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    y[:30].copy_(p)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, m(p, y))


def test_cached_statistics(cuda_device):
    p, y = (t.to(DEV) for t in inputs(CASES["relu_100x64_vs_80x64"]))
    (mp, sp), (my, sy) = ops.fid_moments(p), ops.fid_moments(y)
    got = GM.compute_frechet_distance(mp, sp, my, sy)
    assert got.dtype == F64 and got.is_cuda and torch.equal(got, GM.FIDMetric()(p, y))


def test_input_on_a_non_current_device(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device")
    p, y = (t.to("cuda:1") for t in inputs(CASES["relu_100x64_vs_80x64"]))
    got = GM.FIDMetric()(p, y)
    assert got.device == p.device
    assert abs(float(got) - FIX["relu_100x64_vs_80x64"]["exact"]) <= 1e-10 * FIX["relu_100x64_vs_80x64"]["S"]


@pytest.mark.parametrize("where", ["pred", "y", "both"])
def test_nan_features_give_nan(cuda_device, where):
    p, y = (t.to(DEV) for t in inputs(CASES["relu_100x64_vs_80x64"]))
    if where in ("pred", "both"):
        p[3, 5] = float("nan")
    if where in ("y", "both"):
        y[7, 0] = float("nan")
    assert torch.isnan(GM.FIDMetric()(p, y)).item()


def test_cpu_tensors_raise(cuda_device):
    with pytest.raises(RuntimeError, match="CUDA"):
        GM.FIDMetric()(torch.rand(5, 4), torch.rand(5, 4))
