"""CPU checks of generativemodels_b200.metrics: the host code (argument handling, exceptions, MONAI's buffer and
reductions, MMD's transforms and squeeze) end to end on the CPU stand-in of the C ABI (tests/metrics_backend.py), whose
float64 reading of the
kernels (tests/metrics_emulator.py) and the torch restatement of the reference (oracle/metrics_oracle.py) are both
held to the reference's outputs in tests/golden/g_metrics.pt."""
import re
from pathlib import Path

import pytest
import torch

from generativemodels_b200 import _lib

from generativemodels_b200 import metrics as GM
from generativemodels_b200.metrics import metric as GM_metric
from generativemodels_b200.metrics import mmd as GM_mmd
from generativemodels_b200.metrics import ms_ssim as GM_ms
from generativemodels_b200.metrics import ssim as GM_ssim
from oracle import metrics_oracle as MO
from tests import golden, metrics_backend
from tests.golden.make_golden_metrics import CASES, REDUCTIONS, inputs

FIX = golden.load("g_metrics")
SMALL = [n for n, c in CASES.items() if "brain" not in n and c["shape"] != (3, 3, 144, 144, 144)]


@pytest.fixture
def cpu(monkeypatch):
    metrics_backend.install(monkeypatch)
    for mod in (GM_metric, GM_ssim, GM_ms, GM_mmd):
        monkeypatch.setattr(mod, "require_cuda", lambda *t: None, raising=False)


def _metric(case):
    cls = GM.SSIMMetric if case["kind"] == "ssim" else GM.MultiScaleSSIMMetric
    return cls(**case["kw"])


def _oracle(case, a, b):
    kw = dict(case["kw"])
    sd = kw.pop("spatial_dims")
    ks = kw.pop("kernel_size", 11)
    kw["kernel_size"] = (ks,) * sd
    kw["kernel_sigma"] = (1.5,) * sd
    if case["kind"] == "ssim":
        return MO.ssim(a, b, sd, **kw)
    return MO.ms_ssim(a, b, sd, **kw)


def _scale(name):
    rec = FIX[name]
    return float(rec["terms"].abs().sum()) if rec["kind"] == "mmd" else 1.0


# float64 reading vs the reference's fp32: the reference's own bound (1e-6) on its MS-SSIM cases, 1e-6 relative to
# the Gram terms on MMD.  Elsewhere the fp32 cancellation of sigma = E[x^2] - E[x]^2 in the reference moves the
# means; it is largest where MS-SSIM's coarsest scale has a single voxel per channel (tutorial_ms: 6.1e-6 measured)
TOL = 2e-5


def _tol(name):
    return 1e-6 if CASES[name].get("gen") == "ref_test" else TOL


@pytest.mark.parametrize("name", SMALL + ["ssim_brain", "ms_brain", "mmd_brain", "mmd_ones_3d"])
def test_stand_in_matches_reference_fixture(cpu, name):
    case, rec = CASES[name], FIX[name]
    a, b = inputs(case)
    if case["kind"] == "mmd":
        got = GM.MMDMetric()(a, b)
        assert got.dim() == 0 and got.dtype == torch.float32
        assert abs(float(got) - float(rec["out"])) <= 1e-6 * _scale(name) + 1e-12
        return
    m = _metric(case)
    got = m(a, b)
    assert got.shape == rec["out"].shape == (case["shape"][0], 1) and got.dtype == torch.float32
    assert (got - rec["out"]).abs().max().item() <= _tol(name)


@pytest.mark.parametrize("name", [n for n in SMALL if CASES[n]["kind"] != "mmd"] + ["ssim_brain"])
def test_oracle_matches_reference_fixture(name):
    case, rec = CASES[name], FIX[name]
    a, b = inputs(case)
    assert (_oracle(case, a, b) - rec["out"]).abs().max().item() <= 1e-6


def test_oracle_mmd_matches_reference_fixture():
    for name in ("mmd_ones_2d", "mmd_brain"):
        a, b = inputs(CASES[name])
        assert abs(float(MO.mmd(a, b)) - float(FIX[name]["out"])) <= 1e-6 * _scale(name) + 1e-12


def test_mmd_is_the_difference_of_the_gram_terms():
    """mmd_brain: the reference's fp32 GEMMs lose the answer (it comes out negative); the column reduction gives the
    float64 value of the terms' combination."""
    rec = FIX["mmd_brain"]
    a, b = inputs(CASES["mmd_brain"])
    exact = float(rec["terms"][0] + rec["terms"][1] - 2 * rec["terms"][2])
    from tests import metrics_emulator as M
    assert abs(float(M.mmd(a, b)) - exact) <= 1e-9 * _scale("mmd_brain")
    assert float(M.mmd(a, b)) > 0 > float(rec["out"])


@pytest.mark.parametrize("name", ["tutorial_ssim", "tutorial_ms"])
def test_aggregate_every_reduction(cpu, name):
    case, rec = CASES[name], FIX[name]
    a, b = inputs(case)
    m = _metric(case)
    m(a, b)
    m(b, a)
    for r in REDUCTIONS:
        want = rec["aggregate"][r]
        got = m.aggregate(r)
        assert got.shape == want.shape, r
        assert (got - want).abs().max().item() <= TOL * max(1.0, want.abs().max().item()), r
    m.get_not_nans = True
    for r in REDUCTIONS:
        f, nn = m.aggregate(r)
        wf, wn = rec["aggregate_not_nans"][r]
        assert torch.equal(nn, wn) and (f - wf).abs().max().item() <= TOL * max(1.0, wf.abs().max().item()), r
    m.reset()
    with pytest.raises(ValueError):
        m.aggregate()


def test_reduction_excludes_nans():
    f = torch.tensor([[1.0, float("nan")], [3.0, 5.0], [float("nan"), float("nan")]])
    out, nn = GM.do_metric_reduction(f.clone(), "mean")
    assert out.item() == pytest.approx((1.0 + 4.0) / 2) and nn.item() == 2
    out, nn = GM.do_metric_reduction(f.clone(), "sum_batch")
    assert out.tolist() == [4.0, 5.0] and nn.tolist() == [2.0, 1.0]
    out, nn = GM.do_metric_reduction(f.clone(), "mean_channel")
    assert out.tolist() == [1.0, 4.0, 0.0] and nn.tolist() == [1.0, 2.0, 0.0]
    out, nn = GM.do_metric_reduction(f.clone(), "none")
    assert torch.isnan(out).sum() == 3 and nn.sum() == 3
    with pytest.raises(ValueError):
        GM.do_metric_reduction(f.clone(), "median")


def test_list_inputs_and_buffer(cpu):
    a, b = torch.rand(3, 1, 16, 16), torch.rand(3, 1, 16, 16)
    m = GM.SSIMMetric(2, kernel_size=5)
    batch = m(a, b)
    items = m(list(a), list(b))
    assert torch.allclose(batch, items) and m.get_buffer().shape == (6, 1)
    assert m.aggregate("none").shape == (6, 1)


def test_exceptions(cpu):
    s2, s3 = GM.SSIMMetric(2), GM.SSIMMetric(3)
    with pytest.raises(ValueError):
        s2(torch.rand(1, 1, 16, 16, 16), torch.rand(1, 1, 16, 16, 16))
    with pytest.raises(ValueError):
        s3(torch.rand(1, 1, 16, 16), torch.rand(1, 1, 16, 16))
    with pytest.raises(ValueError):
        s2(torch.rand(1, 1, 16, 16), torch.rand(1, 1, 16, 17))
    with pytest.raises(ValueError):
        GM.compute_ssim_and_cs(torch.rand(1, 1, 16, 16), torch.rand(1, 1, 16, 17), 2)
    with pytest.raises(UnboundLocalError):
        GM.SSIMMetric(2, kernel_type="box")(torch.rand(1, 1, 16, 16), torch.rand(1, 1, 16, 16))
    with pytest.raises(ValueError):
        GM.MultiScaleSSIMMetric(3, weights=[0.5, 0.5])(torch.rand(1, 1, 64, 64), torch.rand(1, 1, 64, 64))
    with pytest.raises(RuntimeError):
        GM.SSIMMetric(2)(torch.rand(1, 1, 8, 8), torch.rand(1, 1, 8, 8))
    with pytest.raises(ValueError):
        GM.MMDMetric()(torch.ones(3, 3, 144, 144), torch.ones(3, 3, 145, 145))
    with pytest.raises(ValueError):
        GM.MMDMetric(y_transform=lambda t: t[:, :, :-1])(torch.ones(2, 1, 8, 8), torch.ones(2, 1, 8, 8))


def test_ms_ssim_size_check_divisor_is_a_square(cpu):
    """max(1, len(weights) - 1) ** 2: 3 weights divide by 4 (not 2 ** 2 = 4 by accident: 4 weights divide by 9)."""
    ms = GM.MultiScaleSSIMMetric(2, kernel_size=3, weights=[0.25] * 4)
    with pytest.raises(ValueError, match="larger than 18"):
        ms(torch.rand(1, 1, 18, 18), torch.rand(1, 1, 18, 18))      # 18 // 9 = 2 <= 2
    assert ms(torch.rand(1, 1, 27, 27), torch.rand(1, 1, 27, 27)).shape == (1, 1)   # 27 // 9 = 3 > 2


def test_mmd_transforms_and_squeeze(cpu):
    y, p = torch.rand(3, 2, 5, 1), torch.rand(3, 2, 5, 1)
    m = GM.MMDMetric(y_transform=lambda t: 2 * t, y_pred_transform=lambda t: t + 1)
    got = m(y, p)
    assert float(got) == pytest.approx(float(MO.mmd(2 * y, p + 1)), rel=1e-5, abs=1e-7)
    assert float(GM.MMDMetric()(y[..., 0], p[..., 0])) == pytest.approx(float(GM.MMDMetric()(y, p)), rel=1e-6)
    # non-contiguous views are read in place
    big_y, big_p = torch.rand(4, 3, 10, 12), torch.rand(4, 3, 10, 12)
    got = GM.MMDMetric()(big_y[:, :, ::2, 1:], big_p.transpose(2, 3).transpose(2, 3)[:, :, ::2, 1:])
    assert float(got) == pytest.approx(float(MO.mmd(big_y[:, :, ::2, 1:].contiguous(),
                                                    big_p[:, :, ::2, 1:].contiguous())), rel=1e-5)


def test_compute_ssim_and_cs_maps(cpu):
    torch.manual_seed(3)
    a, b = torch.rand(2, 2, 20, 18, 17), torch.rand(2, 2, 20, 18, 17)
    s, cs = GM.compute_ssim_and_cs(a, b, 3, kernel_size=(5, 4, 3), kernel_sigma=(1.0, 1.5, 0.7))
    ws, wcs = MO.ssim_and_cs(a, b, 3, kernel_size=(5, 4, 3), kernel_sigma=(1.0, 1.5, 0.7))
    assert s.shape == ws.shape == (2, 2, 16, 15, 15) and s.dtype == torch.float32
    assert (s - ws).abs().max() < 1e-4 and (cs - wcs).abs().max() < 1e-4


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError, match="CUDA"):
        GM.SSIMMetric(2, kernel_size=3)(torch.rand(1, 1, 8, 8), torch.rand(1, 1, 8, 8))
    with pytest.raises(RuntimeError, match="CUDA"):
        GM.MMDMetric()(torch.rand(2, 1, 8, 8), torch.rand(2, 1, 8, 8))


def test_library_exports_every_metric_symbol():
    """include/b200gen_metrics.h, _lib.METRIC_SIGNATURES and the library agree, and the metric structs have one size."""
    header = (Path(__file__).resolve().parents[1] / "include" / "b200gen_metrics.h").read_text()
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_lib.METRIC_SIGNATURES), declared ^ set(_lib.METRIC_SIGNATURES)
    assert not declared & set(_lib.SIGNATURES)
    lib = _lib.load()
    import ctypes as C
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.b200_abi_sizeof(10) == C.sizeof(_lib.SsimParams)
    assert lib.b200_abi_sizeof(11) == C.sizeof(_lib.SsimCombineParams)


def test_cpu_stand_in_covers_every_metric_entry_point():
    missing = sorted(n for n in _lib.METRIC_SIGNATURES
                     if not callable(getattr(metrics_backend.MetricsFakeLib, n, None)))
    assert not missing, missing
