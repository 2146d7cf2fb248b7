"""CPU checks of FIDMetric, get_fid_score and compute_frechet_distance: the host code (argument handling, the
reference's exceptions) end to end on the CPU stand-in of the C ABI (tests/fid_backend.py), whose float64 reading of
b200_fid_moments / b200_frechet (tests/fid_emulator.py) is held to the exact values and the reference's outputs in
tests/golden/g_fid.pt; the pivoted Cholesky factor of that reading; and the distance's analytic identities."""
import numpy as np
import pytest
import torch

from generativemodels_b200 import metrics as GM
from generativemodels_b200.metrics import fid as GM_fid
from tests import fid_oracle as MO
from tests import fid_backend, golden
from tests import fid_emulator as M
from tests.golden.make_golden_fid import CASES, checksum, features, inputs

F64 = torch.float64
FIX = golden.load("g_fid")
SMALL = [n for n, c in CASES.items() if c.get("F", 2) <= 256]


@pytest.fixture
def cpu(monkeypatch):
    fid_backend.install(monkeypatch)
    monkeypatch.setattr(GM_fid, "require_cuda", lambda *t: None)


def scale(p, y):
    """S = tr Sigma_p + tr Sigma_y + |mu_p - mu_y|^2, the scale of the tolerances."""
    (mp, sp), (my, sy) = M.fid_moments(p), M.fid_moments(y)
    return float(torch.trace(sp) + torch.trace(sy) + (mp - my) @ (mp - my))


@pytest.mark.parametrize("name", SMALL)
def test_stand_in_matches_fixture(cpu, name):
    case, rec = CASES[name], FIX[name]
    p, y = inputs(case)
    assert all(torch.equal(checksum(t), c) for t, c in zip((p, y), rec["checksum"]))
    got = GM.FIDMetric()(p, y)
    assert got.dim() == 0 and got.dtype == F64
    assert abs(float(got) - rec["exact"]) <= 1e-10 * rec["S"]
    if rec["error"] is None:
        tol = 1e-7 if case["singular"] else 1e-10
        assert abs(float(got) - float(rec["out"])) <= tol * rec["S"]
    assert float(GM.get_fid_score(p, y)) == float(got)


@pytest.mark.parametrize("name", SMALL)
def test_oracle_matches_fixture(name):
    case, rec = CASES[name], FIX[name]
    p, y = inputs(case)
    if rec["error"] is not None:
        with pytest.raises(ValueError, match="Imaginary component"):
            MO.fid(p, y)
        return
    assert abs(float(MO.fid(p, y)) - float(rec["out"])) <= 1e-12 * rec["S"]


BAD_SHAPES = [
    (torch.rand(3, 4, 5), torch.rand(3, 4)),    # y_pred not 2-D
    (torch.rand(4), torch.rand(3, 4)),          # a 1-D input
    (torch.rand(3, 4), torch.rand(4)),
    (torch.rand(1, 4), torch.rand(3, 4)),       # a single row
    (torch.rand(3, 4), torch.rand(1, 4)),
    (torch.rand(3, 4), torch.rand(3, 5)),       # different feature counts
]


def test_errors_mirror_the_reference(cpu):
    with pytest.raises(ValueError, match="Inputs should have"):     # the reference's test_input_dimensions
        GM.FIDMetric()(torch.ones([3, 3, 144, 144]), torch.ones([3, 3, 145, 145]))
    for p, y in BAD_SHAPES:
        with pytest.raises(RuntimeError):
            GM.FIDMetric()(p, y)
        with pytest.raises(RuntimeError):       # the reference's own arithmetic fails the same way
            MO.fid(p, y)
    mu, s = torch.zeros(4, dtype=F64), torch.eye(4, dtype=F64)
    for args in ((mu, s, mu[:3], s), (mu, s, mu, s[:3]), (mu, s[0], mu, s), (mu[:0], s[:0, :0], mu[:0], s[:0, :0])):
        with pytest.raises(RuntimeError):
            GM.compute_frechet_distance(*args)


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError, match="CUDA"):
        GM.FIDMetric()(torch.rand(5, 4), torch.rand(5, 4))
    mu, s = torch.zeros(4, dtype=F64), torch.eye(4, dtype=F64)
    with pytest.raises(RuntimeError, match="CUDA"):
        GM.compute_frechet_distance(mu, s, mu, s)


@pytest.mark.parametrize("n,F,dead", [(30, 64, 0), (200, 64, 8), (500, 40, 0), (2, 8, 0)])
def test_pivoted_cholesky_reconstructs(n, F, dead):
    _, s = M.fid_moments(features(n, F, 31 + n, dead=dead))
    s = s.numpy()
    G, r = M.pivoted_cholesky(s)
    assert r == np.linalg.matrix_rank(s) == min(n - 1, F - dead)
    assert (G[:, r:] == 0).all()
    assert np.abs(G @ G.T - s).max() <= 1e-12 * np.diag(s).max()


def test_pivot_rule():
    """Largest remaining diagonal first, lowest feature index on a tie; a zero matrix has rank 0."""
    s = np.diag([1.0, 4.0, 4.0, 0.0])
    G, r = M.pivoted_cholesky(s)
    assert r == 3 and G[1, 0] == 2.0 and G[2, 1] == 2.0 and G[0, 2] == 1.0
    assert M.pivoted_cholesky(np.zeros((3, 3)))[1] == 0


@pytest.mark.parametrize("n,F", [(60, 16), (12, 40)])
def test_affine_copy_identity(cpu, n, F):
    """y_pred = c y + b (c > 0): FID = |mu_p - mu_y|^2 + (1 - c)^2 tr Sigma_y, singular or not."""
    y = features(n, F, 7 + F).double()
    c, b = 0.5, torch.linspace(-1.0, 1.0, F, dtype=F64)
    p = c * y + b
    mu_y, s_y = M.fid_moments(y)
    d = (c - 1) * mu_y + b
    want = float(d @ d + (1 - c) ** 2 * torch.trace(s_y))
    assert abs(float(GM.FIDMetric()(p, y)) - want) <= 1e-12 * scale(p, y)


@pytest.mark.parametrize("n,F", [(60, 16), (12, 40)])
def test_identical_sets(cpu, n, F):
    y = features(n, F, 3 + n)
    assert abs(float(GM.FIDMetric()(y, y))) <= 1e-12 * scale(y, y)


def test_compute_frechet_distance_on_cached_statistics(cpu):
    p, y = inputs(CASES["relu_100x64_vs_80x64"])
    (mp, sp), (my, sy) = M.fid_moments(p), M.fid_moments(y)
    got = GM.compute_frechet_distance(mp.float(), sp.float(), my, sy, epsilon=1e-3)
    assert got.dim() == 0 and got.dtype == F64
    want = M.frechet(mp.float().double(), sp.float().double(), my, sy)[0]
    assert float(got) == want


def test_library_exports_every_fid_symbol():
    """include/b200gen_fid.h, _lib.FID_SIGNATURES and the library agree, and the FID structs have one size."""
    import ctypes as C
    import re
    from pathlib import Path

    from generativemodels_b200 import _lib
    header = (Path(__file__).resolve().parents[1] / "include" / "b200gen_fid.h").read_text()
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_lib.FID_SIGNATURES), declared ^ set(_lib.FID_SIGNATURES)
    assert not declared & (set(_lib.SIGNATURES) | set(_lib.METRIC_SIGNATURES))
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.b200_abi_sizeof(12) == C.sizeof(_lib.FidMomentsParams)
    assert lib.b200_abi_sizeof(13) == C.sizeof(_lib.FrechetParams)
    assert lib.b200_frechet_workspace_bytes(0) == -1 and lib.b200_frechet_workspace_bytes(_lib.FID_MAX_F + 1) == -1


def test_cpu_stand_in_covers_every_fid_entry_point():
    from generativemodels_b200 import _lib
    missing = sorted(n for n in _lib.FID_SIGNATURES if not callable(getattr(fid_backend.FidFakeLib, n, None)))
    assert not missing, missing
