"""Pin tests/fid_oracle.fid against the UNMODIFIED reference FIDMetric beyond the fixture's cases.  The reference's
fid.py needs numpy.float_ (gone in NumPy 2) and sqrtm's `disp` argument (gone in SciPy 1.18); both are restored here
with monkeypatch for these tests only.  Runs only where the reference tree exists."""
import sys

import numpy as np
import pytest
import scipy.linalg
import torch

from tests import fid_oracle as MO
from oracle import ref_import
from tests.golden.make_golden_fid import features

pytestmark = pytest.mark.skipif(not ref_import.available(), reason="the reference checkout is not present")


@pytest.fixture(scope="module")
def ref():
    """The reference's `generative.metrics` for this module only (see tests/test_metrics_oracle_vs_reference.py)."""
    saved = {k: v for k, v in sys.modules.items() if k == "generative" or k.startswith("generative.")}
    for k in saved:
        del sys.modules[k]
    path, meta = list(sys.path), list(sys.meta_path)
    sys.meta_path[:] = [f for f in meta if type(f).__name__ != "_AliasFinder"]
    ref_import.import_reference()
    import generative.metrics as gm
    yield gm
    for k in [k for k in sys.modules if k == "generative" or k.startswith("generative.")]:
        del sys.modules[k]
    sys.modules.update(saved)
    sys.path[:] = path
    sys.meta_path[:] = meta


@pytest.fixture
def shims(monkeypatch):
    sqrtm = scipy.linalg.sqrtm
    monkeypatch.setattr(np, "float_", np.float64, raising=False)
    monkeypatch.setattr(scipy.linalg, "sqrtm", lambda a, disp=True: (sqrtm(a), 0.0))


@pytest.mark.parametrize("n_p,n_y,F", [(40, 30, 8), (25, 60, 24), (10, 12, 32), (300, 200, 16)])
def test_fid(ref, shims, n_p, n_y, F):
    p, y = features(n_p, F, n_p, shift=0.2), features(n_y, F, 100 + n_y)
    want = float(ref.FIDMetric()(p, y))
    got = float(MO.fid(p, y))
    assert abs(got - want) <= 1e-12 * abs(want)


def test_compute_frechet_distance_and_errors(ref, shims):
    p, y = features(50, 12, 1).double(), features(70, 12, 2).double()
    args = (p.mean(0), MO.cov(p), y.mean(0), MO.cov(y))
    assert float(ref.fid.compute_frechet_distance(*args)) == float(MO.frechet_distance(*args))
    with pytest.raises(ValueError):
        ref.FIDMetric()(torch.ones([3, 3, 144, 144]), torch.ones([3, 3, 145, 145]))
    with pytest.raises(RuntimeError):
        ref.FIDMetric()(torch.rand(1, 4), torch.rand(3, 4))
    with pytest.raises(RuntimeError):
        ref.FIDMetric()(torch.rand(3, 4), torch.rand(3, 5))
