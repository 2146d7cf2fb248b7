"""Pin oracle/metrics_oracle.py against the UNMODIFIED reference metrics (imported from the reference checkout on the
MONAI shim), beyond the fixture's cases: anisotropic kernels and sigmas, the uniform kernel, several channels.  Runs
only where the reference tree exists."""
import sys

import pytest
import torch

from oracle import metrics_oracle as MO
from oracle import ref_import

pytestmark = pytest.mark.skipif(not ref_import.available(), reason="the reference checkout is not present")


@pytest.fixture(scope="module")
def ref():
    """The reference's `generative` for this module only: this repository's own `generative` alias (its modules and its
    import hook) is set aside and restored afterwards."""
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


CASES = [
    (2, (2, 3, 40, 37), "gaussian", (5, 7), (0.8, 2.0)),
    (2, (1, 2, 30, 33), "uniform", (4, 6), (1.5, 1.5)),
    (3, (1, 2, 20, 17, 22), "gaussian", (3, 5, 4), (1.0, 0.7, 1.5)),
    (3, (2, 1, 16, 18, 15), "uniform", (4, 4, 4), (1.5, 1.5, 1.5)),
]


@pytest.mark.parametrize("sd,shape,kt,ks,sig", CASES)
def test_ssim_and_cs(ref, sd, shape, kt, ks, sig):
    g = torch.Generator().manual_seed(len(shape) * 10 + ks[0])
    a, b = torch.rand(shape, generator=g), torch.rand(shape, generator=g)
    want = ref.ssim.compute_ssim_and_cs(a, b, sd, kernel_type=kt, kernel_size=ks, kernel_sigma=sig)
    got = MO.ssim_and_cs(a, b, sd, kernel_type=kt, kernel_size=ks, kernel_sigma=sig)
    for w, o in zip(want, got):
        assert (w - o).abs().max().item() <= 1e-6
    m = ref.SSIMMetric(sd, kernel_type=kt, kernel_size=ks, kernel_sigma=sig)
    assert (m(a, b) - MO.ssim(a, b, sd, kernel_type=kt, kernel_size=ks, kernel_sigma=sig)).abs().max() <= 1e-6


def test_ms_ssim_and_mmd(ref):
    g = torch.Generator().manual_seed(9)
    a, b = torch.rand(2, 2, 45, 51, generator=g), torch.rand(2, 2, 45, 51, generator=g)
    kw = dict(kernel_size=(3, 3), kernel_sigma=(1.5, 1.5))
    want = ref.MultiScaleSSIMMetric(2, kernel_size=3, weights=[0.3, 0.3, 0.4])(a, b)
    assert (want - MO.ms_ssim(a, b, 2, weights=[0.3, 0.3, 0.4], **kw)).abs().max() <= 1e-6
    y, p = torch.rand(3, 2, 9, 7, generator=g), torch.rand(3, 2, 9, 7, generator=g)
    assert abs(float(ref.MMDMetric()(y, p)) - float(MO.mmd(y, p))) <= 1e-7
