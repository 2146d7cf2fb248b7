"""Generate the sample-quality metrics fixture (tests/golden/g_metrics.pt) by running the UNMODIFIED reference metrics
(the reference checkout named by REFERENCE_DIR, CPU fp32, MONAI shim):   python -m tests.golden.make_golden_metrics

Inputs are regenerated from each case's seed by `inputs` below, so the fixture stores the seeds, the arguments and the
reference's outputs only.  Cases:
  ms2d_gaussian, ms2d_uniform, ms3d_gaussian   the reference's tests/test_compute_multiscalessim_metric.py (64^2, 64^3,
                                               weights [0.5, 0.5], abs(randn) / max after seed 0)
  mmd_ones_2d, mmd_ones_3d                     the reference's tests/test_compute_mmd_metric.py (ones, 3x3x144^2 / ^3)
  tutorial_ssim, tutorial_ms                   the realism-diversity tutorial's settings: kernel_size=4, default weights,
                                               a batch of 4 at 2x64^2; aggregate() under every reduction mode, with and
                                               without get_not_nans
  ssim_brain                                   SSIM, k = 11, 1x1x160x224x160
  ms_brain                                     MS-SSIM 3-D, k = 4, default weights, 1x1x160x224x160
  mmd_brain                                    MMD on 4 such volumes with y_pred = y + 1e-3 noise (the terms cancel)
MMD cases also record the three terms mean(YY^T), mean(PP^T), mean(PY^T) in float64, the scale of its tolerance.
"""
import torch

from tests.golden import save
from oracle import ref_import

REDUCTIONS = ["none", "mean", "sum", "mean_batch", "sum_batch", "mean_channel", "sum_channel"]
BRAIN = (1, 1, 160, 224, 160)

CASES = {
    "ms2d_gaussian": dict(kind="ms", shape=(1, 1, 64, 64), seed=0, gen="ref_test",
                          kw=dict(spatial_dims=2, data_range=1.0, kernel_type="gaussian", weights=[0.5, 0.5])),
    "ms2d_uniform": dict(kind="ms", shape=(1, 1, 64, 64), seed=0, gen="ref_test",
                         kw=dict(spatial_dims=2, data_range=1.0, kernel_type="uniform", weights=[0.5, 0.5])),
    "ms3d_gaussian": dict(kind="ms", shape=(1, 1, 64, 64, 64), seed=0, gen="ref_test",
                          kw=dict(spatial_dims=3, data_range=1.0, kernel_type="gaussian", weights=[0.5, 0.5])),
    "mmd_ones_2d": dict(kind="mmd", shape=(3, 3, 144, 144), seed=0, gen="ones"),
    "mmd_ones_3d": dict(kind="mmd", shape=(3, 3, 144, 144, 144), seed=0, gen="ones"),
    "tutorial_ssim": dict(kind="ssim", shape=(4, 2, 64, 64), seed=11, gen="rand",
                          kw=dict(spatial_dims=2, data_range=1.0, kernel_size=4)),
    "tutorial_ms": dict(kind="ms", shape=(4, 2, 64, 64), seed=12, gen="rand",
                        kw=dict(spatial_dims=2, data_range=1.0, kernel_size=4)),
    "ssim_brain": dict(kind="ssim", shape=BRAIN, seed=21, gen="rand", kw=dict(spatial_dims=3, data_range=1.0)),
    "ms_brain": dict(kind="ms", shape=BRAIN, seed=22, gen="rand", kw=dict(spatial_dims=3, data_range=1.0, kernel_size=4)),
    "mmd_brain": dict(kind="mmd", shape=(4, *BRAIN[1:]), seed=23, gen="close"),
}


def inputs(case):
    """(y_pred, y) for SSIM / MS-SSIM cases, (y, y_pred) for MMD cases, fp32 on the CPU."""
    shape, gen = case["shape"], case["gen"]
    g = torch.Generator().manual_seed(case["seed"])
    if gen == "ones":
        return torch.ones(shape), torch.ones(shape)
    if gen == "ref_test":      # set_determinism(0); abs(randn) / max, preds first
        a = torch.abs(torch.randn(shape, generator=g))
        b = torch.abs(torch.randn(shape, generator=g))
        return a / a.max(), b / b.max()
    a = torch.rand(shape, generator=g)
    if gen == "close":
        return a, a + 1e-3 * torch.randn(shape, generator=g)
    return a, (a + 0.2 * torch.randn(shape, generator=g)).clamp(0, 1)


def mmd_terms(y, p):
    y, p = y.double().reshape(y.shape[0], -1), p.double().reshape(p.shape[0], -1)
    V = y.shape[1]
    ym, pm = y.mean(0), p.mean(0)
    return torch.stack([(ym @ ym) / V, (pm @ pm) / V, (pm @ ym) / V])


def main():
    ref_import.import_reference()
    from generative.metrics import MMDMetric, MultiScaleSSIMMetric, SSIMMetric
    out = {}
    for name, case in CASES.items():
        rec = {k: v for k, v in case.items()}
        a, b = inputs(case)
        if case["kind"] == "mmd":
            rec["out"] = MMDMetric()(a, b)
            rec["terms"] = mmd_terms(a, b)
        else:
            cls = SSIMMetric if case["kind"] == "ssim" else MultiScaleSSIMMetric
            m = cls(**case["kw"])
            rec["out"] = m(a, b)
            m(b, a)        # a second call: the buffer holds 2 batches
            rec["aggregate"] = {r: m.aggregate(r) for r in REDUCTIONS}
            m.get_not_nans = True
            rec["aggregate_not_nans"] = {r: m.aggregate(r) for r in REDUCTIONS}
        out[name] = rec
        print(name, rec["out"].reshape(-1)[:4].tolist(), flush=True)
    save(out, "g_metrics")


if __name__ == "__main__":
    main()
