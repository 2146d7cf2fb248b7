"""Time the sample-quality metrics on one GPU with CUDA events after a warm-up, beside the torch restatement of the
reference's arithmetic (oracle/metrics_oracle.py: full-kernel F.conv{2,3}d, F.avg_pool, three torch.mm) on the same
card, and record the card's name and power limit from the same run.  Prints one JSON line; --out also writes it to a
file.

FID rows time FIDMetric / compute_frechet_distance against tests/fid_oracle.py (torch fp64 moments on the GPU, scipy
sqrtm on the host; one untimed-warm-up-free call, as the host sqrtm dominates) and add a per-stage split and the launch
count from a separate torch.profiler pass: moments, factor (pivoted Cholesky), M (the two GEMMs), tridiagonalisation,
bisection and finish.

    python tools/metrics_probe.py [--iters 10] [--out results/metrics_probe.json]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from generativemodels_b200 import metrics as GM  # noqa: E402
from generativemodels_b200 import ops  # noqa: E402
from oracle import metrics_oracle as MO  # noqa: E402
from tests import fid_oracle as FO  # noqa: E402
from tests.golden.make_golden_fid import features  # noqa: E402

BRAIN = (1, 1, 160, 224, 160)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "unknown"


def time_ms(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


STAGES = [("moments", ("fid_colmean",)), ("factor", ("fid_chol",)), ("tridiagonalisation", ("fid_house", "fid_symv",
           "fid_rank2", "fid_tri_tail")), ("bisection", ("fid_bisect",)), ("finish", ("fid_finish",))]


def fid_stages(moments, frechet):
    """Per-stage kernel time (ms) and launch count of one call, from torch.profiler: fid_dgemm is the moments' Gram
    under `moments` and the M products under `frechet`."""
    from torch.profiler import ProfilerActivity, profile
    split, launches = {}, 0
    for part, fn in (("moments", moments), ("frechet", frechet)):
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            if ev.device_type != torch.autograd.DeviceType.CUDA or "fid_" not in ev.key:
                continue
            stage = "M" if "fid_dgemm" in ev.key and part == "frechet" else "moments" if "fid_dgemm" in ev.key else \
                next((n for n, keys in STAGES if any(k in ev.key for k in keys)), "other")
            split[stage] = round(split.get(stage, 0.0) + ev.device_time_total / 1e3, 3)
            launches += ev.count
    return split, launches


def fid_rows(iters):
    rows = {}
    for name, (n, F) in {"fid_1000x2048_vs_1000x2048": (1000, 2048), "fid_10000x2048_vs_10000x2048": (10000, 2048),
                         "fid_5000x4096_vs_5000x4096": (5000, 4096)}.items():
        p, y = features(n, F, 1, shift=0.1).cuda(), features(n, F, 2).cuda()
        stats = [ops.fid_moments(p), ops.fid_moments(y)]
        rows[name] = (lambda p=p, y=y: GM.FIDMetric()(p, y), lambda p=p, y=y: FO.fid(p, y),
                      lambda p=p, y=y: (ops.fid_moments(p), ops.fid_moments(y)),
                      lambda s=stats: ops.frechet(*s[0], *s[1]))
        if F == 2048 and n == 10000:
            rows["compute_frechet_distance_cached_F2048"] = (
                lambda s=stats: GM.compute_frechet_distance(*s[0], *s[1]),
                lambda s=stats: FO.frechet_distance(*s[0], *s[1]), lambda: None,
                lambda s=stats: ops.frechet(*s[0], *s[1]))
    out = {}
    for name, (ours, base, mom, fre) in rows.items():
        o = time_ms(ours, iters)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ref = base()
        torch.cuda.synchronize()
        bl = (time.perf_counter() - t0) * 1e3
        split, launches = fid_stages(mom, fre)
        got = float(ours())
        out[name] = {"ms": round(o, 3), "oracle_ms": round(bl, 1), "speedup": round(bl / o, 1),
                     "stages_ms": split, "launches": launches, "fid": got,
                     "rel_diff_vs_oracle": abs(got - float(ref)) / max(abs(float(ref)), 1e-300)}
        print(name, out[name], flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "metrics_probe needs a CUDA device"
    torch.manual_seed(0)
    a = torch.rand(BRAIN, device="cuda")
    b = (a + 0.2 * torch.randn_like(a)).clamp(0, 1)
    y4 = torch.rand((4, *BRAIN[1:]), device="cuda")
    p4 = y4 + 1e-3 * torch.randn_like(y4)
    t2a = torch.rand(4, 2, 64, 64, device="cuda")
    t2b = torch.rand(4, 2, 64, 64, device="cuda")
    s3 = dict(kernel_size=(11, 11, 11), kernel_sigma=(1.5, 1.5, 1.5))
    s4 = dict(kernel_size=(4, 4, 4), kernel_sigma=(1.5, 1.5, 1.5))
    cases = {
        "ssim_k11_1x1x160x224x160": (lambda: GM.SSIMMetric(3)(a, b), lambda: MO.ssim(a, b, 3, **s3), 1),
        "ms_ssim_k4_1x1x160x224x160": (lambda: GM.MultiScaleSSIMMetric(3, kernel_size=4)(a, b),
                                       lambda: MO.ms_ssim(a, b, 3, **s4), 1),
        "mmd_4x1x160x224x160": (lambda: GM.MMDMetric()(y4, p4), lambda: MO.mmd(y4, p4), 1),
        "ms_ssim_k4_4x2x64x64": (lambda: GM.MultiScaleSSIMMetric(2, kernel_size=4)(t2a, t2b),
                                 lambda: MO.ms_ssim(t2a, t2b, 2, kernel_size=(4, 4), kernel_sigma=(1.5, 1.5)), 1),
    }
    res = {"card": card(), "iters": args.iters, "cases": {}}
    with torch.no_grad():
        for name, (ours, base, _) in cases.items():
            o = time_ms(ours, args.iters)
            bl = time_ms(base, max(2, args.iters // 5), warmup=1)
            diff = (ours().double().reshape(-1) - base().double().reshape(-1)).abs().max().item()
            res["cases"][name] = {"ms": round(o, 4), "torch_restatement_ms": round(bl, 4),
                                  "speedup": round(bl / o, 1), "max_abs_diff_vs_restatement": diff}
            print(name, res["cases"][name], flush=True)
    res["cases"].update(fid_rows(max(2, args.iters // 5)))
    print(json.dumps(res))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
