"""Time the sample-quality metrics on one GPU with CUDA events after a warm-up, beside the torch restatement of the
reference's arithmetic (oracle/metrics_oracle.py: full-kernel F.conv{2,3}d, F.avg_pool, three torch.mm) on the same
card, and record the card's name and power limit from the same run.  Prints one JSON line; --out also writes it to a
file.

    python tools/metrics_probe.py [--iters 10] [--out results/metrics_probe.json]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from generativemodels_b200 import metrics as GM  # noqa: E402
from oracle import metrics_oracle as MO  # noqa: E402

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
    print(json.dumps(res))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
