"""Timing of DiffusionModelEncoder on the CUDA path, eager and CUDA-graph replayed, with CUDA events: the classifier of
the classifier-guided anomaly-detection tutorial ((32, 64, 64), attention at the two deeper levels, 64-channel heads)
on 1x64x64 images with one broadcast timestep, at batch 1 and 64.  Prints the card name, power limit and maximum SM
clock first, then one JSON line per (batch, mode) with the median and best ms per call.

    python tools/encoder_probe.py [--reps 50] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

from generativemodels_b200.cuda_graph import graphed  # noqa: E402
from generativemodels_b200.networks.nets.diffusion_model_unet import DiffusionModelEncoder  # noqa: E402

TUTORIAL = dict(spatial_dims=2, in_channels=1, out_channels=2, num_channels=(32, 64, 64),
                attention_levels=(False, True, True), num_res_blocks=(1, 1, 1), num_head_channels=64,
                with_conditioning=False)


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:          # the timing does not depend on it; say what is missing
        return f"{torch.cuda.get_device_name()} (power limit and clock unknown: {e})"


def time_ms(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out), min(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    info = card()
    print(f"card: {info}", flush=True)
    torch.manual_seed(0)
    clf = DiffusionModelEncoder(**TUTORIAL).eval().cuda()
    t = torch.Tensor((500,)).cuda()
    rows = []
    with torch.no_grad():
        for n in (1, 64):
            x = torch.randn(n, 1, 64, 64, device="cuda")
            for mode in ("eager", "graph"):
                mod = clf if mode == "eager" else graphed(clf)
                med, best = time_ms(lambda: mod(x, t), args.reps)
                row = dict(case=f"tutorial_classifier_b{n}", mode=mode, ms_median=round(med, 3), ms_min=round(best, 3),
                           reps=args.reps)
                rows.append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "encoder_probe.json").write_text(json.dumps(dict(card=info, rows=rows), indent=1))


if __name__ == "__main__":
    main()
