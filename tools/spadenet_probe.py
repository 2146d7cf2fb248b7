"""Timing of SPADENet on the CUDA path, eager and CUDA-graph replayed, with CUDA events:
  - the 2d_spade_gan tutorial's network (128^2, label_nc 6, [16, 32, 64, 128], z 16), VAE forward at batch 1 and 32;
  - decode of a 3-D 128^3 volume (label_nc 3, [16, 32, 64, 128], z 16), batch 1.
Prints the card name and power limit first, then one JSON line per (case, mode) with the median ms per call.

    python tools/spadenet_probe.py [--reps 10] [--out DIR]
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
import torch.nn.functional as F  # noqa: E402

from generativemodels_b200.cuda_graph import graphed  # noqa: E402
from generativemodels_b200.networks.nets import SPADENet  # noqa: E402


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:          # the timing does not depend on it; say what is missing
        return f"{torch.cuda.get_device_name()} (power limit unknown: {e})"


def seg_map(n, label_nc, shape):
    lab = torch.randint(0, label_nc, (n, *[s // 8 for s in shape]), device="cuda")
    lab = F.interpolate(lab[:, None].float(), size=tuple(shape), mode="nearest")[:, 0].long()
    return F.one_hot(lab, label_nc).movedim(-1, 1).float().contiguous()


def time_ms(fn, reps):
    for _ in range(2):
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
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print(f"card: {card()}", flush=True)
    rows = []
    torch.manual_seed(0)
    tut = SPADENet(2, 1, 1, 6, [128, 128], [16, 32, 64, 128], 16, True).eval().cuda()
    vol = SPADENet(3, 1, 1, 3, [128, 128, 128], [16, 32, 64, 128], 16, True).eval().cuda()
    cases = []
    for n in (1, 32):
        seg, x = seg_map(n, 6, (128, 128)), torch.randn(n, 1, 128, 128, device="cuda")
        cases.append((f"tutorial2d_forward_b{n}", tut, (seg, x)))
    cases.append(("decode3d_128", vol.decoder, (seg_map(1, 3, (128, 128, 128)), torch.randn(1, 16, device="cuda"))))
    with torch.no_grad():
        for name, mod, inp in cases:
            for mode in ("eager", "graph"):
                fn_mod = mod if mode == "eager" else graphed(mod)
                med, best = time_ms(lambda: fn_mod(*inp), args.reps)
                row = dict(case=name, mode=mode, ms_median=round(med, 3), ms_min=round(best, 3), reps=args.reps)
                rows.append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "spadenet_probe.json").write_text(json.dumps(dict(card=card(), rows=rows), indent=1))


if __name__ == "__main__":
    main()
