"""Graph-replayed timing of each convolution class of the C3 UNet (3-D, channels (256, 256, 512), 160 x 224 x 160) at
its real size, with the 128-column kernel (impl = 2) and with the planner's choice (impl = 0; pass --impl 3 to force the
128 x 256 two-CTA kernel), alternated in one process.  Prints ms and algorithmic TFLOP/s per class and how far the two
outputs (and their GroupNorm partials) are apart.

    python tools/conv_probe.py [--reps 5] [--rounds 3] [--impl 0|3] [--only name,...]
"""
from __future__ import annotations

import argparse
import json
import math
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

from generativemodels_b200 import ops  # noqa: E402

L0, L1, L2 = (160, 224, 160), (80, 112, 80), (40, 56, 40)


def cl(c, sp):
    return ops.to_cl(torch.randn(1, c, *sp, device="cuda"))


def packed(cout, cin, splits=None, stride=1):
    w = torch.randn(cout, cin, 3, 3, 3, device="cuda") / math.sqrt(cin * 27)
    return ops.PackedConv(w, torch.randn(cout, device="cuda") * 0.1, stride, 1, splits=splits)


def classes():
    """name -> (setup() -> fn(impl) -> CL, algorithmic FLOP of one call)."""
    v0, v1, v2 = (math.prod(s) for s in (L0, L1, L2))

    def l0_conv1():
        x, pc, rv = cl(256, L0), packed(256, 256), torch.randn(1, 256, device="cuda")
        return lambda impl: ops.conv(x, pc, rowvec=rv, impl=impl)

    def l0_conv2():
        x, pc, res = cl(256, L0), packed(256, 256), cl(256, L0)
        return lambda impl: ops.conv(x, pc, residual=res, impl=impl)

    def l0_concat_conv1():
        a, b, pc, rv = cl(256, L0), cl(256, L0), packed(256, 512, splits=[256, 256]), torch.randn(1, 256, device="cuda")
        return lambda impl: ops.conv([a, b], pc, rowvec=rv, impl=impl)

    def l0_upsample():
        x = cl(256, L1)
        pu = ops.PackedUpsampleConv(torch.randn(256, 256, 3, 3, 3, device="cuda") / 80, torch.randn(256, device="cuda"))
        return lambda impl: ops.conv_upsample2x(x, pu, impl=impl)

    def l1_conv():
        x, pc, rv = cl(256, L1), packed(256, 256), torch.randn(1, 256, device="cuda")
        return lambda impl: ops.conv(x, pc, rowvec=rv, impl=impl)

    def l2_conv():
        x, pc, res = cl(512, L2), packed(512, 512), cl(512, L2)
        return lambda impl: ops.conv(x, pc, residual=res, impl=impl)

    return {
        "l0_conv1_rowvec_gn": (l0_conv1, 2 * v0 * 256 * 27 * 256),
        "l0_conv2_residual_gn": (l0_conv2, 2 * v0 * 256 * 27 * 256),
        "l0_concat512_conv1": (l0_concat_conv1, 2 * v0 * 256 * 27 * 512),
        "l0_upsample_phases": (l0_upsample, 2 * v1 * 8 * 256 * 8 * 256),
        "l1_conv": (l1_conv, 2 * v1 * 256 * 27 * 256),
        "l2_conv512": (l2_conv, 2 * v2 * 512 * 27 * 512),
    }


def graph(fn, reps):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    return g


def time_graph(g, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def compare(a, b):
    """(max |a - b| in units of b's 16-bit ulp, relative L2 of the GroupNorm partial sums)"""
    x, y = a.t[..., :a.C].float(), b.t[..., :b.C].float()
    mant = 7 if ops.H16 == torch.bfloat16 else 10
    ulp = torch.exp2(torch.floor(torch.log2(torch.maximum(x.abs(), y.abs()).clamp_min(2.0 ** -14))) - mant)
    ulps = ((x - y).abs() / ulp).max().item()
    gn = None
    if a.gn is not None and b.gn is not None:
        ga, gb = a.gn.double().sum(1), b.gn.double().sum(1)
        gn = ((ga - gb).norm() / gb.norm()).item()
    return ulps, gn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="calls per graph replay")
    ap.add_argument("--rounds", type=int, default=3, help="alternated replays per implementation")
    ap.add_argument("--impl", type=int, default=0, choices=[0, 3])
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "conv_probe needs a CUDA device"
    torch.manual_seed(0)
    only = set(filter(None, args.only.split(",")))
    for name, (setup, flop) in classes().items():
        if only and name not in only:
            continue
        fn = setup()
        ulps, gn = compare(fn(args.impl), fn(2))
        g_old, g_new = graph(lambda: fn(2), args.reps), graph(lambda: fn(args.impl), args.reps)
        t_old, t_new = [], []
        for _ in range(args.rounds):
            t_old.append(time_graph(g_old, args.reps))
            t_new.append(time_graph(g_new, args.reps))
        mo, mn = statistics.median(t_old), statistics.median(t_new)
        print(json.dumps({"class": name, "impl2_ms": round(mo, 3), f"impl{args.impl}_ms": round(mn, 3),
                          "impl2_tflops": round(flop / mo / 1e9, 1), f"impl{args.impl}_tflops": round(flop / mn / 1e9, 1),
                          "speedup": round(mo / mn, 3), "max_ulps": ulps, "gn_rel_l2": gn,
                          "runs_ms": {"impl2": [round(t, 3) for t in t_old], f"impl{args.impl}": [round(t, 3) for t in t_new]}}),
              flush=True)
        del g_old, g_new, fn
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
