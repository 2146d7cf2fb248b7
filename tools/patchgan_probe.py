"""Timing of the PatchGAN discriminators on the CUDA path, eager and CUDA-graph replayed, with CUDA events:
  - the 2d_ldm tutorial's PatchDiscriminator (BATCH, 64 channels) at batch 16 x 1 x 64^2;
  - the 3d_ldm tutorial's 3-D PatchDiscriminator (BATCH, 32 channels) at batch 2 x 1 x 96 x 96 x 64;
  - the 2d_spade_vae tutorial's MultiScalePatchDiscriminator (INSTANCE, 2 scales, 7 channels) at batch 8 x 7 x 128^2.
Prints the card name and power limit first, then one JSON line per (case, mode) with the median ms per call.

    python tools/patchgan_probe.py [--reps 20] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

from generativemodels_b200.cuda_graph import graphed  # noqa: E402
from generativemodels_b200.networks.nets import MultiScalePatchDiscriminator, PatchDiscriminator  # noqa: E402
from tools.spadenet_probe import card, time_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print(f"card: {card()}", flush=True)
    torch.manual_seed(0)
    cases = [
        ("ldm2d_b16", PatchDiscriminator(spatial_dims=2, num_layers_d=3, num_channels=64, in_channels=1,
                                         out_channels=1), (16, 1, 64, 64)),
        ("ldm3d_b2", PatchDiscriminator(spatial_dims=3, num_layers_d=3, num_channels=32, in_channels=1,
                                        out_channels=1), (2, 1, 96, 96, 64)),
        ("spade_vae_b8", MultiScalePatchDiscriminator(num_d=2, num_layers_d=3, spatial_dims=2, num_channels=8,
                                                      in_channels=7, out_channels=7, minimum_size_im=128,
                                                      norm="INSTANCE", kernel_size=3), (8, 7, 128, 128)),
    ]
    rows = []
    with torch.no_grad():
        for name, mod, shape in cases:
            mod = mod.eval().cuda()
            x = torch.randn(shape, device="cuda")
            for mode in ("eager", "graph"):
                fn_mod = mod if mode == "eager" else graphed(mod)
                med, best = time_ms(lambda: fn_mod(x), args.reps)
                row = dict(case=name, mode=mode, ms_median=round(med, 3), ms_min=round(best, 3), reps=args.reps)
                rows.append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "patchgan_probe.json").write_text(json.dumps(dict(card=card(), rows=rows), indent=1))


if __name__ == "__main__":
    main()
