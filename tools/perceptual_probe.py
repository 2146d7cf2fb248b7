"""Time PerceptualLoss(network_type="resnet50") on one GPU with CUDA events after a warm-up (median of --reps
repetitions), beside the torch oracle (oracle/perceptual_oracle.py: torchvision's ResNet-50 in fp32 with TF32 off, as
the reference computes, and under fp16 autocast) on the same card, and record the card's name, power limit and
maximum SM clock from the same run.  Workloads: 2-D at 8 x 1 x 256 x 256 and the 2.5-D loss of the brain-LDM volume
1 x 1 x 160 x 224 x 160 (ratio 0.5: 2 x 272 slices).  The stem (tap gather, its GEMM and the max-pool) and the head
(b200_perceptual_distance and _mean) are timed alone on the same images, to give their share of the call.  Prints one
JSON line; --out also writes it to a file.

    python tools/perceptual_probe.py [--reps 7] [--out results/perceptual_probe.json]
"""
import argparse
import ctypes
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from generativemodels_b200 import ops  # noqa: E402
from generativemodels_b200.losses import PerceptualLoss  # noqa: E402
from oracle import perceptual_oracle as O  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "unknown"


def median_ms(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    return statistics.median(times)


def stem_and_head(m, n_img, H, W, reps):
    """Median ms of the stem and of the head for n_img image pairs of H x W."""
    feats = m.perceptual_function.model
    x = ops.CL(torch.zeros((2 * n_img, 1, H, W, 8), dtype=ops.H16, device="cuda"), 3, 2)
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    geom = (ctypes.c_int32 * 16)(x.N, 1, H, W, 1, OH, OW, 1, 7, 7, 1, 2, 2, 0, 3, 3)

    def stem():
        h = ops.linear(ops.tap_gather(x, geom, 49), feats._stem(), act1=ops.ACT_RELU, split_k=False)
        ops.pool_s2(h, 3, 1, "max")
    f = feats.forward_cl(x)
    image = torch.empty(n_img, dtype=torch.float64, device="cuda")

    def head():
        ops.perceptual_distance(f[:n_img], f[n_img:], 2048, image)
        ops.perceptual_mean(image, [n_img])
    return median_ms(stem, reps), median_ms(head, reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card": card(), "reps": a.reps, "rows": []}
    torch.manual_seed(0)
    m2 = PerceptualLoss(2, "resnet50", pretrained=False).cuda()
    m3 = PerceptualLoss(3, "resnet50", pretrained=False, is_fake_3d=True).cuda()
    m3.load_state_dict(m2.state_dict())
    net = torch.nn.Module()
    for k in ("conv1", "bn1", "relu", "maxpool", "layer1", "layer2", "layer3", "layer4"):
        net.add_module(k, getattr(m2.perceptual_function.model, k))
    net = net.eval()
    for name, shape, m, dims in (("2d_8x1x256x256", (8, 1, 256, 256), m2, 2),
                                 ("fake3d_1x1x160x224x160", (1, 1, 160, 224, 160), m3, 3)):
        x = torch.rand(shape, device="cuda")
        y = (x + 0.05 * torch.randn_like(x)).clamp(0, 1)
        with torch.no_grad():
            ours = median_ms(lambda: m(x, y), a.reps)
            ref32 = median_ms(lambda: O.loss(net, x, y, dims), a.reps)
            with torch.autocast("cuda", dtype=torch.float16):
                ref16 = median_ms(lambda: O.loss(net, x, y, dims), a.reps)
            if dims == 2:
                stem, head = stem_and_head(m, 8, 256, 256, a.reps)
                stem_head = [stem, head]
            else:          # the three axes' slice sets, at their own extents
                parts = [stem_and_head(m, 80, 224, 160, a.reps), stem_and_head(m, 112, 160, 160, a.reps),
                         stem_and_head(m, 80, 160, 224, a.reps)]
                stem_head = [sum(p[0] for p in parts), sum(p[1] for p in parts)]
        res["rows"].append({"workload": name, "ours_ms": round(ours, 3), "oracle_fp32_ms": round(ref32, 3),
                            "oracle_fp16_autocast_ms": round(ref16, 3), "stem_ms": round(stem_head[0], 3),
                            "head_ms": round(stem_head[1], 3), "stem_share": round(stem_head[0] / ours, 3),
                            "head_share": round(stem_head[1] / ours, 3)})
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
