"""Dev probe: the MedNIST DDPM bundle (model-zoo/models/mednist_ddpm) at its published size — 2-D UNet (64, 128, 128),
attention at the two lower levels (head 128), DDPMScheduler(1000) — resolved from its stored YAML configs
(tests/golden/mednist_ddpm_common.yaml + mednist_ddpm_infer.yaml) on one GPU, random-init weights (zero-initialised
tensors redrawn).

Times the bundle's own ``sample`` (1000 DDPM steps at batch 1, the UNet replayed from its CUDA graph) with CUDA events
after a warm-up sample: median, min and max of --repeats samples.  The per-step time is then split into
* the graph replay: the UNet wrapper called back to back 1000 times on one input (inputs copied in, graph replayed,
  output cloned), with nothing between the calls;
* the host part: the scheduler's CPU ``torch.randn`` of the step noise and its synchronising copy to the device,
  timed alone 1000 times;
and the rest (the step kernel and the launch overheads between them).  The card's name and power limit are read in
the same run.  Prints one JSON line; --out also writes it to a file.

    python tools/mednist_probe.py [--repeats 5] [--out results/mednist_probe.json]
"""
import argparse
import json
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch

from generativemodels_b200.bundle.config import BundleConfig

CONFIGS = [str(ROOT / "tests/golden/mednist_ddpm_common.yaml"), str(ROOT / "tests/golden/mednist_ddpm_infer.yaml")]
IMPORTS = ["$import os", "$import datetime", "$import torch", "$import scripts", "$import generative",
           "$import torch.distributed as dist"]
STEPS = 1000


def redraw(m):
    with torch.no_grad():
        for p in m.parameters():
            if float(p.detach().abs().max()) == 0:
                p.normal_(0, 0.02)
    return m


def card():
    q = subprocess.run(["nvidia-smi", "--id=" + str(torch.cuda.current_device()),
                        "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def timed_ms(fn, repeats):
    times = []
    for _ in range(repeats):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        fn()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    return statistics.median(times), min(times), max(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mednist_probe: no CUDA device")
    with tempfile.TemporaryDirectory() as tmp:
        (Path(tmp) / "scripts").mkdir()                       # `$import scripts`: the bundle's holds a training helper
        (Path(tmp) / "scripts" / "__init__.py").write_text("")
        sys.path.insert(0, tmp)
        torch.manual_seed(0)
        cfg = BundleConfig(CONFIGS, {"imports": IMPORTS}, bundle="mednist_ddpm")
        net = redraw(cfg.get("network")).eval()
        sample, noise = cfg.get("sample"), cfg.get("noise").cuda()
        sched = cfg.get("scheduler")
        assert len(sched.timesteps) == STEPS

    sample(noise)                                             # packs the weights, captures the graph
    torch.cuda.synchronize()
    whole = timed_ms(lambda: sample(noise), args.repeats)

    replay_fn = net.__dict__["_b200_auto_graph"]              # the inferer's cached CUDA-graph wrapper
    ts = torch.Tensor((500,)).cuda()

    def replays():
        for _ in range(STEPS):
            replay_fn(noise, timesteps=ts)
    replay = timed_ms(replays, args.repeats)

    def host():
        for _ in range(STEPS):
            torch.randn(noise.size(), dtype=noise.dtype).to(noise.device)
    host_part = timed_ms(host, args.repeats)

    step_ms = whole[0] / STEPS
    res = {"probe": "mednist_ddpm", "steps": STEPS, "batch": 1, "repeats": args.repeats,
           "unet_params_M": round(sum(p.numel() for p in net.parameters()) / 1e6, 2),
           "sample_ms_median_min_max": [round(v, 1) for v in whole],
           "step_ms": round(step_ms, 4),
           "graph_replay_ms_per_step": round(replay[0] / STEPS, 4),
           "host_randn_copy_ms_per_step": round(host_part[0] / STEPS, 4),
           "rest_ms_per_step": round(step_ms - (replay[0] + host_part[0]) / STEPS, 4),
           "peak_memory_GiB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), **card()}
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
