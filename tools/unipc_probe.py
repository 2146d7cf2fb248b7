"""UniPCMultistepScheduler on one GPU, with CUDA events:

  1. the step kernel b200_unipc_step (corrector with two earlier estimates, predictor of order 2: five input streams,
     three outputs; and the largest case, three earlier estimates) beside b200_dpm_solver_step (2M: three input streams,
     two outputs) and b200_ddim_step, at the C3 volume (1x1x160x224x160): device microseconds per launch (median over
     50 windows of 20 launches) and the fp32 bytes each launch must move over that time;
  2. LatentDiffusionInferer.sample on the C2 networks (2d_ldm_tutorial autoencoder and latent UNet, recipe weights,
     1x3x64x64 latent, decode to 256x256 included) with UniPC-2 (bh2) and DPM-Solver++ 2M at 10 and 20 steps, and
     DDIM-50: wall time per sample (median of --reps);
  3. each sample's distance (relative L2 of the decoded image) to a DDIM-1000 run from the same noise.  The weights are
     random, so this is only a proxy for sample quality.

Prints the card's name, power limit and maximum SM clock first, then one JSON line per measurement; --out also writes
them to a file.

    python tools/unipc_probe.py [--reps 5] [--out results/unipc_probe.jsonl]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import ctypes as C  # noqa: E402

import torch  # noqa: E402

from generativemodels_b200 import _lib  # noqa: E402
from generativemodels_b200.inferers import LatentDiffusionInferer  # noqa: E402
from generativemodels_b200.networks.nets import AutoencoderKL, DiffusionModelUNet  # noqa: E402
from generativemodels_b200.networks.schedulers import (DDIMScheduler, DPMSolverMultistepScheduler,  # noqa: E402
                                                       UniPCMultistepScheduler)
from tests.golden import configs as G  # noqa: E402


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:          # the timing does not depend on it; say what is missing
        return f"{torch.cuda.get_device_name()} (power limit and clock unknown: {e})"


def time_ms(fn, reps):
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
    return statistics.median(out)


def kernel_times(shape, reps, emit):
    """Device time per launch of the step kernels alone: 20 back-to-back launches between two events."""
    g = torch.Generator(device="cuda").manual_seed(0)
    x, m, last, h0, h1, h2 = (torch.randn(shape, device="cuda", generator=g) for _ in range(6))
    prev, x0, xc = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    lib, stream, n = _lib.require_device(), torch.cuda.current_stream().cuda_stream, x.numel()
    dpm = _lib.DpmCoef(alpha_s=0.5, sigma_s=0.8, c_x=0.9, clip_min=-1, clip_max=1, prediction_type=0)
    dpm.w[0], dpm.w[1] = 0.3, -0.2
    uni = _lib.UniPCCoef(alpha_s=0.5, sigma_s=0.8, c_last=0.9, c_xc=0.95, clip_min=-1, clip_max=1, prediction_type=0)
    for k, w in enumerate((0.2, 0.1, -0.05, 0.01)):
        uni.v[k] = w
    for k, w in enumerate((0.3, -0.2, 0.05)):
        uni.u[k] = w
    ddim = _lib.DdimCoef(sqrt_alpha_prod_t=0.5, sqrt_beta_prod_t=0.8, sqrt_alpha_prod_prev=0.6, dir_coef=0.7,
                         clip_min=-1, clip_max=1)
    hist = (C.c_void_p * 3)(h0.data_ptr(), h1.data_ptr(), h2.data_ptr())
    calls = {
        "DDIM (b200_ddim_step)": (4, lambda: lib.b200_ddim_step(m.data_ptr(), x.data_ptr(), None, C.byref(ddim),
                                                                prev.data_ptr(), x0.data_ptr(), n, stream)),
        "DPM-Solver++ 2M (b200_dpm_solver_step, 1 history tensor)": (
            5, lambda: lib.b200_dpm_solver_step(m.data_ptr(), x.data_ptr(), hist, 1, None, C.byref(dpm),
                                                prev.data_ptr(), x0.data_ptr(), n, stream)),
        "UniPC-2 (b200_unipc_step, last + 2 history tensors)": (
            8, lambda: lib.b200_unipc_step(m.data_ptr(), x.data_ptr(), last.data_ptr(), hist, 2, C.byref(uni),
                                           prev.data_ptr(), x0.data_ptr(), xc.data_ptr(), n, stream)),
        "UniPC-3 (b200_unipc_step, last + 3 history tensors)": (
            9, lambda: lib.b200_unipc_step(m.data_ptr(), x.data_ptr(), last.data_ptr(), hist, 3, C.byref(uni),
                                           prev.data_ptr(), x0.data_ptr(), xc.data_ptr(), n, stream)),
    }
    for label, (streams, fn) in calls.items():
        def twenty():
            for _ in range(20):
                assert fn() == 0
        us = 1e3 * time_ms(twenty, reps) / 20
        emit(dict(what="step_kernel", shape=list(shape), kernel=label, us=us,
                  TB_per_s=streams * 4 * n / (us * 1e-6) / 1e12))


def c2_sampling(reps, emit):
    ae, un = AutoencoderKL(**G.C2_AEKL).eval(), DiffusionModelUNet(**G.C2_UNET).eval()
    G.recipe_state_dict(ae, 7)
    G.recipe_state_dict(un, 8)
    ae, un = ae.cuda(), un.cuda()
    noise = torch.randn(*G.C2_LATENT, generator=torch.Generator().manual_seed(2)).cuda()
    kw = dict(G.C2_SCHEDULER, clip_sample=False)

    def run(sched, n):
        sched.set_timesteps(n)
        inf = LatentDiffusionInferer(sched, scale_factor=1.0)
        out = {}

        def once():
            out["img"] = inf.sample(noise, ae, un, sched, verbose=False)
        return time_ms(once, reps), out["img"]

    ddim1000 = DDIMScheduler(**kw)
    ddim1000.set_timesteps(1000)
    ref = LatentDiffusionInferer(ddim1000, scale_factor=1.0).sample(noise, ae, un, ddim1000, verbose=False)
    runs = [("DDIM", 50, DDIMScheduler(**kw))]
    for n in (10, 20):
        runs += [("DPM-Solver++ 2M", n, DPMSolverMultistepScheduler(**kw)), ("UniPC-2 bh2", n,
                                                                             UniPCMultistepScheduler(**kw))]
    for label, n, sched in runs:
        ms, img = run(sched, n)
        dist = ((img - ref).norm() / ref.norm()).item()
        emit(dict(what="c2_ldm_sample", scheduler=label, steps=n, ms_per_sample=ms, rel_l2_to_ddim1000=dist))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(json.dumps(d))
    print(f"card: {card()}", flush=True)
    with torch.no_grad():
        kernel_times((1, 1, 160, 224, 160), 50, emit)
        c2_sampling(args.reps, emit)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
