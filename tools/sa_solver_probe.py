"""SASolverScheduler on one GPU, with CUDA events:

  1. the step kernel b200_sa_solver_step (corrector and predictor through two earlier estimates, both noise streams:
     seven input streams, three outputs) beside b200_unipc_step (UniPC-2: five input streams, three outputs), at the C3
     volume (1x1x160x224x160) and the C2 latent batch (1x3x64x64): device microseconds per launch (median over 50
     windows of 20 launches) and the fp32 bytes each launch must move over that time;
  2. LatentDiffusionInferer.sample on the C2 networks (2d_ldm_tutorial autoencoder and latent UNet, recipe weights,
     1x3x64x64 latent, decode to 256x256 included) with SA-Solver (predictor 2, corrector 2, default tau) at 10, 20 and
     50 steps: wall time per sample (median of --reps);
  3. the MedNIST DDPM bundle's unmodified YAML configs (random weights: no checkpoint is loaded) with the scheduler's
     _target_ swapped to SASolverScheduler at 50 and 100 steps, against its own DDPMScheduler at 1000 steps: wall time
     of `sample` per image.

Prints the card's name, power limit and maximum SM clock first, then one JSON line per measurement; --out also writes
them to a file.

    python tools/sa_solver_probe.py [--reps 5] [--out results/sa_solver_probe.jsonl]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import ctypes as C  # noqa: E402

import torch  # noqa: E402

from generativemodels_b200 import _lib  # noqa: E402
from generativemodels_b200.inferers import LatentDiffusionInferer  # noqa: E402
from generativemodels_b200.networks.nets import AutoencoderKL, DiffusionModelUNet  # noqa: E402
from generativemodels_b200.networks.schedulers import SASolverScheduler  # noqa: E402
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
    x, m, last, zl, h0, h1, z = (torch.randn(shape, device="cuda", generator=g) for _ in range(7))
    prev, x0, xc = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    lib, stream, n = _lib.require_device(), torch.cuda.current_stream().cuda_stream, x.numel()
    uni = _lib.UniPCCoef(alpha_s=0.5, sigma_s=0.8, c_last=0.9, c_xc=0.95, clip_min=-1, clip_max=1, prediction_type=0)
    sa = _lib.SASolverCoef(alpha_s=0.5, sigma_s=0.8, c_last=0.9, c_zlast=0.3, c_xc=0.95, c_z=0.2, clip_min=-1,
                           clip_max=1, prediction_type=0)
    for k, (v, u) in enumerate(((0.2, 0.3), (0.1, -0.2), (-0.05, 0.05))):
        uni.v[k], uni.u[k], sa.v[k], sa.u[k] = v, u, v, u
    hist = (C.c_void_p * 3)(h0.data_ptr(), h1.data_ptr(), z.data_ptr())
    calls = {
        "UniPC-2 (b200_unipc_step, last + 2 history tensors)": (
            8, lambda: lib.b200_unipc_step(m.data_ptr(), x.data_ptr(), last.data_ptr(), hist, 2, C.byref(uni),
                                           prev.data_ptr(), x0.data_ptr(), xc.data_ptr(), n, stream)),
        "SA-Solver 2/2, tau = 0 (b200_sa_solver_step, last + 1 history tensor)": (
            7, lambda: lib.b200_sa_solver_step(m.data_ptr(), x.data_ptr(), last.data_ptr(), None, hist, 1, None,
                                               C.byref(sa), prev.data_ptr(), x0.data_ptr(), xc.data_ptr(), n, stream)),
        "SA-Solver 2/2, tau > 0 (b200_sa_solver_step, last + 1 history tensor + 2 noise)": (
            9, lambda: lib.b200_sa_solver_step(m.data_ptr(), x.data_ptr(), last.data_ptr(), zl.data_ptr(), hist, 1,
                                               z.data_ptr(), C.byref(sa), prev.data_ptr(), x0.data_ptr(),
                                               xc.data_ptr(), n, stream)),
        "SA-Solver 3/3, tau > 0 (b200_sa_solver_step, last + 2 history tensors + 2 noise)": (
            10, lambda: lib.b200_sa_solver_step(m.data_ptr(), x.data_ptr(), last.data_ptr(), zl.data_ptr(), hist, 2,
                                                z.data_ptr(), C.byref(sa), prev.data_ptr(), x0.data_ptr(),
                                                xc.data_ptr(), n, stream)),
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
    for n in (10, 20, 50):
        sched = SASolverScheduler(**G.C2_SCHEDULER, clip_sample=False)
        sched.set_timesteps(n)
        inf = LatentDiffusionInferer(sched, scale_factor=1.0)
        ms = time_ms(lambda: inf.sample(noise, ae, un, sched, verbose=False), reps)
        emit(dict(what="c2_ldm_sample", scheduler="SA-Solver 2/2, default tau", steps=n, ms_per_sample=ms))


def mednist(reps, emit):
    from generativemodels_b200.bundle.config import BundleConfig
    gold = ROOT / "tests" / "golden"
    configs = [str(gold / "mednist_ddpm_common.yaml"), str(gold / "mednist_ddpm_infer.yaml")]
    imports = ["$import os", "$import datetime", "$import torch", "$import generative",
               "$import torch.distributed as dist"]             # the configs' imports but the bundle's own scripts
    for target, steps in (("DDPMScheduler", 1000), ("SASolverScheduler", 50), ("SASolverScheduler", 100)):
        cfg = BundleConfig(configs, {"imports": imports,
                                     "scheduler#_target_": f"generative.networks.schedulers.{target}"},
                           bundle="mednist_ddpm")
        sched, sample = cfg.get("scheduler"), cfg.get("sample")
        sched.set_timesteps(steps)
        x = cfg.get("noise").to(cfg.get("device"))
        out = []
        for _ in range(reps if steps < 1000 else 2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            img = sample(x)
            torch.cuda.synchronize()
            out.append(1e3 * (time.perf_counter() - t0))
            assert torch.isfinite(img).all()
        emit(dict(what="mednist_bundle_sample", scheduler=type(sched).__name__, steps=steps,
                  ms_per_sample=statistics.median(out)))


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
        kernel_times(G.C2_LATENT, 50, emit)
        c2_sampling(args.reps, emit)
        mednist(args.reps, emit)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
