"""DPMSolverMultistepScheduler on one GPU, with CUDA events:

  1. the step kernel (b200_dpm_solver_step with 0 and 2 history tensors, and with one plus noise) beside
     b200_ddim_step, at the C3 volume (1x1x160x224x160) and at a C2 latent batch (8x3x64x64): device microseconds per
     launch (median over --reps windows of 20 launches) and the fp32 streams moved per second;
  2. LatentDiffusionInferer.sample on the C2 networks (2d_ldm_tutorial autoencoder and latent UNet, recipe weights,
     1x3x64x64 latent) with DPM-Solver++ 2M at 10, 15, 20 and 25 steps against DDIM-50: wall time per sample (median);
  3. the chest X-ray bundle's guided sampler (bundle.CXRSampler, UNet replayed from its CUDA graph) at its published
     size (the networks of tests/golden/cxr_ldm_inference.json, random weights with zero-initialised tensors redrawn,
     a random (2, 77, 1024) prompt context, v-prediction, 512x512 decode included), the same step counts against
     DDIM-50: wall time per sample (median);
  4. each sample's distance (relative L2 of the decoded image) to a DDIM-1000 run from the same noise.  The weights are
     random, so this is only a proxy for sample quality.

Prints the card's name, power limit and maximum SM clock first, then one JSON line per measurement; --out also writes
them to a file.

    python tools/dpm_solver_probe.py [--reps 5] [--out results/dpm_solver_probe.jsonl]
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
from generativemodels_b200.bundle import CXRSampler  # noqa: E402
from generativemodels_b200.inferers import LatentDiffusionInferer  # noqa: E402
from generativemodels_b200.networks.nets import AutoencoderKL, DiffusionModelUNet  # noqa: E402
from generativemodels_b200.networks.schedulers import DDIMScheduler, DPMSolverMultistepScheduler  # noqa: E402
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
    x, m, h0, h1, z = (torch.randn(shape, device="cuda", generator=g) for _ in range(5))
    prev, x0 = torch.empty_like(x), torch.empty_like(x)
    lib, stream, n = _lib.require_device(), torch.cuda.current_stream().cuda_stream, x.numel()
    dpm = _lib.DpmCoef(alpha_s=0.5, sigma_s=0.8, c_x=0.9, c_z=0.1, clip_min=-1, clip_max=1, prediction_type=0)
    dpm.w[0], dpm.w[1], dpm.w[2] = 0.3, -0.2, 0.05
    ddim = _lib.DdimCoef(sqrt_alpha_prod_t=0.5, sqrt_beta_prod_t=0.8, sqrt_alpha_prod_prev=0.6, dir_coef=0.7,
                         clip_min=-1, clip_max=1)
    hist = (C.c_void_p * 2)(h0.data_ptr(), h1.data_ptr())
    calls = {
        "DDIM (b200_ddim_step)": lambda: lib.b200_ddim_step(m.data_ptr(), x.data_ptr(), None, C.byref(ddim),
                                                            prev.data_ptr(), x0.data_ptr(), n, stream),
        "order 1 (no history)": lambda: lib.b200_dpm_solver_step(m.data_ptr(), x.data_ptr(), hist, 0, None,
                                                                 C.byref(dpm), prev.data_ptr(), x0.data_ptr(), n,
                                                                 stream),
        "3M (two history tensors)": lambda: lib.b200_dpm_solver_step(m.data_ptr(), x.data_ptr(), hist, 2, None,
                                                                     C.byref(dpm), prev.data_ptr(), x0.data_ptr(), n,
                                                                     stream),
        "SDE 2M (history + noise)": lambda: lib.b200_dpm_solver_step(m.data_ptr(), x.data_ptr(), hist, 1,
                                                                     z.data_ptr(), C.byref(dpm), prev.data_ptr(),
                                                                     x0.data_ptr(), n, stream),
    }
    streams = {"DDIM (b200_ddim_step)": 4, "order 1 (no history)": 4, "3M (two history tensors)": 6,
               "SDE 2M (history + noise)": 6}
    for label, fn in calls.items():
        def twenty():
            for _ in range(20):
                assert fn() == 0
        us = 1e3 * time_ms(twenty, reps) / 20
        emit(dict(what="step_kernel", shape=list(shape), kernel=label, us=us,
                  GB_per_s=streams[label] * 4 * n / (us * 1e-6) / 1e9))


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
    runs = [("DDIM", 50, DDIMScheduler(**kw))] + [("DPM-Solver++ 2M", n, DPMSolverMultistepScheduler(**kw))
                                                   for n in (10, 15, 20, 25)]
    for label, n, sched in runs:
        ms, img = run(sched, n)
        dist = ((img - ref).norm() / ref.norm()).item()
        emit(dict(what="c2_ldm_sample", scheduler=label, steps=n, ms_per_sample=ms, rel_l2_to_ddim1000=dist))


def cxr_sampling(reps, emit):
    cfg = json.loads((Path(__file__).resolve().parents[1] / "tests/golden/cxr_ldm_inference.json").read_text())

    def kwargs(item):
        return {k: v for k, v in cfg[item].items() if not k.startswith("_")}
    torch.manual_seed(0)
    ae = AutoencoderKL(**kwargs("autoencoder_def")).cuda().eval()
    unet = DiffusionModelUNet(**kwargs("diffusion_def")).eval()
    for p in unet.parameters():
        if float(p.detach().abs().max()) == 0:
            p.normal_(0, 0.02)
    unet = unet.cuda()
    noise = torch.randn(1, 3, 64, 64, generator=torch.Generator().manual_seed(3)).cuda()
    context = torch.randn(2, 77, 1024, generator=torch.Generator().manual_seed(4)).cuda()
    smp = CXRSampler(use_cuda_graph=True)
    kw = kwargs("scheduler")

    def run(sched, n, reps_):
        sched.set_timesteps(n)
        out = {}

        def once():
            out["img"] = smp.sampling_fn(noise, ae, unet, sched, context)
        return (time_ms(once, reps_) if reps_ else once()), out["img"]

    _, ref = run(DDIMScheduler(**kw), 1000, 0)
    runs = [("DDIM", 50, DDIMScheduler(**kw))] + [("DPM-Solver++ 2M", n, DPMSolverMultistepScheduler(**kw))
                                                   for n in (10, 15, 20, 25)]
    for label, n, sched in runs:
        ms, img = run(sched, n, reps)
        dist = ((img - ref).norm() / ref.norm()).item()
        emit(dict(what="cxr_sample", scheduler=label, steps=n, ms_per_sample=ms, rel_l2_to_ddim1000=dist))


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
        for shape in ((1, 1, 160, 224, 160), (8, 3, 64, 64)):
            kernel_times(shape, 50, emit)
        c2_sampling(args.reps, emit)
        cxr_sampling(args.reps, emit)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
