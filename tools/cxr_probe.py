"""Dev probe: the chest X-ray text-to-image bundle at its published size — latent 3x64x64 doubled to batch 2 for
classifier-free guidance, UNet (256, 512, 768) with heads (0, 512, 768) cross-attending to a (2, 77, 1024) context,
AutoencoderKL (64, 128, 128, 128) decoding to 1x1x512x512, DDIM-50 v-prediction — through
generativemodels_b200.bundle.CXRSampler on one GPU, random-init weights (zero-initialised tensors redrawn).

Times, with CUDA events after a warm-up sample: the 50-step guided loop with the UNet replayed from its CUDA graph
(decoder replaced by the identity), the decode alone, and the whole sampling_fn.  Each is the median of --repeats runs.
The card's name and power limit are read in the same run.  Prints one JSON line; --out also writes it to a file.

    python tools/cxr_probe.py [--repeats 5] [--out results/cxr_probe.json]
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch

from generativemodels_b200.bundle import CXRSampler
from generativemodels_b200.networks.nets import AutoencoderKL, DiffusionModelUNet
from generativemodels_b200.networks.schedulers import DDIMScheduler

CFG = json.loads((Path(__file__).resolve().parents[1] / "tests/golden/cxr_ldm_inference.json").read_text())
STEPS = 50


def kwargs(item):
    return {k: v for k, v in CFG[item].items() if not k.startswith("_")}


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


class Identity(torch.nn.Module):
    def decode_stage_2_outputs(self, z):
        return z


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("cxr_probe: no CUDA device")
    torch.manual_seed(0)
    ae = AutoencoderKL(**kwargs("autoencoder_def")).cuda().eval()
    unet = redraw(DiffusionModelUNet(**kwargs("diffusion_def"))).cuda().eval()
    sched = DDIMScheduler(**kwargs("scheduler"))
    sched.set_timesteps(num_inference_steps=STEPS)
    noise = torch.randn(1, 3, 64, 64).cuda()
    prompt_embeds = torch.randn(2, 77, 1024).cuda()
    z = torch.randn(1, 3, 64, 64).cuda() / 0.3
    smp = CXRSampler(use_cuda_graph=True)

    smp.sampling_fn(noise, Identity(), unet, sched, prompt_embeds)          # packs the weights, captures the graph
    ae.decode_stage_2_outputs(z)
    torch.cuda.synchronize()
    loop = timed_ms(lambda: smp.sampling_fn(noise, Identity(), unet, sched, prompt_embeds), args.repeats)
    decode = timed_ms(lambda: ae.decode_stage_2_outputs(z), args.repeats)
    whole = timed_ms(lambda: smp.sampling_fn(noise, ae, unet, sched, prompt_embeds), args.repeats)
    res = {"probe": "cxr_ldm", "steps": STEPS, "repeats": args.repeats,
           "unet_params_M": round(sum(p.numel() for p in unet.parameters()) / 1e6, 1),
           "loop_ms_median_min_max": [round(v, 2) for v in loop],
           "unet_step_ms": round(loop[0] / STEPS, 3),
           "decode_ms_median_min_max": [round(v, 2) for v in decode],
           "sampling_fn_ms_median_min_max": [round(v, 2) for v in whole],
           "peak_memory_GiB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), **card()}
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
