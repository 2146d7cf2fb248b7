"""Generate tests/golden/g_bundle_mednist_ddpm.pt by running the UNMODIFIED reference — its DiffusionModelUNet,
DDPMScheduler and DiffusionInferer.sample — on CPU fp32 over the MONAI shim:      python -m tests.golden.make_golden_mednist

The network and the scheduler are the MedNIST DDPM bundle's (model-zoo/models/mednist_ddpm) configs/common.yaml, stored
verbatim as tests/golden/mednist_ddpm_common.yaml next to its infer.yaml and metadata.json: a 2-D UNet (64, 128, 128)
with attention at the two lower levels (head 128) and DDPMScheduler(num_train_timesteps=1000) without set_timesteps,
so one sample is 1000 DDPM steps.  Weights come from tests.golden.configs.recipe_state_dict (seed UNET_SEED; not
committed).  As the bundle's ``testing`` item runs it: ``torch.manual_seed(SEED)``, the file's own
``torch.rand(1, 1, 64, 64)`` noise, then ``inferer.sample(input_noise=x, diffusion_model=network, scheduler=scheduler)``,
whose DDPM steps draw their noise from the global CPU generator.  Stored: the noise, the UNet input, output and the
scheduler's next sample at the PROBE_T timesteps (for teacher forcing), the sample after the step at every timestep
divisible by 100 (nine intermediates and the final image) and the final image.  About a minute on 8 cores.
"""
import time
from pathlib import Path

import torch

from tests import golden
from tests.golden import configs as G      # before the reference import: the reference checkout has its own `tests` package
from oracle import ref_import

OUT = Path(__file__).resolve().parent
STEM = "g_bundle_mednist_ddpm"
PROBE_T = (999, 900, 750, 500, 250, 100, 1, 0)
EVERY = 100
UNET_SEED, SEED = 19, 2718


def bundle_defs():
    """Constructor kwargs of the network and the scheduler, read from the stored common.yaml."""
    import yaml
    cfg = yaml.safe_load((OUT / "mednist_ddpm_common.yaml").read_text())
    unet = {k: v for k, v in cfg["network_def"].items() if not k.startswith("_")}
    assert cfg["scheduler"]["num_train_timesteps"] == "@num_train_timesteps"
    return unet, {"num_train_timesteps": cfg["num_train_timesteps"]}


def main():
    ref_import.import_reference()
    from generative.inferers import DiffusionInferer
    from generative.networks.nets import DiffusionModelUNet
    from generative.networks.schedulers import DDPMScheduler

    unet_kwargs, sched_kwargs = bundle_defs()
    unet = DiffusionModelUNet(**unet_kwargs).eval()
    G.recipe_state_dict(unet, UNET_SEED)
    scheduler = DDPMScheduler(**sched_kwargs)
    assert len(scheduler.timesteps) == 1000

    probes = {t: {} for t in PROBE_T}
    trajectory = []
    forward, step = unet.forward, scheduler.step

    def rec_forward(x, timesteps, *a, **k):
        y = forward(x, timesteps, *a, **k)
        t = int(timesteps[0])
        if t in probes:
            probes[t].update(x=x.clone(), eps=y.clone())
        return y

    def rec_step(model_output, timestep, sample, *a, **k):
        nxt, x0 = step(model_output, timestep, sample, *a, **k)
        t = int(timestep)
        if t in probes:
            probes[t]["next"] = nxt.clone()
        if t % EVERY == 0:
            trajectory.append(nxt.clone())
        return nxt, x0
    unet.forward, scheduler.step = rec_forward, rec_step

    t0 = time.time()
    torch.manual_seed(SEED)
    noise = torch.rand(1, 1, 64, 64)                          # infer.yaml: noise
    image = DiffusionInferer(scheduler).sample(input_noise=noise, diffusion_model=unet, scheduler=scheduler)
    # the whole run drew the noise and one randn per step at t > 0 from the global generator, nothing else
    after = torch.get_rng_state()
    torch.manual_seed(SEED)
    torch.rand(1, 1, 64, 64)
    for _ in range(999):
        torch.randn(1, 1, 64, 64)
    assert torch.equal(after, torch.get_rng_state())
    assert len(trajectory) == 1000 // EVERY and torch.equal(trajectory[-1], image)
    golden.save(dict(unet_kwargs=unet_kwargs, scheduler_kwargs=sched_kwargs, unet_seed=UNET_SEED, seed=SEED,
                     n_params=sum(p.numel() for p in unet.parameters()), probe_t=list(PROBE_T), every=EVERY,
                     noise=noise, probe_x=[probes[t]["x"] for t in PROBE_T],
                     probe_eps=[probes[t]["eps"] for t in PROBE_T], probe_next=[probes[t]["next"] for t in PROBE_T],
                     trajectory=trajectory, image=image), STEM)
    print(STEM, f"{time.time() - t0:.1f} s", sum(p.numel() for p in unet.parameters()), "params;",
          "mean |x| every 100 steps:", [round(float(x.abs().mean()), 4) for x in trajectory],
          "clipped share:", float((image.abs() > 0.999).float().mean()))


if __name__ == "__main__":
    main()
