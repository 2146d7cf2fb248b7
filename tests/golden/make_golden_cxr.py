"""Generate tests/golden/g_bundle_cxr_ldm.pt by running the UNMODIFIED reference — its networks, its DDIMScheduler and
the chest X-ray bundle's own scripts/sampler.py (model-zoo/models/cxr_image_synthesis_latent_diffusion_model) — on CPU
fp32 over the MONAI shim:      python -m tests.golden.make_golden_cxr

The networks and the scheduler are the bundle's configs/inference.json at its published size (stored verbatim as
tests/golden/cxr_ldm_inference.json): 2-D UNet (256, 512, 768) with heads (0, 512, 768) and cross-attention over a
(2, 77, 1024) context, 4-level 2-D AutoencoderKL (64, 128, 128, 128).  Weights come from
tests.golden.configs.recipe_state_dict (seeds 17 / 18; not committed), which redraws every tensor, the zero-initialised
output convolutions included.  The prompt embeddings are seeded normal draws of the CLIP output's shape; the noise is
the file's own ``torch.randn((1, 3, 64, 64))``; CXR_STEPS DDIM v-prediction steps of the file's schedule.  Stored: the
inputs, the UNet output of every step (uncond | text halves), the latent after every step and the decoded image.
"""
import importlib.util
import json
import time
from pathlib import Path

import torch

from tests import golden
from tests.golden import configs as G      # before the reference import: the reference checkout has its own `tests` package
from oracle import ref_import

OUT = Path(__file__).resolve().parent
BUNDLE = ref_import.REF_ROOT / "model-zoo/models/cxr_image_synthesis_latent_diffusion_model"
CXR_STEPS = 3
UNET_SEED, AEKL_SEED = 17, 18


def bundle_defs():
    """Constructor kwargs of the two networks and the scheduler, read from the stored inference.json."""
    cfg = json.loads((OUT / "cxr_ldm_inference.json").read_text())
    strip = lambda d: {k: v for k, v in d.items() if not k.startswith("_")}          # noqa: E731
    return strip(cfg["autoencoder_def"]), strip(cfg["diffusion_def"]), strip(cfg["scheduler"])


def main():
    ref_import.import_reference()
    from generative.networks.nets import AutoencoderKL, DiffusionModelUNet
    from generative.networks.schedulers import DDIMScheduler
    spec = importlib.util.spec_from_file_location("cxr_bundle_sampler", BUNDLE / "scripts/sampler.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)

    aekl_kwargs, unet_kwargs, sched_kwargs = bundle_defs()
    ae = AutoencoderKL(**aekl_kwargs).eval()
    unet = DiffusionModelUNet(**unet_kwargs).eval()
    G.recipe_state_dict(unet, UNET_SEED)
    G.recipe_state_dict(ae, AEKL_SEED)
    scheduler = DDIMScheduler(**sched_kwargs)
    scheduler.set_timesteps(num_inference_steps=CXR_STEPS)
    torch.manual_seed(1717)
    prompt_embeds = torch.randn(2, 77, 1024)
    torch.manual_seed(1818)
    noise = torch.randn((1, 3, 64, 64))

    # record what the unmodified Sampler feeds through: the UNet output and the scheduler's next latent of every step
    outputs, latents = [], []
    forward, step = unet.forward, scheduler.step

    def rec_forward(*a, **k):
        y = forward(*a, **k)
        outputs.append(y.clone())
        return y

    def rec_step(*a, **k):
        nxt, x0 = step(*a, **k)
        latents.append(nxt.clone())
        return nxt, x0
    unet.forward, scheduler.step = rec_forward, rec_step
    t0 = time.time()
    image = mod.Sampler().sampling_fn(noise, ae, unet, scheduler, prompt_embeds)
    assert len(outputs) == len(latents) == CXR_STEPS and tuple(image.shape) == (1, 1, 512, 512)
    golden.save(dict(aekl_kwargs=aekl_kwargs, unet_kwargs=unet_kwargs, scheduler_kwargs=sched_kwargs,
                     steps=CXR_STEPS, unet_seed=UNET_SEED, aekl_seed=AEKL_SEED,
                     timesteps=[int(t) for t in scheduler.timesteps], guidance_scale=7.0, scale_factor=0.3,
                     n_params=(sum(p.numel() for p in unet.parameters()), sum(p.numel() for p in ae.parameters())),
                     noise=noise, prompt_embeds=prompt_embeds, model_outputs=outputs, latents=latents, image=image),
                "g_bundle_cxr_ldm")
    f = OUT / "g_bundle_cxr_ldm.pt"
    print(f.name, f"{time.time() - t0:.1f} s", [float(x.abs().mean()) for x in latents], float(image.abs().mean()),
          float(image.min()), float(image.max()))


if __name__ == "__main__":
    main()
