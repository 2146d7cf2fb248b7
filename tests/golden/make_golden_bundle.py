"""Generate tests/golden/g_bundle_brain_ldm.pt by running the UNMODIFIED reference — its networks, its DDIMScheduler
and the brain-LDM bundle's own scripts/sampler.py (model-zoo/models/brain_image_synthesis_latent_diffusion_model) —
on CPU fp32 over the MONAI shim:      python -m tests.golden.make_golden_bundle

The architecture is the bundle's configs/inference.json (3-D AutoencoderKL with four levels and no attention; 3-D
UNet with 7 = 3 latent + 4 conditioning input channels, resblock_updown, cross-attention on a length-1 context of
dim 4) at reduced widths so the fixture stays small; 5 DDIM steps of the bundle's schedule.
"""
import importlib.util
from pathlib import Path

import torch

from tests import golden
from tests.golden import configs as G      # before the reference import: /root/reference has its own `tests` package
from oracle import ref_import

OUT = Path(__file__).resolve().parent
BUNDLE = ref_import.REF_ROOT / "model-zoo/models/brain_image_synthesis_latent_diffusion_model"


def main():
    ref_import.import_reference()
    from generative.networks.nets import AutoencoderKL, DiffusionModelUNet
    from generative.networks.schedulers import DDIMScheduler
    spec = importlib.util.spec_from_file_location("bundle_sampler", BUNDLE / "scripts/sampler.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)

    torch.manual_seed(0)
    ae = AutoencoderKL(**G.BUNDLE_AEKL).eval()
    unet = G.randomize_zero_params(DiffusionModelUNet(**G.BUNDLE_UNET)).eval()
    scheduler = DDIMScheduler(**G.BUNDLE_SCHEDULER)
    scheduler.set_timesteps(num_inference_steps=G.BUNDLE_STEPS)
    torch.manual_seed(1)
    noise = torch.randn(G.BUNDLE_NOISE)
    conditioning = torch.tensor([[0.0, 0.1, 0.2, 0.4]]).unsqueeze(1)        # inference.json: gender, age, vols
    sample = mod.Sampler().sampling_fn(noise, ae, unet, scheduler, conditioning)
    golden.save(dict(aekl_kwargs=G.BUNDLE_AEKL, unet_kwargs=G.BUNDLE_UNET, aekl_state=ae.state_dict(),
                    unet_state=unet.state_dict(), noise=noise, conditioning=conditioning, sample=sample),
               "g_bundle_brain_ldm")
    f = OUT / "g_bundle_brain_ldm.pt"
    print(f.name, f.stat().st_size, tuple(sample.shape), float(sample.abs().mean()))


if __name__ == "__main__":
    main()
