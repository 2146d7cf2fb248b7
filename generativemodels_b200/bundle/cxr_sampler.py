"""``Sampler`` of the chest X-ray text-to-image bundle (model-zoo/models/cxr_image_synthesis_latent_diffusion_model/
scripts/sampler.py:11-43): classifier-free-guided DDIM over a 2-D latent UNet that cross-attends to CLIP prompt
embeddings, then the autoencoder's ``decode_stage_2_outputs`` of ``latent / scale_factor``.  Same class name and
``sampling_fn`` signature, so the bundle's ``inference.json`` runs unchanged through
:mod:`generativemodels_b200.bundle.config` (``bundle="cxr"``).

Every step runs the UNet once on the latent doubled to batch 2 against the (2, 77, 1024) context — row 0 the empty
prompt, row 1 the user's — and combines the halves as ``uncond + g * (text - uncond)`` in fp32 tensor ops, in the
reference's order.  On a CUDA device the UNet is replayed from a CUDA graph captured once at batch 2.  The reference
decodes under ``autocast``; here the decoder is 16-bit with fp32 accumulation like every other network, so no autocast
context is used.

The bundle's ``inference.json`` calls ``sampling_fn(@noise, @autoencoder, @diffusion, @scheduler, @prompt_embeds)``:
its ``guidance_scale`` item is never passed, so the guidance is always the default 7.0 and ``--guidance_scale`` has no
effect.  This is the reference's behaviour and it is kept.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .sampler import GraphedUNetSampler


class Sampler(GraphedUNetSampler):
    @torch.no_grad()
    def sampling_fn(self, noise: torch.Tensor, autoencoder_model: nn.Module, diffusion_model: nn.Module,
                    scheduler: nn.Module, prompt_embeds: torch.Tensor, guidance_scale: float = 7.0,
                    scale_factor: float = 0.3) -> torch.Tensor:
        network = self._network(diffusion_model, noise.device)
        for t in scheduler.timesteps:
            ts = torch.Tensor((t,)).to(noise.device).long()
            model_output = network(torch.cat([noise] * 2), timesteps=ts, context=prompt_embeds)
            noise_pred_uncond, noise_pred_text = model_output.chunk(2)
            noise_pred = noise_pred_uncond + guidance_scale * (noise_pred_text - noise_pred_uncond)
            noise, _ = scheduler.step(noise_pred, t, noise)
        return autoencoder_model.decode_stage_2_outputs(noise / scale_factor)
