"""``Sampler`` of the brain-LDM bundle (model-zoo/models/brain_image_synthesis_latent_diffusion_model/scripts/
sampler.py:13-52): DDIM loop over a concat+cross-attention conditioned 3-D latent UNet, then the autoencoder's
``decode_stage_2_outputs``.  Same class name and ``sampling_fn`` signature, so the bundle's ``inference.json`` runs
unchanged through :mod:`generativemodels_b200.bundle.config`.

Performance notes: the latent is 3x20x28x20 (11 200 voxels), so one UNet step is ~250 launches of a few microseconds —
the network is wrapped in a CUDA graph (one capture, 50 replays); the conditioning planes are broadcast once, not per
step; the decoder (15 TFLOP of 64..128-channel 3-D convolutions at up to 160x224x160) runs once on the implicit-GEMM
kernel.  The reference decodes under ``autocast`` (fp16 convolutions); here the decoder is 16-bit (fp16 by default) with fp32 accumulation
like every other network, so no autocast context is needed or used.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ..cuda_graph import GraphedModule, graphed


class GraphedUNetSampler:
    """The UNet replay shared by the bundle samplers: on a CUDA device the diffusion model runs from a CUDA graph
    captured on its first call (one capture per input signature, kept per model); ``use_cuda_graph=False`` runs it
    eagerly.  Both give bit-identical results."""

    def __init__(self, use_cuda_graph: bool = True) -> None:
        super().__init__()
        self.use_cuda_graph = use_cuda_graph
        self._graphed: dict[int, GraphedModule] = {}

    def _network(self, diffusion_model: nn.Module, device: torch.device):
        if not self.use_cuda_graph or device.type != "cuda" or isinstance(diffusion_model, GraphedModule):
            return diffusion_model
        g = self._graphed.get(id(diffusion_model))
        if g is None or g.module is not diffusion_model:
            g = self._graphed[id(diffusion_model)] = graphed(diffusion_model)
        return g


class Sampler(GraphedUNetSampler):
    @torch.no_grad()
    def sampling_fn(self, input_noise: torch.Tensor, autoencoder_model: nn.Module, diffusion_model: nn.Module,
                    scheduler: nn.Module, conditioning: torch.Tensor) -> torch.Tensor:
        network = self._network(diffusion_model, input_noise.device)
        image = input_noise
        # [N, 1, C] -> [N, C, 1, 1, 1] -> one plane per conditioning variable over the latent grid (sampler.py:31-32)
        planes = conditioning.squeeze(1)[(...,) + (None,) * (input_noise.dim() - 2)]
        planes = planes.expand(*planes.shape[:2], *input_noise.shape[2:]).to(input_noise.dtype)
        x = torch.empty(input_noise.shape[0], input_noise.shape[1] + planes.shape[1], *input_noise.shape[2:],
                        dtype=input_noise.dtype, device=input_noise.device)
        x[:, input_noise.shape[1]:] = planes                       # written once; only the latent part changes per step
        for t in scheduler.timesteps:
            x[:, :input_noise.shape[1]] = image
            ts = torch.Tensor((t,)).to(input_noise.device).long()
            model_output = network(x, timesteps=ts, context=conditioning)
            image, _ = scheduler.step(model_output, t, image)
        return autoencoder_model.decode_stage_2_outputs(image)
