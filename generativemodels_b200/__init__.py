"""generativemodels_b200 — H100-native (sm_90a) diffusion sampling behind the MONAI GenerativeModels API.

Only the sampling hot path is implemented (SURVEY.md §8): DiffusionModelUNet / ControlNet / AutoencoderKL / VQVAE
forward, DDPM / DDIM / PNDM scheduler steps and the Diffusion / LatentDiffusion / ControlNet inferers' ``sample``.
All arithmetic runs in ``lib/libb200gen.so`` (hand-written CUDA, C-ABI in ``include/b200gen.h``).
"""
__version__ = "0.1.0"


def invalidate_packed(module):
    """Drop the packed-weight / captured-graph caches under ``module`` — needed only after writing weights through
    ``param.data`` (EMA swaps), which PyTorch's version counters do not see; see networks/_holders.py."""
    from .networks._holders import invalidate_packed as _f
    return _f(module)
