"""App edge of the sampling path (SURVEY.md §8f rank 4): the reference's brain-LDM model-zoo bundle
(model-zoo/models/brain_image_synthesis_latent_diffusion_model) running on this package's classes — its ``Sampler`` and
``NiftiSaver`` scripts, a resolver for the bundle's ``inference.json`` and a pre-packed weight cache file."""
from .config import BundleConfig
from .packed_cache import fingerprint, load_packed, save_packed
from .sampler import Sampler
from .saver import NiftiSaver, nifti1_bytes

__all__ = ["BundleConfig", "Sampler", "NiftiSaver", "nifti1_bytes", "save_packed", "load_packed", "fingerprint"]
