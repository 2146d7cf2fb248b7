"""App edge of the sampling path (SURVEY.md §8f rank 4): the reference's three model-zoo bundles running on this
package's classes — the brain-LDM bundle (model-zoo/models/brain_image_synthesis_latent_diffusion_model: its
``Sampler`` and ``NiftiSaver`` scripts), the chest X-ray text-to-image bundle (model-zoo/models/
cxr_image_synthesis_latent_diffusion_model: its guided ``Sampler`` and ``JPGSaver``) and the MedNIST DDPM bundle
(model-zoo/models/mednist_ddpm: no scripts on the sampling path) — a resolver for the bundles' configs (JSON, or YAML
files merged in order) and a pre-packed weight cache file."""
from .config import BundleConfig
from .cxr_sampler import Sampler as CXRSampler
from .packed_cache import fingerprint, load_packed, save_packed
from .sampler import Sampler
from .saver import JPGSaver, NiftiSaver, nifti1_bytes

__all__ = ["BundleConfig", "Sampler", "CXRSampler", "NiftiSaver", "JPGSaver", "nifti1_bytes", "save_packed",
           "load_packed", "fingerprint"]
