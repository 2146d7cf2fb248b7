from .autoencoderkl import AutoencoderKL  # noqa: F401
from .controlnet import ControlNet  # noqa: F401
from .diffusion_model_unet import DiffusionModelUNet  # noqa: F401
from .vqvae import VQVAE  # noqa: F401
from .spade_diffusion_model_unet import SPADEDiffusionModelUNet  # noqa: F401
from .spade_autoencoderkl import SPADEAutoencoderKL  # noqa: F401
from .transformer import DecoderOnlyTransformer  # noqa: F401
from .spade_network import SPADENet  # noqa: F401
from .patchgan_discriminator import MultiScalePatchDiscriminator, PatchDiscriminator  # noqa: F401
