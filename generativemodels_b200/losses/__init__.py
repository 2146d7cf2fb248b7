"""The reference's ``generative.losses.PerceptualLoss`` on the CUDA path, forward only (scoring), for
``network_type="resnet50"`` (torchvision's ResNet-50, which runs offline): 2-D, and 2.5-D on 3-D volumes.  The
LPIPS, RadImageNet and MedicalNet networks, whose architectures and weights are downloads, raise
``NotImplementedError``. The adversarial and spectral losses are not part of this package."""
from .perceptual import PerceptualLoss, TorchvisionModelPerceptualSimilarity

__all__ = ["PerceptualLoss", "TorchvisionModelPerceptualSimilarity"]
