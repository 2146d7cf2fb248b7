"""PerceptualLoss with ``network_type="resnet50"`` — ``generative/losses/perceptual.py`` on the H100 kernels, forward
only: the distance between two images (2-D) or two volumes (2.5-D, slices along each axis) in the channel-normalised
``layer4`` features of torchvision's ResNet-50, for scoring reconstructions and samples.

Same constructor signature, defaults and exceptions as the reference, the same module tree (``state_dict`` keys
``perceptual_function.model.conv1.weight`` ... ``layer4.2.bn3.*``), and weights acquired through torchvision exactly as
the reference acquires them, so a torchvision ResNet-50 checkpoint or a reference ``PerceptualLoss.state_dict()`` loads
with ``strict=True``.  For 2.5-D the slices are drawn with ``torch.randperm`` on the CPU default generator in the
reference's order (sagittal, coronal, axial), so one seed selects the same slices.

Where the work goes:
- b200_perceptual_prep turns the caller's fp32 / fp16 / bf16 / fp64 tensors of any strides into the network's
  channels-last h16 batch in one launch for both inputs: the 1 -> 3 channel repeat, the ImageNet z-score and, for
  2.5-D, the slice gather;
- the network: the 7x7 stride-2 stem as b200_tap_gather (K = 147) plus one GEMM, max-pool 3x3 s2 p1 on b200_pool_s2,
  and every bottleneck convolution on b200_igemm with its eval-mode BatchNorm folded into the packed weights
  (b200_batchnorm_fold, cached against the parameters and BN buffers, so ``load_state_dict`` repacks), ReLU in the
  epilogue and each block's add + ReLU in conv3's residual epilogue; the last block stores fp32;
- b200_perceptual_distance forms x / (|x| + 1e-10) per pixel in the direct form and the per-image spatial means in
  fp64; b200_perceptual_mean the per-axis means and the loss, without a host synchronisation.
Both inputs run through the network as one batch, and every convolution is one pass (no split reduction) on the
128-column kernel, so a feature vector does not depend on which other images share its batch: ``loss(x, x) == 0`` exactly, repeated calls
are bit-identical and 2.5-D slice chunks of any size give the same result.

Deviations from the reference, by design:
- the caller's tensors are never written (the reference's z-score writes into a 3-channel ``input`` / ``target``);
- a call with grad enabled on an input that requires grad raises ``RuntimeError``: there is no backward pass;
- forward in train mode raises ``RuntimeError`` (BatchNorm would use batch statistics);
- a 2.5-D ratio that selects no slice on some axis raises ``ValueError`` (the reference returns NaN).
"""
from __future__ import annotations

import ctypes

import torch
import torch.nn as nn

from .. import ops
from .._lib import REPACK_TAP_IN
from ..networks._holders import _Cached, on_input_device, require_cuda

__all__ = ["PerceptualLoss", "TorchvisionModelPerceptualSimilarity"]

_FINAL = "layer4.2.relu_2"
# Input pixels (both inputs together) per network pass: bounds the workspace of a 2.5-D volume's slices and large
# 2-D batches.  The peak is at the stem, about 130 bytes of h16 activations per input pixel (the prepared input 16,
# the tap gather 76, the stem's output 32), so about 1 GB per pass; results do not depend on it.
_CHUNK_PIXELS = 1 << 23


def _forward_only(*tensors: torch.Tensor) -> None:
    if torch.is_grad_enabled() and any(t.requires_grad for t in tensors):
        raise RuntimeError("PerceptualLoss on the H100 kernels is forward only (scoring): it has no backward pass. "
                           "Call it under torch.no_grad() or on inputs that do not require grad")


class _ResNet50Features(nn.Module, _Cached):
    """torchvision ResNet-50 up to ``layer4`` (what the reference's ``create_feature_extractor(network,
    ["layer4.2.relu_2"])`` keeps), with torchvision's module names.  ``forward(x)`` takes the z-scored NCHW input and
    returns ``{"layer4.2.relu_2": fp32 NCHW features}``; ``forward_cl`` runs on the channels-last batch."""

    def __init__(self, network: nn.Module):
        super().__init__()
        for name in ("conv1", "bn1", "relu", "maxpool", "layer1", "layer2", "layer3", "layer4"):
            self.add_module(name, getattr(network, name))

    def _packed(self, name: str, conv: nn.Conv2d, bn: nn.BatchNorm2d) -> ops.PackedConv:
        stats = (bn.weight, bn.bias, bn.running_mean, bn.running_var)
        return self._cached(name, (conv.weight, *stats), lambda: ops.PackedConv(
            *ops.batchnorm_fold(conv.weight, None, *stats, bn.eps), conv.stride, conv.padding))

    def _stem(self) -> ops.PackedLinear:
        """conv1 + bn1 as one GEMM over the gathered 7x7x3 taps: [64][tap * 3 + c], K = 147 in three 64-wide chunks."""
        stats = (self.bn1.weight, self.bn1.bias, self.bn1.running_mean, self.bn1.running_var)

        def build():
            w, b = ops.batchnorm_fold(self.conv1.weight, None, *stats, self.bn1.eps)
            w16 = ops.repack(w, 64, 3, 49, None, 64, mode=REPACK_TAP_IN, pitch=192)
            return ops.PackedLinear.from_packed(w16, 64, 147, b)
        return self._cached("stem", (self.conv1.weight, *stats), build)

    def forward_cl(self, x: ops.CL) -> torch.Tensor:
        """z-scored 3-channel h16 images -> fp32 channels-last ``layer4`` features [N, 1, h, w, 2048]."""
        OH, OW = (x.H - 1) // 2 + 1, (x.W - 1) // 2 + 1
        geom = (ctypes.c_int32 * 16)(x.N, 1, x.H, x.W, 1, OH, OW, 1, 7, 7, 1, 2, 2, 0, 3, 3)
        # One kernel variant whatever the batch: no split reduction, and the 128-column kernel only (impl 2), which
        # the planner would otherwise trade for the 128 x 256 one on large batches (the two agree to one ulp, not to
        # the bit).  A feature vector then depends on its own image alone.
        kw = dict(split_k=False, impl=2)
        h = ops.linear(ops.tap_gather(x, geom, 49), self._stem(), act1=ops.ACT_RELU, **kw)
        h = ops.pool_s2(h, 3, 1, "max")
        kw["gn_stats"] = False
        for li in range(1, 5):
            blocks = getattr(self, f"layer{li}")
            for bi, blk in enumerate(blocks):
                pre = f"layer{li}.{bi}."
                last = li == 4 and bi == len(blocks) - 1
                y = ops.conv(h, self._packed(pre + "conv1", blk.conv1, blk.bn1), act1=ops.ACT_RELU, **kw)
                y = ops.conv(y, self._packed(pre + "conv2", blk.conv2, blk.bn2), act1=ops.ACT_RELU, **kw)
                idn = h
                if blk.downsample is not None:
                    idn = ops.conv(h, self._packed(pre + "downsample", blk.downsample[0], blk.downsample[1]), **kw)
                h = ops.conv(y, self._packed(pre + "conv3", blk.conv3, blk.bn3), residual=idn, act2=ops.ACT_RELU,
                             out_f32=last, **kw)
        return h

    @on_input_device
    def forward(self, x: torch.Tensor) -> dict[str, torch.Tensor]:
        require_cuda(x, self)
        _forward_only(x)
        if self.training:
            raise RuntimeError("the ResNet-50 features run the eval-mode BatchNorm only; call .eval()")
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"expected a [N, 3, H, W] input, got shape {tuple(x.shape)}")
        f = self.forward_cl(ops.to_cl(x))
        return {_FINAL: ops.from_cl_f32(f, 2048, 2)}


def _build_resnet50(pretrained: bool, pretrained_path: str | None, pretrained_state_dict_key: str | None):
    """The reference's weight acquisition, through torchvision."""
    from torchvision.models import ResNet50_Weights, resnet50

    if pretrained_path is None:
        return resnet50(weights=ResNet50_Weights.DEFAULT if pretrained else None)
    network = resnet50(weights=None)
    if pretrained is True:
        state_dict = torch.load(pretrained_path)
        if pretrained_state_dict_key is not None:
            state_dict = state_dict[pretrained_state_dict_key]
        network.load_state_dict(state_dict)
    return network


class TorchvisionModelPerceptualSimilarity(nn.Module):
    """Perceptual distance in torchvision ResNet-50 features (reference lines 234-312).  ``forward(input, target)``
    on [B, C, H, W] images in [0, 1] (C = 3, or 1 for both) returns the per-image values, fp32 [B, 1, 1, 1]."""

    def __init__(self, net: str = "resnet50", pretrained: bool = True, pretrained_path: str | None = None,
                 pretrained_state_dict_key: str | None = None) -> None:
        super().__init__()
        supported_networks = ["resnet50"]
        if net not in supported_networks:
            raise NotImplementedError(
                f"'net' {net} is not supported, please select a network from {supported_networks}.")
        network = _build_resnet50(pretrained, pretrained_path, pretrained_state_dict_key)
        self.final_layer = _FINAL
        self.model = _ResNet50Features(network)
        self.eval()
        for param in self.parameters():
            param.requires_grad = False

    def _check(self, input: torch.Tensor, target: torch.Tensor, dims: int) -> int:
        """The channel count the network reads (1 = repeated), after the reference's shape rules."""
        require_cuda(input, self)
        require_cuda(target, self)
        _forward_only(input, target)
        if self.model.training:
            raise RuntimeError("TorchvisionModelPerceptualSimilarity runs the eval-mode BatchNorm only; call .eval()")
        if input.dim() != dims or target.shape != input.shape:
            raise ValueError(f"input and target must be {dims}-D tensors of one shape, got {tuple(input.shape)} and "
                             f"{tuple(target.shape)}")
        if input.shape[1] not in (1, 3):
            raise ValueError(f"the network reads 3 channels (or 1, repeated), got {input.shape[1]}")
        return input.shape[1]

    def per_image(self, x: torch.Tensor, y: torch.Tensor, strides, S: int, OH: int, OW: int,
                  idx: torch.Tensor | None, n: int, image: torch.Tensor, image32: torch.Tensor | None = None) -> None:
        """The n per-image distances of a set of images (see ops.perceptual_prep for the addressing) into
        ``image`` (fp64 [n]) and ``image32``, in chunks of at most _CHUNK_PIXELS input pixels."""
        m_max = max(1, _CHUNK_PIXELS // (2 * OH * OW))
        for b0 in range(0, n, m_max):
            m = min(m_max, n - b0)
            if idx is None:      # 2-D: the chunk's images are a batch slice
                xs, ys, ids = x[b0:b0 + m], y[b0:b0 + m], None
            else:
                xs, ys, ids = x, y, idx[b0:b0 + m]
            buf = torch.empty((2 * m, 1, OH, OW, 8), dtype=ops.H16, device=x.device)
            ops.perceptual_prep(xs, ys, strides, S, OH, OW, ids, m, buf)
            f = self.model.forward_cl(ops.CL(buf, 3, 2))
            ops.perceptual_distance(f[:m], f[m:], 2048, image[b0:b0 + m],
                                    None if image32 is None else image32[b0:b0 + m])

    @on_input_device
    def forward(self, input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        self._check(input, target, 4)
        B, _, H, W = input.shape
        strides = [(s[0], s[1], 0, s[2], s[3]) for s in (input.stride(), target.stride())]
        image = torch.empty(B, dtype=torch.float64, device=input.device)
        image32 = torch.empty(B, dtype=torch.float32, device=input.device)
        self.per_image(input, target, strides, 1, H, W, None, B, image, image32)
        return image32.view(B, 1, 1, 1)


class PerceptualLoss(nn.Module):
    """Perceptual loss (reference lines 21-131) for ``network_type="resnet50"``: 2-D, or 3-D with ``is_fake_3d=True``
    (2.5-D: ``int(n * fake_3d_ratio)`` random slices of the n = B * extent slices along each spatial axis, the loss the
    sum of the three axis means).  ``forward(input, target)`` returns the fp32 0-dim loss."""

    def __init__(self, spatial_dims: int, network_type: str = "alex", is_fake_3d: bool = True,
                 fake_3d_ratio: float = 0.5, cache_dir: str | None = None, pretrained: bool = True,
                 pretrained_path: str | None = None, pretrained_state_dict_key: str | None = None):
        super().__init__()
        if spatial_dims not in [2, 3]:
            raise NotImplementedError("Perceptual loss is implemented only in 2D and 3D.")
        if (spatial_dims == 2 or is_fake_3d) and "medicalnet_" in network_type:
            raise ValueError(
                "MedicalNet networks are only compatible with ``spatial_dims=3``."
                "Argument is_fake_3d must be set to False.")
        if spatial_dims == 3 and is_fake_3d is False:
            raise NotImplementedError(f"network_type={network_type!r} with spatial_dims=3 and is_fake_3d=False (the "
                                      "MedicalNet 3-D networks) is not supported on the CUDA path; the supported "
                                      "network is 'resnet50' in 2-D or 2.5-D (is_fake_3d=True)")
        if network_type != "resnet50":
            raise NotImplementedError(f"network_type={network_type!r} is not supported on the CUDA path (its "
                                      "architecture and weights are downloads); the supported network is 'resnet50'")
        if cache_dir:
            torch.hub.set_dir(cache_dir)
        self.spatial_dims = spatial_dims
        self.perceptual_function = TorchvisionModelPerceptualSimilarity(
            net=network_type, pretrained=pretrained, pretrained_path=pretrained_path,
            pretrained_state_dict_key=pretrained_state_dict_key)
        self.is_fake_3d = is_fake_3d
        self.fake_3d_ratio = fake_3d_ratio

    def _fake_3d(self, input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        pf = self.perceptual_function
        B, _, *ext = input.shape
        plans = []
        for axis in (2, 3, 4):         # sagittal, coronal, axial: the reference's order of randperm draws
            rest = [a for a in (2, 3, 4) if a != axis]
            n = B * input.shape[axis]
            keep = torch.randperm(n)[: int(n * self.fake_3d_ratio)]
            if keep.numel() == 0:
                raise ValueError(f"fake_3d_ratio={self.fake_3d_ratio} selects no slice of the {n} along axis {axis}")
            strides = [(s[0], s[1], s[axis], s[rest[0]], s[rest[1]]) for s in (input.stride(), target.stride())]
            plans.append((strides, input.shape[axis], input.shape[rest[0]], input.shape[rest[1]], keep))
        counts = [p[-1].numel() for p in plans]
        image = torch.empty(sum(counts), dtype=torch.float64, device=input.device)
        o = 0
        for (strides, S, OH, OW, keep), k in zip(plans, counts):
            pf.per_image(input, target, strides, S, OH, OW, keep.to(input.device), k, image[o:o + k])
            o += k
        return ops.perceptual_mean(image, counts)[1]

    @on_input_device
    def forward(self, input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        if target.shape != input.shape:
            raise ValueError(f"ground truth has differing shape ({target.shape}) from input ({input.shape})")
        pf = self.perceptual_function
        if self.spatial_dims == 3 and self.is_fake_3d:
            pf._check(input, target, 5)
            return self._fake_3d(input, target)
        pf._check(input, target, 4)
        B, _, H, W = input.shape
        strides = [(s[0], s[1], 0, s[2], s[3]) for s in (input.stride(), target.stride())]
        image = torch.empty(B, dtype=torch.float64, device=input.device)
        pf.per_image(input, target, strides, 1, H, W, None, B, image)
        return ops.perceptual_mean(image, [B])[1]
