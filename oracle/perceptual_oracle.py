"""Torch restatement of the reference's PerceptualLoss for network_type="resnet50" (generative/losses/perceptual.py):
torchvision's ResNet-50 run to layer4 in fp32 with the reference's input and distance arithmetic.  Pinned against the
unmodified reference by tests/test_perceptual_oracle_vs_reference.py; runs wherever torchvision does (no reference
checkout needed)."""
import torch

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


def zscore(x: torch.Tensor) -> torch.Tensor:
    """torchvision_zscore_norm on a copy (the reference writes into its argument)."""
    x = x.clone()
    for c in range(3):
        x[:, c, :, :] = (x[:, c, :, :] - MEAN[c]) / STD[c]
    return x


def features(net, x: torch.Tensor) -> torch.Tensor:
    """layer4.2.relu_2 of a torchvision ResNet-50 (eval mode) for a z-scored [N, 3, H, W] input."""
    h = net.maxpool(net.relu(net.bn1(net.conv1(x))))
    return net.layer4(net.layer3(net.layer2(net.layer1(h))))


def normalize(f: torch.Tensor, eps: float = 1e-10) -> torch.Tensor:
    return f / (torch.sqrt(torch.sum(f ** 2, dim=1, keepdim=True)) + eps)


def similarity(net, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """TorchvisionModelPerceptualSimilarity.forward: per-image values [B, 1, 1, 1]."""
    if x.shape[1] == 1 and y.shape[1] == 1:
        x, y = x.repeat(1, 3, 1, 1), y.repeat(1, 3, 1, 1)
    fx, fy = normalize(features(net, zscore(x))), normalize(features(net, zscore(y)))
    return ((fx - fy) ** 2).sum(dim=1, keepdim=True).mean([2, 3], keepdim=True)


def slices(x: torch.Tensor, axis: int) -> torch.Tensor:
    """The reference's batchify_axis: [B * extent(axis), C, rest...] in permute(0, axis, 1, rest) order."""
    rest = [a for a in (2, 3, 4) if a != axis]
    s = x.float().permute((0, axis, 1, *rest)).contiguous()
    return s.view(-1, x.shape[1], x.shape[rest[0]], x.shape[rest[1]])


def loss(net, x: torch.Tensor, y: torch.Tensor, spatial_dims: int, ratio: float = 0.5) -> torch.Tensor:
    """PerceptualLoss.forward (2-D, or 2.5-D for spatial_dims=3), drawing the slices from the CPU default generator."""
    if spatial_dims == 2:
        return torch.mean(similarity(net, x, y))
    means = []
    for axis in (2, 3, 4):
        xs = slices(x, axis)
        idx = torch.randperm(xs.shape[0])[: int(xs.shape[0] * ratio)].to(xs.device)
        means.append(torch.mean(similarity(net, xs.index_select(0, idx), slices(y, axis).index_select(0, idx))))
    return torch.mean(means[0] + means[2] + means[1])
