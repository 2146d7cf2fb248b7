"""Generate the PerceptualLoss fixture (tests/golden/g_perceptual.pt) by running the UNMODIFIED reference
PerceptualLoss(network_type="resnet50", pretrained=False) (the reference checkout named by REFERENCE_DIR, CPU fp32,
MONAI shim plus the stub `lpips` of oracle/monai_shim):   python -m tests.golden.make_golden_perceptual

The network is torchvision's ResNet-50 with its own initialisation under torch.manual_seed(SEED): the convolution
weights are regenerated from the seed by `network` below (a checksum in the fixture catches generator drift) and only
the BatchNorm parameters and buffers are stored.  Those are made well-conditioned: statistics calibrated by four
train-mode passes over smooth random images, then every bottleneck's bn3.weight set to BN3_GAIN (damped residual
branches).  With torchvision's init alone (gain 1) the network is chaotic (1 % input noise already decorrelates the
features and the loss sits near its maximum), and a fixture like that would accept almost any output.  Damped too far
(gain 0.2: loss 6e-5 / 1.4e-3 / 2.3e-2 at 1 / 5 / 20 % noise) it is so contractive that a mis-wired network stays
within the feature tolerance.  Gain 0.7 sits between: the script prints the loss over a noise sweep, and the feature
error of the wiring mutants in `wiring_mutants` (each far outside the 2e-2 relative-L2 network tolerance), which is the
record of that conditioning.

Cases (y = x + noise * N(0, 1) on smooth images x in [0, 1]):
  2d_1ch      B=3, 1 channel, 96 x 80 (the reference repeats it to 3 channels); also the fp32 layer4 features of x
  2d_3ch      B=2, 3 channels, 64 x 64 (the case where the reference z-scores its arguments in place)
  fake3d      1 x 1 x 40 x 48 x 36, fake_3d_ratio 0.5, slices drawn after torch.manual_seed(slice_seed)
  odd         B=2, 1 channel, 77 x 53 (every stride-2 extent rounds down)
Each case stores the inputs, the reference's per-image values (2-D) and its loss.
"""
import copy
import sys

import torch
import torch.nn.functional as F

from oracle import ref_import
from tests.golden import load, save

SEED = 1234
NOISE = {"2d_1ch": 0.05, "2d_3ch": 0.05, "fake3d": 0.05, "odd": 0.02}
SHAPES = {"2d_1ch": (3, 1, 96, 80), "2d_3ch": (2, 3, 64, 64), "fake3d": (1, 1, 40, 48, 36), "odd": (2, 1, 77, 53)}
SLICE_SEED = 7
BN3_GAIN = 0.7


def smooth(shape, gen) -> torch.Tensor:
    """Images (or volumes) in [0, 1]: coarse noise upsampled, so neighbouring pixels correlate like natural images."""
    coarse = torch.rand(*shape[:2], *[max(2, s // 8) for s in shape[2:]], generator=gen)
    mode = "bilinear" if len(shape) == 4 else "trilinear"
    return F.interpolate(coarse, size=shape[2:], mode=mode, align_corners=False)


def conv_checksum(net) -> torch.Tensor:
    ws = [m.weight.detach().double().reshape(-1) for m in net.modules() if isinstance(m, torch.nn.Conv2d)]
    return torch.stack([sum(w.abs().sum() for w in ws), sum((w * torch.arange(w.numel(), dtype=w.dtype).remainder(7)).sum()
                                                             for w in ws)])


def bn_layers(net):
    return [(n, m) for n, m in net.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]


def raw_network():
    from torchvision.models import resnet50
    torch.manual_seed(SEED)
    return resnet50(weights=None)


def calibrate(net) -> None:
    gen = torch.Generator().manual_seed(SEED + 1)
    net.train()
    with torch.no_grad():
        for _ in range(4):
            net(smooth((8, 3, 96, 96), gen) * 2 - 1)
        for layer in (net.layer1, net.layer2, net.layer3, net.layer4):
            for blk in layer:
                blk.bn3.weight.fill_(BN3_GAIN)
    net.eval()


def network(fixture=None):
    """The fixture's ResNet-50 (torchvision, eval mode): conv weights from SEED, BatchNorm from the fixture."""
    fixture = load("g_perceptual") if fixture is None else fixture
    net = raw_network()
    assert torch.allclose(conv_checksum(net), fixture["checksum"], rtol=1e-12, atol=0), "RNG drift in resnet50 init"
    with torch.no_grad():
        for n, m in bn_layers(net):
            for k in ("weight", "bias", "running_mean", "running_var"):
                getattr(m, k).copy_(fixture["bn"][n][k])
    return net.eval()


def wiring_mutants(net):
    """(name, copy of net) for wirings a port could get wrong: the stride of layer2.0 on its 1x1 conv1 instead of the
    3x3 conv2 (torchvision v1 against v1.5), the 3x3 taps of layer1.1.conv2 transposed, layer4.2 without its
    residual branch."""
    m = copy.deepcopy(net)
    m.layer2[0].conv1.stride, m.layer2[0].conv2.stride = (2, 2), (1, 1)
    yield "stride_on_conv1", m
    m = copy.deepcopy(net)
    with torch.no_grad():
        w = m.layer1[1].conv2.weight
        w.copy_(w.transpose(2, 3).clone())
    yield "transposed_taps", m
    m = copy.deepcopy(net)
    m.layer4[2].forward = torch.relu
    yield "no_residual_branch", m


def loss_state_dict(net) -> dict:
    """A PerceptualLoss state_dict for the network (keys perceptual_function.model.*; no fc)."""
    return {"perceptual_function.model." + k: v for k, v in net.state_dict().items() if not k.startswith("fc.")}


def inputs(name: str, noise: float | None = None):
    gen = torch.Generator().manual_seed(SEED + 10 + sorted(SHAPES).index(name))
    x = smooth(SHAPES[name], gen)
    y = x + (NOISE[name] if noise is None else noise) * torch.randn(x.shape, generator=gen)
    return x, y


def main():
    ref_import.import_reference()
    if str(ref_import._SHIM) not in sys.path:       # the stub lpips, also where a real MONAI is installed
        sys.path.insert(0, str(ref_import._SHIM))
    import generative.losses as gl

    net = raw_network()
    calibrate(net)
    fixture = {"seed": SEED, "checksum": conv_checksum(net),
               "bn": {n: {k: getattr(m, k).detach().clone() for k in ("weight", "bias", "running_mean", "running_var")}
                      for n, m in bn_layers(net)}}
    sd = loss_state_dict(net)

    def ref_loss(dims, **kw):
        m = gl.PerceptualLoss(spatial_dims=dims, network_type="resnet50", pretrained=False, **kw)
        m.load_state_dict(sd)
        return m.eval()

    with torch.no_grad():
        for name in SHAPES:
            x, y = inputs(name)
            rec = {"x": x, "y": y}
            if name == "fake3d":
                m3 = ref_loss(3, is_fake_3d=True, fake_3d_ratio=0.5)
                torch.manual_seed(SLICE_SEED)
                rec["loss"] = m3(x.clone(), y.clone())
            else:
                m = ref_loss(2)
                rec["per_image"] = m.perceptual_function(x.clone(), y.clone())
                rec["loss"] = m(x.clone(), y.clone())
            if name == "2d_1ch":
                rec["features"] = m.perceptual_function.model(
                    gl.perceptual.torchvision_zscore_norm(x.repeat(1, 3, 1, 1)))["layer4.2.relu_2"]
            fixture[name] = rec
            print(f"{name}: loss {float(rec['loss']):.6e}")
        m = ref_loss(2)
        for noise in (0.0, 0.01, 0.05, 0.2):
            x, y = inputs("2d_1ch", noise)
            print(f"noise sweep 2d_1ch: {noise:.2f} -> loss {float(m(x, y)):.4e}")
        from oracle import perceptual_oracle as O
        z = O.zscore(fixture["2d_1ch"]["x"].repeat(1, 3, 1, 1))
        f0 = fixture["2d_1ch"]["features"]
        for name, mut in wiring_mutants(net):
            f = O.features(mut, z)
            print(f"wiring mutant {name}: features rel-L2 {float((f - f0).norm() / f0.norm()):.3e}")
    save(fixture, "g_perceptual")


if __name__ == "__main__":
    sys.exit(main())
