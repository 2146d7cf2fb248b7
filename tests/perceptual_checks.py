"""Shared by the perceptual tests: the fixture's networks (product and torchvision oracle), the distance delta
between two feature networks, and the tolerances.

delta is the RMS over pixels of the distance between two networks' channel-normalised features of the inputs, summed
over the two inputs.  With A, B the normalised feature maps of the two inputs, sqrt(L) is an L2 norm of A - B over
pixels and channels, so the triangle inequality gives |sqrt(L) - sqrt(L_ref)| <= delta, i.e.
|L - L_ref| <= 2 sqrt(L_ref) delta + delta^2.  The tests hold the product's delta against the reference network to
DELTA_MAX, a fixed ceiling per storage flavour, and the loss to the bound at DELTA_MAX, so neither tolerance grows
with the product's own error.

Tolerances per storage flavour, from the fixture network's measured errors with headroom (DESIGN.md section 2 records
the measurements): features relative L2 / normalised max-abs, DELTA_MAX, and (fp16 only) the loss's relative error.
The wiring mutants of tests/golden/make_golden_perceptual.py are 0.13-0.30 off in features and 0.27-0.61 in delta,
outside every one of them."""
import math

import torch

from generativemodels_b200 import ops
from generativemodels_b200.losses import PerceptualLoss
from oracle import perceptual_oracle as O
from tests.golden import make_golden_perceptual as G

FP16 = ops.H16 == torch.float16
FEATURE_TOL = (5e-3, 1e-2) if FP16 else (2e-2, 4e-2)
DELTA_MAX = 1e-2 if FP16 else 5e-2
LOSS_REL_TOL = 5e-3 if FP16 else None


def networks(fixture, device="cpu", **kw):
    """(product PerceptualLoss loaded from the fixture, oracle torchvision ResNet-50) on `device`."""
    net = G.network(fixture)
    m = PerceptualLoss(network_type="resnet50", pretrained=False, **{"spatial_dims": 2, **kw})
    m.load_state_dict(G.loss_state_dict(net), strict=True)
    return m.to(device).eval(), net.to(device)


def product_features(m):
    return lambda z: m.perceptual_function.model(z)["layer4.2.relu_2"]


def oracle_features(net):
    return lambda z: O.features(net, z)


def delta(fa, fb, x, y):
    """RMS over pixels of |normalised fa features - normalised fb features| (fa, fb: z-scored images -> features),
    summed over x and y."""
    d = 0.0
    for t in (x, y):
        if t.shape[1] == 1:
            t = t.repeat(1, 3, 1, 1)
        z = O.zscore(t.float())
        d += math.sqrt(float(((O.normalize(fa(z)) - O.normalize(fb(z))) ** 2).sum(1).mean()))
    return d


def loss_bound(l_ref: float, d: float = DELTA_MAX) -> float:
    return 2 * math.sqrt(max(l_ref, 0.0)) * d + d * d
