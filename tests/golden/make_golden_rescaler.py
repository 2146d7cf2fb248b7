"""Generate the SpatialRescaler fixture (tests/golden/g_spatial_rescaler.pt) by running the UNMODIFIED reference
(/root/reference, CPU fp32, MONAI shim):   python -m tests.golden.make_golden_rescaler

Parameters come from tests.rescaler_oracle.seeded_weights (keyed by name) and inputs from rescaler_oracle.input_of
(seeded, fp16-exact), so the fixture stores outputs only (fp32).  Cases:
  ref_0 .. ref_6   the seven CASES of the reference's tests/test_encoder_modules.py
  nearest_down, nearest_up, area_down, area_up, bicubic_down, bicubic_up
  linear1d, linear1d_mapper   1-D linear without and with a channel mapper (3 -> 5)
  mult_1_7, mult_0_6_1_3      non-integer multipliers, the second per axis with a mapper
  odd_scale, odd_size         a length-17 axis halved by scale_factor=0.5 and by size=8 (the ratios differ)
  stages_2, stages_3          chained stages
  size_mapper_bias            size with a 3 -> 5 mapper and bias=True
  brain_area, brain_trilinear 3-D 160 x 224 x 160 -> the brain-LDM latent grid 20 x 28 x 20
Each case also records its state_dict keys and shapes, and per-tensor float64 sums of the parameters the constructor
draws after torch.manual_seed(0).
"""
import torch

from tests.golden import save
from tests import rescaler_oracle as RO     # before the reference import: /root/reference has its own `tests` package
from oracle import ref_import

_REF_CASES = [
    (dict(spatial_dims=2, n_stages=1, method="bilinear", multiplier=0.5, in_channels=None, out_channels=None), (1, 1, 16, 16)),
    (dict(spatial_dims=2, n_stages=1, method="bilinear", multiplier=0.5, in_channels=3, out_channels=2), (1, 3, 16, 16)),
    (dict(spatial_dims=3, n_stages=1, method="trilinear", multiplier=0.5, in_channels=None, out_channels=None),
     (1, 1, 16, 16, 16)),
    (dict(spatial_dims=3, n_stages=1, method="trilinear", multiplier=0.5, in_channels=3, out_channels=2),
     (1, 3, 16, 16, 16)),
    (dict(spatial_dims=3, n_stages=1, method="trilinear", multiplier=(0.25, 0.5, 0.75), in_channels=3, out_channels=2),
     (1, 3, 20, 20, 20)),
    (dict(spatial_dims=2, n_stages=1, size=(8, 8), method="bilinear", in_channels=3, out_channels=2), (1, 3, 16, 16)),
    (dict(spatial_dims=3, n_stages=1, size=(8, 8, 8), method="trilinear", in_channels=None, out_channels=None),
     (1, 1, 16, 16, 16)),
]
CASES = {f"ref_{i}": dict(kw=kw, shape=shape) for i, (kw, shape) in enumerate(_REF_CASES)}
CASES.update({
    "nearest_down": dict(kw=dict(method="nearest", multiplier=0.5), shape=(2, 3, 17, 15)),
    "nearest_up": dict(kw=dict(method="nearest", multiplier=1.5, in_channels=5, out_channels=3), shape=(1, 5, 10, 13)),
    "area_down": dict(kw=dict(method="area", multiplier=0.5), shape=(2, 5, 16, 21)),
    "area_up": dict(kw=dict(spatial_dims=3, method="area", multiplier=2.5), shape=(1, 3, 4, 6, 5)),
    "bicubic_down": dict(kw=dict(method="bicubic", multiplier=0.5), shape=(1, 3, 20, 17)),
    "bicubic_up": dict(kw=dict(method="bicubic", multiplier=2.0, in_channels=3, out_channels=5), shape=(1, 3, 9, 12)),
    "linear1d": dict(kw=dict(spatial_dims=1, method="linear", multiplier=0.5), shape=(2, 3, 40)),
    "linear1d_mapper": dict(kw=dict(spatial_dims=1, method="linear", multiplier=1.7, in_channels=3, out_channels=5),
                            shape=(2, 3, 23)),
    "mult_1_7": dict(kw=dict(method="bilinear", multiplier=1.7), shape=(1, 3, 13, 18)),
    "mult_0_6_1_3": dict(kw=dict(method="bilinear", multiplier=(0.6, 1.3), in_channels=5, out_channels=3),
                         shape=(2, 5, 21, 14)),
    "odd_scale": dict(kw=dict(spatial_dims=1, method="linear", multiplier=0.5), shape=(1, 3, 17)),
    "odd_size": dict(kw=dict(spatial_dims=1, method="linear", size=8), shape=(1, 3, 17)),
    "stages_2": dict(kw=dict(method="bilinear", n_stages=2, multiplier=0.5), shape=(1, 3, 32, 27)),
    "stages_3": dict(kw=dict(spatial_dims=3, method="trilinear", n_stages=3, multiplier=0.5, in_channels=3,
                             out_channels=5), shape=(1, 3, 24, 32, 20)),
    "size_mapper_bias": dict(kw=dict(method="bilinear", size=(9, 11), in_channels=3, out_channels=5, bias=True),
                             shape=(2, 3, 16, 20)),
    "brain_area": dict(kw=dict(spatial_dims=3, method="area", size=(20, 28, 20), in_channels=None),
                       shape=(1, 1, 160, 224, 160)),
    "brain_trilinear": dict(kw=dict(spatial_dims=3, method="trilinear", size=(20, 28, 20), in_channels=None),
                            shape=(1, 1, 160, 224, 160)),
})


def init_sums(module):
    return {k: torch.stack([v.double().sum(), (v.double() ** 2).sum()]) for k, v in module.state_dict().items()}


def main():
    ref_import.import_reference()
    from monai.networks.layers.factories import Conv
    assert Conv["CONV", 1] is torch.nn.Conv1d, "the MONAI Conv factory must give Conv1d for spatial_dims=1"
    from generative.networks.blocks import SpatialRescaler
    out = {}
    for i, (name, case) in enumerate(CASES.items()):
        kw = case["kw"]
        torch.manual_seed(0)
        m = SpatialRescaler(**kw)
        rec = dict(kwargs=kw, shape=case["shape"], seed=1000 + i, init_sums=init_sums(m),
                   keys=[(k, tuple(v.shape)) for k, v in m.state_dict().items()])
        m = RO.seeded_weights(m).eval()
        with torch.no_grad():
            rec["out"] = m(RO.input_of(rec))
        out[name] = rec
        print(name, tuple(rec["out"].shape), flush=True)
    save(out, "g_spatial_rescaler")


if __name__ == "__main__":
    main()
