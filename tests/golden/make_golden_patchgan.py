"""Generate the PatchGAN discriminator fixture (tests/golden/g_patchgan.pt + parts) by running the UNMODIFIED reference
(/root/reference, CPU fp32, MONAI shim) in eval mode:   python -m tests.golden.make_golden_patchgan

Parameters and BatchNorm statistics come from tests.patchgan_oracle.seeded_weights (keyed by name, nothing left at its
default), so the fixture stores inputs and outputs only.  Inputs are fp16-exact and stored as fp16; the two large ones
are stored at a reduced extent and repeated along every axis (patchgan_oracle.input_of).  Features are stored as fp16,
the patch scores as fp32.  Cases:
  ldm2d        the 2d_ldm tutorial's PatchDiscriminator (BATCH, k4, 64 channels, 3 layers) at 2 x 1 x 64^2
  ldm3d        the 3d_ldm tutorial's 3-D PatchDiscriminator (32 channels) at 1 x 1 x 96 x 96 x 64: scores only
  spade_vae    the 2d_spade_vae tutorial's MultiScalePatchDiscriminator (INSTANCE, k3, 7 -> 7 channels, 2 scales)
               at 1 x 7 x 128^2
  test_2d, test_3d, test_2d_pool, test_3d_pool, test_layer_list
               the reference test file's configurations (INSTANCE, LEAKYRELU, dropout 0.1) at reduced sizes: 2-D
               1 x 3 x 64 x 128 (test_2d 1 x 3 x 128 x 256), 3-D 1 x 3 x 32 x 128 x 32 (test_3d 1 x 3 x 32 x 128 x 128,
               scores only).  Without pooling the second discriminator halves the input six times; the sizes keep
               at least 4 voxels in its deepest InstanceNorm layers (over 2 voxels InstanceNorm returns about +-1,
               with a sign that storage rounding flips where the two values nearly tie)
  test_2d_full test_2d at its real size, 1 x 3 x 256 x 512: scores only
Each case also records its state_dict keys and shapes, and per-tensor float64 sums of the parameters the constructor
draws after torch.manual_seed(0).
"""
import torch

from tests.golden import save
from tests import patchgan_oracle as PO      # before the reference import: /root/reference has its own `tests` package
from oracle import ref_import

_REF = dict(num_d=2, num_layers_d=3, num_channels=8, in_channels=3, out_channels=1, kernel_size=3,
            activation="LEAKYRELU", norm="instance", bias=False, dropout=0.1, minimum_size_im=256)
PD, MS = "PatchDiscriminator", "MultiScalePatchDiscriminator"
CASES = {
    "ldm2d": dict(cls=PD, kw=dict(spatial_dims=2, num_layers_d=3, num_channels=64, in_channels=1, out_channels=1),
                  shape=(2, 1, 64, 64), repeat=1, features=True),
    "ldm3d": dict(cls=PD, kw=dict(spatial_dims=3, num_layers_d=3, num_channels=32, in_channels=1, out_channels=1),
                  shape=(1, 1, 96, 96, 64), repeat=4, features=False),
    "spade_vae": dict(cls=MS, kw=dict(num_d=2, num_layers_d=3, spatial_dims=2, num_channels=8, in_channels=7,
                                      out_channels=7, minimum_size_im=128, norm="INSTANCE", kernel_size=3),
                      shape=(1, 7, 128, 128), repeat=1, features=True),
    "test_2d": dict(cls=MS, kw=dict(_REF, spatial_dims=2), shape=(1, 3, 128, 256), repeat=2, features=True),
    "test_3d": dict(cls=MS, kw=dict(_REF, spatial_dims=3), shape=(1, 3, 32, 128, 128), repeat=4, features=False),
    "test_2d_pool": dict(cls=MS, kw=dict(_REF, num_d=4, spatial_dims=2, pooling_method="avg"), shape=(1, 3, 64, 128),
                         repeat=1, features=True),
    "test_3d_pool": dict(cls=MS, kw=dict(_REF, spatial_dims=3, pooling_method="max"), shape=(1, 3, 32, 128, 32),
                         repeat=2, features=True),
    "test_layer_list": dict(cls=MS, kw=dict(_REF, num_d=3, num_layers_d=[3, 4, 5], spatial_dims=2),
                            shape=(1, 3, 64, 128), repeat=1, features=True),
    "test_2d_full": dict(cls=MS, kw=dict(_REF, spatial_dims=2), shape=(1, 3, 256, 512), repeat=4, features=False),
}


def init_sums(module):
    return {k: torch.stack([v.double().sum(), (v.double() ** 2).sum()]) for k, v in module.state_dict().items()
            if v.is_floating_point()}


def main():
    ref_import.import_reference()
    import generative.networks.nets.patchgan_discriminator as nets
    out = {}
    for i, (name, case) in enumerate(CASES.items()):
        cls, kw, r = getattr(nets, case["cls"]), case["kw"], case["repeat"]
        torch.manual_seed(0)
        m = cls(**kw)
        rec = dict(cls=case["cls"], kwargs=kw, repeat=r, init_sums=init_sums(m),
                   keys=[(k, tuple(v.shape)) for k, v in m.state_dict().items()])
        m = PO.seeded_weights(m).eval()
        g = torch.Generator().manual_seed(100 + i)
        low = case["shape"][:2] + tuple(s // r for s in case["shape"][2:])
        rec["x16"] = torch.randn(low, generator=g).half()
        with torch.no_grad():
            res = m(PO.input_of(rec))
        if case["cls"] == PD:
            scores, feats = res[-1], res[:-1]
        else:
            scores, feats = res
        rec["scores"] = scores
        if case["features"]:
            rec["features"] = [[f.half() for f in fs] for fs in feats] if case["cls"] == MS else [f.half() for f in feats]
        out[name] = rec
        shapes = [tuple(s.shape) for s in scores] if isinstance(scores, list) else tuple(scores.shape)
        print(name, shapes, flush=True)
    save(out, "g_patchgan")


if __name__ == "__main__":
    main()
