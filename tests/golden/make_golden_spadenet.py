"""Generate the SPADENet fixture (tests/golden/g_spadenet.pt + parts) by running the UNMODIFIED reference
(/root/reference, CPU fp32, MONAI shim):   python -m tests.golden.make_golden_spadenet

Weights come from tests.spadenet_oracle.seeded_weights (keyed by parameter name, nothing left at zero), so the fixture
stores inputs and outputs only; segmentation maps are stored as label images.  Cases:
  tutorial   the 2d_spade_gan tutorial's network (128^2, label_nc 6, [16, 32, 64, 128], z 16), VAE mode: mu, logvar,
             the seeded CPU eps, z, the image and the KL term
  ref3d      the reference test's 3-D case (64^3, label_nc 3), VAE mode, same records
  bilinear / bicubic   the reference test's 2-D case with upsampling_mode bilinear / bicubic and last_act None,
             decode(seg, z)
  gan        SPADENet(2, 1, 1, 8, [32, 32], [8, 8], None, False): the GAN-mode output of shape (N, 1, 32, 2048)
"""
import torch

from tests.golden import save
from tests import spadenet_oracle as SO      # before the reference import: /root/reference has its own `tests` package
from oracle import ref_import

CASES = {
    "tutorial": dict(kw=dict(spatial_dims=2, in_channels=1, out_channels=1, label_nc=6, input_shape=[128, 128],
                             num_channels=[16, 32, 64, 128], z_dim=16, is_vae=True), batch=2),
    "ref3d": dict(kw=dict(spatial_dims=3, in_channels=1, out_channels=1, label_nc=3, input_shape=[64, 64, 64],
                          num_channels=[16, 32, 64, 128], z_dim=16, is_vae=True), batch=1),
    "bilinear": dict(kw=dict(spatial_dims=2, in_channels=1, out_channels=1, label_nc=3, input_shape=[64, 64],
                             num_channels=[16, 32, 64, 128], z_dim=16, is_vae=True, upsampling_mode="bilinear",
                             last_act=None), batch=2),
    "bicubic": dict(kw=dict(spatial_dims=2, in_channels=1, out_channels=1, label_nc=3, input_shape=[64, 64],
                            num_channels=[16, 32, 64, 128], z_dim=16, is_vae=True, upsampling_mode="bicubic",
                            last_act=None), batch=2),
    "gan": dict(kw=dict(spatial_dims=2, in_channels=1, out_channels=1, label_nc=8, input_shape=[32, 32],
                        num_channels=[8, 8], z_dim=None, is_vae=False), batch=1),
}


def build(nets, kw):
    kw = dict(kw)
    kw["num_channels"] = list(kw["num_channels"])
    return SO.seeded_weights(nets.SPADENet(**kw)).eval()


def main():
    ref_import.import_reference()
    import generative.networks.nets.spade_network as nets
    out = {}
    for i, (name, case) in enumerate(CASES.items()):
        kw, n = case["kw"], case["batch"]
        m = build(nets, kw)
        shape = kw["input_shape"]
        labels = SO.one_hot_seg(n, kw["label_nc"], shape, seed=i).argmax(1).to(torch.uint8)
        seg = SO.labels_to_onehot(labels, kw["label_nc"])
        rec = dict(kwargs=kw, labels=labels)
        torch.manual_seed(100 + i)
        with torch.no_grad():
            if kw["is_vae"]:
                x = torch.randn(n, kw["in_channels"], *shape)
                mu, logvar = m.encoder(x)
                eps = torch.randn_like(mu)
                z = eps * torch.exp(0.5 * logvar) + mu
                rec.update(x=x, mu=mu, logvar=logvar, eps=eps, z=z, kld=m.kld_loss(mu, logvar), out=m.decode(seg, z))
            else:
                rec.update(out=m(seg)[0])
        out[name] = rec
        print(name, tuple(rec["out"].shape), flush=True)
    save(out, "g_spadenet")


if __name__ == "__main__":
    main()
