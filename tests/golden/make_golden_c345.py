"""BASELINE.json configs[2..4] (C3, C4, C5) through the UNMODIFIED reference on CPU fp32:
    python -m tests.golden.make_golden_c345 [c3] [c4] [c5]

C3  3-D DiffusionModelUNet (256, 256, 512), attention (F, F, T), head 512 — the bench's headline model — on the
    tutorial volume 1x1x32x40x32: one forward at t = 500 and DiffusionInferer.sample with DDIM-5.
C4  3-D VQVAE (256, 256), 256 codes of dimension 32, on 1x1x64^3: encoder output, code indices, best/second-best
    distance margins (so the CUDA twin can tell a rounding flip at a near-tie from a wrong index), reconstruction.
C5  ControlNet + conditioned 2-D UNet at 3x256x256: one classifier-free-guidance DDIM step (guidance 7, context
    [-1, +1], disc mask as control image), T = 16 384 self-attention at 128^2.
Weights come from tests.golden.configs.recipe_state_dict (seeds 13 / 14 / 15, 16; not committed)."""
import sys
import time
from pathlib import Path

import torch

from tests import golden
from tests.golden import configs as G      # before the reference import: /root/reference has its own `tests` package
from oracle import ref_import

OUT = Path(__file__).resolve().parent


def make_c3():
    from generative.inferers import DiffusionInferer
    from generative.networks.nets import DiffusionModelUNet
    from generative.networks.schedulers import DDIMScheduler
    m = DiffusionModelUNet(**G.C3_UNET).eval()
    G.recipe_state_dict(m, 13)
    s = DDIMScheduler(**G.C3_SCHEDULER)
    s.set_timesteps(G.C3_STEPS)
    torch.manual_seed(1313)
    noise = torch.randn(G.C3_SHAPE)
    with torch.no_grad():
        y500 = m(noise, torch.Tensor((500,)))
        sample, inter = DiffusionInferer(s).sample(input_noise=noise, diffusion_model=m, scheduler=s, verbose=False,
                                                   save_intermediates=True, intermediate_steps=1)
    golden.save(dict(noise=noise, y500=y500, sample=sample, intermediates=inter, timesteps=[int(t) for t in s.timesteps],
                    n_params=sum(p.numel() for p in m.parameters())), "g_c3")
    print("g_c3.pt", (OUT / "g_c3.pt").stat().st_size, float(y500.abs().mean()), float(sample.abs().mean()))


def make_c4():
    from generative.networks.nets import VQVAE
    m = VQVAE(**G.C4_VQVAE).eval()
    G.recipe_state_dict(m, 14)
    torch.manual_seed(1414)
    x = torch.rand(G.C4_SHAPE)
    with torch.no_grad():
        z = m.encode(x)
        idx = m.index_quantize(x)
        recon, loss = m(x)
        cb = m.quantizer.quantizer.embedding.weight
        flat = z.permute(0, 2, 3, 4, 1).reshape(-1, z.shape[1])
        d = (flat ** 2).sum(1, keepdim=True) + (cb.t() ** 2).sum(0, keepdim=True) - 2 * flat @ cb.t()
        two = torch.topk(-d, 2, dim=1)[0]
        margin = (two[:, 0] - two[:, 1]).reshape(idx.shape)          # >= 0: distance gap second-best minus best
        assert torch.equal(torch.max(-d, 1)[1].reshape(idx.shape), idx)
        recon_from_idx = m.decode_samples(idx)
    golden.save(dict(x=x, z=z, indices=idx, margin=margin, recon=recon, loss=loss, recon_from_idx=recon_from_idx,
                    n_params=sum(p.numel() for p in m.parameters())), "g_c4")
    print("g_c4.pt", (OUT / "g_c4.pt").stat().st_size, float(recon.abs().mean()), int(idx.unique().numel()),
          float(margin.min()), float(margin.median()))


def make_c5():
    from generative.networks.nets import ControlNet, DiffusionModelUNet
    from generative.networks.schedulers import DDIMScheduler
    unet = DiffusionModelUNet(**G.C5_UNET).eval()
    cn = ControlNet(**G.C5_CONTROLNET).eval()
    G.recipe_state_dict(unet, 15)
    G.recipe_state_dict(cn, 16)
    s = DDIMScheduler(num_train_timesteps=1000)
    s.set_timesteps(50)
    t = int(s.timesteps[G.C5_T_INDEX])
    torch.manual_seed(1515)
    x = torch.randn(G.C5_SHAPE)
    mask = G.c5_mask()
    ctx = torch.cat([-1 * torch.ones(1, 1, 1), torch.ones(1, 1, 1)], dim=0)
    with torch.no_grad():
        x2 = torch.cat([x] * 2)
        ts = torch.Tensor((t,))
        down, mid = cn(x=x2, timesteps=ts, controlnet_cond=torch.cat([mask] * 2), context=ctx)
        eps2 = unet(x2, timesteps=ts, context=ctx, down_block_additional_residuals=down,
                    mid_block_additional_residual=mid)
        eu, et = eps2.chunk(2)
        eps = eu + G.C5_GUIDANCE * (et - eu)
        nxt, _ = s.step(eps, t, x)
    golden.save(dict(x=x, t=t, eps2=eps2, eps=eps, nxt=nxt, mid_mean=mid.mean((2, 3)), down_means=[d.mean((2, 3)) for d in down],
                    n_params=(sum(p.numel() for p in unet.parameters()), sum(p.numel() for p in cn.parameters()))),
               "g_c5")
    print("g_c5.pt", (OUT / "g_c5.pt").stat().st_size, float(eps2.abs().mean()), float(nxt.abs().mean()))


def main():
    ref_import.import_reference()
    which = [a.lower() for a in sys.argv[1:]] or ["c3", "c4", "c5"]
    for name, fn in (("c3", make_c3), ("c4", make_c4), ("c5", make_c5)):
        if name in which:
            t0 = time.time()
            fn()
            print(f"  {name}: {time.time() - t0:.1f} s")


if __name__ == "__main__":
    main()
