"""Checks at BASELINE.json's FULL sizes (config C3: 160 x 224 x 160, T = 89 600 tokens; config C4: 32 768 vectors),
where the CPU oracle cannot run: size-independent properties and cross-implementation agreement on the GPU.

* full-resolution 3x3x3 convolution: the wgmma/TMA kernel against the independent CUDA-core cross-check kernel
  (same bf16 operands, fp32 accumulation) — they share only the parameter block, not the data path;
* full-length attention (one head of 512, 89 600 keys): the flash kernel against the GEMM + softmax + GEMM path on a
  slab of query rows, plus the invariant that rows of softmax sum to one (constant V gives back the constant);
* GroupNorm at full resolution: output statistics per group are (0, 1) before the affine;
* DDIM step: linear in (sample, model_output) for epsilon prediction without clipping, and x0 round trip;
* VQ: quantising codebook rows returns their own index; quantisation is idempotent.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

FULL = (160, 224, 160)


def _ops():
    from generativemodels_b200 import ops
    return ops


def test_conv_fullres_tc_vs_crosscheck(cuda_device):
    ops = _ops()
    torch.manual_seed(0)
    D, H, W = FULL
    C = 256
    a = ops.CL((torch.randn(1, D, H, W, C, device="cuda") * 0.5).to(ops.H16), C, 3)
    w = torch.randn(C, C, 3, 3, 3, device="cuda") / math.sqrt(C * 27)
    b = torch.randn(C, device="cuda")
    pc = ops.PackedConv(w, b, 1, 1)
    y_tc = ops.conv(a, pc, impl=0).t
    # cross-check on a sub-volume that includes every face of the padding (corners, edges) and the interior:
    # run the CUDA-core kernel on crops and compare with the matching region of the full-size result
    for (d0, h0, w0) in ((0, 0, 0), (D - 6, H - 10, W - 12), (77, 100, 64)):
        d1, h1, w1 = min(D, d0 + 6), min(H, h0 + 10), min(W, w0 + 12)
        lo = (max(d0 - 1, 0), max(h0 - 1, 0), max(w0 - 1, 0))
        hi = (min(d1 + 1, D), min(h1 + 1, H), min(w1 + 1, W))
        crop = ops.CL(a.t[:, lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]].contiguous(), C, 3)
        y_ck = ops.conv(crop, pc, impl=1).t
        # interior of the crop result corresponds to [d0:d1, h0:h1, w0:w1] only where the crop edge is the volume edge
        sl_full = (slice(None), slice(d0, d1), slice(h0, h1), slice(w0, w1))
        sl_crop = (slice(None), slice(d0 - lo[0], d1 - lo[0]), slice(h0 - lo[1], h1 - lo[1]), slice(w0 - lo[2], w1 - lo[2]))
        got, want = y_tc[sl_full].float(), y_ck[sl_crop].float()
        err = (got - want).abs().max().item()
        assert err <= 2e-2 * max(1.0, want.abs().max().item()), f"crop {(d0, h0, w0)}: max abs err {err:.3e}"


def test_attention_full_length(cuda_device):
    ops = _ops()
    torch.manual_seed(1)
    T = S = FULL[0] // 4 * FULL[1] // 4 * FULL[2] // 4       # 89 600 tokens at the attention level
    assert T == 89600
    dh = 512
    q = (torch.randn(1, T, dh, device="cuda") * 0.5).to(ops.H16)
    k = (torch.randn(1, S, dh, device="cuda") * 0.5).to(ops.H16)
    v = torch.randn(1, S, dh, device="cuda").to(ops.H16)
    vt = v.transpose(1, 2).contiguous()
    scale = 1 / math.sqrt(dh)
    out = ops.attention(q, k, None, 1, dh, scale, vt=vt)
    assert torch.isfinite(out.float()).all()
    # (a) flash kernel vs the GEMM + softmax + GEMM path on a slab of queries spread over the sequence
    rows = torch.cat([torch.arange(0, 256), torch.arange(44800, 45056), torch.arange(T - 256, T)]).cuda()
    ops_unf = ops
    old = ops._FORCE_UNFUSED_ATTENTION
    ops._FORCE_UNFUSED_ATTENTION = True
    try:
        ref = ops_unf.attention(q[:, rows].contiguous(), k, None, 1, dh, scale, vt=vt)
    finally:
        ops._FORCE_UNFUSED_ATTENTION = old
    got = out[:, rows]
    rel = ((got.float() - ref.float()).norm() / ref.float().norm()).item()
    assert rel < 2e-2, f"flash vs unfused at T = 89600: rel L2 {rel:.3e}"
    # (b) softmax rows sum to one: a constant value matrix must come back unchanged (up to bf16 rounding)
    vc = torch.full((1, dh, S), 0.75, device="cuda", dtype=ops.H16)
    outc = ops.attention(q[:, :1024].contiguous(), k, None, 1, dh, scale, vt=vc)
    assert (outc.float() - 0.75).abs().max().item() < 1e-2


def test_groupnorm_full_resolution_statistics(cuda_device):
    ops = _ops()
    torch.manual_seed(2)
    D, H, W = FULL
    C, G = 256, 32
    x = ops.CL((torch.randn(1, D // 2, H, W, C, device="cuda") * 3 + 1.5).to(ops.H16), C, 3)
    y = ops.groupnorm(x, G, 1e-6, torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")).t.float()
    g = y.view(-1, G, C // G)
    mean = g.mean(dim=(0, 2))
    var = g.var(dim=(0, 2), unbiased=False)
    assert mean.abs().max().item() < 5e-3 and (var - 1).abs().max().item() < 1e-2


def test_ddim_step_properties_full_volume(cuda_device):
    from generativemodels_b200.networks.schedulers import DDIMScheduler
    s = DDIMScheduler(num_train_timesteps=1000, schedule="scaled_linear_beta", beta_start=0.0005, beta_end=0.0195,
                      clip_sample=False)
    s.set_timesteps(50)
    torch.manual_seed(3)
    shape = (1, 1, *FULL)
    x, e = torch.randn(shape, device="cuda"), torch.randn(shape, device="cuda")
    p1, x0 = s.step(e, 500, x)
    p2, _ = s.step(2 * e, 500, 2 * x)
    assert (p2 - 2 * p1).abs().max().item() < 1e-5            # linearity (epsilon prediction, no clipping)
    a_t = s.alphas_cumprod[500]
    assert (x0 * a_t ** 0.5 + (1 - a_t) ** 0.5 * e - x).abs().max().item() < 1e-5   # x0 <-> x_t round trip


def test_vq_properties_full_size(cuda_device):
    from generativemodels_b200.networks.layers import EMAQuantizer
    torch.manual_seed(4)
    q = EMAQuantizer(spatial_dims=3, num_embeddings=256, embedding_dim=32).cuda().eval()
    cb = q.embedding.weight.detach()
    # every codebook row quantises to itself
    z = cb.t().reshape(1, 32, 4, 8, 8).contiguous()
    _, _, idx = q(z)
    assert torch.equal(idx.flatten().cpu(), torch.arange(256))
    # idempotence on a C4-sized latent (32 768 vectors)
    z = torch.randn(1, 32, 32, 32, 32, device="cuda") * 0.7
    zq, _, idx1 = q(z)
    _, _, idx2 = q(zq)
    assert torch.equal(idx1, idx2)
