"""Dev probe for ncu: one launch each of the HBM-bound kernels at the sizes the BASELINE configs give them —
GroupNorm statistics + apply(+SiLU) on a 1x160x224x160x256 tensor (C3 level 0), the DDIM step on 1x1x160x224x160 fp32,
the VQ nearest-code search at M = 32 768 x 32 with 256 codes (C4 at 128^3); and, launch-bound, the fused GroupNorm at
the C2 UNet's deep levels and rows_linear's LayerNorm-prologue GEMV at M = 8, K = 512 (--norm-only: just those).
CUDA-event timings are printed for the roofline table; under `ncu --set full -k regex:...` the same launches give dram__bytes_{read,write}."""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch
from generativemodels_b200 import ops
from generativemodels_b200.networks.layers import EMAQuantizer
from generativemodels_b200.networks.schedulers import DDIMScheduler

torch.manual_seed(0)
dev = "cuda"
HBM = 6582.5
NORM_ONLY = "--norm-only" in sys.argv      # only the launch-bound normalisation timings below (for A/B runs)


def timed(fn, n=5):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return min(ts)


def many(fn, n):
    def run():
        for _ in range(n):
            fn()
    return run


# launch-bound normalisation: the fused GroupNorm at the C2 UNet's deep levels (N = 1, latent 64 x 64 -> 32^2 x 256
# and 16^2 x 512, 32 groups) and the LayerNorm-prologue GEMV of decoding (rows_linear, M = 8, K = O = 512)
from generativemodels_b200 import _lib
import ctypes as Cc
props = torch.cuda.get_device_properties(0)
print(f"device: {props.name}")
for hw, ch in ((32, 256), (16, 512)):
    xs = ops.CL(torch.randn(1, 1, hw, hw, ch, device=dev).to(ops.H16), ch, 2)
    g1, b1 = torch.ones(ch, device=dev), torch.zeros(ch, device=dev)
    fn = lambda: ops.groupnorm(xs, 32, 1e-6, g1, b1, act=ops.ACT_SILU)
    ms = timed(many(fn, 200), n=7) / 200
    print(f"fused GroupNorm(32)+SiLU 1x{hw}x{hw}x{ch}: {ms*1e3:.2f} us per call (200 back-to-back calls, best of 7)")
lib = _lib.require_device()
M, K = 8, 512
xr = torch.randn(M, K, device=dev).to(ops.H16)
W = (torch.randn(K, K, device=dev) * 0.05).to(ops.H16)
lg, lb = torch.ones(K, device=dev), torch.zeros(K, device=dev)
yr = torch.empty(M, K, device=dev, dtype=ops.H16)
def rows_linear():
    _lib.check(lib.b200_rows_linear(xr.data_ptr(), K, M, K, lg.data_ptr(), lb.data_ptr(), 1e-5, W.data_ptr(), K, K,
                                    None, 0, None, 0, yr.data_ptr(), K, 0, ops._stream()), "rows_linear")
ms = timed(many(rows_linear, 500), n=7) / 500
print(f"rows_linear + LayerNorm prologue M={M} K=O={K}: {ms*1e3:.2f} us per call (500 back-to-back calls, best of 7)")
if NORM_ONLY:
    sys.exit(0)

C = 256
x = ops.CL((torch.randn(1, 160, 224, 160, C, device=dev) * 0.7 + 0.1).to(ops.H16), C, 3)
gamma, beta = torch.ones(C, device=dev), torch.zeros(C, device=dev)
nbytes = x.t.numel() * 2
ms = timed(lambda: ops.groupnorm(x, 32, 1e-6, gamma, beta, act=ops.ACT_SILU))
print(f"GroupNorm(32)+SiLU stats+apply on {tuple(x.t.shape)} ({nbytes/1e9:.2f} GB): {ms:.3f} ms  -> "
      f"{3*nbytes/ms/1e6:.0f} GB/s algorithmic (2 reads + 1 write), {3*nbytes/ms/1e6/HBM:.3f} of measured copy bandwidth")
aff = ops.groupnorm_affine(x, 32, 1e-6, gamma, beta)
out = x.like()
def apply_only():
    _, ap = ops._gn_params([x])
    ap.affine, ap.act = aff.data_ptr(), ops.ACT_SILU
    ap.y_ptr, ap.y_pitch = out.t.data_ptr(), out.pitch
    _lib.check(_lib.require_device().b200_groupnorm_apply(Cc.byref(ap), ops._stream()), "apply")
ms = timed(apply_only)
print(f"gn_apply_kernel alone: {ms:.3f} ms -> {2*nbytes/ms/1e6:.0f} GB/s (1 read + 1 write), {2*nbytes/ms/1e6/HBM:.3f} of measured")
ms = timed(lambda: ops.groupnorm_affine(x, 32, 1e-6, gamma, beta))
print(f"gn statistics alone (partial + finalize): {ms:.3f} ms -> {nbytes/ms/1e6:.0f} GB/s (1 read), {nbytes/ms/1e6/HBM:.3f} of measured")
del x, out

s = DDIMScheduler(num_train_timesteps=1000, schedule="scaled_linear_beta", beta_start=0.0005, beta_end=0.0195, clip_sample=False)
s.set_timesteps(50)
eps = torch.randn(1, 1, 160, 224, 160, device=dev)
xt = torch.randn_like(eps)
n = eps.numel()
for rep in (1, 8):
    e, xx = eps.repeat(rep, 1, 1, 1, 1), xt.repeat(rep, 1, 1, 1, 1)
    ms = timed(lambda: s.step(e, 500, xx))
    print(f"ddim_step_kernel on {rep} x 1x160x224x160 fp32: {ms*1e3:.1f} us -> {16*n*rep/ms/1e6:.0f} GB/s (2 reads + 2 writes), "
          f"{16*n*rep/ms/1e6/HBM:.3f} of measured")

q = EMAQuantizer(spatial_dims=3, num_embeddings=256, embedding_dim=32).to(dev).eval()
z = torch.randn(1, 32, 32, 32, 32, device=dev)
for rep in (1, 16):
    zz = z.repeat(rep, 1, 1, 1, 1)
    zc = q._z_channels_last(zz)
    M = zc.numel() // 32
    ms = timed(lambda: q.quantize_cl(zc, want_f32=False))
    byts = M * 32 * 4 + 256 * 32 * 4 + M * 8 + M * 32 * 2
    print(f"vq_argmin_kernel M = {M} x 32, 256 codes: {ms*1e3:.1f} us -> {byts/ms/1e6:.0f} GB/s algorithmic, "
          f"{byts/ms/1e6/HBM:.3f} of measured; {2*M*256*32/ms/1e9:.2f} TFLOP/s fp32 distance math")
