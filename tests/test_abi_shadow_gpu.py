"""Every C-ABI call of real network forwards, checked against its float64 contract reading (tests/abi_shadow.py).

The contract tests hold each kernel to its emulator on argument sets their authors chose; the network tests compare
whole forwards at network tolerance (2e-2 relative L2).  Here each call a network makes runs on the GPU and on the
CPU stand-in with the call's own device inputs, under the per-element bound of its family, and every byte outside
its outputs must survive.  The sized cases use the models' real channel widths at batch sizes and volumes that cross
ops._TAP_MIN_ROWS / ops._GN_FUSE_MIN_ROWS (32768 rows), reach split-K on the latent UNets' deep levels, the two-CTA
256-column kernel, flash attention at head dims 256 and 512 and the GEGLU GEMM.  Most of the file's time is the float64
emulation on the host.  The last test asserts which kernel
paths the file reached, so that a threshold or planner change that routes the networks around one of them shows."""
import time

import pytest
import torch

from generativemodels_b200 import ops
from tests import abi_shadow
from tests.golden import configs as G

pytestmark = pytest.mark.gpu

REACHED = set()


def nets():
    from generativemodels_b200.networks import nets as N
    return N


def shadowed(monkeypatch, name, fn):
    """Run fn() with every C-ABI call shadowed; assert no violation; print the per-entry table."""
    torch.cuda.synchronize()
    t0 = time.time()
    with abi_shadow.shadow(monkeypatch) as sh, torch.no_grad():
        fn()
    REACHED.update(sh.paths())
    print(f"\n== {name}: {len(sh.calls)} calls, {time.time() - t0:.1f} s\n{sh.table()}")
    assert sh.calls, f"{name}: no C-ABI call was shadowed"
    assert not sh.violations, f"{name}: {len(sh.violations)} violations\n{sh.report()}"


def _unet(kw, cls=None):
    torch.manual_seed(0)
    return G.randomize_zero_params((cls or nets().DiffusionModelUNet)(**kw)).eval().cuda()


# ------------------------------------------------------------------------------------------------------------------
# the configurations of tests/golden/configs.py
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(G.UNET_CASES))
def test_unet_cases(cuda_device, monkeypatch, name):
    kw, inp = G.UNET_CASES[name], G.UNET_INPUTS[name]
    m = _unet(kw)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(inp["shape"], generator=g).cuda()
    t = torch.tensor([10, 500][:x.shape[0]] * (x.shape[0] // min(2, x.shape[0]))).cuda()
    ctx = torch.randn(inp["context"], generator=g).cuda() if "context" in inp else None
    cls = torch.arange(x.shape[0]).cuda() if inp.get("classes") else None
    shadowed(monkeypatch, name, lambda: m(x, t, context=ctx, class_labels=cls))


def test_controlnet_case(cuda_device, monkeypatch):
    kw = G.CONTROLNET_CASE
    torch.manual_seed(0)
    cn = G.randomize_zero_params(nets().ControlNet(**kw)).eval().cuda()
    ukw = {k: v for k, v in kw.items() if not k.startswith("conditioning_embedding")}
    un = _unet(dict(ukw, out_channels=kw["in_channels"]))
    g = torch.Generator().manual_seed(2)
    x, ctx = torch.randn(2, 3, 16, 16, generator=g).cuda(), torch.randn(2, 3, 8, generator=g).cuda()
    cond, t = torch.rand(2, 1, 16, 16, generator=g).cuda(), torch.tensor([3, 700]).cuda()

    def fwd():
        down, mid = cn(x, t, cond, conditioning_scale=1.0, context=ctx)
        un(x, t, context=ctx, down_block_additional_residuals=down, mid_block_additional_residual=mid)
    shadowed(monkeypatch, "controlnet", fwd)


@pytest.mark.parametrize("name", list(G.AEKL_CASES))
def test_autoencoderkl_cases(cuda_device, monkeypatch, name):
    torch.manual_seed(0)
    m = G.randomize_zero_params(nets().AutoencoderKL(**G.AEKL_CASES[name])).eval().cuda()
    x = torch.randn(G.AEKL_INPUTS[name], generator=torch.Generator().manual_seed(3)).cuda()
    shadowed(monkeypatch, name, lambda: m.decode(m.encode(x)[0]))


@pytest.mark.parametrize("name", list(G.VQVAE_CASES))
def test_vqvae_cases(cuda_device, monkeypatch, name):
    torch.manual_seed(0)
    m = G.randomize_zero_params(nets().VQVAE(**G.VQVAE_CASES[name])).eval().cuda()
    x = torch.randn(G.VQVAE_INPUTS[name], generator=torch.Generator().manual_seed(4)).cuda()
    shadowed(monkeypatch, name, lambda: m(x))


@pytest.mark.parametrize("name", list(G.SPADE_UNET_CASES))
def test_spade_unet_cases(cuda_device, monkeypatch, name):
    kw, inp = G.SPADE_UNET_CASES[name], G.SPADE_UNET_INPUTS[name]
    m = _unet(kw, nets().SPADEDiffusionModelUNet)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(inp["shape"], generator=g).cuda()
    seg = G.seg_onehot(inp["seg"]).cuda()
    ctx = torch.randn(inp["context"], generator=g).cuda() if "context" in inp else None
    t = torch.tensor([20] * x.shape[0]).cuda()
    shadowed(monkeypatch, name, lambda: m(x, t, seg, context=ctx))


@pytest.mark.parametrize("name", list(G.SPADE_AEKL_CASES))
def test_spade_autoencoderkl_cases(cuda_device, monkeypatch, name):
    torch.manual_seed(0)
    m = G.randomize_zero_params(nets().SPADEAutoencoderKL(**G.SPADE_AEKL_CASES[name])).eval().cuda()
    shape = G.SPADE_AEKL_INPUTS[name]
    x = torch.randn(shape, generator=torch.Generator().manual_seed(6)).cuda()
    seg = G.seg_onehot((shape[0], G.SPADE_AEKL_CASES[name]["label_nc"], *shape[2:])).cuda()
    shadowed(monkeypatch, name, lambda: m.decode(m.encode(x)[0], seg))


def test_transformer_and_vqvae_transformer_inferer(cuda_device, monkeypatch):
    """Teacher-forced forward and key/value-cache decoding: embed_tokens, the cache append, attention_decode,
    rows_linear.  Eager steps: the inferer's sampler replays them from a CUDA graph, which the shadow cannot see."""
    from generativemodels_b200.inferers import VQVAETransformerInferer
    from generativemodels_b200.utils.ordering import Ordering
    kw = G.VQVAE_CASES["vqvae2d"]
    K = kw["num_embeddings"]
    torch.manual_seed(0)
    vq = nets().VQVAE(**kw).eval().cuda()
    tr = nets().DecoderOnlyTransformer(num_tokens=K + 1, max_seq_len=10, attn_layers_dim=32, attn_layers_depth=2,
                                       attn_layers_heads=4).eval().cuda()
    ordering = Ordering("s_curve", 2, (1, 4, 4), reflected_spatial_dims=(True, False))
    inf = VQVAETransformerInferer()
    x = torch.randn(2, 1, 16, 16, generator=torch.Generator().manual_seed(7)).cuda()

    tok = torch.randint(0, K + 1, (2, 9), generator=torch.Generator().manual_seed(8)).cuda()

    def fwd():
        inf(x, vq, tr, ordering)
        cache = tr.new_cache(2, tok.device, None)                 # eager key/value-cache steps (no CUDA graph)
        tr.step(tok[:, :4], cache)
        for i in range(4, 9):
            tr.step(tok[:, i:i + 1], cache)
        dyn = tr.new_cache(2, tok.device, None)                   # the position-in-device-memory form
        for i in range(9):
            tr._step_dyn(tok[:, i:i + 1].contiguous(), dyn)
    shadowed(monkeypatch, "transformer + VQVAETransformerInferer", fwd)


# ------------------------------------------------------------------------------------------------------------------
# the other networks at their golden-fixture configurations
# ------------------------------------------------------------------------------------------------------------------
def test_patch_discriminators(cuda_device, monkeypatch):
    """Every PatchDiscriminator / MultiScalePatchDiscriminator fixture, on its input: folded BatchNorm, instance norm,
    strided pooling."""
    from tests import patchgan_oracle as PO
    from tests.test_patchgan_gpu import CLASSES, GOLD
    for name, g in GOLD.items():
        net = PO.seeded_weights(CLASSES[g["cls"]](**g["kwargs"])).eval().cuda()
        x = PO.input_of(g).cuda()
        shadowed(monkeypatch, f"{g['cls']} {name}", lambda: net(x))


def test_spadenet(cuda_device, monkeypatch):
    from tests.test_spadenet_gpu import GOLD, _net, _seg
    for name in ("tutorial", "ref3d"):
        g = GOLD[name]
        net = _net(g["kwargs"])
        shadowed(monkeypatch, f"spadenet {name}",
                 lambda: (net.encoder(g["x"].cuda()), net.decode(_seg(g), g["z"].cuda())))


def test_spatial_rescaler(cuda_device, monkeypatch):
    from tests import rescaler_oracle as RO
    from tests.test_spatial_rescaler_gpu import GOLD, _rescaler
    for name, g in GOLD.items():
        m = _rescaler(g["kwargs"])
        x = RO.input_of(g).cuda()
        shadowed(monkeypatch, f"rescaler {name}", lambda: m(x))


def test_diffusion_model_encoder(cuda_device, monkeypatch):
    from tests.test_diffusion_encoder_gpu import CASES, _inputs, _net
    for name in CASES:
        m = _net(name)
        x, t, ctx, labels = _inputs(name)
        shadowed(monkeypatch, f"encoder {name}", lambda: m(x, t, context=ctx, class_labels=labels))


# ------------------------------------------------------------------------------------------------------------------
# scheduler steps
# ------------------------------------------------------------------------------------------------------------------
def test_scheduler_steps(cuda_device, monkeypatch):
    from generativemodels_b200.networks.schedulers import DDIMScheduler, DDPMScheduler, PNDMScheduler
    from generativemodels_b200.networks.schedulers.dpm_solver import DPMSolverMultistepScheduler
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 3, 16, 16, generator=g).cuda()
    eps = [torch.randn(2, 3, 16, 16, generator=g).cuda() for _ in range(4)]
    for name, s in (("ddpm", DDPMScheduler(num_train_timesteps=1000)),
                    ("ddim", DDIMScheduler(num_train_timesteps=1000)),
                    ("pndm", PNDMScheduler(num_train_timesteps=1000, skip_prk_steps=True)),
                    ("dpm", DPMSolverMultistepScheduler(num_train_timesteps=1000))):
        s.set_timesteps(10)

        def steps():
            y = x
            for i, t in enumerate(s.timesteps[:4]):
                y = s.step(eps[i], t, y)[0]
        shadowed(monkeypatch, f"{name} steps", steps)


# ------------------------------------------------------------------------------------------------------------------
# sized cases: the models' real channel widths past the 32768-row thresholds, split-K, wide tiles, big heads
# ------------------------------------------------------------------------------------------------------------------
def test_c1_unet_past_the_row_thresholds(cuda_device, monkeypatch):
    m = _unet(G.C1_UNET)
    N_, H = 8, 64                                   # 8 x 64 x 64 = 32768 level-0 rows
    assert N_ * H * H >= ops._TAP_MIN_ROWS and N_ * H * H >= ops._GN_FUSE_MIN_ROWS
    x = torch.randn(N_, 1, H, H, generator=torch.Generator().manual_seed(9)).cuda()
    t = torch.arange(N_).cuda() * 100
    shadowed(monkeypatch, "C1 UNet 8x64x64", lambda: m(x, t))


def test_brain_ldm_latent_unet_split_k(cuda_device, monkeypatch):
    kw = dict(spatial_dims=3, in_channels=7, out_channels=3, num_channels=(256, 512, 768), num_res_blocks=1,
              attention_levels=(False, True, True), norm_num_groups=32, norm_eps=1e-6, resblock_updown=True,
              num_head_channels=(0, 512, 768), with_conditioning=True, transformer_num_layers=1,
              cross_attention_dim=4, upcast_attention=True)
    m = _unet(kw)
    g = torch.Generator().manual_seed(10)
    x = torch.randn(1, 7, 20, 28, 20, generator=g).cuda()
    ctx = torch.randn(1, 1, 4, generator=g).cuda()
    shadowed(monkeypatch, "brain-LDM latent UNet 20x28x20", lambda: m(x, torch.tensor([500]).cuda(), context=ctx))


def test_c3_unet_wide_tap_gn8_flash512(cuda_device, monkeypatch):
    """The C3 network (256, 256, 512, head 512, two res blocks) at 32 x 40 x 32: 40960 level-0 rows of 256 channels
    reach the 3-D tap gather / tap sum, GroupNorm from 8-channel partials and the wide kernel; flash at head dim 512
    on the deepest level."""
    m = _unet(G.C3_UNET)
    x = torch.randn(G.C3_SHAPE, generator=torch.Generator().manual_seed(11)).cuda()
    assert x[0, 0].numel() >= ops._TAP_MIN_ROWS
    shadowed(monkeypatch, "C3 UNet 32x40x32", lambda: m(x, torch.tensor([250]).cuda()))


def test_c2_autoencoderkl(cuda_device, monkeypatch):
    torch.manual_seed(0)
    m = G.randomize_zero_params(nets().AutoencoderKL(**G.C2_AEKL)).eval().cuda()
    x = torch.randn(1, 1, 64, 64, generator=torch.Generator().manual_seed(12)).cuda()
    shadowed(monkeypatch, "C2 AutoencoderKL encode + decode", lambda: m.decode(m.encode(x)[0]))


def test_controlnet_cross_attention_geglu_77_tokens(cuda_device, monkeypatch):
    common = dict(spatial_dims=2, in_channels=3, num_res_blocks=1, num_channels=(128, 256, 256),
                  attention_levels=(False, True, True), num_head_channels=256, with_conditioning=True,
                  cross_attention_dim=64)
    torch.manual_seed(0)
    cn = G.randomize_zero_params(nets().ControlNet(conditioning_embedding_in_channels=1,
                                                   conditioning_embedding_num_channels=(16,), **common)).eval().cuda()
    un = _unet(dict(out_channels=3, **common))
    g = torch.Generator().manual_seed(13)
    x, ctx = torch.randn(2, 3, 32, 32, generator=g).cuda(), torch.randn(2, 77, 64, generator=g).cuda()
    cond, t = torch.rand(2, 1, 32, 32, generator=g).cuda(), torch.tensor([480, 480]).cuda()

    def fwd():
        down, mid = cn(x, t, cond, conditioning_scale=1.0, context=ctx)
        un(x, t, context=ctx, down_block_additional_residuals=down, mid_block_additional_residual=mid)
    shadowed(monkeypatch, "ControlNet + cross-attention UNet, 77 tokens", fwd)


# ------------------------------------------------------------------------------------------------------------------
# coverage of the file
# ------------------------------------------------------------------------------------------------------------------
MUST_REACH = {
    # implicit GEMM: column tiles, split-K, store paths, GroupNorm partial producers (planner-derived, not hard-coded)
    "igemm bn64", "igemm bn128", "igemm bn256", "igemm wide", "igemm split", "igemm lean", "igemm fast",
    "igemm geglu", "igemm general vector", "igemm stat", "igemm gn4", "igemm gn8", "igemm sampled rows",
    # the large-shape reformulations and their consumers
    "b200_tap_gather", "b200_tap_sum", "gn_from_partials gw4", "gn_from_partials gw8",
    # attention: every head dim of ops._FLASH_HEAD_DIMS a case uses, the CUDA-core kernels, the decode path
    "flash dh64", "flash dh256", "flash dh512", "b200_attention_small", "b200_attention_small_ex",
    "b200_attention_decode", "b200_softmax_rows_partials",
    # everything else the networks call
    "b200_cache_append", "b200_embed_tokens", "b200_rows_linear", "b200_advance_i32", "b200_layernorm",
    "b200_groupnorm_fused", "b200_groupnorm_stats", "b200_groupnorm_apply", "b200_spade_apply",
    "b200_interpolate", "b200_pool_s2", "b200_batchnorm_fold", "b200_repack_weight", "b200_vq_argmin_gather",
    "b200_timestep_embedding", "b200_small_linear", "b200_pndm_step", "b200_dpm_solver_step", "b200_ddim_step",
    "b200_ddpm_step", "b200_axpy_h16", "b200_exp_half_clamped", "b200_nchw_to_nhwc", "b200_nhwc_to_nchw",
}
RAN = set()


@pytest.fixture(autouse=True)
def _ran(request):
    yield
    RAN.add(request.node.name)


def _cases_in_file():
    n = 0
    for name, fn in globals().items():
        if name.startswith("test_") and name != "test_zz_paths_reached":
            marks = [m for m in getattr(fn, "pytestmark", []) if m.name == "parametrize"]
            n += len(marks[0].args[1]) if marks else 1
    return n


def test_zz_paths_reached(cuda_device):
    """The paths the whole file reached (REACHED is filled by the cases above, in this process): skipped when only a
    selection of the cases ran."""
    RAN.discard("test_zz_paths_reached")
    if len(RAN) < _cases_in_file():
        pytest.skip(f"only {len(RAN)} of the file's {_cases_in_file()} cases ran")
    print("\npaths reached:", ", ".join(sorted(REACHED)))
    missing = MUST_REACH - REACHED
    assert not missing, f"the networks no longer reach {sorted(missing)}"
