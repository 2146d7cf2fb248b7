"""Every C-ABI call of the schedulers and inferers, checked against its float64 contract reading (tests/abi_shadow.py),
at the arguments real sampling produces.

The kernel tests of the step, noise and likelihood entry points use synthetic arguments, and the whole-trajectory
tests compare at a tolerance sized for a chain of network forwards, which cannot see a per-call error of a few
ulp-bounds.  Here the public inferer and scheduler API runs with every call shadowed: the history pointers are the x0
buffers earlier steps stored, in the order the host rotates them; `last` / `last_noise` come and go with the
corrector order and tau; `lower_order_final` and the last step of each trajectory are reached; the likelihood loop
reaches t = 0.  The networks are the reference-suite sizes of tests/golden/configs.py, and the scheduler variants
beyond one per family are driven by a pure-torch model, so that the file stays affordable.

Sampling replays the network from a CUDA graph by default (inferer.AUTO_CUDA_GRAPH), which the shadow cannot see:
the shadowed runs are eager, and test_eager_equals_graphed ties them to the default path bit for bit.  The last test
asserts which entry points and kernel paths the file reached (abi_shadow.step_paths labels)."""
import time

import pytest
import torch

from tests import abi_shadow
from tests.golden import configs as G

pytestmark = pytest.mark.gpu

REACHED = set()
STEPS = 10                    # below 15: lower_order_final shapes the last two steps
SHORT = 5                     # the latent, ControlNet and likelihood runs: each step is several network forwards


@pytest.fixture(autouse=True)
def _eager(monkeypatch):
    import generativemodels_b200.inferers.inferer as I
    monkeypatch.setattr(I, "AUTO_CUDA_GRAPH", False)


def nets():
    from generativemodels_b200.networks import nets as N
    return N


def sch():
    from generativemodels_b200.networks import schedulers as S
    return S


def inf():
    from generativemodels_b200 import inferers
    return inferers


def shadowed(monkeypatch, name, fn):
    """Run fn() with every C-ABI call shadowed; assert no violation; print the per-entry table."""
    torch.cuda.synchronize()
    t0 = time.time()
    with abi_shadow.shadow(monkeypatch) as sh, torch.no_grad():
        out = fn()
    REACHED.update(sh.paths())
    print(f"\n== {name}: {len(sh.calls)} calls, {time.time() - t0:.1f} s\n{sh.table()}")
    assert sh.calls, f"{name}: no C-ABI call was shadowed"
    assert not sh.violations, f"{name}: {len(sh.violations)} violations\n{sh.report()}"
    return out


def _seeded(module):
    torch.manual_seed(0)
    return G.randomize_zero_params(module).eval().cuda()


def unet(base="unet2d_small_heads", **kw):
    return _seeded(nets().DiffusionModelUNet(**dict(G.UNET_CASES[base], **kw)))


def aekl():
    return _seeded(nets().AutoencoderKL(**G.AEKL_CASES["aekl2d"]))        # 1 x 16 x 16 -> 3 x 8 x 8


def controlnet_pair():
    kw = G.CONTROLNET_CASE
    cn = _seeded(nets().ControlNet(**kw))
    ukw = {k: v for k, v in kw.items() if not k.startswith("conditioning_embedding")}
    return _seeded(nets().DiffusionModelUNet(**dict(ukw, out_channels=kw["in_channels"]))), cn


def randn(*shape, seed=0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).cuda()


def ready(s, steps=STEPS):
    s.set_timesteps(steps)
    return s


def const(tau):
    return lambda t: tau


# ------------------------------------------------------------------------------------------------------------------
# DiffusionInferer.sample, every scheduler
# ------------------------------------------------------------------------------------------------------------------
def _sample_cases():
    S = sch()
    return {
        "ddpm fixed, eps, clip, intermediates": lambda: S.DDPMScheduler(),
        "ddpm learned_range, v": lambda: S.DDPMScheduler(variance_type="learned_range", prediction_type="v_prediction",
                                                         clip_sample=False),
        "ddim sample-pred, concat": lambda: S.DDIMScheduler(prediction_type="sample"),
        "pndm plms, eps": lambda: S.PNDMScheduler(skip_prk_steps=True),
        "pndm prk, v": lambda: S.PNDMScheduler(prediction_type="v_prediction"),
        "dpm order 2, cross-attention": lambda: S.DPMSolverMultistepScheduler(),
        "dpm order 3, v": lambda: S.DPMSolverMultistepScheduler(solver_order=3, prediction_type="v_prediction",
                                                                clip_sample=False),
        "dpm sde order 2, sample-pred": lambda: S.DPMSolverMultistepScheduler(algorithm_type="sde-dpmsolver++",
                                                                              prediction_type="sample"),
        "unipc bh1": lambda: S.UniPCMultistepScheduler(solver_type="bh1", prediction_type="v_prediction"),
        "unipc bh2 order 3": lambda: S.UniPCMultistepScheduler(solver_order=3, clip_sample=False),
        "unipc corrector disabled": lambda: S.UniPCMultistepScheduler(disable_corrector=[1, 4, 5],
                                                                      prediction_type="sample"),
        "sa 1/1 tau 0": lambda: S.SASolverScheduler(predictor_order=1, corrector_order=1, tau_func=const(0.0)),
        "sa 2/2 tau 0.6, v": lambda: S.SASolverScheduler(tau_func=const(0.6), prediction_type="v_prediction",
                                                         clip_sample=False),
        "sa 3/3 tau 1, sample-pred": lambda: S.SASolverScheduler(predictor_order=3, corrector_order=3,
                                                                 tau_func=const(1.0), prediction_type="sample"),
        "sa 3/1 default tau": lambda: S.SASolverScheduler(predictor_order=3, corrector_order=1),
    }


SAMPLE_CASES = [
    "ddpm fixed, eps, clip, intermediates", "ddpm learned_range, v", "ddim sample-pred, concat", "pndm plms, eps",
    "pndm prk, v", "dpm order 2, cross-attention", "dpm order 3, v", "dpm sde order 2, sample-pred", "unipc bh1",
    "unipc bh2 order 3", "unipc corrector disabled", "sa 1/1 tau 0", "sa 2/2 tau 0.6, v", "sa 3/3 tau 1, sample-pred",
    "sa 3/1 default tau"]


# one case of each scheduler family samples with a network; the other variants drive the same loop with toy_model(),
# which makes no C-ABI call of its own, so that only their step calls are shadowed
NET_CASES = {"ddpm learned_range, v", "ddim sample-pred, concat", "pndm prk, v", "dpm order 2, cross-attention",
             "unipc bh2 order 3", "sa 3/1 default tau"}


@pytest.mark.parametrize("name", SAMPLE_CASES)
def test_diffusion_inferer_sample(cuda_device, monkeypatch, name):
    s = ready(_sample_cases()[name]())
    x = randn(2, 3, 8, 8, seed=1)
    kw = {}
    if name not in NET_CASES:
        m = toy_model()
    elif name.startswith("ddpm learned_range"):
        m = unet(out_channels=6)
    elif "concat" in name:
        m = unet(in_channels=4)
        kw = dict(mode="concat", conditioning=randn(2, 1, 8, 8, seed=2))
    elif "cross-attention" in name:
        m = unet("unet2d_cross")
        kw = dict(conditioning=randn(2, 3, 8, seed=2))
    else:
        m = unet()
    if "intermediates" in name:
        kw.update(save_intermediates=True, intermediate_steps=200)
    torch.manual_seed(3)
    out = shadowed(monkeypatch, f"DiffusionInferer.sample, {name}",
                   lambda: inf().DiffusionInferer(s).sample(x, m, s, verbose=False, **kw))
    img = out[0] if "intermediates" in name else out
    assert torch.isfinite(img).all()
    if "intermediates" in name:
        assert len(out[1]) == 5


# ------------------------------------------------------------------------------------------------------------------
# training forwards, distinct per-sample timesteps
# ------------------------------------------------------------------------------------------------------------------
T2 = (17, 640)


def test_training_forwards(cuda_device, monkeypatch):
    I = inf()
    t = torch.tensor(T2).cuda()
    ddpm = sch().DDPMScheduler()
    m, ae = unet(), aekl()
    un, cn = controlnet_pair()
    img = randn(2, 1, 16, 16, seed=4)
    shadowed(monkeypatch, "DiffusionInferer.__call__",
             lambda: I.DiffusionInferer(ddpm)(randn(2, 3, 8, 8, seed=5), m, randn(2, 3, 8, 8, seed=6), t))
    shadowed(monkeypatch, "LatentDiffusionInferer.__call__ (AutoencoderKL)",
             lambda: I.LatentDiffusionInferer(ddpm, scale_factor=0.7)(img, ae, m, randn(2, 3, 8, 8, seed=6), t))
    ctx, cond = randn(2, 3, 8, seed=7), torch.rand(2, 1, 16, 16, generator=torch.Generator().manual_seed(8)).cuda()
    shadowed(monkeypatch, "ControlNetDiffusionInferer.__call__",
             lambda: I.ControlNetDiffusionInferer(ddpm)(randn(2, 3, 16, 16, seed=5), un, cn,
                                                        randn(2, 3, 16, 16, seed=6), t, cond, condition=ctx))
    shadowed(monkeypatch, "ControlNetLatentDiffusionInferer.__call__ (AutoencoderKL)",
             lambda: I.ControlNetLatentDiffusionInferer(ddpm, scale_factor=0.7)(img, ae, un, cn,
                                                                                randn(2, 3, 8, 8, seed=6), t, cond,
                                                                                condition=ctx))


# ------------------------------------------------------------------------------------------------------------------
# LatentDiffusionInferer
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", ["unipc", "sa"])
def test_latent_sample(cuda_device, monkeypatch, solver):
    s = ready(sch().UniPCMultistepScheduler() if solver == "unipc" else sch().SASolverScheduler(tau_func=const(0.6)),
              SHORT)
    m, ae = unet(), aekl()
    x = randn(2, 3, 8, 8, seed=9)
    torch.manual_seed(3)
    out = shadowed(monkeypatch, f"LatentDiffusionInferer.sample, {solver}",
                   lambda: inf().LatentDiffusionInferer(s, scale_factor=0.7).sample(x, ae, m, s, verbose=False))
    assert out.shape == (2, 1, 16, 16) and torch.isfinite(out).all()


def test_latent_pad_and_crop(cuda_device, monkeypatch):
    """ldm_latent_shape 10 x 10 around the autoencoder's 8 x 8 latent: sampling crops, the training forward pads."""
    s = ready(sch().DPMSolverMultistepScheduler(), SHORT)
    m, ae = unet(), aekl()
    li = inf().LatentDiffusionInferer(s, scale_factor=0.7, ldm_latent_shape=[10, 10], autoencoder_latent_shape=[8, 8])
    out = shadowed(monkeypatch, "LatentDiffusionInferer.sample, pad / crop",
                   lambda: li.sample(randn(2, 3, 10, 10, seed=10), ae, m, s, verbose=False))
    assert out.shape == (2, 1, 16, 16)
    shadowed(monkeypatch, "LatentDiffusionInferer.__call__, pad",
             lambda: li(randn(2, 1, 16, 16, seed=11), ae, m, randn(2, 3, 10, 10, seed=12), torch.tensor(T2).cuda()))


def test_latent_vqvae_first_stage(cuda_device, monkeypatch):
    """A VQVAE first stage (16-channel 8 x 8 latent): training forwards with quantized True and False, and sampling,
    whose decode re-quantises."""
    vq = _seeded(nets().VQVAE(**G.VQVAE_CASES["vqvae2d"]))
    m = unet(in_channels=16, out_channels=16)
    s = ready(sch().DDIMScheduler(), SHORT)
    li = inf().LatentDiffusionInferer(s, scale_factor=0.5)
    img, t = randn(2, 1, 32, 32, seed=13), torch.tensor(T2).cuda()
    for q in (True, False):
        shadowed(monkeypatch, f"LatentDiffusionInferer.__call__ (VQVAE, quantized={q})",
                 lambda: li(img, vq, m, randn(2, 16, 8, 8, seed=14), t, quantized=q))
    out = shadowed(monkeypatch, "LatentDiffusionInferer.sample (VQVAE)",
                   lambda: li.sample(randn(2, 16, 8, 8, seed=15), vq, m, s, verbose=False))
    assert torch.isfinite(out).all()


def test_latent_spade_pair(cuda_device, monkeypatch):
    ae = _seeded(nets().SPADEAutoencoderKL(**G.SPADE_AEKL_CASES["spade_aekl2d"]))          # 1 x 16 x 16 -> 4 x 4 x 4
    m = _seeded(nets().SPADEDiffusionModelUNet(**dict(G.SPADE_UNET_CASES["spade_unet2d"], in_channels=4,
                                                       out_channels=4)))
    seg = G.seg_onehot((1, 3, 16, 16)).cuda()
    s = ready(sch().SASolverScheduler(), SHORT)
    torch.manual_seed(3)
    out = shadowed(monkeypatch, "LatentDiffusionInferer.sample, SPADE pair",
                   lambda: inf().LatentDiffusionInferer(s).sample(randn(1, 4, 4, 4, seed=16), ae, m, s, verbose=False,
                                                                  seg=seg))
    assert out.shape == (1, 1, 16, 16) and torch.isfinite(out).all()


# ------------------------------------------------------------------------------------------------------------------
# ControlNet inferers
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", ["dpm", "sa"])
def test_controlnet_sample(cuda_device, monkeypatch, solver):
    S, I = sch(), inf()
    s = ready(S.DPMSolverMultistepScheduler(solver_order=3) if solver == "dpm" else S.SASolverScheduler(), SHORT)
    un, cn = controlnet_pair()
    ctx = randn(2, 3, 8, seed=17)
    cond = torch.rand(2, 1, 16, 16, generator=torch.Generator().manual_seed(18)).cuda()
    torch.manual_seed(3)
    shadowed(monkeypatch, f"ControlNetDiffusionInferer.sample, {solver}",
             lambda: I.ControlNetDiffusionInferer(s).sample(randn(2, 3, 16, 16, seed=19), un, cn, cond, s,
                                                            conditioning=ctx, verbose=False))
    torch.manual_seed(3)
    out = shadowed(monkeypatch, f"ControlNetLatentDiffusionInferer.sample, {solver}",
                   lambda: I.ControlNetLatentDiffusionInferer(s, scale_factor=0.7).sample(
                       randn(2, 3, 8, 8, seed=20), aekl(), un, cn, cond, s, conditioning=ctx, verbose=False))
    assert out.shape == (2, 1, 16, 16) and torch.isfinite(out).all()


# ------------------------------------------------------------------------------------------------------------------
# get_likelihood: the DDPM grid of 5 steps ends at t = 0, so both b200_ddpm_kl branches run
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pred,clip", [("epsilon", True), ("v_prediction", False), ("sample", True)])
def test_likelihood(cuda_device, monkeypatch, pred, clip):
    s = ready(sch().DDPMScheduler(prediction_type=pred, clip_sample=clip), SHORT)
    assert int(s.timesteps[-1]) == 0
    x = torch.rand(2, 3, 8, 8, generator=torch.Generator().manual_seed(21)).cuda() * 2 - 1
    x[0, 0, 0] = torch.tensor([-1.0, 1.0, 0.9995, -0.9995, 0.0, 0.5, -0.5, 0.25])      # the edge bins of t = 0
    inter = pred == "epsilon"
    torch.manual_seed(3)
    out = shadowed(monkeypatch, f"DiffusionInferer.get_likelihood, {pred}, clip {clip}",
                   lambda: inf().DiffusionInferer(s).get_likelihood(x, unet(), s, save_intermediates=inter,
                                                                    verbose=False))
    kl = out[0] if inter else out
    assert kl.shape == (2,) and torch.isfinite(kl).all()


def test_latent_likelihood_resampled(cuda_device, monkeypatch):
    s = ready(sch().DDPMScheduler(), SHORT)
    img = randn(2, 1, 16, 16, seed=22)
    torch.manual_seed(3)
    kl, maps = shadowed(monkeypatch, "LatentDiffusionInferer.get_likelihood, resampled",
                        lambda: inf().LatentDiffusionInferer(s, scale_factor=0.7).get_likelihood(
                            img, aekl(), unet(), s, save_intermediates=True, resample_latent_likelihoods=True,
                            resample_interpolation_mode="bilinear", verbose=False))
    assert len(maps) == SHORT and maps[0].shape[-2:] == (16, 16)


# ------------------------------------------------------------------------------------------------------------------
# VQVAETransformerInferer
# ------------------------------------------------------------------------------------------------------------------
def _vq_transformer():
    from generativemodels_b200.utils.ordering import Ordering
    kw = G.VQVAE_CASES["vqvae2d"]
    vq = _seeded(nets().VQVAE(**kw))
    torch.manual_seed(0)
    tr = nets().DecoderOnlyTransformer(num_tokens=kw["num_embeddings"] + 1, max_seq_len=10, attn_layers_dim=32,
                                       attn_layers_depth=2, attn_layers_heads=4).eval().cuda()
    return vq, tr, Ordering("s_curve", 2, (1, 4, 4), reflected_spatial_dims=(True, False))


def test_vqvae_transformer_inferer(cuda_device, monkeypatch):
    """sample on a key/value cache forced eager (new_cache always with graph=False), which reaches b200_vq_gather in
    VQVAE.decode_samples; get_likelihood of a 16-token sequence through a 10-token window, which slides."""
    vq, tr, ordering = _vq_transformer()
    new_cache = tr.new_cache
    monkeypatch.setattr(tr, "new_cache", lambda *a, graph=False, **k: new_cache(*a, graph=False, **k))
    K = G.VQVAE_CASES["vqvae2d"]["num_embeddings"]
    start = torch.full((2, 1), K, dtype=torch.long).cuda()
    torch.manual_seed(3)
    out = shadowed(monkeypatch, "VQVAETransformerInferer.sample, eager cache",
                   lambda: inf().VQVAETransformerInferer().sample((4, 4), start, vq, tr, ordering, verbose=False))
    assert out.shape == (2, 1, 16, 16)
    lp = shadowed(monkeypatch, "VQVAETransformerInferer.get_likelihood, sliding window",
                  lambda: inf().VQVAETransformerInferer().get_likelihood(randn(2, 1, 16, 16, seed=23), vq, tr,
                                                                         ordering))
    assert lp.shape == (2, 4, 4) and torch.isfinite(lp).all()


def test_spadenet_vae_forward(cuda_device, monkeypatch):
    """SPADENet's VAE forward: the reparameterisation and its KL term (b200_vae_reparam_kld)."""
    from tests.test_spadenet_gpu import GOLD, _net, _seg
    g = GOLD["tutorial"]
    net = _net(g["kwargs"])
    torch.manual_seed(3)
    shadowed(monkeypatch, "SPADENet forward", lambda: net(_seg(g), g["x"].cuda()))


# ------------------------------------------------------------------------------------------------------------------
# steps only: a pure-torch model makes no C-ABI call, so the step kernels are shadowed cheaply at edge sizes
# ------------------------------------------------------------------------------------------------------------------
def toy_model(unaligned=False):
    """A smooth, timestep-dependent model output.  unaligned: a channel slice of a wider batch-1 output with odd H W,
    a contiguous view whose pointer is 4 (mod 16) bytes into its allocation, as a user model may return it."""
    def f(x, timesteps=None, context=None):
        y = 0.5 * torch.tanh(x) + 0.1 * torch.cos(3 * x + float(timesteps.flatten()[0]) / 100)
        if not unaligned:
            return y
        wide = torch.empty(y.shape[0], y.shape[1] + 1, *y.shape[2:], device=y.device)
        wide[:, 1:] = y
        v = wide[:, 1:]
        assert v.is_contiguous() and v.data_ptr() % 16 != 0
        return v
    return f


def _step_schedulers():
    S = sch()
    return {"ddim": lambda: S.DDIMScheduler(), "dpm": lambda: S.DPMSolverMultistepScheduler(
        algorithm_type="sde-dpmsolver++"), "unipc": lambda: S.UniPCMultistepScheduler(solver_order=3),
            "sa": lambda: S.SASolverScheduler(tau_func=const(0.6))}


EDGES = {"tail": ((1, 3, 5, 5), False), "scalar": ((1, 3, 5, 5), True), "vec": (G.C3_SHAPE, False)}


@pytest.mark.parametrize("edge", list(EDGES))
def test_steps_at_edge_sizes(cuda_device, monkeypatch, edge):
    shape, unaligned = EDGES[edge]
    for fam, make in _step_schedulers().items():
        s = ready(make())
        torch.manual_seed(3)
        out = shadowed(monkeypatch, f"{fam} steps, {edge} {shape}",
                       lambda: inf().DiffusionInferer(s).sample(randn(*shape, seed=24), toy_model(unaligned), s,
                                                                verbose=False))
        assert out.shape == shape and torch.isfinite(out).all()
    s = ready(sch().DDIMScheduler())
    x, g = randn(*shape, seed=25), torch.Generator().manual_seed(4)

    def others():
        y = x
        for t in s.timesteps[:3]:                  # DDIM with eta > 0 draws noise
            y = s.step(toy_model(unaligned)(y, torch.tensor([t])), t, y, eta=0.5, generator=g)[0]
        return s.get_velocity(y, x, torch.tensor([300]).cuda())
    shadowed(monkeypatch, f"DDIM eta 0.5 and get_velocity, {edge}", others)


def teacher_forced_error(s, emulator, x):
    """The largest relative distance, over the steps of one trajectory of `s` driven by toy_model(), between the
    scheduler's next sample and the float64 solver of `emulator` (tests/*_emulator.EmulatorScheduler, the formulas
    unfolded, no code shared with the host's folding) stepped from the same sample with the same model output.  The
    shadow holds each kernel to the coefficients the host hands it; this holds the host's coefficients to the solver."""
    E, f, worst = emulator(s), toy_model(), 0.0
    for t in s.timesteps:
        m = f(x, torch.tensor([int(t)]))
        want, _ = E.step(m.double().cpu(), x.double().cpu())
        x = s.step(m, t, x)[0]
        worst = max(worst, float((x.double().cpu() - want).abs().max() / want.abs().max()))
    return worst


def likelihood_f64(s, x, seed):
    """DiffusionInferer.get_likelihood of toy_model() restated in float64 from the scheduler's plain-tensor posterior
    (_get_mean, _get_variance) and the inferer's plain-tensor decoder log-likelihood, with the same noise draw."""
    torch.manual_seed(seed)
    noise = torch.randn_like(x).double()
    f, x64, total = toy_model(), x.double(), torch.zeros(x.shape[0], dtype=torch.float64, device=x.device)
    for t in (int(v) for v in s.timesteps):
        a = s.alphas_cumprod[t].double()
        xt = a.sqrt() * x64 + (1 - a).sqrt() * noise
        mo = f(xt.float(), torch.tensor([t])).double()
        p0 = {"epsilon": (xt - (1 - a).sqrt() * mo) / a.sqrt(), "sample": mo,
              "v_prediction": a.sqrt() * xt - (1 - a).sqrt() * mo}[str(s.prediction_type)]
        p0 = p0.clamp(-1, 1) if s.clip_sample else p0
        pred, post = s._get_mean(t, p0, xt), s._get_mean(t, x64, xt)
        lv = torch.log(s._get_variance(t)).double()
        if t == 0:
            kl = -inf().DiffusionInferer(s)._get_decoder_log_likelihood(x64, pred, 0.5 * lv)
        else:
            kl = 0.5 * (pred - post) ** 2 * torch.exp(-lv)
        total += kl.flatten(1).mean(1)
    return total


def test_scheduler_coefficients_against_the_solvers(cuda_device, monkeypatch):
    """Teacher-forced trajectories of the deterministic multistep solvers (every coefficient the host folds, the last
    step and lower_order_final included) and the likelihood of every prediction type, shadowed, against float64
    restatements."""
    from tests import dpm_solver_emulator as DE, sa_solver_emulator as SE, unipc_emulator as UE
    S = sch()
    cases = [("dpm order 3", S.DPMSolverMultistepScheduler(solver_order=3), DE.EmulatorScheduler),
             ("unipc bh2 order 3", S.UniPCMultistepScheduler(solver_order=3, prediction_type="v_prediction"),
              UE.EmulatorScheduler),
             ("unipc bh1, corrector disabled", S.UniPCMultistepScheduler(solver_type="bh1", disable_corrector=[3]),
              UE.EmulatorScheduler),
             ("sa 3/3 tau 0", S.SASolverScheduler(predictor_order=3, corrector_order=3, tau_func=const(0.0),
                                                  prediction_type="sample"), SE.EmulatorScheduler)]
    x = randn(1, 3, 5, 5, seed=27)
    for name, s, emulator in cases:
        err = shadowed(monkeypatch, f"{name} teacher-forced", lambda: teacher_forced_error(ready(s), emulator, x))
        print(f"{name}: largest relative distance to the float64 solver {err:.3g}")
        assert err < 1e-4, (name, err)
    img = torch.rand(2, 3, 5, 5, generator=torch.Generator().manual_seed(28)).cuda() * 2 - 1
    for pred, clip in (("epsilon", True), ("v_prediction", False), ("sample", True)):
        s = ready(S.DDPMScheduler(prediction_type=pred, clip_sample=clip))
        torch.manual_seed(29)
        got = shadowed(monkeypatch, f"get_likelihood {pred}, toy model",
                       lambda: inf().DiffusionInferer(s).get_likelihood(img, toy_model(), s, verbose=False))
        want = likelihood_f64(s, img, 29)
        rel = float(((got.double() - want).abs() / want.abs()).max())
        print(f"get_likelihood {pred}: relative distance to float64 {rel:.3g}")
        assert rel < 1e-3, (pred, got, want)


# ------------------------------------------------------------------------------------------------------------------
# eager equals graphed: the shadowed runs above are eager, the default replays the network from a CUDA graph
# ------------------------------------------------------------------------------------------------------------------
def _graph_cases():
    S = sch()
    return {  # the DiffusionInferer defaults of test_{unipc,sa_solver}_gpu.py's graph tests are not repeated
        "diffusion, unipc bh1 v": ("diffusion", lambda: S.UniPCMultistepScheduler(solver_type="bh1",
                                                                                   prediction_type="v_prediction")),
        "diffusion, sa 1/1 tau 1": ("diffusion", lambda: S.SASolverScheduler(predictor_order=1, corrector_order=1,
                                                                             tau_func=const(1.0))),
        "latent, unipc": ("latent", lambda: S.UniPCMultistepScheduler()),
        "latent, sa": ("latent", lambda: S.SASolverScheduler()),
    }


@pytest.mark.parametrize("name", ["diffusion, unipc bh1 v", "diffusion, sa 1/1 tau 1", "latent, unipc", "latent, sa"])
def test_eager_equals_graphed(cuda_device, monkeypatch, name):
    import generativemodels_b200.inferers.inferer as I
    kind, make = _graph_cases()[name]
    s = ready(make())
    m, ae = unet(), aekl()
    x = randn(2, 3, 8, 8, seed=26)
    outs = {}
    for graph in (False, True):
        monkeypatch.setattr(I, "AUTO_CUDA_GRAPH", graph)
        torch.manual_seed(3)
        with torch.no_grad():
            if kind == "diffusion":
                outs[graph] = I.DiffusionInferer(s).sample(x, m, s, verbose=False)
            else:
                outs[graph] = I.LatentDiffusionInferer(s, scale_factor=0.7).sample(x, ae, m, s, verbose=False)
        assert ("_b200_auto_graph" in m.__dict__) == graph
    assert torch.isfinite(outs[True]).all()
    assert torch.equal(outs[False], outs[True]), "eager sampling differs from graph-replayed sampling"


# ------------------------------------------------------------------------------------------------------------------
# coverage of the file
# ------------------------------------------------------------------------------------------------------------------
MUST_REACH = {
    # the scheduler and inferer entry points (the three sampler steps, include/b200gen_samplers.h, among them)
    "b200_ddim_step", "b200_ddpm_step", "b200_pndm_step", "b200_dpm_solver_step", "b200_unipc_step",
    "b200_sa_solver_step", "b200_add_noise", "b200_ddpm_kl", "b200_scale_f32", "b200_fma_f32",
    "b200_exp_half_clamped", "b200_vq_gather", "b200_vae_reparam_kld",
    # history depths and optional streams, as the host code rotates and drops them
    "dpm nh0", "dpm nh1", "dpm nh2", "dpm nh0 noise", "dpm nh1 noise",
    "unipc nh0", "unipc nh1", "unipc nh1 last", "unipc nh2 last", "unipc nh3 last",
    "sa nh0", "sa nh0 z", "sa nh0 last", "sa nh1 last", "sa nh1 last zl z", "sa nh2 last zl z", "sa nh2 last zl",
    "ddim", "ddim noise", "ddpm var0", "ddpm var2", "ddpm no noise",
    "pndm nh1", "pndm nh2", "pndm nh3", "pndm nh4",
    "ddpm_kl t0", "ddpm_kl t", "add_noise +", "add_noise -", "scale div", "scale mul",
    # the access paths of the four vectorised step kernels
    *(f"{fam} step {kind}" for fam in ("ddim", "dpm", "unipc", "sa") for kind in ("vec", "tail", "scalar")),
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
    assert not missing, f"the inferers no longer reach {sorted(missing)}"
