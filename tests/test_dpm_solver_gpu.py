"""DPMSolverMultistepScheduler on the GPU: b200_dpm_solver_step against the float64 solver reading
(tests/dpm_solver_emulator.py), order 1 against DDIM, the Gaussian model's exact endpoint, the golden C1 / C2 networks
and the brain-LDM bundle config against the CPU oracle driving the emulator scheduler, CUDA-graph replay and repeat
runs.  Runs in whichever storage flavour the library was loaded in (B200_ACT_DTYPE)."""
import ctypes as C
import json
import math
from pathlib import Path

import pytest
import torch

from generativemodels_b200 import _lib
from generativemodels_b200.networks.schedulers.dpm_solver import dpm_solver_weights
from oracle import torch_oracle as O
from tests import dpm_solver_emulator as E
from tests import golden
from tests.golden import configs as G

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"
MU, STD = 0.3, 0.5
TRAJ_TOL, TRAJ_MAX = 5e-2, 1e-1      # multi-step network trajectories (relative L2, max-abs of the reference's peak)


def _sched(**kw):
    from generativemodels_b200.networks.schedulers import DPMSolverMultistepScheduler
    return DPMSolverMultistepScheduler(**kw)


def _check_traj(got, want, what):
    got, want = got.detach().float().cpu(), want.detach().float().cpu()
    r = ((got - want).norm() / want.norm()).item()
    m = ((got - want).abs().max() / want.abs().max()).item()
    assert r < TRAJ_TOL and m < TRAJ_MAX, f"{what}: relative L2 {r:.3e}, max-abs {m:.3e}"
    return r


# ------------------------------------------------------------------------------------------------ the kernel
def _plan(pred, clip, n_hist, sde):
    s = _sched()
    acp = s.alphas_cumprod.double()
    a, sg = acp.sqrt(), (1 - acp).sqrt()
    lam = (a.log() - sg.log()).tolist()
    t_s, t_t, hist_t = 400, 330, (470, 560)
    return E.Step(pred, float(a[t_s]), float(sg[t_s]), float(a[t_t]), float(sg[t_t]),
                  [lam[t_s]] + [lam[t] for t in hist_t][:n_hist], n_hist + 1, sde, clip, -1.0, 1.0)


def _coef(p):
    c_x, w, c_z = dpm_solver_weights(p.alpha_s, p.sigma_s, p.alpha_t, p.sigma_t, p.lambdas, p.order, p.sde)
    c = _lib.DpmCoef(alpha_s=p.alpha_s, sigma_s=p.sigma_s, c_x=c_x, c_z=c_z, clip_min=p.clip_min, clip_max=p.clip_max,
                     prediction_type=p.pred, clip=int(p.clip))
    for k in range(3):
        c.w[k] = w[k]
    return c


def _launch(c, m, s, hist, z, prev, x0):
    lib = _lib.require_device()
    ptrs = (C.c_void_p * 2)(*[h.data_ptr() for h in hist])
    _lib.check(lib.b200_dpm_solver_step(m.data_ptr(), s.data_ptr(), ptrs, len(hist), None if z is None else
                                        z.data_ptr(), C.byref(c), prev.data_ptr(), x0.data_ptr(), m.numel(),
                                        torch.cuda.current_stream().cuda_stream), "b200_dpm_solver_step")


def _run_kernel(p, n, offset, seed):
    """Inputs of n elements at element `offset` of their buffers (offset 1: no 16-byte alignment); outputs likewise,
    with a NaN sentinel around them."""
    g = torch.Generator().manual_seed(seed)
    host = [1.5 * torch.randn(n, generator=g) for _ in range(5)]
    dev = []
    for h in host:
        buf = torch.full((n + offset + 3,), float("nan"), device="cuda")
        buf[offset:offset + n] = h.cuda()
        dev.append(buf[offset:offset + n])
    m, s, h0, h1, z = dev
    hist = [h0, h1][:p.order - 1]
    outs = [torch.full((n + offset + 3,), float("nan"), device="cuda") for _ in range(2)]
    prev, x0 = (o[offset:offset + n] for o in outs)
    c = _coef(p)
    _launch(c, m, s, hist, z if p.sde else None, prev, x0)
    torch.cuda.synchronize()
    for o in outs:
        assert torch.isnan(o[:offset]).all() and torch.isnan(o[offset + n:]).all(), "write outside the outputs"
    return host, c, prev.cpu(), x0.cpu()


CASES = [(pred, clip, nh, sde) for pred in (E.PRED_EPSILON, E.PRED_SAMPLE, E.PRED_V) for clip in (False, True)
         for nh in (0, 1, 2) for sde in (False, True) if not (sde and nh == 2)]


@pytest.mark.parametrize("pred,clip,n_hist,sde", CASES)
def test_kernel_matches_the_solver(cuda_device, pred, clip, n_hist, sde):
    p = _plan(pred, clip, n_hist, sde)
    worst = 0.0
    for n in (1, 7, 8, 4099):
        for offset in (0, 1):
            (m, s, h0, h1, z), c, prev, x0 = _run_kernel(p, n, offset, seed=n + offset)
            hist = [h0, h1][:n_hist]
            want_p, want_x = E.solver_step(m, s, hist, z if sde else None, p)
            ex_p, ex_x = E.excess(want_p, prev).max().item(), E.excess(want_x, x0).max().item()
            assert ex_p <= 1.0 and ex_x <= 1.0, (n, offset, ex_p, ex_x)
            abi_p, abi_x = E.abi_step(m, s, hist, z if sde else None, c, n)
            assert E.excess(abi_p, prev).max() <= 1.0 and E.excess(abi_x, x0).max() <= 1.0, (n, offset)
            worst = max(worst, ex_p, ex_x)
    print(f"dpm_solver_step pred={pred} clip={clip} n_hist={n_hist} sde={sde}: largest err/bound {worst:.3f}")


@pytest.mark.parametrize("n_hist,sde", [(2, False), (1, True)])
def test_kernel_at_the_c3_volume(cuda_device, n_hist, sde):
    n = 160 * 224 * 160
    p = _plan(E.PRED_EPSILON, True, n_hist, sde)
    (m, s, h0, h1, z), _, prev, x0 = _run_kernel(p, n, 0, seed=3)
    want_p, want_x = E.solver_step(m, s, [h0, h1][:n_hist], z if sde else None, p)
    assert E.excess(want_p, prev).max() <= 1.0 and E.excess(want_x, x0).max() <= 1.0


def test_kernel_repeats_bit_identical(cuda_device):
    p = _plan(E.PRED_V, True, 2, False)
    _, _, a, ax = _run_kernel(p, 4099, 0, seed=9)
    _, _, b, bx = _run_kernel(p, 4099, 0, seed=9)
    assert torch.equal(a, b) and torch.equal(ax, bx)


# ------------------------------------------------------------------------------------------------ order 1 = DDIM
def test_order_one_on_the_leading_grid_is_ddim(cuda_device):
    from generativemodels_b200.networks.schedulers import DDIMScheduler
    d = DDIMScheduler(clip_sample=False)
    s = _sched(solver_order=1, timestep_spacing="leading", clip_sample=False)
    d.set_timesteps(50)
    s.set_timesteps(50)
    assert torch.equal(d.timesteps, s.timesteps)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 3, 16, 16, generator=g).cuda()
    acp = d.alphas_cumprod.double()
    for i, t in enumerate(d.timesteps):
        m = torch.randn(2, 3, 16, 16, generator=g).cuda()
        want, want_x0 = d.step(m, t, x)
        got, got_x0 = s.step(m, t, x)
        tp = int(t) - 1000 // 50
        a_t, s_t = (math.sqrt(float(acp[tp])), math.sqrt(1 - float(acp[tp]))) if tp >= 0 else (1.0, 0.0)
        a_s, s_s = math.sqrt(float(acp[int(t)])), math.sqrt(1 - float(acp[int(t)]))
        x0_terms = (x.abs() + s_s * m.abs()).double() / a_s          # the magnitudes x0 is formed from
        terms = a_t * x0_terms + s_t * m.abs().double() + (s_t / s_s) * x.abs().double()
        assert ((got.double() - want.double()).abs() <= 8 * 2.0 ** -24 * terms).all(), i
        assert ((got_x0.double() - want_x0.double()).abs() <= 4 * 2.0 ** -24 * x0_terms).all(), i
        x = want


# ------------------------------------------------------------------------------------------------ the Gaussian model
def _gaussian_model(sched, pred="epsilon"):
    acp = sched.alphas_cumprod.double()

    def model(x, timesteps, context=None):
        t = int(timesteps[0])
        a, s = math.sqrt(float(acp[t])), math.sqrt(1.0 - float(acp[t]))
        x0 = E.gaussian_x0(x.double(), a, s, MU, STD)
        eps = (x.double() - a * x0) / s
        return {"epsilon": eps, "sample": x0, "v_prediction": a * eps - s * x0}[pred].to(x.dtype)
    return model


def _emulator_trajectory(sched, x_T, pred="epsilon"):
    em = E.EmulatorScheduler(sched)
    model = _gaussian_model(sched, pred)
    x = x_T.double()
    for t in sched.timesteps:
        x, _ = em.step(model(x, torch.tensor([int(t)])).double(), x)
    return x


@pytest.mark.parametrize("n", [10, 20])
def test_gaussian_model_on_the_logsnr_grid(cuda_device, n):
    from generativemodels_b200.inferers import DiffusionInferer
    x_T = torch.randn(1, 4, 64, 64, generator=torch.Generator().manual_seed(0))
    err = {}
    for order in (1, 2, 3):
        s = _sched(solver_order=order, clip_sample=False)
        s.set_timesteps(n)
        got = DiffusionInferer(s).sample(x_T.cuda(), _gaussian_model(s), s, verbose=False).cpu().double()
        want = _emulator_trajectory(s, x_T)
        assert ((got - want).norm() / want.norm()).item() < 1e-5, order
        acp = s.alphas_cumprod.double()
        exact = E.pf_ode_endpoint(x_T.double(), math.sqrt(float(acp[999])), math.sqrt(1 - float(acp[999])), MU, STD)
        err[order] = ((got - exact).norm() / exact.norm()).item()
    print(f"Gaussian model, {n} steps on the log-SNR grid: endpoint error order 1 {err[1]:.3e}, 2M {err[2]:.3e}, "
          f"3M {err[3]:.3e} ({err[1] / err[2]:.1f}x)")
    if n == 10:
        assert err[1] / err[2] >= 5.0, err


# ------------------------------------------------------------------------------------------------ networks
class _EmulatorDriver:
    """The emulator scheduler with the oracle's step(model_output, t, x) interface (fp32 in, fp32 out)."""

    def __init__(self, sched):
        self.em = E.EmulatorScheduler(sched)
        self.timesteps = sched.timesteps.cpu()

    def step(self, out, t, x):
        prev, x0 = self.em.step(out.double(), x.double())
        return prev.float(), x0.float()


def _recipe(module, seed):
    sd = G.recipe_state_dict(module, seed)
    return {k: v.clone() for k, v in sd.items()}


def test_c1_unet_sampling_vs_oracle(cuda_device):
    from generativemodels_b200.inferers import DiffusionInferer
    from generativemodels_b200.networks.nets import DiffusionModelUNet
    m = DiffusionModelUNet(**G.C1_UNET).eval()
    sd = _recipe(m, 2024)
    # no clip: the random network's x0 saturates it, and a 16-bit rounding difference then sends an element to the
    # other bound
    s = _sched(clip_sample=False)
    s.set_timesteps(5)
    noise = torch.randn(*G.C1_SHAPE, generator=torch.Generator().manual_seed(1))
    cfg = G.unet_oracle_cfg(G.C1_UNET)
    with torch.no_grad():
        want = O.diffusion_sample(lambda x, t, c: O.unet_forward(sd, cfg, x, t, context=c), _EmulatorDriver(s), noise)
    got = DiffusionInferer(s).sample(noise.cuda(), m.cuda(), s, verbose=False)
    print(f"C1 DPM-Solver++ 5 steps vs oracle: rel L2 {_check_traj(got, want, 'C1 sample'):.3e}")


def test_c2_latent_sampling_vs_oracle(cuda_device):
    from generativemodels_b200.inferers import LatentDiffusionInferer
    from generativemodels_b200.networks.nets import AutoencoderKL, DiffusionModelUNet
    ae, un = AutoencoderKL(**G.C2_AEKL).eval(), DiffusionModelUNet(**G.C2_UNET).eval()
    asd, usd = _recipe(ae, 7), _recipe(un, 8)
    s = _sched(clip_sample=False, **G.C2_SCHEDULER)
    s.set_timesteps(5)
    noise = torch.randn(*G.C2_LATENT, generator=torch.Generator().manual_seed(2))
    ucfg, acfg = G.unet_oracle_cfg(G.C2_UNET), G.aekl_oracle_cfg(G.C2_AEKL)
    with torch.no_grad():
        lat = O.diffusion_sample(lambda x, t, c: O.unet_forward(usd, ucfg, x, t, context=c), _EmulatorDriver(s), noise)
        want = O.autoencoderkl_decode(asd, acfg, lat)
    got = LatentDiffusionInferer(s, scale_factor=1.0).sample(noise.cuda(), ae.cuda(), un.cuda(), s, verbose=False)
    print(f"C2 latent DPM-Solver++ 5 steps vs oracle: rel L2 {_check_traj(got, want, 'C2 sample'):.3e}")


def _small_unet():
    from generativemodels_b200.networks.nets import DiffusionModelUNet
    torch.manual_seed(0)
    return G.randomize_zero_params(DiffusionModelUNet(**G.UNET_CASES["unet2d_attn"])).cuda().eval()


@pytest.mark.parametrize("kw", [dict(), dict(solver_order=3), dict(algorithm_type="sde-dpmsolver++")])
def test_graph_replay_and_repeats_bit_identical(cuda_device, monkeypatch, kw):
    """The auto-graph path (>= 8 steps) reuses the network's output buffer; the history holds the kernel's own x0, so
    replayed and eager sampling agree bit for bit, and so do repeated runs of one scheduler object."""
    import generativemodels_b200.inferers.inferer as I
    from generativemodels_b200.inferers import DiffusionInferer
    m = _small_unet()
    x = torch.randn(2, 1, 16, 16, generator=torch.Generator().manual_seed(1)).cuda()
    s = _sched(**kw)
    s.set_timesteps(10)
    outs = {}
    for graph in (False, True, True):
        monkeypatch.setattr(I, "AUTO_CUDA_GRAPH", graph)
        torch.manual_seed(4)                      # the SDE form's noise
        outs.setdefault(graph, []).append(DiffusionInferer(s).sample(x, m, s, verbose=False))
    assert "_b200_auto_graph" in m.__dict__
    assert torch.equal(outs[False][0], outs[True][0]), "graph-replayed sampling differs from eager"
    assert torch.equal(outs[True][0], outs[True][1]), "repeated sampling differs"
    assert torch.isfinite(outs[True][0]).all()


def test_brain_ldm_bundle_config_with_the_scheduler_swapped(cuda_device):
    """The bundle's unmodified inference.json with the scheduler's _target_ swapped, resolved at the fixture's reduced
    widths, against the oracle networks driving the emulator scheduler."""
    from generativemodels_b200.bundle import BundleConfig
    from generativemodels_b200.networks.schedulers import DPMSolverMultistepScheduler
    fx = golden.load("g_bundle_brain_ldm")
    over = {"load_autoencoder": "$@autoencoder_def.load_state_dict(@states['aekl_state'])",
            "load_diffusion": "$@diffusion_def.load_state_dict(@states['unet_state'])",
            "noise": "$@states['noise'].to(@device)", "states": "$None",
            "scheduler#_target_": "generative.networks.schedulers.DPMSolverMultistepScheduler",
            "set_timesteps": "$@scheduler.set_timesteps(num_inference_steps=10)"}
    for item, kw in (("autoencoder_def", G.BUNDLE_AEKL), ("diffusion_def", G.BUNDLE_UNET)):
        for k, v in kw.items():
            over[f"{item}#{k}"] = list(v) if isinstance(v, tuple) else v
    cfg = BundleConfig(str(GOLD / "brain_ldm_inference.json"), json.loads(json.dumps(over)))
    cfg._resolved["states"] = fx
    got = cfg.get("sample")
    s = cfg.get("scheduler")
    assert isinstance(s, DPMSolverMultistepScheduler) and len(s.timesteps) == 10 and not s.clip_sample
    ucfg, acfg = G.unet_oracle_cfg(fx["unet_kwargs"]), G.aekl_oracle_cfg(fx["aekl_kwargs"])
    ref = _sched(**G.BUNDLE_SCHEDULER)
    ref.set_timesteps(10)
    with torch.no_grad():
        want = O.bundle_sampling_fn(lambda x, t, c: O.unet_forward(fx["unet_state"], ucfg, x, t, context=c),
                                    lambda z: O.autoencoderkl_decode(fx["aekl_state"], acfg, z), _EmulatorDriver(ref),
                                    fx["noise"], fx["conditioning"])
    print(f"brain-LDM config, DPM-Solver++ 10 steps vs oracle: rel L2 {_check_traj(got, want, 'bundle'):.3e}")
