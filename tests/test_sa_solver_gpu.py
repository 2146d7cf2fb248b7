"""SASolverScheduler on the GPU: b200_sa_solver_step against the float64 readings (tests/sa_solver_emulator.py), the
tau = 1 order-1 step against DPMSolverMultistepScheduler's SDE order 1, the Gaussian model's weak and strong
convergence, the golden C1 / C2 networks and the brain-LDM bundle config against the CPU oracle driving the emulator
scheduler with the same noise, CUDA-graph replay and repeat runs.  Runs in whichever storage flavour the library was
loaded in (B200_ACT_DTYPE)."""
import ctypes as C
import json
import math
from pathlib import Path

import pytest
import torch

from generativemodels_b200 import _lib
from generativemodels_b200.networks.schedulers.sa_solver import sa_solver_weights
from oracle import torch_oracle as O
from tests import golden
from tests import sa_solver_emulator as E
from tests.golden import configs as G

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"
MU, STD = 0.3, 0.5
TRAJ_TOL, TRAJ_MAX = 5e-2, 1e-1      # multi-step network trajectories, as tests/test_dpm_solver_gpu.py


def _sched(**kw):
    from generativemodels_b200.networks.schedulers import SASolverScheduler
    return SASolverScheduler(**kw)


def _const(tau):
    return lambda t: tau


def _check_traj(got, want, what):
    got, want = got.detach().float().cpu(), want.detach().float().cpu()
    r = ((got - want).norm() / want.norm()).item()
    m = ((got - want).abs().max() / want.abs().max()).item()
    assert r < TRAJ_TOL and m < TRAJ_MAX, f"{what}: relative L2 {r:.3e}, max-abs {m:.3e}"
    return r


# ------------------------------------------------------------------------------------------------ the kernel
def _plan(pred, clip, n_hist, last, noise, last_noise):
    """A step at t = 400 predicting to 330, earlier estimates at 470 and 560: predictor order n_hist + 1 and, with
    `last`, a corrector of the same order from 470; tau 1 (0 without `noise`), the previous step's 0.7 (0 without
    `last_noise`).  -> (emulator Step, folded weights)."""
    s = _sched()
    acp = s.alphas_cumprod.double()
    a, sg = acp.sqrt(), (1 - acp).sqrt()
    lam = (a.log() - sg.log())
    ts, tgt = [400, 470, 560], 330
    p, q = n_hist + 1, (n_hist + 1 if last else 0)
    tau, tau_last = (1.0 if noise else 0.0), (0.7 if last_noise else 0.0)
    f = lambda v: [float(v[t]) for t in ts]         # noqa: E731
    folded = sa_solver_weights(f(a), f(sg), f(lam), float(a[tgt]), float(sg[tgt]), p, q, tau, tau_last)
    pr = E.Interval(f(a)[0], f(sg)[0], float(a[tgt]), float(sg[tgt]), f(lam)[:p], tau)
    cor = E.Interval(f(a)[1], f(sg)[1], f(a)[0], f(sg)[0], f(lam)[:q], tau_last) if q else None
    return E.Step(pred, f(a)[0], f(sg)[0], pr, cor, clip, -1.0, 1.0), folded


def _coef(p, folded):
    c_last, v, c_zl, c_xc, u, c_z = folded
    c = _lib.SASolverCoef(alpha_s=p.alpha_s, sigma_s=p.sigma_s, c_last=c_last, c_zlast=c_zl, c_xc=c_xc, c_z=c_z,
                          clip_min=p.clip_min, clip_max=p.clip_max, prediction_type=p.pred, clip=int(p.clip))
    for k in range(3):
        c.v[k], c.u[k] = v[k], u[k]
    return c


def _launch(c, m, s, last, zl, hist, z, prev, x0, xc):
    lib = _lib.require_device()
    ptrs = (C.c_void_p * 2)(*[h.data_ptr() for h in hist])
    ptr = (lambda t: None if t is None else t.data_ptr())                # noqa: E731
    _lib.check(lib.b200_sa_solver_step(m.data_ptr(), s.data_ptr(), ptr(last), ptr(zl), ptrs, len(hist), ptr(z),
                                       C.byref(c), prev.data_ptr(), x0.data_ptr(), xc.data_ptr(), m.numel(),
                                       torch.cuda.current_stream().cuda_stream), "b200_sa_solver_step")


def _run_kernel(p, folded, n_hist, last, noise, last_noise, n, offset, seed):
    """Inputs of n elements at element `offset` of their buffers (offset 1: no 16-byte alignment); outputs likewise,
    with a NaN sentinel around them."""
    g = torch.Generator().manual_seed(seed)
    host = [1.5 * torch.randn(n, generator=g) for _ in range(7)]
    dev = []
    for h in host:
        buf = torch.full((n + offset + 3,), float("nan"), device="cuda")
        buf[offset:offset + n] = h.cuda()
        dev.append(buf[offset:offset + n])
    m, s, l_, zl, h0, h1, z = dev
    outs = [torch.full((n + offset + 3,), float("nan"), device="cuda") for _ in range(3)]
    prev, x0, xc = (o[offset:offset + n] for o in outs)
    c = _coef(p, folded)
    _launch(c, m, s, l_ if last else None, zl if last_noise else None, [h0, h1][:n_hist], z if noise else None,
            prev, x0, xc)
    torch.cuda.synchronize()
    for o in outs:
        assert torch.isnan(o[:offset]).all() and torch.isnan(o[offset + n:]).all(), "write outside the outputs"
    return host, c, prev.cpu(), x0.cpu(), xc.cpu()


CASES = [(pred, clip, nh, last, noise, zl) for pred in (E.PRED_EPSILON, E.PRED_SAMPLE, E.PRED_V) for clip in (False, True)
         for nh in (0, 1, 2) for last in (False, True) for noise in (False, True)
         for zl in ((False, True) if last else (False,))]


@pytest.mark.parametrize("pred,clip,n_hist,last,noise,last_noise", CASES)
def test_kernel_matches_the_solver(cuda_device, pred, clip, n_hist, last, noise, last_noise):
    p, folded = _plan(pred, clip, n_hist, last, noise, last_noise)
    worst = 0.0
    for n in (1, 7, 8, 4099):
        for offset in (0, 1):
            (m, s, l_, zl, h0, h1, z), c, prev, x0, xc = _run_kernel(p, folded, n_hist, last, noise, last_noise, n,
                                                                     offset, n + offset)
            hist = [h0, h1][:n_hist]
            want = E.solver_step(m, s, l_, zl, hist, z, p)
            abi = E.abi_step(m, s, l_ if last else None, zl if last_noise else None, hist, z if noise else None, c, n)
            for w, a, got in zip(want, abi, (prev, x0, xc)):
                ex = E.excess(w, got).max().item()
                assert ex <= 1.0 and E.excess(a, got).max() <= 1.0, (n, offset, ex)
                worst = max(worst, ex)
            if not last:
                assert torch.equal(xc, s), "without a corrector the corrected sample is the sample"
    print(f"sa_solver_step pred={pred} clip={clip} n_hist={n_hist} last={last} noise={noise} last_noise={last_noise}: "
          f"largest err/bound {worst:.3f}")


def test_kernel_at_the_c3_volume(cuda_device):
    n = 160 * 224 * 160
    p, folded = _plan(E.PRED_EPSILON, True, 2, True, True, True)
    (m, s, l_, zl, h0, h1, z), _, prev, x0, xc = _run_kernel(p, folded, 2, True, True, True, n, 0, 3)
    for w, got in zip(E.solver_step(m, s, l_, zl, [h0, h1], z, p), (prev, x0, xc)):
        assert E.excess(w, got).max() <= 1.0


def test_kernel_repeats_bit_identical(cuda_device):
    p, folded = _plan(E.PRED_V, True, 2, True, True, True)
    a = _run_kernel(p, folded, 2, True, True, True, 4099, 0, 9)
    b = _run_kernel(p, folded, 2, True, True, True, 4099, 0, 9)
    assert all(torch.equal(x, y) for x, y in zip(a[2:], b[2:]))


# ------------------------------------------------------------------------------------------------ tau = 1 vs SDE
def test_tau_one_order_one_is_dpm_solver_sde_order_one(cuda_device):
    """tau = 1, predictor order 1, no corrector against DPMSolverMultistepScheduler's SDE order 1 over 50 steps, from
    the same inputs and one seed at each step: where the two hosts' fp32 weights are equal the kernels' samples are
    bit-identical (one product and the same fmas in the same order, on the same noise); elsewhere the weights differ by
    an fp32 rounding, so the samples differ by at most 10 u times the terms' magnitudes."""
    from generativemodels_b200.networks.schedulers import DPMSolverMultistepScheduler
    from generativemodels_b200.networks.schedulers.dpm_solver import dpm_solver_weights
    sa = _sched(predictor_order=1, corrector_order=0, tau_func=_const(1.0), clip_sample=False)
    d = DPMSolverMultistepScheduler(solver_order=1, algorithm_type="sde-dpmsolver++", clip_sample=False)
    sa.set_timesteps(50)
    d.set_timesteps(50)
    acp = d.alphas_cumprod.double()
    a, sg = acp.sqrt(), (1 - acp).sqrt()
    lam = a.log() - sg.log()
    g = torch.Generator().manual_seed(0)
    gs, gd = torch.Generator().manual_seed(1), torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, 16, 16, generator=g).cuda()
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))       # noqa: E731
    equal_w, same = 0, 0
    for i, t in enumerate(sa.timesteps.tolist()):
        m = torch.randn(2, 3, 16, 16, generator=g).cuda()
        state = gd.get_state()
        got, got_x0 = sa.step(m, t, x, generator=gs)
        want, want_x0 = d.step(m, t, x, generator=gd)
        assert torch.equal(got_x0, want_x0) and torch.equal(gs.get_state(), gd.get_state()), i
        a_t, s_t = d._targets[i]
        _, _, _, c_xc, u, c_z = sa_solver_weights([float(a[t])], [float(sg[t])], [float(lam[t])], a_t, s_t, 1, 0, 1.0)
        c_x, w, c_zd = dpm_solver_weights(float(a[t]), float(sg[t]), a_t, s_t, [float(lam[t])], 1, True)
        if (f32(c_xc), f32(u[0]), f32(c_z)) == (f32(c_x), f32(w[0]), f32(c_zd)):
            equal_w += 1
            assert torch.equal(got, want), i
        z = torch.zeros_like(x)
        if c_zd:
            gd2 = torch.Generator()
            gd2.set_state(state)
            z = torch.randn(x.shape, generator=gd2).cuda()
        terms = abs(c_x) * x.abs() + abs(w[0]) * want_x0.abs() + abs(c_zd) * z.abs()
        assert ((got - want).abs() <= 10 * 2.0 ** -24 * terms).all(), i
        same += bool(torch.equal(got, want))
        x = want
    print(f"tau = 1 order 1 vs SDE order 1, 50 steps: fp32 weights equal at {equal_w}, samples bit-identical at {same}")
    assert equal_w >= 25, equal_w


# ------------------------------------------------------------------------------------------------ the Gaussian model
# (predictor order, corrector order) -> the slopes tests/test_sa_solver_cpu.py measured with the float64 formulas
GPU_SLOPES = {"tau=1": {(1, 0): (0.89, 0.95), (1, 2): (1.77, 1.94), (2, 2): (2.91, 2.80), (2, 3): (2.72, 2.53)},
              "default tau": {(1, 0): (1.01, 0.95), (1, 2): (2.16, 1.94), (2, 2): (2.92, 2.57), (2, 3): (2.64, 2.42)},
              "tau=0": {(1, 0): (0.99, 1.00), (1, 2): (2.06, 2.03), (2, 2): (3.98, 4.01), (2, 3): (3.05, 2.88)}}


@pytest.mark.parametrize("which", list(GPU_SLOPES))
def test_gaussian_model_convergence(cuda_device, monkeypatch, which):
    """The scheduler on the GPU, its kernel carrying the Gaussian model's coefficient vectors (an fp32 tensor over
    (1, zeta, xi_0, xi_1, ...)) and each noise draw the unit vector of that step's xi: the errors at 20, 40 and 80 steps
    track the float64 formulas' within 2 %, and the slopes are within 0.3 of the measured ones."""
    tau = {"tau=1": _const(1.0), "default tau": None, "tau=0": _const(0.0)}[which]
    weak = which != "tau=0"
    real_randn, queue = torch.randn, []

    def randn(shape, dtype=None, generator=None):
        return queue.pop().reshape(shape).to(dtype)
    lines = []
    for (p, q), want in GPU_SLOPES[which].items():
        errs, ref = [], []
        for n in (20, 40, 80):
            kw = dict(predictor_order=p, corrector_order=q, tau_func=tau, prediction_type="sample", clip_sample=False,
                      lower_order_final=False)
            s = _sched(**kw)
            s.set_timesteps(n)

            def step(m, t, x, z, s=s):
                queue[:] = [z.float()]
                out, _ = s.step(m.float().reshape(1, -1).cuda(), t, x.float().reshape(1, -1).cuda())
                return out.double().cpu().reshape(-1)
            monkeypatch.setattr(torch, "randn", randn)
            errs.append(E.gaussian_errors(s, step, MU, STD, weak))
            monkeypatch.setattr(torch, "randn", real_randn)
            ref.append(E.emulator_gaussian_error(_sched(**kw), n, MU, STD, weak))
        slopes = [math.log2(errs[k] / errs[k + 1]) for k in range(2)]
        lines.append(f"p={p} q={q}: errors {', '.join(f'{e:.3e}' for e in errs)} (float64 "
                     f"{', '.join(f'{e:.3e}' for e in ref)}), slopes {', '.join(f'{x:.2f}' for x in slopes)}")
        assert all(abs(a / b - 1.0) < 0.02 for a, b in zip(errs, ref)), (p, q, errs, ref)
        assert all(abs(a - b) <= 0.3 for a, b in zip(slopes, want)), (p, q, slopes, want)
    print(f"Gaussian model on the GPU, {which}:\n  " + "\n  ".join(lines))


# ------------------------------------------------------------------------------------------------ networks
class _EmulatorDriver:
    """The emulator scheduler with the oracle's step(model_output, t, x) interface (fp32 in, fp32 out), drawing each
    step's noise as the scheduler does: torch.randn of the output's shape on the global CPU generator, where the step
    injects noise."""

    def __init__(self, sched):
        self.em = E.EmulatorScheduler(sched)
        self.timesteps = sched.timesteps.cpu()

    def step(self, out, t, x):
        z = None
        if E.draws_noise(self.em.plan(self.em.i).predictor):
            z = torch.randn(out.shape, dtype=out.dtype)
        prev, x0 = self.em.step(out.double(), x.double(), None if z is None else z.double())
        return prev.float(), x0.float()


def _recipe(module, seed):
    sd = G.recipe_state_dict(module, seed)
    return {k: v.clone() for k, v in sd.items()}


def test_c1_unet_sampling_vs_oracle(cuda_device):
    from generativemodels_b200.inferers import DiffusionInferer
    from generativemodels_b200.networks.nets import DiffusionModelUNet
    m = DiffusionModelUNet(**G.C1_UNET).eval()
    sd = _recipe(m, 2024)
    s = _sched(clip_sample=False, tau_func=_const(1.0))    # no clip, for the reason tests/test_dpm_solver_gpu.py gives
    s.set_timesteps(5)
    noise = torch.randn(*G.C1_SHAPE, generator=torch.Generator().manual_seed(1))
    cfg = G.unet_oracle_cfg(G.C1_UNET)
    torch.manual_seed(5)
    with torch.no_grad():
        want = O.diffusion_sample(lambda x, t, c: O.unet_forward(sd, cfg, x, t, context=c), _EmulatorDriver(s), noise)
    torch.manual_seed(5)
    got = DiffusionInferer(s).sample(noise.cuda(), m.cuda(), s, verbose=False)
    print(f"C1 SA-Solver 5 steps (tau = 1) vs oracle: rel L2 {_check_traj(got, want, 'C1 sample'):.3e}")


def test_c2_latent_sampling_vs_oracle(cuda_device):
    from generativemodels_b200.inferers import LatentDiffusionInferer
    from generativemodels_b200.networks.nets import AutoencoderKL, DiffusionModelUNet
    ae, un = AutoencoderKL(**G.C2_AEKL).eval(), DiffusionModelUNet(**G.C2_UNET).eval()
    asd, usd = _recipe(ae, 7), _recipe(un, 8)
    s = _sched(clip_sample=False, **G.C2_SCHEDULER)
    s.set_timesteps(10)
    noise = torch.randn(*G.C2_LATENT, generator=torch.Generator().manual_seed(2))
    ucfg, acfg = G.unet_oracle_cfg(G.C2_UNET), G.aekl_oracle_cfg(G.C2_AEKL)
    torch.manual_seed(6)
    with torch.no_grad():
        lat = O.diffusion_sample(lambda x, t, c: O.unet_forward(usd, ucfg, x, t, context=c), _EmulatorDriver(s), noise)
        want = O.autoencoderkl_decode(asd, acfg, lat)
    torch.manual_seed(6)
    got = LatentDiffusionInferer(s, scale_factor=1.0).sample(noise.cuda(), ae.cuda(), un.cuda(), s, verbose=False)
    print(f"C2 latent SA-Solver 10 steps vs oracle: rel L2 {_check_traj(got, want, 'C2 sample'):.3e}")


def _small_unet():
    from generativemodels_b200.networks.nets import DiffusionModelUNet
    torch.manual_seed(0)
    return G.randomize_zero_params(DiffusionModelUNet(**G.UNET_CASES["unet2d_attn"])).cuda().eval()


@pytest.mark.parametrize("kw", [dict(), dict(predictor_order=3, corrector_order=3, tau_func=_const(0.6))])
def test_graph_replay_and_repeats_bit_identical(cuda_device, monkeypatch, kw):
    """The auto-graph path (>= 8 steps) reuses the network's output buffer; the history holds the kernel's own x0 and
    corrected sample and the scheduler's own noise, so replayed and eager sampling from one seed agree bit for bit,
    and so do repeated runs of one scheduler."""
    import generativemodels_b200.inferers.inferer as I
    from generativemodels_b200.inferers import DiffusionInferer
    m = _small_unet()
    x = torch.randn(2, 1, 16, 16, generator=torch.Generator().manual_seed(1)).cuda()
    s = _sched(**kw)
    s.set_timesteps(10)
    outs = {}
    for graph in (False, True, True):
        monkeypatch.setattr(I, "AUTO_CUDA_GRAPH", graph)
        torch.manual_seed(3)
        outs.setdefault(graph, []).append(DiffusionInferer(s).sample(x, m, s, verbose=False))
    assert "_b200_auto_graph" in m.__dict__
    assert torch.equal(outs[False][0], outs[True][0]), "graph-replayed sampling differs from eager"
    assert torch.equal(outs[True][0], outs[True][1]), "repeated sampling differs"
    assert torch.isfinite(outs[True][0]).all()


def test_brain_ldm_bundle_config_with_the_scheduler_swapped(cuda_device):
    """The bundle's unmodified inference.json with the scheduler's _target_ swapped, resolved at the fixture's reduced
    widths, against the oracle networks driving the emulator scheduler with the same noise."""
    from generativemodels_b200.bundle import BundleConfig
    from generativemodels_b200.networks.schedulers import SASolverScheduler
    fx = golden.load("g_bundle_brain_ldm")
    over = {"load_autoencoder": "$@autoencoder_def.load_state_dict(@states['aekl_state'])",
            "load_diffusion": "$@diffusion_def.load_state_dict(@states['unet_state'])",
            "noise": "$@states['noise'].to(@device)", "states": "$None",
            "scheduler#_target_": "generative.networks.schedulers.SASolverScheduler",
            "set_timesteps": "$@scheduler.set_timesteps(num_inference_steps=10)"}
    for item, kw in (("autoencoder_def", G.BUNDLE_AEKL), ("diffusion_def", G.BUNDLE_UNET)):
        for k, v in kw.items():
            over[f"{item}#{k}"] = list(v) if isinstance(v, tuple) else v
    cfg = BundleConfig(str(GOLD / "brain_ldm_inference.json"), json.loads(json.dumps(over)))
    cfg._resolved["states"] = fx
    s = cfg.get("scheduler")
    assert isinstance(s, SASolverScheduler) and not s.clip_sample
    torch.manual_seed(7)
    got = cfg.get("sample")
    assert len(s.timesteps) == 10
    ucfg, acfg = G.unet_oracle_cfg(fx["unet_kwargs"]), G.aekl_oracle_cfg(fx["aekl_kwargs"])
    ref = _sched(**G.BUNDLE_SCHEDULER)
    ref.set_timesteps(10)
    torch.manual_seed(7)
    with torch.no_grad():
        want = O.bundle_sampling_fn(lambda x, t, c: O.unet_forward(fx["unet_state"], ucfg, x, t, context=c),
                                    lambda z: O.autoencoderkl_decode(fx["aekl_state"], acfg, z), _EmulatorDriver(ref),
                                    fx["noise"], fx["conditioning"])
    print(f"brain-LDM config, SA-Solver 10 steps vs oracle: rel L2 {_check_traj(got, want, 'bundle'):.3e}")
