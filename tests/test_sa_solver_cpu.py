"""SASolverScheduler without a GPU: constructor, grids and orders (DPMSolverMultistepScheduler's), the host's folding
(sa_solver_weights) against scipy's quadrature of the exact integral and against the unfolded formulas
(tests/sa_solver_emulator.py), tau = 1 order 1 against DPM-Solver++ SDE order 1, the noise draws, the corrector rules,
history and dtypes through the CPU stand-in of the C ABI (tests/sa_solver_backend.py), every inferer's sample, and
the measured weak and strong convergence on a Gaussian model propagated exactly."""
import ctypes as C
import math
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch
from scipy.integrate import quad

from generativemodels_b200 import _lib
from generativemodels_b200.inferers import (ControlNetDiffusionInferer, ControlNetLatentDiffusionInferer,
                                            DiffusionInferer, LatentDiffusionInferer)
from generativemodels_b200.networks.schedulers import DPMSolverMultistepScheduler, SASolverScheduler
from generativemodels_b200.networks.schedulers.dpm_solver import dpm_solver_weights
from generativemodels_b200.networks.schedulers.sa_solver import default_tau, sa_solver_weights
from tests import sa_solver_backend
from tests import sa_solver_emulator as E

ROOT = Path(__file__).resolve().parents[1]
MU, STD = 0.3, 0.5


@pytest.fixture
def fake(monkeypatch):
    return sa_solver_backend.install(monkeypatch)


def _tables(s):
    acp = s.alphas_cumprod.double()
    a, sg = acp.sqrt(), (1 - acp).sqrt()
    return a, sg, (a.log() - sg.log())


def _const(tau):
    return lambda t: tau


# ------------------------------------------------------------------------------------------------ constructor
def test_defaults_follow_dpm_solver():
    s, d = SASolverScheduler(), DPMSolverMultistepScheduler()
    assert s.predictor_order == 2 and s.corrector_order == 2 and s.tau_func is default_tau
    assert [default_tau(t) for t in (0, 199, 200, 500, 800, 801, 999)] == [0.0, 0.0, 1.0, 1.0, 1.0, 0.0, 0.0]
    for k in ("num_train_timesteps", "prediction_type", "clip_sample", "clip_sample_values", "timestep_spacing",
              "steps_offset", "lower_order_final", "solver_order"):
        assert getattr(s, k) == getattr(d, k), k
    assert torch.equal(s.final_alpha_cumprod, d.final_alpha_cumprod) and torch.equal(s.betas, d.betas)
    assert torch.equal(s.timesteps, d.timesteps) and s.orders == d.orders
    s2 = SASolverScheduler(schedule="scaled_linear_beta", beta_start=0.0015, beta_end=0.0205, set_alpha_to_one=False,
                           predictor_order=3, corrector_order=0, tau_func=_const(0.5))
    assert torch.equal(s2.alphas_cumprod, DPMSolverMultistepScheduler(schedule="scaled_linear_beta", beta_start=0.0015,
                                                                      beta_end=0.0205).alphas_cumprod)
    assert s2.solver_order == 3 and s2.corrector_order == 0 and s2.tau_func(7) == 0.5


@pytest.mark.parametrize("kw,msg", [
    (dict(prediction_type="x0"), "prediction_type"),
    (dict(clip_sample_min=1, clip_sample_max=1), "clip_sample_min"),
    (dict(predictor_order=0), "predictor_order"),
    (dict(predictor_order=4), "predictor_order"),
    (dict(corrector_order=-1), "corrector_order"),
    (dict(corrector_order=4), "corrector_order"),
    (dict(tau_func=1.0), "tau_func"),
    (dict(timestep_spacing="linspace"), "timestep_spacing"),
    (dict(steps_offset=999), "steps_offset"),
    (dict(steps_offset=-1), "steps_offset"),
])
def test_constructor_errors(kw, msg):
    with pytest.raises(ValueError, match=msg):
        SASolverScheduler(**kw)


@pytest.mark.parametrize("tau", [-0.5, math.inf, math.nan])
def test_a_bad_tau_is_refused_at_the_step(fake, tau):
    s = SASolverScheduler(tau_func=_const(tau))
    s.set_timesteps(5)
    with pytest.raises(ValueError, match="tau_func"):
        s.step(torch.zeros(1, 1, 4, 4), s.timesteps[0], torch.zeros(1, 1, 4, 4))
    assert s.counter == 0


def test_alias_and_exports():
    """Under the reference's import path, in a fresh interpreter."""
    code = ("import generative.networks.schedulers as G, generativemodels_b200.networks.schedulers as S; "
            "assert G.SASolverScheduler is S.SASolverScheduler")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    for p in (1, 2, 3):
        for q in (0, 1, 2, 3):
            SASolverScheduler(predictor_order=p, corrector_order=q)


# ------------------------------------------------------------------------------------------------ grids and orders
GRIDS = [dict(), dict(predictor_order=3), dict(predictor_order=1), dict(steps_offset=3), dict(schedule="cosine"),
         dict(lower_order_final=False, predictor_order=3), dict(set_alpha_to_one=False, lower_order_final=False),
         dict(timestep_spacing="leading"), dict(timestep_spacing="leading", steps_offset=1, set_alpha_to_one=False),
         dict(timestep_spacing="leading", schedule="cosine")]


@pytest.mark.parametrize("kw", GRIDS, ids=[",".join(f"{k}={v}" for k, v in g.items()) or "default" for g in GRIDS])
@pytest.mark.parametrize("n", [2, 3, 5, 10, 14, 15, 16, 25, 50, 333])
def test_grid_targets_and_orders_are_dpm_solvers(kw, n):
    dkw = {("solver_order" if k == "predictor_order" else k): v for k, v in kw.items()}
    s, d = SASolverScheduler(**kw), DPMSolverMultistepScheduler(**dkw)
    s.set_timesteps(n)
    d.set_timesteps(n)
    assert torch.equal(s.timesteps, d.timesteps) and s.orders == d.orders and s._targets == d._targets


def test_grid_errors_are_dpm_solvers():
    s = SASolverScheduler()
    for n in (0, 1):
        with pytest.raises(ValueError):
            s.set_timesteps(n)
    with pytest.raises(ValueError, match="cannot be larger"):
        s.set_timesteps(1001)
    with pytest.raises(ValueError, match="past the last trained timestep"):
        SASolverScheduler(timestep_spacing="leading", steps_offset=1).set_timesteps(1000)


# ------------------------------------------------------------------------------------------------ folding
def _quad_update(a_s, s_s, a_t, s_t, nodes, tau):
    """(c_x, [w_k], c_z) of one update from scipy's adaptive quadrature of the exact integral with the Lagrange basis
    in lambda, in float64."""
    lam_s, lam_t = math.log(a_s) - math.log(s_s), math.log(a_t) - math.log(s_t)
    h, t2 = lam_t - lam_s, tau * tau
    c = 1.0 + t2

    def basis(k, lam):
        return math.prod((lam - lj) / (nodes[k] - lj) for j, lj in enumerate(nodes) if j != k)
    w = [a_t * c * quad(lambda u: math.exp(-c * u) * basis(k, lam_t - u), 0.0, h, epsabs=0.0, epsrel=1e-13)[0]
         for k in range(len(nodes))]
    return s_t / s_s * math.exp(-t2 * h), w, s_t * math.sqrt(1.0 - math.exp(-2.0 * t2 * h))


FOLD = ([(p, q, tau, "next") for p in (1, 2, 3) for q in (0, 1, 2, 3) for tau in (0.0, 0.5, 1.0)]
        + [(1, q, tau, t) for t in ("sigma0", "h0") for q in (0, 1, 2, 3) for tau in (0.0, 0.5, 1.0)])


@pytest.mark.parametrize("order,q,tau,target", FOLD)
def test_sa_solver_weights_match_the_exact_integral(order, q, tau, target):
    """The host's closed-form folding against scipy.integrate.quad of the exact integral, predictor and corrector, to
    float64 rounding (the corrector's tau is a different one, 0.7, as the previous step's would be).  A step to sigma = 0
    is x_t = alpha_t x0 without noise, a step over h = 0 leaves the sample as it is.  Then the fp32-rounded weights
    through the entry point's reading stay within the unfolded formulas' bound (what the GPU test holds the kernel
    to)."""
    s = SASolverScheduler()
    a, sg, lam = _tables(s)
    ts = [400, 470, 560]
    tgt = {"next": 300, "sigma0": -1, "h0": 400}[target]
    a_t, s_t = (float(a[tgt]), float(sg[tgt])) if tgt >= 0 else (1.0, 0.0)
    f = lambda v: [float(v[t]) for t in ts]         # noqa: E731
    tau_last = 0.7
    c_last, v, c_zl, c_xc, u, c_z = sa_solver_weights(f(a), f(sg), f(lam), a_t, s_t, order, q, tau, tau_last)
    assert all(isinstance(x, float) for x in [c_last, c_zl, c_xc, c_z] + v + u)
    if target == "next":
        want_x, want_w, want_z = _quad_update(f(a)[0], f(sg)[0], a_t, s_t, f(lam)[:order], tau)
    elif target == "sigma0":
        want_x, want_w, want_z = 0.0, [1.0], 0.0
    else:
        want_x, want_w, want_z = 1.0, [0.0], 0.0
    scale = abs(want_x) + sum(abs(w) for w in want_w) + abs(want_z)
    got = [c_xc] + u[:order] + [c_z]
    assert max(abs(x - y) for x, y in zip(got, [want_x] + want_w + [want_z])) <= 1e-13 * scale, (got, want_w)
    assert u[order:] == [0.0] * (3 - order)
    if q:
        want_x, want_w, want_z = _quad_update(f(a)[1], f(sg)[1], f(a)[0], f(sg)[0], f(lam)[:q], tau_last)
        scale = abs(want_x) + sum(abs(w) for w in want_w) + abs(want_z)
        got = [c_last] + v[:q] + [c_zl]
        assert max(abs(x - y) for x, y in zip(got, [want_x] + want_w + [want_z])) <= 1e-13 * scale, (got, want_w)
    else:
        assert (c_last, v, c_zl) == (0.0, [0.0] * 3, 0.0)
    # the fp32 weights through the entry point's reading, against the unfolded formulas' bound
    pr = E.Interval(f(a)[0], f(sg)[0], a_t, s_t, f(lam)[:order], tau)
    cor = E.Interval(f(a)[1], f(sg)[1], f(a)[0], f(sg)[0], f(lam)[:q], tau_last) if q else None
    step = E.Step(E.PRED_EPSILON, f(a)[0], f(sg)[0], pr, cor, True)
    g = torch.Generator().manual_seed(order * 17 + q * 3 + int(10 * tau))
    n = 4099
    m, x, last, zl, h0, h1, z = (torch.randn(n, generator=g) for _ in range(7))
    hist = [h0, h1][:max(order, q) - 1]
    c = _coef(E.PRED_EPSILON, step.alpha_s, step.sigma_s, (c_last, v, c_zl, c_xc, u, c_z), clip=True)
    got = E.abi_step(m, x, last if q else None, zl if c_zl else None, hist, z if c_z else None, c, n)
    want = E.solver_step(m, x, last, zl, hist, z, step)
    for w, g_ in zip(want, got):
        assert E.excess(w, g_.out).max() <= 1.0


def _coef(pred, a_s, s_s, folded, clip=False):
    c_last, v, c_zl, c_xc, u, c_z = folded
    c = _lib.SASolverCoef(alpha_s=a_s, sigma_s=s_s, c_last=c_last, c_zlast=c_zl, c_xc=c_xc, c_z=c_z, clip_min=-1,
                          clip_max=1, prediction_type=pred, clip=int(clip))
    for k in range(3):
        c.v[k], c.u[k] = v[k], u[k]
    return c


def test_bound_rejects_a_wrong_weight():
    """A folding that moves the corrector's weight of the older estimate onto x0 is far outside the bound."""
    s = SASolverScheduler()
    a, sg, lam = _tables(s)
    ts = [400, 470, 560]
    f = lambda v: [float(v[t]) for t in ts]         # noqa: E731
    folded = list(sa_solver_weights(f(a), f(sg), f(lam), float(a[300]), float(sg[300]), 2, 2, 1.0, 1.0))
    c = _coef(E.PRED_SAMPLE, f(a)[0], f(sg)[0], folded)
    c.v[0], c.v[1] = c.v[0] + c.v[1], 0.0
    pr = E.Interval(f(a)[0], f(sg)[0], float(a[300]), float(sg[300]), f(lam)[:2], 1.0)
    cor = E.Interval(f(a)[1], f(sg)[1], f(a)[0], f(sg)[0], f(lam)[:2], 1.0)
    step = E.Step(E.PRED_SAMPLE, f(a)[0], f(sg)[0], pr, cor)
    m, x, last, zl, h0, z = (torch.randn(64, generator=torch.Generator().manual_seed(i)) for i in range(6))
    bad = E.abi_step(m, x, last, zl, [h0], z, c, 64)
    want = E.solver_step(m, x, last, zl, [h0], z, step)
    assert E.excess(want[2], bad[2].out).max() > 100 and E.excess(want[0], bad[0].out).max() > 100


# ------------------------------------------------------------------------------------------------ tau = 1 vs SDE
@pytest.mark.parametrize("kw", [dict(), dict(timestep_spacing="leading"),
                                dict(set_alpha_to_one=False, schedule="scaled_linear_beta", beta_start=0.0015,
                                     beta_end=0.0205)])
def test_tau_one_order_one_is_dpm_solver_sde_order_one(fake, kw):
    """tau = 1, predictor order 1 and no corrector is DPM-Solver++ SDE order 1: the weights agree to float64 rounding
    at every step of 50, one seed draws the same noise, and the trajectories through the stand-in agree within its
    bound (bit for bit wherever the fp32 weights are equal)."""
    sa = SASolverScheduler(predictor_order=1, corrector_order=0, tau_func=_const(1.0), clip_sample=False, **kw)
    d = DPMSolverMultistepScheduler(solver_order=1, algorithm_type="sde-dpmsolver++", clip_sample=False, **kw)
    sa.set_timesteps(50)
    d.set_timesteps(50)
    a, sg, lam = _tables(sa)
    ts = sa.timesteps.tolist()
    for i, t in enumerate(ts):
        a_t, s_t = d._targets[i]
        _, _, _, c_xc, u, c_z = sa_solver_weights([float(a[t])], [float(sg[t])], [float(lam[t])], a_t, s_t, 1, 0, 1.0)
        c_x, w, c_zd = dpm_solver_weights(float(a[t]), float(sg[t]), a_t, s_t, [float(lam[t])], 1, True)
        scale = abs(c_x) + abs(w[0]) + abs(c_zd)
        assert max(abs(c_xc - c_x), abs(u[0] - w[0]), abs(c_z - c_zd)) <= 1e-13 * scale, i
    gs, gd = torch.Generator().manual_seed(0), torch.Generator().manual_seed(0)
    x = torch.randn(1, 2, 8, 8, generator=torch.Generator().manual_seed(1))
    same = 0
    for t in ts:
        m = torch.randn(1, 2, 8, 8, generator=torch.Generator().manual_seed(100 + int(t)))
        x_s, x0_s = sa.step(m, t, x, generator=gs)
        x_d, x0_d = d.step(m, t, x, generator=gd)
        assert torch.equal(x0_s, x0_d) and torch.equal(gs.get_state(), gd.get_state())
        assert ((x_s - x_d).abs() <= 1e-5 * (1 + x_d.abs())).all()
        same += bool(torch.equal(x_s, x_d))
        x = x_d
    print(f"tau = 1 order 1 vs DPM-Solver++ SDE order 1, 50 steps: bit-identical at {same}")
    assert same >= 25, same


# ------------------------------------------------------------------------------------------------ noise draws
def test_noise_draws_count_and_order(fake):
    """One torch.randn of the model output's shape and dtype on the given CPU generator per step whose tau > 0 and
    whose target has sigma > 0, in step order; none where tau = 0.  The kernel receives each step's noise, and the
    next step's corrector receives it again."""
    s = SASolverScheduler(clip_sample=False)
    s.set_timesteps(20)
    ts = s.timesteps.tolist()
    lib = _lib.require_device()
    calls = []
    orig = type(lib).b200_sa_solver_step

    def spy(self, m, x, last, zl, hist, n_hist, z, c, prev, x0o, xco, n, stream):
        calls.append((zl, z))
        return orig(self, m, x, last, zl, hist, n_hist, z, c, prev, x0o, xco, n, stream)
    type(lib).b200_sa_solver_step = spy
    try:
        g, g2 = torch.Generator().manual_seed(3), torch.Generator().manual_seed(3)
        x = torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(0), dtype=torch.float16)
        drawn = []
        for i, t in enumerate(ts):
            x, _ = s.step(torch.randn(1, 1, 8, 8, dtype=torch.float16), t, x, generator=g)
            draws = default_tau(t) > 0
            if draws:
                want = torch.randn(1, 1, 8, 8, dtype=torch.float16, generator=g2).float()
                assert torch.equal(s._noise, want), i
                drawn.append(i)
            else:
                assert s._noise is None, i
            assert torch.equal(g.get_state(), g2.get_state()), i
    finally:
        type(lib).b200_sa_solver_step = orig
    assert 0 < len(drawn) < len(ts)
    for i, (zl, z) in enumerate(calls):
        assert bool(z) == (i in drawn)
        assert bool(zl) == (i - 1 in drawn), i


# ------------------------------------------------------------------------------------------------ inferers
def _analytic_model(sched, pred):
    acp = sched.alphas_cumprod.double()

    def model(x, timesteps, context=None, **kw):
        t = int(timesteps[0])
        a, s = math.sqrt(float(acp[t])), math.sqrt(1.0 - float(acp[t]))
        x0 = E.gaussian_x0(x.double(), a, s, MU, STD)
        eps = (x.double() - a * x0) / s if s > 0 else torch.zeros_like(x0)      # sigma = 0 at t = 0 of the cosine
        return {"epsilon": eps, "sample": x0, "v_prediction": a * eps - s * x0}[pred].to(x.dtype)
    return model


PATHS = [
    dict(),
    dict(tau_func=_const(0.0)),
    dict(tau_func=_const(1.0), predictor_order=1, corrector_order=0),
    dict(predictor_order=1, corrector_order=1),
    dict(predictor_order=3, corrector_order=3, tau_func=_const(0.5)),
    dict(predictor_order=3, corrector_order=3, lower_order_final=False),
    dict(predictor_order=1, corrector_order=3),
    dict(prediction_type="v_prediction"),
    dict(prediction_type="sample", predictor_order=3),
    dict(timestep_spacing="leading"),
    dict(timestep_spacing="leading", set_alpha_to_one=False, steps_offset=1),
    dict(timestep_spacing="leading", schedule="cosine"),       # the last timestep has sigma = 0
    dict(steps_offset=3, predictor_order=3, set_alpha_to_one=False),
    dict(clip_sample=True, clip_sample_min=-0.5, clip_sample_max=0.8),
]


def _path_id(p):
    return ",".join(f"{k}={v(500) if callable(v) else v}" for k, v in p.items()) or "default"


@pytest.mark.parametrize("kw", PATHS, ids=[_path_id(p) for p in PATHS])
def test_scheduler_paths_through_the_inferer(fake, kw):
    """DiffusionInferer.sample with the analytic model through the stand-in, the noise drawn from one seeded
    generator: every step equals the emulator scheduler's step from the same inputs and the same noise, within its
    bound, and every step after the first corrects unless corrector_order is 0."""
    kw = dict(dict(clip_sample=False), **kw)
    s = SASolverScheduler(**kw)
    s.set_timesteps(12)
    em = E.EmulatorScheduler(s)
    model = _analytic_model(s, kw.get("prediction_type", "epsilon"))
    x_T = torch.randn(1, 2, 16, 16, generator=torch.Generator().manual_seed(3))
    seen = []

    def spy(x, timesteps, context=None):
        out = model(x, timesteps, context)
        seen.append((x.clone(), out.clone()))
        return out
    g = torch.Generator().manual_seed(11)
    orig_step = s.step
    s.step = lambda m, t, x, generator=None: orig_step(m, t, x, generator=g)
    got = DiffusionInferer(s).sample(x_T, spy, s, verbose=False)
    assert len(seen) == 12 and s.counter == 12
    g2 = torch.Generator().manual_seed(11)
    corrected = 0
    for i, (x, m) in enumerate(seen):
        p = em.plan(i)
        corrected += p.corrector is not None
        z = torch.randn(m.shape, dtype=m.dtype, generator=g2) if E.draws_noise(p.predictor) else None
        hist = [h.reshape(-1) for h, _ in reversed(em.hist)]
        flat = (lambda t: None if t is None else t.reshape(-1))          # noqa: E731
        want_p, want_x, want_c = E.solver_step(m.reshape(-1), x.reshape(-1), flat(em.last), flat(em.last_noise), hist,
                                               flat(z), p)
        nxt = seen[i + 1][0] if i + 1 < len(seen) else got
        assert E.excess(want_p, nxt.reshape(-1)).max() <= 1.0, i
        em.hist = (em.hist + [(want_x.out.view(x.shape), em.grid[i])])[-2:]
        em.last, em.last_noise, em.tau = want_c.out.view(x.shape), z, p.predictor.tau
    assert torch.equal(g.get_state(), g2.get_state())
    assert corrected == (11 if kw.get("corrector_order", 2) else 0)


class _IdentityAutoencoder:
    def decode_stage_2_outputs(self, z):
        return z


def test_every_inferer_samples_with_sa_solver(fake):
    """DiffusionInferer, LatentDiffusionInferer and the two ControlNet inferers drive the same trajectory from the
    same seed (the ControlNet adds zero residuals, the autoencoder decodes to the latent itself), noise included."""
    s = SASolverScheduler(clip_sample=False)
    s.set_timesteps(10)
    model = _analytic_model(s, "epsilon")
    x_T = torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(5))

    def controlnet(x, timesteps, controlnet_cond, context=None):
        return [torch.zeros_like(x)], torch.zeros_like(x)

    def unet(x, timesteps, context=None, down_block_additional_residuals=None, mid_block_additional_residual=None):
        return model(x, timesteps)
    cond = torch.zeros(1, 1, 8, 8)
    runs = [lambda: DiffusionInferer(s).sample(x_T, model, s, verbose=False),
            lambda: LatentDiffusionInferer(s).sample(x_T, _IdentityAutoencoder(), model, s, verbose=False),
            lambda: ControlNetDiffusionInferer(s).sample(x_T, unet, controlnet, cond, s, verbose=False),
            lambda: ControlNetLatentDiffusionInferer(s).sample(x_T, _IdentityAutoencoder(), unet, controlnet, cond, s,
                                                               verbose=False)]
    outs = []
    for run in runs:
        torch.manual_seed(0)
        outs.append(run())
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    assert torch.isfinite(outs[0]).all() and not torch.equal(outs[0], x_T)


# ------------------------------------------------------------------------------------------------ convergence
# Measured on the 1000-step linear_beta schedule's log-SNR grid, lower_order_final off, prediction_type "sample", at
# 20 -> 40 -> 80 steps: (predictor order, corrector order) -> the two slopes at tau = 1 and at the default tau_func
# (weak error), and at tau = 0 (strong error of the ODE).  None: not asserted (pre-asymptotic at these step counts).
WEAK_TAU1 = {(1, 0): (0.89, 0.95), (1, 1): None, (1, 2): (1.77, 1.94), (1, 3): (1.81, 1.97),
             (2, 0): (2.13, 2.08), (2, 1): (1.04, 0.92), (2, 2): (2.91, 2.80), (2, 3): (2.72, 2.53),
             (3, 0): (2.35, 1.93), (3, 1): None, (3, 2): (3.38, 1.91), (3, 3): (2.57, 1.77)}
WEAK_DEFAULT = {(1, 0): (1.01, 0.95), (1, 1): None, (1, 2): (2.16, 1.94), (1, 3): (2.21, 1.94),
                (2, 0): (1.97, 2.14), (2, 1): (0.99, 0.93), (2, 2): (2.92, 2.57), (2, 3): (2.64, 2.42),
                (3, 0): (2.16, 2.37), (3, 1): None, (3, 2): (2.67, 1.98), (3, 3): (2.05, 2.00)}
STRONG_ODE = {(1, 0): (0.99, 1.00), (1, 1): None, (1, 2): (2.06, 2.03), (1, 3): (2.12, 2.07),
              (2, 0): (2.11, 2.07), (2, 1): (1.01, 0.97), (2, 2): (3.98, 4.01), (2, 3): (3.05, 2.88),
              (3, 0): None, (3, 1): None, (3, 2): None, (3, 3): None}
NS = (20, 40, 80)


def _slopes(kw, weak):
    errs = [E.emulator_gaussian_error(SASolverScheduler(prediction_type="sample", clip_sample=False,
                                                        lower_order_final=False, **kw), n, MU, STD, weak) for n in NS]
    return errs, [math.log2(errs[k] / errs[k + 1]) for k in range(len(NS) - 1)]


@pytest.mark.parametrize("which,table", [("tau=1", WEAK_TAU1), ("default tau", WEAK_DEFAULT), ("tau=0", STRONG_ODE)])
def test_convergence_on_the_gaussian_model(which, table):
    """The exact law (weak) or the exact ODE path (strong, tau = 0) of the sample at the last evaluated timestep,
    against the float64 formulas run on the Gaussian model's exact propagation: every slope within 0.3 of the one
    measured, and in every case the error at 80 steps below the one at 20."""
    tau = {"tau=1": _const(1.0), "default tau": None, "tau=0": _const(0.0)}[which]
    lines = []
    for (p, q), want in table.items():
        errs, slopes = _slopes(dict(predictor_order=p, corrector_order=q, tau_func=tau), which != "tau=0")
        lines.append(f"p={p} q={q}: errors {', '.join(f'{e:.2e}' for e in errs)}, slopes "
                     f"{', '.join(f'{x:.2f}' for x in slopes)}")
        assert errs[-1] < errs[0], (p, q, errs)
        if want is not None:
            assert all(abs(a - b) <= 0.3 for a, b in zip(slopes, want)), (p, q, slopes, want)
    print(f"Gaussian model, {which}, 20-40-80 steps:\n  " + "\n  ".join(lines))


# ------------------------------------------------------------------------------------------------ state
def test_counter_history_and_corrector_state(fake):
    s = SASolverScheduler(clip_sample=False, predictor_order=3, corrector_order=3, tau_func=_const(0.5))
    s.set_timesteps(6)
    ts = s.timesteps.tolist()
    x = torch.randn(2, 3, 4, 4)
    m = torch.randn(2, 3, 4, 4)
    with pytest.raises(ValueError, match="out of order"):
        s.step(m, ts[1], x)
    outs = []
    for i, t in enumerate(ts):
        prev, x0 = s.step(m, t, x)
        outs.append(x0)
        assert s.counter == i + 1 and len(s._hist) == min(i + 1, 2)
        assert s._hist[-1][0] is x0 and x0.data_ptr() != m.data_ptr()
        assert s._last is not None and s._last.data_ptr() not in (x.data_ptr(), m.data_ptr(), prev.data_ptr())
        assert (s._noise is None) == (i == len(ts) - 1)               # the last step goes to sigma = 0: no noise
        x = prev
    with pytest.raises(ValueError, match="finished"):
        s.step(m, 0, x)
    kept = [o.clone() for o in outs]
    s.step(m, ts[0], x)                                  # a finished trajectory: timesteps[0] starts the next one
    assert s.counter == 1 and len(s._hist) == 1
    assert all(torch.equal(a, b) for a, b in zip(outs, kept))
    with pytest.raises(ValueError, match="expected"):
        s.step(m, ts[0], x)
    s.set_timesteps(6)
    assert s.counter == 0 and s._hist == [] and s._last is None and s._noise is None
    s.step(m, ts[0], x)
    with pytest.raises(ValueError, match="changed shape"):
        s.step(m[:1], ts[1], x[:1])
    with pytest.raises(ValueError, match="changed shape"):
        s.step(m.reshape(3, 2, 4, 4), ts[1], x.reshape(3, 2, 4, 4))
    s.step(m, ts[1], x)


def test_corrector_over_a_zero_length_interval_is_skipped(fake):
    """Where two grid timesteps share one alphas_cumprod value, the step from the first to the second is order 1 and
    noise-free (DPM-Solver's rule for h = 0), and the second step's corrector, over an empty interval, is skipped: its
    corrected sample is the sample it was given."""
    s = SASolverScheduler(timestep_spacing="leading", clip_sample=False, prediction_type="sample", predictor_order=1,
                          corrector_order=1, tau_func=_const(1.0))
    s.set_timesteps(6)
    t = s.timesteps.tolist()
    for table in (s._alpha, s._sigma, s._lambda):
        table[t[2]] = table[t[1]]
    s.set_timesteps(6)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, 1, 4, 4, generator=g)
    for i, tt in enumerate(t):
        x_in = x
        x, _ = s.step(torch.randn(1, 1, 4, 4, generator=g), tt, x, generator=torch.Generator().manual_seed(i))
        assert torch.isfinite(x).all() and torch.isfinite(s._last).all()
        assert torch.equal(s._last, x_in) == (i in (0, 2)), i
        assert (s._noise is None) == (i in (1, 5)), i


def test_model_output_buffer_reuse_does_not_alias_history(fake):
    """A graph-replayed network hands back one buffer every step: the history must hold x0, the start sample and the
    noise in the scheduler's own tensors, not that buffer or the caller's sample."""
    def run(reuse):
        s = SASolverScheduler(clip_sample=False, prediction_type="sample", predictor_order=3, corrector_order=3,
                              tau_func=_const(0.8))
        s.set_timesteps(7)
        buf, xbuf = torch.empty(1, 1, 8, 8), torch.empty(1, 1, 8, 8)
        x = torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(1))
        g = torch.Generator().manual_seed(2)
        for i, t in enumerate(s.timesteps):
            v = torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(10 + i))
            if reuse:
                buf.copy_(v)
                xbuf.copy_(x)
                x, _ = s.step(buf, t, xbuf, generator=g)
            else:
                x, _ = s.step(v.clone(), t, x.clone(), generator=g)
        return x
    assert torch.equal(run(True), run(False))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_dtype_round_trip(fake, dtype):
    s = SASolverScheduler(tau_func=_const(1.0))
    s.set_timesteps(4)
    x = torch.randn(1, 2, 8, 8).to(dtype)
    for t in s.timesteps:
        x, x0 = s.step(torch.randn(1, 2, 8, 8).to(dtype), t, x)
        assert x.dtype == dtype and x0.dtype == dtype and x.shape == (1, 2, 8, 8)
    assert s._hist[-1][0].dtype == torch.float32 and s._last.dtype == torch.float32


# ------------------------------------------------------------------------------------------------ ABI
def test_header_binding_and_struct():
    text = (ROOT / "include" / "b200gen_samplers.h").read_text()
    declared = set(re.findall(r"^int (b200_\w+)\(", text, re.M))
    assert "b200_sa_solver_step" in declared and declared == set(_lib.SAMPLER_SIGNATURES)
    assert "B200_SA_SOLVER_MAX_HIST 2" in text and _lib.SA_SOLVER_MAX_HIST == 2
    assert "b200_abi_sizeof(16) is sizeof(b200_sa_solver_coef)" in text
    lib = _lib.load()
    assert lib.b200_abi_sizeof(16) == C.sizeof(_lib.SASolverCoef) == 64
    assert callable(getattr(sa_solver_backend.SASolverFakeLib, "b200_sa_solver_step"))


def test_entry_point_rejects_bad_arguments():
    """Argument checks run on the host before any launch, so they hold without a GPU."""
    lib = _lib.load()
    c = _lib.SASolverCoef(alpha_s=1.0, sigma_s=0.5, prediction_type=0)
    none = (C.c_void_p * 1)()
    args = dict(m=8, s=8, last=None, zl=None, hist=none, nh=0, z=None, c=C.byref(c), p=8, x0=8, xc=8, n=4)

    def call(**kw):
        a = dict(args, **kw)
        return lib.b200_sa_solver_step(a["m"], a["s"], a["last"], a["zl"], a["hist"], a["nh"], a["z"], a["c"], a["p"],
                                       a["x0"], a["xc"], a["n"], None)
    for bad in (dict(m=None), dict(s=None), dict(p=None), dict(x0=None), dict(xc=None), dict(n=0), dict(nh=3),
                dict(nh=-1), dict(nh=1), dict(c=None), dict(zl=8)):
        assert call(**bad) == _lib.B200_EINVAL, bad
    c.prediction_type = 7
    assert call() == _lib.B200_EINVAL
