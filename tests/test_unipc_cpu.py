"""UniPCMultistepScheduler without a GPU: constructor, grids and orders (DPMSolverMultistepScheduler's), the corrector
rules, history and dtypes through the CPU stand-in of the C ABI (tests/unipc_backend.py); the host's folding
(unipc_weights) against the unfolded formulas (tests/unipc_emulator.py); every inferer's sample; the formulas' order of
convergence on a Gaussian model; and UniPC-2 bh2 with every corrector disabled against DPM-Solver++ 2M."""
import ctypes as C
import math
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from generativemodels_b200 import _lib
from generativemodels_b200.inferers import (ControlNetDiffusionInferer, ControlNetLatentDiffusionInferer,
                                            DiffusionInferer, LatentDiffusionInferer)
from generativemodels_b200.networks.schedulers import DPMSolverMultistepScheduler, UniPCMultistepScheduler
from generativemodels_b200.networks.schedulers.dpm_solver import dpm_solver_weights
from generativemodels_b200.networks.schedulers.unipc import unipc_weights
from tests import unipc_backend
from tests import unipc_emulator as E

ROOT = Path(__file__).resolve().parents[1]
MU, STD = 0.3, 0.5
ALL_STEPS = tuple(range(1000))          # disable_corrector: every corrector off


@pytest.fixture
def fake(monkeypatch):
    return unipc_backend.install(monkeypatch)


def _tables(s):
    acp = s.alphas_cumprod.double()
    a, sg = acp.sqrt(), (1 - acp).sqrt()
    return a, sg, (a.log() - sg.log())


# ------------------------------------------------------------------------------------------------ constructor
def test_defaults_follow_dpm_solver():
    s, d = UniPCMultistepScheduler(), DPMSolverMultistepScheduler()
    assert s.solver_order == 2 and s.solver_type == "bh2" and s.disable_corrector == []
    for k in ("num_train_timesteps", "prediction_type", "clip_sample", "clip_sample_values", "timestep_spacing",
              "steps_offset", "lower_order_final"):
        assert getattr(s, k) == getattr(d, k), k
    assert torch.equal(s.final_alpha_cumprod, d.final_alpha_cumprod) and torch.equal(s.betas, d.betas)
    assert torch.equal(s.timesteps, d.timesteps) and s.orders == d.orders
    s2 = UniPCMultistepScheduler(schedule="scaled_linear_beta", beta_start=0.0015, beta_end=0.0205,
                                 set_alpha_to_one=False, disable_corrector=[0, 3])
    assert torch.equal(s2.alphas_cumprod, DPMSolverMultistepScheduler(schedule="scaled_linear_beta", beta_start=0.0015,
                                                                      beta_end=0.0205).alphas_cumprod)
    assert torch.equal(s2.final_alpha_cumprod, s2.alphas_cumprod[0]) and s2.disable_corrector == [0, 3]


@pytest.mark.parametrize("kw,msg", [
    (dict(prediction_type="x0"), "prediction_type"),
    (dict(clip_sample_min=1, clip_sample_max=1), "clip_sample_min"),
    (dict(solver_order=0), "solver_order"),
    (dict(solver_order=4), "solver_order"),
    (dict(solver_type="bh3"), "solver_type"),
    (dict(timestep_spacing="linspace"), "timestep_spacing"),
    (dict(steps_offset=999), "steps_offset"),
    (dict(steps_offset=-1), "steps_offset"),
])
def test_constructor_errors(kw, msg):
    with pytest.raises(ValueError, match=msg):
        UniPCMultistepScheduler(**kw)


def test_alias_and_exports():
    """Under the reference's import path, in a fresh interpreter."""
    code = ("import generative.networks.schedulers as G, generativemodels_b200.networks.schedulers as S; "
            "assert G.UniPCMultistepScheduler is S.UniPCMultistepScheduler")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    for order in (1, 2, 3):
        for bh in ("bh1", "bh2"):
            UniPCMultistepScheduler(solver_order=order, solver_type=bh)


# ------------------------------------------------------------------------------------------------ grids and orders
GRIDS = [dict(), dict(solver_order=3), dict(solver_order=1), dict(steps_offset=3), dict(schedule="cosine"),
         dict(lower_order_final=False, solver_order=3), dict(set_alpha_to_one=False, lower_order_final=False),
         dict(timestep_spacing="leading"), dict(timestep_spacing="leading", steps_offset=1, set_alpha_to_one=False),
         dict(timestep_spacing="leading", schedule="cosine")]


@pytest.mark.parametrize("kw", GRIDS, ids=[",".join(f"{k}={v}" for k, v in g.items()) or "default" for g in GRIDS])
@pytest.mark.parametrize("n", [2, 3, 5, 10, 14, 15, 16, 25, 50, 333])
def test_grid_targets_and_orders_are_dpm_solvers(kw, n):
    s, d = UniPCMultistepScheduler(**kw), DPMSolverMultistepScheduler(**kw)
    s.set_timesteps(n)
    d.set_timesteps(n)
    assert torch.equal(s.timesteps, d.timesteps) and s.orders == d.orders and s._targets == d._targets


def test_grid_errors_are_dpm_solvers():
    s = UniPCMultistepScheduler()
    for n in (0, 1):
        with pytest.raises(ValueError):
            s.set_timesteps(n)
    with pytest.raises(ValueError, match="cannot be larger"):
        s.set_timesteps(1001)
    with pytest.raises(ValueError, match="past the last trained timestep"):
        UniPCMultistepScheduler(timestep_spacing="leading", steps_offset=1).set_timesteps(1000)


# ------------------------------------------------------------------------------------------------ folding
def _one_hot_weights(step):
    """The unfolded formulas' own weights, in float64: each input in turn set to 1 (x^c_(i-1), m_i, m_(i-1), m_(i-2),
    m_(i-3) for the corrector; x^c, m_i, m_(i-1), m_(i-2) for the predictor)."""
    def unit(k, n):
        return [torch.tensor([1.0 if j == k else 0.0], dtype=torch.float64) for j in range(n)]
    cor = None
    if step.corrector is not None:
        q = step.corrector.order
        cor = []
        for k in range(5):
            last, mt, m0, m1, m2 = unit(k, 5)
            cor.append(float(E._apply(step.corrector, True, last, m0, [m1, m2][:q - 1], mt, False)))
    o = step.predictor.order
    pre = []
    for k in range(4):
        xc, m0, m1, m2 = unit(k, 4)
        pre.append(float(E._apply(step.predictor, False, xc, m0, [m1, m2][:o - 1], None, False)))
    return cor, pre


def _coef(pred, a_s, s_s, folded, clip=False):
    c_last, v, c_xc, u = folded
    c = _lib.UniPCCoef(alpha_s=a_s, sigma_s=s_s, c_last=c_last, c_xc=c_xc, clip_min=-1, clip_max=1,
                       prediction_type=pred, clip=int(clip))
    for k in range(4):
        c.v[k] = v[k]
    for k in range(3):
        c.u[k] = u[k]
    return c


def _case(s, ts, target, order, q, bh, pred=E.PRED_SAMPLE, clip=False):
    """A step at ts[0] with the earlier estimates at ts[1:], predicting to `target` (a timestep, or -1 for sigma = 0);
    corrector order q (0: none).  -> (emulator Step, folded weights)."""
    a, sg, lam = _tables(s)
    a_t, s_t = (float(a[target]), float(sg[target])) if target >= 0 else (1.0, 0.0)
    f = lambda v: [float(v[t]) for t in ts]         # noqa: E731
    folded = unipc_weights(f(a), f(sg), f(lam), a_t, s_t, order, q, bh)
    lams = f(lam)
    pr = E.Interval(f(a)[0], f(sg)[0], a_t, s_t, lams[:order], order, bh)
    cor = E.Interval(f(a)[1], f(sg)[1], f(a)[0], f(sg)[0], lams[1:q + 1], q, bh) if q else None
    return E.Step(pred, f(a)[0], f(sg)[0], pr, cor, clip), folded


FOLD = ([(o, q, bh, "next") for o in (1, 2, 3) for q in (0, 1, 2, 3) for bh in ("bh1", "bh2")]
        + [(1, q, bh, t) for t in ("sigma0", "h0") for q in (0, 1, 2, 3) for bh in ("bh1", "bh2")])


@pytest.mark.parametrize("order,q,bh,target", FOLD)
def test_unipc_weights_match_the_formulas(order, q, bh, target):
    """The host's float64 folding equals the unfolded formulas' weights to float64 rounding, and its fp32-rounded
    weights through the entry point's reading stay within the solver reading's bound (what the GPU test holds the
    kernel to).  A step to sigma = 0 or to its own timestep (h = 0) is order 1."""
    tgt = {"next": 300, "sigma0": -1, "h0": 400}[target]
    s = UniPCMultistepScheduler()
    ts = [400, 470, 560, 700]
    step, folded = _case(s, ts, tgt, order, q, bh, pred=E.PRED_EPSILON, clip=True)
    cor, pre = _one_hot_weights(step)
    c_last, v, c_xc, u = folded
    scale = sum(abs(w) for w in pre) + (sum(abs(w) for w in cor) if cor else 0.0)
    assert max(abs(a - b) for a, b in zip([c_xc] + u, pre)) <= 1e-12 * scale, ([c_xc] + u, pre)
    if cor:
        assert max(abs(a - b) for a, b in zip([c_last] + [v[0]] + v[1:], cor)) <= 1e-12 * scale, (v, cor)
    else:
        assert c_last == 0.0 and v == [0.0] * 4
    g = torch.Generator().manual_seed(order * 17 + q * 3 + len(bh))
    n = 4099
    m, x, last, h0, h1, h2 = (torch.randn(n, generator=g) for _ in range(6))
    n_hist = max(order - 1, q)
    hist = [h0, h1, h2][:n_hist]
    c = _coef(E.PRED_EPSILON, step.alpha_s, step.sigma_s, folded, clip=True)
    got = E.abi_step(m, x, last if q else None, hist, c, n)
    want = E.solver_step(m, x, last, hist, step)
    for w, g_ in zip(want, got):
        assert E.excess(w, g_.out).max() <= 1.0


def test_corrector_over_a_zero_length_interval_is_skipped(fake):
    """Where two grid timesteps share one alphas_cumprod value, the step from the first to the second is order 1
    (DPM-Solver's rule for h = 0) and the second step's corrector, over an empty interval, is skipped: its corrected
    sample is the sample it was given."""
    s = UniPCMultistepScheduler(timestep_spacing="leading", clip_sample=False, prediction_type="sample",
                                solver_order=1)
    s.set_timesteps(6)
    t = s.timesteps.tolist()
    for table in (s._alpha, s._sigma, s._lambda):
        table[t[2]] = table[t[1]]
    s.set_timesteps(6)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, 1, 4, 4, generator=g)
    for i, tt in enumerate(t):
        x_in = x
        x, _ = s.step(torch.randn(1, 1, 4, 4, generator=g), tt, x)
        assert torch.isfinite(x).all() and torch.isfinite(s._last).all()
        assert torch.equal(s._last, x_in) == (i in (0, 2)), i


def test_bound_rejects_a_wrong_weight():
    """A folding that drops the corrector's older-estimate term is far outside the bound."""
    s = UniPCMultistepScheduler()
    step, folded = _case(s, [400, 470, 560], 300, 2, 2, "bh2")
    c = _coef(E.PRED_SAMPLE, step.alpha_s, step.sigma_s, folded)
    c.v[1], c.v[2] = c.v[1] + c.v[2], 0.0
    m, x, last, h0, h1 = (torch.randn(64, generator=torch.Generator().manual_seed(i)) for i in range(5))
    bad = E.abi_step(m, x, last, [h0, h1], c, 64)
    want = E.solver_step(m, x, last, [h0, h1], step)
    assert E.excess(want[2], bad[2].out).max() > 100 and E.excess(want[0], bad[0].out).max() > 100


# ------------------------------------------------------------------------------------------------ UniPC-2 vs 2M
@pytest.mark.parametrize("kw", [dict(), dict(timestep_spacing="leading"), dict(lower_order_final=False),
                                dict(set_alpha_to_one=False, schedule="scaled_linear_beta", beta_start=0.0015,
                                     beta_end=0.0205)])
def test_correctors_off_is_dpm_solver_2m(fake, kw):
    """UniPC-2 bh2 with every corrector disabled is DPM-Solver++ 2M: the folded weights agree to float64 rounding at
    every step of 50, and the trajectories through the stand-in agree within the stand-in's bound (bit for bit wherever
    the fp32 weights are equal)."""
    u = UniPCMultistepScheduler(disable_corrector=ALL_STEPS, clip_sample=False, **kw)
    d = DPMSolverMultistepScheduler(clip_sample=False, **kw)
    u.set_timesteps(50)
    d.set_timesteps(50)
    a, sg, lam = _tables(u)
    ts = u.timesteps.tolist()
    for i, t in enumerate(ts):
        o = d.orders[i]
        a_t, s_t = d._targets[i]
        hist_t = ts[max(i - o + 1, 0):i][::-1]
        c_last, v, c_xc, uw = unipc_weights([float(a[k]) for k in [t] + hist_t], [float(sg[k]) for k in [t] + hist_t],
                                            [float(lam[k]) for k in [t] + hist_t], a_t, s_t, o, 0, "bh2")
        c_x, w, _ = dpm_solver_weights(float(a[t]), float(sg[t]), a_t, s_t, [float(lam[k]) for k in [t] + hist_t], o,
                                       False)
        scale = abs(c_x) + sum(abs(x) for x in w)
        assert abs(c_xc - c_x) <= 1e-13 * scale and max(abs(p - q) for p, q in zip(uw, w)) <= 1e-13 * scale, i
    g = torch.Generator().manual_seed(0)
    x_u = x_d = torch.randn(1, 2, 8, 8, generator=g)
    same = 0
    for t in ts:
        m = torch.randn(1, 2, 8, 8, generator=g)
        x_u, x0_u = u.step(m, t, x_u)
        x_d, x0_d = d.step(m, t, x_d)
        assert torch.equal(x0_u, x0_d)
        assert ((x_u - x_d).abs() <= 1e-5 * (1 + x_d.abs())).all()
        same += bool(torch.equal(x_u, x_d))
        x_u = x_d                                         # one trajectory: compare each step from the same inputs
    assert same >= 25, same


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
    dict(solver_type="bh1"),
    dict(solver_order=1),
    dict(solver_order=3),
    dict(solver_order=3, solver_type="bh1", lower_order_final=False),
    dict(prediction_type="v_prediction"),
    dict(prediction_type="sample", solver_order=3),
    dict(disable_corrector=[0, 4, 5]),
    dict(timestep_spacing="leading"),
    dict(timestep_spacing="leading", set_alpha_to_one=False, steps_offset=1),
    dict(timestep_spacing="leading", schedule="cosine"),       # the last timestep has sigma = 0
    dict(steps_offset=3, solver_order=3, set_alpha_to_one=False),
    dict(clip_sample=True, clip_sample_min=-0.5, clip_sample_max=0.8),
]


@pytest.mark.parametrize("kw", PATHS, ids=[",".join(f"{k}={v}" for k, v in p.items()) or "default" for p in PATHS])
def test_scheduler_paths_through_the_inferer(fake, kw):
    """DiffusionInferer.sample with the analytic model through the stand-in: every step equals the emulator
    scheduler's step from the same inputs, within its bound, and the sample reaches the exact endpoint."""
    kw = dict(dict(clip_sample=False), **kw)
    s = UniPCMultistepScheduler(**kw)
    s.set_timesteps(12)
    em = E.EmulatorScheduler(s)
    model = _analytic_model(s, kw.get("prediction_type", "epsilon"))
    x_T = torch.randn(1, 2, 16, 16, generator=torch.Generator().manual_seed(3))
    seen = []

    def spy(x, timesteps, context=None):
        out = model(x, timesteps, context)
        seen.append((x.clone(), out.clone()))
        return out
    got = DiffusionInferer(s).sample(x_T, spy, s, verbose=False)
    assert len(seen) == 12 and s.counter == 12
    corrected = 0
    for i, (x, m) in enumerate(seen):
        p = em.plan(i)
        corrected += p.corrector is not None
        hist = [h.reshape(-1) for h, _ in reversed(em.hist)]
        want_p, want_x, want_c = E.solver_step(m.reshape(-1), x.reshape(-1), None if em.last is None else
                                               em.last.reshape(-1), hist, p)
        nxt = seen[i + 1][0] if i + 1 < len(seen) else got
        assert E.excess(want_p, nxt.reshape(-1)).max() <= 1.0, i
        em.hist = (em.hist + [(want_x.out.view(x.shape), em.grid[i])])[-3:]
        em.last = want_c.out.view(x.shape)
    disabled = {k for k in kw.get("disable_corrector", ()) if k < 11}
    assert corrected == 11 - len(disabled)
    if not kw.get("clip_sample") and kw.get("timestep_spacing") != "leading":
        a_T, s_T = float(em.alpha[999]), float(em.sigma[999])
        exact = E.pf_ode_endpoint(x_T.double(), a_T, s_T, MU, STD)
        assert ((got.double() - exact).norm() / exact.norm()).item() < 0.2


class _IdentityAutoencoder:
    def decode_stage_2_outputs(self, z):
        return z


def test_every_inferer_samples_with_unipc(fake):
    """DiffusionInferer, LatentDiffusionInferer and the two ControlNet inferers drive the same trajectory (the
    ControlNet adds zero residuals, the autoencoder decodes to the latent itself)."""
    s = UniPCMultistepScheduler(clip_sample=False)
    s.set_timesteps(10)
    model = _analytic_model(s, "epsilon")
    x_T = torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(5))

    def controlnet(x, timesteps, controlnet_cond, context=None):
        return [torch.zeros_like(x)], torch.zeros_like(x)

    def unet(x, timesteps, context=None, down_block_additional_residuals=None, mid_block_additional_residual=None):
        return model(x, timesteps)
    cond = torch.zeros(1, 1, 8, 8)
    outs = [DiffusionInferer(s).sample(x_T, model, s, verbose=False),
            LatentDiffusionInferer(s).sample(x_T, _IdentityAutoencoder(), model, s, verbose=False),
            ControlNetDiffusionInferer(s).sample(x_T, unet, controlnet, cond, s, verbose=False),
            ControlNetLatentDiffusionInferer(s).sample(x_T, _IdentityAutoencoder(), unet, controlnet, cond, s,
                                                       verbose=False)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    acp = s.alphas_cumprod.double()
    exact = E.pf_ode_endpoint(x_T.double(), math.sqrt(float(acp[999])), math.sqrt(1 - float(acp[999])), MU, STD)
    assert ((outs[0].double() - exact).norm() / exact.norm()).item() < 0.05


# ------------------------------------------------------------------------------------------------ convergence
def _last_point_error(sched, n):
    """The emulator scheduler (float64) on the Gaussian model with x0 prediction: the relative error of the sample the
    network is evaluated on at the last timestep, against the probability-flow ODE's exact solution there."""
    sched.set_timesteps(n)
    em = (E.EmulatorScheduler if isinstance(sched, UniPCMultistepScheduler) else
          E.D.EmulatorScheduler)(sched)
    a, sg = em.alpha, em.sigma
    ts = em.grid
    x = torch.randn(4096, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    a0, s0 = float(a[ts[0]]), float(sg[ts[0]])
    xi = (x - a0 * MU) / math.sqrt(a0 * a0 * STD * STD + s0 * s0)
    for t in ts[:-1]:
        x, _ = em.step(E.gaussian_x0(x, float(a[t]), float(sg[t]), MU, STD), x)
    al, sl = float(a[ts[-1]]), float(sg[ts[-1]])
    exact = al * MU + math.sqrt(al * al * STD * STD + sl * sl) * xi
    return ((x - exact).norm() / exact.norm()).item()


def _slopes(cls, kw, ns):
    errs = [_last_point_error(cls(prediction_type="sample", clip_sample=False, lower_order_final=False, **kw), n)
            for n in ns]
    return errs, [math.log(errs[k] / errs[k + 1]) / math.log(ns[k + 1] / ns[k]) for k in range(len(ns) - 1)]


def test_convergence_order_on_the_logsnr_grid():
    """Measured at 20 -> 40 -> 80 steps of the 1000-step linear_beta schedule's log-SNR grid: UniPC-1 2.0, 2.0;
    UniPC-2 bh2 2.94, 2.83 (bh1 3.21, 2.95); DPM-Solver++ 2M 1.96, 2.03.  Past about 80 steps the integer timesteps
    near t = 0 stop shrinking the last intervals and every slope falls."""
    ns = (20, 40, 80)
    _, p1 = _slopes(UniPCMultistepScheduler, dict(solver_order=1), ns)
    e2, p2 = _slopes(UniPCMultistepScheduler, dict(), ns)
    _, p2b = _slopes(UniPCMultistepScheduler, dict(solver_type="bh1"), ns)
    ed, pd = _slopes(DPMSolverMultistepScheduler, dict(), ns)
    print(f"log-SNR grid slopes 20-40-80: UniPC-1 {p1}, UniPC-2 bh2 {p2}, bh1 {p2b}, DPM-Solver++ 2M {pd}")
    assert all(1.8 <= p <= 2.3 for p in p1), p1
    assert all(2.6 <= p <= 3.4 for p in p2 + p2b), (p2, p2b)
    assert all(1.8 <= p <= 2.3 for p in pd), pd
    assert e2[-1] < ed[-1] / 4, (e2, ed)


def test_convergence_order_on_the_leading_grid():
    """Measured at 50 -> 100 -> 200 steps of the leading grid (uniform in t, so the last intervals shrink slowly in
    lambda, which is singular at t = 0): UniPC-1 1.60, 1.68; UniPC-2 bh2 2.17, 2.31; UniPC-3 2.49, 2.82;
    DPM-Solver++ 2M 1.95, 2.04.  Below p + 1, but each order still gains on the one below."""
    ns = (50, 100, 200)
    _, p1 = _slopes(UniPCMultistepScheduler, dict(solver_order=1, timestep_spacing="leading"), ns)
    e2, p2 = _slopes(UniPCMultistepScheduler, dict(timestep_spacing="leading"), ns)
    _, p3 = _slopes(UniPCMultistepScheduler, dict(solver_order=3, timestep_spacing="leading"), ns)
    ed, pd = _slopes(DPMSolverMultistepScheduler, dict(timestep_spacing="leading"), ns)
    print(f"leading grid slopes 50-100-200: UniPC-1 {p1}, UniPC-2 {p2}, UniPC-3 {p3}, DPM-Solver++ 2M {pd}")
    assert all(1.5 <= p <= 2.1 for p in p1), p1
    assert all(2.1 <= p <= 3.1 for p in p2), p2
    assert p3[-1] >= 2.7, p3
    assert e2[-1] < ed[-1], (e2, ed)


# ------------------------------------------------------------------------------------------------ state
def test_counter_history_and_corrector_state(fake):
    s = UniPCMultistepScheduler(clip_sample=False, solver_order=3)
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
        assert s.counter == i + 1 and len(s._hist) == min(i + 1, 3)
        assert s._hist[-1][0] is x0 and x0.data_ptr() != m.data_ptr()
        assert s._last is not None and s._last.data_ptr() not in (x.data_ptr(), m.data_ptr(), prev.data_ptr())
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
    assert s.counter == 0 and s._hist == [] and s._last is None
    s.step(m, ts[0], x)
    with pytest.raises(ValueError, match="changed shape"):
        s.step(m[:1], ts[1], x[:1])
    with pytest.raises(ValueError, match="changed shape"):
        s.step(m.reshape(3, 2, 4, 4), ts[1], x.reshape(3, 2, 4, 4))
    s.step(m, ts[1], x)


def test_disable_corrector_skips_the_next_steps_corrector(fake):
    """disable_corrector=[k] leaves the sample of step k + 1 uncorrected: that step's corrected sample is the sample it
    was given, and every other step after the first corrects."""
    s = UniPCMultistepScheduler(clip_sample=False, disable_corrector=[2])
    s.set_timesteps(6)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 1, 8, 8, generator=g)
    for i, t in enumerate(s.timesteps):
        x_in = x
        x, _ = s.step(torch.randn(1, 1, 8, 8, generator=g), t, x)
        assert torch.equal(s._last, x_in) == (i in (0, 3)), i


def test_model_output_buffer_reuse_does_not_alias_history(fake):
    """A graph-replayed network hands back one buffer every step: the history must hold x0 and the corrected sample,
    not that buffer or the caller's sample."""
    s = UniPCMultistepScheduler(clip_sample=False, prediction_type="sample", solver_order=3)
    s.set_timesteps(7)
    buf, xbuf = torch.empty(1, 1, 8, 8), torch.empty(1, 1, 8, 8)
    x_a = x_b = torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(1))
    vals = [torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(10 + i)) for i in range(7)]
    for t, v in zip(s.timesteps, vals):
        buf.copy_(v)
        xbuf.copy_(x_a)
        x_a, _ = s.step(buf, t, xbuf)
    s2 = UniPCMultistepScheduler(clip_sample=False, prediction_type="sample", solver_order=3)
    s2.set_timesteps(7)
    for t, v in zip(s2.timesteps, vals):
        x_b, _ = s2.step(v.clone(), t, x_b.clone())
    assert torch.equal(x_a, x_b)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_dtype_round_trip(fake, dtype):
    s = UniPCMultistepScheduler()
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
    assert "b200_unipc_step" in declared and declared == set(_lib.SAMPLER_SIGNATURES)
    assert "B200_UNIPC_MAX_HIST 3" in text and _lib.UNIPC_MAX_HIST == 3
    assert "b200_abi_sizeof(15) is sizeof(b200_unipc_coef)" in text
    lib = _lib.load()
    assert lib.b200_abi_sizeof(15) == C.sizeof(_lib.UniPCCoef) == 60
    assert callable(getattr(unipc_backend.UniPCFakeLib, "b200_unipc_step"))


def test_entry_point_rejects_bad_arguments():
    """Argument checks run on the host before any launch, so they hold without a GPU."""
    lib = _lib.load()
    c = _lib.UniPCCoef(alpha_s=1.0, sigma_s=0.5, prediction_type=0)
    none = (C.c_void_p * 1)()
    args = dict(m=8, s=8, last=None, hist=none, nh=0, c=C.byref(c), p=8, x0=8, xc=8, n=4)

    def call(**kw):
        a = dict(args, **kw)
        return lib.b200_unipc_step(a["m"], a["s"], a["last"], a["hist"], a["nh"], a["c"], a["p"], a["x0"], a["xc"],
                                   a["n"], None)
    for bad in (dict(m=None), dict(s=None), dict(p=None), dict(x0=None), dict(xc=None), dict(n=0), dict(nh=4),
                dict(nh=-1), dict(nh=1), dict(c=None)):
        assert call(**bad) == _lib.B200_EINVAL, bad
    c.prediction_type = 7
    assert call() == _lib.B200_EINVAL
