"""DPMSolverMultistepScheduler without a GPU: constructor, both grids, order schedule, history rules and dtypes through
the CPU stand-in of the C ABI (tests/samplers_backend.py), and the solver's formulas (tests/dpm_solver_emulator.py)
against the exact probability-flow ODE solution of a Gaussian model."""
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
from generativemodels_b200.inferers import DiffusionInferer
from generativemodels_b200.networks.schedulers import DDIMScheduler, DPMSolverMultistepScheduler
from generativemodels_b200.networks.schedulers.dpm_solver import dpm_solver_weights
from tests import dpm_solver_emulator as E
from tests import samplers_backend

ROOT = Path(__file__).resolve().parents[1]
MU, STD = 0.3, 0.5


@pytest.fixture
def fake(monkeypatch):
    return samplers_backend.install(monkeypatch)


# ------------------------------------------------------------------------------------------------ constructor
def test_defaults_follow_ddim():
    s = DPMSolverMultistepScheduler()
    d = DDIMScheduler()
    assert s.num_train_timesteps == 1000 and s.solver_order == 2 and s.algorithm_type == "dpmsolver++"
    assert s.prediction_type == "epsilon" and s.clip_sample is True and s.clip_sample_values == [-1, 1]
    assert s.timestep_spacing == "logsnr" and s.steps_offset == 0 and s.lower_order_final is True
    assert float(s.final_alpha_cumprod) == 1.0
    assert torch.equal(s.alphas_cumprod, d.alphas_cumprod) and torch.equal(s.betas, d.betas)
    assert len(s.timesteps) == 1000 and torch.equal(s.timesteps, torch.arange(999, -1, -1))
    s2 = DPMSolverMultistepScheduler(schedule="scaled_linear_beta", beta_start=0.0015, beta_end=0.0205,
                                     set_alpha_to_one=False)
    assert torch.equal(s2.alphas_cumprod, DDIMScheduler(schedule="scaled_linear_beta", beta_start=0.0015,
                                                        beta_end=0.0205).alphas_cumprod)
    assert torch.equal(s2.final_alpha_cumprod, s2.alphas_cumprod[0])


@pytest.mark.parametrize("kw,msg", [
    (dict(prediction_type="x0"), "prediction_type"),
    (dict(clip_sample_min=1, clip_sample_max=1), "clip_sample_min"),
    (dict(solver_order=0), "solver_order"),
    (dict(solver_order=4), "solver_order"),
    (dict(algorithm_type="dpmsolver"), "algorithm_type"),
    (dict(algorithm_type="sde-dpmsolver++", solver_order=3), "sde-dpmsolver"),
    (dict(timestep_spacing="linspace"), "timestep_spacing"),
])
def test_constructor_errors(kw, msg):
    with pytest.raises(ValueError, match=msg):
        DPMSolverMultistepScheduler(**kw)


def test_alias_and_exports():
    """Under the reference's import path, in a fresh interpreter (this process may hold the reference itself as
    ``generative`` for the oracle tests)."""
    code = ("import generative.networks.schedulers as G, generativemodels_b200.networks.schedulers as S; "
            "assert G.DPMSolverMultistepScheduler is S.DPMSolverMultistepScheduler")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    for algo, order in (("dpmsolver++", 3), ("sde-dpmsolver++", 2), ("sde-dpmsolver++", 1)):
        DPMSolverMultistepScheduler(algorithm_type=algo, solver_order=order)


# ------------------------------------------------------------------------------------------------ grids
@pytest.mark.parametrize("n,offset", [(1, 0), (7, 0), (50, 0), (50, 1), (333, 0), (1000, 0)])
def test_leading_grid_is_ddims(n, offset):
    s = DPMSolverMultistepScheduler(timestep_spacing="leading", steps_offset=offset)
    d = DDIMScheduler(steps_offset=offset)
    s.set_timesteps(n)
    d.set_timesteps(n)
    assert torch.equal(s.timesteps, d.timesteps)


def _lam(s):
    acp = s.alphas_cumprod.double()
    return 0.5 * (acp.log() - (1 - acp).log())


@pytest.mark.parametrize("schedule,kw", [("linear_beta", {}), ("scaled_linear_beta", dict(beta_start=0.0015,
                                                                                            beta_end=0.0205)),
                                         ("cosine", {}), ("sigmoid_beta", {})])
@pytest.mark.parametrize("n", [2, 3, 10, 15, 20, 25, 50, 200, 999])
def test_logsnr_grid(schedule, kw, n):
    s = DPMSolverMultistepScheduler(schedule=schedule, **kw)
    s.set_timesteps(n)
    t = s.timesteps.numpy()
    t0 = 1 if schedule == "cosine" else 0                 # the cosine schedule has alphas_cumprod[0] = 1
    assert float(s.alphas_cumprod[0]) == 1.0 or t0 == 0
    assert len(t) == n and t[0] == 999 and t[-1] == t0 and np.all(np.diff(t) < 0)
    lam = _lam(s).numpy()[t0:]
    targets = np.linspace(lam[-1], lam[0], n)
    # away from collisions every timestep is the integer nearest (in t) to its lambda target
    tc = np.interp(targets, lam[::-1], np.arange(999, t0 - 1, -1))
    free = np.abs(t - tc) <= 0.5 + 1e-9
    if n <= 25:
        assert free.all(), (t, tc)
    for i in np.flatnonzero(~free):                       # the others were moved by the collision rule
        assert t[i] in (t[i + 1] + 1, t0 + n - 1 - i, 999 - i), (i, t[i], tc[i])


def test_logsnr_collision_rule():
    """Where several lambda targets round to one integer, the clamp into the feasible band and the push from the t = 0
    end give a fixed, strictly decreasing grid."""
    s = DPMSolverMultistepScheduler(num_train_timesteps=20)
    s.set_timesteps(15)
    t = s.timesteps.numpy()
    lam = _lam(s).numpy()
    raw = np.rint(np.interp(np.linspace(lam[19], lam[0], 15), lam[::-1], np.arange(19, -1, -1.0))).astype(int)
    assert len(set(raw.tolist())) < 15                    # the case has collisions
    i = np.arange(15)
    want = np.clip(raw, 14 - i, 19 - i)
    for k in range(13, -1, -1):
        want[k] = max(want[k], want[k + 1] + 1)
    assert t.tolist() == want.tolist() and t[0] == 19 and t[-1] == 0 and np.all(np.diff(t) < 0)
    s.set_timesteps(20)
    assert s.timesteps.tolist() == list(range(19, -1, -1))


def test_grid_errors_and_offset():
    s = DPMSolverMultistepScheduler()
    for n in (0, 1):
        with pytest.raises(ValueError):
            s.set_timesteps(n)
    with pytest.raises(ValueError, match="cannot be larger"):
        s.set_timesteps(1001)
    with pytest.raises(ValueError, match="strictly decreasing"):
        DPMSolverMultistepScheduler(num_train_timesteps=1000, beta_start=0.0, beta_end=0.0)
    for bad in (-1, 999, 1000):
        with pytest.raises(ValueError, match="steps_offset"):
            DPMSolverMultistepScheduler(steps_offset=bad)


@pytest.mark.parametrize("offset", [1, 3, 100])
def test_logsnr_grid_with_steps_offset(offset):
    """On the log-SNR grid steps_offset is the last timestep evaluated: the grid runs from T - 1 down to it, evenly in
    lambda over that range, and never past T - 1."""
    o = DPMSolverMultistepScheduler(steps_offset=offset)
    assert o.timesteps.tolist() == list(range(999, offset - 1, -1))           # the constructor's full grid
    o.set_timesteps(10)
    t = o.timesteps.numpy()
    assert t[0] == 999 and t[-1] == offset and np.all(np.diff(t) < 0)
    lam = _lam(o).numpy()[offset:]
    tc = np.interp(np.linspace(lam[-1], lam[0], 10), lam[::-1], np.arange(999, offset - 1, -1))
    assert np.all(np.abs(t - tc) <= 0.5 + 1e-9), (t, tc)
    o.set_timesteps(1000 - offset)
    with pytest.raises(ValueError, match="inference steps"):
        o.set_timesteps(1001 - offset)


def test_leading_grid_with_steps_offset_stays_in_range():
    s = DPMSolverMultistepScheduler(timestep_spacing="leading", steps_offset=1)
    assert s.timesteps.tolist() == list(range(999, 0, -1))
    s.set_timesteps(50)
    assert s.timesteps[0] == 981 and s.timesteps[-1] == 1
    with pytest.raises(ValueError, match="past the last trained timestep"):
        s.set_timesteps(1000)


# ------------------------------------------------------------------------------------------------ orders
@pytest.mark.parametrize("kw,n,want", [
    (dict(), 10, [1, 2, 2, 2, 2, 2, 2, 2, 2, 1]),
    (dict(solver_order=3), 10, [1, 2, 3, 3, 3, 3, 3, 3, 2, 1]),
    (dict(solver_order=3), 3, [1, 2, 1]),
    (dict(solver_order=3, lower_order_final=False), 5, [1, 2, 3, 3, 1]),        # last target sigma = 0
    (dict(solver_order=3), 16, [1, 2] + [3] * 13 + [1]),
    (dict(solver_order=1), 10, [1] * 10),
    (dict(algorithm_type="sde-dpmsolver++"), 6, [1, 2, 2, 2, 2, 1]),
    (dict(set_alpha_to_one=False, lower_order_final=False), 5, [1, 2, 2, 2, 1]),  # last step has h = 0
    (dict(timestep_spacing="leading", set_alpha_to_one=False, steps_offset=1, lower_order_final=False), 5,
     [1, 2, 2, 2, 2]),
    (dict(timestep_spacing="leading", set_alpha_to_one=False, steps_offset=1), 5, [1, 2, 2, 2, 1]),
])
def test_order_schedule(kw, n, want):
    s = DPMSolverMultistepScheduler(**kw)
    s.set_timesteps(n)
    assert s.orders == want


# ------------------------------------------------------------------------------------------------ folding
@pytest.mark.parametrize("order,sde", [(1, False), (2, False), (3, False), (1, True), (2, True)])
@pytest.mark.parametrize("pred", [E.PRED_EPSILON, E.PRED_SAMPLE, E.PRED_V])
def test_folded_weights_match_the_formulas(order, sde, pred):
    """The host's fp32-rounded weights through the entry point's reading agree with the unfolded formulas within the
    solver reading's bound (what the GPU test holds the kernel to)."""
    g = torch.Generator().manual_seed(order * 7 + pred)
    s = DPMSolverMultistepScheduler()
    lam = _lam(s)
    t_s, t_t, t_1, t_2 = 400, 300, 500, 650
    a, sg = s.alphas_cumprod.double().sqrt(), (1 - s.alphas_cumprod.double()).sqrt()
    p = E.Step(pred, float(a[t_s]), float(sg[t_s]), float(a[t_t]), float(sg[t_t]),
               [float(lam[t_s]), float(lam[t_1]), float(lam[t_2])][:order], order, sde, clip=True)
    n = 4099
    m, x, h0, h1, z = (torch.randn(n, generator=g) for _ in range(5))
    hist = [h0, h1][:order - 1]
    c_x, w, c_z = dpm_solver_weights(p.alpha_s, p.sigma_s, p.alpha_t, p.sigma_t, p.lambdas, order, sde)
    c = _lib.DpmCoef(alpha_s=p.alpha_s, sigma_s=p.sigma_s, c_x=c_x, c_z=c_z, clip_min=-1, clip_max=1,
                     prediction_type=pred, clip=1)
    for k in range(3):
        c.w[k] = w[k]
    got_p, got_x = E.abi_step(m, x, hist, z if sde else None, c, n)
    want_p, want_x = E.solver_step(m, x, hist, z if sde else None, p)
    assert E.excess(want_p, got_p.out).max() <= 1.0
    assert E.excess(want_x, got_x.out).max() <= 1.0


def test_bound_rejects_a_wrong_weight():
    """A folding that drops the 2M correction's history term is far outside the bound."""
    s = DPMSolverMultistepScheduler()
    lam = _lam(s)
    a, sg = s.alphas_cumprod.double().sqrt(), (1 - s.alphas_cumprod.double()).sqrt()
    p = E.Step(E.PRED_SAMPLE, float(a[400]), float(sg[400]), float(a[300]), float(sg[300]),
               [float(lam[400]), float(lam[500])], 2)
    m, x, h0 = (torch.randn(64, generator=torch.Generator().manual_seed(i)) for i in range(3))
    c_x, w, _ = dpm_solver_weights(p.alpha_s, p.sigma_s, p.alpha_t, p.sigma_t, p.lambdas, 2, False)
    c = _lib.DpmCoef(alpha_s=p.alpha_s, sigma_s=p.sigma_s, c_x=c_x, prediction_type=E.PRED_SAMPLE)
    c.w[0], c.w[1] = w[0] + w[1], 0.0
    bad, _ = E.abi_step(m, x, [h0], None, c, 64)
    want, _ = E.solver_step(m, x, [h0], None, p)
    assert E.excess(want, bad.out).max() > 100


# ------------------------------------------------------------------------------------------------ the Gaussian model
def _vp(lam):
    """alpha, sigma of the continuous variance-preserving schedule at log-SNR/2 = lam."""
    return math.sqrt(1.0 / (1.0 + math.exp(-2 * lam))), math.sqrt(1.0 / (1.0 + math.exp(2 * lam)))


def _continuous_run(n, order, x_T, lam_lo=-5.0, lam_hi=9.0):
    """The emulator's formulas on a lambda-uniform grid of n evaluations from lam_lo to lam_hi, then to sigma = 0."""
    lams = np.linspace(lam_lo, lam_hi, n).tolist()
    x, hist = x_T.clone(), []
    for i, lam_s in enumerate(lams):
        a_s, s_s = _vp(lam_s)
        a_t, s_t = _vp(lams[i + 1]) if i + 1 < n else (1.0, 0.0)
        o = 1 if s_t == 0.0 else min(order, i + 1)
        m = E.gaussian_x0(x, a_s, s_s, MU, STD)
        p = E.Step(E.PRED_SAMPLE, a_s, s_s, a_t, s_t, [lam_s] + [lam for _, lam in reversed(hist)][:o - 1], o)
        rp, rx = E.solver_step(m, x, [h for h, _ in reversed(hist)][:o - 1], None, p)
        x = rp.exact
        hist = (hist + [(rx.exact, lam_s)])[-2:]
    return x


def test_formulas_reach_the_exact_endpoint_at_second_order():
    x_T = torch.randn(4096, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    a_T, s_T = _vp(-5.0)
    exact = E.pf_ode_endpoint(x_T, a_T, s_T, MU, STD)
    err = {}
    for order in (1, 2, 3):
        for n in (10, 20, 40, 80, 160):
            x = _continuous_run(n, order, x_T)
            err[order, n] = ((x - exact).norm() / exact.norm()).item()
    assert err[2, 40] / err[2, 80] >= 3.5, err
    assert err[2, 80] / err[2, 160] >= 3.5, err
    assert err[1, 40] / err[1, 80] < 2.5, err                   # first order
    # 3M: its order-1 and order-2 warm-up steps keep the global error at second order, with a smaller constant
    assert err[3, 40] / err[3, 80] >= 3.5 and err[3, 160] < err[2, 160] < 5e-4, err


def _analytic_model(sched, pred):
    acp = sched.alphas_cumprod.double()

    def model(x, timesteps, context=None):
        t = int(timesteps[0])
        a, s = math.sqrt(float(acp[t])), math.sqrt(1.0 - float(acp[t]))
        x0 = E.gaussian_x0(x.double(), a, s, MU, STD)
        eps = (x.double() - a * x0) / s
        out = {"epsilon": eps, "sample": x0, "v_prediction": a * eps - s * x0}[pred]
        return out.to(x.dtype)
    return model


PATHS = [
    dict(),
    dict(solver_order=1),
    dict(solver_order=3),
    dict(prediction_type="v_prediction"),
    dict(prediction_type="sample", solver_order=3, lower_order_final=False),
    dict(timestep_spacing="leading"),
    dict(timestep_spacing="leading", set_alpha_to_one=False, steps_offset=1),
    dict(steps_offset=1),
    dict(steps_offset=3, solver_order=3, set_alpha_to_one=False),
    dict(algorithm_type="sde-dpmsolver++"),
    dict(algorithm_type="sde-dpmsolver++", solver_order=1, prediction_type="v_prediction"),
    dict(clip_sample=True, clip_sample_min=-0.5, clip_sample_max=0.8),
]


@pytest.mark.parametrize("kw", PATHS, ids=[",".join(f"{k}={v}" for k, v in p.items()) or "default" for p in PATHS])
def test_scheduler_paths_through_the_inferer(fake, kw):
    """DiffusionInferer.sample with the analytic model through the stand-in: every step equals the emulator scheduler's
    step from the same inputs, within its bound, and the ODE reaches the exact endpoint about as well as the formulas
    do in float64."""
    kw = dict(dict(clip_sample=False), **kw)
    s = DPMSolverMultistepScheduler(**kw)
    s.set_timesteps(12)
    em = E.EmulatorScheduler(s)
    model = _analytic_model(s, kw.get("prediction_type", "epsilon"))
    sde = kw.get("algorithm_type") == "sde-dpmsolver++"
    x_T = torch.randn(1, 2, 16, 16, generator=torch.Generator().manual_seed(3))
    seen = []

    def spy(x, timesteps, context=None):
        out = model(x, timesteps, context)
        seen.append((x.clone(), out.clone()))
        return out
    g = torch.Generator().manual_seed(11)
    orig_step = s.step

    def step(m, t, x, generator=None):
        return orig_step(m, t, x, generator=g)
    s.step = step
    got = DiffusionInferer(s).sample(x_T, spy, s, verbose=False)
    assert len(seen) == 12 and s.counter == 12
    g2 = torch.Generator().manual_seed(11)
    for i, (x, m) in enumerate(seen):
        p = em.plan(i)
        z = None
        if sde and em.targets[i][1] > 0:
            z = torch.randn(m.shape, dtype=m.dtype, generator=g2)
        hist = [h for h, _ in reversed(em.hist)][:p.order - 1]
        want_p, want_x = E.solver_step(m.reshape(-1), x.reshape(-1), [h.reshape(-1) for h in hist],
                                       None if z is None else z.reshape(-1), p)
        nxt = seen[i + 1][0] if i + 1 < len(seen) else got
        assert E.excess(want_p, nxt.reshape(-1)).max() <= 1.0, i
        em.hist = (em.hist + [(want_x.out.view(x.shape), p.lambdas[0])])[-2:]
    if not sde and not kw.get("clip_sample"):
        a_T, s_T = float(em.alpha[999]), float(em.sigma[999])
        if kw.get("timestep_spacing") != "leading":
            exact = E.pf_ode_endpoint(x_T.double(), a_T, s_T, MU, STD)
            assert ((got.double() - exact).norm() / exact.norm()).item() < 0.2


def _gaussian_sample(fake_unused, n, order, spacing="logsnr"):
    s = DPMSolverMultistepScheduler(solver_order=order, clip_sample=False, timestep_spacing=spacing)
    s.set_timesteps(n)
    x_T = torch.randn(1, 1, 64, 64, generator=torch.Generator().manual_seed(0))
    got = DiffusionInferer(s).sample(x_T, _analytic_model(s, "epsilon"), s, verbose=False)
    acp = s.alphas_cumprod.double()
    exact = E.pf_ode_endpoint(x_T.double(), math.sqrt(float(acp[999])), math.sqrt(1 - float(acp[999])), MU, STD)
    return ((got.double() - exact).norm() / exact.norm()).item()


def test_second_order_beats_ddim_on_the_logsnr_grid(fake):
    e1, e2 = _gaussian_sample(fake, 10, 1), _gaussian_sample(fake, 10, 2)
    assert e1 / e2 >= 5.0, (e1, e2)
    assert _gaussian_sample(fake, 20, 2) < e2


# ------------------------------------------------------------------------------------------------ state
def test_counter_and_history(fake):
    s = DPMSolverMultistepScheduler(clip_sample=False)
    s.set_timesteps(5)
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
        x = prev
    with pytest.raises(ValueError, match="finished"):
        s.step(m, 0, x)
    kept = [o.clone() for o in outs]
    # once the trajectory is finished, a step at timesteps[0] starts the next one
    s.step(m, ts[0], x)
    assert s.counter == 1 and len(s._hist) == 1
    assert all(torch.equal(a, b) for a, b in zip(outs, kept))          # earlier returned x0 never overwritten
    # ... but not mid-trajectory: a repeated first step is an error, and so is an unfinished trajectory restarted
    with pytest.raises(ValueError, match="expected"):
        s.step(m, ts[0], x)
    s.step(m, ts[1], x)
    with pytest.raises(ValueError, match="expected"):
        s.step(m, ts[0], x)
    s.set_timesteps(5)
    assert s.counter == 0 and s._hist == []
    with pytest.raises(ValueError, match="out of order"):
        s.step(m, ts[2], x)
    s.step(m, ts[0], x)
    with pytest.raises(ValueError, match="changed shape"):
        s.step(m[:1], ts[1], x[:1])
    with pytest.raises(ValueError, match="changed shape"):                  # same number of elements, other shape
        s.step(m.reshape(3, 2, 4, 4), ts[1], x.reshape(3, 2, 4, 4))
    s.step(m, ts[1], x)


def test_model_output_buffer_reuse_does_not_alias_history(fake):
    """A graph-replayed network hands back one buffer every step: the history must hold x0, not that buffer."""
    s = DPMSolverMultistepScheduler(clip_sample=False, prediction_type="sample")
    s.set_timesteps(6)
    buf = torch.empty(1, 1, 8, 8)
    x_a = x_b = torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(1))
    vals = [torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(10 + i)) for i in range(6)]
    for t, v in zip(s.timesteps, vals):
        buf.copy_(v)
        x_a, _ = s.step(buf, t, x_a)
    s2 = DPMSolverMultistepScheduler(clip_sample=False, prediction_type="sample")
    s2.set_timesteps(6)
    for t, v in zip(s2.timesteps, vals):
        x_b, _ = s2.step(v.clone(), t, x_b)
    assert torch.equal(x_a, x_b)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_dtype_round_trip(fake, dtype):
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(4)
    x = torch.randn(1, 2, 8, 8).to(dtype)
    for t in s.timesteps:
        x, x0 = s.step(torch.randn(1, 2, 8, 8).to(dtype), t, x)
        assert x.dtype == dtype and x0.dtype == dtype and x.shape == (1, 2, 8, 8)
    assert s._hist[-1][0].dtype == torch.float32


def test_sde_noise_follows_the_generator(fake):
    outs = []
    for _ in range(2):
        s = DPMSolverMultistepScheduler(algorithm_type="sde-dpmsolver++", clip_sample=False)
        s.set_timesteps(4)
        x = torch.ones(1, 1, 4, 4)
        g = torch.Generator().manual_seed(5)
        for t in s.timesteps:
            x, _ = s.step(torch.zeros(1, 1, 4, 4), t, x, generator=g)
        outs.append(x)
    assert torch.equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------ ABI
def test_header_binding_and_struct():
    text = (ROOT / "include" / "b200gen_samplers.h").read_text()
    declared = set(re.findall(r"^int (b200_\w+)\(", text, re.M))
    assert declared == set(_lib.SAMPLER_SIGNATURES)
    others = (set(_lib.SIGNATURES) | set(_lib.METRIC_SIGNATURES) | set(_lib.FID_SIGNATURES)
              | set(_lib.PERCEPTUAL_SIGNATURES) | set(_lib.LOSS_SIGNATURES))
    assert not declared & others
    assert "B200_DPM_MAX_HIST 2" in text and _lib.DPM_MAX_HIST == 2
    lib = _lib.load()
    assert lib.b200_abi_sizeof(14) == C.sizeof(_lib.DpmCoef) == 44
    assert callable(getattr(samplers_backend.SamplersFakeLib, "b200_dpm_solver_step"))


def test_entry_point_rejects_bad_arguments():
    """Argument checks run on the host before any launch, so they hold without a GPU."""
    lib = _lib.load()
    c = _lib.DpmCoef(alpha_s=1.0, sigma_s=0.5, prediction_type=0)
    none = (C.c_void_p * 1)()
    args = dict(m=8, s=8, hist=none, nh=0, z=None, c=C.byref(c), p=8, x0=8, n=4)

    def call(**kw):
        a = dict(args, **kw)
        return lib.b200_dpm_solver_step(a["m"], a["s"], a["hist"], a["nh"], a["z"], a["c"], a["p"], a["x0"], a["n"],
                                        None)
    for bad in (dict(m=None), dict(s=None), dict(p=None), dict(x0=None), dict(n=0), dict(nh=3), dict(nh=-1),
                dict(nh=1), dict(c=None)):
        assert call(**bad) == _lib.B200_EINVAL, bad
    c.prediction_type = 7
    assert call() == _lib.B200_EINVAL
