"""Float64 reading of DPMSolverMultistepScheduler.step and of its entry point b200_dpm_solver_step
(include/b200gen_samplers.h) (CPU only; test infrastructure).

Two readings, both returning tests/elementwise_emulator.Result pairs (prev_sample, pred_x0) with kind "f32":

  abi_step      the entry point's contract on the fp32 coefficients it is handed: x0 per prediction type, clip, then
                c_x s + w0 x0 + w1 hist[0] + w2 hist[1] + c_z z.  The CPU stand-in of the library stores its `out`.
  solver_step   the solver from its formulas (Lu et al. 2022, arXiv 2211.01095), unfolded: D1 = (m0 - m1) / r0 and,
                for order 3, D1_0, D1_1, D1 and D2 as written in the paper's multistep form, from the solver's float64
                alpha, sigma and lambda.  It shares no code with the host's folding (dpm_solver_weights), so holding
                the kernel to it checks the folding and the kernel together.

The bound of solver_step, with u = 2^-24:
  x0            epsilon: 3u (|s| + sigma_s |m|) / alpha_s + 2u |x0|;  v: 3u (alpha_s |s| + sigma_s |m|);  sample: 0
                (alpha_s and sigma_s are rounded to fp32 once; fma / product, sum and division one rounding each).
                The clip is 1-Lipschitz, so it does not grow the error.
  prev          E + (k + 2) u S.  S is the update with every coefficient and every difference taken in absolute value
                (|c_x s| + the x0 terms' magnitudes + |c_z z|): it bounds sum_i |w_i m_i| of any folding of the formula.
                k is the number of terms (sample, x0, history, noise): one product and k - 1 fmas round once each
                against partial sums <= S, and rounding the folded weights to fp32 costs u S more.  E is the x0 error
                carried through the same absolute-value formula.
abi_step's bound is the same with the struct's fp32 values taken as exact: |w0| e0 + (k + 1) u sum |terms|.

EmulatorScheduler restates the solver's step rules (targets, orders, history) over a DPMSolverMultistepScheduler's
grid and tables, in float64, for trajectories.  The grid itself is checked separately (tests/test_dpm_solver_cpu.py).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch

from tests.elementwise_emulator import Result, U, excess, f32  # noqa: F401  (excess: for the tests)

F64 = torch.float64
PRED_EPSILON, PRED_SAMPLE, PRED_V = 0, 1, 2
PRED_CODES = {"epsilon": PRED_EPSILON, "sample": PRED_SAMPLE, "v_prediction": PRED_V}


def _res(exact, err):
    return Result(exact, f32(exact), err, "f32")


@dataclass
class Step:
    """One solver step: prediction type and clip, the current (s) and target (t) alpha and sigma, the lambdas of the
    estimates m0, m1, m2 (newest first, as many as `order`), the order and the SDE form."""
    pred: int
    alpha_s: float
    sigma_s: float
    alpha_t: float
    sigma_t: float
    lambdas: list = field(default_factory=list)
    order: int = 1
    sde: bool = False
    clip: bool = False
    clip_min: float = -1.0
    clip_max: float = 1.0


def _x0(m, s, pred, alpha, sigma, clip, lo, hi, rounded_coefs):
    """x0 and its error; rounded_coefs adds the fp32 rounding of alpha and sigma."""
    k = 3 if rounded_coefs else 2
    if pred == PRED_EPSILON:
        x0 = (s - sigma * m) / alpha
        err = k * U * (s.abs() + abs(sigma) * m.abs()) / abs(alpha) + (k - 1) * U * x0.abs()
    elif pred == PRED_V:
        x0 = alpha * s - sigma * m
        err = k * U * (abs(alpha) * s.abs() + abs(sigma) * m.abs())
    else:
        x0, err = m.clone(), torch.zeros_like(m)
    if clip:
        x0 = x0.clamp(lo, hi)
    return x0, err


def _emh(p: Step):
    return (p.sigma_t / p.alpha_t) * (p.alpha_s / p.sigma_s)


def _x0_terms(p: Step, m0, m1, m2, absolute: bool):
    """The update's terms in the estimates, from the formulas; `absolute` takes every coefficient and difference in
    absolute value (the magnitude the rounding acts on)."""
    A = abs if absolute else (lambda v: v)

    def sub(a, b):
        return a + b if absolute else a - b

    emh = _emh(p)
    if p.order > 1:
        lam_t = math.log(p.alpha_t) - math.log(p.sigma_t)
        h = lam_t - p.lambdas[0]
        r0 = (p.lambdas[0] - p.lambdas[1]) / h
    if p.sde:
        q = p.alpha_t * (1.0 - emh * emh)
        out = A(q) * m0
        if p.order == 2:
            out = out + A(0.5 * q) * (sub(m0, m1) / A(r0))
        return out
    phi = p.alpha_t * (emh - 1.0)
    out = A(-phi) * m0
    if p.order == 2:
        d1 = sub(m0, m1) / A(r0)
        out = out + A(-0.5 * phi) * d1
    elif p.order == 3:
        r1 = (p.lambdas[1] - p.lambdas[2]) / h
        d1_0, d1_1 = sub(m0, m1) / A(r0), sub(m1, m2) / A(r1)
        d1 = d1_0 + A(r0 / (r0 + r1)) * sub(d1_0, d1_1)
        d2 = sub(d1_0, d1_1) / A(r0 + r1)
        c1 = p.alpha_t * ((emh - 1.0) / h + 1.0)
        c2 = p.alpha_t * ((emh - 1.0 + h) / (h * h) - 0.5)
        out = sub(out + A(c1) * d1, A(c2) * d2)
    return out


def _sample_and_noise_coefs(p: Step):
    emh = _emh(p)
    if p.sde:
        return (p.sigma_t / p.sigma_s) * emh, p.sigma_t * math.sqrt(max(1.0 - emh * emh, 0.0))
    return p.sigma_t / p.sigma_s, 0.0


def solver_step(m, s, hist, noise, p: Step):
    """(prev_sample, pred_x0) Results of one solver step from the formulas.  m, s, hist entries (m1, m2) and noise are
    flat tensors; hist needs p.order - 1 entries."""
    m, s = m.to(F64), s.to(F64)
    hist = [h.to(F64) for h in hist]
    x0, e0 = _x0(m, s, p.pred, p.alpha_s, p.sigma_s, p.clip, p.clip_min, p.clip_max, True)
    zero = torch.zeros_like(s)
    m1 = hist[0] if p.order > 1 else zero
    m2 = hist[1] if p.order > 2 else zero
    c_x, c_z = _sample_and_noise_coefs(p)
    z = noise.to(F64) if (noise is not None and c_z != 0.0) else zero
    prev = c_x * s + _x0_terms(p, x0, m1, m2, False) + c_z * z
    scale = abs(c_x) * s.abs() + _x0_terms(p, x0.abs(), m1.abs(), m2.abs(), True) + abs(c_z) * z.abs()
    k = 2 + (p.order - 1) + (1 if noise is not None and c_z != 0.0 else 0)
    err = _x0_terms(p, e0, zero, zero, True) + (k + 2) * U * scale
    return _res(prev, err), _res(x0, e0)


def abi_step(m, s, hist, noise, c, n):
    """(prev_sample, pred_x0) Results of b200_dpm_solver_step on the fp32 coefficients of the struct `c`."""
    m, s = m[:n].to(F64), s[:n].to(F64)
    x0, e0 = _x0(m, s, c.prediction_type, c.alpha_s, c.sigma_s, bool(c.clip), c.clip_min, c.clip_max, False)
    terms = [c.c_x * s, c.w[0] * x0] + [c.w[k + 1] * hist[k][:n].to(F64) for k in range(len(hist))]
    if noise is not None:
        terms.append(c.c_z * noise[:n].to(F64))
    prev = sum(terms)
    err = abs(c.w[0]) * e0 + (len(terms) + 1) * U * sum(t.abs() for t in terms)
    return _res(prev, err), _res(x0, e0)


class EmulatorScheduler:
    """DPMSolverMultistepScheduler.step in float64 over the grid and alphas_cumprod of `sched` (a
    DPMSolverMultistepScheduler after set_timesteps): targets, order rules and history restated from the solver's
    definition.  step() takes and returns float64 tensors; `noise` is the SDE form's z (ignored otherwise)."""

    def __init__(self, sched):
        acp = sched.alphas_cumprod.to(F64)
        self.alpha, self.sigma = acp.sqrt(), (1.0 - acp).sqrt()
        self.T = sched.num_train_timesteps
        self.grid = [int(t) for t in sched.timesteps.cpu()]
        n = len(self.grid)
        a_f = float(sched.final_alpha_cumprod)
        final = (math.sqrt(a_f), math.sqrt(1.0 - a_f))
        if sched.timestep_spacing == "logsnr":
            prevs = self.grid[1:] + [-1]
        else:
            prevs = [t - self.T // n for t in self.grid]
        self.targets = [(float(self.alpha[q]), float(self.sigma[q])) if q >= 0 else final for q in prevs]
        self.solver_order, self.lower_order_final = sched.solver_order, sched.lower_order_final
        self.sde = sched.algorithm_type == "sde-dpmsolver++"
        self.pred = PRED_CODES[str(sched.prediction_type)]
        self.clip, (self.lo, self.hi) = bool(sched.clip_sample), sched.clip_sample_values
        self.i, self.hist = 0, []

    def lam(self, t):
        return math.log(float(self.alpha[t])) - math.log(float(self.sigma[t]))

    def order(self, i):
        n = len(self.grid)
        o = min(self.solver_order, i + 1)
        if self.lower_order_final and n < 15:
            if i == n - 1:
                o = 1
            elif i == n - 2:
                o = min(o, 2)
        a_t, s_t = self.targets[i]
        t = self.grid[i]
        if s_t == 0.0 or (a_t == float(self.alpha[t]) and s_t == float(self.sigma[t])):
            o = 1
        return o

    def plan(self, i) -> Step:
        t = self.grid[i]
        o = self.order(i)
        lams = [self.lam(t)] + [lam for _, lam in reversed(self.hist)][:o - 1]
        a_t, s_t = self.targets[i]
        return Step(self.pred, float(self.alpha[t]), float(self.sigma[t]), a_t, s_t, lams, o, self.sde, self.clip,
                    float(self.lo), float(self.hi))

    def step(self, m, x, noise=None):
        p = self.plan(self.i)
        hist = [h for h, _ in reversed(self.hist)][:p.order - 1]
        shape = x.shape
        rp, rx = solver_step(m.reshape(-1), x.reshape(-1), [h.reshape(-1) for h in hist],
                             None if noise is None else noise.reshape(-1), p)
        self.hist = (self.hist + [(rx.exact.view(shape), p.lambdas[0])])[-2:]
        self.i += 1
        return rp.exact.view(shape), rx.exact.view(shape)


# ---------------------------------------------------------------------------------------------------------------------
# the Gaussian model: data x0 ~ N(mu, std^2) per element, whose probability-flow ODE is solved exactly
# ---------------------------------------------------------------------------------------------------------------------
def gaussian_x0(x, alpha, sigma, mu, std):
    """E[x0 | x_t = x] for x0 ~ N(mu, std^2): the exact x0-predictor."""
    return mu + alpha * std * std / (alpha * alpha * std * std + sigma * sigma) * (x - alpha * mu)


def gaussian_eps(x, alpha, sigma, mu, std):
    return (x - alpha * gaussian_x0(x, alpha, sigma, mu, std)) / sigma


def pf_ode_endpoint(x_T, alpha_T, sigma_T, mu, std):
    """The probability-flow ODE's solution at sigma = 0 from x_T at (alpha_T, sigma_T)."""
    return mu + std * (x_T - alpha_T * mu) / math.sqrt(alpha_T * alpha_T * std * std + sigma_T * sigma_T)
