"""Float64 reading of UniPCMultistepScheduler.step and of its entry point b200_unipc_step (include/b200gen_samplers.h)
(CPU only; test infrastructure).

Two readings, both returning tests/elementwise_emulator.Result triples (prev_sample, pred_x0, corrected):

  abi_step      the entry point's contract on the fp32 coefficients it is handed: x0 per prediction type, clip; the
                corrected sample xc = c_last last + v0 x0 + sum v_k hist[k-1] (or the sample itself when there is no
                `last`); then c_xc xc + u0 x0 + sum u_k hist[k-1].  The CPU stand-in of the library stores its `out`.
  solver_step   the solver from its formulas (Zhao et al. 2023, arXiv 2302.04867, data prediction), unfolded: phi1, B(h),
                the b_k recursion, the R rho = b solves and the D_k = (m_k - m0) / r_k differences, from the solver's
                float64 alpha, sigma and lambda.  It shares no code with the host's folding (unipc_weights), so holding
                the kernel to it checks the folding and the kernel together.

The bound of solver_step, with u = 2^-24 (the reasoning of tests/dpm_solver_emulator.py, applied twice):
  x0            as in tests/dpm_solver_emulator.py.
  corrected     E_c = |alpha_t B rho_q| e0 + (k_c + 2) u S_c, where S_c is the corrector with every coefficient and
                difference taken in absolute value and k_c = 2 + q the number of its terms (last, x0, q estimates): one
                product and k_c - 1 fmas round once each against partial sums <= S_c, and rounding the folded weights
                to fp32 costs u S_c more.  Without a corrector the kernel copies the sample: exact.
  prev          |c_xc| E_c + (the predictor's x0 coefficients in absolute value) e0 + (k_p + 2) u S_p, with S_p the
                predictor in absolute value over |corrected| and k_p = 1 + p.
abi_step's bound is the same with the struct's fp32 values taken as exact: (number of terms + 1) u sum |terms|.

EmulatorScheduler restates the step rules (which steps correct, with which order, from which history) over a
UniPCMultistepScheduler's grid, with the targets and the order schedule of tests/dpm_solver_emulator.EmulatorScheduler.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from tests import dpm_solver_emulator as D
from tests.dpm_solver_emulator import _x0, gaussian_x0, pf_ode_endpoint  # noqa: F401  (the last two: for the tests)
from tests.elementwise_emulator import Result, U, copy, excess, f32  # noqa: F401  (excess: for the tests)

F64 = torch.float64
PRED_EPSILON, PRED_SAMPLE, PRED_V, PRED_CODES = D.PRED_EPSILON, D.PRED_SAMPLE, D.PRED_V, D.PRED_CODES


def _res(exact, err):
    return Result(exact, f32(exact), err, "f32")


@dataclass
class Interval:
    """One UniPC update from (x, lambdas[0]) at (alpha_s0, sigma_s0) to (alpha_t, sigma_t).  lambdas: of the estimate
    m0 and of the older ones m1, m2, ... (newest first), `order` of them."""
    alpha_s0: float
    sigma_s0: float
    alpha_t: float
    sigma_t: float
    lambdas: list
    order: int
    solver_type: str = "bh2"


@dataclass
class Step:
    """One scheduler step: x0 from the network output, the corrector (None: skipped), the predictor."""
    pred: int
    alpha_s: float
    sigma_s: float
    predictor: Interval
    corrector: Interval | None = None
    clip: bool = False
    clip_min: float = -1.0
    clip_max: float = 1.0


def _terms(iv: Interval, corrector: bool):
    """(c_x, phi1, B, r, rho) of the update from the formulas.  rho weighs D_1..D_(p-1) (and, for the corrector, last
    of all m_t - m0)."""
    if iv.sigma_t == 0.0:                                  # h infinite: phi1 = B = -1; order 1
        assert iv.order == 1
        return 0.0, -1.0, -1.0, [], ([0.5] if corrector else [])
    lam_t = math.log(iv.alpha_t) - math.log(iv.sigma_t)
    h = lam_t - iv.lambdas[0]
    hh = -h
    phi1 = math.expm1(hh)
    B = hh if iv.solver_type == "bh1" else math.expm1(hh)
    c_x = iv.sigma_t / iv.sigma_s0
    p = iv.order
    if p == 1 and not corrector:
        return c_x, phi1, B, [], []
    r = [(iv.lambdas[k] - iv.lambdas[0]) / h for k in range(1, p)] + [1.0]
    g, fact, b = math.expm1(hh) / hh - 1.0, 1.0, []
    for k in range(1, p + 1):
        b.append(g * fact / B)
        fact *= k + 1
        g = g / hh - 1.0 / fact
    R = torch.tensor([[rk ** (k - 1) for rk in r] for k in range(1, p + 1)], dtype=F64)
    b = torch.tensor(b, dtype=F64)
    if corrector:
        rho = [0.5] if p == 1 else torch.linalg.solve(R, b).tolist()
    else:
        rho = [0.5] if p == 2 else torch.linalg.solve(R[:p - 1, :p - 1], b[:p - 1]).tolist()
    return c_x, phi1, B, r, rho


def _apply(iv: Interval, corrector: bool, x, m0, older, m_t, absolute: bool):
    """x_t = c_x x - alpha_t phi1 m0 - alpha_t B (sum_k rho_k D_k [+ rho_q (m_t - m0)]); `absolute` takes every
    coefficient and difference in absolute value (the magnitude the rounding acts on)."""
    A = abs if absolute else (lambda v: v)

    def sub(a, b):
        return a + b if absolute else a - b

    if iv.sigma_s0 == 0.0:                                 # a noise-free sample: x_t = alpha_t m0
        return A(iv.alpha_t) * m0
    c_x, phi1, B, r, rho = _terms(iv, corrector)
    res = torch.zeros_like(m0)
    for k in range(1, iv.order):
        res = res + A(rho[k - 1]) * (sub(older[k - 1], m0) / A(r[k - 1]))
    if corrector:
        res = res + A(rho[-1]) * sub(m_t, m0)
    return sub(sub(A(c_x) * x, A(iv.alpha_t * phi1) * m0), A(iv.alpha_t * B) * res)


def solver_step(m, s, last, hist, p: Step):
    """(prev_sample, pred_x0, corrected) Results of one step from the formulas.  m, s, last and the hist entries (the
    previous x0 estimates, newest first: as many as the corrector's order and the predictor's order - 1 need) are flat
    tensors; `last` (the previous corrected sample) is only read by the corrector."""
    m, s = m.to(F64), s.to(F64)
    hist = [h.to(F64) for h in hist]
    x0, e0 = _x0(m, s, p.pred, p.alpha_s, p.sigma_s, p.clip, p.clip_min, p.clip_max, True)
    zero = torch.zeros_like(s)
    cor = p.corrector
    if cor is None:
        rc = copy(s)
    else:
        q, last = cor.order, last.to(F64)
        xc = _apply(cor, True, last, hist[0], hist[1:q], x0, False)
        scale = _apply(cor, True, last.abs(), hist[0].abs(), [h.abs() for h in hist[1:q]], x0.abs(), True)
        err = _apply(cor, True, zero, zero, [zero] * (q - 1), e0, True) + (q + 4) * U * scale
        rc = _res(xc, err)
    pr, o = p.predictor, p.predictor.order
    older = hist[:o - 1]
    prev = _apply(pr, False, rc.exact, x0, older, None, False)
    scale = _apply(pr, False, rc.exact.abs(), x0.abs(), [h.abs() for h in older], None, True)
    carried = _apply(pr, False, rc.err, e0, [zero] * (o - 1), None, True)
    return _res(prev, carried + (o + 3) * U * scale), _res(x0, e0), rc


def abi_step(m, s, last, hist, c, n):
    """(prev_sample, pred_x0, corrected) Results of b200_unipc_step on the fp32 coefficients of the struct `c`."""
    m, s = m[:n].to(F64), s[:n].to(F64)
    hist = [h[:n].to(F64) for h in hist]
    x0, e0 = _x0(m, s, c.prediction_type, c.alpha_s, c.sigma_s, bool(c.clip), c.clip_min, c.clip_max, False)
    if last is None:
        rc = copy(s)
    else:
        terms = [c.c_last * last[:n].to(F64), c.v[0] * x0] + [c.v[k + 1] * h for k, h in enumerate(hist)]
        rc = _res(sum(terms), abs(c.v[0]) * e0 + (len(terms) + 1) * U * sum(t.abs() for t in terms))
    terms = [c.c_xc * rc.exact, c.u[0] * x0] + [c.u[k + 1] * h for k, h in enumerate(hist[:2])]
    err = abs(c.c_xc) * rc.err + abs(c.u[0]) * e0 + (len(terms) + 1) * U * sum(t.abs() for t in terms)
    return _res(sum(terms), err), _res(x0, e0), rc


class EmulatorScheduler(D.EmulatorScheduler):
    """UniPCMultistepScheduler.step in float64 over the grid and alphas_cumprod of `sched` (after set_timesteps): the
    targets and orders of DPM-Solver's emulator scheduler, the corrector rules restated from UniPC's definition.
    step() takes and returns float64 tensors."""

    def __init__(self, sched):
        super().__init__(sched)
        self.solver_type = str(sched.solver_type)
        self.disabled = set(sched.disable_corrector)
        self.last = None

    def lam(self, t):
        return math.inf if float(self.sigma[t]) == 0.0 else super().lam(t)

    def plan(self, i) -> Step:
        t = self.grid[i]
        o = self.order(i)
        past = list(reversed(self.hist))                           # (x0, timestep), newest first
        a_s, s_s = float(self.alpha[t]), float(self.sigma[t])
        cor = None
        if i > 0 and i - 1 not in self.disabled and self.lam(past[0][1]) != self.lam(t):
            q, t0 = self.order(i - 1), past[0][1]
            cor = Interval(float(self.alpha[t0]), float(self.sigma[t0]), a_s, s_s,
                           [self.lam(tk) for _, tk in past[:q]], q, self.solver_type)
        a_t, s_t = self.targets[i]
        pr = Interval(a_s, s_s, a_t, s_t, [self.lam(t)] + [self.lam(tk) for _, tk in past[:o - 1]], o,
                      self.solver_type)
        return Step(self.pred, a_s, s_s, pr, cor, self.clip, float(self.lo), float(self.hi))

    def step(self, m, x, noise=None):
        p = self.plan(self.i)
        hist = [h.reshape(-1) for h, _ in reversed(self.hist)]
        shape = x.shape
        rp, rx, rc = solver_step(m.reshape(-1), x.reshape(-1), None if self.last is None else self.last.reshape(-1),
                                 hist, p)
        self.hist = (self.hist + [(rx.exact.view(shape), self.grid[self.i])])[-3:]
        self.last = rc.exact.view(shape)
        self.i += 1
        return rp.exact.view(shape), rx.exact.view(shape)
