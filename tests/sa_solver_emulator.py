"""Float64 reading of SASolverScheduler.step and of its entry point b200_sa_solver_step (include/b200gen_samplers.h)
(CPU only; test infrastructure).

Two readings, both returning tests/elementwise_emulator.Result triples (prev_sample, pred_x0, corrected):

  abi_step      the entry point's contract on the fp32 coefficients it is handed: x0 per prediction type, clip; the
                corrected sample xc = c_last last + v0 x0 + sum v_k hist[k-1] + c_zlast last_noise (or the sample itself
                when there is no `last`); then c_xc xc + u0 x0 + sum u_k hist[k-1] + c_z noise.  The CPU stand-in of the
                library stores its `out`.
  solver_step   the solver from its formulas (Xue et al. 2023, arXiv 2309.05019, data prediction), unfolded: x0(lambda)
                is the Lagrange interpolant of the estimates, evaluated at the nodes of a 48-point Gauss-Legendre rule
                on [0, h], and the integral alpha_t c int_0^h e^(-c u) x0(lambda_t - u) du is that rule's sum; the
                sample and noise coefficients are (sigma_t / sigma_s) e^(-tau^2 h) and sigma_t sqrt(1 - e^(-2 tau^2 h)).
                It shares no code with the host's folding (sa_solver_weights, closed-form integrals of the monomials),
                so holding the kernel to it checks the folding and the kernel together.  The rule integrates e^(-c u)
                times a polynomial of degree <= 2 to float64 rounding for the c h of any grid step.

The bound of solver_step, with u = 2^-24 (the reasoning of tests/dpm_solver_emulator.py, applied twice):
  x0            as in tests/dpm_solver_emulator.py.
  corrected     E_c = A_0 e0 + (k_c + 2) u S_c, where S_c is the corrector with every coefficient taken in absolute value
                (|c_x| |last| + alpha_t c sum_g W_g e^(-c u_g) sum_k |l_k| |m_k| + |c_z| |last_noise|, l_k the Lagrange
                basis), A_0 the x0 estimate's share of it per unit, and k_c the number of its terms (last, x0, the
                earlier estimates, the noise): one product and k_c - 1 fmas round once each against partial sums <= S_c,
                and rounding the folded weights to fp32 costs u S_c more.  Without a corrector the kernel copies the
                sample: exact.
  prev          |c_xc| E_c + A_0 e0 + (k_p + 2) u S_p, with S_p the predictor in absolute value over |corrected|.
abi_step's bound is the same with the struct's fp32 values taken as exact: (number of terms + 1) u sum |terms|.

EmulatorScheduler restates the step rules (which steps correct, with which order, which tau, which noise) over a
SASolverScheduler's grid, with the targets and the predictor's order schedule of
tests/dpm_solver_emulator.EmulatorScheduler.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from tests import dpm_solver_emulator as D
from tests.dpm_solver_emulator import _x0, gaussian_x0  # noqa: F401  (gaussian_x0: for the tests)
from tests.elementwise_emulator import Result, U, copy, excess, f32  # noqa: F401  (excess: for the tests)

F64 = torch.float64
PRED_EPSILON, PRED_SAMPLE, PRED_V, PRED_CODES = D.PRED_EPSILON, D.PRED_SAMPLE, D.PRED_V, D.PRED_CODES
_GL_X, _GL_W = np.polynomial.legendre.leggauss(48)


def _res(exact, err):
    return Result(exact, f32(exact), err, "f32")


@dataclass
class Interval:
    """One SA-Solver update from (x_s, lambda_s) at (alpha_s, sigma_s) to (alpha_t, sigma_t) with a constant tau,
    through the x0 estimates at `lambdas` (newest first)."""
    alpha_s: float
    sigma_s: float
    alpha_t: float
    sigma_t: float
    lambdas: list
    tau: float


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


def coefficients(iv: Interval):
    """(c_x, c_z, [(lambda_g, K_g)]) of the update: x_t = c_x x_s + sum_g K_g x0(lambda_g) + c_z xi."""
    if iv.sigma_s == 0.0 or iv.sigma_t == 0.0:            # x_t = alpha_t x0 of the newest estimate, no noise
        return 0.0, 0.0, None
    lam_s = math.log(iv.alpha_s) - math.log(iv.sigma_s)
    lam_t = math.log(iv.alpha_t) - math.log(iv.sigma_t)
    h = lam_t - lam_s
    t2 = iv.tau * iv.tau
    c = 1.0 + t2
    c_x = iv.sigma_t / iv.sigma_s * math.exp(-t2 * h)
    c_z = iv.sigma_t * math.sqrt(1.0 - math.exp(-2.0 * t2 * h))
    us = 0.5 * h * (_GL_X + 1.0)
    ks = 0.5 * h * _GL_W * iv.alpha_t * c * np.exp(-c * us)
    return c_x, c_z, [(lam_t - u, k) for u, k in zip(us.tolist(), ks.tolist())]


def _basis(lambdas, k, lam):
    out = 1.0
    for j, lj in enumerate(lambdas):
        if j != k:
            out *= (lam - lj) / (lambdas[k] - lj)
    return out


def _apply(iv: Interval, x, ms, z, absolute: bool):
    """c_x x + sum_g K_g P(lambda_g) + c_z z with P the Lagrange interpolant of the estimates `ms` (newest first, one
    per iv.lambdas) or, with `absolute`, every coefficient and basis value in absolute value over the inputs given."""
    A = abs if absolute else (lambda v: v)
    c_x, c_z, rule = coefficients(iv)
    if rule is None:
        return A(iv.alpha_t) * ms[0]
    out = A(c_x) * x
    for k, m in enumerate(ms):                            # the rule's sum of K_g P(lambda_g), taken per estimate
        out = out + sum(kg * A(_basis(iv.lambdas, k, lam)) for lam, kg in rule) * m
    if z is not None and c_z != 0.0:
        out = out + A(c_z) * z
    return out


def draws_noise(iv: Interval) -> bool:
    return coefficients(iv)[1] != 0.0


def solver_step(m, s, last, last_noise, hist, noise, p: Step):
    """(prev_sample, pred_x0, corrected) Results of one step from the formulas.  m, s and the tensors are flat; hist
    holds the previous x0 estimates, newest first, as many as the orders need; `last` and `last_noise` (the previous
    step's start sample and noise, None when it drew none) are only read by the corrector, `noise` only when the
    predictor injects noise."""
    m, s = m.to(F64), s.to(F64)
    hist = [h.to(F64) for h in hist]
    x0, e0 = _x0(m, s, p.pred, p.alpha_s, p.sigma_s, p.clip, p.clip_min, p.clip_max, True)
    zero = torch.zeros_like(s)
    cor = p.corrector
    if cor is None:
        rc = copy(s)
    else:
        q = len(cor.lambdas)
        ms = [x0] + hist[:q - 1]
        zl = last_noise.to(F64) if draws_noise(cor) else None
        last = last.to(F64)
        xc = _apply(cor, last, ms, zl, False)
        scale = _apply(cor, last.abs(), [t.abs() for t in ms], None if zl is None else zl.abs(), True)
        k = 1 + q + (zl is not None)
        err = _apply(cor, zero, [e0] + [zero] * (q - 1), None, True) + (k + 2) * U * scale
        rc = _res(xc, err)
    pr = p.predictor
    o = len(pr.lambdas)
    ms = [x0] + hist[:o - 1]
    z = noise.to(F64) if draws_noise(pr) else None
    prev = _apply(pr, rc.exact, ms, z, False)
    scale = _apply(pr, rc.exact.abs(), [t.abs() for t in ms], None if z is None else z.abs(), True)
    carried = _apply(pr, rc.err, [e0] + [zero] * (o - 1), None, True)
    k = 1 + o + (z is not None)
    return _res(prev, carried + (k + 2) * U * scale), _res(x0, e0), rc


def abi_step(m, s, last, last_noise, hist, noise, c, n):
    """(prev_sample, pred_x0, corrected) Results of b200_sa_solver_step on the fp32 coefficients of the struct `c`."""
    m, s = m[:n].to(F64), s[:n].to(F64)
    hist = [h[:n].to(F64) for h in hist]
    x0, e0 = _x0(m, s, c.prediction_type, c.alpha_s, c.sigma_s, bool(c.clip), c.clip_min, c.clip_max, False)
    if last is None:
        rc = copy(s)
    else:
        terms = [c.c_last * last[:n].to(F64), c.v[0] * x0] + [c.v[k + 1] * h for k, h in enumerate(hist)]
        if last_noise is not None:
            terms.append(c.c_zlast * last_noise[:n].to(F64))
        rc = _res(sum(terms), abs(c.v[0]) * e0 + (len(terms) + 1) * U * sum(t.abs() for t in terms))
    terms = [c.c_xc * rc.exact, c.u[0] * x0] + [c.u[k + 1] * h for k, h in enumerate(hist)]
    if noise is not None:
        terms.append(c.c_z * noise[:n].to(F64))
    err = abs(c.c_xc) * rc.err + abs(c.u[0]) * e0 + (len(terms) + 1) * U * sum(t.abs() for t in terms)
    return _res(sum(terms), err), _res(x0, e0), rc


class EmulatorScheduler(D.EmulatorScheduler):
    """SASolverScheduler.step in float64 over the grid and alphas_cumprod of `sched` (after set_timesteps): the
    targets and predictor orders of DPM-Solver's emulator scheduler, the corrector, tau and noise rules restated from
    SA-Solver's definition.  step() takes and returns float64 tensors; `noise` is the step's xi (read only when the
    step injects noise)."""

    def __init__(self, sched):
        super().__init__(sched)
        self.corrector_order, self.tau_func = sched.corrector_order, sched.tau_func
        self.last, self.last_noise, self.tau = None, None, 0.0

    def lam(self, t):
        return math.inf if float(self.sigma[t]) == 0.0 else super().lam(t)

    def plan(self, i) -> Step:
        t = self.grid[i]
        o = self.order(i)
        past = list(reversed(self.hist))                           # (x0, timestep), newest first
        a_s, s_s = float(self.alpha[t]), float(self.sigma[t])
        cor = None
        if self.corrector_order and i > 0 and self.lam(past[0][1]) != self.lam(t):
            q = 1 if s_s == 0.0 else min(self.corrector_order, i + 1)
            t0 = past[0][1]
            cor = Interval(float(self.alpha[t0]), float(self.sigma[t0]), a_s, s_s,
                           [self.lam(t)] + [self.lam(tk) for _, tk in past[:q - 1]], self.tau)
        a_t, s_t = self.targets[i]
        pr = Interval(a_s, s_s, a_t, s_t, [self.lam(t)] + [self.lam(tk) for _, tk in past[:o - 1]],
                      float(self.tau_func(t)))
        return Step(self.pred, a_s, s_s, pr, cor, self.clip, float(self.lo), float(self.hi))

    def step(self, m, x, noise=None):
        p = self.plan(self.i)
        hist = [h.reshape(-1) for h, _ in reversed(self.hist)]
        shape = x.shape
        flat = (lambda t: None if t is None else t.reshape(-1))          # noqa: E731
        rp, rx, rc = solver_step(m.reshape(-1), x.reshape(-1), flat(self.last), flat(self.last_noise), hist,
                                 flat(noise), p)
        self.hist = (self.hist + [(rx.exact.view(shape), self.grid[self.i])])[-2:]
        self.last = rc.exact.view(shape)
        self.last_noise = noise if draws_noise(p.predictor) else None
        self.tau = p.predictor.tau
        self.i += 1
        return rp.exact.view(shape), rx.exact.view(shape)


# ---------------------------------------------------------------------------------------------------------------------
# the Gaussian model, propagated exactly: data x0 ~ N(mu, std^2) per element.  Its x0-predictor is exact and affine, and
# every step is affine in the sample, the estimates and the noise, so each quantity is carried as a coefficient vector
# over (1, zeta, xi_0, xi_1, ...): zeta the starting draw, xi_i the noise of step i, all independent standard normals.
# Its mean is the first coefficient and its variance the squared norm of the others: no Monte Carlo.
# ---------------------------------------------------------------------------------------------------------------------
def gaussian_errors(sched, step, mu, std, weak: bool) -> float:
    """The relative error of the sample the network is evaluated on at the last timestep of `sched` (after
    set_timesteps; prediction_type "sample", no clip), run by step(model_output, timestep, sample, noise) -> next
    sample on float64 coefficient vectors.  weak: the start is the exact marginal at timesteps[0], and the error is the
    2-Wasserstein distance of the sample's law to the exact marginal N(alpha mu, alpha^2 std^2 + sigma^2) over that
    law's root mean square.  Otherwise (the ODE, tau = 0) the start is N(0, 1), and the error is the root-mean-square
    distance to the probability-flow ODE's solution from the same start, relative."""
    acp = sched.alphas_cumprod.to(F64)
    alpha, sigma = acp.sqrt(), (1.0 - acp).sqrt()
    ts = [int(t) for t in sched.timesteps.cpu()]
    K = 2 + len(ts)
    a0, s0 = float(alpha[ts[0]]), float(sigma[ts[0]])
    sd0 = math.sqrt(a0 * a0 * std * std + s0 * s0)
    x = torch.zeros(K, dtype=F64)
    if weak:
        x[0], x[1] = a0 * mu, sd0
    else:
        x[1] = 1.0
    for i, t in enumerate(ts[:-1]):
        a, s = float(alpha[t]), float(sigma[t])
        gain = a * std * std / (a * a * std * std + s * s)
        m = gain * x
        m[0] += mu - gain * a * mu
        z = torch.zeros(K, dtype=F64)
        z[2 + i] = 1.0
        x = step(m, t, x, z)
    a, s = float(alpha[ts[-1]]), float(sigma[ts[-1]])
    sd = math.sqrt(a * a * std * std + s * s)
    if weak:
        return math.hypot(float(x[0]) - a * mu, float(x[1:].norm()) - sd) / math.hypot(a * mu, sd)
    exact = torch.zeros(K, dtype=F64)
    exact[0], exact[1] = a * mu - sd * a0 * mu / sd0, sd / sd0
    return float((x - exact).norm() / exact.norm())


def emulator_gaussian_error(sched, n, mu, std, weak: bool) -> float:
    """gaussian_errors with the float64 emulator scheduler over `sched`'s grid at n steps."""
    sched.set_timesteps(n)
    em = EmulatorScheduler(sched)
    return gaussian_errors(sched, lambda m, t, x, z: em.step(m, x, z)[0], mu, std, weak)
