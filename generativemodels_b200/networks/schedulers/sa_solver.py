"""SASolverScheduler: SA-Solver (Xue et al. 2023, arXiv 2309.05019), the stochastic Adams multistep predictor-corrector
solver of the diffusion SDE, in its data-prediction (x0) form.  The amount of noise injected per step is tau, a
function of the timestep: tau = 0 is a deterministic Adams solver of the probability-flow ODE, and tau = 1 with order 1
is DPM-Solver++ SDE's first-order step.  A step costs one network evaluation: the corrector reuses the x0 estimate the
step forms anyway.

The grid, the target of each step and the predictor's order schedule are DPMSolverMultistepScheduler's (this class
derives from it, with ``solver_order = predictor_order``).

The host folds the corrector and the predictor into one weight per input stream in float64 (``sa_solver_weights``);
``step`` is then one fused kernel launch (b200_sa_solver_step, include/b200gen_samplers.h) that forms x0 from the model
output, clips it, corrects the sample and predicts the next one.

Notation as in dpm_solver.py: alpha = sqrt(alphas_cumprod), sigma = sqrt(1 - alphas_cumprod), lambda = log alpha -
log sigma.  With tau constant over an update from (x_s, lambda_s) to lambda_t, h = lambda_t - lambda_s and
c = 1 + tau^2, the exact solution that both the predictor and the corrector approximate is

    x_t = (sigma_t / sigma_s) e^(-tau^2 h) x_s + alpha_t c int_0^h e^(-c u) x0(lambda_t - u) du
          + sigma_t sqrt(1 - e^(-2 tau^2 h)) xi.

Each replaces x0(lambda) by the Lagrange polynomial through some of the x0 estimates; the integral of each basis
polynomial is taken in closed form from J_n(x) = int_0^1 v^n e^(-x v) dv, with u = h v.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from ... import _lib
from .scheduler import PRED_CODES, _f, _prep, _stream
from .dpm_solver import DPMSolverMultistepScheduler, DPMSolverPredictionType, DPMSolverTimestepSpacing
from .._holders import on_input_device


def default_tau(t: int) -> float:
    """tau = 1 (noise injected as in DPM-Solver++ SDE) for 200 <= t <= 800, else 0 (the ODE)."""
    return 1.0 if 200 <= t <= 800 else 0.0


def _exp_moments(x: float, n_max: int) -> list[float]:
    """J_n(x) = int_0^1 v^n e^(-x v) dv for n = 0..n_max, x >= 0, in float64.  Below x = 2 from the series
    e^-x sum_m x^m n! / (m + n + 1)!, whose terms are all positive; above, from n! / x^(n+1) (1 - e^-x sum_(j<=n)
    x^j / j!), whose cancellation is then at most a factor of e^2 / 2."""
    out = []
    for n in range(n_max + 1):
        if x < 2.0:
            term, total = 1.0 / (n + 1), 0.0
            for m in range(60):
                total += term
                term *= x / (m + n + 2)
            out.append(math.exp(-x) * total)
        else:
            partial, term = 0.0, 1.0
            for j in range(n + 1):
                partial += term
                term *= x / (j + 1)
            out.append(math.factorial(n) / x ** (n + 1) * (1.0 - math.exp(-x) * partial))
    return out


def _update(alpha_s: float, sigma_s: float, alpha_t: float, sigma_t: float, lam_s: float, nodes, tau: float
            ) -> tuple[float, list[float], float]:
    """One update from (x_s, lam_s) at (alpha_s, sigma_s) to (alpha_t, sigma_t) with tau held constant, as weights
    (c_x, w, c_z) in float64: x_t = c_x x_s + sum_k w[k] m_k + c_z xi, where m_k is the x0 estimate at lambda
    nodes[k] and x0(lambda) is the Lagrange polynomial through them."""
    w = [0.0] * len(nodes)
    if sigma_s == 0.0:                                   # a noise-free sample: x_t = alpha_t x0
        w[0] = alpha_t
        return 0.0, w, 0.0
    if sigma_t == 0.0:                                   # to sigma = 0: h is infinite, x_t = alpha_t x0
        if len(nodes) != 1:
            raise ValueError("an SA-Solver update to sigma = 0 must be order 1")
        w[0] = alpha_t
        return 0.0, w, 0.0
    h = (math.log(alpha_t) - math.log(sigma_t)) - lam_s
    lam_t = lam_s + h
    t2 = tau * tau
    c = 1.0 + t2
    c_x = (sigma_t / sigma_s) * math.exp(-t2 * h)
    c_z = sigma_t * math.sqrt(max(-math.expm1(-2.0 * t2 * h), 0.0))
    J = _exp_moments(c * h, len(nodes) - 1)
    v = [(lam_t - lam) / h for lam in nodes] if len(nodes) > 1 else []
    for k in range(len(nodes)):
        basis = np.array([1.0])                          # the k-th Lagrange basis polynomial in v, lowest power first
        for j in range(len(nodes)):
            if j != k:
                basis = np.polynomial.polynomial.polymul(basis, [-v[j], 1.0]) / (v[k] - v[j])
        w[k] = alpha_t * c * h * sum(a * J[n] for n, a in enumerate(basis))
    return c_x, w, c_z


def sa_solver_weights(alphas, sigmas, lambdas, alpha_t: float, sigma_t: float, order: int, corrector_order: int,
                      tau: float, tau_last: float = 0.0) -> tuple[float, list[float], float, float, list[float], float]:
    """(c_last, [v0, v1, v2], c_zlast, c_xc, [u0, u1, u2], c_z) of step i, in float64.  ``alphas``, ``sigmas`` and
    ``lambdas`` are those of the current timestep s_i first, then of the previous ones s_(i-1), s_(i-2), where the
    earlier x0 estimates m_(i-1), m_(i-2) were formed (as many as the orders need).

    Corrector of order q = ``corrector_order`` (0: none): step i - 1 again, from its start sample x^c_(i-1) at s_(i-1)
    to s_i with its tau (``tau_last``) and its noise xi_(i-1), through m_i, ..., m_(i-q+1):
    x^c = c_last x^c_(i-1) + v0 m_i + v1 m_(i-1) + v2 m_(i-2) + c_zlast xi_(i-1).  Predictor of order p = ``order``
    from (x^c, s_i) to (alpha_t, sigma_t) with ``tau``, through m_i, ..., m_(i-p+1):
    x_(i+1) = c_xc x^c + u0 m_i + u1 m_(i-1) + u2 m_(i-2) + c_z xi_i."""
    c_last, v, c_zlast = 0.0, [0.0] * 3, 0.0
    if corrector_order:
        c_last, w, c_zlast = _update(alphas[1], sigmas[1], alphas[0], sigmas[0], lambdas[1],
                                     lambdas[:corrector_order], tau_last)
        v[:corrector_order] = w
    c_xc, w, c_z = _update(alphas[0], sigmas[0], alpha_t, sigma_t, lambdas[0], lambdas[:order], tau)
    return c_last, v, c_zlast, c_xc, w + [0.0] * (3 - len(w)), c_z


class SASolverScheduler(DPMSolverMultistepScheduler):
    """SA-Solver multistep sampler (data prediction) with the interface of DPMSolverMultistepScheduler.

    Args:
        num_train_timesteps, schedule, prediction_type, clip_sample, clip_sample_min, clip_sample_max,
        set_alpha_to_one, timestep_spacing, steps_offset, lower_order_final, schedule_args: as in
            DPMSolverMultistepScheduler (same defaults, same grids, targets and order schedule).
        predictor_order: 1, 2 or 3, the number of x0 estimates the predictor interpolates (DPM-Solver's
            ``solver_order``: the same warm-up, ``lower_order_final`` and order-1 rules).
        corrector_order: 0, 1, 2 or 3, the number of x0 estimates the corrector interpolates, the new one included
            (0: no corrector).  Step i's corrector has order min(corrector_order, i + 1), 1 at a timestep with
            sigma = 0.
        tau_func: timestep -> tau >= 0, the noise injected over the step that starts at that timestep.  The default
            is 1 for 200 <= t <= 800 and 0 elsewhere.

    ``step`` forms the x0 estimate from the network output and the sample it is given, corrects that sample (from
    the second step on, and not across an interval of zero length) by re-integrating the previous step from its start
    sample with the noise it drew, then predicts the next sample from the corrected one, drawing fresh noise where
    tau > 0.  It keeps the two previous x0 estimates, the last start sample and the last noise, all kernel outputs or
    its own buffers; ``set_timesteps`` clears them.  The step order rules are DPMSolverMultistepScheduler's.
    """

    def __init__(self, num_train_timesteps: int = 1000, schedule: str = "linear_beta", predictor_order: int = 2,
                 corrector_order: int = 2, tau_func=None, prediction_type: str = DPMSolverPredictionType.EPSILON,
                 clip_sample: bool = True, clip_sample_min: int = -1, clip_sample_max: int = 1,
                 set_alpha_to_one: bool = True, timestep_spacing: str = DPMSolverTimestepSpacing.LOGSNR,
                 steps_offset: int = 0, lower_order_final: bool = True, **schedule_args) -> None:
        if predictor_order not in (1, 2, 3):
            raise ValueError(f"predictor_order must be 1, 2 or 3, got {predictor_order}")
        if corrector_order not in (0, 1, 2, 3):
            raise ValueError(f"corrector_order must be 0, 1, 2 or 3, got {corrector_order}")
        if tau_func is not None and not callable(tau_func):
            raise ValueError(f"tau_func must be a callable from the timestep to tau >= 0, got {tau_func!r}")
        super().__init__(num_train_timesteps, schedule, solver_order=predictor_order, prediction_type=prediction_type,
                         clip_sample=clip_sample, clip_sample_min=clip_sample_min, clip_sample_max=clip_sample_max,
                         set_alpha_to_one=set_alpha_to_one, timestep_spacing=timestep_spacing,
                         steps_offset=steps_offset, lower_order_final=lower_order_final, **schedule_args)
        self.predictor_order = predictor_order
        self.corrector_order = corrector_order
        self.tau_func = default_tau if tau_func is None else tau_func

    def set_timesteps(self, num_inference_steps: int, device: str | torch.device | None = None) -> None:
        """Sets the discrete timesteps of the chain and clears the solver's history."""
        super().set_timesteps(num_inference_steps, device)
        self._hist: list[tuple[torch.Tensor, int]] = []           # (x0 estimate, timestep it was formed at)
        self._last: torch.Tensor | None = None                      # the previous step's start (corrected) sample
        self._noise: torch.Tensor | None = None                     # the noise the previous step drew, if any
        self._tau = 0.0                                             # the previous step's tau

    def _tau_at(self, timestep: int) -> float:
        tau = float(self.tau_func(timestep))
        if not (math.isfinite(tau) and tau >= 0.0):
            raise ValueError(f"tau_func must return a finite tau >= 0, got {tau} at timestep {timestep}")
        return tau

    @on_input_device
    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor,
             generator: torch.Generator | None = None) -> tuple[torch.Tensor, torch.Tensor]:
        """One corrector-predictor step at ``timestep`` -> (prev_sample, pred_original_sample), the latter the x0
        estimate from ``sample`` as given (before the correction).  ``generator`` draws the noise of a step with
        tau > 0 (on the CPU, like DPMSolverMultistepScheduler's SDE form)."""
        timestep = int(timestep)
        i = self.counter
        if i == len(self._grid) and timestep == int(self._grid[0]):
            i, self._hist, self._last, self._noise = 0, [], None, None   # the previous trajectory is finished
        elif i >= len(self._grid) or timestep != int(self._grid[i]):
            want = (f"the trajectory is finished; the next one starts at {int(self._grid[0])}" if i >= len(self._grid)
                    else f"expected {int(self._grid[i])}")
            raise ValueError(f"SASolverScheduler.step: timestep {timestep} is out of order ({want}); the solver "
                             "keeps the previous steps' estimates, so steps must follow `timesteps` from the first "
                             "(call set_timesteps to start over)")
        tau = self._tau_at(timestep)
        order = self.orders[i]
        past = list(reversed(self._hist))                                   # newest first
        corrector_order = 0
        if self.corrector_order and i > 0 and self._lambda[past[0][1]] != self._lambda[timestep]:
            corrector_order = 1 if self._sigma[timestep] == 0.0 else min(self.corrector_order, i + 1)
        n_hist = max(order, corrector_order) - 1
        n_ts = max(n_hist, 1 if corrector_order else 0)                     # s_(i-1) is the corrector's start
        ts = [timestep] + [t for _, t in past[:n_ts]]
        alpha_t, sigma_t = self._targets[i]
        c_last, v, c_zlast, c_xc, u, c_z = sa_solver_weights(self._alpha[ts].tolist(), self._sigma[ts].tolist(),
                                                             self._lambda[ts].tolist(), alpha_t, sigma_t, order,
                                                             corrector_order, tau, self._tau)
        noise = None
        if c_z != 0.0:
            noise = torch.randn(model_output.shape, dtype=model_output.dtype, generator=generator).to(model_output.device)
        lib = _lib.require_device()
        m, s, nz = _prep(model_output, sample, noise)
        hist = [x for x, _ in past[:n_hist]]
        last = self._last if corrector_order else None
        last_noise = self._noise if corrector_order and c_zlast != 0.0 else None
        for h in hist + [t for t in (last, last_noise) if t is not None]:
            if h.shape != s.shape or h.device != s.device:
                raise ValueError("SASolverScheduler.step: the sample changed shape or device mid-trajectory "
                                 "(call set_timesteps to start over)")
        c = _lib.SASolverCoef()
        c.alpha_s, c.sigma_s = _f(self._alpha[timestep]), _f(self._sigma[timestep])
        c.c_last, c.c_zlast, c.c_xc, c.c_z = _f(c_last), _f(c_zlast), _f(c_xc), _f(c_z)
        for k in range(3):
            c.v[k], c.u[k] = _f(v[k]), _f(u[k])
        c.clip_min, c.clip_max = float(self.clip_sample_values[0]), float(self.clip_sample_values[1])
        c.prediction_type, c.clip = PRED_CODES[str(self.prediction_type)], int(bool(self.clip_sample))
        prev, x0, xc = torch.empty_like(s), torch.empty_like(s), torch.empty_like(s)
        ptrs = (C.c_void_p * max(n_hist, 1))(*[h.data_ptr() for h in hist])
        _lib.check(lib.b200_sa_solver_step(m.data_ptr(), s.data_ptr(), None if last is None else last.data_ptr(),
                                           None if last_noise is None else last_noise.data_ptr(), ptrs, n_hist,
                                           None if nz is None else nz.data_ptr(), C.byref(c), prev.data_ptr(),
                                           x0.data_ptr(), xc.data_ptr(), s.numel(), _stream()), "b200_sa_solver_step")
        self._hist = (self._hist + [(x0, timestep)])[-_lib.SA_SOLVER_MAX_HIST:]
        self._last, self._noise, self._tau = xc, nz, tau
        self.counter = i + 1
        if sample.dtype != torch.float32:
            prev, x0 = prev.to(sample.dtype), x0.to(sample.dtype)
        return prev, x0
