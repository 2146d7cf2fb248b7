"""UniPCMultistepScheduler: UniPC (Zhao et al. 2023, arXiv 2302.04867), the unified predictor-corrector multistep solver
of the probability-flow ODE, in its data-prediction (x0) form with the B(h) = h (``"bh1"``) or e^h - 1 (``"bh2"``)
variants.  A step still costs one network evaluation: the corrector (UniC) reuses the x0 estimate the step forms
anyway, and raises the order of the predictor (UniP) by one.

The grid, the target of each step and the order schedule are DPMSolverMultistepScheduler's (this class derives from
it).  With every corrector disabled, UniPC-2 bh2 is DPM-Solver++ 2M.

The host folds the corrector and the predictor into weights in float64 (``unipc_weights``); ``step`` is then one fused
kernel launch (b200_unipc_step, include/b200gen_samplers.h) that forms x0 from the model output, clips it, corrects the
sample and predicts the next one.

Notation as in dpm_solver.py: alpha = sqrt(alphas_cumprod), sigma = sqrt(1 - alphas_cumprod), lambda = log alpha -
log sigma.  An update runs from (x, lambda_s0) to lambda_t with h = lambda_t - lambda_s0, hh = -h, phi1 = expm1(hh),
B = hh (bh1) or expm1(hh) (bh2); b_k = g_k k! / B with g_1 = phi1 / hh - 1, g_(k+1) = g_k / hh - 1 / (k+1)!; R has
rows r^(k-1) over r = (r_1, ..., r_(p-1), 1) with r_k = (lambda_(s_k) - lambda_s0) / h, and D_k = (m_k - m0) / r_k.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from ... import _lib
from .scheduler import PRED_CODES, StrEnum, _f, _prep, _stream
from .dpm_solver import DPMSolverMultistepScheduler, DPMSolverPredictionType, DPMSolverTimestepSpacing
from .._holders import on_input_device


class UniPCSolverType(StrEnum):
    BH1 = "bh1"
    BH2 = "bh2"


def _update(alpha_s0: float, sigma_s0: float, alpha_t: float, sigma_t: float, lambdas, order: int, solver_type: str,
            corrector: bool) -> tuple[float, list[float]]:
    """One UniPC update from (x, lambdas[0]) to (alpha_t, sigma_t) as weights (c_x, w), in float64:
    x_t = c_x x + sum_k w[k] m_k, where m_0 is the x0 estimate at lambdas[0] and m_k the k-th previous one (at
    lambdas[k], k < order).  The predictor (order p) has p weights; the corrector (order q) has q + 1, the last one for
    m_t, the x0 estimate at the target."""
    w = [0.0] * (order + 1 if corrector else order)
    if sigma_s0 == 0.0:                                  # a noise-free sample: x_t = alpha_t x0
        w[0] = alpha_t
        return 0.0, w
    if sigma_t == 0.0:                                   # to sigma = 0: h is infinite, phi1 = B = -1
        if order != 1:
            raise ValueError("a UniPC update to sigma = 0 must be order 1")
        w[0] = alpha_t
        if corrector:                                    # - alpha_t B rho (m_t - m0), rho = 1/2
            w[0], w[1] = 0.5 * alpha_t, 0.5 * alpha_t
        return 0.0, w
    h = (math.log(alpha_t) - math.log(sigma_t)) - lambdas[0]
    hh = -h
    phi1 = math.expm1(hh)
    c_x, w[0] = sigma_t / sigma_s0, -alpha_t * phi1
    n_rho = order if corrector else order - 1
    if n_rho == 0:
        return c_x, w
    B = hh if solver_type == UniPCSolverType.BH1 else phi1
    r = [(lambdas[k] - lambdas[0]) / h for k in range(1, order)] + [1.0]
    if n_rho == 1:
        rho = [0.5]
    else:
        b, g, fac = [], phi1 / hh - 1.0, 1.0
        for k in range(1, n_rho + 1):
            b.append(g * fac / B)
            fac *= k + 1
            g = g / hh - 1.0 / fac
        R = np.array([[rk ** i for rk in r[:n_rho]] for i in range(n_rho)])
        rho = np.linalg.solve(R, np.array(b)).tolist()
    for k in range(1, order):                            # - alpha_t B rho_k D_k
        c = -alpha_t * B * rho[k - 1] / r[k - 1]
        w[0], w[k] = w[0] - c, w[k] + c
    if corrector:                                        # - alpha_t B rho_q (m_t - m0)
        c = -alpha_t * B * rho[-1]
        w[0], w[-1] = w[0] - c, w[-1] + c
    return c_x, w


def unipc_weights(alphas, sigmas, lambdas, alpha_t: float, sigma_t: float, order: int, corrector_order: int,
                  solver_type: str) -> tuple[float, list[float], float, list[float]]:
    """(c_last, [v0, v1, v2, v3], c_xc, [u0, u1, u2]) of step i, in float64.  ``alphas``, ``sigmas`` and ``lambdas``
    are those of the current timestep s_i first, then of the previous ones s_(i-1), s_(i-2), ..., where the earlier x0
    estimates m_(i-1), m_(i-2), ... were formed (as many as the orders need).

    Corrector of order q = ``corrector_order`` (0: none), from the previous corrected sample at s_(i-1) to s_i:
    x^c = c_last x^c_(i-1) + v0 m_i + sum_(k=1..3) v_k m_(i-k).  Predictor of order p = ``order`` from (x^c, s_i) to
    (alpha_t, sigma_t): x_(i+1) = c_xc x^c + u0 m_i + sum_(k=1..2) u_k m_(i-k)."""
    c_last, v = 0.0, [0.0] * 4
    if corrector_order:
        c_last, w = _update(alphas[1], sigmas[1], alphas[0], sigmas[0], lambdas[1:], corrector_order, solver_type, True)
        v[0] = w[-1]
        v[1:corrector_order + 1] = w[:-1]
    c_xc, w = _update(alphas[0], sigmas[0], alpha_t, sigma_t, lambdas, order, solver_type, False)
    return c_last, v, c_xc, w + [0.0] * (3 - len(w))


class UniPCMultistepScheduler(DPMSolverMultistepScheduler):
    """UniPC multistep sampler (data prediction) with the interface of DPMSolverMultistepScheduler.

    Args:
        num_train_timesteps, schedule, prediction_type, clip_sample, clip_sample_min, clip_sample_max,
        set_alpha_to_one, timestep_spacing, steps_offset, lower_order_final, schedule_args: as in
            DPMSolverMultistepScheduler (same defaults, same grids, targets and order schedule).
        solver_order: 1, 2 or 3, the predictor's order; with the corrector the step's order is one higher.
        solver_type: ``"bh2"`` (B(h) = e^h - 1) or ``"bh1"`` (B(h) = h).
        disable_corrector: step indices; the corrector of step i is skipped when i - 1 is in the list.

    ``step`` forms the x0 estimate from the network output and the sample it is given, corrects that sample (from
    the second step on, unless disabled, and not across an interval of zero length), then predicts the next one from
    the corrected sample.  It keeps the x0 estimates of the three previous steps and the last corrected sample, all
    the kernel's own outputs; ``set_timesteps`` clears them.  The step order rules are DPMSolverMultistepScheduler's.
    """

    def __init__(self, num_train_timesteps: int = 1000, schedule: str = "linear_beta", solver_order: int = 2,
                 solver_type: str = UniPCSolverType.BH2, prediction_type: str = DPMSolverPredictionType.EPSILON,
                 clip_sample: bool = True, clip_sample_min: int = -1, clip_sample_max: int = 1,
                 set_alpha_to_one: bool = True, timestep_spacing: str = DPMSolverTimestepSpacing.LOGSNR,
                 steps_offset: int = 0, lower_order_final: bool = True, disable_corrector=(), **schedule_args) -> None:
        super().__init__(num_train_timesteps, schedule, solver_order=solver_order, prediction_type=prediction_type,
                         clip_sample=clip_sample, clip_sample_min=clip_sample_min, clip_sample_max=clip_sample_max,
                         set_alpha_to_one=set_alpha_to_one, timestep_spacing=timestep_spacing,
                         steps_offset=steps_offset, lower_order_final=lower_order_final, **schedule_args)
        if solver_type not in UniPCSolverType.__members__.values():
            raise ValueError("Argument `solver_type` must be a member of UniPCSolverType")
        self.solver_type = solver_type
        self.disable_corrector = [int(k) for k in disable_corrector]

    def set_timesteps(self, num_inference_steps: int, device: str | torch.device | None = None) -> None:
        """Sets the discrete timesteps of the chain and clears the solver's history."""
        super().set_timesteps(num_inference_steps, device)
        self._hist: list[tuple[torch.Tensor, int]] = []           # (x0 estimate, timestep it was formed at)
        self._last: torch.Tensor | None = None                      # the previous step's corrected sample

    @on_input_device
    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor,
             generator: torch.Generator | None = None) -> tuple[torch.Tensor, torch.Tensor]:
        """One corrector-predictor step at ``timestep`` -> (prev_sample, pred_original_sample), the latter the x0
        estimate from ``sample`` as given (before the correction).  ``generator`` is accepted for the common interface
        and unused."""
        timestep = int(timestep)
        i = self.counter
        if i == len(self._grid) and timestep == int(self._grid[0]):
            i, self._hist, self._last = 0, [], None      # the previous trajectory is finished: start the next one
        elif i >= len(self._grid) or timestep != int(self._grid[i]):
            want = (f"the trajectory is finished; the next one starts at {int(self._grid[0])}" if i >= len(self._grid)
                    else f"expected {int(self._grid[i])}")
            raise ValueError(f"UniPCMultistepScheduler.step: timestep {timestep} is out of order ({want}); the solver "
                             "keeps the previous steps' estimates, so steps must follow `timesteps` from the first "
                             "(call set_timesteps to start over)")
        order = self.orders[i]
        past = list(reversed(self._hist))                                   # newest first
        corrector_order = 0
        if i > 0 and i - 1 not in self.disable_corrector and self._lambda[past[0][1]] != self._lambda[timestep]:
            corrector_order = self.orders[i - 1]
        n_hist = max(order - 1, corrector_order)
        ts = [timestep] + [t for _, t in past[:n_hist]]
        alpha_t, sigma_t = self._targets[i]
        c_last, v, c_xc, u = unipc_weights(self._alpha[ts].tolist(), self._sigma[ts].tolist(),
                                           self._lambda[ts].tolist(), alpha_t, sigma_t, order, corrector_order,
                                           self.solver_type)
        lib = _lib.require_device()
        m, s = _prep(model_output, sample)
        hist = [x for x, _ in past[:n_hist]]
        last = self._last if corrector_order else None
        for h in hist + ([last] if last is not None else []):
            if h.shape != s.shape or h.device != s.device:
                raise ValueError("UniPCMultistepScheduler.step: the sample changed shape or device mid-trajectory "
                                 "(call set_timesteps to start over)")
        c = _lib.UniPCCoef()
        c.alpha_s, c.sigma_s = _f(self._alpha[timestep]), _f(self._sigma[timestep])
        c.c_last, c.c_xc = _f(c_last), _f(c_xc)
        for k in range(4):
            c.v[k] = _f(v[k])
        for k in range(3):
            c.u[k] = _f(u[k])
        c.clip_min, c.clip_max = float(self.clip_sample_values[0]), float(self.clip_sample_values[1])
        c.prediction_type, c.clip = PRED_CODES[str(self.prediction_type)], int(bool(self.clip_sample))
        prev, x0, xc = torch.empty_like(s), torch.empty_like(s), torch.empty_like(s)
        ptrs = (C.c_void_p * max(n_hist, 1))(*[h.data_ptr() for h in hist])
        _lib.check(lib.b200_unipc_step(m.data_ptr(), s.data_ptr(), None if last is None else last.data_ptr(), ptrs,
                                       n_hist, C.byref(c), prev.data_ptr(), x0.data_ptr(), xc.data_ptr(), s.numel(),
                                       _stream()), "b200_unipc_step")
        self._hist = (self._hist + [(x0, timestep)])[-_lib.UNIPC_MAX_HIST:]
        self._last = xc
        self.counter = i + 1
        if sample.dtype != torch.float32:
            prev, x0 = prev.to(sample.dtype), x0.to(sample.dtype)
        return prev, x0
