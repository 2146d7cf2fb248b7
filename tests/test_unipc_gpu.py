"""UniPCMultistepScheduler on the GPU: b200_unipc_step against the float64 readings (tests/unipc_emulator.py), UniPC-2
bh2 with every corrector disabled against DPMSolverMultistepScheduler 2M, the Gaussian model's convergence, the golden
C1 / C2 networks and the brain-LDM bundle config against the CPU oracle driving the emulator scheduler, CUDA-graph
replay and repeat runs.  Runs in whichever storage flavour the library was loaded in (B200_ACT_DTYPE)."""
import ctypes as C
import json
import math
from pathlib import Path

import pytest
import torch

from generativemodels_b200 import _lib
from generativemodels_b200.networks.schedulers.unipc import unipc_weights
from oracle import torch_oracle as O
from tests import golden
from tests import unipc_emulator as E
from tests.golden import configs as G

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"
MU, STD = 0.3, 0.5
TRAJ_TOL, TRAJ_MAX = 5e-2, 1e-1      # multi-step network trajectories, as tests/test_dpm_solver_gpu.py
ALL_STEPS = tuple(range(1000))


def _sched(**kw):
    from generativemodels_b200.networks.schedulers import UniPCMultistepScheduler
    return UniPCMultistepScheduler(**kw)


def _check_traj(got, want, what):
    got, want = got.detach().float().cpu(), want.detach().float().cpu()
    r = ((got - want).norm() / want.norm()).item()
    m = ((got - want).abs().max() / want.abs().max()).item()
    assert r < TRAJ_TOL and m < TRAJ_MAX, f"{what}: relative L2 {r:.3e}, max-abs {m:.3e}"
    return r


# ------------------------------------------------------------------------------------------------ the kernel
def _plan(pred, clip, n_hist, last, bh="bh2"):
    """A step at t = 400 predicting to 330, earlier estimates at 470, 560, 650; predictor order min(n_hist, 2) + 1 and,
    with `last`, a corrector of order n_hist.  -> (emulator Step, folded weights)."""
    s = _sched()
    acp = s.alphas_cumprod.double()
    a, sg = acp.sqrt(), (1 - acp).sqrt()
    lam = (a.log() - sg.log())
    ts, tgt = [400, 470, 560, 650], 330
    p, q = min(n_hist, 2) + 1, (n_hist if last else 0)
    f = lambda v: [float(v[t]) for t in ts]         # noqa: E731
    folded = unipc_weights(f(a), f(sg), f(lam), float(a[tgt]), float(sg[tgt]), p, q, bh)
    pr = E.Interval(f(a)[0], f(sg)[0], float(a[tgt]), float(sg[tgt]), f(lam)[:p], p, bh)
    cor = E.Interval(f(a)[1], f(sg)[1], f(a)[0], f(sg)[0], f(lam)[1:q + 1], q, bh) if q else None
    return E.Step(pred, f(a)[0], f(sg)[0], pr, cor, clip, -1.0, 1.0), folded


def _coef(p, folded):
    c_last, v, c_xc, u = folded
    c = _lib.UniPCCoef(alpha_s=p.alpha_s, sigma_s=p.sigma_s, c_last=c_last, c_xc=c_xc, clip_min=p.clip_min,
                       clip_max=p.clip_max, prediction_type=p.pred, clip=int(p.clip))
    for k in range(4):
        c.v[k] = v[k]
    for k in range(3):
        c.u[k] = u[k]
    return c


def _launch(c, m, s, last, hist, prev, x0, xc):
    lib = _lib.require_device()
    ptrs = (C.c_void_p * 3)(*[h.data_ptr() for h in hist])
    _lib.check(lib.b200_unipc_step(m.data_ptr(), s.data_ptr(), None if last is None else last.data_ptr(), ptrs,
                                   len(hist), C.byref(c), prev.data_ptr(), x0.data_ptr(), xc.data_ptr(), m.numel(),
                                   torch.cuda.current_stream().cuda_stream), "b200_unipc_step")


def _run_kernel(p, folded, n_hist, last, n, offset, seed):
    """Inputs of n elements at element `offset` of their buffers (offset 1: no 16-byte alignment); outputs likewise,
    with a NaN sentinel around them."""
    g = torch.Generator().manual_seed(seed)
    host = [1.5 * torch.randn(n, generator=g) for _ in range(6)]
    dev = []
    for h in host:
        buf = torch.full((n + offset + 3,), float("nan"), device="cuda")
        buf[offset:offset + n] = h.cuda()
        dev.append(buf[offset:offset + n])
    m, s, l_, h0, h1, h2 = dev
    outs = [torch.full((n + offset + 3,), float("nan"), device="cuda") for _ in range(3)]
    prev, x0, xc = (o[offset:offset + n] for o in outs)
    c = _coef(p, folded)
    _launch(c, m, s, l_ if last else None, [h0, h1, h2][:n_hist], prev, x0, xc)
    torch.cuda.synchronize()
    for o in outs:
        assert torch.isnan(o[:offset]).all() and torch.isnan(o[offset + n:]).all(), "write outside the outputs"
    return host, c, prev.cpu(), x0.cpu(), xc.cpu()


CASES = [(pred, clip, nh, last) for pred in (E.PRED_EPSILON, E.PRED_SAMPLE, E.PRED_V) for clip in (False, True)
         for nh, last in ((0, False), (1, False), (2, False), (1, True), (2, True), (3, True))]


@pytest.mark.parametrize("pred,clip,n_hist,last", CASES)
def test_kernel_matches_the_solver(cuda_device, pred, clip, n_hist, last):
    worst = 0.0
    for bh in ("bh1", "bh2"):
        p, folded = _plan(pred, clip, n_hist, last, bh)
        for n in (1, 7, 8, 4099):
            for offset in (0, 1):
                (m, s, l_, h0, h1, h2), c, prev, x0, xc = _run_kernel(p, folded, n_hist, last, n, offset, n + offset)
                hist = [h0, h1, h2][:n_hist]
                want = E.solver_step(m, s, l_, hist, p)
                abi = E.abi_step(m, s, l_ if last else None, hist, c, n)
                for w, a, got in zip(want, abi, (prev, x0, xc)):
                    ex = E.excess(w, got).max().item()
                    assert ex <= 1.0 and E.excess(a, got).max() <= 1.0, (bh, n, offset, ex)
                    worst = max(worst, ex)
                if not last:
                    assert torch.equal(xc, s), "without a corrector the corrected sample is the sample"
    print(f"unipc_step pred={pred} clip={clip} n_hist={n_hist} last={last}: largest err/bound {worst:.3f}")


def test_kernel_at_the_c3_volume(cuda_device):
    n = 160 * 224 * 160
    p, folded = _plan(E.PRED_EPSILON, True, 3, True)
    (m, s, l_, h0, h1, h2), _, prev, x0, xc = _run_kernel(p, folded, 3, True, n, 0, 3)
    for w, got in zip(E.solver_step(m, s, l_, [h0, h1, h2], p), (prev, x0, xc)):
        assert E.excess(w, got).max() <= 1.0


def test_kernel_repeats_bit_identical(cuda_device):
    p, folded = _plan(E.PRED_V, True, 3, True)
    a = _run_kernel(p, folded, 3, True, 4099, 0, 9)
    b = _run_kernel(p, folded, 3, True, 4099, 0, 9)
    assert all(torch.equal(x, y) for x, y in zip(a[2:], b[2:]))


# ------------------------------------------------------------------------------------------------ correctors off = 2M
def test_correctors_off_is_dpm_solver_2m(cuda_device):
    """UniPC-2 bh2 with every corrector disabled against DPMSolverMultistepScheduler 2M over 50 steps, from the same
    inputs at each step: where the two hosts' fp32 weights are equal the kernels' samples are bit-identical (one
    product and the same fmas in the same order); elsewhere the weights differ by an fp32 rounding, so the samples
    differ by at most 12 u times the terms' magnitudes."""
    from generativemodels_b200.networks.schedulers import DPMSolverMultistepScheduler
    from generativemodels_b200.networks.schedulers.dpm_solver import dpm_solver_weights
    u = _sched(disable_corrector=ALL_STEPS, clip_sample=False)
    d = DPMSolverMultistepScheduler(clip_sample=False)
    u.set_timesteps(50)
    d.set_timesteps(50)
    assert torch.equal(u.timesteps, d.timesteps) and u.orders == d.orders
    acp = d.alphas_cumprod.double()
    a, sg = acp.sqrt(), (1 - acp).sqrt()
    lam = a.log() - sg.log()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 3, 16, 16, generator=g).cuda()
    ts, equal_w, same = u.timesteps.tolist(), 0, 0
    for i, t in enumerate(ts):
        m = torch.randn(2, 3, 16, 16, generator=g).cuda()
        got, got_x0 = u.step(m, t, x)
        want, want_x0 = d.step(m, t, x)
        assert torch.equal(got_x0, want_x0), i
        o, (a_t, s_t) = d.orders[i], d._targets[i]
        hist_t = ts[max(i - o + 1, 0):i][::-1]
        lams = [float(lam[k]) for k in [t] + hist_t]
        _, _, c_xc, uw = unipc_weights([float(a[k]) for k in [t] + hist_t], [float(sg[k]) for k in [t] + hist_t],
                                       lams, a_t, s_t, o, 0, "bh2")
        c_x, w, _ = dpm_solver_weights(float(a[t]), float(sg[t]), a_t, s_t, lams, o, False)
        f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))       # noqa: E731
        if f32(c_xc) == f32(c_x) and all(f32(p) == f32(q) for p, q in zip(uw, w)):
            equal_w += 1
            assert torch.equal(got, want), i
        hist = [h for h, _ in reversed(d._hist)][1:o]
        terms = abs(c_x) * x.abs() + abs(w[0]) * want_x0.abs() + sum(abs(w[k + 1]) * h.abs() for k, h in enumerate(hist))
        assert ((got - want).abs() <= 12 * 2.0 ** -24 * terms).all(), i
        same += bool(torch.equal(got, want))
        x = want
    print(f"correctors off vs 2M, 50 steps: fp32 weights equal at {equal_w}, samples bit-identical at {same}")
    assert equal_w >= 25, equal_w


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


def test_gaussian_model_convergence(cuda_device):
    """DiffusionInferer.sample on the GPU with the exact x0-predictor of a Gaussian, log-SNR grid, lower_order_final
    off: the sample the network sees at the last timestep tracks the float64 emulator scheduler, and its error against
    the probability-flow ODE's exact solution there falls at third order for UniPC-2 (second for UniPC-1)."""
    from generativemodels_b200.inferers import DiffusionInferer
    x_T = torch.randn(1, 4, 64, 64, generator=torch.Generator().manual_seed(0))
    err = {}
    for kw in (dict(solver_order=1), dict(), dict(solver_type="bh1")):
        for n in (20, 40, 80):
            s = _sched(clip_sample=False, lower_order_final=False, prediction_type="sample", **kw)
            s.set_timesteps(n)
            model, seen = _gaussian_model(s, "sample"), []

            def spy(x, timesteps, context=None):
                seen.append(x.double().cpu())
                return model(x, timesteps, context)
            DiffusionInferer(s).sample(x_T.cuda(), spy, s, verbose=False)
            em = E.EmulatorScheduler(s)
            x = x_T.double()
            for t in s.timesteps[:-1]:
                x, _ = em.step(model(x, torch.tensor([int(t)])).double(), x)
            assert ((seen[-1] - x).norm() / x.norm()).item() < 1e-5
            acp = s.alphas_cumprod.double()
            t0, tl = int(s.timesteps[0]), int(s.timesteps[-1])
            a0, s0, al, sl = (math.sqrt(float(acp[t0])), math.sqrt(1 - float(acp[t0])), math.sqrt(float(acp[tl])),
                              math.sqrt(1 - float(acp[tl])))
            xi = (x_T.double() - a0 * MU) / math.sqrt(a0 * a0 * STD * STD + s0 * s0)
            exact = al * MU + math.sqrt(al * al * STD * STD + sl * sl) * xi
            err[str(kw), n] = ((seen[-1] - exact).norm() / exact.norm()).item()
    slopes = {k: [math.log2(err[k, n] / err[k, 2 * n]) for n in (20, 40)] for k in {k for k, _ in err}}
    print("Gaussian model, log-SNR grid, error at the last evaluated timestep:",
          {f"{k} {n}": f"{e:.3e}" for (k, n), e in err.items()}, "slopes", slopes)
    assert all(1.8 <= p <= 2.3 for p in slopes[str(dict(solver_order=1))])
    assert all(2.6 <= p <= 3.4 for p in slopes[str(dict())] + slopes[str(dict(solver_type="bh1"))])


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
    s = _sched(clip_sample=False)             # no clip, for the reason tests/test_dpm_solver_gpu.py gives
    s.set_timesteps(5)
    noise = torch.randn(*G.C1_SHAPE, generator=torch.Generator().manual_seed(1))
    cfg = G.unet_oracle_cfg(G.C1_UNET)
    with torch.no_grad():
        want = O.diffusion_sample(lambda x, t, c: O.unet_forward(sd, cfg, x, t, context=c), _EmulatorDriver(s), noise)
    got = DiffusionInferer(s).sample(noise.cuda(), m.cuda(), s, verbose=False)
    print(f"C1 UniPC 5 steps vs oracle: rel L2 {_check_traj(got, want, 'C1 sample'):.3e}")


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
    print(f"C2 latent UniPC 5 steps vs oracle: rel L2 {_check_traj(got, want, 'C2 sample'):.3e}")


def _small_unet():
    from generativemodels_b200.networks.nets import DiffusionModelUNet
    torch.manual_seed(0)
    return G.randomize_zero_params(DiffusionModelUNet(**G.UNET_CASES["unet2d_attn"])).cuda().eval()


@pytest.mark.parametrize("kw", [dict(), dict(solver_order=3, solver_type="bh1")])
def test_graph_replay_and_repeats_bit_identical(cuda_device, monkeypatch, kw):
    """The auto-graph path (>= 8 steps) reuses the network's output buffer; the history holds the kernel's own x0 and
    corrected sample, so replayed and eager sampling agree bit for bit, and so do repeated runs of one scheduler."""
    import generativemodels_b200.inferers.inferer as I
    from generativemodels_b200.inferers import DiffusionInferer
    m = _small_unet()
    x = torch.randn(2, 1, 16, 16, generator=torch.Generator().manual_seed(1)).cuda()
    s = _sched(**kw)
    s.set_timesteps(10)
    outs = {}
    for graph in (False, True, True):
        monkeypatch.setattr(I, "AUTO_CUDA_GRAPH", graph)
        outs.setdefault(graph, []).append(DiffusionInferer(s).sample(x, m, s, verbose=False))
    assert "_b200_auto_graph" in m.__dict__
    assert torch.equal(outs[False][0], outs[True][0]), "graph-replayed sampling differs from eager"
    assert torch.equal(outs[True][0], outs[True][1]), "repeated sampling differs"
    assert torch.isfinite(outs[True][0]).all()


def test_brain_ldm_bundle_config_with_the_scheduler_swapped(cuda_device):
    """The bundle's unmodified inference.json with the scheduler's _target_ swapped, resolved at the fixture's reduced
    widths, against the oracle networks driving the emulator scheduler."""
    from generativemodels_b200.bundle import BundleConfig
    from generativemodels_b200.networks.schedulers import UniPCMultistepScheduler
    fx = golden.load("g_bundle_brain_ldm")
    over = {"load_autoencoder": "$@autoencoder_def.load_state_dict(@states['aekl_state'])",
            "load_diffusion": "$@diffusion_def.load_state_dict(@states['unet_state'])",
            "noise": "$@states['noise'].to(@device)", "states": "$None",
            "scheduler#_target_": "generative.networks.schedulers.UniPCMultistepScheduler",
            "set_timesteps": "$@scheduler.set_timesteps(num_inference_steps=10)"}
    for item, kw in (("autoencoder_def", G.BUNDLE_AEKL), ("diffusion_def", G.BUNDLE_UNET)):
        for k, v in kw.items():
            over[f"{item}#{k}"] = list(v) if isinstance(v, tuple) else v
    cfg = BundleConfig(str(GOLD / "brain_ldm_inference.json"), json.loads(json.dumps(over)))
    cfg._resolved["states"] = fx
    got = cfg.get("sample")
    s = cfg.get("scheduler")
    assert isinstance(s, UniPCMultistepScheduler) and len(s.timesteps) == 10 and not s.clip_sample
    ucfg, acfg = G.unet_oracle_cfg(fx["unet_kwargs"]), G.aekl_oracle_cfg(fx["aekl_kwargs"])
    ref = _sched(**G.BUNDLE_SCHEDULER)
    ref.set_timesteps(10)
    with torch.no_grad():
        want = O.bundle_sampling_fn(lambda x, t, c: O.unet_forward(fx["unet_state"], ucfg, x, t, context=c),
                                    lambda z: O.autoencoderkl_decode(fx["aekl_state"], acfg, z), _EmulatorDriver(ref),
                                    fx["noise"], fx["conditioning"])
    print(f"brain-LDM config, UniPC 10 steps vs oracle: rel L2 {_check_traj(got, want, 'bundle'):.3e}")
