"""The shadow-call harness (tests/abi_shadow.py) on the metric, FID, perceptual and loss entry points, on host memory:
host tensors stand in for allocator segments and a mutated CPU stand-in plays the real library, as in
tests/test_abi_shadow_cpu.py.  The unmutated stand-in must pass one call of each entry point; each kernel-shaped mutant
must be rejected by the rule written for it, and the test prints by what factor (the worst err / tol of the call, inf
for a NaN or a value the reading does not have; a write outside the outputs has no factor)."""
import ctypes as C

import numpy as np
import pytest
import torch

from generativemodels_b200 import _lib, ops
from generativemodels_b200._lib import FidMomentsParams, FrechetParams, SsimCombineParams, SsimParams
from generativemodels_b200.metrics.ssim import separable_kernel
from tests import abi_shadow
from tests import losses_emulator as LE
from tests import perceptual_emulator as PE
from tests.test_abi_shadow_cpu import Buffers, _bytes

SLOTS = 3          # partial slots per item of the 'real' SSIM


def _f32(ptr, n):
    return np.ctypeslib.as_array(C.cast(int(ptr), C.POINTER(C.c_float)), shape=(int(n),))


def _f64(ptr, n):
    return np.ctypeslib.as_array(C.cast(int(ptr), C.POINTER(C.c_double)), shape=(int(n),))


class Real(abi_shadow.StandIn):
    """The stand-in as a 'real' library: SLOTS partial slots per SSIM item, scratch it leaves alone, and the mutations
    that change how b200_ssim / b200_ssim_combine / b200_perceptual_prep compute (`mutate`, a name)."""
    mutate = None

    def b200_ssim_workspace_bytes(self, p):
        return _obj(p).N * 16 * SLOTS

    def b200_mmd_workspace_bytes(self, shape):
        return 64

    def b200_frechet_workspace_bytes(self, F):
        return 64

    def b200_ssim(self, p, stream):
        q = SsimParams.from_buffer_copy(_obj(p))
        if self.mutate == "ssim_scale_twice":
            q.scale = q.scale * q.scale
        if self.mutate == "ssim_swapped_hw_taps":
            q.taps_h, q.taps_w, q.kh, q.kw = q.taps_w, q.taps_h, q.kw, q.kh
        super().b200_ssim(C.byref(q), stream)
        part = _f64(q.partials, q.N * SLOTS * 2).reshape(q.N, SLOTS, 2)
        count = q.C * (q.D - q.kd + 1) * (q.H - q.kh + 1) * (q.W - q.kw + 1)
        for k, ptr in enumerate((q.ssim_map, q.cs_map)):
            if ptr:                             # a kernel sums the fp32 values it stores
                part[:, 0, k] = _f32(ptr, q.N * count).reshape(q.N, count).astype(np.float64).sum(1)
        part[:, 1] = part[:, 0] * 0.25          # spread each item's sums over the slots (exact in fp64)
        part[:, 2] = part[:, 0] * 0.25
        part[:, 0] *= 0.5
        if self.mutate == "ssim_dropped_slot":
            part[:, 1] = 0.0
        return 0

    def b200_ssim_combine(self, p, stream):
        super().b200_ssim_combine(p, stream)
        if self.mutate == "combine_last_scale_cs":
            q = _obj(p)
            S, N_ = q.n_scales, q.N
            cs = torch.from_numpy(_f32(q.cs_mean, S * N_).copy()).view(S, N_)
            w = torch.tensor(list(q.weights[:S]), dtype=torch.float64).view(-1, 1)
            _f32(q.ms_ssim, N_)[:] = torch.prod(cs.double().clamp_min(0) ** w, 0).float().numpy()
        return 0

    def b200_perceptual_prep(self, *args):
        if self.mutate != "prep_mean_std_swapped":
            return super().b200_perceptual_prep(*args)
        mean, std = PE.MEAN32, PE.STD32
        PE.MEAN32, PE.STD32 = std, mean
        try:
            return super().b200_perceptual_prep(*args)
        finally:
            PE.MEAN32, PE.STD32 = mean, std


class After:
    """`real` with fn(args) applied to the memory after each call of `entry` (a kernel that stored something else)."""

    def __init__(self, real, entry, fn):
        self.real, self.entry, self.fn = real, entry, fn

    def __getattr__(self, name):
        f = getattr(self.real, name)
        if name != self.entry:
            return f

        def call(*args):
            rc = f(*args)
            self.fn(args)
            return rc
        return call


def _obj(a):
    return a._obj if hasattr(a, "_obj") else a


def run(monkeypatch, bufs, name, args, real=None):
    real = real if real is not None else Real()
    with abi_shadow.shadow(monkeypatch, memory=bufs.memory(), real=real) as sh:
        rc = getattr(_lib.require_device(), name)(*args)
    assert rc == 0
    return sh


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------------
# one call of each entry point, on host buffers
# ------------------------------------------------------------------------------------------------------------------
def ssim_call(kernel="uniform", maps=True):
    """b200_ssim on 2 items of 1 x 20 x 20 (D = 1): a 5 x 5 uniform kernel, or the anisotropic Gaussian (3, 9)."""
    bufs = Buffers()
    g = _gen(1)
    shape = (2, 1, 1, 20, 20)
    a = torch.rand(shape, generator=g)
    x, y = bufs(a), bufs((a + 0.2 * torch.randn(shape, generator=g)).clamp(0, 1))
    if kernel == "uniform":
        taps, scale = separable_kernel(2, "uniform", 5, 1.5)
    else:
        taps, scale = separable_kernel(2, "gaussian", (3, 9), (0.8, 2.0))
    p = SsimParams()
    p.x, p.y, p.x_dtype, p.y_dtype = x.data_ptr(), y.data_ptr(), _lib.DT_F32, _lib.DT_F32
    p.x_strides[:], p.y_strides[:] = x.stride(), y.stride()
    p.N, p.C, p.D, p.H, p.W = shape
    p.kd, p.kh, p.kw = (len(t) for t in taps)
    for dst, t in zip((p.taps_d, p.taps_h, p.taps_w), taps):
        dst[:len(t)] = list(t)
    p.scale, p.c1, p.c2 = scale, 1e-4, 9e-4
    out = (shape[0], 1, 1, 20 - p.kh + 1, 20 - p.kw + 1)
    sm, cm = (bufs(torch.full(out, float("nan"))) for _ in range(2)) if maps else (None, None)
    part = bufs(torch.zeros(shape[0] * SLOTS * 2, dtype=torch.float64))
    p.ssim_map, p.cs_map = (sm.data_ptr(), cm.data_ptr()) if maps else (None, None)
    p.partials = part.data_ptr()
    return bufs, (C.byref(p), None), p


def combine_call():
    """b200_ssim_combine over two scales of SSIM partials the 'real' b200_ssim left (SLOTS slots per item)."""
    bufs = Buffers()
    parts, counts = [], []
    for k, seed in ((5, 2), (3, 3)):
        g = _gen(seed)
        shape = (2, 1, 1, 16, 16)
        a = torch.rand(shape, generator=g)
        x, y = bufs(a), bufs((a + 0.3 * torch.randn(shape, generator=g)).clamp(0, 1) * 0.7)
        taps, scale = separable_kernel(2, "gaussian", k, 1.5)
        p = SsimParams()
        p.x, p.y, p.x_dtype, p.y_dtype = x.data_ptr(), y.data_ptr(), _lib.DT_F32, _lib.DT_F32
        p.x_strides[:], p.y_strides[:] = x.stride(), y.stride()
        p.N, p.C, p.D, p.H, p.W = shape
        p.kd, p.kh, p.kw = (len(t) for t in taps)
        for dst, t in zip((p.taps_d, p.taps_h, p.taps_w), taps):
            dst[:len(t)] = list(t)
        p.scale, p.c1, p.c2 = scale, 1e-4, 9e-4
        part = bufs(torch.zeros(2 * SLOTS * 2, dtype=torch.float64))
        p.partials = part.data_ptr()
        assert Real().b200_ssim(C.byref(p), None) == 0
        parts.append(part)
        counts.append((16 - k + 1) ** 2)
    q = SsimCombineParams()
    for i, (part, n) in enumerate(zip(parts, counts)):
        q.partials[i], q.slots[i], q.count[i], q.weights[i] = part.data_ptr(), SLOTS, n, (0.4, 0.6)[i]
    q.N, q.n_scales = 2, 2
    sm, cm, ms = bufs(torch.zeros(4)), bufs(torch.zeros(4)), bufs(torch.zeros(2))
    q.ssim_mean, q.cs_mean, q.ms_ssim = sm.data_ptr(), cm.data_ptr(), ms.data_ptr()
    return bufs, (C.byref(q), None), q


def mmd_call():
    bufs = Buffers()
    g = _gen(4)
    a = torch.rand(3, 2, 5, 7, generator=g)
    y, p = bufs(a), bufs(a + 0.05 * torch.randn(3, 2, 5, 7, generator=g))
    shape = (C.c_int64 * 5)(3, 2, 5, 7, 1)
    st = (C.c_int64 * 5)(*y.stride(), 1)
    ws, out = bufs(torch.zeros(8, dtype=torch.float64)), bufs(torch.zeros(1))
    return bufs, (y.data_ptr(), _lib.DT_F32, st, p.data_ptr(), _lib.DT_F32, st, shape, ws.data_ptr(), out.data_ptr(),
                  None), out


def moments_call():
    bufs = Buffers()
    x = bufs(torch.randn(40, 6, generator=_gen(5)).abs())
    mu, sigma = bufs(torch.zeros(6, dtype=torch.float64)), bufs(torch.zeros(36, dtype=torch.float64))
    p = FidMomentsParams()
    p.x, p.x_dtype, p.F, p.n = x.data_ptr(), _lib.DT_F32, 6, 40
    p.x_strides[:] = x.stride()
    p.mu, p.sigma = mu.data_ptr(), sigma.data_ptr()
    return bufs, (C.byref(p), None)


def frechet_call():
    from tests import fid_emulator as FE
    bufs = Buffers()
    g = _gen(6)
    (mx, sx), (my, sy) = (FE.fid_moments(torch.randn(n, 8, generator=g) + s) for n, s in ((30, 0.1), (25, 0.0)))
    t = [bufs(v.contiguous()) for v in (mx, sx, my, sy)]
    ws, out = bufs(torch.zeros(8, dtype=torch.float64)), bufs(torch.zeros(1, dtype=torch.float64))
    eig, rank = bufs(torch.zeros(8, dtype=torch.float64)), bufs(torch.zeros(1, dtype=torch.int32))
    p = FrechetParams()
    p.mu_x, p.sigma_x, p.mu_y, p.sigma_y = (v.data_ptr() for v in t)
    p.F, p.workspace, p.out, p.eigvals, p.rank = 8, ws.data_ptr(), out.data_ptr(), eig.data_ptr(), rank.data_ptr()
    return bufs, (C.byref(p), None)


def prep_call():
    bufs = Buffers()
    g = _gen(7)
    x, y = bufs(torch.rand(2, 3, 6, 5, generator=g)), bufs(torch.rand(2, 3, 6, 5, generator=g))
    out = bufs(torch.full((2 * 2 * 6 * 5 * 8,), float("nan")).to(ops.H16))
    st = [(C.c_int64 * 5)(t.stride(0), t.stride(1), 0, t.stride(2), t.stride(3)) for t in (x, y)]
    half = 2 * 6 * 5 * 8 * 2
    return bufs, (x.data_ptr(), _lib.DT_F32, st[0], y.data_ptr(), _lib.DT_F32, st[1], 3, 1, 6, 5, None, 2,
                  out.data_ptr(), out.data_ptr() + half, None)


def distance_call():
    """Two images of 6 pixels, 48 of 64 channels; pixel 2 of image 0 is an all-zero (dead) feature vector in x."""
    bufs = Buffers()
    g = _gen(8)
    fx = torch.randn(2, 6, 64, generator=g).relu()
    fy = (fx + 0.3 * torch.randn(2, 6, 64, generator=g)).relu()
    fx[0, 2] = 0.0
    x, y = bufs(fx), bufs(fy)
    pixel, image, image32 = bufs(torch.zeros(12)), bufs(torch.zeros(2, dtype=torch.float64)), bufs(torch.zeros(2))
    return bufs, (x.data_ptr(), y.data_ptr(), _lib.DT_F32, 2, 6, 48, 64, pixel.data_ptr(), image.data_ptr(),
                  image32.data_ptr(), None)


def mean_call():
    bufs = Buffers()
    image = bufs(torch.rand(5, generator=_gen(9), dtype=torch.float64))
    means, loss = bufs(torch.zeros(3, dtype=torch.float64)), bufs(torch.zeros(1))
    return bufs, (image.data_ptr(), 2, (C.c_int32 * 2)(2, 3), means.data_ptr(), loss.data_ptr(), None)


SIG = (1, 1, 6, 8)           # nC, n1, n2, n3: a 2-D 6 x 8 image, even n3


def fft_call():
    bufs = Buffers()
    g = _gen(10)
    x, y = bufs(torch.randn(2, 1, 6, 8, generator=g)), bufs(torch.randn(2, 1, 6, 8, generator=g))
    spec = bufs(torch.zeros(2 * 2 * 6 * 5, dtype=torch.complex64))
    st = [(C.c_int64 * 5)(t.stride(0), t.stride(1), 0, t.stride(2), t.stride(3)) for t in (x, y)]
    return bufs, (x.data_ptr(), _lib.DT_F32, st[0], y.data_ptr(), _lib.DT_F32, st[1], 2, (C.c_int32 * 4)(*SIG),
                  (C.c_int32 * 4)(*SIG), spec.data_ptr(), None)


def spectral_distance_call(reduction=_lib.REDUCTION_MEAN):
    bufs = Buffers()
    g = _gen(11)
    s = LE.spectral_fft(torch.randn(2, 1, 6, 8, generator=g), torch.randn(2, 1, 6, 8, generator=g), SIG[:1] + SIG[2:])
    spec = bufs(s.reshape(-1).to(torch.complex64))
    if reduction == _lib.REDUCTION_NONE:
        out, partials, result = bufs(torch.zeros(2 * 6 * 8)), None, None
    else:
        out = bufs(torch.zeros(1))
        partials = bufs(torch.zeros(_lib.SPECTRAL_PARTIALS, dtype=torch.float64))
        result = bufs(torch.zeros(2, dtype=torch.float64))
    ptr = lambda t: None if t is None else t.data_ptr()
    return bufs, (spec.data_ptr(), 2, (C.c_int32 * 4)(*SIG), 0.125, reduction, out.data_ptr(), ptr(partials),
                  ptr(result), None)


def adversarial_call(criterion=_lib.ADV_BCE, real=True, reduction=_lib.REDUCTION_NONE):
    """Two discriminator outputs; the first holds logits of -120 and +40, where BCE's -100 clamp decides."""
    bufs = Buffers()
    g = _gen(12)
    a, b = 3 * torch.randn(2, 1, 4, 4, generator=g), 3 * torch.randn(2, 1, 3, 3, generator=g)
    a[0, 0, 0, :2] = torch.tensor([-120.0, 40.0])
    xs = [bufs(a), bufs(b)]
    n = len(xs)
    shapes = (C.c_int64 * 10)(1, 2, 1, 4, 4, 1, 2, 1, 3, 3)
    strides = (C.c_int64 * 10)(0, *a.stride(), 0, *b.stride())
    elem = None
    if reduction == _lib.REDUCTION_NONE and criterion != _lib.ADV_HINGE:
        el = [bufs(torch.zeros(t.numel())) for t in xs]
        elem = (C.c_void_p * n)(*[t.data_ptr() for t in el])
    partials = bufs(torch.zeros(_lib.ADV_PARTIALS, dtype=torch.float64))
    losses, losses32 = bufs(torch.zeros(n + 1, dtype=torch.float64)), bufs(torch.zeros(n + 1))
    return bufs, ((C.c_void_p * n)(*[t.data_ptr() for t in xs]), (C.c_int32 * n)(_lib.DT_F32, _lib.DT_F32), shapes,
                  strides, n, criterion, int(real), reduction, elem, partials.data_ptr(), losses.data_ptr(),
                  losses32.data_ptr(), None)


CALLS = {
    "b200_ssim": lambda: ssim_call("uniform")[:2],
    "b200_ssim_combine": lambda: combine_call()[:2],
    "b200_mmd": lambda: mmd_call()[:2],
    "b200_fid_moments": moments_call,
    "b200_frechet": frechet_call,
    "b200_perceptual_prep": prep_call,
    "b200_perceptual_distance": distance_call,
    "b200_perceptual_mean": mean_call,
    "b200_spectral_fft": fft_call,
    "b200_spectral_distance": spectral_distance_call,
    "b200_adversarial": adversarial_call,
}


@pytest.mark.parametrize("name", list(CALLS))
def test_unmutated_stand_in_passes(monkeypatch, name):
    bufs, args = CALLS[name]()
    sh = run(monkeypatch, bufs, name, args)
    assert not sh.violations, sh.report()
    assert [c.name for c in sh.calls] == [name]


def test_more_calls_pass(monkeypatch):
    """The other shapes of the new rules: SSIM without maps and on the anisotropic kernel, the spectral distance's
    full-spectrum output and sum, every adversarial criterion with and without per-element outputs."""
    cases = [("b200_ssim", ssim_call("uniform", maps=False)[:2]), ("b200_ssim", ssim_call("aniso")[:2]),
             ("b200_spectral_distance", spectral_distance_call(_lib.REDUCTION_NONE)),
             ("b200_spectral_distance", spectral_distance_call(_lib.REDUCTION_SUM))]
    for crit in (_lib.ADV_BCE, _lib.ADV_HINGE, _lib.ADV_LEAST_SQUARES, _lib.ADV_LEAST_SQUARES_RAW):
        for real in (True, False):
            for red in (_lib.REDUCTION_NONE, _lib.REDUCTION_MEAN, _lib.REDUCTION_SUM):
                cases.append(("b200_adversarial", adversarial_call(crit, real, red)))
    for name, (bufs, args) in cases:
        sh = run(monkeypatch, bufs, name, args)
        assert not sh.violations, (name, sh.report())


# ------------------------------------------------------------------------------------------------------------------
# mutants
# ------------------------------------------------------------------------------------------------------------------
def mmd_over_bv(args):
    _f32(args[8], 1)[0] *= 3            # sum / (B V) instead of sum / (B^2 V), B = 3


def frechet_unsorted(args):
    p = _obj(args[0])
    e = _f64(p.eigvals, p.F)
    e[:] = e[::-1].copy()


def frechet_rank_off(args):
    p = _obj(args[0])
    np.ctypeslib.as_array(C.cast(p.rank, C.POINTER(C.c_int32)), shape=(1,))[0] += 1


def fft_conjugate(args):
    s = np.ctypeslib.as_array(C.cast(args[9], C.POINTER(C.c_float)), shape=(2 * 2 * 6 * 5 * 2,))
    s[1::2] *= -1


def nyquist_twice(args):
    """Weight 2 on the k3 = n3 / 2 bins of an even n3: the sum gains them once more."""
    spec, B, sig, scale, red, out, partials, result = args[:8]
    s = torch.from_numpy(np.ctypeslib.as_array(C.cast(spec, C.POINTER(C.c_float)), shape=(2 * 2 * 6 * 5 * 2,))
                         .copy()).view(torch.complex64).view(2, 2, 1, 1, 6, 5)
    a = (s.to(torch.complex128) * float(np.float32(scale))).abs()
    extra = float(((a[0] - a[1]) ** 2)[..., -1].sum())
    r = _f64(result, 2)
    r[0] += extra
    r[1] = r[0] / (2 * 6 * 8)
    _f32(out, 1)[0] = np.float32(r[1])


def adversarial_no_clamp(args):
    """BCE without the -100 clamp: -log p of a saturated sigmoid is +inf."""
    x = torch.from_numpy(_f32(args[0][0], 32).copy())
    p = torch.sigmoid(x)
    v = -torch.log(p)
    _f32(args[8][0], 32)[:] = v.numpy()
    ls = _f64(args[10], 3)
    ls[0], ls[2] = float(v.double().mean()), float(v.double().mean() + ls[1]) / 2
    _f32(args[11], 3)[:] = ls.astype(np.float32)


def hinge_sign(args):
    """Hinge with tanh not negated for a fake target."""
    xs = [torch.from_numpy(_f32(args[0][i], n).copy()).double() for i, n in ((0, 32), (1, 18))]
    per = [-torch.clamp(torch.tanh(t) - 1, max=0).mean() for t in xs]
    ls = _f64(args[10], 3)
    ls[:] = [float(per[0]), float(per[1]), float(per[0] + per[1]) / 2]
    _f32(args[11], 3)[:] = ls.astype(np.float32)


def eps_outside_quotient(args):
    """x_c / n_x + eps instead of x_c / (n_x + eps): a dead (all-zero) pixel gives 0 / 0."""
    x, y, dt, B, HW, C_, pitch, pixel, image, image32 = args[:10]
    fx, fy = (torch.from_numpy(_f32(t, B * HW * pitch).copy()).view(B, HW, pitch)[..., :C_].double() for t in (x, y))
    nx, ny = (t.pow(2).sum(-1, keepdim=True).sqrt() for t in (fx, fy))
    v = (fx / nx + PE.EPS32 - fy / ny - PE.EPS32).pow(2).sum(-1)
    _f32(pixel, B * HW)[:] = v.reshape(-1).float().numpy()
    _f64(image, B)[:] = v.mean(1).numpy()
    _f32(image32, B)[:] = v.mean(1).float().numpy()


def scratch_overrun(offset_arg, nbytes):
    """One 8-byte element written past the end of a scratch region (argument `offset_arg`, `nbytes` long)."""
    def fn(args):
        ptr = args[offset_arg]
        ptr = (_obj(ptr).workspace if hasattr(_obj(ptr), "workspace") else ptr)
        _bytes(int(ptr) + nbytes, 8)[:] = 0x7F
    return fn


def ssim_partials_overrun(args):
    p = _obj(args[0])
    _bytes(p.partials + p.N * 16 * SLOTS, 8)[:] = 0x7F


MUTANTS = {  # name: (entry, call, mutation: a Real.mutate name or a function of the arguments, what is violated)
    "ssim_scale_applied_twice": ("b200_ssim", lambda: ssim_call("uniform")[:2], "ssim_scale_twice", "stored values"),
    "ssim_swapped_hw_taps_3x9": ("b200_ssim", lambda: ssim_call("aniso")[:2], "ssim_swapped_hw_taps",
                                 "stored values"),
    "ssim_one_partial_slot_dropped": ("b200_ssim", lambda: ssim_call("uniform")[:2], "ssim_dropped_slot",
                                      "SSIM partial slots vs the kernel's own map"),
    "ssim_slot_dropped_without_maps": ("b200_ssim", lambda: ssim_call("uniform", maps=False)[:2],
                                       "ssim_dropped_slot", "SSIM partial slots vs the reading"),
    "combine_last_scale_uses_cs": ("b200_ssim_combine", lambda: combine_call()[:2], "combine_last_scale_cs",
                                   "stored values"),
    "mmd_divided_by_b_v": ("b200_mmd", lambda: mmd_call()[:2], mmd_over_bv, "stored values"),
    "frechet_eigenvalues_unsorted": ("b200_frechet", frechet_call, frechet_unsorted, "stored values"),
    "frechet_rank_off_by_one": ("b200_frechet", frechet_call, frechet_rank_off, "stored values"),
    "fft_conjugate_spectrum": ("b200_spectral_fft", fft_call, fft_conjugate, "stored values"),
    "spectral_nyquist_weighted_2": ("b200_spectral_distance", spectral_distance_call, nyquist_twice,
                                    "stored values"),
    "adversarial_clamp_dropped": ("b200_adversarial", adversarial_call, adversarial_no_clamp, "stored values"),
    "adversarial_hinge_sign_flipped": ("b200_adversarial",
                                       lambda: adversarial_call(_lib.ADV_HINGE, False, _lib.REDUCTION_MEAN),
                                       hinge_sign, "stored values"),
    "perceptual_eps_outside_quotient": ("b200_perceptual_distance", distance_call, eps_outside_quotient,
                                        "stored values"),
    "perceptual_mean_and_std_swapped": ("b200_perceptual_prep", prep_call, "prep_mean_std_swapped",
                                        "stored values"),
    "overrun_ssim_partials": ("b200_ssim", lambda: ssim_call("uniform")[:2], ssim_partials_overrun,
                              "outside the outputs"),
    "overrun_mmd_workspace": ("b200_mmd", lambda: mmd_call()[:2], scratch_overrun(7, 64), "outside the outputs"),
    "overrun_frechet_workspace": ("b200_frechet", frechet_call, scratch_overrun(0, 64), "outside the outputs"),
    "overrun_spectral_partials": ("b200_spectral_distance", spectral_distance_call,
                                  scratch_overrun(6, _lib.SPECTRAL_PARTIALS * 8), "outside the outputs"),
    "overrun_adversarial_partials": ("b200_adversarial", adversarial_call, scratch_overrun(9, _lib.ADV_PARTIALS * 8),
                                     "outside the outputs"),
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_rejects_mutant(monkeypatch, name):
    entry, make, mutate, what = MUTANTS[name]
    bufs, args = make()
    real = Real()
    if isinstance(mutate, str):
        real.mutate = mutate
    else:
        real = After(real, entry, mutate)
    sh = run(monkeypatch, bufs, entry, args, real)
    assert sh.violations, f"{name} passed the shadow check"
    assert any(what in v for v in sh.violations), sh.violations
    if what == "outside the outputs":
        print(f"\n{name}: rejected, bytes changed outside the outputs")
        return
    worst = max(c.excess for c in sh.calls)
    print(f"\n{name}: rejected by '{what}', worst err / tol {worst:.3g}")
    assert worst > 1.0
