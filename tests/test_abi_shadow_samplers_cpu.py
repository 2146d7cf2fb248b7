"""The shadow-call harness (tests/abi_shadow.py) on the scheduler, sampler-step and inferer entry points, on host memory:
host tensors stand in for allocator segments and a mutated CPU stand-in plays the real library, as in
tests/test_abi_shadow_cpu.py.  The unmutated stand-in must pass one call of each entry point (and the variants whose
path labels tests/test_abi_shadow_inferers_gpu.py asks for); each kernel-shaped mutant must be rejected by the rule
written for it, and the test prints by what factor (the worst err / tol of the call, inf for a NaN or a value the
reading does not have; a write outside the outputs has no factor).

The step calls run on N_EL = 75 elements (n % 4 = 3, the vector kernels' scalar tail) with 16-byte aligned buffers,
and every output buffer has SLACK floats after its n elements, so that a store past n lands inside the segment where
the footprint check sees it."""
import ctypes as C

import numpy as np
import pytest
import torch

from generativemodels_b200 import _lib, ops
from generativemodels_b200._lib import DdimCoef, DdpmCoef, DpmCoef, KlCoef, SASolverCoef, UniPCCoef
from tests import abi_shadow
from tests.test_abi_shadow_cpu import Buffers, pndm_call

N_EL = 75
SLACK = 4
EPS, SAMPLE, V = _lib.PRED_EPSILON, _lib.PRED_SAMPLE, _lib.PRED_V


def _obj(a):
    return a._obj if hasattr(a, "_obj") else a


def _f32(ptr, n):
    return np.ctypeslib.as_array(C.cast(int(ptr), C.POINTER(C.c_float)), shape=(int(n),))


def _f64(ptr, n):
    return np.ctypeslib.as_array(C.cast(int(ptr), C.POINTER(C.c_double)), shape=(int(n),))


class Wrap:
    """`real` with `entry` replaced by fn(f, args), f the real entry point (a kernel that computes something else)."""

    def __init__(self, real, entry, fn):
        self.real, self.entry, self.fn = real, entry, fn

    def __getattr__(self, name):
        f = getattr(self.real, name)
        return f if name != self.entry else (lambda *args: self.fn(f, args))


def run(monkeypatch, bufs, name, args, real=None):
    with abi_shadow.shadow(monkeypatch, memory=bufs.memory(),
                           real=real if real is not None else abi_shadow.StandIn()) as sh:
        rc = getattr(_lib.require_device(), name)(*args)
    assert rc == 0
    return sh


# ------------------------------------------------------------------------------------------------------------------
# one call of each entry point, on host buffers
# ------------------------------------------------------------------------------------------------------------------
class Bufs(Buffers):
    """Buffers with the inputs and outputs of a step call: seeded inputs, NaN outputs with SLACK floats after n; an
    input `unaligned` sits 4 bytes into its segment."""

    def __init__(self, seed):
        super().__init__()
        self.g = torch.Generator().manual_seed(seed)

    def inp(self, n=N_EL, scale=1.0, unaligned=False):
        t = self(scale * torch.randn(n + 1, generator=self.g))
        return (t[1:] if unaligned else t[:n]).data_ptr()

    def out(self, n=N_EL, dtype=torch.float32):
        return self(torch.full((n + SLACK,), float("nan"), dtype=dtype)).data_ptr()


def _hist(ptrs, size):
    return (C.c_void_p * max(size, 1))(*ptrs)


def ddim_call(noise=True, pred=EPS, unaligned=False, n=N_EL):
    b = Bufs(1)
    c = DdimCoef(0.6, 0.8, 0.75, 0.6, 0.2 if noise else 0.0, -1.0, 1.0, pred, 1)
    m, s = b.inp(n, unaligned=unaligned), b.inp(n, 1.5)
    z = b.inp(n) if noise else None
    return b, (m, s, z, C.byref(c), b.out(n), b.out(n), n, None)


def ddpm_call(var_mode=2, noise=True, pred=V):
    b = Bufs(2)
    c = DdpmCoef(0.6, 0.8, 0.3, 0.9, 0.1, -1.0, 1.0, 0.01, 0.02, var_mode, pred, 1)
    m, s = b.inp(), b.inp(scale=1.5)
    z = b.inp() if noise else None
    pv = b(torch.rand(N_EL, generator=b.g) * 2 - 1).data_ptr() if var_mode else None
    return b, (m, s, z, pv, C.byref(c), b.out(), b.out(), N_EL, None)


def dpm_call(nh=2, noise=True, unaligned=False, n=N_EL):
    b = Bufs(3)
    c = DpmCoef(0.6, 0.8, 0.7, (C.c_float * 3)(0.5, -0.2, 0.1), 0.3 if noise else 0.0, -1.0, 1.0, EPS, 1)
    m, s = b.inp(n, unaligned=unaligned), b.inp(n, 1.5)
    h = [b.inp(n) for _ in range(nh)]
    z = b.inp(n) if noise else None
    return b, (m, s, _hist(h, nh), nh, z, C.byref(c), b.out(n), b.out(n), n, None)


def unipc_call(nh=3, last=True, unaligned=False, n=N_EL, pred=EPS):
    b = Bufs(4)
    c = UniPCCoef(0.6, 0.8, 0.9, (C.c_float * 4)(0.3, 0.2, -0.15, 0.05), 0.8, (C.c_float * 3)(0.4, -0.3, 0.1),
                  -1.0, 1.0, pred, 1)
    m, s = b.inp(n, unaligned=unaligned), b.inp(n, 1.5)
    lp = b.inp(n) if last else None
    h = [b.inp(n) for _ in range(nh)]
    return b, (m, s, lp, _hist(h, nh), nh, C.byref(c), b.out(n), b.out(n), b.out(n), n, None)


def sa_call(nh=2, last=True, zl=True, z=True, unaligned=False, n=N_EL, pred=SAMPLE):
    b = Bufs(5)
    c = SASolverCoef(0.6, 0.8, 0.85, (C.c_float * 3)(0.3, 0.2, -0.1), 0.25 if zl else 0.0, 0.8,
                     (C.c_float * 3)(0.4, -0.3, 0.1), 0.35 if z else 0.0, -1.0, 1.0, pred, 1)
    m, s = b.inp(n, 1.5, unaligned=unaligned), b.inp(n, 1.5)
    lp = b.inp(n) if last else None
    zlp = b.inp(n) if zl else None
    h = [b.inp(n) for _ in range(nh)]
    zp = b.inp(n) if z else None
    return b, (m, s, lp, zlp, _hist(h, nh), nh, zp, C.byref(c), b.out(n), b.out(n), b.out(n), n, None)


def add_noise_call(sign=1.0):
    b = Bufs(6)
    ca = torch.tensor([0.9, 0.5, 0.2])
    x0, z = b.inp(), b.inp()
    cap, cbp = b(ca).data_ptr(), b((1 - ca * ca).sqrt()).data_ptr()
    return b, (x0, z, cap, cbp, sign, 3, N_EL // 3, b.out(), None)


def ddpm_kl_call(t0=True, pred=EPS, clip=1):
    """Three items of 25; the image holds values at and beyond the t = 0 edge bins (|a| > 0.999)."""
    b = Bufs(7)
    a = torch.rand(N_EL, generator=b.g) * 2 - 1
    a[::7], a[3::7] = 1.0, -1.0
    x0 = b(a)
    xt = b(0.9 * a + 0.4 * torch.randn(N_EL, generator=b.g)).data_ptr()
    c = KlCoef(0.95, 0.31, 0.5, 0.45, -5.0, -5.0, 2.0 / 255, pred, clip, int(t0))
    ssum = b(torch.zeros(3, dtype=torch.float64)).data_ptr()
    return b, (x0.data_ptr(), xt, b.inp(), C.byref(c), b.out(), ssum, 3, N_EL // 3, None)


def scale_call(div=True):
    b = Bufs(8)
    mul, d = (1.0, 0.18215) if div else (0.18215, 1.0)
    return b, (b.inp(), mul, d, b.out(), N_EL, None)


def fma_call():
    b = Bufs(9)
    return b, (b.inp(), b.inp(), b.inp(), b.out(), N_EL, None)


def exp_half_call():
    b = Bufs(10)
    return b, (b.inp(scale=20.0), -30.0, 20.0, b.out(), N_EL, None)


def vq_gather_call():
    b = Bufs(11)
    M, K, D, qp = 10, 6, 8, 8
    idx = b(torch.randint(0, K, (M,), generator=b.g)).data_ptr()
    return b, (idx, M, b.inp(K * D), K, D, b.out(M * qp, ops.H16), qp, None)


def vae_reparam_call():
    b = Bufs(12)
    return b, (b.inp(), b.inp(), b.inp(), b.out(), b.out(1), N_EL, None)


CALLS = {
    "b200_ddim_step": ddim_call,
    "b200_ddpm_step": ddpm_call,
    "b200_pndm_step": lambda: pndm_call()[:2],
    "b200_dpm_solver_step": dpm_call,
    "b200_unipc_step": unipc_call,
    "b200_sa_solver_step": sa_call,
    "b200_add_noise": add_noise_call,
    "b200_ddpm_kl": ddpm_kl_call,
    "b200_scale_f32": scale_call,
    "b200_fma_f32": fma_call,
    "b200_exp_half_clamped": exp_half_call,
    "b200_vq_gather": vq_gather_call,
    "b200_vae_reparam_kld": vae_reparam_call,
}


@pytest.mark.parametrize("name", list(CALLS))
def test_unmutated_stand_in_passes(monkeypatch, name):
    bufs, args = CALLS[name]()
    sh = run(monkeypatch, bufs, name, args)
    assert not sh.violations, sh.report()
    assert [c.name for c in sh.calls] == [name]


VARIANTS = [  # (entry, call, the path labels it must carry)
    ("b200_ddim_step", lambda: ddim_call(False, SAMPLE), {"ddim", "ddim step tail"}),
    ("b200_ddim_step", lambda: ddim_call(True, V, unaligned=True), {"ddim noise", "ddim step scalar"}),
    ("b200_ddim_step", lambda: ddim_call(n=64), {"ddim step vec"}),
    ("b200_ddpm_step", lambda: ddpm_call(0, pred=EPS), {"ddpm var0"}),
    ("b200_ddpm_step", lambda: ddpm_call(1, pred=SAMPLE), {"ddpm var1"}),
    ("b200_ddpm_step", lambda: ddpm_call(2), {"ddpm var2"}),
    ("b200_ddpm_step", lambda: ddpm_call(2, noise=False), {"ddpm no noise"}),
    ("b200_dpm_solver_step", lambda: dpm_call(0, False), {"dpm nh0", "dpm step tail"}),
    ("b200_dpm_solver_step", lambda: dpm_call(1, True, unaligned=True), {"dpm nh1 noise", "dpm step scalar"}),
    ("b200_dpm_solver_step", lambda: dpm_call(2, False, n=64), {"dpm nh2", "dpm step vec"}),
    ("b200_unipc_step", lambda: unipc_call(0, False, pred=V), {"unipc nh0", "unipc step tail"}),
    ("b200_unipc_step", lambda: unipc_call(1, True, unaligned=True), {"unipc nh1 last", "unipc step scalar"}),
    ("b200_unipc_step", lambda: unipc_call(2, True, n=64, pred=SAMPLE), {"unipc nh2 last", "unipc step vec"}),
    ("b200_sa_solver_step", lambda: sa_call(0, False, False, False, pred=EPS), {"sa nh0", "sa step tail"}),
    ("b200_sa_solver_step", lambda: sa_call(1, True, False, True, unaligned=True),
     {"sa nh1 last z", "sa step scalar"}),
    ("b200_sa_solver_step", lambda: sa_call(2, True, True, False, n=64, pred=V), {"sa nh2 last zl", "sa step vec"}),
    ("b200_add_noise", lambda: add_noise_call(-1.0), {"add_noise -"}),
    ("b200_ddpm_kl", lambda: ddpm_kl_call(False, V, 0), {"ddpm_kl t"}),
    ("b200_ddpm_kl", lambda: ddpm_kl_call(True, SAMPLE, 0), {"ddpm_kl t0"}),
    ("b200_scale_f32", lambda: scale_call(False), {"scale mul"}),
]


def test_variants_pass_and_carry_their_path_labels(monkeypatch):
    """Every path label the GPU file asks for, on the unmutated stand-in: history depths, optional streams, variance
    modes, both likelihood branches, both signs and scale forms, and the three access paths of the step kernels."""
    for name, make, want in VARIANTS:
        bufs, args = make()
        sh = run(monkeypatch, bufs, name, args)
        assert not sh.violations, (name, want, sh.report())
        assert want <= sh.paths(), (name, want, sh.paths())


# ------------------------------------------------------------------------------------------------------------------
# mutants
# ------------------------------------------------------------------------------------------------------------------
N_ARG = {"b200_ddim_step": 6, "b200_dpm_solver_step": 8, "b200_unipc_step": 9, "b200_sa_solver_step": 11}
OUT_ARGS = {"b200_ddim_step": (4, 5), "b200_dpm_solver_step": (6, 7), "b200_unipc_step": (6, 7, 8),
            "b200_sa_solver_step": (8, 9, 10)}
COEF_ARG = {"b200_ddim_step": 3, "b200_ddpm_step": 4, "b200_dpm_solver_step": 5, "b200_unipc_step": 5,
            "b200_sa_solver_step": 7, "b200_ddpm_kl": 3}
STEP_CALLS = {"b200_ddim_step": ddim_call, "b200_dpm_solver_step": dpm_call, "b200_unipc_step": unipc_call,
              "b200_sa_solver_step": sa_call}


def with_args(change):
    """The entry point called with the arguments change(list(args)) (a kernel that reads the wrong stream)."""
    return lambda f, args: f(*change(list(args)))


def with_coef(entry, **fields):
    """The entry point called with a copy of its coefficient struct with `fields` set (values, or functions of the
    old value)."""
    i = COEF_ARG[entry]

    def fn(f, args):
        q = type(_obj(args[i])).from_buffer_copy(_obj(args[i]))
        for k, v in fields.items():
            setattr(q, k, v(getattr(q, k)) if callable(v) else v)
        return f(*args[:i], C.byref(q), *args[i + 1:])
    return fn


def _swap01(arr):
    v = list(arr)
    return type(arr)(v[1], v[0], *v[2:])


def unwritten(k):
    """Output argument k keeps what it held before the call."""
    def fn(f, args):
        n = args[N_ARG["b200_unipc_step"]]
        keep = _f32(args[k], n).copy()
        rc = f(*args)
        _f32(args[k], n)[:] = keep
        return rc
    return fn


def tail_skipped(entry):
    """The scalar tail skipped: the last n % 4 elements of every output keep what they held."""
    def fn(f, args):
        n = args[N_ARG[entry]]
        lo = n - n % 4
        keep = [(args[i], _f32(args[i], n)[lo:].copy()) for i in OUT_ARGS[entry] if args[i]]
        rc = f(*args)
        for p, k in keep:
            _f32(p, n)[lo:] = k
        return rc
    return fn


def float4_past_n(entry):
    """The tail stored as one whole float4: the first output is also written from n up to the next multiple of 4."""
    def fn(f, args):
        rc = f(*args)
        n = args[N_ARG[entry]]
        end = (n + 3) // 4 * 4
        _f32(args[OUT_ARGS[entry][0]], end)[n:end] = 0.0
        return rc
    return fn


def kl_sum_to_other_item(f, args):
    """Each item's sum added into the next item's slot."""
    rc = f(*args)
    s = _f64(args[5], args[6])
    s[:] = np.roll(s.copy(), 1)
    return rc


def add_noise_item0_coefs(f, args):
    """Item 0's coefficients applied to every item."""
    rc = f(*args)
    x0, z, ca, cb, sign, N_, per, out = args[:8]
    a, b = np.float32(_f32(ca, N_)[0]), np.float32(_f32(cb, N_)[0]) * np.float32(sign)
    _f32(out, N_ * per)[:] = a * _f32(x0, N_ * per) + b * _f32(z, N_ * per)
    return rc


MUTANTS = {  # name: (entry, call, fn(f, args), what is violated)
    "unipc_corrector_dropped": ("b200_unipc_step", unipc_call, with_args(lambda a: a[:2] + [None] + a[3:]),
                                "stored values"),
    "unipc_hist0_hist1_swapped": ("b200_unipc_step", unipc_call,
                                  with_args(lambda a: a[:3] + [_swap01(a[3])] + a[4:]), "stored values"),
    "unipc_xc_out_unwritten": ("b200_unipc_step", unipc_call, unwritten(8), "stored values"),
    "sa_z_used_for_zl": ("b200_sa_solver_step", sa_call, with_args(lambda a: a[:3] + [a[6]] + a[4:]),
                         "stored values"),
    "sa_noise_added_twice": ("b200_sa_solver_step", sa_call, with_coef("b200_sa_solver_step", c_z=lambda v: 2 * v),
                             "stored values"),
    "dpm_sde_noise_dropped": ("b200_dpm_solver_step", dpm_call, with_args(lambda a: a[:4] + [None] + a[5:]),
                              "stored values"),
    "ddpm_kl_kl_at_t0": ("b200_ddpm_kl", ddpm_kl_call, with_coef("b200_ddpm_kl", is_t0=0), "stored values"),
    "ddpm_kl_sum_into_wrong_item": ("b200_ddpm_kl", lambda: ddpm_kl_call(False), kl_sum_to_other_item,
                                    "stored values"),
    "add_noise_item0_coefficients": ("b200_add_noise", add_noise_call, add_noise_item0_coefs, "stored values"),
    "ddpm_clip_ignored": ("b200_ddpm_step", ddpm_call, with_coef("b200_ddpm_step", clip=0), "stored values"),
    "scale_multiplies_by_divide_by": ("b200_scale_f32", scale_call, with_args(lambda a: [a[0], a[2], 1.0] + a[3:]),
                                      "stored values"),
}
for _e, _make in STEP_CALLS.items():
    _fam = _e[5:-5]
    MUTANTS[f"{_fam}_tail_skipped"] = (_e, _make, tail_skipped(_e), "stored values")
    MUTANTS[f"{_fam}_float4_past_n"] = (_e, _make, float4_past_n(_e), "outside the outputs")
    MUTANTS[f"{_fam}_clip_ignored"] = (_e, _make, with_coef(_e, clip=0), "stored values")


@pytest.mark.parametrize("name", list(MUTANTS))
def test_rejects_mutant(monkeypatch, name):
    entry, make, fn, what = MUTANTS[name]
    bufs, args = make()
    sh = run(monkeypatch, bufs, entry, args, Wrap(abi_shadow.StandIn(), entry, fn))
    assert sh.violations, f"{name} passed the shadow check"
    assert any(what in v for v in sh.violations), sh.violations
    if what == "outside the outputs":
        print(f"\n{name}: rejected, bytes changed outside the outputs")
        return
    worst = max(c.excess for c in sh.calls)
    print(f"\n{name}: rejected by '{what}', worst err / tol {worst:.3g}")
    assert worst > 1.0
