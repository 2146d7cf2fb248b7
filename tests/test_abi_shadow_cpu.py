"""The shadow-call harness (tests/abi_shadow.py) on host memory: host tensors stand in for allocator segments and a
mutated CPU stand-in plays the real library.  The unmutated stand-in must pass on an igemm call with GroupNorm
partials and a split-K workspace, a two-source GroupNorm, flash attention with a workspace and a PNDM step; each
kernel-shaped mutant must be rejected; pointer translation must reach every place a pointer can hide and leave the
caller's struct alone."""
import ctypes as C

import numpy as np
import pytest
import torch

from generativemodels_b200 import _lib, ops
from generativemodels_b200._lib import ACT_SILU, FlashParams, GnApplyParams, GnStatsParams, IgemmParams, PndmCoef
from tests import abi_shadow, igemm_emulator as E, samplers_backend
from tests import test_igemm_contract_gpu as T


class Real(samplers_backend.SamplersFakeLib):
    """The stand-in as a 'real' library: host queries, scratch it scribbles on, and one mutation per test."""
    mutate = None

    def b200_igemm_plan(self, p, nsm, splits, out):
        out[0], out[1] = 64, 2 if _obj(p).split_ws else 1
        return 0

    def b200_igemm(self, p, stream):
        p = _obj(p)
        if p.split_ws:
            _bytes(p.split_ws, p.split_ws_bytes)[:] = 0xA5           # scratch: any bytes may be left there
        if self.mutate == "unwritten":
            return 0
        if self.mutate == "chunk":
            q = IgemmParams.from_buffer_copy(p)
            q.seg[q.n_seg - 1].nchunks -= 1
            E.emulate(q)
        else:
            E.emulate(p)
        if self.mutate is not None and self.mutate != "chunk":
            self.mutate(p)
        return 0

    def b200_groupnorm_fused(self, sp, ap, stream):
        s = _obj(sp)
        if s.partial:
            _bytes(s.partial, 16)[:] = 0x5A
        return super().b200_groupnorm_fused(sp, ap, stream)

    def b200_attention_flash(self, a, stream):
        o = _obj(a)
        if o.workspace:
            _bytes(o.workspace, o.workspace_bytes)[:] = 0x3C
        return super().b200_attention_flash(a, stream)


def _obj(a):
    return a._obj if hasattr(a, "_obj") else a


def _bytes(ptr, n):
    return np.ctypeslib.as_array(C.cast(int(ptr), C.POINTER(C.c_uint8)), shape=(int(n),))


def seg(x):
    """x copied into its own 'segment': a fresh buffer padded to a multiple of 8 bytes plus 8 guard bytes."""
    nb = x.numel() * x.element_size()
    raw = torch.zeros((nb + 7) // 8 * 8 + 8, dtype=torch.uint8)
    v = raw[:nb].view(x.dtype).view(x.shape)
    v.copy_(x)
    return raw, v


class Buffers:
    def __init__(self):
        self.raw = []

    def __call__(self, x):
        raw, v = seg(x)
        self.raw.append(raw)
        return v

    def memory(self):
        return abi_shadow.HostMemory(self.raw)


def run(monkeypatch, bufs, name, args, mutate=None):
    real = Real()
    real.mutate = mutate
    with abi_shadow.shadow(monkeypatch, memory=bufs.memory(), real=real) as sh:
        rc = getattr(_lib.require_device(), name)(*args)
    assert rc == 0
    return sh


# ------------------------------------------------------------------------------------------------------------------
# the calls
# ------------------------------------------------------------------------------------------------------------------
IGEMM = T.conv("shadow_gn8_split", "fast", None, 2, (1, 8, 6), [128], 64, act1=ACT_SILU, gn=8, out_pad=8)
PAD = T.conv("shadow_pad_cols", "general scalar", None, 1, (1, 5, 7), [64], 60, out_cols=64, w_rows=64)


def igemm_call(case=IGEMM):
    g = T.Geom(case, 2)
    bufs = Buffers()
    t = {k: bufs(v) for k, v in T.make_operands(case, g).items()}
    p = T.fill(case, g, T.host_ptrs(t))
    ws = bufs(torch.zeros(4096, dtype=torch.uint8))
    p.split_ws, p.split_ws_bytes = ws.data_ptr(), 4096
    return bufs, t, p


def test_accepts_igemm_with_gn_partials_and_split_workspace(monkeypatch):
    bufs, t, p = igemm_call()
    before = bytes(p)
    sh = run(monkeypatch, bufs, "b200_igemm", (C.byref(p), None))
    assert not sh.violations, sh.report()
    assert bytes(p) == before, "the caller's struct changed"
    assert {"igemm gn8", "igemm bn64", "igemm split"} <= sh.paths()
    assert (t["gn"].sum() != 0) and torch.isfinite(t["out"][:1]).all()


def two_source_gn():
    bufs = Buffers()
    g = torch.Generator().manual_seed(3)
    Nn, S, C0, C1 = 2, 16, 32, 32
    x0, x1 = bufs(torch.randn(Nn * S * 40, generator=g).to(ops.H16)), bufs(torch.randn(Nn * S * 32, generator=g).to(ops.H16))
    gamma, beta = bufs(1 + 0.1 * torch.randn(C0 + C1, generator=g)), bufs(0.1 * torch.randn(C0 + C1, generator=g))
    y, ws = bufs(torch.full((Nn * S * 72,), float("nan")).to(ops.H16)), bufs(torch.zeros(4, dtype=torch.float32))
    sp, ap = GnStatsParams(), GnApplyParams()
    for q in (sp, ap):
        q.x_ptr[0], q.x_ptr[1], q.x_C[0], q.x_C[1], q.x_pitch[0], q.x_pitch[1] = x0.data_ptr(), x1.data_ptr(), C0, C1, 40, 32
        q.N, q.spatial = Nn, S
    sp.groups, sp.eps, sp.gamma, sp.beta, sp.partial = 8, 1e-5, gamma.data_ptr(), beta.data_ptr(), ws.data_ptr()
    ap.act, ap.y_ptr, ap.y_pitch = ACT_SILU, y.data_ptr(), 72
    return bufs, (C.byref(sp), C.byref(ap), None), y


def test_accepts_two_source_groupnorm(monkeypatch):
    bufs, args, y = two_source_gn()
    sh = run(monkeypatch, bufs, "b200_groupnorm_fused", args)
    assert not sh.violations, sh.report()
    assert torch.isfinite(y.view(-1, 72)[:, :64]).all()


def flash_call():
    bufs = Buffers()
    g = torch.Generator().manual_seed(4)
    B, T_, S, heads, dh = 1, 64, 64, 1, 64
    q, k = bufs(torch.randn(B * T_ * dh, generator=g).to(ops.H16)), bufs(torch.randn(B * S * dh, generator=g).to(ops.H16))
    vt, out = bufs(torch.randn(B * dh * S, generator=g).to(ops.H16)), bufs(torch.zeros(B * T_ * dh, dtype=ops.H16))
    ws = bufs(torch.zeros(256, dtype=torch.uint8))
    a = FlashParams()
    a.q, a.k, a.vt, a.out, a.res = q.data_ptr(), k.data_ptr(), vt.data_ptr(), out.data_ptr(), None
    a.B, a.T, a.S, a.heads, a.dh = B, T_, S, heads, dh
    a.q_pitch = a.k_pitch = a.out_pitch = dh
    a.vt_pitch, a.scale, a.workspace, a.workspace_bytes = S, dh ** -0.5, ws.data_ptr(), 256
    return bufs, (C.byref(a), None)


def test_accepts_flash_with_workspace(monkeypatch):
    bufs, args = flash_call()
    sh = run(monkeypatch, bufs, "b200_attention_flash", args)
    assert not sh.violations, sh.report()
    assert "flash dh64" in sh.paths()


def pndm_call():
    bufs = Buffers()
    g = torch.Generator().manual_seed(5)
    n = 100
    h0, h1, s = (bufs(torch.randn(n, generator=g)) for _ in range(3))
    prev, eps = bufs(torch.zeros(n)), bufs(torch.zeros(n))
    c = PndmCoef()
    c.w[0], c.w[1], c.n_hist, c.sample_coeff, c.eps_coeff, c.prediction_type = 1.5, -0.5, 2, 1.01, 0.04, 0
    hist = (C.c_void_p * 2)(h0.data_ptr(), h1.data_ptr())
    return bufs, (hist, s.data_ptr(), C.byref(c), prev.data_ptr(), eps.data_ptr(), n, None), prev


def test_accepts_pndm_step(monkeypatch):
    bufs, args, prev = pndm_call()
    sh = run(monkeypatch, bufs, "b200_pndm_step", args)
    assert not sh.violations, sh.report()
    assert (prev != 0).all()


# ------------------------------------------------------------------------------------------------------------------
# mutants
# ------------------------------------------------------------------------------------------------------------------
def _out16(p, count):
    return torch.from_numpy(np.ctypeslib.as_array(C.cast(p.out_ptr, C.POINTER(C.c_uint16)),
                                                  shape=(count,)).view(np.int16)).view(ops.H16)


def move_by_twice_the_bound(p):
    """One element moved by a 16-bit value more than twice its bound away."""
    fp = E.footprint(p)
    out = _out16(p, int(fp.max()) + 1)
    want = out.double().numpy()[fp]
    tol = float(E.bound(p, want, want)[0, 0, 2, 3, 5])
    i = int(fp[0, 0, 2, 3, 5])
    out[i] = torch.tensor(float(out[i]) + 2.5 * tol).to(ops.H16)


def write_past_row(p):
    i = int(E.footprint(p)[0, 0, 1, 1, -1]) + 1
    _out16(p, i + 1)[i] = 1.0


def write_padding_column(p):
    i = int(E.footprint(p)[0, 0, 1, 1, p.cout])
    _out16(p, i + 1)[i] = -0.0


def write_input(p):
    a = torch.from_numpy(np.ctypeslib.as_array(C.cast(p.a_ptr[0], C.POINTER(C.c_uint16)), shape=(8,)).view(np.int16))
    a[3] ^= 1


def wrong_slot_sum(p):
    gw = p.gn_group or 8
    part = np.ctypeslib.as_array(C.cast(p.gn_partial, C.POINTER(C.c_float)),
                                 shape=(p.out_N * p.gn_slots * (p.cout // gw) * 2,))
    part[p.gn_slot0 * (p.cout // gw) * 2 + 2] *= 1.01


MUTANTS = {
    "moved_by_twice_the_bound": (IGEMM, move_by_twice_the_bound, "igemm output"),
    "dropped_64_channel_chunk": (IGEMM, "chunk", "igemm output"),
    "output_unwritten": (IGEMM, "unwritten", "igemm output"),
    "write_one_past_the_row": (IGEMM, write_past_row, "outside the outputs"),
    "write_into_padding_column": (PAD, write_padding_column, "padding columns"),
    "write_into_an_input": (IGEMM, write_input, "outside the outputs"),
    "wrong_gn_slot_sum": (IGEMM, wrong_slot_sum, "GroupNorm partial sums"),
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_rejects_mutant(monkeypatch, name):
    case, mutate, what = MUTANTS[name]
    bufs, t, p = igemm_call(case)
    sh = run(monkeypatch, bufs, "b200_igemm", (C.byref(p), None), mutate=mutate)
    assert sh.violations, f"{name} passed the shadow check"
    assert any(what in v for v in sh.violations), sh.violations


def test_pad_case_passes_unmutated(monkeypatch):
    bufs, t, p = igemm_call(PAD)
    sh = run(monkeypatch, bufs, "b200_igemm", (C.byref(p), None))
    assert not sh.violations, sh.report()


def test_mutated_elementwise_store_is_rejected(monkeypatch):
    """A wrong value stored through the recorder path (not b200_igemm): PNDM's prev off by 1e-3 relative."""
    class Off(Real):
        def b200_pndm_step(self, hist, s, c, prev, eps_out, n, stream):
            super().b200_pndm_step(hist, s, c, prev, eps_out, n, stream)
            np.ctypeslib.as_array(C.cast(prev, C.POINTER(C.c_float)), shape=(n,))[7] *= 1.001
            return 0
    bufs, args, _ = pndm_call()
    with abi_shadow.shadow(monkeypatch, memory=bufs.memory(), real=Off()) as sh:
        _lib.require_device().b200_pndm_step(*args)
    assert any("stored values" in v for v in sh.violations), sh.violations


# ------------------------------------------------------------------------------------------------------------------
# pointer translation
# ------------------------------------------------------------------------------------------------------------------
def test_translation_reaches_every_pointer_and_leaves_the_struct_alone():
    p = GnStatsParams()
    p.x_ptr[0], p.x_ptr[1], p.gamma, p.partial, p.N = 0x1000, 0x2000, 0x3000, 0, 7
    arr = (C.c_void_p * 2)(0x4000, None)
    ints = (C.c_int32 * 2)(5, 6)
    args = [C.byref(p), arr, ints, 0x5000, None]
    types = [C.POINTER(GnStatsParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    before = bytes(p)
    found = abi_shadow.pointers(args, types)
    assert sorted(found) == [0x1000, 0x2000, 0x3000, 0x4000, 0x5000]
    out = abi_shadow.translate(args, types, lambda v: v + 1)
    q = out[0]._obj
    assert (q.x_ptr[0], q.x_ptr[1], q.gamma, q.partial, q.N) == (0x1001, 0x2001, 0x3001, None, 7)
    assert (out[1][0], out[1][1]) == (0x4001, None)
    assert out[2] is ints and out[3] == 0x5001 and out[4] is None
    assert bytes(p) == before and arr[0] == 0x4000


def test_unknown_pointer_and_unknown_entry_fail(monkeypatch):
    bufs, args, _ = pndm_call()
    bad = list(args)
    bad[3] = 0x10            # prev outside every segment
    with abi_shadow.shadow(monkeypatch, memory=bufs.memory(), real=Real()):
        with pytest.raises(AssertionError, match="no allocator segment"):
            _lib.require_device().b200_pndm_step(*bad)
        with pytest.raises(AssertionError, match="neither a host query"):
            _lib.require_device().b200_not_an_entry_point


BIG = T.gemm("shadow_sampled_rows", "lean", None, 9000, 64, 64, out_pad=8)


def test_large_igemm_checks_a_deterministic_subset_of_rows(monkeypatch):
    """A call of more than 8192 output rows is compared on igemm_emulator.sample_voxels's rows; an output left
    unwritten or a wrong value on a sampled row is still rejected, and the footprint check still sees every row."""
    bufs, t, p = igemm_call(BIG)
    sh = run(monkeypatch, bufs, "b200_igemm", (C.byref(p), None))
    assert not sh.violations, sh.report()
    assert "igemm sampled rows" in sh.paths()

    def one_percent_off(q):
        out = _out16(q, 64)
        out[5] = torch.tensor(float(out[5]) * 1.01 + 0.01).to(ops.H16)
    def write_past_an_unsampled_row(q):
        i = int(E.footprint(q)[0, 0, 0, 4000, -1]) + 1
        _out16(q, i + 1)[i] = 1.0
    assert 4000 not in E.sample_voxels(p)
    for mutate, what in (("unwritten", "igemm output"), (one_percent_off, "igemm output"),
                         (write_past_an_unsampled_row, "outside the outputs")):
        bufs, t, p = igemm_call(BIG)
        sh = run(monkeypatch, bufs, "b200_igemm", (C.byref(p), None), mutate=mutate)
        assert any(what in v for v in sh.violations), (mutate, sh.violations)
