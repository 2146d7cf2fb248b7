"""Shadow calls: every C-ABI call a network, metric, loss, scheduler or inferer makes runs on the real library AND on
the CPU stand-in (StandIn below: tests/losses_backend.LossesFakeLib, which carries the metric, FID and perceptual entry
points, and tests/{unipc,sa_solver}_backend's stand-ins, which carry the three sampler steps) with the call's own inputs, and the two are compared under the bound of the
entry point's family.  Test infrastructure only.

    with abi_shadow.shadow(monkeypatch) as sh:
        model(x)
    assert not sh.violations, sh.report()

For each b200_* call the proxy installed in place of _lib.require_device()

  1. passes host queries (PASSTHROUGH) to the real library: the split-K workspace size in particular, so that the
     networks take the same paths as without the shadow;
  2. finds every device pointer of the call (plain c_void_p arguments, c_void_p fields and c_void_p array fields of
     the parameter structs, ctypes pointer arrays such as the partial-sum list of GroupNorm or the history of the PNDM
     and DPM steps) and the allocator segment holding it; a pointer in no segment fails the call;
  3. copies those segments to the host, runs the real entry point, and copies them again (no device allocation in
     between);
  4. runs the stand-in on a host copy of the pre-call segments, with every pointer translated into that copy in a
     cloned struct or array (the caller's struct is never touched: ops caches parameter templates);
  5. compares every region the stand-in stored (cpu_backend.RECORDER reports the view and the emulator's Result)
     with the device's bytes under the family's rule: elementwise / norm / attention excess <= 1, copies (resampling,
     weight repacking, VQ indices, the perceptual input preparation) bit for bit, GroupNorm affine tables by
     affine_excess; the metric and loss outputs under the bounds of tests/{metrics,fid,perceptual,losses}_emulator.py
     (fp32 and fp64 values per element, the FFT's spectra norm-wise per (side, image)); b200_ssim's partial slots
     summed per item, against the float64 sums of the kernel's own maps when it stores them and against the reading's
     sums within the sum of its per-voxel bounds always; b200_igemm under
     igemm_emulator.bound on its footprint (calls of more than 8192 output voxels per sample on the deterministic
     subset igemm_emulator.sample_voxels; the footprint, padding and partial-sum checks below see every voxel),
     padding columns +0, GroupNorm partials summed over slots against the
     float64 sums of the kernel's own stored output and softmax partials against the kernel's own fp32 rows, as
     tests/test_igemm_contract_gpu.py does;
  6. checks the footprint: every other byte of every touched segment is bit-identical before and after the call,
     except the declared scratch (split-K split_ws, the flash workspace, the GroupNorm statistics workspace, the MMD,
     Frechet, spectral-distance and adversarial workspaces).

Each call is logged with a compact argument signature, its worst excess and, for b200_igemm, the planner's column
tile and split factor and the store path (the predicates of tests/test_igemm_contract_gpu.py's docstring), so that a
test can assert which kernel paths the networks reached.  The scheduler and inferer entry points carry path labels
too (step_paths), derived from the call's arguments with the predicates the .cu files choose their kernels by.
"""
from __future__ import annotations

import bisect
import contextlib
import ctypes as C
import math
from collections import defaultdict
from dataclasses import dataclass, field

import numpy as np
import torch

from generativemodels_b200 import _lib
from tests import attention_emulator as A
from tests import cpu_backend
from tests import elementwise_emulator as W
from tests import igemm_emulator as E
from tests import losses_backend
from tests import losses_emulator as LE
from tests import metrics_emulator as ME
from tests import norm_emulator as N
from tests import sa_solver_backend
from tests import unipc_backend

PASSTHROUGH = {"b200_sm_count", "b200_igemm_split_workspace_bytes", "b200_attention_flash_workspace_bytes",
               "b200_groupnorm_workspace_bytes", "b200_igemm_plan", "b200_version", "b200_act_dtype",
               "b200_device_check", "b200_last_error_string", "b200_abi_sizeof", "b200_ssim_workspace_bytes",
               "b200_mmd_workspace_bytes", "b200_frechet_workspace_bytes"}
ARGTYPES = {**_lib.SIGNATURES, **_lib.METRIC_SIGNATURES, **_lib.FID_SIGNATURES, **_lib.PERCEPTUAL_SIGNATURES,
            **_lib.LOSS_SIGNATURES, **_lib.SAMPLER_SIGNATURES}
GN_PARTIAL_REL = 2e-4          # GroupNorm partial sums vs the kernel's own output (test_igemm_contract_gpu.py)
SOFTMAX_SUM_REL = 1e-5         # softmax partial sums vs the kernel's own rows (test_igemm_contract_gpu.py)
_SIGNED = {1: torch.int8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


class StandIn(losses_backend.LossesFakeLib, unipc_backend.UniPCFakeLib, sa_solver_backend.SASolverFakeLib):
    """The CPU stand-in of every entry point: the network, metric, FID, perceptual and loss stand-ins, and the
    three sampler steps' (DPM-Solver++, UniPC, SA-Solver)."""


def _excess(got, want, tol):
    """|got - want| / tol elementwise (torch, float64); equal values (NaN included) are 0, other non-finite ones inf."""
    same = (got == want) | (torch.isnan(got) & torch.isnan(want))
    ratio = ((got - want).abs() / tol).nan_to_num(math.inf, math.inf)
    return torch.where(same, torch.zeros_like(ratio), ratio)


# ----------------------------------------------------------------------------------------------------------------
# memory maps: where a pointer's bytes live, and how to copy them to the host
# ----------------------------------------------------------------------------------------------------------------
class _CudaArray:
    def __init__(self, addr, size):
        self.__cuda_array_interface__ = {"shape": (size,), "typestr": "|u1", "data": (addr, False), "version": 3}


class DeviceMemory:
    """Segments of PyTorch's CUDA caching allocator on the current device (torch.cuda.memory_snapshot()), cached and
    re-read whenever the allocator has created or released a segment since, or a pointer is not found."""

    def __init__(self):
        self._key, self._bases, self._sizes = None, [], []

    def _refresh(self):
        dev = torch.cuda.current_device()
        segs = sorted((s["address"], s["total_size"]) for s in torch.cuda.memory_snapshot() if s["device"] == dev)
        self._bases, self._sizes = [b for b, _ in segs], [s for _, s in segs]

    def _lookup(self, ptr):
        i = bisect.bisect_right(self._bases, ptr) - 1
        if i >= 0 and ptr < self._bases[i] + self._sizes[i]:
            return self._bases[i], self._sizes[i]
        return None

    def find(self, ptr):
        st = torch.cuda.memory_stats()
        key = (st.get("segment.all.allocated", 0), st.get("segment.all.freed", 0))
        if key != self._key:
            self._key = key
            self._refresh()
        hit = self._lookup(ptr)
        if hit is None:
            self._refresh()
            hit = self._lookup(ptr)
        return hit

    def sync(self):
        torch.cuda.synchronize()

    def read(self, base, size):
        t = torch.as_tensor(_CudaArray(base, size), device="cuda")
        assert t.data_ptr() == base, "the segment view does not start at the segment"
        return t.cpu()


class HostMemory:
    """Host tensors standing in for allocator segments (the harness's own CPU test)."""

    def __init__(self, tensors):
        segs = sorted((t.data_ptr(), t.numel() * t.element_size()) for t in tensors)
        self._bases, self._sizes = [b for b, _ in segs], [s for _, s in segs]
        self._keep = list(tensors)

    def find(self, ptr):
        i = bisect.bisect_right(self._bases, ptr) - 1
        if i >= 0 and ptr < self._bases[i] + self._sizes[i]:
            return self._bases[i], self._sizes[i]
        return None

    def sync(self):
        pass

    def read(self, base, size):
        return torch.from_numpy(np.ctypeslib.as_array(C.cast(base, C.POINTER(C.c_uint8)), shape=(size,))).clone()


# ----------------------------------------------------------------------------------------------------------------
# pointers of a call
# ----------------------------------------------------------------------------------------------------------------
def _obj(a):
    return a._obj if hasattr(a, "_obj") else a


def _is_ptr_array(a):
    return isinstance(a, C.Array) and a._type_ is C.c_void_p


def _struct_ptr_fields(s):
    """(name, index or None) of every c_void_p field and c_void_p array element of a ctypes struct."""
    out = []
    for name, typ in s._fields_:
        if typ is C.c_void_p:
            out.append((name, None))
        elif isinstance(typ, type) and issubclass(typ, C.Array) and typ._type_ is C.c_void_p:
            out.extend((name, i) for i in range(typ._length_))
    return out


def pointers(args, argtypes):
    """Every nonzero device pointer the arguments carry (the last argument, the stream, excluded)."""
    found = []
    for a, at in zip(args[:-1], argtypes):
        o = _obj(a)
        if isinstance(o, C.Structure):
            for name, i in _struct_ptr_fields(o):
                v = getattr(o, name) if i is None else getattr(o, name)[i]
                if v:
                    found.append(int(v))
        elif _is_ptr_array(o):
            found.extend(int(v) for v in o if v)
        elif at is C.c_void_p and isinstance(o, int) and o:
            found.append(o)
    return found


def translate(args, argtypes, tr):
    """The arguments with every pointer p replaced by tr(p): structs and pointer arrays are cloned, never mutated."""
    out = []
    for k, a in enumerate(args):
        o = _obj(a)
        if k == len(args) - 1:
            out.append(a)
        elif isinstance(o, C.Structure):
            c = type(o).from_buffer_copy(o)
            for name, i in _struct_ptr_fields(c):
                v = getattr(c, name) if i is None else getattr(c, name)[i]
                if v:
                    if i is None:
                        setattr(c, name, tr(int(v)))
                    else:
                        getattr(c, name)[i] = tr(int(v))
            out.append(C.byref(c))
        elif _is_ptr_array(o):
            out.append(type(o)(*[tr(int(v)) if v else None for v in o]))
        elif argtypes[k] is C.c_void_p and isinstance(o, int) and o:
            out.append(tr(o))
        else:
            out.append(a)
    return out


def signature(name, args):
    """A compact, hashable description of the call's shape: scalar arguments and scalar struct fields."""
    parts = []
    for a, at in zip(args[:-1], ARGTYPES[name]):
        o = _obj(a)
        if isinstance(o, C.Structure):
            if isinstance(o, _lib.IgemmParams):
                parts.append(("N", o.in_N, "in", (o.in_D, o.in_H, o.in_W), "out", (o.out_D, o.out_H, o.out_W),
                              "aC", tuple(o.a_C), "pitch", tuple(o.a_pitch), "cout", o.cout, "cols", o.out_cols,
                              "n_seg", o.n_seg, "dt", o.out_dtype, "act", (o.act1, o.act2), "res", bool(o.res_ptr),
                              "gn", o.gn_group if o.gn_partial else 0, "stat", bool(o.stat_ptr), "impl", o.impl))
                continue
            ptr = {n for n, _ in _struct_ptr_fields(o)}
            for n, typ in o._fields_:
                if n in ptr:
                    continue
                v = getattr(o, n)
                parts.append((n, tuple(v) if isinstance(v, C.Array) else v))
        elif isinstance(o, C.Array):
            if not _is_ptr_array(o) and not issubclass(o._type_, C.Structure):
                parts.append(tuple(o))
        elif isinstance(o, (int, float)) and at is not C.c_void_p:
            parts.append(o)
    return (name, tuple(parts))


# ----------------------------------------------------------------------------------------------------------------
# the igemm store path (tests/test_igemm_contract_gpu.py's docstring; generativemodels_b200/csrc/igemm.cu)
# ----------------------------------------------------------------------------------------------------------------
def igemm_path(p, plan):
    bn, splits = plan
    if bn == 256:
        return "wide"
    if splits > 1:
        return "split"
    if p.act1 == _lib.ACT_GEGLU:
        return "geglu"
    g = 8 if p.out_dtype == _lib.DT_H16 else 4
    vec = lambda cols, *s, ptr: cols % g == 0 and all(x % g == 0 for x in s) and ptr % 16 == 0
    out_vec = vec(p.out_cols, p.out_sN, p.out_sD, p.out_sH, p.out_sW, ptr=p.out_ptr or 0)
    if not out_vec:
        return "general scalar"
    esz = 2 if p.out_dtype == _lib.DT_H16 else 4
    staged = p.out_dtype == _lib.DT_F32 and p.out_sW * esz > 2048
    # the residual's vector width is its own dtype's: an h16 residual needs multiples of 8 (igemm.cu, res_vec)
    rvec = lambda cols, *s, ptr: cols % 8 == 0 and all(x % 8 == 0 for x in s) and ptr % 16 == 0
    res_vec = (not p.res_ptr) or (p.res_dtype == _lib.DT_H16 and rvec(p.out_cols, p.res_sN, p.res_sD, p.res_sH,
                                                                       p.res_sW, ptr=p.res_ptr))
    fast = not staged and not p.stat_ptr and res_vec
    if staged:
        return "staged"
    if not fast:
        return "general vector"
    lean = (p.act1 == p.act2 == _lib.ACT_NONE and p.scale == 1.0 and not p.row_bias and not p.gn_partial
            and p.out_dtype == _lib.DT_H16)
    return "lean" if lean else "fast"


# ----------------------------------------------------------------------------------------------------------------
# the scheduler and inferer paths (generativemodels_b200/csrc/{samplers,elementwise}.cu)
# ----------------------------------------------------------------------------------------------------------------
def _vec_kind(ptrs, n):
    """The step kernels' access path: 'scalar' (VEC = 0) unless every pointer the entry point ORs into its alignment
    test is 16-byte aligned; then 'vec', or 'tail' when n % 4 elements are left to the scalar tail."""
    if any((p or 0) % 16 for p in ptrs):
        return "scalar"
    return "vec" if n % 4 == 0 else "tail"


def step_paths(name, o):
    """Path labels of one call of a scheduler / inferer entry point from its arguments `o` (the ctypes objects),
    with the kernel-selection predicates of the entry point; () for other entry points."""
    def hist(arr, nh):
        return [int(arr[k] or 0) for k in range(nh)]
    if name == "b200_dpm_solver_step":
        m, s, h, nh, z, c, prev, x0, n = o[:9]
        return (f"dpm nh{nh}" + (" noise" if z else ""),
                "dpm step " + _vec_kind([m, s, *hist(h, nh), z, prev, x0], n))
    if name == "b200_unipc_step":
        m, s, last, h, nh, c, prev, x0, xc, n = o[:10]
        return (f"unipc nh{nh}" + (" last" if last else ""),
                "unipc step " + _vec_kind([m, s, last, *hist(h, nh), prev, x0, xc], n))
    if name == "b200_sa_solver_step":
        m, s, last, zl, h, nh, z, c, prev, x0, xc, n = o[:12]
        zl = zl if last else None                       # the kernel reads last_noise only with last
        return (f"sa nh{nh}" + (" last" if last else "") + (" zl" if zl else "") + (" z" if z else ""),
                "sa step " + _vec_kind([m, s, last, zl, *hist(h, nh), z, prev, x0, xc], n))
    if name == "b200_ddim_step":
        m, s, z, c, prev, x0, n = o[:7]
        return ("ddim" + (" noise" if z else ""), "ddim step " + _vec_kind([m, s, z, prev, x0], n))
    if name == "b200_ddpm_step":
        z, c = o[2], o[4]
        return (f"ddpm var{c.var_mode}" if z else "ddpm no noise",)      # var_mode is read only with noise
    if name == "b200_pndm_step":
        return (f"pndm nh{o[2].n_hist}",)
    if name == "b200_ddpm_kl":
        return ("ddpm_kl t0" if o[3].is_t0 else "ddpm_kl t",)
    if name == "b200_add_noise":
        return ("add_noise +" if o[4] > 0 else "add_noise -",)
    if name == "b200_scale_f32":
        return ("scale div" if o[2] != 1.0 else "scale mul",)
    return ()


# ----------------------------------------------------------------------------------------------------------------
# the proxy
# ----------------------------------------------------------------------------------------------------------------
@dataclass
class Call:
    name: str
    sig: tuple
    excess: float
    paths: tuple = ()


@dataclass
class Shadow:
    real: object
    memory: object
    stand_in: object = field(default_factory=StandIn)
    calls: list = field(default_factory=list)
    violations: list = field(default_factory=list)

    def __getattr__(self, name):
        if not name.startswith("b200_"):
            raise AttributeError(name)
        if name in PASSTHROUGH:
            return getattr(self.real, name)
        if name not in ARGTYPES or not hasattr(self.stand_in, name):
            raise AssertionError(f"{name}: neither a host query nor an entry point of the CPU stand-in")
        return lambda *args: self.call(name, args)

    # -- one call --------------------------------------------------------------------------------------------
    def call(self, name, args):
        segs = {}
        for p in pointers(args, ARGTYPES[name]):
            hit = self.memory.find(p)
            if hit is None:
                raise AssertionError(f"{name}: pointer {p:#x} lies in no allocator segment")
            segs[hit[0]] = hit[1]
        self.memory.sync()
        pre = {b: self.memory.read(b, s) for b, s in segs.items()}
        rc = getattr(self.real, name)(*args)
        self.memory.sync()
        post = {b: self.memory.read(b, s) for b, s in segs.items()}
        if rc != 0:
            return rc
        emu = {b: t.clone() for b, t in pre.items()}
        ctx = _Compare(name, args, segs, pre, post, emu, self)
        ctx.run()
        self.calls.append(Call(name, signature(name, args), ctx.worst, tuple(ctx.paths)))
        return rc

    # -- summary -----------------------------------------------------------------------------------------------
    def paths(self):
        return {p for c in self.calls for p in c.paths} | {c.name for c in self.calls}

    def table(self):
        rows = defaultdict(lambda: [0, set(), 0.0, None])
        for c in self.calls:
            r = rows[c.name]
            r[0] += 1
            r[1].add(c.sig)
            if c.excess >= r[2]:
                r[2], r[3] = c.excess, c.sig
        lines = [f"{'entry':34s} {'calls':>6s} {'shapes':>6s} {'worst excess':>12s}  worst call"]
        for n in sorted(rows):
            k, sigs, ex, sig = rows[n]
            lines.append(f"{n:34s} {k:6d} {len(sigs):6d} {ex:12.3g}  {str(sig[1])[:150]}")
        ig = defaultdict(int)
        for c in self.calls:
            for p in c.paths:
                ig[p] += 1
        lines.append("paths: " + ", ".join(f"{p} x{k}" for p, k in sorted(ig.items())))
        return "\n".join(lines)

    def report(self):
        return "\n".join(self.violations[:20]) + "\n" + self.table()


class _Compare:
    """The emulation and comparison of one call (steps 4 to 6 of the module docstring)."""

    def __init__(self, name, args, segs, pre, post, emu, shadow):
        self.name, self.args, self.segs, self.pre, self.post, self.emu = name, args, segs, pre, post, emu
        self.sh = shadow
        self.worst = 0.0
        self.paths = []
        self.voxels = None
        self.slot_sums = None
        self.mask = {b: torch.zeros(s, dtype=torch.bool) for b, s in segs.items()}
        self.host = {b: t.data_ptr() for b, t in emu.items()}
        self.pre_host = {b: t.data_ptr() for b, t in pre.items()}

    def seg_of(self, ptr):
        for b, s in self.segs.items():
            if b <= ptr < b + s:
                return b
        raise AssertionError(f"{self.name}: {ptr:#x} outside the call's segments")

    def to_emu(self, ptr):
        b = self.seg_of(ptr)
        return self.host[b] + (ptr - b)

    def to_pre(self, ptr):
        b = self.seg_of(ptr)
        return self.pre_host[b] + (ptr - b)

    def fail(self, msg):
        self.sh.violations.append(f"{self.name} {signature(self.name, self.args)[1]}: {msg}")

    def note(self, ex, what):
        ex = float(ex)
        if not ex <= self.worst:
            self.worst = ex if not math.isnan(ex) else math.inf
        if not ex <= 1.0:
            self.fail(f"{what}: excess {ex:.3g}")

    def mark(self, dev_ptr, nbytes):
        b = self.seg_of(dev_ptr)
        self.mask[b][dev_ptr - b:dev_ptr - b + nbytes] = True

    # -- views of the emulation copy and the device's bytes ------------------------------------------------------
    def _emu_seg(self, view):
        p = view.data_ptr()
        for b, h in self.host.items():
            if h <= p < h + self.segs[b]:
                return b
        raise AssertionError(f"{self.name}: the stand-in stored outside the call's segments")

    def device_view(self, view, which="post"):
        b = self._emu_seg(view)
        es = view.element_size()
        off = view.data_ptr() - self.host[b]
        assert off % es == 0
        src = (self.post if which == "post" else self.pre)[b]
        return torch.as_strided(src.view(view.dtype), view.shape, view.stride(), off // es)

    def mark_view(self, view):
        b = self._emu_seg(view)
        es = view.element_size()
        off = view.data_ptr() - self.host[b]
        m = torch.zeros(self.segs[b], dtype=torch.uint8)
        torch.as_strided(m.view(_SIGNED[es]), view.shape, view.stride(), off // es).fill_(-1)
        self.mask[b] |= m.bool()

    # -- steps 4 to 6 --------------------------------------------------------------------------------------------
    def run(self):
        records = []
        fake_args = translate(self.args, ARGTYPES[self.name], self.to_emu)
        cpu_backend.RECORDER = lambda view, r: records.append((view, r))
        try:
            if self.name == "b200_igemm":      # the stand-in's emulate, on a deterministic subset of a large call's rows
                self.voxels = E.sample_voxels(_obj(self.args[0]))
                E.emulate(_obj(fake_args[0]), self.voxels)
            else:
                getattr(self.sh.stand_in, self.name)(*fake_args)
        finally:
            cpu_backend.RECORDER = None
        for view, r in records:
            self.mark_view(view)
            got = self.device_view(view)
            if isinstance(r, ME.SlotSums):         # compared summed per item, in entry_specific
                self.slot_sums = r
                continue
            if isinstance(r, N.Affine):
                ex = N.affine_excess(r, got)
            elif isinstance(r, LE.Spectra):
                ex = LE.norm_excess(r, got.reshape(r.out.shape))
            else:
                got = got.reshape(r.out.shape)
                fam = W if isinstance(r, W.Result) else N if isinstance(r, N.Result) else A
                assert isinstance(r, (W.Result, N.Result, A.Result)), type(r)
                ex = fam.excess(r, got)
            self.note(ex.max() if ex.numel() else 0.0, f"stored values ({tuple(view.shape)})")
        self.entry_specific()
        for b in self.segs:
            stand = (self.emu[b] != self.pre[b]) & ~self.mask[b]
            if stand.any():
                raise AssertionError(f"{self.name}: the stand-in changed {int(stand.sum())} bytes it did not report")
            dev = (self.post[b] != self.pre[b]) & ~self.mask[b]
            if dev.any():
                i = int(torch.nonzero(dev)[0])
                self.fail(f"{int(dev.sum())} bytes changed outside the outputs, first at segment offset {i}")

    def entry_specific(self):
        o = [_obj(a) for a in self.args]
        self.paths += step_paths(self.name, o)
        if self.name == "b200_igemm":
            self.igemm(o[0])
        elif self.name == "b200_attention_flash":
            a = o[0]
            self.paths.append(f"flash dh{a.dh}")
            if a.workspace:
                self.mark(a.workspace, a.workspace_bytes)
        elif self.name == "b200_ssim":
            self.ssim_slots(o[0])
        elif self.name == "b200_mmd":
            self.mark(o[7], int(self.sh.real.b200_mmd_workspace_bytes(o[6])))
        elif self.name == "b200_frechet":
            self.mark(o[0].workspace, int(self.sh.real.b200_frechet_workspace_bytes(o[0].F)))
        elif self.name == "b200_spectral_distance":
            if o[6]:
                self.mark(o[6], _lib.SPECTRAL_PARTIALS * 8)
        elif self.name == "b200_adversarial":
            self.mark(o[9], _lib.ADV_PARTIALS * 8)
        elif self.name == "b200_perceptual_distance" and o[9]:
            image, image32 = (self.f64_at(o[8], o[3]), self.post_at(o[9], o[3], torch.float32))
            if not torch.equal(image.float().view(torch.int32), image32.view(torch.int32)):
                self.note(math.inf, "image32 is not the fp32 rounding of the kernel's own image")
        elif self.name in ("b200_groupnorm_stats", "b200_groupnorm_fused", "b200_groupnorm_from_partials_ex"):
            p = o[0]
            if p.partial:
                Ct = p.x_C[0] + (p.x_C[1] if p.x_ptr[1] else 0)
                self.mark(p.partial, int(self.sh.real.b200_groupnorm_workspace_bytes(p.N, p.spatial, Ct)))
            if self.name == "b200_groupnorm_from_partials_ex":
                for i in range(2):
                    if o[1][i]:
                        self.paths.append(f"gn_from_partials gw{(o[3][i] or 8) if o[3] is not None else 8}")

    def post_at(self, ptr, count, dtype):
        b = self.seg_of(ptr)
        es = torch.empty((), dtype=dtype).element_size()
        assert (ptr - b) % es == 0
        return self.post[b].view(dtype)[(ptr - b) // es:(ptr - b) // es + count]

    def f64_at(self, ptr, count):
        return self.post_at(ptr, count, torch.float64)

    def ssim_slots(self, p):
        """The partial slots of b200_ssim, whose layout is the device's own: per item, the sum over its slots against
        the float64 sum of the kernel's own stored maps (within fp64 summation error) and against the reading's sum
        (within the sum of the per-voxel bounds, metrics_emulator.slot_sums)."""
        nbytes = int(self.sh.real.b200_ssim_workspace_bytes(C.byref(p)))
        slots = nbytes // (16 * p.N)
        self.mark(p.partials, nbytes)
        dev = self.f64_at(p.partials, p.N * slots * 2).view(p.N, slots, 2).sum(1)
        r = self.slot_sums
        self.note(_excess(dev, r.exact, r.err).max(), "SSIM partial slots vs the reading's sums")
        count = p.C * (p.D - p.kd + 1) * (p.H - p.kh + 1) * (p.W - p.kw + 1)
        for k, ptr in enumerate((p.ssim_map, p.cs_map)):
            if ptr:
                own = self.post_at(ptr, p.N * count, torch.float32).double().view(p.N, count)
                tol = (count + slots + 2) * ME.E53 * own.abs().sum(1)
                self.note(_excess(dev[:, k], own.sum(1), tol).max(), "SSIM partial slots vs the kernel's own map")

    def igemm(self, p):
        nsm = int(self.sh.real.b200_sm_count())
        plan = (C.c_int32 * 4)()
        assert self.sh.real.b200_igemm_plan(C.byref(p), nsm, int(bool(p.split_ws)), plan) == 0
        bn, splits = int(plan[0]), int(plan[1])
        self.paths += [f"igemm bn{bn}", f"igemm {igemm_path(p, (bn, splits))}"]
        if p.split_ws:
            self.mark(p.split_ws, p.split_ws_bytes)
        h16 = p.out_dtype == _lib.DT_H16
        dt, es = (torch.int16, 2) if h16 else (torch.int32, 4)
        idx = torch.from_numpy(E.footprint(p))
        b = self.seg_of(p.out_ptr)
        off = p.out_ptr - b
        assert off % es == 0
        flat = idx + off // es
        fl = (lambda t: t.view(torch.float16 if E.ACT_DTYPE == "fp16" else torch.bfloat16)) if h16 else \
            (lambda t: t.view(torch.float32))
        got = fl(self.post[b].view(dt)[flat]).double().numpy()
        want = fl(self.emu[b].view(dt)[flat]).double().numpy()
        m = torch.zeros(self.segs[b] // es, dtype=torch.bool)
        m[flat.reshape(-1)] = True
        self.mask[b] |= m.view(-1, 1).expand(-1, es).reshape(-1) if es > 1 else m
        cv = p.cout // 2 if p.act1 == _lib.ACT_GEGLU else p.cout
        if cv < p.out_cols and (self.post[b].view(dt)[flat[..., cv:]] != 0).any():
            self.fail("padding columns are not +0")
            self.note(math.inf, "padding columns")
        hp = _lib.IgemmParams.from_buffer_copy(translate([C.byref(p), None], ARGTYPES["b200_igemm"],
                                                         self.to_pre)[0]._obj)
        gs, ws = got, want
        if self.voxels is not None:
            self.paths.append("igemm sampled rows")
            gs, ws = (x.reshape(p.out_N, -1, p.out_cols)[:, self.voxels] for x in (got, want))
        tol = E.bound(hp, gs, ws, voxels=self.voxels)
        same = (gs == ws) | (np.isnan(gs) & np.isnan(ws))
        ratio = np.where(same, 0.0, np.abs(gs - ws) / tol)
        ratio = np.where(np.isfinite(ratio), ratio, np.inf)
        self.note(ratio.max() if ratio.size else 0.0, "igemm output")
        if p.gn_partial:
            self.paths.append(f"igemm gn{p.gn_group or 8}")
            gw = p.gn_group or 8
            cnt = p.out_N * p.gn_slots * (p.cout // gw) * 2
            self.mark(p.gn_partial, cnt * 4)
            gb = self.seg_of(p.gn_partial)
            go = (p.gn_partial - gb) // 4
            shape = (p.out_N, p.gn_slots, p.cout // gw, 2)
            gsum = self.post[gb].view(torch.float32)[go:go + cnt].view(shape).double().sum(1).numpy()
            psum = self.pre[gb].view(torch.float32)[go:go + cnt].view(shape).double().sum(1).numpy()
            own = got[..., :p.cout].reshape(p.out_N, -1, p.cout // gw, gw)
            wantp = psum + np.stack([own.sum((1, 3)), (own * own).sum((1, 3))], -1)
            size = np.stack([np.abs(own).sum((1, 3)), (own * own).sum((1, 3))], -1) + 1 + np.abs(psum)
            r = np.abs(gsum - wantp) / size / GN_PARTIAL_REL
            self.note(np.nan_to_num(r, nan=np.inf).max(), "GroupNorm partial sums vs the kernel's own output")
        if p.stat_ptr:
            self.paths.append("igemm stat")
            cols, nt = p.out_cols, (p.out_cols + 127) // 128
            cnt = p.out_W * nt * 2
            self.mark(p.stat_ptr, cnt * 4)
            sb = self.seg_of(p.stat_ptr)
            so = (p.stat_ptr - sb) // 4
            st = self.post[sb].view(torch.float32)[so:so + cnt].view(p.out_W, nt, 2).double().numpy()
            rows = got.reshape(p.out_W, cols)
            worst = 0.0
            for t in range(nt):
                seg = rows[:, t * 128:min((t + 1) * 128, p.cout)]
                if seg.shape[1] == 0:
                    ok = (st[:, t, 0] == -np.inf).all() and (st[:, t, 1] == 0).all()
                    worst = max(worst, 0.0 if ok else math.inf)
                    continue
                mx = seg.max(1)
                if not (st[:, t, 0] == mx).all():
                    worst = math.inf
                s = np.exp(seg - mx[:, None]).sum(1)
                worst = max(worst, float(np.nan_to_num(np.abs(st[:, t, 1] - s) / (SOFTMAX_SUM_REL * s),
                                                       nan=np.inf).max()))
            self.note(worst, "softmax partials vs the kernel's own rows")


@contextlib.contextmanager
def shadow(monkeypatch, memory=None, real=None, stand_in=None):
    """Route every C-ABI call of the product through a Shadow of the real library (or `real`) over `memory`
    (default: the CUDA caching allocator's segments)."""
    sh = Shadow(real if real is not None else _lib.require_device(), memory if memory is not None else DeviceMemory(),
                **({"stand_in": stand_in} if stand_in is not None else {}))
    old = _lib.require_device
    monkeypatch.setattr(_lib, "require_device", lambda: sh)
    try:
        yield sh
    finally:
        monkeypatch.setattr(_lib, "require_device", old)
