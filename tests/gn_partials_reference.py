"""Float64 reference for GroupNorm fed by the partial sums of b200_igemm's epilogue (test infrastructure; the tensors may
live on the CPU or the GPU).

The chain: a convolution stores its h16 output and adds (sum, sum of squares) of the stored values per producer group
(gn_group = 4 or 8 channels) into private fp32 slots, one per epilogue warp of each persistent CTA; ops.groupnorm_affine
then folds the slots in fp64 with b200_groupnorm_from_partials_ex into the [N, C, 2] affine table.  `check` holds the
library's table and slot buffers to three bars (each a ratio, > 1 fails):

  contract  the header's from-partials accuracy.  Every slot is an fp32 sum of at most T terms, T = (work items per
            slot) x 32 rows x gn_group, from the launch's tile plan (work_per_slot).  With u = 2^-24, e = T u and s =
            sqrt(var + eps), the sums carry |d sum| <= e sum |x| and |d sumsq| <= e sum x^2, so
                |d mean| <= e (|mean| + s),  |d var| <= e (mean^2 + var) + 2 |mean| d_mean + d_mean^2,
                |d rstd| <= rstd |d var| / s^2
            -- about (mean / s)^2 T 2^-24, as include/b200gen.h states.
  product   the bound b200_groupnorm_stats is held to (norm_emulator.stats_affine: 2^-12 against the group's pivot).
  totals    the slot totals against the float64 sums of the STORED values per producer group, within the rounding
            depth of the epilogue's order of summation: a tree over the group's channels and a tile's 32 rows of the
            slot, then one fp32 add per work item and at most two per flush (8 + 3 x work items per slot roundings of
            any term).  A producer that sums its fp32 accumulators instead of the rounded stores fails it where the
            16-bit rounding errors of a group add up to more than that (small groups, or a biased rounding).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import torch

from generativemodels_b200 import _lib, ops
from tests import norm_emulator as N

F64 = torch.float64
U = 2.0 ** -24
ROWS_PER_SLOT = 32      # rows of a work item one slot receives: a warp's 32 rows of a 128-row tile (128-column kernel),
                        # 16 rows from each of the two consumers of a 128-row CTA half (two-CTA kernel)


def work_per_slot(p, sm_count: int) -> int:
    """Work items one slot sums, at most: b200_igemm_plan's items over the persistent CTAs (128-column kernel: one per
    SM up to the item count) or clusters (two-CTA kernel: counted as a quarter of the SM count, since how many clusters
    are co-resident is a device query; at least half the SM pairs hold one)."""
    out = (C.c_int32 * 4)()
    q = _lib.IgemmParams.from_buffer_copy(p)
    rc = _lib.load().b200_igemm_plan(C.byref(q), sm_count, 0, out)
    assert rc == 0, "b200_igemm_plan rejected a parameter block b200_igemm ran"
    items = int(out[2])
    workers = min(items, max(1, sm_count // 4) if out[0] == 256 else sm_count)
    return -(-items // workers)


class Producers:
    """Wraps ops.igemm_raw (context manager) to record, per GroupNorm partial buffer, the most work items any of its
    slots receives over the launches that write it (conv_upsample2x: one launch per phase, each on its own slots)."""

    def __init__(self, sm_count: int):
        self.sm_count = sm_count
        self.wps: dict[int, int] = {}

    def __enter__(self):
        self._orig = ops.igemm_raw

        def wrapped(p, *a, **k):
            if p.gn_partial:
                key, w = int(p.gn_partial), work_per_slot(p, self.sm_count)
                self.wps[key] = w if p.gn_slot0 == 0 else max(w, self.wps.get(key, 0))
            return self._orig(p, *a, **k)
        ops.igemm_raw = wrapped
        return self

    def __exit__(self, *exc):
        ops.igemm_raw = self._orig
        return False

    def of(self, a: ops.CL) -> int:
        return self.wps[a.gn.data_ptr()]


def takes_partials(srcs, groups) -> bool:
    """ops.groupnorm_affine's rule for reading the producers' partials instead of running the statistics pass."""
    cpg = sum(a.C for a in srcs) // groups
    return (ops._GN_FUSE and all(a.gn is not None for a in srcs) and all(cpg % ops._gn_group(a) == 0 for a in srcs)
            and srcs[0].C % cpg == 0)


@dataclass
class Moments:
    mean: torch.Tensor        # [N, groups] float64, over the virtual concat of the sources
    var: torch.Tensor
    piv: torch.Tensor
    prod: list = field(default_factory=list)   # per source: [N, C / gn_group, 3] float64 (sum, sum of squares, sum |x|)


def _voxels(a: ops.CL):
    return a.t.view(a.N, a.spatial, a.pitch)[..., :a.C]


def moments(srcs, groups, chunk=1 << 25) -> Moments:
    """Two float64 passes over the stored h16 values in chunks of voxels (a full-size C3 tensor is 1.5 G values)."""
    cpg = sum(a.C for a in srcs) // groups
    means, vars_, pivs, prod = [], [], [], []
    for a in srcs:
        gw = ops._gn_group(a) if a.gn is not None else cpg
        x = _voxels(a)
        step = max(1, chunk // a.C)
        P = torch.zeros(a.N, a.C // gw, 3, dtype=F64, device=x.device)
        for s0 in range(0, a.spatial, step):
            v = x[:, s0:s0 + step].to(F64).reshape(a.N, -1, a.C // gw, gw)
            P[..., 0] += v.sum((1, 3))
            P[..., 1] += (v * v).sum((1, 3))
            P[..., 2] += v.abs().sum((1, 3))
        mean = P[..., 0].reshape(a.N, a.C // cpg, -1).sum(-1) / (a.spatial * cpg)
        m2 = torch.zeros_like(mean)
        for s0 in range(0, a.spatial, step):
            v = x[:, s0:s0 + step].to(F64).reshape(a.N, -1, a.C // cpg, cpg)
            m2 += ((v - mean[:, None, :, None]) ** 2).sum((1, 3))
        means.append(mean)
        vars_.append(m2 / (a.spatial * cpg))
        pivs.append(x[:, 0].to(F64).reshape(a.N, a.C // cpg, cpg)[..., 0])
        prod.append(P)
    return Moments(torch.cat(means, 1), torch.cat(vars_, 1), torch.cat(pivs, 1), prod)


def contract_affine(m: Moments, terms, eps, gamma, beta, groups):
    """The table's accuracy under the header's from-partials note; terms [groups]: T of the source each group lies in."""
    mean, var = m.mean, m.var
    s2 = var + eps
    s, rstd = torch.sqrt(s2), 1.0 / torch.sqrt(s2)
    e = terms[None] * U * (1 + 1e-3) + N.STAT_PARTIALS
    d_mean = e * (mean.abs() + s)
    d_var = e * (mean ** 2 + var) + 2 * mean.abs() * d_mean + d_mean ** 2
    return N.affine_table(mean, rstd, d_mean, rstd * d_var / s2, gamma, beta, groups)


@dataclass
class Report:
    k: float                  # largest |mean| / std over the (sample, group)s
    contract: float           # largest err / tol of each bar
    product: float
    totals: float
    work_per_slot: int        # largest over the sources
    terms: int                # largest T


def check(srcs, groups, eps, gamma, beta, table, wps) -> Report:
    """Ratios of the library's affine table [N, C, 2] and the sources' partial buffers against the float64 reference
    of the stored values; wps[i]: work items per slot of source i (Producers.of)."""
    srcs = [srcs] if isinstance(srcs, ops.CL) else list(srcs)
    dev = srcs[0].t.device
    Ct = sum(a.C for a in srcs)
    cpg = Ct // groups
    gamma = torch.ones(Ct, device=dev) if gamma is None else gamma
    beta = torch.zeros(Ct, device=dev) if beta is None else beta
    m = moments(srcs, groups)
    terms = torch.cat([torch.full((a.C // cpg,), float(w * ROWS_PER_SLOT * ops._gn_group(a)), dtype=F64, device=dev)
                       for a, w in zip(srcs, wps)])
    got = table.view(srcs[0].N, Ct, 2)
    contract = N.affine_excess(contract_affine(m, terms, eps, gamma, beta, groups), got)
    product = N.affine_excess(N.stats_affine(m.mean, m.var, m.piv, eps, gamma, beta, groups), got)
    totals = 0.0
    for a, w, P in zip(srcs, wps, m.prod):
        tot = a.gn.to(F64).sum(1)                                   # [N, C / gw, 2]
        e = (8 + 3 * w) * U * (1 + 1e-3)
        rs = (tot[..., 0] - P[..., 0]).abs() / (e * P[..., 2] + 1e-300)
        rq = (tot[..., 1] - P[..., 1]).abs() / (e * P[..., 1] + 1e-300)
        totals = max(totals, float(torch.maximum(rs, rq).max()))
    k = float((m.mean.abs() / torch.sqrt(m.var + eps)).max())
    return Report(k, float(contract.max()), float(product.max()), totals, max(wps), int(terms.max()))


def fmt(r: Report) -> str:
    return (f"k {r.k:7.2f}  work/slot {r.work_per_slot:4d}  T {r.terms:7d}  err/tol contract {r.contract:.3g}  "
            f"product {r.product:.3g}  totals {r.totals:.3g}")
