"""tests/norm_emulator.py against float64 PyTorch, and its bound against kernel-shaped mutants (CPU only).

The emulator has to agree with F.group_norm / F.layer_norm / F.interpolate(mode="nearest") in float64 to within its
own bound, and that bound has to be narrow enough to reject the mistakes a normalisation kernel makes: an unbiased
variance, eps outside the square root, a voxel per chunk dropped, the second source normalised with the first source's
statistics, the two LeakyReLU slopes swapped, SPADE's gamma and beta halves swapped, a partial slot read off by one,
a pad channel left unwritten, the exact-rational nearest index, and E[x^2] - mean^2 from fp32 sums at a large offset.
Each mutant prints its excess factor (max err / tol) in both storage flavours.
"""
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import norm_emulator as E
from tests import rescaler_oracle as R

F64 = torch.float64
FLAVOURS = [torch.float16, torch.bfloat16]
FL_IDS = ["fp16", "bf16"]
MARGIN = 4.0            # a mutant must leave the bound by at least this factor


def gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def torch_act(y, code):
    if code == E.ACT_SILU:
        return F.silu(y)
    if code in E.SLOPE:
        return F.leaky_relu(y, E.SLOPE[code])
    return y


class GN:
    """One GroupNorm operand set in the ABI layout: two sources (C0, C1 channels, pitches with pad), N samples."""

    def __init__(self, name, N, spatial, C0, C1, groups, eps=0.1, k=0.0, act=E.ACT_NONE, offset1=0.0):
        g = gen(name)
        self.N, self.S, self.C0, self.C1, self.groups, self.eps, self.act = N, spatial, C0, C1, groups, eps, act
        self.C = C0 + C1
        self.p0, self.p1, self.yp = C0 + 3, C1 + 5, self.C + 8
        X = torch.randn(N, spatial, self.C, generator=g, dtype=F64) + k
        X[..., C0:] += offset1
        self.gamma = (1 + 0.5 * torch.randn(self.C, generator=g)).float()
        self.beta = (0.5 * torch.randn(self.C, generator=g)).float()
        self.x0 = torch.full((N * spatial * self.p0,), math.nan, dtype=E.H16)
        self.x0.view(-1, self.p0)[:, :C0] = X.reshape(-1, self.C)[:, :C0].to(E.H16)
        self.x1 = torch.full((N * spatial * self.p1,), math.nan, dtype=E.H16)
        if C1:
            self.x1.view(-1, self.p1)[:, :C1] = X.reshape(-1, self.C)[:, C0:].to(E.H16)
        self.X = E.concat(self.x0, self.x1, C0, C1, self.p0, self.p1, N, spatial)

    def emulate(self):
        return E.groupnorm(self.x0, self.x1, self.C0, self.C1, self.p0, self.p1, self.N, self.S, self.groups,
                           self.eps, self.gamma, self.beta, self.act, self.yp)

    def store(self, y, pad=0.0):
        """[N, spatial, C] float64 -> output rows [N * spatial, y_pitch] as a kernel would store them."""
        out = torch.full((self.N * self.S, self.yp), pad, dtype=F64)
        out[:, :self.C] = E.h16(y.reshape(-1, self.C))
        return out

    def mutant(self, var_fn=None, rstd_fn=None, stat_x=None, stat_of=None, slope=None):
        """GroupNorm in float64 with one piece changed."""
        N, S, C, G = self.N, self.S, self.C, self.groups
        Xs = self.X if stat_x is None else stat_x
        Xg = Xs.reshape(N, -1, G, C // G)
        mean = Xg.mean((1, 3))
        var = ((Xg - mean[:, None, :, None]) ** 2).mean((1, 3))
        if var_fn:
            var = var_fn(var, Xg[0, :, 0].numel())
        rstd = rstd_fn(var, self.eps) if rstd_fn else 1 / torch.sqrt(var + self.eps)
        if stat_of is not None:
            mean, rstd = mean[:, stat_of], rstd[:, stat_of]
        ex = lambda t: t.repeat_interleave(C // G, 1)[:, None]
        y = (self.X - ex(mean)) * ex(rstd) * self.gamma.double() + self.beta.double()
        if slope is not None:
            y = torch.where(y > 0, y, slope * y)
        else:
            y = torch_act(y, self.act)
        return self.store(y)


def report(name, flavour, r):
    print(f"\nMUTANT {name} {flavour} excess = {r:.1f}")


# ----------------------------------------------------------------------------------------------------------------
# the emulator against float64 PyTorch
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
@pytest.mark.parametrize("k", [0, 10, 100, 256])
@pytest.mark.parametrize("act", [E.ACT_NONE, E.ACT_SILU, E.ACT_LEAKYRELU, E.ACT_LEAKYRELU02])
def test_groupnorm_emulator_matches_torch(dt, k, act):
    with E.storage(dt):
        c = GN(f"gn{k}{act}", 2, 37, 24, 8, 8, eps=1e-5, k=k, act=act)
        r, t = c.emulate()
        Xn = c.X.permute(0, 2, 1)                                        # [N, C, spatial]
        y = F.group_norm(Xn, c.groups, c.gamma.double(), c.beta.double(), c.eps).permute(0, 2, 1)
        want = c.store(torch_act(y, act))
        assert E.excess(r, want).max() <= 1
        assert (r.out[:, c.C:] == 0).all()
        # the affine table: a ~ rstd gamma, b ~ beta - mean a against torch's own moments
        var, mean = torch.var_mean(Xn.reshape(2, 8, -1), dim=2, unbiased=False)
        a = (1 / torch.sqrt(var + c.eps)).repeat_interleave(4, 1) * c.gamma.double()
        b = c.beta.double() - mean.repeat_interleave(4, 1) * a
        assert E.affine_excess(t, torch.stack([a, b], -1)).max() <= 1


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
@pytest.mark.parametrize("k", [0, 100, 256])
def test_layernorm_emulator_matches_torch(dt, k):
    with E.storage(dt):
        g = gen(f"ln{k}")
        M, C, xp, yp = 9, 264, 272, 280
        x = torch.full((M * xp,), math.nan, dtype=E.H16)
        x.view(M, xp)[:, :C] = (torch.randn(M, C, generator=g) + k).to(E.H16)
        gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
        r = E.layernorm(x, M, C, xp, gamma, beta, 1e-5, yp)
        y = F.layer_norm(x.view(M, xp)[:, :C].double(), (C,), gamma.double(), beta.double(), 1e-5)
        want = torch.zeros(M, yp, dtype=F64)
        want[:, :C] = E.h16(y)
        assert E.excess(r, want).max() <= 1


def test_nearest_index_is_f_interpolates_for_every_pair_up_to_79():
    # on fp32 / fp16 tensors: for float64 ones F.interpolate forms the scale in double (32 of these pairs differ)
    for n_in in range(1, 80):
        src = torch.arange(n_in, dtype=torch.float32).view(1, 1, n_in)
        for n_out in range(1, 80):
            got = F.interpolate(src, size=n_out, mode="nearest").view(-1).long()
            index = R.axis_weights(R.NEAREST, n_in, n_out, np.float32(n_in) / np.float32(n_out)).argmax(1)
            assert torch.equal(torch.from_numpy(index), got), (n_in, n_out)


@pytest.mark.parametrize("dims", [2, 3])
def test_resize_nearest_emulator_matches_f_interpolate(dims):
    g = gen(f"rs{dims}")
    N, pitch = 2, 8
    D, H, W, OD, OH, OW = (1, 26, 6, 1, 22, 74) if dims == 2 else (14, 6, 26, 46, 74, 22)
    x = torch.randn(N, D, H, W, pitch, generator=g)
    got = R.resample_cl(x, (OD, OH, OW), R.NEAREST)
    ncd = x.permute(0, 4, 1, 2, 3)
    if dims == 2:
        want = F.interpolate(ncd[:, :, 0], size=(OH, OW), mode="nearest")[:, :, None]
    else:
        want = F.interpolate(ncd, size=(OD, OH, OW), mode="nearest")
    assert torch.equal(got, want.permute(0, 2, 3, 4, 1))


# ----------------------------------------------------------------------------------------------------------------
# mutants
# ----------------------------------------------------------------------------------------------------------------
def gn_case():
    # 6 values per group (3 voxels x 2 channels): a one-element change to the statistics moves rstd by percents
    return GN("mut", 2, 3, 8, 4, 6, eps=0.1, k=2.0)


def worst(r, got):
    return float(E.excess(r, got).max())


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_bound_rejects_groupnorm_mutants(dt):
    with E.storage(dt):
        c = gn_case()
        r, _ = c.emulate()
        assert worst(r, c.mutant()) <= 1
        muts = {
            "unbiased_variance": c.mutant(var_fn=lambda v, n: v * n / (n - 1)),
            "eps_outside_sqrt": c.mutant(rstd_fn=lambda v, e: 1 / (torch.sqrt(v) + e)),
            "voxel_per_chunk_dropped": c.mutant(stat_x=c.X[:, :-1]),
            "pad_channel_unwritten": c.store(c.X * 0 + r.exact.view(c.N, c.S, -1)[..., :c.C], pad=math.nan),
        }
        for name, got in muts.items():
            ex = worst(r, got)
            report(name, dt, ex)
            assert ex > MARGIN, name


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_bound_rejects_second_source_with_first_source_statistics(dt):
    with E.storage(dt):
        c = GN("mut2", 2, 3, 8, 8, 8, k=0.5, offset1=2.0)          # groups 4..7 live in the second source
        r, _ = c.emulate()
        got = c.mutant(stat_of=torch.tensor([0, 1, 2, 3, 0, 1, 2, 3]))
        ex = worst(r, got)
        report("second_source_first_source_stats", dt, ex)
        assert ex > MARGIN


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_bound_rejects_swapped_leakyrelu_slopes(dt):
    with E.storage(dt):
        for act, other in ((E.ACT_LEAKYRELU, 0.2), (E.ACT_LEAKYRELU02, 0.01)):
            c = GN("mut3", 2, 3, 8, 4, 6, act=act)
            r, _ = c.emulate()
            assert worst(r, c.mutant()) <= 1
            ex = worst(r, c.mutant(slope=other))
            report(f"leakyrelu_slope_{E.SLOPE[act]}_as_{other}", dt, ex)
            assert ex > MARGIN


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_bound_rejects_swapped_spade_halves(dt):
    with E.storage(dt):
        g = gen("spade")
        N, S, C, gbp, yp = 2, 5, 8, 24, 16
        x = torch.randn(N * S * C, generator=g).to(E.H16)
        gb = torch.randn(N * S * gbp, generator=g).to(E.H16)
        ax = torch.randn(N, C, 2, generator=g)
        gba = torch.randn(N, 2 * C, 2, generator=g)
        r = E.spade(x, None, C, 0, C, 0, N, S, ax, gb, gbp, gba, E.ACT_LEAKYRELU02, yp)
        X = x.double().view(N, S, C)
        G = gb.double().view(N, S, gbp)
        nx = X * ax[:, None, :, 0] + ax[:, None, :, 1]
        gg = G[..., :C] * gba[:, None, :C, 0] + gba[:, None, :C, 1]
        tt = G[..., C:2 * C] * gba[:, None, C:, 0] + gba[:, None, C:, 1]

        def store(v):
            out = torch.zeros(N * S, yp, dtype=F64)
            out[:, :C] = E.h16(F.leaky_relu(v, 0.2).reshape(-1, C))
            return out

        assert worst(r, store(nx * (1 + gg) + tt)) <= 1
        ex = worst(r, store(nx * (1 + tt) + gg))
        report("spade_gamma_beta_swapped", dt, ex)
        assert ex > MARGIN


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_bound_rejects_partial_slot_read_off_by_one(dt):
    with E.storage(dt):
        c = GN("mut_part", 2, 40, 16, 8, 3, eps=1e-5)
        P0, P1 = E.partials_from(c.X[..., :16], 5, 8), E.partials_from(c.X[..., 16:], 3, 4)
        args = (16, 8, c.N, c.S, c.groups, c.eps, c.gamma, c.beta)
        t = E.gn_from_partials([P0.reshape(-1), P1.reshape(-1)], [5, 3], [8, 4], *args)
        want = E.gn_affine(c.X, c.groups, c.eps, c.gamma, c.beta)
        assert E.affine_excess(t, torch.stack([want.a, want.b], -1)).max() <= 1
        shifted = torch.roll(P0, -1, dims=1)
        shifted[:, -1] = 0                                      # slots 1..5 read as 0..4: the last one past the buffer
        m = E.gn_from_partials([shifted.reshape(-1), P1.reshape(-1)], [5, 3], [8, 4], *args)
        ex = float(E.affine_excess(t, torch.stack([m.a, m.b], -1)).max())
        report("partial_slot_off_by_one", dt, ex)
        assert ex > MARGIN


def test_exact_rational_nearest_index_differs():
    for n_in, n_out in ((26, 22), (6, 74), (14, 46)):
        rational = torch.minimum(torch.arange(n_out) * n_in // n_out, torch.tensor(n_in - 1))
        index = R.axis_weights(R.NEAREST, n_in, n_out, np.float32(n_in) / np.float32(n_out)).argmax(1)
        bad = int((rational != torch.from_numpy(index)).sum())
        print(f"\nMUTANT exact_rational_nearest {n_in}->{n_out} differs at {bad} of {n_out} indices")
        assert bad > 0


def one_pass_fp32_rows(X, lanes, fold32=False):
    """E[x^2] - mean^2 from fp32 sums: `lanes` sequential chains (one per thread), folded in fp64 (the GroupNorm
    kernels' block reduction) or, with fold32, in an fp32 warp tree with the moments in fp32 too (rows_linear's old
    prologue).  X [R, n] float64; returns mean, var per row."""
    R, n = X.shape
    x = X.float()
    pad = (-n) % lanes
    x = torch.cat([x, torch.zeros(R, pad)], 1).view(R, -1, lanes)
    s = torch.zeros(R, lanes)
    q = torch.zeros(R, lanes)
    for i in range(x.shape[1]):
        s = s + x[:, i]
        q = torch.addcmul(q, x[:, i], x[:, i])
    if fold32:
        while s.shape[1] > 1:
            h = s.shape[1] // 2
            s, q = s[:, :h] + s[:, h:], q[:, :h] + q[:, h:]
        mean = s[:, 0] / n
        return mean.double(), (q[:, 0] / n - mean * mean).clamp_min(0.0).double()
    s, q = s.double().sum(1), q.double().sum(1)
    mean = s / n
    return mean, (q / n - mean ** 2).clamp_min(0.0)


@pytest.mark.parametrize("dt", FLAVOURS, ids=FL_IDS)
def test_bound_rejects_one_pass_fp32_statistics_at_large_offset(dt):
    with E.storage(dt):
        # GroupNorm: 8 channels x 2048 voxels per group summed by 32 threads in fp32 (the fused kernel's shape)
        c = GN("mut_k", 1, 2048, 16, 0, 2, eps=1e-5, k=256.0)
        r, _ = c.emulate()
        Xg = c.X.reshape(1, 2048, 2, 8).permute(0, 2, 1, 3).reshape(2, -1)
        mean, var = one_pass_fp32_rows(Xg, 32)
        rstd = 1 / torch.sqrt(var + c.eps)
        ex = lambda t: t.repeat_interleave(8)[None, None]
        y = (c.X - ex(mean)) * ex(rstd) * c.gamma.double() + c.beta.double()
        e_gn = worst(r, c.store(y))
        report("groupnorm_one_pass_fp32_k256", dt, e_gn)
        assert e_gn > MARGIN
        # LayerNorm (rows_linear's old prologue): one warp per row of 512.  At k = 256 its rstd is ~0.5 % off: several
        # fp16 ulps of the output but under one bf16 ulp, so the bf16 flavour shows it at k = 1024
        g = gen("mut_ln")
        M, K = 8, 512
        x = (torch.randn(M, K, generator=g) + (256 if dt is torch.float16 else 1024)).to(E.H16)
        gamma, beta = torch.ones(K), torch.zeros(K)
        rl = E.rows_linear_ln(x.reshape(-1), M, K, K, gamma, beta, 1e-5)
        mean, var = one_pass_fp32_rows(x.double(), 32, fold32=True)
        y = (x.double() - mean[:, None]) / torch.sqrt(var[:, None] + 1e-5)
        e_ln = worst(rl, E.h16(y))
        report("rows_linear_one_pass_fp32_k256" if dt is torch.float16 else "rows_linear_one_pass_fp32_k1024", dt, e_ln)
        assert e_ln > MARGIN
