"""CPU tests of the host-side logic in generativemodels_b200.ops: weight packing, tap tables, asymmetric padding,
stride, transposed-conv phases, virtual concat, GEMM/attention parameter blocks.  The C-ABI call is replaced by
tests/igemm_emulator.py (a literal reading of include/b200gen.h), so what is verified here is exactly the struct the
GPU kernel receives.  That the kernels compute what the emulator computes, on every store path and kernel of b200_igemm,
is checked on the GPU by tests/test_igemm_contract_gpu.py."""
import math

import pytest
import torch
import torch.nn.functional as F

from generativemodels_b200 import ops
from tests import cpu_backend, igemm_emulator


@pytest.fixture(autouse=True)
def _emulated(monkeypatch):
    cpu_backend.install(monkeypatch)          # weight repacking and the GEMM both go through the C-ABI stand-in
    monkeypatch.setattr(ops, "igemm_raw", igemm_emulator.emulate)


def bf(x):
    return x.to(ops.H16).float()


def cl_cpu(x):
    """NC[D]HW fp32 -> CL on CPU (test-only stand-in for the layout kernel)."""
    sd = x.dim() - 2
    t = x.movedim(1, -1)
    if sd == 2:
        t = t.unsqueeze(1)
    C_ = x.shape[1]
    P = ops.round_up(C_, 8)
    t = F.pad(t, (0, P - C_)).to(ops.H16).contiguous()
    return ops.CL(t, C_, sd)


def back(a):
    t = a.t[..., : a.C].float()
    if a.spatial_dims == 2:
        t = t.squeeze(1)
    return t.movedim(-1, 1)


def close(a, b, tol=1.5e-2):
    err = (a - b).norm() / (b.norm() + 1e-12)
    assert err < tol, f"rel err {err:.3e}"


CASES = [
    (2, 2, 20, 24, (9, 7), 3, 1, 1), (2, 1, 3, 8, (6, 6), 3, 1, 1), (2, 1, 70, 5, (5, 8), 1, 1, 0),
    (3, 1, 12, 16, (4, 5, 6), 3, 1, 1), (2, 1, 16, 16, (9, 11), 3, 2, 1), (3, 1, 8, 8, (6, 6, 7), 3, 2, 1),
    (3, 1, 8, 12, (6, 8, 6), 4, 2, 1), (2, 1, 130, 16, (4, 4), 3, 1, 1),
]


@pytest.mark.parametrize("case", CASES, ids=[str(c) for c in CASES])
def test_conv_host_logic(case):
    sd, N, Cin, Cout, sp, k, s, p = case
    torch.manual_seed(0)
    x = torch.randn(N, Cin, *sp)
    w = torch.randn(Cout, Cin, *([k] * sd)) / math.sqrt(Cin * k ** sd)
    b = torch.randn(Cout)
    conv = F.conv2d if sd == 2 else F.conv3d
    ref = conv(bf(x), bf(w), b, stride=s, padding=p)
    out = ops.conv(cl_cpu(x), ops.PackedConv(w, b, s, p))
    assert tuple(back(out).shape) == tuple(ref.shape)
    close(back(out), ref)
    assert out.t[..., out.C:].abs().sum() == 0


@pytest.mark.parametrize("sd,Cin,Cout,sp,k,s,p,kw", [
    (3, 1, 16, (6, 7, 5), 3, 1, 1, {}), (2, 3, 24, (9, 8), 3, 1, 1, dict(act1=2)), (3, 2, 16, (8, 8, 6), 3, 2, 1, {}),
    (3, 64, 1, (5, 6, 7), 3, 1, 1, dict(out_f32=True)), (2, 72, 3, (9, 7), 3, 1, 1, {}), (3, 64, 2, (4, 4, 4), 3, 1, 1, {}),
])
def test_tap_reformulations_host_logic(monkeypatch, sd, Cin, Cout, sp, k, s, p, kw):
    """conv_in-like (few input channels -> b200_tap_gather + one-chunk GEMM) and out-conv-like (few output channels ->
    1x1 GEMM with taps as columns + b200_tap_sum) routes of ops.conv against F.conv (diffusion_model_unet.py:1744-1752,
    1856-1867), forced on for small shapes."""
    from tests import cpu_backend
    cpu_backend.install(monkeypatch)
    monkeypatch.setattr(ops, "_TAP_MIN_ROWS", 1)
    torch.manual_seed(3)
    x = torch.randn(2, Cin, *sp)
    w = torch.randn(Cout, Cin, *([k] * sd)) / math.sqrt(Cin * k ** sd)
    b = torch.randn(Cout)
    pc = ops.PackedConv(w, b, s, p)
    assert (pc.tap_in is not None) == (Cin * k ** sd <= 64) and (pc.tap_out is not None) == (Cout <= 4 and Cin >= 64)
    conv = F.conv2d if sd == 2 else F.conv3d
    ref = conv(bf(x), bf(w), b, stride=s, padding=p)
    if kw.get("act1") == 2:
        ref = F.silu(ref)
    out = ops.conv(cl_cpu(x), pc, **kw)
    if kw.get("out_f32"):
        got = out[..., :Cout].movedim(-1, 1)
        assert out[..., Cout:].abs().sum() == 0
    else:
        got = back(out)
        assert out.t[..., out.C:].abs().sum() == 0
    assert tuple(got.shape) == tuple(ref.shape)
    close(got, ref)


def test_groupnorm_from_conv_partials_host_logic(monkeypatch):
    """GroupNorm statistics taken from the partial sums the producing convolutions leave behind (b200_igemm gn_partial
    -> b200_groupnorm_from_partials) against the ordinary two-pass GroupNorm: single source, virtual concat of two
    producers with different channel counts (groups of 24 = 3 producer groups), the 8-phase upsample convolution,
    and invalidation by an in-place update."""
    from tests import cpu_backend
    cpu_backend.install(monkeypatch)
    monkeypatch.setattr(ops, "_GN_FUSE_MIN_ROWS", 1)
    torch.manual_seed(5)
    x = torch.randn(2, 16, 5, 6, 4)
    mk = lambda co, ci: ops.PackedConv(torch.randn(co, ci, 3, 3, 3) / math.sqrt(ci * 27), torch.randn(co), 1, 1)
    a = ops.conv(cl_cpu(x), mk(64, 16))
    b = ops.conv(cl_cpu(x), mk(32, 16))
    # narrow tensors (<= 128 channels) leave 4-channel partial groups, wider ones 8-channel groups
    assert a.gn is not None and tuple(a.gn.shape) == (2, ops._gn_slots(), 16, 2) and b.gn is not None
    wide = ops.conv(cl_cpu(x), mk(160, 16))
    assert tuple(wide.gn.shape) == (2, ops._gn_slots(), 20, 2)

    def both(srcs, groups):
        Ct = sum(t.C for t in srcs)
        g, be = torch.randn(Ct), torch.randn(Ct)
        fused = ops.groupnorm(srcs, groups, 1e-5, g, be, act=ops.ACT_SILU)
        monkeypatch.setattr(ops, "_GN_FUSE", False)
        plain = ops.groupnorm(srcs, groups, 1e-5, g, be, act=ops.ACT_SILU)
        monkeypatch.setattr(ops, "_GN_FUSE", True)
        close(back(fused), back(plain), 1e-2)
        ref = F.silu(F.group_norm(torch.cat([back(t) for t in srcs], 1), groups, g, be, 1e-5))
        close(back(fused), ref, 1e-2)

    calls = []
    real = cpu_backend.FakeLib.b200_groupnorm_from_partials_ex
    monkeypatch.setattr(cpu_backend.FakeLib, "b200_groupnorm_from_partials_ex",
                        lambda self, *args: (calls.append(1), real(self, *args))[1])
    both([a], 8)                  # 8 channels per group = one producer group
    both([a], 2)                  # 32 channels per group
    both([a, b], 4)               # concat 96 channels, groups of 24 (64 % 24 != 0 -> falls back to the full pass)
    assert len(calls) == 2
    both([a, b], 6)               # groups of 16: 4 groups in a, 2 in b -> fused
    assert len(calls) == 3
    both([a], 16)                 # GroupNorm groups of 4 channels (32 groups over 128 channels in the 2-D UNets)
    both([wide, a], 28)           # groups of 8 over an 8-channel-partial source and a 4-channel-partial source
    both([wide], 40)              # groups of 4 over 8-channel partials: falls back to the statistics pass
    assert len(calls) == 5
    up = ops.conv_upsample2x(a, ops.PackedUpsampleConv(torch.randn(32, 64, 3, 3, 3) / 40, torch.randn(32)))
    assert up.gn is not None and up.gn.shape[1] == 8 * ops._gn_slots()
    both([up], 4)
    assert len(calls) == 6
    c = ops.axpy(a, a, 0.5, inplace=True)
    assert c.gn is None           # an in-place update invalidates the producer's sums
    both([c], 8)
    assert len(calls) == 6


def test_asym_pad_host_logic():
    for sd, sp in ((2, (8, 10)), (3, (4, 6, 5))):
        x = torch.randn(1, 16, *sp)
        w = torch.randn(16, 16, *([3] * sd)) / 10
        conv = F.conv2d if sd == 2 else F.conv3d
        ref = conv(F.pad(bf(x), (0, 1) * sd), bf(w), None, stride=2)
        out = ops.conv(cl_cpu(x), ops.PackedConv(w, None, 2, [(0, 1)] * sd))
        assert tuple(back(out).shape) == tuple(ref.shape)
        close(back(out), ref)


def test_concat_epilogue_host_logic():
    torch.manual_seed(1)
    N, C0, C1, Cout, sp = 2, 24, 8, 20, (3, 4, 5)
    x0, x1 = torch.randn(N, C0, *sp), torch.randn(N, C1, *sp)
    w = torch.randn(Cout, C0 + C1, 3, 3, 3) / 20
    b, temb, res = torch.randn(Cout), torch.randn(N, Cout), torch.randn(N, Cout, *sp)
    ref = F.conv3d(torch.cat([bf(x0), bf(x1)], 1), bf(w), b, padding=1) + temb[:, :, None, None, None]
    ref = F.relu(bf(res) + 0.5 * F.silu(ref))
    pc = ops.PackedConv(w, b, 1, 1, splits=[C0, C1])
    out = ops.conv([cl_cpu(x0), cl_cpu(x1)], pc, rowvec=temb, act1=ops.ACT_SILU, scale=0.5, residual=cl_cpu(res),
                   act2=ops.ACT_RELU)
    close(back(out), ref)
    out32 = ops.conv([cl_cpu(x0), cl_cpu(x1)], pc, rowvec=temb[:1], out_f32=True)
    ref32 = F.conv3d(torch.cat([bf(x0), bf(x1)], 1), bf(w), b, padding=1) + temb[:1, :, None, None, None]
    close(out32[..., :Cout].movedim(-1, 1), ref32, 1e-3)


@pytest.mark.parametrize("sd,sp,k,s,p,op", [(2, (5, 6), 4, 2, 1, 0), (3, (3, 4, 5), 4, 2, 1, 0), (2, (4, 4), 3, 2, 1, 1)])
def test_conv_transpose_host_logic(sd, sp, k, s, p, op):
    torch.manual_seed(2)
    x = torch.randn(2, 12, *sp)
    w = torch.randn(12, 10, *([k] * sd)) / 5
    b = torch.randn(10)
    convt = F.conv_transpose2d if sd == 2 else F.conv_transpose3d
    ref = F.relu(convt(bf(x), bf(w), b, stride=s, padding=p, output_padding=op))
    out = ops.conv_transpose(cl_cpu(x), ops.PackedConvTranspose(w, b, s, p, op), act1=ops.ACT_RELU)
    assert tuple(back(out).shape) == tuple(ref.shape)
    close(back(out), ref)


@pytest.mark.parametrize("sd,sp", [(2, (5, 6)), (3, (3, 4, 5))])
def test_upsample_conv_host_logic(sd, sp):
    """nearest x2 + k3 conv folded into per-phase 2-tap convolutions == F.interpolate + F.conv."""
    torch.manual_seed(5)
    x = torch.randn(2, 12, *sp)
    w = torch.randn(10, 12, *([3] * sd)) / 6
    b = torch.randn(10)
    conv = F.conv2d if sd == 2 else F.conv3d
    ref = conv(F.interpolate(bf(x), scale_factor=2.0, mode="nearest"), w, b, padding=1)   # fp32 weights: the fold
    out = ops.conv_upsample2x(cl_cpu(x), ops.PackedUpsampleConv(w, b))                  # sums taps before bf16
    assert tuple(back(out).shape) == tuple(ref.shape)
    close(back(out), ref)


def test_linear_and_transposed_host_logic():
    torch.manual_seed(3)
    M, K, O = 37, 40, 24
    x = torch.randn(1, K, 1, M)
    w, b = torch.randn(O, K) / 6, torch.randn(O)
    ref = F.linear(bf(x)[0, :, 0].t(), bf(w), b)
    pl = ops.PackedLinear(w, b)
    a = cl_cpu(x)
    out = ops.linear(a, pl)
    close(out.t[0, 0, 0, :, :O].float(), ref)
    vt = ops.linear_transposed(a.t.reshape(1, M, -1), K, pl)
    close(vt[0, :, :M].float(), ref.t())
    # a batch goes through ONE launch: the projection matrix is the broadcast A operand, sample b's rows are weight
    # batch b (b200gen.h a_broadcast / w_batched)
    xb = torch.randn(3, K, 1, M)
    ab = cl_cpu(xb)
    vtb = ops.linear_transposed(ab.t.reshape(3, M, -1), K, pl)
    for i in range(3):
        close(vtb[i, :, :M].float(), F.linear(bf(xb)[i, :, 0].t(), bf(w), b).t())


def test_linear_geglu_host_logic():
    """linear1 + GEGLU gating as one GEMM: interleaved [32 a | 32 gate] weight rows, B200_ACT_GEGLU epilogue
    (MLPBlock act="GEGLU": a * gelu(gate), a, gate = chunk(linear1(x), 2, -1))."""
    torch.manual_seed(5)
    for M, K, H in ((37, 40, 32), (130, 64, 160), (9, 256, 1024)):
        x = torch.randn(1, K, 1, M)
        w, b = torch.randn(2 * H, K) / K ** 0.5, torch.randn(2 * H)
        a, gate = F.linear(bf(x)[0, :, 0].t(), bf(w), b).chunk(2, -1)
        ref = a * F.gelu(gate)
        out = ops.linear_geglu(cl_cpu(x), ops.PackedLinear.geglu(w, b))
        assert out.C == H and out.t.shape[-1] == H
        close(out.t[0, 0, 0, :, :H].float(), ref)
    with pytest.raises(ValueError):
        ops.PackedLinear.geglu(torch.randn(2 * 40, 16), None)          # hidden width not a multiple of 32


def test_attention_tc_host_logic(monkeypatch):
    """The tensor-core attention parameter blocks (QK^T, PV with V^T) — softmax emulated on CPU."""
    torch.manual_seed(4)
    B, T, heads, dh = 2, 70, 2, 64
    Cc = heads * dh
    q, k, v = (torch.randn(B, T, Cc) for _ in range(3))

    class FakeLib:
        def b200_softmax_rows_partials(self, s, M, S, sp, part, n_tiles, p, pp, stream):
            from tests.cpu_backend import FakeLib as F2
            return F2().b200_softmax_rows_partials(s, M, S, sp, part, n_tiles, p, pp, stream)

        def b200_softmax_rows(self, s, M, S, sp, p, pp, stream):
            import ctypes as C
            import numpy as np
            sc = np.ctypeslib.as_array(C.cast(s, C.POINTER(C.c_float)), shape=(M * sp,)).reshape(M, sp)[:, :S]
            e = np.exp(sc - sc.max(1, keepdims=True))
            pr = e / e.sum(1, keepdims=True)
            dst = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint16)), shape=(M * pp,)).reshape(M, pp)
            dst[:] = 0
            dst[:, :S] = igemm_emulator._f32_to_bf16(pr.astype(np.float32)).reshape(M, S)
            return 0

    monkeypatch.setattr(ops._lib, "require_device", lambda: FakeLib())
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops, "_FORCE_UNFUSED_ATTENTION", True)     # this test covers the GEMM + softmax + GEMM blocks
    qb, kb, vb = (t.to(ops.H16).contiguous() for t in (q, k, v))
    vt = F.pad(vb.transpose(1, 2), (0, ops.round_up(T, 8) - T)).contiguous()
    out = ops.attention(qb, kb, None, heads, dh, 1 / math.sqrt(dh), vt=vt)
    qh, kh, vh = (bf(t).view(B, T, heads, dh).transpose(1, 2) for t in (q, k, v))
    ref = (torch.softmax(qh @ kh.transpose(-1, -2) / math.sqrt(dh), -1) @ vh).transpose(1, 2).reshape(B, T, Cc)
    close(out[..., :Cc].float(), ref, 2e-2)


def test_auto_cuda_graph_policy(monkeypatch):
    """inferers.AUTO_CUDA_GRAPH (on by default since round 2): which sample() calls replay the network from a CUDA graph."""
    import torch.nn as nn

    import generativemodels_b200.inferers.inferer as I

    class FakeNoise:
        def __init__(self, per_sample, cuda=True):
            self.is_cuda, self._n = cuda, per_sample

        def __getitem__(self, i):
            return torch.empty(self._n, device="meta")

    class Sched:
        def __init__(self, n):
            self.timesteps = list(range(n))

    made = []
    monkeypatch.setattr(I, "graphed", lambda m: (made.append(m), ("graph-of", m))[1])
    net = nn.Linear(2, 2)
    assert I.AUTO_CUDA_GRAPH is True
    monkeypatch.setattr(I, "AUTO_CUDA_GRAPH", False)
    assert I._maybe_graphed(net, FakeNoise(100), Sched(50), None) is net
    monkeypatch.setattr(I, "AUTO_CUDA_GRAPH", True)
    w = I._maybe_graphed(net, FakeNoise(3 * 64 * 64), Sched(50), None)
    assert w == ("graph-of", net) and I._maybe_graphed(net, FakeNoise(3 * 64 * 64), Sched(50), None) is w
    assert len(made) == 1 and "_b200_auto_graph" not in dict(net.named_modules()) and not net.state_dict().keys() - {
        "weight", "bias"}
    other = nn.Linear(2, 2)
    assert I._maybe_graphed(other, FakeNoise(160 * 224 * 160), Sched(50), None) is other      # work-bound volume
    assert I._maybe_graphed(other, FakeNoise(4096), Sched(4), None) is other                 # too few steps to amortise
    assert I._maybe_graphed(other, FakeNoise(4096, cuda=False), Sched(50), None) is other
    assert I._maybe_graphed(other, FakeNoise(4096), Sched(50), object()) is other             # SPADE: seg is bound late
    fn = lambda *a, **k: None                                                                 # noqa: E731
    assert I._maybe_graphed(fn, FakeNoise(4096), Sched(50), None) is fn and len(made) == 1


def test_transformer_block_host_paths(monkeypatch):
    """Host choices of the conditioned transformer block (second half of round 2): linear1 + GEGLU as one GEMM when the
    hidden width is a multiple of 32 (else linear + b200_geglu), the to_k / to_v projections of a handful of context
    tokens through the GEMV entry point, and ops.fork() as a no-op outside a CUDA-graph capture — each against the
    plain formulation."""
    from generativemodels_b200.networks.nets.diffusion_model_unet import (BasicTransformerBlock, GEGLUFeedForward,
                                                                          _few_rows_linear)
    from generativemodels_b200.networks._holders import packed_linear
    torch.manual_seed(9)
    calls = {"rows_linear": 0, "geglu": 0}
    real_rl, real_gg = cpu_backend.FakeLib.b200_rows_linear, cpu_backend.FakeLib.b200_geglu
    monkeypatch.setattr(cpu_backend.FakeLib, "b200_rows_linear",
                        lambda self, *a: (calls.__setitem__("rows_linear", calls["rows_linear"] + 1), real_rl(self, *a))[1])
    monkeypatch.setattr(cpu_backend.FakeLib, "b200_geglu",
                        lambda self, *a: (calls.__setitem__("geglu", calls["geglu"] + 1), real_gg(self, *a))[1])

    # feed-forward: hidden 4 * 16 = 64 (fused) and 4 * 12 = 48 (not a multiple of 32 -> separate gating kernel)
    for C_, fused in ((16, True), (12, False)):
        ff = GEGLUFeedForward(C_, 4 * C_).eval()
        x = torch.randn(1, C_, 1, 23)
        xs = bf(x)[0, :, 0].t()
        a, gate = F.linear(xs, bf(ff.linear1.weight), ff.linear1.bias).chunk(2, -1)
        ref = F.linear(bf(a * F.gelu(gate)), bf(ff.linear2.weight), ff.linear2.bias)
        before = calls["geglu"]
        with torch.no_grad():
            out = ff(cl_cpu(x))
        assert (calls["geglu"] == before) == fused
        close(out.t[0, 0, 0, :, :C_].float(), ref, 2e-2)

    # context projections: 2 tokens in total -> GEMV entry point; 9 tokens -> the GEMM path; same numbers
    blk = BasicTransformerBlock(32, 2, 16, cross_attention_dim=8).eval()
    pl = packed_linear(blk.attn2, "to_k")
    for n_tok, gemv in ((2, True), (9, False)):
        ctx = torch.randn(n_tok, 8, 1, 1)                      # N = n_tok samples, one context token each
        before = calls["rows_linear"]
        rows = _few_rows_linear(cl_cpu(ctx), pl)
        assert (calls["rows_linear"] == before + 1) == gemv
        close(rows[:, 0, :32].float(), F.linear(bf(ctx)[:, :, 0, 0], bf(blk.attn2.to_k.weight)), 2e-2)

    with ops.fork() as f:                                       # no GPU, no capture: nothing happens
        assert not f.active
    f.join()
