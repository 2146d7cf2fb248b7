"""The metric kernels on the GPU: every case of tests/golden/g_metrics.pt against the reference's outputs, a sweep
against the float64 reading of their contract (tests/metrics_emulator.py), bit-identical repeats and CUDA-graph
capture of a metric call."""
import pytest
import torch

from generativemodels_b200 import metrics as GM
from generativemodels_b200 import ops
from tests import metrics_emulator as M
from tests.golden import load
from tests.golden.make_golden_metrics import CASES, inputs

pytestmark = pytest.mark.gpu
FIX = load("g_metrics")
DEV = "cuda"


def _metric(case):
    return (GM.SSIMMetric if case["kind"] == "ssim" else GM.MultiScaleSSIMMetric)(**case["kw"])


# The reference's own bounds on its cases: 1e-6 absolute on MS-SSIM, rtol 1e-4 on MMD (scaled by the Gram terms, whose
# difference is the result).  Other SSIM / MS-SSIM cases: 2e-5, the fp32 error of the reference's moments (its
# sigma = E[x^2] - E[x]^2 cancels), largest at MS-SSIM's single-voxel coarsest scale (6.1e-6 in float64).
@pytest.mark.parametrize("name", list(CASES))
def test_fixture_case(cuda_device, name):
    case, rec = CASES[name], FIX[name]
    a, b = (t.to(DEV) for t in inputs(case))
    if case["kind"] == "mmd":
        got = GM.MMDMetric()(a, b)
        assert got.dim() == 0 and got.dtype == torch.float32 and got.is_cuda
        err = abs(float(got) - float(rec["out"]))
        print(f"{name}: |mmd - ref| = {err:.3e}, terms {float(rec['terms'].abs().sum()):.3e}")
        assert err <= 1e-4 * float(rec["terms"].abs().sum()) + 1e-12
        return
    got = _metric(case)(a, b)
    assert got.shape == (case["shape"][0], 1) and got.dtype == torch.float32
    err = (got.cpu() - rec["out"]).abs().max().item()
    print(f"{name}: max |metric - ref| = {err:.3e}")
    assert err <= (1e-6 if case["gen"] == "ref_test" else 2e-5)


def _views(shape, dtype, strided, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(shape, generator=g)
    b = (a + 0.3 * torch.randn(shape, generator=g)).clamp(0, 1)
    if strided:          # a channels-last layout and a view with a step along the last axis
        big = list(shape)
        big[-1] *= 2
        a2 = torch.zeros(big)
        a2[..., ::2] = a
        a = a2.to(DEV, dtype)[..., ::2]
        b = b.to(DEV, dtype).movedim(1, -1).contiguous().movedim(-1, 1)
        assert not a.is_contiguous()
        return a, b
    return a.to(DEV, dtype), b.to(DEV, dtype)


SWEEP = [  # (spatial_dims, shape, kernel_size, kernel_type, sigma)
    (2, (2, 1, 33, 40), 1, "gaussian", 1.5),
    (2, (1, 3, 37, 29), 4, "gaussian", 1.5),
    (2, (2, 2, 30, 45), 7, "uniform", 1.5),
    (2, (1, 4, 64, 50), 11, "gaussian", 1.5),
    (2, (1, 2, 40, 41), (3, 9), "gaussian", (0.8, 2.0)),
    (3, (1, 1, 20, 18, 23), 4, "gaussian", 1.5),
    (3, (2, 2, 24, 21, 26), 11, "uniform", 1.5),
    (3, (1, 3, 17, 20, 19), (5, 3, 7), "gaussian", (1.0, 0.5, 2.0)),
    (3, (1, 1, 46, 44, 45), 41, "gaussian", 6.0),     # ring of 41 planes: 4-row tiles
    (2, (1, 1, 160, 150), 101, "uniform", 1.5),       # a 108 x 132 staging tile
]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.float64])
@pytest.mark.parametrize("strided", [False, True])
@pytest.mark.parametrize("i", range(len(SWEEP)))
def test_ssim_maps_and_means_match_the_contract(cuda_device, i, dtype, strided):
    sd, shape, ks, kt, sig = SWEEP[i]
    a, b = _views(shape, dtype, strided, 100 + i)
    s, cs = GM.compute_ssim_and_cs(a, b, sd, kernel_type=kt, kernel_size=ks, kernel_sigma=sig)
    taps, scale = GM.ssim.separable_kernel(sd, kt, ks, sig)
    a5, b5 = (t.cpu() if sd == 3 else t.cpu().unsqueeze(2) for t in (a, b))
    ws, wcs = M.ssim(a5, b5, taps, scale, 1e-4, 9e-4)
    if sd == 2:
        ws, wcs = ws.squeeze(2), wcs.squeeze(2)
    assert s.shape == ws.shape and s.dtype == torch.float32
    assert (s.cpu() - ws).abs().max().item() < 5e-4 and (cs.cpu() - wcs).abs().max().item() < 5e-4
    mean = GM.SSIMMetric(sd, kernel_type=kt, kernel_size=ks, kernel_sigma=sig)(a, b)
    assert (mean.cpu().double().view(-1) - M.per_item_means(ws)).abs().max().item() < 2e-6


@pytest.mark.parametrize("sd,shape,ks,w", [(2, (2, 2, 45, 51), 3, [0.3, 0.3, 0.4]),
                                           (3, (1, 2, 37, 41, 35), (3, 2, 3), [0.2, 0.3, 0.5]),
                                           (2, (1, 1, 64, 64), 4, [0.0448, 0.2856, 0.3001, 0.2363, 0.1333])])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_ms_ssim_odd_extents_match_the_contract(cuda_device, sd, shape, ks, w, dtype):
    a, b = _views(shape, dtype, dtype == torch.float16, 7)
    got = GM.MultiScaleSSIMMetric(sd, kernel_size=ks, weights=w)(a, b).cpu()
    taps, scale = GM.ssim.separable_kernel(sd, "gaussian", ks, 1.5)
    x, y = (t.cpu() if sd == 3 else t.cpu().unsqueeze(2) for t in (a, b))
    ss, cc = [], []
    for s in range(len(w)):
        sm, cm = M.ssim(x, y, taps, scale, 1e-4, 9e-4)
        ss.append(M.per_item_means(sm).float())
        cc.append(M.per_item_means(cm).float())
        x, y = M.pool(x, sd), M.pool(y, sd)
    want = M.combine(torch.stack(ss), torch.stack(cc), w)
    err = (got.double().view(-1) - want).abs().max().item()
    print(f"ms-ssim {shape} k={ks} {dtype}: max |got - reading| = {err:.3e}")
    # 1e-4: with 5 weights the coarsest 4 x 4 scale has one voxel per channel, whose fp32 variance cancels
    assert err < 1e-4


def test_pooling_is_exact(cuda_device):
    x = torch.rand(2, 3, 9, 13, 11, device=DEV)[:, :, :, 1:, :]
    for sd, v in ((3, x), (2, x[:, :, :1])):
        got = ops.avgpool2_f32(v, sd).cpu()
        assert torch.equal(got, M.pool(v.cpu(), sd))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.float64])
def test_mmd_matches_the_contract(cuda_device, dtype):
    g = torch.Generator().manual_seed(5)
    y = torch.rand(5, 2, 30, 31, generator=g)
    p = y + 0.01 * torch.randn(5, 2, 30, 31, generator=g)
    for yy, pp in ((y, p), (y.transpose(2, 3), p.transpose(2, 3)), (y[:, :, ::2], p[:, :, ::2])):
        got = GM.MMDMetric()(yy.to(DEV, dtype), pp.to(DEV, dtype))
        assert got.dtype == dtype
        want = M.mmd(yy.to(dtype), pp.to(dtype))
        # a 16-bit result is the fp32 value rounded to the inputs' dtype, as the reference returns it
        # (fp16 holds ~2e-5 as a subnormal, 2^-24 apart)
        tol = torch.finfo(dtype).eps * float(want) + 2.0 ** -24 if dtype in (torch.float16, torch.bfloat16) else \
            1e-6 * float(want)
        assert abs(float(got) - float(want)) <= tol


def test_repeat_calls_are_bit_identical(cuda_device):
    a, b = (t.to(DEV) for t in inputs(CASES["ms_brain"]))
    for m in (GM.SSIMMetric(3), GM.MultiScaleSSIMMetric(3, kernel_size=4)):
        assert torch.equal(m(a, b), m(a, b))
    y, p = (t.to(DEV) for t in inputs(CASES["mmd_brain"]))
    assert torch.equal(GM.MMDMetric()(y, p), GM.MMDMetric()(y, p))


def test_cuda_graph_capture(cuda_device):
    a, b = (t.to(DEV) for t in inputs(CASES["tutorial_ms"]))
    ssim, ms, mmd = GM.SSIMMetric(2, kernel_size=4), GM.MultiScaleSSIMMetric(2, kernel_size=4), GM.MMDMetric()
    eager = [ssim(a, b), ms(a, b), mmd(a, b)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        warm = [ssim(a, b), ms(a, b), mmd(a, b)]
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = [ssim(a, b), ms(a, b), mmd(a, b)]
    a.copy_(b)
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(w, e) for w, e in zip(warm, eager))
    same = [ssim(a, b), ms(a, b), mmd(a, b)]
    assert all(torch.equal(o, e) for o, e in zip(out, same))
    assert float(out[2]) == 0.0 and torch.allclose(out[0], torch.ones_like(out[0]))


def test_cpu_tensors_raise(cuda_device):
    with pytest.raises(RuntimeError, match="CUDA"):
        GM.MultiScaleSSIMMetric(2, kernel_size=3, weights=[0.5, 0.5])(torch.rand(1, 1, 16, 16), torch.rand(1, 1, 16, 16))


def test_kernel_too_large_for_a_tile_raises(cuda_device):
    x = torch.rand(1, 1, 128, 128, 128, device=DEV)
    with pytest.raises(NotImplementedError):
        GM.SSIMMetric(3, kernel_size=120, kernel_type="uniform")(x, x)
