"""Every C-ABI call of the sample-quality metrics, FID, the perceptual loss and the spectral / adversarial losses,
checked against its float64 contract reading (tests/abi_shadow.py).

The metric and loss GPU tests compare module outputs with fixtures and emulator sweeps at tolerances sized for the
whole result.  Here each call a module makes, as users call it, runs on the GPU and on the CPU stand-in with the
call's own device inputs, under the per-element bounds of tests/{metrics,fid,perceptual,losses}_emulator.py; SSIM's
partial slots are checked summed per item, and every byte outside the outputs and the declared scratch must survive.
The cases are the committed fixtures' inputs plus one sized case per family at the brain-LDM volume 160 x 224 x 160;
the perceptual networks are built inside the shadowed call, so their BatchNorm folding and weight repacking are
checked too.  The last test asserts which entry points and kernel paths the file reached and prints the largest
err / tol per entry point."""
import time
import warnings

import pytest
import torch

from generativemodels_b200 import metrics as GM
from generativemodels_b200 import ops
from tests import abi_shadow

pytestmark = pytest.mark.gpu

REACHED = set()
CALLS = []
DEV = "cuda"
BRAIN = (1, 1, 160, 224, 160)


def shadowed(monkeypatch, name, fn):
    """Run fn() with every C-ABI call shadowed; assert no violation; print the per-entry table."""
    torch.cuda.synchronize()
    t0 = time.time()
    with abi_shadow.shadow(monkeypatch) as sh, torch.no_grad():
        out = fn()
    REACHED.update(sh.paths())
    CALLS.extend(sh.calls)
    print(f"\n== {name}: {len(sh.calls)} calls, {time.time() - t0:.1f} s\n{sh.table()}")
    assert sh.calls, f"{name}: no C-ABI call was shadowed"
    assert not sh.violations, f"{name}: {len(sh.violations)} violations\n{sh.report()}"
    return out


def _brain_pair(seed):
    """A smooth brain-sized volume and a noisy copy, as tests/test_losses_gpu.py builds them."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    coarse = torch.rand(1, 1, 20, 28, 20, device=DEV, generator=g)
    x = torch.nn.functional.interpolate(coarse, size=BRAIN[2:], mode="trilinear", align_corners=False)
    return x, (x + 0.01 * torch.randn(x.shape, device=DEV, generator=g)).clamp(0, 1)


# ------------------------------------------------------------------------------------------------------------------
# SSIM, MS-SSIM, MMD: the fixture cases of tests/golden/make_golden_metrics.py, maps, views, every tile height
# ------------------------------------------------------------------------------------------------------------------
def _metric_cases():
    from tests.golden.make_golden_metrics import CASES
    return CASES


@pytest.mark.parametrize("name", list(_metric_cases()))
def test_metric_fixture_cases(cuda_device, monkeypatch, name):
    from tests.golden.make_golden_metrics import inputs
    case = _metric_cases()[name]
    a, b = (t.to(DEV) for t in inputs(case))
    if case["kind"] == "mmd":
        shadowed(monkeypatch, name, lambda: GM.MMDMetric()(a, b))
    else:
        cls = GM.SSIMMetric if case["kind"] == "ssim" else GM.MultiScaleSSIMMetric
        shadowed(monkeypatch, name, lambda: cls(**case["kw"])(a, b))


# (spatial_dims, shape, kernel_size, kernel_type, sigma, dtype, strided): the maps in 2-D and 3-D, a strided fp16 view,
# and kernel sizes whose tiles are 8 (k = 11), 4 (k = 41), 2 (k = 60) and 1 (k = 90) rows high in 3-D
MAP_CASES = {
    "2d_maps": (2, (2, 3, 37, 29), 4, "gaussian", 1.5, torch.float32, False),
    "3d_maps": (3, (1, 2, 20, 18, 23), (5, 3, 7), "gaussian", (1.0, 0.5, 2.0), torch.float32, False),
    "2d_fp16_strided": (2, (2, 2, 30, 45), 7, "uniform", 1.5, torch.float16, True),
    "3d_bf16_strided": (3, (1, 1, 20, 18, 23), 4, "gaussian", 1.5, torch.bfloat16, True),
    "aniso_3x9": (2, (1, 2, 40, 41), (3, 9), "gaussian", (0.8, 2.0), torch.float64, False),
    "tile8_k11": (3, (1, 1, 24, 21, 26), 11, "uniform", 1.5, torch.float32, False),
    "tile4_k41": (3, (1, 1, 46, 44, 45), 41, "gaussian", 6.0, torch.float32, False),
    "tile2_k60": (3, (1, 1, 62, 61, 64), 60, "uniform", 1.5, torch.float32, False),
    "tile1_k90": (3, (1, 1, 91, 92, 94), 90, "uniform", 1.5, torch.float32, False),
}


@pytest.mark.parametrize("name", list(MAP_CASES))
def test_ssim_maps_views_and_tiles(cuda_device, monkeypatch, name):
    from tests.test_metrics_gpu import _views
    sd, shape, ks, kt, sig, dtype, strided = MAP_CASES[name]
    a, b = _views(shape, dtype, strided, 7)

    def run():
        GM.compute_ssim_and_cs(a, b, sd, kernel_type=kt, kernel_size=ks, kernel_sigma=sig)
        GM.SSIMMetric(sd, kernel_type=kt, kernel_size=ks, kernel_sigma=sig)(a, b)
    shadowed(monkeypatch, name, run)


def test_ms_ssim_fp64_inputs_and_area_pooling(cuda_device, monkeypatch):
    """MS-SSIM of fp64 inputs: the AREA pooling between scales reads fp64 and writes fp32."""
    from tests.test_metrics_gpu import _views
    a, b = _views((1, 2, 37, 41, 35), torch.float64, False, 8)
    shadowed(monkeypatch, "ms-ssim fp64", lambda: GM.MultiScaleSSIMMetric(3, kernel_size=(3, 2, 3),
                                                                          weights=[0.2, 0.3, 0.5])(a, b))


def test_mmd_views_and_fp16(cuda_device, monkeypatch):
    g = torch.Generator().manual_seed(5)
    y = torch.rand(5, 2, 30, 31, generator=g)
    p = y + 0.01 * torch.randn(5, 2, 30, 31, generator=g)
    yd, pd = y.to(DEV), p.to(DEV)
    shadowed(monkeypatch, "mmd transposed", lambda: GM.MMDMetric()(yd.transpose(2, 3), pd.transpose(2, 3)))
    shadowed(monkeypatch, "mmd fp16", lambda: GM.MMDMetric()(yd.half(), pd.half()))


# ------------------------------------------------------------------------------------------------------------------
# FID
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tutorial_1000x2048", "large_4000x2048", "singular_30x256_vs_40x256", "fp16"])
def test_fid_cases(cuda_device, monkeypatch, name):
    from tests.golden.make_golden_fid import CASES, inputs
    p, y = (t.to(DEV) for t in inputs(CASES[name]))
    shadowed(monkeypatch, name, lambda: GM.FIDMetric()(p, y))


def test_frechet_details(cuda_device, monkeypatch):
    """The eigenvalue and rank outputs, which FIDMetric does not ask for."""
    from tests.golden.make_golden_fid import CASES, inputs
    p, y = (t.to(DEV) for t in inputs(CASES["singular_30x256_vs_40x256"]))
    mp, sp = ops.fid_moments(p)
    my, sy = ops.fid_moments(y)
    shadowed(monkeypatch, "frechet details", lambda: ops.frechet(mp, sp, my, sy, details=True))


# ------------------------------------------------------------------------------------------------------------------
# PerceptualLoss(network_type="resnet50"): the network is built inside the shadowed call
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def perceptual_fixture():
    from tests import golden
    return golden.load("g_perceptual")


@pytest.mark.parametrize("name", ["2d_1ch", "2d_3ch", "odd", "fake3d"])
def test_perceptual_fixture_cases(cuda_device, monkeypatch, perceptual_fixture, name):
    from tests import perceptual_checks as K
    from tests.golden import make_golden_perceptual as G
    rec = perceptual_fixture[name]
    x, y = rec["x"].to(DEV), rec["y"].to(DEV)
    kw = dict(spatial_dims=3, is_fake_3d=True, fake_3d_ratio=0.5) if name == "fake3d" else {}

    def run():
        m = K.networks(perceptual_fixture, DEV, **kw)[0]
        torch.manual_seed(G.SLICE_SEED)
        return m(x, y)
    shadowed(monkeypatch, f"perceptual {name}", run)


def test_perceptual_brain_volume(cuda_device, monkeypatch, perceptual_fixture):
    """2.5-D at 160 x 224 x 160: 1 + 2 + 1 slices (fake_3d_ratio 0.01) of 224 x 160, 160 x 160 and 160 x 224; the stem
    GEMM has more than 8192 rows per image, so the igemm check compares its sampled rows.  The ratio keeps the float64
    emulation of the network's GEMMs to about a minute."""
    from tests import perceptual_checks as K
    x, y = _brain_pair(31)

    def run():
        m = K.networks(perceptual_fixture, DEV, spatial_dims=3, is_fake_3d=True, fake_3d_ratio=0.01)[0]
        torch.manual_seed(0)
        return m(x, y)
    shadowed(monkeypatch, "perceptual brain volume", run)


# ------------------------------------------------------------------------------------------------------------------
# JukeboxLoss, PatchAdversarialLoss
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def losses_fixture():
    from tests.golden import load
    return load("g_losses")


def test_jukebox_fixture_cases(cuda_device, monkeypatch, losses_fixture):
    from generativemodels_b200.losses import JukeboxLoss
    for name, case in losses_fixture["spectral"].items():
        x, y = case["x"].float().to(DEV), case["y"].float().to(DEV)
        for norm, red in case["runs"]:
            loss = JukeboxLoss(case["spatial_dims"], fft_signal_size=case["fft_signal_size"], fft_norm=norm,
                               reduction=red)
            shadowed(monkeypatch, f"jukebox {name} {norm} {red}", lambda: loss(x, y))


def test_jukebox_brain_volume(cuda_device, monkeypatch):
    from generativemodels_b200.losses import JukeboxLoss
    x, y = _brain_pair(32)
    shadowed(monkeypatch, "jukebox brain volume", lambda: JukeboxLoss(3, reduction="mean")(x, y))


def _discriminator_logits():
    from generativemodels_b200.networks.nets import MultiScalePatchDiscriminator
    torch.manual_seed(0)
    net = MultiScalePatchDiscriminator(num_d=3, num_layers_d=2, spatial_dims=2, num_channels=8, in_channels=1,
                                       out_channels=1).eval().to(DEV)
    with torch.no_grad():
        logits, _ = net(torch.rand(2, 1, 128, 128, device=DEV))
    return [t[-1] if isinstance(t, list) else t for t in logits]


def test_adversarial_on_multiscale_discriminator(cuda_device, monkeypatch):
    from generativemodels_b200.losses import PatchAdversarialLoss
    from tests.test_losses_cpu import CRIT
    logits = _discriminator_logits()
    for crit, noact in CRIT:
        for red in ("mean", "sum", "none"):
            loss = PatchAdversarialLoss(reduction=red, criterion=crit, no_activation_leastsq=noact)
            for real in (True, False):
                for disc in (True, False):
                    with warnings.catch_warnings():
                        warnings.simplefilter("ignore")
                        shadowed(monkeypatch, f"adversarial {crit} noact={noact} {red} real={real} disc={disc}",
                                 lambda: loss(logits, target_is_real=real, for_discriminator=disc))


def test_adversarial_fp16_and_strided_logits(cuda_device, monkeypatch):
    from generativemodels_b200.losses import PatchAdversarialLoss
    logits = _discriminator_logits()
    x16 = [t.half() for t in logits]
    wide = [torch.cat([t, t], dim=-1)[..., ::2] for t in logits]          # a step along the last axis
    assert not wide[0].is_contiguous()
    for crit in ("bce", "least_squares", "hinge"):
        for red in ("mean", "none"):
            loss = PatchAdversarialLoss(reduction=red, criterion=crit)
            shadowed(monkeypatch, f"adversarial fp16 {crit} {red}",
                     lambda: loss(x16, target_is_real=True, for_discriminator=True))
            shadowed(monkeypatch, f"adversarial strided {crit} {red}",
                     lambda: loss(wide, target_is_real=False, for_discriminator=True))


# ------------------------------------------------------------------------------------------------------------------
# coverage of the file
# ------------------------------------------------------------------------------------------------------------------
MUST_REACH = {
    # the 11 entry points of b200gen_metrics.h, b200gen_fid.h, b200gen_perceptual.h and b200gen_losses.h
    "b200_ssim", "b200_ssim_combine", "b200_mmd", "b200_fid_moments", "b200_frechet", "b200_perceptual_prep",
    "b200_perceptual_distance", "b200_perceptual_mean", "b200_spectral_fft", "b200_spectral_distance",
    "b200_adversarial",
    # the ResNet-50 on b200gen.h: the stem's tap gather (K = 147), max-pooling 3x3 s2 p1, the folded and repacked
    # weights, the last block's fp32 store at 2048 columns; MS-SSIM's AREA pooling
    "b200_tap_gather", "b200_pool_s2", "b200_batchnorm_fold", "b200_repack_weight", "b200_interpolate",
    "igemm staged",
}
RAN = set()


@pytest.fixture(autouse=True)
def _ran(request):
    yield
    RAN.add(request.node.name)


def _cases_in_file():
    n = 0
    for name, fn in globals().items():
        if name.startswith("test_") and name != "test_zz_paths_reached":
            marks = [m for m in getattr(fn, "pytestmark", []) if m.name == "parametrize"]
            n += len(marks[0].args[1]) if marks else 1
    return n


def test_zz_paths_reached(cuda_device):
    """The paths the whole file reached (REACHED is filled by the cases above, in this process) and the per-entry table
    of all its calls (calls, distinct argument shapes, largest err / tol): skipped when only a selection of the cases
    ran."""
    RAN.discard("test_zz_paths_reached")
    if len(RAN) < _cases_in_file():
        pytest.skip(f"only {len(RAN)} of the file's {_cases_in_file()} cases ran")
    print(f"\nstorage {ops.H16}, the whole file:\n{abi_shadow.Shadow(None, None, calls=CALLS).table()}")
    print("paths reached:", ", ".join(sorted(REACHED)))
    missing = MUST_REACH - REACHED
    assert not missing, f"the modules no longer reach {sorted(missing)}"
