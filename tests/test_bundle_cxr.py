"""The chest X-ray text-to-image bundle (model-zoo/models/cxr_image_synthesis_latent_diffusion_model) on this package:
its guided ``Sampler`` against the fixture written by the reference's own scripts/sampler.py at the published size
(tests/golden/make_golden_cxr.py), its ``JPGSaver`` against a numpy restatement, the unmodified ``inference.json``
(stored as tests/golden/cxr_ldm_inference.json) through the resolver and the CLI, with the offline prompt-embedding
route.  CPU tests need no GPU; the ``gpu`` tests run the bundle on the CUDA path."""
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import torch_oracle as O
from tests import cpu_backend, golden
from tests.fixture_checks import TOL_MAX, TOL_REL, TOL_TRAJ, close, rel, relmax
from tests.golden import configs as G

GOLD = Path(__file__).resolve().parent / "golden"
CXR_JSON = GOLD / "cxr_ldm_inference.json"
# the file's imports without transformers: the offline route, with the prompt embeddings overridden
OFFLINE_IMPORTS = ["$import torch", "$from datetime import datetime", "$from pathlib import Path"]


def _fixture():
    return golden.load("g_bundle_cxr_ldm")


def _guided(eps2, g):
    uncond, text = eps2.chunk(2)
    return uncond + g * (text - uncond)


def _recipe_states(fx):
    """The fixture's weights: the seeded recipe drawn over this package's modules (same keys and shapes as the
    reference's)."""
    from generativemodels_b200.networks.nets import AutoencoderKL, DiffusionModelUNet
    unet = DiffusionModelUNet(**fx["unet_kwargs"]).eval()
    ae = AutoencoderKL(**fx["aekl_kwargs"]).eval()
    assert (sum(p.numel() for p in unet.parameters()), sum(p.numel() for p in ae.parameters())) == tuple(fx["n_params"])
    return unet, G.recipe_state_dict(unet, fx["unet_seed"]), ae, G.recipe_state_dict(ae, fx["aekl_seed"])


def _scheduler(fx):
    from generativemodels_b200.networks.schedulers import DDIMScheduler
    s = DDIMScheduler(**fx["scheduler_kwargs"])
    s.set_timesteps(num_inference_steps=fx["steps"])
    assert [int(t) for t in s.timesteps] == fx["timesteps"]
    return s


def _recording(scheduler):
    """Wrap ``scheduler.step`` to record the guided model output it is given and the latent it returns."""
    guided, latents = [], []
    step = scheduler.step

    def rec(model_output, t, sample, *a, **k):
        nxt, x0 = step(model_output, t, sample, *a, **k)
        guided.append(model_output.clone())
        latents.append(nxt.clone())
        return nxt, x0
    scheduler.step = rec
    return guided, latents


def _offline_overrides(root, **extra):
    return {"imports": OFFLINE_IMPORTS, "bundle_root": str(root), "load_autoencoder": "$None",
            "load_diffusion": "$None", **extra}


# ------------------------------------------------------------------------------------------------------------------
# oracle pinned to the reference's own bundle script
# ------------------------------------------------------------------------------------------------------------------
def test_oracle_guided_sampler_matches_reference_fixture():
    """The guided sampler restated on the fp32 torch oracle reproduces the reference's run step by step."""
    fx = _fixture()
    _, unet_sd, _, ae_sd = _recipe_states(fx)
    sched = O.DDIMOracle(**fx["scheduler_kwargs"])
    sched.set_timesteps(fx["steps"])
    ucfg, acfg = G.unet_oracle_cfg(fx["unet_kwargs"]), G.aekl_oracle_cfg(fx["aekl_kwargs"])
    noise = fx["noise"]
    with torch.no_grad():
        for k, t in enumerate(sched.timesteps):
            eps2 = O.unet_forward(unet_sd, ucfg, torch.cat([noise] * 2), torch.Tensor((t,)).long(),
                                  context=fx["prompt_embeds"])
            assert rel(eps2, fx["model_outputs"][k]) < 1e-4, (k, rel(eps2, fx["model_outputs"][k]))
            noise, _ = sched.step(_guided(eps2, fx["guidance_scale"]), int(t), noise)
            assert rel(noise, fx["latents"][k]) < 1e-4, (k, rel(noise, fx["latents"][k]))
        image = O.autoencoderkl_decode(ae_sd, acfg, noise / fx["scale_factor"])
    assert image.shape == fx["image"].shape and rel(image, fx["image"]) < 1e-4, rel(image, fx["image"])


def test_guidance_and_scheduler_teacher_forced_cpu(monkeypatch):
    """The package's DDIMScheduler (v-prediction, the file's schedule) on the reference's own UNet outputs."""
    cpu_backend.install(monkeypatch)
    fx = _fixture()
    s = _scheduler(fx)
    x = fx["noise"]
    for k, t in enumerate(s.timesteps):
        x, _ = s.step(_guided(fx["model_outputs"][k], fx["guidance_scale"]), t, x)
        assert rel(x, fx["latents"][k]) < 1e-5, (k, rel(x, fx["latents"][k]))


# ------------------------------------------------------------------------------------------------------------------
# resolver, script sets and CLI
# ------------------------------------------------------------------------------------------------------------------
def test_script_set_selection():
    from generativemodels_b200.bundle import CXRSampler, JPGSaver, NiftiSaver, Sampler
    from generativemodels_b200.bundle.config import BUNDLES, BundleConfig, _locate, detect_bundle
    sampler = {"s": {"_target_": "scripts.sampler.Sampler"}}
    # the default is the brain set, for dicts and for paths outside a bundle directory alike
    assert BundleConfig(dict(sampler)).bundle == "brain" and type(BundleConfig(dict(sampler)).get("s")) is Sampler
    assert detect_bundle(None) == "brain" and detect_bundle(str(CXR_JSON)) == "brain"
    assert type(BundleConfig(dict(sampler), bundle="cxr").get("s")) is CXRSampler
    assert CXRSampler is not Sampler and not issubclass(CXRSampler, Sampler)
    assert _locate("scripts.saver.NiftiSaver") is NiftiSaver
    assert _locate("scripts.saver.JPGSaver", BUNDLES["cxr"][1]) is JPGSaver
    with pytest.raises(ModuleNotFoundError):                   # the brain set does not map the CXR saver
        BundleConfig({"v": {"_target_": "scripts.saver.JPGSaver", "output_dir": "."}}).get("v")
    with pytest.raises(ValueError, match="unknown bundle"):
        BundleConfig({}, bundle="mednist")
    # detection from the reference bundle's directory name
    for name, (dirname, _) in BUNDLES.items():
        assert detect_bundle(f"/x/model-zoo/models/{dirname}/configs/inference.json") == name
        assert detect_bundle(Path("rel") / dirname / "configs" / "inference.json") == name


def test_detected_from_path_and_brain_unchanged(monkeypatch, tmp_path):
    cpu_backend.install(monkeypatch)
    from generativemodels_b200.bundle import CXRSampler, Sampler
    from generativemodels_b200.bundle.config import BundleConfig
    cfg_dir = tmp_path / "cxr_image_synthesis_latent_diffusion_model" / "configs"
    cfg_dir.mkdir(parents=True)
    (cfg_dir / "inference.json").write_text(CXR_JSON.read_text())
    cfg = BundleConfig(str(cfg_dir / "inference.json"), _offline_overrides(tmp_path))
    assert cfg.bundle == "cxr" and type(cfg.get("sampler")) is CXRSampler
    assert BundleConfig(str(cfg_dir / "inference.json"), _offline_overrides(tmp_path), bundle="brain").bundle == "brain"
    brain = BundleConfig(str(GOLD / "brain_ldm_inference.json"), {"load_autoencoder": "$None", "load_diffusion": "$None",
                                                                   "device": "$'cpu'"})
    assert brain.bundle == "brain" and type(brain.get("sampler")) is Sampler


def test_cxr_inference_json_resolves_offline(monkeypatch, tmp_path):
    """The unmodified file resolves on this package without transformers: ``imports`` and ``prompt_embeds``
    overridden, and lazy resolution never builds ``tokenizer`` / ``text_encoder``."""
    from generativemodels_b200.bundle import CXRSampler, JPGSaver
    from generativemodels_b200.bundle.config import BundleConfig
    from generativemodels_b200.networks.nets import AutoencoderKL, DiffusionModelUNet
    from generativemodels_b200.networks.schedulers import DDIMScheduler
    monkeypatch.setitem(sys.modules, "transformers", None)    # import transformers -> ImportError
    raw = json.loads(CXR_JSON.read_text())
    with pytest.raises(ImportError):                           # the file's own imports need transformers
        BundleConfig(str(CXR_JSON), {"device": "$'cpu'"}, bundle="cxr").get("prompt_list")
    emb = tmp_path / "emb.pt"
    torch.save(torch.randn(2, 77, 1024), emb)
    cfg = BundleConfig(str(CXR_JSON), _offline_overrides(tmp_path, device="$'cpu'",
                                                         prompt_embeds=f"$torch.load({str(emb)!r}).to(@device)"),
                       bundle="cxr")
    assert torch.equal(cfg.get("prompt_embeds"), torch.load(emb))
    sampler, sched, saver = cfg.get("sampler"), cfg.get("scheduler"), cfg.get("saver")
    assert type(sampler) is CXRSampler and isinstance(saver, JPGSaver) and (tmp_path / "output").is_dir()
    assert isinstance(sched, DDIMScheduler) and sched.prediction_type == "v_prediction" and len(sched.timesteps) == 50
    assert tuple(cfg.get("noise").shape) == (1, 3, 64, 64) and cfg.get("prompt_list") == ["", raw["prompt"]]
    ae, unet = cfg.get("autoencoder"), cfg.get("diffusion")
    assert isinstance(ae, AutoencoderKL) and isinstance(unet, DiffusionModelUNet)
    assert unet.in_channels == 3 and list(unet.block_out_channels) == [256, 512, 768]
    assert "tokenizer" not in cfg._resolved and "text_encoder" not in cfg._resolved
    # the reference's quirk: the file's guidance_scale is never passed to sampling_fn
    assert "guidance_scale" not in raw["sample"] and cfg.get("guidance_scale") == 7.0
    assert BundleConfig(str(CXR_JSON), {"guidance_scale": 3.0}, bundle="cxr").get("guidance_scale") == 3.0


def test_cxr_cli_end_to_end_cpu(monkeypatch, tmp_path):
    """``python -m generativemodels_b200.bundle run save_jpg save --bundle cxr ...`` on the CPU stand-in, at reduced
    widths and two steps: writes the .jpg and the .pt."""
    cpu_backend.install(monkeypatch)
    pytest.importorskip("PIL")
    from PIL import Image

    from generativemodels_b200.bundle.__main__ import main
    monkeypatch.setitem(sys.modules, "transformers", None)
    torch.save(torch.randn(2, 77, 1024), tmp_path / "emb.pt")
    args = ["run", "save_jpg", "save", "--config_file", str(CXR_JSON), "--bundle", "cxr",
            "--imports", json.dumps(OFFLINE_IMPORTS), "--bundle_root", str(tmp_path), "--device", "$'cpu'",
            "--load_autoencoder", "$None", "--load_diffusion", "$None", "--out_file", "cxr",
            "--prompt_embeds", f"$torch.load({str(tmp_path / 'emb.pt')!r})",
            "--diffusion_def#num_channels", "[32, 64, 64]", "--diffusion_def#num_head_channels", "[0, 64, 64]",
            "--autoencoder_def#num_channels", "[32, 32, 32, 32]",
            "--set_timesteps", "$@scheduler.set_timesteps(num_inference_steps=2)"]
    assert main(args) == 0
    sample = torch.load(tmp_path / "output" / "cxr.pt")
    assert tuple(sample.shape) == (1, 1, 512, 512) and bool(torch.isfinite(sample).all())
    with Image.open(tmp_path / "output" / "cxr.jpg") as im:
        assert im.format == "JPEG" and im.size == (512, 512) and im.mode == "L"
    assert main(["run", "save", "--config_file", str(CXR_JSON), "--bundle", "nope"]) == 2


# ------------------------------------------------------------------------------------------------------------------
# JPGSaver
# ------------------------------------------------------------------------------------------------------------------
def _jpg_restatement(image: torch.Tensor) -> np.ndarray:
    """scripts/saver.py:14-16 in numpy."""
    a = np.clip(image.cpu().numpy(), 0, 1)
    return (a * 255).astype(np.uint8)[0, 0]


def _saved_array(monkeypatch, saver, image, name):
    from PIL import Image
    seen = []
    fromarray = Image.fromarray
    monkeypatch.setattr(Image, "fromarray", lambda a, *r, **k: (seen.append(a.copy()), fromarray(a, *r, **k))[1])
    saver.save(image, name)
    assert len(seen) == 1
    return seen[0]


def test_jpg_saver_array_equals_numpy_cpu(monkeypatch, tmp_path):
    pytest.importorskip("PIL")
    from PIL import Image

    from generativemodels_b200.bundle import JPGSaver
    g = torch.Generator().manual_seed(5)
    image = torch.randn(1, 1, 96, 80, generator=g) * 0.6 + 0.5         # a quarter of the values are clipped
    image[0, 0, 0, :4] = torch.tensor([0.0, 1.0, 254.5 / 255, 0.99 / 255])
    saver = JPGSaver(str(tmp_path))
    got = _saved_array(monkeypatch, saver, image, "img")
    want = _jpg_restatement(image)
    assert got.dtype == np.uint8 and got.shape == (96, 80) and np.array_equal(got, want)
    assert got[0, :4].tolist() == want[0, :4].tolist() == [0, 255, 254, 0]   # truncation, not rounding
    with Image.open(tmp_path / "img.jpg") as im:
        assert im.format == "JPEG" and im.size == (80, 96)


def test_jpg_saver_without_pil(monkeypatch, tmp_path):
    # importing the bundle package needs no PIL (a fresh interpreter in which PIL cannot be imported)
    code = ("import sys; sys.modules['PIL'] = None; import generativemodels_b200.bundle as b; "
            "assert b.JPGSaver and 'PIL.Image' not in sys.modules")
    root = Path(__file__).resolve().parents[1]
    subprocess.run([sys.executable, "-c", code], cwd=root, check=True, env={**os.environ, "PYTHONPATH": str(root)})
    from generativemodels_b200.bundle import JPGSaver
    monkeypatch.setitem(sys.modules, "PIL", None)
    monkeypatch.setitem(sys.modules, "PIL.Image", None)
    with pytest.raises(ImportError, match="Pillow"):
        JPGSaver(str(tmp_path)).save(torch.zeros(1, 1, 8, 8), "x")
    assert not (tmp_path / "x.jpg").exists()


# ------------------------------------------------------------------------------------------------------------------
# CUDA path
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cxr_models():
    fx = _fixture()
    unet, _, ae, _ = _recipe_states(fx)
    return fx, ae.cuda(), unet.cuda()


def _run(fx, ae, unet, graph):
    from generativemodels_b200.bundle import CXRSampler
    sched = _scheduler(fx)
    guided, latents = _recording(sched)
    image = CXRSampler(use_cuda_graph=graph).sampling_fn(fx["noise"].cuda(), ae, unet, sched,
                                                         fx["prompt_embeds"].cuda())
    torch.cuda.synchronize()
    return image, guided, latents


@pytest.mark.gpu
def test_cxr_sampler_golden_gpu(cxr_models):
    """Full size against the reference's fp32 run: the guided output and the latent of every step, and the image."""
    fx, ae, unet = cxr_models
    ts = torch.Tensor((fx["timesteps"][0],)).long().cuda()
    eps2 = unet(torch.cat([fx["noise"]] * 2).cuda(), timesteps=ts, context=fx["prompt_embeds"].cuda())
    image, guided, latents = _run(fx, ae, unet, graph=True)
    assert len(latents) == fx["steps"]
    # (name, got, want, rel-L2 tolerance): the first step's UNet output is a forward from the reference's own input;
    # the guided outputs (guidance 7 amplifies the text - uncond difference, as in C5), latents and image are
    # trajectory values
    checks = [("UNet output, first step (uncond | text)", eps2, fx["model_outputs"][0], TOL_REL)]
    for k in range(fx["steps"]):
        checks.append((f"guided output, step {k + 1}", guided[k], _guided(fx["model_outputs"][k], fx["guidance_scale"]),
                       TOL_TRAJ))
        checks.append((f"latent after step {k + 1}", latents[k], fx["latents"][k], TOL_TRAJ))
    checks.append(("decoded image", image, fx["image"], TOL_TRAJ))
    print("CXR fixture (rel-L2, max-abs):", {n: (f"{rel(a, b):.3e}", f"{relmax(a, b):.3e}") for n, a, b, _ in checks})
    for name, got, want, tol in checks:
        close(got, want, "CXR " + name, tol, TOL_MAX if tol == TOL_REL else 2 * tol)


@pytest.mark.gpu
def test_cxr_graph_replay_bit_identical_to_eager(cxr_models):
    fx, ae, unet = cxr_models
    eager = _run(fx, ae, unet, graph=False)
    replay = _run(fx, ae, unet, graph=True)
    assert torch.equal(eager[0], replay[0])
    for a, b in zip(eager[1] + eager[2], replay[1] + replay[2]):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_cxr_jpg_saver_gpu_equals_numpy(monkeypatch, cxr_models, tmp_path):
    pytest.importorskip("PIL")
    from generativemodels_b200.bundle import JPGSaver
    fx, ae, _ = cxr_models
    image = ae.decode_stage_2_outputs(fx["latents"][-1].cuda() / fx["scale_factor"]) * 0.25 + 0.5   # ~half clipped
    assert image.is_cuda
    got = _saved_array(monkeypatch, JPGSaver(str(tmp_path)), image, "cxr")
    assert np.array_equal(got, _jpg_restatement(image)) and got.shape == (512, 512)
    assert 0 < int((got == 0).sum()) + int((got == 255).sum()) < got.size


@pytest.mark.gpu
def test_cxr_cli_end_to_end_gpu(monkeypatch, tmp_path):
    """The published-size bundle with random weights: 50 guided steps on the device, .jpg and .pt written."""
    pytest.importorskip("PIL")
    from PIL import Image

    from generativemodels_b200.bundle.__main__ import main
    monkeypatch.setitem(sys.modules, "transformers", None)
    torch.save(torch.randn(2, 77, 1024), tmp_path / "emb.pt")
    args = ["run", "save_jpg", "save", "--config_file", str(CXR_JSON), "--bundle", "cxr",
            "--imports", json.dumps(OFFLINE_IMPORTS), "--bundle_root", str(tmp_path), "--out_file", "cxr",
            "--load_autoencoder", "$None", "--load_diffusion", "$None",
            "--prompt_embeds", f"$torch.load({str(tmp_path / 'emb.pt')!r}).to(@device)"]
    assert main(args) == 0
    sample = torch.load(tmp_path / "output" / "cxr.pt")
    assert tuple(sample.shape) == (1, 1, 512, 512) and sample.is_cuda and bool(torch.isfinite(sample).all())
    with Image.open(tmp_path / "output" / "cxr.jpg") as im:
        assert im.format == "JPEG" and im.size == (512, 512) and im.mode == "L"
