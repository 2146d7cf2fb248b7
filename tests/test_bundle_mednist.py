"""The MedNIST DDPM bundle (model-zoo/models/mednist_ddpm) on this package: its unmodified YAML configs (common.yaml +
infer.yaml, with metadata.json as the meta file; stored as tests/golden/mednist_ddpm_*) through the resolver and the
CLI in the notebook's call shape, and its 1000-step DDPM sample against the reference's own fp32 run
(tests/golden/make_golden_mednist.py).  CPU tests need no GPU; the ``gpu`` tests run the bundle on the CUDA path."""
import json
import sys
import types
from pathlib import Path

import pytest
import torch

from oracle import torch_oracle as O
from tests import cpu_backend, golden
from tests.fixture_checks import TOL_MAX, TOL_REL, close, rel, relmax
from tests.golden import configs as G

GOLD = Path(__file__).resolve().parent / "golden"
COMMON, INFER, META = (GOLD / f"mednist_ddpm_{n}" for n in ("common.yaml", "infer.yaml", "metadata.json"))
CONFIGS = [str(COMMON), str(INFER)]
# common.yaml's imports without monai: the offline route (MONAI is only needed by infer.yaml's save_trans)
OFFLINE_IMPORTS = ["$import os", "$import datetime", "$import torch", "$import scripts", "$import generative",
                   "$import torch.distributed as dist"]


def _fixture():
    return golden.load("g_bundle_mednist_ddpm")


def _generative_modules():
    return {k: v for k, v in sys.modules.items() if k == "generative" or k.startswith("generative.")}


@pytest.fixture
def scripts_pkg(monkeypatch, tmp_path):
    """An empty ``scripts`` package on sys.path, so that ``$import scripts`` resolves (the bundle's own only holds a
    training helper).  The file's ``$import generative`` installs this repository's ``generative`` alias; it is undone
    afterwards, so that tests importing the reference under that name still find the reference."""
    root = tmp_path / "bundle_scripts"
    (root / "scripts").mkdir(parents=True)
    (root / "scripts" / "__init__.py").write_text("")
    monkeypatch.delitem(sys.modules, "scripts", raising=False)
    monkeypatch.syspath_prepend(str(root))
    monkeypatch.setattr(sys, "meta_path", list(sys.meta_path))
    before = _generative_modules()
    yield root
    for k in set(_generative_modules()) - set(before):
        del sys.modules[k]
    sys.modules.update(before)


def _noise_generator(seed: int, t: int) -> torch.Generator:
    """A generator in the state the global one is in when the bundle's sample reaches the step at timestep ``t``:
    after the file's ``torch.rand`` noise and one ``randn`` per earlier step."""
    g = torch.Generator().manual_seed(seed)
    torch.rand(1, 1, 64, 64, generator=g)
    for _ in range(999 - t):
        torch.randn(1, 1, 64, 64, generator=g)
    return g


def _recipe_unet(fx):
    from generativemodels_b200.networks.nets import DiffusionModelUNet
    unet = DiffusionModelUNet(**fx["unet_kwargs"]).eval()
    assert sum(p.numel() for p in unet.parameters()) == fx["n_params"]
    return unet, G.recipe_state_dict(unet, fx["unet_seed"])


# ------------------------------------------------------------------------------------------------------------------
# config loading
# ------------------------------------------------------------------------------------------------------------------
def test_yaml_loading(monkeypatch, tmp_path):
    import yaml

    from generativemodels_b200.bundle.config import BundleConfig
    cfg = BundleConfig(str(COMMON))
    assert cfg.config == yaml.safe_load(COMMON.read_text())
    assert cfg.get("image_size") == [1, 64, 64] and cfg.get("num_train_timesteps") == 1000
    (tmp_path / "c.yml").write_text("a: 1\nb: '$@a + 1'\n")
    assert BundleConfig(tmp_path / "c.yml").get("b") == 2
    monkeypatch.setitem(sys.modules, "yaml", None)
    with pytest.raises(ImportError, match="PyYAML"):
        BundleConfig(str(COMMON))
    (tmp_path / "c.json").write_text('{"a": 3}')
    assert BundleConfig(str(tmp_path / "c.json")).get("a") == 3            # JSON needs no PyYAML


def test_list_merge_later_file_wins_top_level_only(tmp_path):
    from generativemodels_b200.bundle.config import BundleConfig
    (tmp_path / "a.yaml").write_text("x: 1\nkeep: 5\nd: {p: 1, q: 2}\n")
    (tmp_path / "b.json").write_text('{"x": 2, "d": {"p": 3}}')
    a, b = str(tmp_path / "a.yaml"), str(tmp_path / "b.json")
    cfg = BundleConfig([a, b])
    assert cfg.config == {"x": 2, "keep": 5, "d": {"p": 3}}               # d replaced whole, not merged
    assert BundleConfig((b, Path(a))).config == {"x": 1, "keep": 5, "d": {"p": 1, "q": 2}}
    # the stored bundle: infer.yaml's items on top of common.yaml's
    both = BundleConfig(CONFIGS)
    assert {"network_def", "scheduler", "inferer", "noise", "sample", "testing", "testing_jpg"} <= set(both.config)
    assert "_meta_" not in both.config


def test_meta_file(tmp_path):
    from generativemodels_b200.bundle.config import BundleConfig
    meta = json.loads(META.read_text())
    cfg = BundleConfig(CONFIGS, meta_file=str(META))
    assert cfg.config["_meta_"] == meta and cfg.get("_meta_#network_data_format#inputs#image#num_channels") == 1
    assert BundleConfig(CONFIGS, meta_file={"version": "x"}).config["_meta_"] == {"version": "x"}
    (tmp_path / "own.json").write_text('{"_meta_": {"own": 1}}')           # a config's own _meta_ replaces the file's
    assert BundleConfig([str(tmp_path / "own.json")], meta_file=str(META)).config["_meta_"] == {"own": 1}


def test_cli_config_file_forms_and_meta_file(monkeypatch, tmp_path):
    from generativemodels_b200.bundle import __main__ as cli
    seen = []

    class Recorder:
        def __init__(self, config, overrides, bundle=None, meta_file=None):
            seen.append((config, overrides, bundle, meta_file))

        def run(self, *ids):
            seen[-1] += (ids,)
    monkeypatch.setattr(cli, "BundleConfig", Recorder)
    a, b = CONFIGS
    for form in (f"['{a}', '{b}']", f"'{a}', '{b}'"):
        assert cli.main(["run", "testing", "--meta_file", str(META), "--config_file", form, "--out_file", "t.pt"]) == 0
        assert seen[-1] == ([a, b], {"out_file": "t.pt"}, None, str(META), ("testing",))
    assert cli.main(["run", "testing", "--config_file", a, "--bundle", "mednist_ddpm"]) == 0
    assert seen[-1] == (a, {}, "mednist_ddpm", None, ("testing",))
    assert cli.parse_config_file("missing.json") == "missing.json"        # no literal: left to open() to report
    assert cli.parse_config_file(f"'{a}'") == a
    # a file whose name parses as a literal is still the file
    odd = tmp_path / "'x'"
    odd.write_text("{}")
    assert cli.parse_config_file(str(odd)) == str(odd)
    assert cli.main(["run", "testing", "--config_file", a, "--bundle", "mednist"]) == 2
    assert cli.main(["run", "testing", "--meta_file"]) == 2


def test_path_detection():
    from generativemodels_b200.bundle.config import BundleConfig, detect_bundle
    root = "/x/model-zoo/models/mednist_ddpm/bundle/configs"
    assert detect_bundle(f"{root}/common.yaml") == "mednist_ddpm"
    assert detect_bundle([f"{root}/common.yaml", "/elsewhere/infer.yaml"]) == "mednist_ddpm"
    assert detect_bundle(["/elsewhere/infer.yaml", f"{root}/common.yaml"]) == "brain"     # the first file decides
    assert detect_bundle(CONFIGS) == "brain" and detect_bundle(None) == "brain"
    with pytest.raises(ValueError, match="unknown bundle"):
        BundleConfig({}, bundle="mednist")


def test_dotless_target_needs_monai(monkeypatch):
    from generativemodels_b200.bundle.config import BundleConfig
    monkeypatch.setitem(sys.modules, "monai", None)
    with pytest.raises(ModuleNotFoundError) as e:
        BundleConfig({"t": {"_target_": "ScaleIntensity", "minv": 0.0}}).get("t")
    assert "MONAI" in str(e.value) and "ScaleIntensity" in str(e.value)


def test_dotless_target_resolves_in_monai(monkeypatch):
    from generativemodels_b200.bundle.config import BundleConfig
    compose_mod = types.ModuleType("monai.transforms.compose")
    intensity_mod = types.ModuleType("monai.transforms.intensity.array")

    class Compose:
        def __init__(self, transforms):
            self.transforms = transforms

    class ScaleIntensity:
        def __init__(self, minv, maxv):
            self.minv, self.maxv = minv, maxv
    Compose.__module__, ScaleIntensity.__module__ = compose_mod.__name__, intensity_mod.__name__
    compose_mod.Compose, intensity_mod.ScaleIntensity = Compose, ScaleIntensity
    transforms = types.ModuleType("monai.transforms")
    transforms.Compose, transforms.ScaleIntensity = Compose, ScaleIntensity      # re-exports, defined elsewhere
    monai = types.ModuleType("monai")
    monai.transforms = transforms
    for m in (monai, transforms, compose_mod, intensity_mod):
        monkeypatch.setitem(sys.modules, m.__name__, m)
    cfg = BundleConfig({"t": {"_target_": "Compose", "transforms": [
        {"_target_": "ScaleIntensity", "minv": 0.0, "maxv": 255.0}]}})
    t = cfg.get("t")
    assert type(t) is Compose and type(t.transforms[0]) is ScaleIntensity and t.transforms[0].maxv == 255.0
    with pytest.raises(ValueError, match="NotInMonai"):
        BundleConfig({"t": {"_target_": "NotInMonai"}}).get("t")


def test_stored_configs_resolve_offline(monkeypatch, scripts_pkg):
    """The unmodified files resolve on this package with MONAI unimportable: only ``imports`` is overridden."""
    from generativemodels_b200.bundle.config import BundleConfig
    from generativemodels_b200.inferers import DiffusionInferer
    from generativemodels_b200.networks.nets import DiffusionModelUNet
    from generativemodels_b200.networks.schedulers import DDPMScheduler
    monkeypatch.setitem(sys.modules, "monai", None)
    with pytest.raises(ImportError):                           # the file's own imports need monai
        BundleConfig(CONFIGS, bundle="mednist_ddpm").get("noise")
    cfg = BundleConfig(CONFIGS, {"imports": OFFLINE_IMPORTS}, bundle="mednist_ddpm", meta_file=str(META))
    net = cfg.get("network")
    assert type(net) is DiffusionModelUNet and net.in_channels == 1 and net.out_channels == 1
    assert list(net.block_out_channels) == [64, 128, 128] and sum(p.numel() for p in net.parameters()) == 4634305
    assert cfg.get("network_def") is net                       # network is network_def moved to the device
    sched = cfg.get("scheduler")
    assert type(sched) is DDPMScheduler and sched.num_train_timesteps == 1000 and len(sched.timesteps) == 1000
    assert [int(t) for t in sched.timesteps[[0, -1]]] == [999, 0] and sched.clip_sample
    noise = cfg.get("noise")
    assert tuple(noise.shape) == (1, 1, 64, 64) and noise.dtype == torch.float32
    assert float(noise.min()) >= 0.0 and float(noise.max()) < 1.0
    inferer = cfg.get("inferer")
    assert type(inferer) is DiffusionInferer and inferer.scheduler is sched and callable(cfg.get("sample"))
    assert cfg.get("ckpt_path") == "./models/model.pt" and cfg.get("out_file") == ""
    with pytest.raises(ModuleNotFoundError, match="MONAI"):   # testing_jpg's transforms are MONAI's
        cfg.get("save_trans")


# ------------------------------------------------------------------------------------------------------------------
# oracle and scheduler pinned to the reference's own 1000-step run
# ------------------------------------------------------------------------------------------------------------------
def test_fixture_layout():
    fx = _fixture()
    assert fx["probe_t"] == [999, 900, 750, 500, 250, 100, 1, 0] and fx["every"] == 100
    assert len(fx["trajectory"]) == 10 and torch.equal(fx["trajectory"][-1], fx["image"])
    assert torch.equal(fx["probe_x"][0], fx["noise"])
    g = torch.Generator().manual_seed(fx["seed"])
    assert torch.equal(torch.rand(1, 1, 64, 64, generator=g), fx["noise"])
    for t, nxt in zip(fx["probe_t"], fx["probe_next"]):
        if t % 100 == 0:                                       # the sample after the step at t = 900, 800, ..., 0
            assert torch.equal(nxt, fx["trajectory"][(900 - t) // 100]), t
    assert torch.equal(fx["probe_next"][fx["probe_t"].index(1)], fx["probe_x"][fx["probe_t"].index(0)])


def test_oracle_teacher_forced_matches_reference_fixture():
    """The fp32 torch oracle's UNet and DDPM step reproduce the reference's at every recorded timestep."""
    fx = _fixture()
    _, sd = _recipe_unet(fx)
    cfg = G.unet_oracle_cfg(fx["unet_kwargs"])
    sched = O.DDPMOracle(**fx["scheduler_kwargs"])
    with torch.no_grad():
        for t, x, eps, nxt in zip(fx["probe_t"], fx["probe_x"], fx["probe_eps"], fx["probe_next"]):
            y = O.unet_forward(sd, cfg, x, torch.Tensor((t,)).long())
            assert rel(y, eps) < 1e-4, (t, rel(y, eps))
            got, _ = sched.step(eps, t, x, generator=_noise_generator(fx["seed"], t))
            assert rel(got, nxt) < 1e-5, (t, rel(got, nxt))


def test_ddpm_scheduler_teacher_forced_cpu(monkeypatch):
    """The package's DDPMScheduler on the reference's UNet outputs, with the same noise draws."""
    cpu_backend.install(monkeypatch)
    from generativemodels_b200.networks.schedulers import DDPMScheduler
    fx = _fixture()
    s = DDPMScheduler(**fx["scheduler_kwargs"])
    for t, x, eps, nxt in zip(fx["probe_t"], fx["probe_x"], fx["probe_eps"], fx["probe_next"]):
        got, _ = s.step(eps, t, x, generator=_noise_generator(fx["seed"], t))
        assert rel(got, nxt) < 1e-5, (t, rel(got, nxt))


# ------------------------------------------------------------------------------------------------------------------
# CLI, the notebook's call shape
# ------------------------------------------------------------------------------------------------------------------
def _reduced_unet(**kw):
    from generativemodels_b200.networks.nets import DiffusionModelUNet
    return DiffusionModelUNet(**{**dict(spatial_dims=2, in_channels=1, out_channels=1, num_channels=[16, 32, 32],
                                        attention_levels=[False, True, True], num_res_blocks=1, num_head_channels=32,
                                        norm_num_groups=8), **kw})


REDUCED = ["--network_def#num_channels", "[16, 32, 32]", "--network_def#num_head_channels", "32",
           "--network_def#norm_num_groups", "8"]


def test_cli_testing_end_to_end_cpu(monkeypatch, tmp_path, scripts_pkg):
    """``run testing --meta_file ... --config_file "'common.yaml', 'infer.yaml'" --ckpt_path ... --bundle_root .
    --out_file ...`` on the CPU stand-in at reduced width and 4 DDPM steps, loading a checkpoint saved here."""
    cpu_backend.install(monkeypatch)
    from generativemodels_b200.bundle.__main__ import main
    monkeypatch.setitem(sys.modules, "monai", None)
    monkeypatch.chdir(tmp_path)
    torch.manual_seed(3)
    torch.save(G.randomize_zero_params(_reduced_unet()).state_dict(), tmp_path / "model.pt")
    args = ["run", "testing", "--meta_file", str(META), "--config_file", f"'{CONFIGS[0]}', '{CONFIGS[1]}'",
            "--ckpt_path", "model.pt", "--bundle_root", ".", "--out_file", "test.pt", "--bundle", "mednist_ddpm",
            "--imports", json.dumps(OFFLINE_IMPORTS), "--device", "$torch.device('cpu')",
            "--num_train_timesteps", "4", *REDUCED]
    assert main(args) == 0
    sample = torch.load(tmp_path / "test.pt")
    assert tuple(sample.shape) == (1, 1, 64, 64) and bool(torch.isfinite(sample).all())
    # a checkpoint of another width does not load: the file's load_state really reads --ckpt_path
    torch.save(_reduced_unet(num_res_blocks=2).state_dict(), tmp_path / "model.pt")
    with pytest.raises(RuntimeError, match="state_dict"):
        main(args)


# ------------------------------------------------------------------------------------------------------------------
# CUDA path
# ------------------------------------------------------------------------------------------------------------------
# Drift of the graph-replayed 1000-step sample from the reference's fp32 run, relative L2 / normalised max-abs of the
# sample after the step at t = 900, 800, ..., 0 (the last is the final image), measured on an H100 80GB HBM3 at a
# 700 W power limit:
#   fp16 library: 1.2e-5/2.5e-5  1.9e-5/4.4e-5  3.5e-5/6.6e-5  6.4e-5/1.4e-4  1.1e-4/2.1e-4
#                 1.7e-4/4.2e-4  2.6e-4/7.3e-4  3.6e-4/1.1e-3  5.1e-4/2.3e-3  7.7e-4/3.9e-3
#   bf16 library: 8.5e-5/1.8e-4  1.5e-4/3.3e-4  2.7e-4/5.1e-4  4.7e-4/1.2e-3  8.0e-4/2.1e-3
#                 1.3e-3/3.2e-3  1.7e-3/4.4e-3  2.4e-3/5.7e-3  3.6e-3/1.5e-2  5.3e-3/3.5e-2
# The teacher-forced UNet outputs are 1.3e-3 - 1.8e-3 (fp16) and 1.1e-2 - 1.5e-2 (bf16) off the reference, yet the
# chain stays bounded: the drift grows steadily but stays below one forward's error over the whole run, because
# clipping x0 to [-1, 1] discards most of the model output's error at large t.  The bounds leave 3-5x headroom over
# the final image's numbers and lie inside the suite's trajectory tolerance (TOL_TRAJ, 2 * TOL_TRAJ).
TRAJ_TOL = {torch.float16: (4e-3, 2e-2), torch.bfloat16: (2e-2, 1e-1)}


@pytest.fixture(scope="module")
def mednist_unet():
    fx = _fixture()
    unet, sd = _recipe_unet(fx)
    return fx, unet.cuda(), sd


@pytest.mark.gpu
def test_mednist_unet_teacher_forced_gpu(mednist_unet):
    """The UNet at the bundle's shapes (GroupNorm(32) over 64 channels, head-128 attention at T = 1024 and 256) on the
    reference's own inputs at every recorded timestep."""
    fx, unet, _ = mednist_unet
    report = {}
    for t, x, eps in zip(fx["probe_t"], fx["probe_x"], fx["probe_eps"]):
        y = unet(x.cuda(), timesteps=torch.Tensor((t,)).cuda())
        report[t] = close(y, eps, f"MedNIST UNet output t={t}", TOL_REL, TOL_MAX)
    print("MedNIST teacher-forced UNet (rel-L2, max-abs):", {t: (f"{r:.2e}", f"{m:.2e}") for t, (r, m) in report.items()})


@pytest.mark.gpu
def test_mednist_testing_1000_steps_gpu(mednist_unet, scripts_pkg, tmp_path):
    """The bundle's ``testing`` item resolved in-process on the CUDA path, seeded as the fixture: the checkpoint is
    loaded into the device network, the file's noise and 999 DDPM noise draws come from the global CPU generator
    (graph capture and warm-up draw nothing), and the trajectory stays within TRAJ_TOL of the reference's."""
    from generativemodels_b200 import ops
    from generativemodels_b200.bundle.config import BundleConfig
    fx, _, sd = mednist_unet
    torch.save(sd, tmp_path / "model.pt")
    cfg = BundleConfig(CONFIGS, {"imports": OFFLINE_IMPORTS, "ckpt_path": str(tmp_path / "model.pt"),
                                 "out_file": str(tmp_path / "test.pt")}, bundle="mednist_ddpm", meta_file=str(META))
    sched = cfg.get("scheduler")
    traj, step = [], sched.step

    def rec(model_output, timestep, sample, *a, **k):
        nxt, x0 = step(model_output, timestep, sample, *a, **k)
        if int(timestep) % fx["every"] == 0:
            traj.append(nxt.clone())
        return nxt, x0
    sched.step = rec
    cfg.get("load_state")                                      # the file's order: weights first, then the noise
    net = cfg.get("network")
    assert next(net.parameters()).is_cuda
    assert all(torch.equal(v.cpu(), sd[k]) for k, v in net.state_dict().items())
    torch.manual_seed(fx["seed"])
    cfg.get("testing")
    torch.cuda.synchronize()
    after = torch.get_rng_state()
    g = _noise_generator(fx["seed"], 0)
    assert torch.equal(after, g.get_state()), "the sample drew from the global CPU generator beyond the DDPM noise"
    assert torch.equal(cfg.get("noise"), fx["noise"])
    image = torch.load(tmp_path / "test.pt")
    assert len(traj) == len(fx["trajectory"]) and torch.equal(image, traj[-1])
    curve = [(rel(a, b), relmax(a, b)) for a, b in zip(traj, fx["trajectory"])]
    print("MedNIST 1000-step drift, rel-L2 / max-abs after t = 900 ... 0:",
          [f"{r:.2e}/{m:.2e}" for r, m in curve])
    tol_rel, tol_max = TRAJ_TOL[ops.H16]
    for k, (a, b) in enumerate(zip(traj, fx["trajectory"])):
        close(a, b, f"MedNIST sample after t={900 - 100 * k}", tol_rel, tol_max)
    close(image, fx["image"], "MedNIST final image", tol_rel, tol_max)


@pytest.mark.gpu
def test_mednist_graph_replay_bit_identical_to_eager(monkeypatch, mednist_unet):
    from generativemodels_b200.inferers import DiffusionInferer
    from generativemodels_b200.inferers import inferer as inferer_mod
    from generativemodels_b200.networks.schedulers import DDPMScheduler
    fx, unet, _ = mednist_unet
    runs = {}
    for graph in (False, True):
        monkeypatch.setattr(inferer_mod, "AUTO_CUDA_GRAPH", graph)
        s = DDPMScheduler(**fx["scheduler_kwargs"])
        s.set_timesteps(40)
        torch.manual_seed(fx["seed"])
        runs[graph] = DiffusionInferer(s).sample(fx["noise"].cuda(), unet, s, save_intermediates=True,
                                                 intermediate_steps=1, verbose=False)
    assert "_b200_auto_graph" in unet.__dict__
    assert len(runs[True][1]) == len(runs[False][1]) == 40
    for a, b in zip(runs[False][1], runs[True][1]):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_mednist_cli_testing_gpu(monkeypatch, tmp_path, scripts_pkg):
    """The notebook's command at the published size with a saved random-weight checkpoint: 1000 DDPM steps on the
    device, test.pt written."""
    from generativemodels_b200.bundle.__main__ import main
    from generativemodels_b200.networks.nets import DiffusionModelUNet
    monkeypatch.setitem(sys.modules, "monai", None)
    monkeypatch.chdir(tmp_path)
    fx = _fixture()
    unet = DiffusionModelUNet(**fx["unet_kwargs"])
    G.recipe_state_dict(unet, 7)
    torch.save(unet.state_dict(), tmp_path / "model.pt")
    args = ["run", "testing", "--meta_file", str(META), "--config_file", f"'{CONFIGS[0]}', '{CONFIGS[1]}'",
            "--ckpt_path", "model.pt", "--bundle_root", ".", "--out_file", "test.pt", "--bundle", "mednist_ddpm",
            "--imports", json.dumps(OFFLINE_IMPORTS)]
    assert main(args) == 0
    sample = torch.load(tmp_path / "test.pt")
    assert tuple(sample.shape) == (1, 1, 64, 64) and sample.is_cuda and bool(torch.isfinite(sample).all())
