"""DiffusionModelEncoder on the H100 kernels: every case of the reference fixture (tests/golden/g_diffusion_encoder.pt)
within the network tolerance, in the loaded storage flavour and (through B200_ACT_DTYPE, in a fresh interpreter) the
other one; repeat calls and CUDA-graph replays bit for bit; a sample's logits against the same sample run alone; the
tutorial's import line, classifier and DDIM encoding loop with only ``sys.path`` changed."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from generativemodels_b200 import ops
from generativemodels_b200.cuda_graph import graphed
from generativemodels_b200.networks.nets.diffusion_model_unet import DiffusionModelEncoder
from tests.fixture_checks import TOL_MAX, TOL_REL, TOL_TRAJ, close
from tests.golden import configs as G
from tests.golden import load

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
GOLD = load("g_diffusion_encoder")
CASES = [k for k in GOLD if k != "ddim_encode"]
RUNS = [(k, i) for k in CASES for i in range(len(GOLD[k]["runs"]))]


def _net(name):
    g = GOLD[name]
    m = DiffusionModelEncoder(**g["kwargs"]).eval()
    G.recipe_state_dict(m, g["seed"])
    return m.cuda()


def _inputs(name, i=-1):
    g = GOLD[name]
    cuda = lambda t: None if t is None else t.cuda()
    return cuda(g["x"]), cuda(g["runs"][i]["t"]), cuda(g["context"]), cuda(g["class_labels"])


def _check_logits(got, want, what):
    close(got.float().cpu(), want, what, TOL_REL, TOL_MAX)
    # where the reference's top logit leads the runner-up by more than twice the max-abs tolerance, the class agrees
    top2 = want.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 2 * TOL_MAX * want.abs().max()
    assert torch.equal(got.float().cpu().argmax(1)[clear], want.argmax(1)[clear]), f"{what}: argmax differs"


@pytest.mark.parametrize("name,i", RUNS, ids=[f"{k}-{i}" for k, i in RUNS])
def test_vs_fixture(cuda_device, name, i):
    m = _net(name)
    x, t, ctx, labels = _inputs(name, i)
    got = m(x, t, context=ctx, class_labels=labels)
    assert got.dtype == torch.float32 and got.is_cuda
    _check_logits(got, GOLD[name]["runs"][i]["logits"], f"{name} run {i}")


def test_other_storage_flavour(cuda_device):
    """The same checks with the library built for the other 16-bit storage type (B200_ACT_DTYPE is read at import)."""
    other = "bf16" if ops.H16 is torch.float16 else "fp16"
    code = f'''
import sys
sys.path.insert(0, {str(ROOT)!r})
import torch
from generativemodels_b200 import ops
assert ops.H16 is (torch.bfloat16 if {other!r} == "bf16" else torch.float16)
import tests.test_diffusion_encoder_gpu as T
for name, i in T.RUNS:
    m = T._net(name)
    x, t, ctx, labels = T._inputs(name, i)
    T._check_logits(m(x, t, context=ctx, class_labels=labels), T.GOLD[name]["runs"][i]["logits"], name)
print("ok")
'''
    env = dict(os.environ, B200_ACT_DTYPE=other)
    env.pop("PYTHONPATH", None)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=str(ROOT),
                       timeout=900)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_half_input_returns_input_dtype(cuda_device):
    m = _net("tutorial")
    x, t, _, _ = _inputs("tutorial", 0)
    got = m(x.half(), t)
    assert got.dtype == torch.float16
    _check_logits(got, GOLD["tutorial"]["runs"][0]["logits"], "fp16 input")


def test_batch_of_eight_takes_the_gemm_head(cuda_device):
    """More than four samples of 4096 features leave the GEMV kernel for the tensor-core GEMM head."""
    m = _net("tutorial")
    x, t, _, _ = _inputs("tutorial")
    got = m(torch.cat([x, x.flip(0)]), torch.cat([t, t.flip(0)]))
    want = GOLD["tutorial"]["runs"][-1]["logits"]
    _check_logits(got, torch.cat([want, want.flip(0)]), "batch 8")


def test_train_mode_equals_eval_mode(cuda_device):
    m = _net("tutorial")
    x, t, _, _ = _inputs("tutorial")
    a = m(x, t)
    b = m.train()(x, t)
    assert torch.equal(a, b)


def test_repeat_calls_bit_identical(cuda_device):
    for name in ("tutorial", "cross", "class"):
        m = _net(name)
        x, t, ctx, labels = _inputs(name)
        a = m(x, t, context=ctx, class_labels=labels)
        b = m(x, t, context=ctx, class_labels=labels)
        assert torch.equal(a, b), name


def test_sample_independent_of_its_batch(cuda_device):
    """One call at batch 4 against four calls at batch 1, to the bit: no kernel the tutorial's classifier reaches mixes
    samples or orders a sample's sums by the batch size (its reductions are too short for the split-K path, whose
    split follows the number of output tiles, and the head's GEMV reduces each row on its own)."""
    m = _net("tutorial")
    x, t, _, _ = _inputs("tutorial")
    whole = m(x, t)
    alone = torch.cat([m(x[i:i + 1], t[i:i + 1]) for i in range(x.shape[0])])
    assert torch.equal(whole, alone), (whole - alone).abs().max().item()


@pytest.mark.parametrize("name", ["tutorial", "cross", "class"])
def test_graph_replay_equals_eager(cuda_device, name):
    m = _net(name)
    x, t, ctx, labels = _inputs(name)
    eager = m(x, t, context=ctx, class_labels=labels)
    gm = graphed(m)
    first = gm(x, t, context=ctx, class_labels=labels)
    second = gm(x, t, context=ctx, class_labels=labels)
    assert torch.equal(first, eager) and torch.equal(second, eager)


# anomalydetection_tutorial_classifier_guidance.py:66 (imports), 304-315 (classifier), 176-188 (diffusion model and
# scheduler), 430-442 (the reversed DDIM encoding loop); trained weights are replaced by a load_state_dict of the
# fixture's seeded recipe, and the loop runs its first steps only
_TUTORIAL_CELLS = '''
import sys
sys.path.insert(0, {root!r})                 # <- the only change: this repository instead of the reference checkout
import torch
from torch.cuda.amp import autocast
from generative.networks.nets.diffusion_model_unet import DiffusionModelEncoder, DiffusionModelUNet
from generative.networks.schedulers.ddim import DDIMScheduler

device = torch.device("cuda")
data = torch.load({inputs!r})

model = DiffusionModelUNet(
    spatial_dims=2,
    in_channels=1,
    out_channels=1,
    num_channels=(64, 64, 64),
    attention_levels=(False, False, True),
    num_res_blocks=1,
    num_head_channels=64,
    with_conditioning=False,
)
model.load_state_dict(data["unet"])
model.to(device)
scheduler = DDIMScheduler(num_train_timesteps=1000)

classifier = DiffusionModelEncoder(
    spatial_dims=2,
    in_channels=1,
    out_channels=2,
    num_channels=(32, 64, 64),
    attention_levels=(False, True, True),
    num_res_blocks=(1, 1, 1),
    num_head_channels=64,
    with_conditioning=False,
)
classifier.load_state_dict(data["classifier"])
classifier.to(device)

model.eval()
classifier.eval()
images = data["images"].to(device)
logits = []
for t in data["timesteps"]:
    with torch.no_grad():
        logits.append(classifier(images, timesteps=torch.Tensor((t,)).to(device)).cpu())

L = data["steps"]
current_img = data["inputimg"][None, ...].to(device)
scheduler.set_timesteps(num_inference_steps=1000)
outputs, samples = [], []
for t in range(L):
    with autocast(enabled=False):
        with torch.no_grad():
            model_output = model(current_img, timesteps=torch.Tensor((t,)).to(current_img.device))
    current_img, _ = scheduler.reversed_step(model_output, t, current_img)
    outputs.append(model_output.cpu())
    samples.append(current_img.cpu())
torch.save(dict(logits=logits, outputs=outputs, samples=samples), {out!r})
'''


def test_tutorial_dropin(cuda_device, tmp_path):
    from generativemodels_b200.networks.nets import DiffusionModelUNet
    g, d = GOLD["tutorial"], GOLD["ddim_encode"]
    broadcast = [r for r in g["runs"] if r["t"].numel() == 1]
    inputs, out = tmp_path / "inputs.pt", tmp_path / "out.pt"
    torch.save(dict(classifier=G.recipe_state_dict(DiffusionModelEncoder(**g["kwargs"]), g["seed"]),
                    unet=G.recipe_state_dict(DiffusionModelUNet(**d["unet_kwargs"]), d["seed"]),
                    images=g["x"], timesteps=[int(r["t"].item()) for r in broadcast], inputimg=d["x"][0],
                    steps=d["steps"]), inputs)
    env = dict(os.environ)
    env.pop("PYTHONPATH", None)
    r = subprocess.run([sys.executable, "-W", "ignore", "-c",
                        _TUTORIAL_CELLS.format(root=str(ROOT), inputs=str(inputs), out=str(out))],
                       capture_output=True, text=True, env=env, cwd="/tmp", timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = torch.load(out)
    for logits, run in zip(got["logits"], broadcast):
        _check_logits(logits, run["logits"], f"tutorial classifier at t={int(run['t'].item())}")
    for k in range(d["steps"]):
        close(got["outputs"][k], d["model_outputs"][k], f"DDIM encoding step {k}: model output", TOL_REL, TOL_MAX)
        # the step moves the image by a small amount: compare the displacement, not the image
        close(got["samples"][k] - d["x"], d["samples"][k] - d["x"], f"DDIM encoding step {k}: displacement",
              TOL_TRAJ, 2 * TOL_TRAJ)
