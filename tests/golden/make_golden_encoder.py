"""Generate the DiffusionModelEncoder fixture (tests/golden/g_diffusion_encoder.pt + parts) by running the UNMODIFIED
reference (/root/reference, CPU fp32, MONAI shim):   python -m tests.golden.make_golden_encoder

Weights come from tests.golden.configs.recipe_state_dict (sorted keys, one seeded generator, nothing left at zero), so
the fixture stores the seed, inputs and logits, and the reference's state_dict keys with their shapes.  Every case's
last feature map flattens to the 4096 features of the reference's hard-coded head.  Cases:
  tutorial   the classifier of the classifier-guided anomaly-detection tutorial, batch 4, 1x64x64: logits for one
             broadcast float timestep torch.Tensor((t,)) at several t, and for per-sample int64 timesteps
  3d         a 3-D classifier on 16^3 volumes
  cross      with_conditioning=True, a (N, 1, cross_attention_dim) context
  class      num_class_embeds with labels; 256 channels on a 4x4 map at the head
  updown     resblock_updown=True (ResnetBlock downsamplers, the last level's included)
  heads      a tuple num_head_channels (two heads of 32 at 32x32) and norm_num_groups 16
The updown weights use seed 308 rather than 304: with 304 its logits are a few tenths, small against the head's
4096-term sums, and their relative error under bfloat16 storage (8-bit mantissa) is 4e-2 where the other cases are at
1e-2 or below.
And ``ddim_encode``: the tutorial's DDIM reversed_step encoding loop (its DiffusionModelUNet, 1x1x64x64, the first
``steps`` timesteps of a 1000-step schedule) with the model output of every step.
"""
import torch

from tests.golden import configs as G
from tests.golden import save
from oracle import ref_import

TUTORIAL = dict(spatial_dims=2, in_channels=1, out_channels=2, num_channels=(32, 64, 64),
                attention_levels=(False, True, True), num_res_blocks=(1, 1, 1), num_head_channels=64,
                with_conditioning=False)
CASES = {
    "tutorial": dict(kw=TUTORIAL, shape=(4, 1, 64, 64)),
    "3d": dict(kw=dict(spatial_dims=3, in_channels=1, out_channels=3, num_channels=(32, 64),
                       attention_levels=(False, True), num_res_blocks=(1, 1), num_head_channels=64),
               shape=(2, 1, 16, 16, 16)),
    "cross": dict(kw=dict(spatial_dims=2, in_channels=1, out_channels=2, num_channels=(32, 64),
                          attention_levels=(False, True), num_res_blocks=(1, 1), num_head_channels=32,
                          with_conditioning=True, cross_attention_dim=8),
                  shape=(2, 1, 32, 32), context=8),
    "class": dict(kw=dict(spatial_dims=2, in_channels=1, out_channels=2, num_channels=(32, 64, 256),
                          attention_levels=(False, False, True), num_res_blocks=(1, 1, 1), num_head_channels=64,
                          num_class_embeds=3),
                  shape=(3, 1, 32, 32), classes=3),
    "updown": dict(kw=dict(spatial_dims=2, in_channels=2, out_channels=2, num_channels=(32, 64),
                           attention_levels=(False, True), num_res_blocks=(2, 1), num_head_channels=64,
                           resblock_updown=True),
                   shape=(2, 2, 32, 32), seed=308),
    "heads": dict(kw=dict(spatial_dims=2, in_channels=2, out_channels=4, num_channels=(32, 64, 64),
                          attention_levels=(False, True, True), num_res_blocks=(1, 1, 1),
                          num_head_channels=(0, 32, 64), norm_num_groups=16),
                  shape=(2, 2, 64, 64)),
}
TUTORIAL_TIMESTEPS = (0, 250, 999)
# anomalydetection_tutorial_classifier_guidance.py:176-188 (the diffusion model and its scheduler)
TUTORIAL_UNET = dict(spatial_dims=2, in_channels=1, out_channels=1, num_channels=(64, 64, 64),
                     attention_levels=(False, False, True), num_res_blocks=1, num_head_channels=64,
                     with_conditioning=False)
DDIM_STEPS = 3


def main():
    ref_import.import_reference()
    from generative.networks.nets.diffusion_model_unet import DiffusionModelEncoder, DiffusionModelUNet
    from generative.networks.schedulers.ddim import DDIMScheduler

    torch.set_grad_enabled(False)
    out = {}
    for i, (name, case) in enumerate(CASES.items()):
        m = DiffusionModelEncoder(**case["kw"]).eval()
        seed = case.get("seed", 300 + i)
        G.recipe_state_dict(m, seed)
        torch.manual_seed(400 + i)
        n = case["shape"][0]
        x = torch.randn(case["shape"])
        ctx = torch.randn(n, 1, case["context"]) if "context" in case else None
        labels = torch.randint(0, case["classes"], (n,)) if "classes" in case else None
        runs = []
        if name == "tutorial":
            for t in TUTORIAL_TIMESTEPS:
                ts = torch.Tensor((t,))
                runs.append(dict(t=ts, logits=m(x, ts)))
        ts = torch.randint(0, 1000, (n,)).long()
        runs.append(dict(t=ts, logits=m(x, ts, context=ctx, class_labels=labels)))
        out[name] = dict(kwargs=case["kw"], seed=seed, x=x, context=ctx, class_labels=labels, runs=runs,
                         keys=[(k, tuple(v.shape)) for k, v in m.state_dict().items()])
        print(name, [tuple(r["logits"].shape) for r in runs], flush=True)

    unet = DiffusionModelUNet(**TUTORIAL_UNET).eval()
    G.recipe_state_dict(unet, 310)
    scheduler = DDIMScheduler(num_train_timesteps=1000)
    scheduler.set_timesteps(num_inference_steps=1000)
    torch.manual_seed(410)
    img = torch.rand(1, 1, 64, 64)
    current, outputs, samples = img, [], []
    for t in range(DDIM_STEPS):                # the tutorial's encoding loop (:435-442), first DDIM_STEPS steps
        model_output = unet(current, timesteps=torch.Tensor((t,)))
        current, _ = scheduler.reversed_step(model_output, t, current)
        outputs.append(model_output)
        samples.append(current)
    out["ddim_encode"] = dict(unet_kwargs=TUTORIAL_UNET, seed=310, steps=DDIM_STEPS, x=img, model_outputs=outputs,
                              samples=samples)
    save(out, "g_diffusion_encoder")


if __name__ == "__main__":
    main()
