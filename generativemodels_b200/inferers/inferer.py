"""Sampling drivers with the interface of generative/inferers/inferer.py: DiffusionInferer (30-143),
LatentDiffusionInferer (323-487), ControlNetDiffusionInferer (561-707), ControlNetLatentDiffusionInferer (856-1038).

The loops are the reference's: one network forward + one ``scheduler.step`` per timestep, the sample travelling
between them as an NC[D]HW fp32 CUDA tensor.  What differs is underneath — each forward is the fused-kernel UNet, each
step one elementwise kernel, and ControlNet residuals are handed to the UNet as channels-last handles without a
layout round trip.  ``get_likelihood`` (SURVEY.md §8f rank 1) runs the same networks and one fused KL kernel per step.
"""
from __future__ import annotations

import os
from abc import ABC, abstractmethod
from collections.abc import Callable
from functools import partial

import torch
import torch.nn as nn

from .. import ops
from ..cuda_graph import GraphedModule, graphed
from ..networks.nets import VQVAE, ControlNet, SPADEAutoencoderKL, SPADEDiffusionModelUNet

try:  # tqdm is optional, like in the reference
    from tqdm import tqdm
    has_tqdm = True
except Exception:  # pragma: no cover
    has_tqdm = False


class Inferer(ABC):
    """Minimal stand-in for monai.inferers.Inferer (an ABC with ``__call__``)."""

    @abstractmethod
    def __call__(self, inputs, network, *args, **kwargs):
        raise NotImplementedError


def _check_mode(mode: str) -> None:
    if mode not in ["crossattn", "concat"]:
        raise NotImplementedError(f"{mode} condition is not supported")


def _with_seg(diffusion_model, seg):
    """SPADE networks take the segmentation map as an extra argument (inferer.py:121-125, 210-214, 445-446)."""
    return partial(diffusion_model, seg=seg) if isinstance(diffusion_model, SPADEDiffusionModelUNet) else diffusion_model


# Replay the network from a CUDA graph inside ``sample`` when one step is launch-latency-bound (a latent UNet step is
# 150-500 dependent launches of a few microseconds).  On by default (the -m gpu suite runs with it; graph-replayed and
# eager sampling are bit-identical, incl. PNDM's history).
# ``B200_AUTO_GRAPH=0`` or setting this flag to False turns it off.
AUTO_CUDA_GRAPH = os.environ.get("B200_AUTO_GRAPH", "1") != "0"
_AUTO_GRAPH_MAX_NUMEL = 1 << 18          # per-sample elements of the network input (64^3, 512^2): above, work dominates
_AUTO_GRAPH_MIN_STEPS = 8                # capture costs ~3 forwards


def _maybe_graphed(diffusion_model, input_noise: torch.Tensor, scheduler, seg):
    """The network itself, or its CUDA-graph wrapper (cached on the module) when AUTO_CUDA_GRAPH applies."""
    if not AUTO_CUDA_GRAPH or seg is not None or not isinstance(diffusion_model, nn.Module) or \
            isinstance(diffusion_model, GraphedModule) or not input_noise.is_cuda:
        return diffusion_model
    if input_noise[0].numel() > _AUTO_GRAPH_MAX_NUMEL or len(scheduler.timesteps) < _AUTO_GRAPH_MIN_STEPS:
        return diffusion_model
    wrapper = diffusion_model.__dict__.get("_b200_auto_graph")
    if wrapper is None:
        wrapper = graphed(diffusion_model)
        diffusion_model.__dict__["_b200_auto_graph"] = wrapper      # not a registered submodule: no state_dict change
    return wrapper


def _progress(scheduler, verbose: bool):
    return tqdm(scheduler.timesteps) if (verbose and has_tqdm) else iter(scheduler.timesteps)


def _spatial_pad(img: torch.Tensor, size) -> torch.Tensor:
    """monai SpatialPad (symmetric, zero) on a channel-first item without batch dim."""
    sp = img.shape[1:]
    pads = []
    for d in reversed(range(len(sp))):
        tot = max(size[d] - sp[d], 0)
        pads += [tot // 2, tot - tot // 2]
    return torch.nn.functional.pad(img, pads)


def _center_crop(img: torch.Tensor, roi) -> torch.Tensor:
    """monai CenterSpatialCrop on a channel-first item; non-positive roi entries keep the dim."""
    sl = [slice(None)]
    for d, n in enumerate(img.shape[1:]):
        r = n if roi[d] <= 0 else min(roi[d], n)
        start = max(n // 2 - r // 2, 0)
        sl.append(slice(start, start + r))
    return img[tuple(sl)]


class DiffusionInferer(Inferer):
    """inferer.py:30-143."""

    def __init__(self, scheduler: nn.Module) -> None:
        Inferer.__init__(self)
        self.scheduler = scheduler

    def __call__(self, inputs: torch.Tensor, diffusion_model: Callable[..., torch.Tensor], noise: torch.Tensor,
                 timesteps: torch.Tensor, condition: torch.Tensor | None = None, mode: str = "crossattn",
                 seg: torch.Tensor | None = None) -> torch.Tensor:
        """Training-style forward (inferer.py:44-81): add noise at per-sample timesteps, predict."""
        _check_mode(mode)
        diffusion_model = _with_seg(diffusion_model, seg)
        noisy_image = self.scheduler.add_noise(original_samples=inputs, noise=noise, timesteps=timesteps)
        if mode == "concat":
            noisy_image = torch.cat([noisy_image, condition], dim=1)
            condition = None
        return diffusion_model(x=noisy_image, timesteps=timesteps, context=condition)

    @torch.no_grad()
    def sample(self, input_noise: torch.Tensor, diffusion_model: Callable[..., torch.Tensor],
               scheduler: Callable[..., torch.Tensor] | None = None, save_intermediates: bool | None = False,
               intermediate_steps: int | None = 100, conditioning: torch.Tensor | None = None,
               mode: str = "crossattn", verbose: bool = True, seg: torch.Tensor | None = None):
        _check_mode(mode)
        if not scheduler:
            scheduler = self.scheduler
        diffusion_model = _with_seg(_maybe_graphed(diffusion_model, input_noise, scheduler, seg), seg)
        image = input_noise
        intermediates = []
        for t in _progress(scheduler, verbose):
            ts = torch.Tensor((t,)).to(input_noise.device)
            if mode == "concat":
                model_output = diffusion_model(torch.cat([image, conditioning], dim=1), timesteps=ts, context=None)
            else:
                model_output = diffusion_model(image, timesteps=ts, context=conditioning)
            image, _ = scheduler.step(model_output, t, image)
            if save_intermediates and t % intermediate_steps == 0:
                intermediates.append(image)
        return (image, intermediates) if save_intermediates else image

    @torch.no_grad()
    def get_likelihood(self, inputs: torch.Tensor, diffusion_model: Callable[..., torch.Tensor],
                       scheduler: Callable[..., torch.Tensor] | None = None, save_intermediates: bool | None = False,
                       conditioning: torch.Tensor | None = None, mode: str = "crossattn",
                       original_input_range: tuple | None = (0, 255), scaled_input_range: tuple | None = (0, 1),
                       verbose: bool = True, seg: torch.Tensor | None = None):
        """Variational lower bound per sample (inferer.py:145-277): for every timestep add noise, run the network,
        and accumulate the KL between the true posterior and the predicted one (decoder NLL at t = 0).  The whole
        per-step tail — predicted x0, clip, both means, KL / discretised-Gaussian term, per-sample mean — is one
        fused kernel (b200_ddpm_kl).  Fixed-variance DDPM schedulers (the reference's learned-variance branch
        evaluates ``if predicted_variance`` on a tensor and cannot run)."""
        diffusion_model = _with_seg(diffusion_model, seg)

        def predict(noisy_image, timesteps):
            if mode == "concat":
                return diffusion_model(torch.cat([noisy_image, conditioning], dim=1), timesteps=timesteps, context=None)
            return diffusion_model(x=noisy_image, timesteps=timesteps, context=conditioning)

        return self._likelihood_loop(inputs, predict, scheduler, save_intermediates, mode, original_input_range,
                                     scaled_input_range, verbose)

    def _likelihood_loop(self, inputs, predict, scheduler, save_intermediates, mode, original_input_range,
                         scaled_input_range, verbose):
        import ctypes as C

        from .. import _lib

        if not scheduler:
            scheduler = self.scheduler
        if scheduler._get_name() != "DDPMScheduler":
            raise NotImplementedError(f"Likelihood computation is only compatible with DDPMScheduler,"
                                      f" you are using {scheduler._get_name()}")
        _check_mode(mode)
        if scheduler.variance_type in ["learned", "learned_range"]:
            raise NotImplementedError("get_likelihood with a learned variance is not supported")
        lib = _lib.require_device()
        x0 = inputs.contiguous().float()
        N = x0.shape[0]
        per = x0.numel() // N
        noise = torch.randn_like(inputs).to(inputs.device)
        total_kl = torch.zeros(N, device=inputs.device)
        intermediates = []
        bin_width = (scaled_input_range[1] - scaled_input_range[0]) / (original_input_range[1] - original_input_range[0])
        for t in _progress(scheduler, verbose):
            t = int(t)
            timesteps = torch.full(inputs.shape[:1], t, device=inputs.device).long()
            noisy_image = self.scheduler.add_noise(original_samples=inputs, noise=noise, timesteps=timesteps)
            model_output = predict(noisy_image, timesteps)
            a_t = scheduler.alphas_cumprod[t]
            a_prev = scheduler.alphas_cumprod[t - 1] if t > 0 else scheduler.one
            b_t, b_prev = 1 - a_t, 1 - a_prev
            c = _lib.KlCoef()
            c.sqrt_alpha_prod_t, c.sqrt_beta_prod_t = float(a_t ** 0.5), float(b_t ** 0.5)
            c.coef_x0 = float((a_prev ** 0.5 * scheduler.betas[t]) / b_t)
            c.coef_xt = float(scheduler.alphas[t] ** 0.5 * b_prev / b_t)
            log_post = torch.log(scheduler._get_variance(timestep=t, predicted_variance=None))
            c.log_post_var = c.log_pred_var = float(log_post)
            c.bin_width = float(bin_width)
            c.prediction_type = {"epsilon": _lib.PRED_EPSILON, "sample": _lib.PRED_SAMPLE,
                                 "v_prediction": _lib.PRED_V}[str(scheduler.prediction_type)]
            c.clip, c.is_t0 = int(bool(scheduler.clip_sample)), int(t == 0)
            xt = noisy_image.contiguous().float()
            mo = model_output.contiguous().float()
            kl = torch.empty_like(x0) if save_intermediates else None
            ssum = torch.zeros(N, dtype=torch.float64, device=inputs.device)
            _lib.check(lib.b200_ddpm_kl(x0.data_ptr(), xt.data_ptr(), mo.data_ptr(), C.byref(c),
                                        None if kl is None else kl.data_ptr(), ssum.data_ptr(), N, per, ops._stream()),
                       "b200_ddpm_kl")
            total_kl += (ssum / per).float()
            if save_intermediates:
                intermediates.append(kl.cpu())
        return (total_kl, intermediates) if save_intermediates else total_kl

    def _approx_standard_normal_cdf(self, x):
        """inferer.py:279-283 (tanh approximation; the reference's only value-level unit test pins it vs scipy)."""
        import math
        return 0.5 * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3))))

    def _get_decoder_log_likelihood(self, inputs: torch.Tensor, means: torch.Tensor, log_scales: torch.Tensor,
                                    original_input_range: tuple | None = (0, 255),
                                    scaled_input_range: tuple | None = (0, 1)) -> torch.Tensor:
        """inferer.py:285-321, kept as a plain tensor expression for API parity (get_likelihood itself uses the
        fused kernel)."""
        assert inputs.shape == means.shape
        bin_width = (scaled_input_range[1] - scaled_input_range[0]) / (original_input_range[1] - original_input_range[0])
        centered_x = inputs - means
        inv_stdv = torch.exp(-log_scales)
        cdf_plus = self._approx_standard_normal_cdf(inv_stdv * (centered_x + bin_width / 2))
        cdf_min = self._approx_standard_normal_cdf(inv_stdv * (centered_x - bin_width / 2))
        log_cdf_plus = torch.log(cdf_plus.clamp(min=1e-12))
        log_one_minus_cdf_min = torch.log((1.0 - cdf_min).clamp(min=1e-12))
        cdf_delta = cdf_plus - cdf_min
        return torch.where(inputs < -0.999, log_cdf_plus,
                           torch.where(inputs > 0.999, log_one_minus_cdf_min, torch.log(cdf_delta.clamp(min=1e-12))))


class _LatentMixin:
    def _init_latent(self, scale_factor, ldm_latent_shape, autoencoder_latent_shape):
        self.scale_factor = scale_factor
        if (ldm_latent_shape is None) ^ (autoencoder_latent_shape is None):
            raise ValueError("If ldm_latent_shape is None, autoencoder_latent_shape must be None" "and vice versa.")
        self.ldm_latent_shape = ldm_latent_shape
        self.autoencoder_latent_shape = autoencoder_latent_shape

    def _encode_latent(self, inputs, autoencoder_model, quantized):
        with torch.no_grad():
            if isinstance(autoencoder_model, VQVAE):
                latent = autoencoder_model.encode_stage_2_inputs(inputs, quantized=quantized)
            else:
                latent = autoencoder_model.encode_stage_2_inputs(inputs)
            latent = ops.scale_f32(latent, self.scale_factor)
        if self.ldm_latent_shape is not None:
            latent = torch.stack([_spatial_pad(i, self.ldm_latent_shape) for i in latent], 0)
        return latent

    @staticmethod
    def _check_resample(resample_latent_likelihoods, resample_interpolation_mode):
        if resample_latent_likelihoods and resample_interpolation_mode not in ("nearest", "bilinear", "trilinear"):
            raise ValueError(f"resample_interpolation mode should be either nearest, bilinear, or trilinear,"
                             f" got {resample_interpolation_mode}")

    @staticmethod
    def _resample_maps(outputs, size, save_intermediates, resample_latent_likelihoods, resample_interpolation_mode):
        """KL maps upsampled to the image grid (inferer.py:557-562); a host-side post-processing of saved maps."""
        if save_intermediates and resample_latent_likelihoods:
            resizer = nn.Upsample(size=tuple(size), mode=resample_interpolation_mode)
            outputs = (outputs[0], [resizer(x) for x in outputs[1]])
        return outputs

    def _decode_latent(self, latent, autoencoder_model, seg=None):
        if self.autoencoder_latent_shape is not None:
            latent = torch.stack([_center_crop(i, self.autoencoder_latent_shape) for i in latent], 0)
        decode = autoencoder_model.decode_stage_2_outputs
        if isinstance(autoencoder_model, SPADEAutoencoderKL):          # inferer.py:473-474
            decode = partial(autoencoder_model.decode_stage_2_outputs, seg=seg)
        return decode(ops.scale_f32(latent, 1.0 / self.scale_factor, divide_by=self.scale_factor))


class LatentDiffusionInferer(DiffusionInferer, _LatentMixin):
    """inferer.py:323-487."""

    def __init__(self, scheduler: nn.Module, scale_factor: float = 1.0, ldm_latent_shape: list | None = None,
                 autoencoder_latent_shape: list | None = None) -> None:
        super().__init__(scheduler=scheduler)
        self._init_latent(scale_factor, ldm_latent_shape, autoencoder_latent_shape)

    def __call__(self, inputs: torch.Tensor, autoencoder_model, diffusion_model, noise: torch.Tensor,
                 timesteps: torch.Tensor, condition: torch.Tensor | None = None, mode: str = "crossattn",
                 seg: torch.Tensor | None = None, quantized: bool = True) -> torch.Tensor:
        latent = self._encode_latent(inputs, autoencoder_model, quantized)
        return super().__call__(inputs=latent, diffusion_model=diffusion_model, noise=noise, timesteps=timesteps,
                                condition=condition, mode=mode, seg=seg)

    @torch.no_grad()
    def sample(self, input_noise: torch.Tensor, autoencoder_model, diffusion_model,
               scheduler: Callable[..., torch.Tensor] | None = None, save_intermediates: bool | None = False,
               intermediate_steps: int | None = 100, conditioning: torch.Tensor | None = None,
               mode: str = "crossattn", verbose: bool = True, seg: torch.Tensor | None = None):
        if isinstance(autoencoder_model, SPADEAutoencoderKL) and isinstance(diffusion_model, SPADEDiffusionModelUNet) \
                and autoencoder_model.decoder.label_nc != diffusion_model.label_nc:
            raise ValueError(f"If both autoencoder_model and diffusion_model implement SPADE, the number of semantic"
                             f"labels for each must be compatible. Got {autoencoder_model.decoder.label_nc} and "
                             f"{diffusion_model.label_nc}")                                    # inferer.py:431-440
        outputs = super().sample(input_noise=input_noise, diffusion_model=diffusion_model, scheduler=scheduler,
                                 save_intermediates=save_intermediates, intermediate_steps=intermediate_steps,
                                 conditioning=conditioning, mode=mode, verbose=verbose, seg=seg)
        latent, latent_intermediates = outputs if save_intermediates else (outputs, [])
        image = self._decode_latent(latent, autoencoder_model, seg)
        if save_intermediates:
            return image, [self._decode_latent(l, autoencoder_model, seg) for l in latent_intermediates]
        return image


    @torch.no_grad()
    def get_likelihood(self, inputs: torch.Tensor, autoencoder_model, diffusion_model,
                       scheduler: Callable[..., torch.Tensor] | None = None, save_intermediates: bool | None = False,
                       conditioning: torch.Tensor | None = None, mode: str = "crossattn",
                       original_input_range: tuple | None = (0, 255), scaled_input_range: tuple | None = (0, 1),
                       verbose: bool = True, resample_latent_likelihoods: bool = False,
                       resample_interpolation_mode: str = "nearest", seg: torch.Tensor | None = None,
                       quantized: bool = True):
        """Likelihood of the latent representation (inferer.py:489-562)."""
        self._check_resample(resample_latent_likelihoods, resample_interpolation_mode)
        latents = self._encode_latent(inputs, autoencoder_model, quantized)
        outputs = super().get_likelihood(inputs=latents, diffusion_model=diffusion_model, scheduler=scheduler,
                                         save_intermediates=save_intermediates, conditioning=conditioning, mode=mode,
                                         verbose=verbose, seg=seg)
        return self._resample_maps(outputs, inputs.shape[2:], save_intermediates, resample_latent_likelihoods,
                                   resample_interpolation_mode)


class ControlNetDiffusionInferer(DiffusionInferer):
    """inferer.py:561-707."""

    def __init__(self, scheduler: nn.Module) -> None:
        Inferer.__init__(self)
        self.scheduler = scheduler

    def __call__(self, inputs: torch.Tensor, diffusion_model, controlnet, noise: torch.Tensor,
                 timesteps: torch.Tensor, cn_cond: torch.Tensor, condition: torch.Tensor | None = None,
                 mode: str = "crossattn", seg: torch.Tensor | None = None) -> torch.Tensor:
        _check_mode(mode)
        noisy_image = self.scheduler.add_noise(original_samples=inputs, noise=noise, timesteps=timesteps)
        if mode == "concat":
            noisy_image = torch.cat([noisy_image, condition], dim=1)
            condition = None
        down, mid = _run_controlnet(controlnet, noisy_image, timesteps, cn_cond, condition)
        return _with_seg(diffusion_model, seg)(x=noisy_image, timesteps=timesteps, context=condition,
                                               down_block_additional_residuals=down,
                                               mid_block_additional_residual=mid)

    @torch.no_grad()
    def sample(self, input_noise: torch.Tensor, diffusion_model, controlnet, cn_cond: torch.Tensor,
               scheduler: Callable[..., torch.Tensor] | None = None, save_intermediates: bool | None = False,
               intermediate_steps: int | None = 100, conditioning: torch.Tensor | None = None,
               mode: str = "crossattn", verbose: bool = True, seg: torch.Tensor | None = None):
        _check_mode(mode)
        if not scheduler:
            scheduler = self.scheduler
        diffusion_model = _with_seg(diffusion_model, seg)
        image = input_noise
        intermediates = []
        for t in _progress(scheduler, verbose):
            if mode == "concat":
                model_input, context_ = torch.cat([image, conditioning], dim=1), None
            else:
                model_input, context_ = image, conditioning
            ts = torch.Tensor((t,)).to(input_noise.device)
            down, mid = _run_controlnet(controlnet, model_input, ts, cn_cond, context_)
            model_output = diffusion_model(model_input, timesteps=ts, context=context_,
                                           down_block_additional_residuals=down, mid_block_additional_residual=mid)
            image, _ = scheduler.step(model_output, t, image)
            if save_intermediates and t % intermediate_steps == 0:
                intermediates.append(image)
        return (image, intermediates) if save_intermediates else image


    @torch.no_grad()
    def get_likelihood(self, inputs: torch.Tensor, diffusion_model, controlnet, cn_cond: torch.Tensor,
                       scheduler: Callable[..., torch.Tensor] | None = None, save_intermediates: bool | None = False,
                       conditioning: torch.Tensor | None = None, mode: str = "crossattn",
                       original_input_range: tuple | None = (0, 255), scaled_input_range: tuple | None = (0, 1),
                       verbose: bool = True, seg: torch.Tensor | None = None):
        """inferer.py:710-853: as DiffusionInferer.get_likelihood with the ControlNet residuals fed to the UNet.  (The
        reference's concat branch overwrites ``conditioning`` inside the loop and fails on its second step; here the
        concatenation is per step, as in ``sample``.)"""
        diffusion_model = _with_seg(diffusion_model, seg)

        def predict(noisy_image, timesteps):
            if mode == "concat":
                model_input, context_ = torch.cat([noisy_image, conditioning], dim=1), None
            else:
                model_input, context_ = noisy_image, conditioning
            down, mid = _run_controlnet(controlnet, model_input, timesteps, cn_cond, context_)
            return diffusion_model(model_input, timesteps=timesteps, context=context_,
                                   down_block_additional_residuals=down, mid_block_additional_residual=mid)

        return self._likelihood_loop(inputs, predict, scheduler, save_intermediates, mode, original_input_range,
                                     scaled_input_range, verbose)


def _run_controlnet(controlnet, x, timesteps, cn_cond, context):
    if isinstance(controlnet, ControlNet):      # keep the residuals channels-last between the two networks
        return controlnet(x=x, timesteps=timesteps, controlnet_cond=cn_cond, context=context, _internal=True)
    return controlnet(x=x, timesteps=timesteps, controlnet_cond=cn_cond, context=context)


class ControlNetLatentDiffusionInferer(ControlNetDiffusionInferer, _LatentMixin):
    """inferer.py:856-1038."""

    def __init__(self, scheduler: nn.Module, scale_factor: float = 1.0, ldm_latent_shape: list | None = None,
                 autoencoder_latent_shape: list | None = None) -> None:
        super().__init__(scheduler=scheduler)
        self._init_latent(scale_factor, ldm_latent_shape, autoencoder_latent_shape)

    def _match_cond(self, cn_cond: torch.Tensor, spatial) -> torch.Tensor:
        """Conditioning image resized to the latent grid (inferer.py:915-917 / 1001-1003)."""
        if tuple(cn_cond.shape[2:]) != tuple(spatial):
            cn_cond = torch.nn.functional.interpolate(cn_cond, tuple(spatial))
        return cn_cond

    def __call__(self, inputs: torch.Tensor, autoencoder_model, diffusion_model, controlnet, noise: torch.Tensor,
                 timesteps: torch.Tensor, cn_cond: torch.Tensor, condition: torch.Tensor | None = None,
                 mode: str = "crossattn", seg: torch.Tensor | None = None, quantized: bool = True) -> torch.Tensor:
        latent = self._encode_latent(inputs, autoencoder_model, quantized)
        cn_cond = self._match_cond(cn_cond, latent.shape[2:])
        return super().__call__(inputs=latent, diffusion_model=diffusion_model, controlnet=controlnet, noise=noise,
                                timesteps=timesteps, cn_cond=cn_cond, condition=condition, mode=mode, seg=seg)

    @torch.no_grad()
    def sample(self, input_noise: torch.Tensor, autoencoder_model, diffusion_model, controlnet,
               cn_cond: torch.Tensor, scheduler: Callable[..., torch.Tensor] | None = None,
               save_intermediates: bool | None = False, intermediate_steps: int | None = 100,
               conditioning: torch.Tensor | None = None, mode: str = "crossattn", verbose: bool = True,
               seg: torch.Tensor | None = None):
        cn_cond = self._match_cond(cn_cond, input_noise.shape[2:])
        outputs = super().sample(input_noise=input_noise, diffusion_model=diffusion_model, controlnet=controlnet,
                                 cn_cond=cn_cond, scheduler=scheduler, save_intermediates=save_intermediates,
                                 intermediate_steps=intermediate_steps, conditioning=conditioning, mode=mode,
                                 verbose=verbose, seg=seg)
        latent, latent_intermediates = outputs if save_intermediates else (outputs, [])
        image = self._decode_latent(latent, autoencoder_model, seg)
        if save_intermediates:
            return image, [self._decode_latent(l, autoencoder_model, seg) for l in latent_intermediates]
        return image

    @torch.no_grad()
    def get_likelihood(self, inputs: torch.Tensor, autoencoder_model, diffusion_model, controlnet,
                       cn_cond: torch.Tensor, scheduler: Callable[..., torch.Tensor] | None = None,
                       save_intermediates: bool | None = False, conditioning: torch.Tensor | None = None,
                       mode: str = "crossattn", original_input_range: tuple | None = (0, 255),
                       scaled_input_range: tuple | None = (0, 1), verbose: bool = True,
                       resample_latent_likelihoods: bool = False, resample_interpolation_mode: str = "nearest",
                       seg: torch.Tensor | None = None, quantized: bool = True):
        """inferer.py:1041-1124."""
        self._check_resample(resample_latent_likelihoods, resample_interpolation_mode)
        latents = self._encode_latent(inputs, autoencoder_model, quantized)
        cn_cond = self._match_cond(cn_cond, latents.shape[2:])
        outputs = super().get_likelihood(inputs=latents, diffusion_model=diffusion_model, controlnet=controlnet,
                                         cn_cond=cn_cond, scheduler=scheduler, save_intermediates=save_intermediates,
                                         conditioning=conditioning, mode=mode, verbose=verbose, seg=seg)
        return self._resample_maps(outputs, inputs.shape[2:], save_intermediates, resample_latent_likelihoods,
                                   resample_interpolation_mode)


class VQVAETransformerInferer(Inferer):
    """inferer.py:1126-1330 — VQ-VAE indices + autoregressive transformer (SURVEY.md §8f rank 3)."""

    def __init__(self) -> None:
        Inferer.__init__(self)

    @staticmethod
    def _ordered_latent(inputs, vqvae_model, ordering):
        with torch.no_grad():
            latent = vqvae_model.index_quantize(inputs)
        latent_spatial_dim = tuple(latent.shape[1:])
        latent = latent.reshape(latent.shape[0], -1)
        return latent[:, ordering.get_sequence_ordering()], latent_spatial_dim

    def __call__(self, inputs: torch.Tensor, vqvae_model, transformer_model, ordering,
                 condition: torch.Tensor | None = None, return_latent: bool = False):
        """Teacher-forced forward of a training iteration (inferer.py:1134-1181): BOS-prefixed ordered indices in,
        next-token logits out (a random max_seq_len window if the sequence is longer)."""
        latent, latent_spatial_dim = self._ordered_latent(inputs, vqvae_model, ordering)
        target = latent.clone()
        latent = torch.nn.functional.pad(latent, (1, 0), "constant", vqvae_model.num_embeddings)
        latent = latent[:, :-1].long()
        seq_len = latent.shape[1]
        max_seq_len = transformer_model.max_seq_len
        start = torch.randint(low=0, high=seq_len + 1 - max_seq_len, size=(1,)).item() if max_seq_len < seq_len else 0
        prediction = transformer_model(x=latent[:, start:start + max_seq_len], context=condition)
        if return_latent:
            return prediction, target[:, start:start + max_seq_len], latent_spatial_dim
        return prediction

    @torch.no_grad()
    def sample(self, latent_spatial_dim, starting_tokens: torch.Tensor, vqvae_model, transformer_model, ordering,
               conditioning: torch.Tensor | None = None, temperature: float = 1.0, top_k: int | None = None,
               verbose: bool = True) -> torch.Tensor:
        """inferer.py:1183-1245.  Token by token: logits of the last position / temperature -> optional top-k ->
        softmax -> BOS probability zeroed -> torch.multinomial (the draw stays with PyTorch's generator).  While the
        sequence fits ``max_seq_len`` the logits come from the transformer's key/value cache (one row per step);
        once the window slides the whole window is recomputed per token, as the reference always does."""
        import math
        seq_len = math.prod(latent_spatial_dim)
        steps = tqdm(range(seq_len)) if (verbose and has_tqdm) else iter(range(seq_len))
        latent_seq = starting_tokens.long()
        incremental = hasattr(transformer_model, "new_cache") and latent_seq.size(1) <= transformer_model.max_seq_len
        cache = transformer_model.new_cache(latent_seq.shape[0], latent_seq.device, conditioning,
                                            graph=latent_seq.is_cuda) if incremental else None
        pending = latent_seq                      # tokens the cache has not seen yet
        for _ in steps:
            if cache is not None and cache.length + pending.size(1) <= transformer_model.max_seq_len:
                logits = transformer_model.step(pending, cache)
            else:
                cache = None
                idx_cond = latent_seq[:, -transformer_model.max_seq_len:]      # the whole sequence while it fits
                logits = transformer_model(x=idx_cond, context=conditioning)
            logits = logits[:, -1, :] / temperature          # (a fresh tensor: graph steps return a static buffer)
            if top_k is not None:
                v, _ = torch.topk(logits, min(top_k, logits.size(-1)))
                logits[logits < v[:, [-1]]] = -float("Inf")
            probs = torch.nn.functional.softmax(logits, dim=-1)
            probs[:, vqvae_model.num_embeddings] = 0          # never sample the BOS token
            idx_next = torch.multinomial(probs, num_samples=1)
            latent_seq = torch.cat((latent_seq, idx_next), dim=1)
            pending = idx_next
        latent_seq = latent_seq[:, 1:]
        latent_seq = latent_seq[:, ordering.get_revert_sequence_ordering()]
        latent = latent_seq.reshape((starting_tokens.shape[0],) + tuple(latent_spatial_dim))
        return vqvae_model.decode_samples(latent)

    @torch.no_grad()
    def get_likelihood(self, inputs: torch.Tensor, vqvae_model, transformer_model, ordering,
                       condition: torch.Tensor | None = None, resample_latent_likelihoods: bool = False,
                       resample_interpolation_mode: str = "nearest", verbose: bool = False) -> torch.Tensor:
        """Log-likelihood of every latent token given its predecessors (inferer.py:1247-1330)."""
        import math
        if resample_latent_likelihoods and resample_interpolation_mode not in ("nearest", "bilinear", "trilinear"):
            raise ValueError(f"resample_interpolation mode should be either nearest, bilinear, or trilinear,"
                             f" got {resample_interpolation_mode}")
        latent, latent_spatial_dim = self._ordered_latent(inputs, vqvae_model, ordering)
        seq_len = math.prod(latent_spatial_dim)
        latent = torch.nn.functional.pad(latent, (1, 0), "constant", vqvae_model.num_embeddings).long()
        L = transformer_model.max_seq_len
        logits = transformer_model(x=latent[:, :L], context=condition)
        probs = torch.nn.functional.softmax(logits, dim=-1)
        target = latent[:, 1:]
        probs = torch.gather(probs, 2, target[:, :L].unsqueeze(2)).squeeze(2)
        if probs.shape[1] < target.shape[1]:
            steps = tqdm(range(L, seq_len)) if (verbose and has_tqdm) else iter(range(L, seq_len))
            for i in steps:
                lg = transformer_model(x=latent[:, i + 1 - L:i + 1], context=condition)[:, -1, :]
                p = torch.gather(torch.nn.functional.softmax(lg, dim=-1), 1, target[:, i].unsqueeze(1))
                probs = torch.cat((probs, p), dim=1)
        probs = torch.log(probs)
        probs = probs[:, ordering.get_revert_sequence_ordering()]
        probs_reshaped = probs.reshape((inputs.shape[0],) + latent_spatial_dim)
        if resample_latent_likelihoods:
            probs_reshaped = nn.Upsample(size=inputs.shape[2:], mode=resample_interpolation_mode)(
                probs_reshaped[:, None, ...])
        return probs_reshaped
