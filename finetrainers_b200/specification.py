"""``LTXVideoModelSpecification`` hot-path mirror: the ``forward`` contract finetrainers' ``SFTTrainer`` calls
(``finetrainers/models/modeling_utils.py:183-186``;
LTX: ``finetrainers/models/ltx_video/base_specification.py:271-345``), same argument names, same dict
mutation (``pop`` of latents / latents_mean / latents_std, insertion of ``hidden_states``), same return triple
``(pred, target, sigmas)``.  Normalise + noising + packing + target run as ONE libb2d kernel (K15) instead of ~12 ATen
launches; with ``compute_posterior=False`` the same launch first samples the latent from precomputed VAE moments
(``finetrainers/models/utils.py:8-31``).  Everything else is delegated to the H100 transformer module.
"""
from __future__ import annotations

import random
from typing import Dict, Optional, Tuple

import torch

from . import ops, sampling
from .model import B200LTXTransformer, LTXConfig


def moments_channels(shape, in_channels: int) -> int:
    """Latent channel count C of precomputed VAE moments ``[B, 2C, F, H, W]`` (mean | logvar); ``ValueError`` naming the
    shape unless dim 1 is even and equals ``2 * in_channels``."""
    if len(shape) != 5 or shape[1] % 2 or shape[1] != 2 * in_channels:
        raise ValueError(f"compute_posterior=False expects VAE moments [B, 2 * {in_channels}, F, H, W] (mean | logvar), "
                         f"got shape {tuple(shape)}")
    return shape[1] // 2


class LTXVideoModelSpecification:
    # TODO(aryan)-marked constants of the reference forward (base_specification.py:281-282, 325-334)
    first_frame_conditioning_p = 0.1
    min_first_frame_sigma = 0.25
    frame_rate = 25
    temporal_compression_ratio = 8
    vae_spatial_compression_ratio = 32

    def __init__(self, transformer_config: Optional[LTXConfig] = None, transformer_dtype=torch.bfloat16):
        self.transformer_config = transformer_config or LTXConfig()
        self.transformer_dtype = transformer_dtype

    # -- load_diffusion_models (base_specification.py:173-190) with random-init weights (no hub access here)
    def load_diffusion_models(self, device="cuda") -> Dict[str, object]:
        transformer = B200LTXTransformer(self.transformer_config, self.transformer_dtype, device)
        return {"transformer": transformer, "scheduler": FlowMatchSchedulerTable()}

    # -- modeling_utils.py:156-181
    def collate_conditions(self, data):
        from .data import collate
        return collate(data)

    def collate_latents(self, data):
        from .data import collate
        return collate(data)

    def forward(self, transformer: B200LTXTransformer, condition_model_conditions: Dict[str, torch.Tensor],
                latent_model_conditions: Dict[str, torch.Tensor], sigmas: torch.Tensor,
                generator: Optional[torch.Generator] = None, compute_posterior: bool = True,
                noise: Optional[torch.Tensor] = None, posterior_noise: Optional[torch.Tensor] = None,
                **kwargs) -> Tuple[torch.Tensor, ...]:
        """``compute_posterior=False``: ``latents`` holds the VAE moments ``[B, 2C, F, H, W]`` (mean | logvar), as the
        reference precomputes them; the latent is sampled from them inside the prologue kernel with eps drawn from
        ``generator`` before the noise (or ``posterior_noise`` when given), as ``DiagonalGaussianDistribution.sample``
        does."""
        latents = latent_model_conditions.pop("latents")
        latents_mean = latent_model_conditions.pop("latents_mean")
        latents_std = latent_model_conditions.pop("latents_std")
        dev = latents.device
        eps = None
        if compute_posterior:
            B, C, Fr, Hh, Ww = latents.shape
        else:
            C = moments_channels(latents.shape, transformer.cfg.in_channels)
            B, _, Fr, Hh, Ww = latents.shape
        latents = latents.to(torch.bfloat16).contiguous()
        if not compute_posterior:
            if posterior_noise is None:
                # models/utils.py:23-29: randn_tensor(mean.shape, generator, device, dtype) before the flow-match noise
                eps = torch.randn((B, C, Fr, Hh, Ww), generator=generator, device=dev, dtype=torch.bfloat16)
            else:
                eps = posterior_noise.to(torch.bfloat16).contiguous()
        if noise is None:
            # same draw as the reference: torch.zeros_like(latents).normal_(generator=generator) (:296)
            noise = torch.zeros((B, C, Fr, Hh, Ww), dtype=torch.bfloat16, device=dev).normal_(generator=generator)
        else:
            noise = noise.to(torch.bfloat16).contiguous()
        sig = sigmas.reshape(B).to(torch.float32).contiguous()
        sig_ff = None
        if random.random() < self.first_frame_conditioning_p:
            # base_specification.py:298-310: first latent frame gets sigma_1 = min(U[0,1) * sigma, 0.25)
            ff = torch.rand_like(sig) * sig
            sig_ff = torch.min(ff, torch.full_like(sig, self.min_first_frame_sigma)).contiguous()
        S = Fr * Hh * Ww
        x_t = torch.empty(B, S, C, dtype=torch.bfloat16, device=dev)
        target = torch.empty_like(x_t)
        mean32 = latents_mean.reshape(B, C).to(torch.float32).contiguous()
        std32 = latents_std.reshape(B, C).to(torch.float32).contiguous()
        if eps is None:
            ops.prep_noise_pack(latents, noise, mean32, std32, sig, sig_ff, x_t, target, B, C, Fr, Hh * Ww)
        else:
            ops.prep_posterior_noise_pack(latents, eps, noise, mean32, std32, sig, sig_ff, x_t, target, B, C, Fr, Hh * Ww)
        sig_tok = sig.view(B, 1, 1).expand(B, S, 1)
        timesteps = (sig_tok * 1000.0).long()  # fp32 multiply then truncate, as the reference (:320)
        latent_model_conditions["hidden_states"] = x_t
        latent_frame_rate = self.frame_rate / self.temporal_compression_ratio
        rope_interpolation_scale = [1 / latent_frame_rate, self.vae_spatial_compression_ratio,
                                    self.vae_spatial_compression_ratio]
        latent_model_conditions.setdefault("num_frames", Fr)
        latent_model_conditions.setdefault("height", Hh)
        latent_model_conditions.setdefault("width", Ww)
        pred = transformer(**latent_model_conditions, **condition_model_conditions, timestep=timesteps,
                           rope_interpolation_scale=rope_interpolation_scale, return_dict=False)[0]
        return pred, target, sig_tok

    def generate_latents(self, transformer: B200LTXTransformer, prompt_embeds: torch.Tensor,
                         prompt_attention_mask: torch.Tensor, negative_prompt_embeds: Optional[torch.Tensor] = None,
                         negative_prompt_attention_mask: Optional[torch.Tensor] = None, *, num_frames: int, height: int,
                         width: int, frame_rate: float = 25, num_inference_steps: int = 50,
                         guidance_scale: float = sampling.GUIDANCE_SCALE, generator: Optional[torch.Generator] = None,
                         latents: Optional[torch.Tensor] = None, sigmas=None, cuda_graph: bool = True,
                         image_latents: Optional[torch.Tensor] = None, latents_mean=None,
                         latents_std=None) -> torch.Tensor:
        """Validation sampling without diffusers: what ``LTXPipeline(transformer=..., output_type="latent")`` returns for
        the given prompt embeddings [B, L, caption_channels] and masks [B, L], the packed normalised latents
        [B, S, C] fp32 (VAE decode stays with the caller).  ``num_frames`` / ``height`` / ``width`` are pixel sizes,
        converted to the latent grid by the compression ratios; ``latents`` (packed [B, S, C]) replaces the first draw
        ``randn((B, C, F, H, W), generator)``; ``sigmas`` replaces the base schedule ``linspace(1, 1 / N, N)``.  Guidance
        is on iff ``guidance_scale > 1``.  Each step is a no-grad forward and one guided Euler launch; steps after the
        first replay one CUDA graph (``cuda_graph=False``: every step eager, the same bits; a model sharded with FSDP-2
        always runs eagerly).  Bad input raises ValueError before anything is launched.

        ``image_latents``: image-to-video, what ``LTXImageToVideoPipeline(output_type="latent")`` returns.  It is the raw
        VAE latent of the conditioning image, [B, C, 1, H, W] at the latent grid (the caller encodes), with the VAE's
        ``latents_mean`` and ``latents_std`` ([C]).  As the pipeline's ``prepare_latents`` does in fp32, it is normalised
        to ``(x - mean) * 1.0 / std``, repeated over the F latent frames and blended with the noise as
        ``init * mask + noise * (1 - mask)`` (mask 1 on latent frame 0) before packing; ``latents`` then replaces only
        the noise draw.  Latent frame 0 keeps the normalised image latents through every step.  The pipeline draws its
        VAE posterior sample from ``generator`` before this noise, so a caller that wants the pipeline's random stream
        draws it first."""
        tr, sr = self.temporal_compression_ratio, self.vae_spatial_compression_ratio
        if (num_frames - 1) % tr or num_frames < 1 or height % sr or width % sr or height < sr or width < sr:
            raise ValueError(f"num_frames - 1 must be a multiple of {tr} and height, width positive multiples of {sr} "
                             f"(got {num_frames} x {height} x {width})")
        if sigmas is None and num_inference_steps < 1:
            raise ValueError(f"num_inference_steps must be at least 1, not {num_inference_steps}")
        cfg = guidance_scale > 1.0
        if cfg and (negative_prompt_embeds is None or negative_prompt_attention_mask is None):
            raise ValueError(f"guidance_scale = {guidance_scale} > 1 needs negative_prompt_embeds and "
                             "negative_prompt_attention_mask (classifier-free guidance)")
        B, L = prompt_embeds.shape[:2]
        if tuple(prompt_attention_mask.shape) != (B, L):
            raise ValueError(f"prompt_attention_mask must be [{B}, {L}], not {tuple(prompt_attention_mask.shape)}")
        if cfg and (tuple(negative_prompt_embeds.shape) != tuple(prompt_embeds.shape)
                    or tuple(negative_prompt_attention_mask.shape) != (B, L)):
            raise ValueError(f"negative prompt embeddings {tuple(negative_prompt_embeds.shape)} and mask "
                             f"{tuple(negative_prompt_attention_mask.shape)} must match the prompt's "
                             f"{tuple(prompt_embeds.shape)} and ({B}, {L}): the two halves of the guidance batch share L")
        Fl, Hl, Wl = (num_frames - 1) // tr + 1, height // sr, width // sr
        C, S = transformer.cfg.in_channels, Fl * Hl * Wl
        dev = transformer.proj_in.weight.device
        if latents is not None and tuple(latents.shape) != (B, S, C):
            raise ValueError(f"latents must be packed [{B}, {S}, {C}], not {tuple(latents.shape)}")
        if image_latents is not None:
            mean, std = self._check_image_latents(image_latents, latents_mean, latents_std, B, C, Fl, Hl, Wl)
        elif latents_mean is not None or latents_std is not None:
            raise ValueError("latents_mean and latents_std normalise image_latents, which was not given")
        sig = sampling.ltx_sigmas(num_inference_steps, S, sigmas=sigmas)
        if latents is None:
            # LTXPipeline.prepare_latents -> randn_tensor: drawn on the generator's device when that is the CPU
            gdev = generator.device if (generator is not None and generator.device.type == "cpu") else dev
            noise = torch.randn((B, C, Fl, Hl, Wl), generator=generator, device=gdev, dtype=torch.float32)
        else:
            noise = latents.to(torch.float32).transpose(1, 2).reshape(B, C, Fl, Hl, Wl)
        noise = noise.to(dev)
        if image_latents is not None:
            # LTXImageToVideoPipeline.prepare_latents (fp32): normalise, repeat over the frames, blend with the noise
            init = (image_latents.to(device=dev, dtype=torch.float32) - mean.to(dev).view(1, -1, 1, 1, 1)) * 1.0 \
                / std.to(dev).view(1, -1, 1, 1, 1)
            init = init.repeat(1, 1, Fl, 1, 1)
            mask = torch.zeros((B, 1, Fl, Hl, Wl), dtype=torch.float32, device=dev)
            mask[:, :, 0] = 1.0
            noise = init * mask + noise * (1 - mask)
        latents = sampling.pack_latents(noise).contiguous().clone()
        rope = (tr / frame_rate, sr, sr)
        graph = cuda_graph and getattr(transformer, "_fsdp", None) is None
        return sampling.sample(transformer, prompt_embeds, prompt_attention_mask, negative_prompt_embeds,
                               negative_prompt_attention_mask, latents, sig, num_frames=Fl, height=Hl, width=Wl,
                               rope_interpolation_scale=rope, guidance_scale=guidance_scale, cuda_graph=graph,
                               cond_tokens=Hl * Wl if image_latents is not None else 0)

    @staticmethod
    def _check_image_latents(image_latents, latents_mean, latents_std, B, C, Fl, Hl, Wl):
        """ValueError unless the conditioning image's latents are floating [B, C, 1, Hl, Wl] with mean and std of C
        values, and the video has a latent frame after the image's; -> (mean, std) as fp32 [C]."""
        if not isinstance(image_latents, torch.Tensor) or not image_latents.is_floating_point() \
                or tuple(image_latents.shape) != (B, C, 1, Hl, Wl):
            raise ValueError(f"image_latents must be a floating-point [{B}, {C}, 1, {Hl}, {Wl}] tensor (the VAE latent "
                             f"of the conditioning image), not {getattr(image_latents, 'dtype', type(image_latents))} "
                             f"{tuple(getattr(image_latents, 'shape', ()))}")
        if Fl < 2:
            raise ValueError("image-to-video needs a latent frame after the conditioning image's: num_frames >= 9")
        out = []
        for name, v in (("latents_mean", latents_mean), ("latents_std", latents_std)):
            if v is None:
                raise ValueError(f"image_latents needs {name} (the VAE's, [{C}])")
            t = torch.as_tensor(v)
            if not t.is_floating_point() or tuple(t.shape) != (C,):
                raise ValueError(f"{name} must be floating-point [{C}], not {t.dtype} {tuple(t.shape)}")
            out.append(t.to(torch.float32))
        return out


class FlowMatchSchedulerTable:
    """diffusers ``FlowMatchEulerDiscreteScheduler()`` defaults as far as the trainer reads them
    (``scheduler.sigmas``, ``config.num_train_timesteps``; utils/diffusion.py:66-74): sigmas[i] = (1000 - i)/1000, then 0."""

    class _Cfg:
        num_train_timesteps = 1000

    def __init__(self):
        self.config = self._Cfg()
        ts = torch.linspace(1, 1000, 1000, dtype=torch.float32).flip(0)
        self.sigmas = torch.cat([ts / 1000.0, torch.zeros(1)])
