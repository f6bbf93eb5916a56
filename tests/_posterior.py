"""Test-side restatement of the reference's posterior sampling on precomputed VAE moments (``compute_posterior=False``;
finetrainers/models/ltx_video/base_specification.py:285-290, finetrainers/models/utils.py:8-31), in plain torch, on top
of the CPU oracle (oracle/ltx_oracle.py).  Pinned against the reference's own class by
tests/golden/posterior_golden.pt."""
from typing import Optional

import torch


def posterior_sample(moments: torch.Tensor, generator=None, eps: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``DiagonalGaussianDistribution(moments).sample(generator)``: moments ``[B, 2C, ...]`` = mean | logvar, computed
    in the moments' dtype; diffusers' ``randn_tensor`` on the parameters' device is ``torch.randn``.  ``eps`` may be
    injected in place of the draw."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    std = torch.exp(0.5 * logvar)
    if eps is None:
        eps = torch.randn(mean.shape, generator=generator, device=moments.device, dtype=moments.dtype)
    return mean + std * eps.to(moments.dtype)


def spec_forward_moments(transformer, moments, latents_mean, latents_std, encoder_hidden_states,
                         encoder_attention_mask, sigmas, noise=None, generator=None, first_frame_sigma=None,
                         posterior_eps: Optional[torch.Tensor] = None):
    """The oracle's ``spec_forward`` on the posterior path: the latents are sampled from the moments first (eps from
    ``generator`` before the noise, or ``posterior_eps``)."""
    from oracle.ltx_oracle import spec_forward
    latents = posterior_sample(moments, generator, posterior_eps)
    return spec_forward(transformer, latents, latents_mean, latents_std, encoder_hidden_states, encoder_attention_mask,
                        sigmas, noise=noise, generator=generator, first_frame_sigma=first_frame_sigma)
