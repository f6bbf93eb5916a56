"""Validation sampling: the transformer-only half of ``SFTTrainer._validate``
(``finetrainers/trainer/sft_trainer/trainer.py:583-700``), which hands the training transformer to diffusers'
``LTXPipeline`` and calls it once per denoising step under ``torch.no_grad()``.  Here prompt embeddings go in and the
packed latents come out (``LTXPipeline(..., output_type="latent")``); T5 encoding and VAE decode stay with the caller.

Each step is one no-grad forward of the transformer (its inference plan, ``B200LTXTransformer.workspace_plan(...,
inference=True)``) and one ``b2d_cfg_euler_step`` launch (guidance + Euler update + the next step's bf16 input); with a
conditioning image (``LTXImageToVideoPipeline``), per-frame timesteps and one ``b2d_cfg_euler_step_cond`` launch.  The
first step runs eagerly, the same step is then captured in one CUDA graph and replayed for the rest, with the timestep
and the Euler step size reaching the graph through static device buffers: no host-device synchronisation inside the loop.

Upstream constants, restated from the published sources (diffusers 0.32-0.33; not checked against diffusers, which is not
a dependency of this package; every value stays an argument):

| constant | value | upstream symbol |
|---|---|---|
| base sigmas | ``linspace(1, 1 / N, N)`` in float64, then float32 | ``LTXPipeline.__call__`` (``sigmas=None``); ``FlowMatchEulerDiscreteScheduler.set_timesteps``: ``np.array(sigmas).astype(np.float32)`` |
| shift ``mu`` | ``seq_len * m + b``, ``m = (max_shift - base_shift) / (max_seq_len - base_seq_len)``, ``b = base_shift - m * base_seq_len`` | ``diffusers.pipelines.ltx.pipeline_ltx.calculate_shift`` |
| shift inputs | ``base_image_seq_len 1024``, ``max_image_seq_len 4096``, ``base_shift 0.95``, ``max_shift 2.05`` | LTX-Video ``scheduler/scheduler_config.json`` (read by ``LTXPipeline.__call__``) |
| time shift | ``e^mu / (e^mu + (1 / sigma - 1) ** 1)`` | ``FlowMatchEulerDiscreteScheduler.time_shift`` (``use_dynamic_shifting=True``, ``time_shift_type="exponential"``) |
| terminal stretch | ``1 - (1 - sigma) / ((1 - sigma[-1]) / (1 - shift_terminal))``, ``shift_terminal 0.1`` | ``FlowMatchEulerDiscreteScheduler.stretch_shift_to_terminal``; LTX-Video scheduler config |
| timesteps | ``sigma * 1000`` in float32 (``num_train_timesteps 1000``), then a trailing sigma 0 | ``FlowMatchEulerDiscreteScheduler.set_timesteps`` |
| Euler step | ``x + (sigma_next - sigma) * v`` in float32 | ``FlowMatchEulerDiscreteScheduler.step`` |
| guidance | ``u + g (c - u)`` on ``noise_pred.float().chunk(2)``, ``g = 3.0``, on iff ``g > 1`` | ``LTXPipeline.__call__`` defaults |
| first latents | ``randn((B, C, F, H, W), float32)`` then packed to ``[B, F H W, C]`` | ``LTXPipeline.prepare_latents`` / ``_pack_latents`` |
| image latents | ``(x - mean) * 1.0 / std`` (``scaling_factor 1.0``), repeated over F, ``init * mask + noise * (1 - mask)`` with ``mask`` 1 on latent frame 0 | ``LTXImageToVideoPipeline.prepare_latents`` / ``_normalize_latents`` |
| image timesteps | ``t.expand(rows).unsqueeze(-1) * (1 - mask)``, mask packed to ``[rows, F H W]`` | ``LTXImageToVideoPipeline.__call__`` |
| image step | Euler step on latent frames 1.. only, frame 0 kept | ``LTXImageToVideoPipeline.__call__`` (``noise_pred[:, :, 1:]``, ``torch.cat([latents[:, :, :1], pred_latents], 2)``) |
| RoPE scale | ``(temporal_ratio / frame_rate, spatial_ratio, spatial_ratio)``, ``frame_rate 25`` | ``LTXPipeline.__call__`` |
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import numpy as np
import torch

from . import ops

BASE_IMAGE_SEQ_LEN = 1024
MAX_IMAGE_SEQ_LEN = 4096
BASE_SHIFT = 0.95
MAX_SHIFT = 2.05
SHIFT_TERMINAL = 0.1
GUIDANCE_SCALE = 3.0
NUM_TRAIN_TIMESTEPS = 1000


def calculate_shift(seq_len: int, base_seq_len: int = BASE_IMAGE_SEQ_LEN, max_seq_len: int = MAX_IMAGE_SEQ_LEN,
                    base_shift: float = BASE_SHIFT, max_shift: float = MAX_SHIFT) -> float:
    """``mu`` of the exponential time shift: linear in the latent sequence length (float64, as the pipeline)."""
    m = (max_shift - base_shift) / (max_seq_len - base_seq_len)
    b = base_shift - m * base_seq_len
    return seq_len * m + b


def ltx_sigmas(num_inference_steps: int, video_seq_len: int, *, base_seq_len: int = BASE_IMAGE_SEQ_LEN,
               max_seq_len: int = MAX_IMAGE_SEQ_LEN, base_shift: float = BASE_SHIFT, max_shift: float = MAX_SHIFT,
               shift_terminal: Optional[float] = SHIFT_TERMINAL,
               sigmas: Optional[Sequence[float]] = None) -> torch.Tensor:
    """The sigma schedule ``LTXPipeline`` sets on its scheduler: fp32 ``[N + 1]``, strictly decreasing from ~1 to
    ``shift_terminal`` and then 0.  ``sigmas`` replaces the base ``linspace(1, 1 / N, N)`` (the pipeline's argument of
    that name; N is then its length).  Every step after the float64 linspace runs in float32, as the scheduler's numpy
    float32 arithmetic does.  The timesteps the transformer sees are ``sigmas[:-1] * 1000`` in float32."""
    if sigmas is None:
        if num_inference_steps < 1:
            raise ValueError(f"num_inference_steps must be at least 1, not {num_inference_steps}")
        sigmas = np.linspace(1.0, 1.0 / num_inference_steps, num_inference_steps)
    s = np.asarray(sigmas, dtype=np.float64).astype(np.float32)
    if s.ndim != 1 or s.size < 1:
        raise ValueError(f"sigmas must be a non-empty 1-D sequence, got shape {s.shape}")
    f32 = np.float32
    emu = f32(math.exp(calculate_shift(video_seq_len, base_seq_len, max_seq_len, base_shift, max_shift)))
    s = emu / (emu + (f32(1) / s - f32(1)) ** f32(1))
    if shift_terminal:
        one_minus = f32(1) - s
        if not one_minus[-1] > 0:
            raise ValueError("the stretch to shift_terminal needs a last sigma below 1 (one step of the default "
                             "schedule has none): use num_inference_steps >= 2 or shift_terminal=None")
        s = f32(1) - one_minus / (one_minus[-1] / f32(1 - shift_terminal))
    s = torch.from_numpy(s.astype(np.float32))
    return torch.cat([s, torch.zeros(1, dtype=torch.float32)])


def pack_latents(latents: torch.Tensor) -> torch.Tensor:
    """[B, C, F, H, W] -> [B, F H W, C] (``LTXPipeline._pack_latents`` at patch size 1)."""
    B, C = latents.shape[:2]
    return latents.reshape(B, C, -1).transpose(1, 2).contiguous()


@torch.no_grad()
def sample(transformer, prompt_embeds: torch.Tensor, prompt_attention_mask: torch.Tensor,
           negative_prompt_embeds: Optional[torch.Tensor], negative_prompt_attention_mask: Optional[torch.Tensor],
           latents: torch.Tensor, sigmas: torch.Tensor, *, num_frames: int, height: int, width: int,
           rope_interpolation_scale, guidance_scale: float = GUIDANCE_SCALE, cuda_graph: bool = True,
           cond_tokens: int = 0) -> torch.Tensor:
    """Denoise ``latents`` (fp32 ``[B, S, C]`` on the transformer's device, S = num_frames * height * width latent
    tokens; updated in place and returned) over the schedule ``sigmas`` (``[N + 1]``, as ``ltx_sigmas``).  Inputs are
    checked by the caller (``LTXVideoModelSpecification.generate_latents``).  ``cuda_graph=False`` runs every step
    eagerly; the result is the same bits.

    ``cond_tokens > 0``: the first ``cond_tokens`` tokens of each sample (the conditioning frame) stay as given, as in
    ``LTXImageToVideoPipeline``: the transformer gets the per-token timesteps ``t * (1 - conditioning_mask)`` ([rows,
    S] fp32, 0 on those tokens; the engine embeds them once per latent frame) and the step is
    ``b2d_cfg_euler_step_cond``, which leaves those tokens' latents and next input alone."""
    dev = latents.device
    B, S, C = latents.shape
    cfg = guidance_scale > 1.0  # LTXPipeline.do_classifier_free_guidance; the one place this is decided
    rows = 2 * B if cfg else B
    if cfg:
        ehs = torch.cat([negative_prompt_embeds, prompt_embeds])
        mask = torch.cat([negative_prompt_attention_mask, prompt_attention_mask])
    else:
        ehs, mask = prompt_embeds, prompt_attention_mask
    ehs = ehs.to(device=dev, dtype=torch.bfloat16).contiguous()
    mask = mask.to(dev).contiguous()
    sig = sigmas.to(device=dev, dtype=torch.float32)
    n_steps = sig.numel() - 1
    t_all = sig[:-1] * float(NUM_TRAIN_TIMESTEPS)   # scheduler.timesteps: fp32 sigma * 1000
    dt_all = sig[1:] - sig[:-1]                     # sigma_next - sigma in fp32, as scheduler.step
    # static buffers: what the step reads (x_in, t, dt) and writes (latents, x_in)
    x_in = latents.to(torch.bfloat16).repeat(rows // B, 1, 1)  # torch.cat([latents] * 2).to(bf16)
    if cond_tokens:
        keep = torch.ones(rows, S, dtype=torch.float32, device=dev)  # 1 - conditioning_mask, packed
        keep[:, :cond_tokens] = 0.0
        t_buf = torch.empty(rows, S, dtype=torch.float32, device=dev)
    else:
        t_buf = torch.empty(rows, dtype=torch.float32, device=dev)
    dt_buf = torch.empty(1, dtype=torch.float32, device=dev)
    n = S * C
    rope = tuple(float(r) for r in rope_interpolation_scale)

    def step():
        pred = transformer(hidden_states=x_in, encoder_hidden_states=ehs, timestep=t_buf,
                           encoder_attention_mask=mask, num_frames=num_frames, height=height, width=width,
                           rope_interpolation_scale=rope, return_dict=False)[0]
        if cond_tokens:
            ops.cfg_euler_step_cond(pred, latents, x_in, B, n, cond_tokens * C, cfg, guidance_scale, dt_buf)
        else:
            ops.cfg_euler_step(pred, latents, x_in, B, n, cfg, guidance_scale, dt_buf)

    graph = None
    for i in range(n_steps):
        if cond_tokens:
            torch.mul(t_all[i], keep, out=t_buf)  # t.expand(rows).unsqueeze(-1) * (1 - conditioning_mask)
        else:
            t_buf.copy_(t_all[i].expand(rows))
        dt_buf.copy_(dt_all[i:i + 1])
        if graph is not None:
            graph.replay()
            continue
        step()
        if cuda_graph and i + 1 < n_steps:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                step()
    del graph  # it holds pointers into the inference workspace, which the next forward at another shape frees
    return latents
