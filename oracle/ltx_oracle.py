"""CPU oracle for the LTX-Video DiT training step — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this module.  The product path
(``finetrainers_b200``) never does; it fails loudly when the CUDA library is missing.

What this restates (plain PyTorch, runs on CPU in fp32 or bf16; autograd gives the
reference gradients).  Citations are relative to the reference repository's root:

* top-level transformer forward ........ finetrainers/patches/models/ltx_video/patch.py:38-127
* RoPE application (interleaved pairs) . finetrainers/patches/models/ltx_video/patch.py:23-33
* RMSNorm numerics ..................... finetrainers/patches/dependencies/diffusers/rms_norm.py:17-30
* noising / packing / timesteps / target finetrainers/models/ltx_video/base_specification.py:271-345, 427-459
* flow-match x_t / target .............. finetrainers/functional/diffusion.py:4-11
* sigma sampling, loss weights ......... finetrainers/utils/diffusion.py:38-63, 84-130
* loss + backward ...................... finetrainers/trainer/sft_trainer/trainer.py:463-481
* LoRA policy (r, alpha, fp32 adapters)  finetrainers/trainer/sft_trainer/trainer.py:120-136
* module tree / dims ................... tests/models/ltx_video/_test_tp.py:29-59, 186-245
* tiny plumbing config ................. tests/models/ltx_video/base_specification.py:46-63

PARITY UNPINNED for model output / loss: the arithmetic of the blocks lives in
``diffusers`` (>=0.32.1, tested 0.33.0.dev0; requirements.txt:4, docs/environment.md:6) and
``peft`` (>=0.13.0; requirements.txt:8), neither vendored in the reference nor installed
here, and the reference's own tests hold no golden tensor for this path
(tests/trainer/test_sft_trainer.py:110-113 only assert "does not raise").  The block
dataflow, AdaLN-single, PixArt text projection, LTX RoPE table and peft LoRA forward below
are restated from the published diffusers/peft algorithms.  What IS pinned: the attention
sub-op against ``torch`` math SDPA with the reference's own recipe and tolerances
(tests/models/attention_dispatch.py:41-111; see tests/test_attention_kat.py).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, asdict
from typing import Dict, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------------
# Config (tests/models/ltx_video/_test_tp.py:29-59 real size; tests/models/ltx_video/base_specification.py:46-63 tiny)
# ----------------------------------------------------------------------------------------------
@dataclass
class LTXConfig:
    in_channels: int = 128
    out_channels: int = 128
    patch_size: int = 1
    patch_size_t: int = 1
    num_attention_heads: int = 32
    attention_head_dim: int = 64
    cross_attention_dim: int = 2048
    num_layers: int = 28
    caption_channels: int = 4096
    norm_eps: float = 1e-6
    qk_norm_eps: float = 1e-5  # diffusers Attention default eps for qk_norm="rms_norm_across_heads"
    ffn_mult: int = 4

    @property
    def inner_dim(self) -> int:
        return self.num_attention_heads * self.attention_head_dim

    def to_dict(self):
        return asdict(self)

    @staticmethod
    def ltx_2b() -> "LTXConfig":
        return LTXConfig()

    @staticmethod
    def tiny() -> "LTXConfig":
        # the reference's dummy LTX: tests/models/ltx_video/base_specification.py:46-63
        return LTXConfig(in_channels=8, out_channels=8, num_attention_heads=4, attention_head_dim=8,
                         cross_attention_dim=32, num_layers=1, caption_channels=32)


# ----------------------------------------------------------------------------------------------
# Leaf modules
# ----------------------------------------------------------------------------------------------
class RMSNorm(nn.Module):
    """finetrainers/patches/dependencies/diffusers/rms_norm.py:17-30 (torch>=2.4 branch)."""

    def __init__(self, dim: int, eps: float, elementwise_affine: bool):
        super().__init__()
        self.eps = eps
        self.dim = dim
        self.weight = nn.Parameter(torch.ones(dim)) if elementwise_affine else None

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        input_dtype = x.dtype
        if self.weight is not None and self.weight.dtype in (torch.float16, torch.bfloat16):
            x = x.to(self.weight.dtype)
        x = F.rms_norm(x, (x.shape[-1],), weight=self.weight, eps=self.eps)
        return x.to(input_dtype)


class LoraLinear(nn.Module):
    """peft ``lora.Linear`` restated: y = base(x) + B(A(x.to(A.dtype))) * (alpha/r), result cast back to
    base dtype.  Parameter names follow peft so that state_dicts interchange
    (``base_layer.weight``, ``lora_A.default.weight``, ``lora_B.default.weight``)."""

    def __init__(self, base: nn.Linear, r: int, alpha: float):
        super().__init__()
        self.base_layer = base
        self.lora_A = nn.ModuleDict({"default": nn.Linear(base.in_features, r, bias=False)})
        self.lora_B = nn.ModuleDict({"default": nn.Linear(r, base.out_features, bias=False)})
        self.scaling = alpha / r
        self.r = r
        nn.init.kaiming_uniform_(self.lora_A["default"].weight, a=math.sqrt(5))
        nn.init.zeros_(self.lora_B["default"].weight)
        base.weight.requires_grad_(False)
        if base.bias is not None:
            base.bias.requires_grad_(False)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        result = self.base_layer(x)
        torch_result_dtype = result.dtype
        a = self.lora_A["default"]
        b = self.lora_B["default"]
        xa = x.to(a.weight.dtype)
        result = result + b(a(xa)) * self.scaling
        return result.to(torch_result_dtype)


class TimestepEmbedder(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.linear_1 = nn.Linear(256, dim)
        self.linear_2 = nn.Linear(dim, dim)

    def forward(self, x):
        return self.linear_2(F.silu(self.linear_1(x)))


class _Emb(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.timestep_embedder = TimestepEmbedder(dim)


def sinusoid_256(timesteps: torch.Tensor) -> torch.Tensor:
    """diffusers ``Timesteps(256, flip_sin_to_cos=True, downscale_freq_shift=0)`` -> [cos | sin], fp32."""
    half = 128
    exponent = -math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=timesteps.device) / half
    emb = timesteps[:, None].float() * torch.exp(exponent)[None, :]
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


class AdaLayerNormSingle(nn.Module):
    """diffusers AdaLayerNormSingle (module tree _test_tp.py:188-199): returns (temb[6D], embedded_timestep[D])."""

    def __init__(self, dim: int):
        super().__init__()
        self.emb = _Emb(dim)
        self.linear = nn.Linear(dim, 6 * dim)

    def forward(self, timestep: torch.Tensor, hidden_dtype: torch.dtype):
        proj = sinusoid_256(timestep).to(hidden_dtype)
        embedded = self.emb.timestep_embedder(proj)
        return self.linear(F.silu(embedded)), embedded


class TextProjection(nn.Module):
    """diffusers PixArtAlphaTextProjection (module tree _test_tp.py:200-204)."""

    def __init__(self, in_features: int, hidden: int):
        super().__init__()
        self.linear_1 = nn.Linear(in_features, hidden)
        self.linear_2 = nn.Linear(hidden, hidden)

    def forward(self, x):
        return self.linear_2(F.gelu(self.linear_1(x), approximate="tanh"))


def ltx_rope_table(num_frames: int, height: int, width: int, dim: int, rope_interpolation_scale,
                   batch_size: int = 1, device="cpu", base_num_frames: int = 20, base_height: int = 2048,
                   base_width: int = 2048, patch_size: int = 1, patch_size_t: int = 1, theta: float = 10000.0):
    """diffusers ``LTXVideoRotaryPosEmbed.forward`` restated (called at patch.py:52). fp32 cos/sin [B,S,dim]."""
    grid_f = torch.arange(num_frames, dtype=torch.float32, device=device)
    grid_h = torch.arange(height, dtype=torch.float32, device=device)
    grid_w = torch.arange(width, dtype=torch.float32, device=device)
    grid = torch.stack(torch.meshgrid(grid_f, grid_h, grid_w, indexing="ij"), dim=0)
    grid = grid.unsqueeze(0).repeat(batch_size, 1, 1, 1, 1)
    if rope_interpolation_scale is not None:
        grid[:, 0:1] = grid[:, 0:1] * rope_interpolation_scale[0] * patch_size_t / base_num_frames
        grid[:, 1:2] = grid[:, 1:2] * rope_interpolation_scale[1] * patch_size / base_height
        grid[:, 2:3] = grid[:, 2:3] * rope_interpolation_scale[2] * patch_size / base_width
    grid = grid.flatten(2, 4).transpose(1, 2)  # [B,S,3]
    freqs = theta ** torch.linspace(math.log(1.0, theta), math.log(theta, theta), dim // 6,
                                    device=device, dtype=torch.float32)
    freqs = freqs * math.pi / 2.0
    freqs = freqs * (grid.unsqueeze(-1) * 2 - 1)  # [B,S,3,dim//6]
    freqs = freqs.transpose(-1, -2).flatten(2)  # [B,S,(dim//6)*3], frequency-major then (f,h,w)
    cos = freqs.cos().repeat_interleave(2, dim=-1)
    sin = freqs.sin().repeat_interleave(2, dim=-1)
    if dim % 6 != 0:
        pad = dim % 6
        cos = torch.cat([torch.ones_like(cos[:, :, :pad]), cos], dim=-1)
        sin = torch.cat([torch.zeros_like(sin[:, :, :pad]), sin], dim=-1)
    return cos, sin


def apply_rotary_emb(x: torch.Tensor, freqs) -> torch.Tensor:
    """patch.py:23-33 (value-identical to the upstream ``unbind`` form)."""
    cos, sin = freqs
    x_real, x_imag = x.unflatten(2, (-1, 2)).unbind(-1)
    x_rotated = torch.stack([-x_imag, x_real], dim=-1).flatten(2)
    return (x.float() * cos + x_rotated.float() * sin).to(x.dtype)


class Attention(nn.Module):
    """diffusers ``Attention`` + ``LTXVideoAttentionProcessor2_0`` (module tree _test_tp.py:208-231)."""

    def __init__(self, cfg: LTXConfig, cross: bool):
        super().__init__()
        d = cfg.inner_dim
        kv_in = cfg.cross_attention_dim if cross else d
        self.heads = cfg.num_attention_heads
        self.norm_q = RMSNorm(d, cfg.qk_norm_eps, True)
        self.norm_k = RMSNorm(d, cfg.qk_norm_eps, True)
        self.to_q = nn.Linear(d, d, bias=True)
        self.to_k = nn.Linear(kv_in, d, bias=True)
        self.to_v = nn.Linear(kv_in, d, bias=True)
        self.to_out = nn.ModuleList([nn.Linear(d, d, bias=True), nn.Dropout(0.0)])

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, image_rotary_emb=None,
                sdpa=None):
        B = hidden_states.shape[0]
        if encoder_hidden_states is None:
            encoder_hidden_states = hidden_states
        q = self.to_q(hidden_states)
        k = self.to_k(encoder_hidden_states)
        v = self.to_v(encoder_hidden_states)
        q = self.norm_q(q)
        k = self.norm_k(k)
        if image_rotary_emb is not None:
            q = apply_rotary_emb(q, image_rotary_emb)
            k = apply_rotary_emb(k, image_rotary_emb)
        q = q.unflatten(2, (self.heads, -1)).transpose(1, 2)
        k = k.unflatten(2, (self.heads, -1)).transpose(1, 2)
        v = v.unflatten(2, (self.heads, -1)).transpose(1, 2)
        if attention_mask is not None:
            # [B,1,L] additive bias -> [B,H,1,L] (Attention.prepare_attention_mask + view in the processor)
            attention_mask = attention_mask.unsqueeze(1).expand(B, self.heads, 1, attention_mask.shape[-1])
        fn = sdpa or F.scaled_dot_product_attention
        o = fn(q, k, v, attn_mask=attention_mask, dropout_p=0.0, is_causal=False)
        o = o.transpose(1, 2).flatten(2, 3).to(q.dtype)
        o = self.to_out[0](o)
        return self.to_out[1](o)


class _GELUProj(nn.Module):
    def __init__(self, d_in, d_out):
        super().__init__()
        self.proj = nn.Linear(d_in, d_out)

    def forward(self, x):
        return F.gelu(self.proj(x), approximate="tanh")


class FeedForward(nn.Module):
    """diffusers FeedForward(activation_fn='gelu-approximate') (module tree _test_tp.py:232-240)."""

    def __init__(self, d: int, mult: int):
        super().__init__()
        self.net = nn.ModuleList([_GELUProj(d, d * mult), nn.Dropout(0.0), nn.Linear(d * mult, d)])

    def forward(self, x):
        for m in self.net:
            x = m(x)
        return x


class TransformerBlock(nn.Module):
    """diffusers ``LTXVideoTransformerBlock.forward`` restated."""

    def __init__(self, cfg: LTXConfig):
        super().__init__()
        d = cfg.inner_dim
        self.norm1 = RMSNorm(d, cfg.norm_eps, False)
        self.attn1 = Attention(cfg, cross=False)
        self.norm2 = RMSNorm(d, cfg.norm_eps, False)
        self.attn2 = Attention(cfg, cross=True)
        self.ff = FeedForward(d, cfg.ffn_mult)
        self.scale_shift_table = nn.Parameter(torch.randn(6, d) / d ** 0.5)

    def forward(self, hidden_states, encoder_hidden_states, temb, image_rotary_emb, encoder_attention_mask, sdpa=None):
        B = hidden_states.size(0)
        norm_h = self.norm1(hidden_states)
        ada = self.scale_shift_table[None, None] + temb.reshape(B, temb.size(1), 6, -1)
        shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = ada.unbind(dim=2)
        norm_h = norm_h * (1 + scale_msa) + shift_msa
        attn = self.attn1(norm_h, None, None, image_rotary_emb, sdpa=sdpa)
        hidden_states = hidden_states + attn * gate_msa
        attn = self.attn2(hidden_states, encoder_hidden_states, encoder_attention_mask, None, sdpa=sdpa)
        hidden_states = hidden_states + attn
        norm_h = self.norm2(hidden_states) * (1 + scale_mlp) + shift_mlp
        ff = self.ff(norm_h)
        hidden_states = hidden_states + ff * gate_mlp
        return hidden_states


class LTXTransformerOracle(nn.Module):
    """Same parameter FQNs as diffusers ``LTXVideoTransformer3DModel`` (+ peft after ``add_lora``)."""

    def __init__(self, cfg: LTXConfig):
        super().__init__()
        self.cfg = cfg
        d = cfg.inner_dim
        self.proj_in = nn.Linear(cfg.in_channels, d)
        self.scale_shift_table = nn.Parameter(torch.randn(2, d) / d ** 0.5)
        self.time_embed = AdaLayerNormSingle(d)
        self.caption_projection = TextProjection(cfg.caption_channels, d)
        self.transformer_blocks = nn.ModuleList([TransformerBlock(cfg) for _ in range(cfg.num_layers)])
        self.norm_out = nn.LayerNorm(d, eps=1e-6, elementwise_affine=False)
        self.proj_out = nn.Linear(d, cfg.out_channels)
        self.sdpa = None  # optional attention override (the provider hook, for tests)

    # -- patch.py:38-127 ------------------------------------------------------------------------
    def forward(self, hidden_states, encoder_hidden_states, timestep, encoder_attention_mask, num_frames, height,
                width, rope_interpolation_scale=None, return_dict=False):
        cfg = self.cfg
        B = hidden_states.size(0)
        rope = ltx_rope_table(num_frames, height, width, cfg.inner_dim, rope_interpolation_scale, B,
                              hidden_states.device, patch_size=cfg.patch_size, patch_size_t=cfg.patch_size_t)
        if encoder_attention_mask is not None and encoder_attention_mask.ndim == 2:
            encoder_attention_mask = (1 - encoder_attention_mask.to(hidden_states.dtype)) * -10000.0
            encoder_attention_mask = encoder_attention_mask.unsqueeze(1)
        if timestep.ndim == 1:
            timestep = timestep.view(-1, 1, 1).expand(-1, *hidden_states.shape[1:-1], -1)
        temb, embedded = self.time_embed(timestep.flatten(), hidden_dtype=hidden_states.dtype)
        temb = temb.view(B, *hidden_states.shape[1:-1], temb.size(-1))
        embedded = embedded.view(B, *hidden_states.shape[1:-1], embedded.size(-1))
        hidden_states = self.proj_in(hidden_states)
        encoder_hidden_states = self.caption_projection(encoder_hidden_states)
        encoder_hidden_states = encoder_hidden_states.view(B, -1, hidden_states.size(-1))
        for block in self.transformer_blocks:
            hidden_states = block(hidden_states, encoder_hidden_states, temb, rope, encoder_attention_mask,
                                  sdpa=self.sdpa)
        ssv = self.scale_shift_table[None, None] + embedded[:, :, None]
        shift, scale = ssv[:, :, 0], ssv[:, :, 1]
        hidden_states = self.norm_out(hidden_states)
        hidden_states = hidden_states * (1 + scale) + shift
        out = self.proj_out(hidden_states)
        return (out,)


LORA_TARGETS = ("to_q", "to_k", "to_v", "to_out.0")  # examples/training/sft/ltx_video/crush_smol_lora/train.sh:77


def add_lora(model: LTXTransformerOracle, rank: int, alpha: float) -> None:
    """trainer.py:96-136: freeze everything, inject adapters on to_q|to_k|to_v|to_out.0 of attn1+attn2."""
    for p in model.parameters():
        p.requires_grad_(False)
    for blk in model.transformer_blocks:
        for attn in (blk.attn1, blk.attn2):
            attn.to_q = LoraLinear(attn.to_q, rank, alpha)
            attn.to_k = LoraLinear(attn.to_k, rank, alpha)
            attn.to_v = LoraLinear(attn.to_v, rank, alpha)
            attn.to_out[0] = LoraLinear(attn.to_out[0], rank, alpha)


def synthetic_init_(model: nn.Module, seed: int = 0, lora_b_std: float = 0.01) -> None:
    """SURVEY §8(d) deterministic synthetic init: weights randn*0.02, biases randn*0.02 (non-zero so bias paths
    are exercised), qk-norm weights 1+randn*0.1, scale_shift_tables randn/sqrt(D), LoRA-A kaiming-uniform,
    LoRA-B randn*lora_b_std.  Identical generator walk for oracle and product (same FQN order)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(model.named_parameters(), key=lambda kv: kv[0]):
            shape = p.shape
            if "scale_shift_table" in name:
                v = torch.randn(shape, generator=g) / shape[-1] ** 0.5
            elif "lora_A" in name:
                bound = 1.0 / math.sqrt(shape[1])
                v = (torch.rand(shape, generator=g) * 2 - 1) * bound
            elif "lora_B" in name:
                v = torch.randn(shape, generator=g) * lora_b_std
            elif "norm_q" in name or "norm_k" in name:
                v = 1.0 + torch.randn(shape, generator=g) * 0.1
            else:
                v = torch.randn(shape, generator=g) * 0.02
            p.copy_(v.to(p.dtype))


# ----------------------------------------------------------------------------------------------
# ModelSpecification.forward / loss (base_specification.py:271-345, trainer.py:463-481)
# ----------------------------------------------------------------------------------------------
def normalize_latents(latents, latents_mean, latents_std, scaling_factor: float = 1.0):
    B = latents.shape[0]
    m = latents_mean.view(B, -1, 1, 1, 1).to(latents.device)
    s = latents_std.view(B, -1, 1, 1, 1).to(latents.device)
    return ((latents.float() - m) * scaling_factor / s).to(latents)


def pack_latents(latents, patch_size: int = 1, patch_size_t: int = 1):
    B, C, Fr, H, W = latents.shape
    latents = latents.reshape(B, -1, Fr // patch_size_t, patch_size_t, H // patch_size, patch_size,
                              W // patch_size, patch_size)
    return latents.permute(0, 2, 4, 6, 1, 3, 5, 7).flatten(4, 7).flatten(1, 3)


def flow_match_xt(x0, n, t):
    return (1.0 - t) * x0 + t * n


def flow_match_target(n, x0):
    return n - x0


def prepare_sigmas(scheduler_sigmas: torch.Tensor, batch_size: int, num_train_timesteps: int = 1000,
                   flow_weighting_scheme: str = "none", flow_logit_mean: float = 0.0, flow_logit_std: float = 1.0,
                   flow_mode_scale: float = 1.29, device="cpu", generator=None):
    """utils/diffusion.py:38-63,84-114."""
    if flow_weighting_scheme == "logit_normal":
        u = torch.normal(mean=flow_logit_mean, std=flow_logit_std, size=(batch_size,), device=device,
                         generator=generator)
        u = torch.sigmoid(u)
    elif flow_weighting_scheme == "mode":
        u = torch.rand(size=(batch_size,), device=device, generator=generator)
        u = 1 - u - flow_mode_scale * (torch.cos(math.pi * u / 2) ** 2 - 1 + u)
    else:
        u = torch.rand(size=(batch_size,), device=device, generator=generator)
    idx = (u * num_train_timesteps).long()
    return scheduler_sigmas[idx]


def flow_match_scheduler_sigmas(num_train_timesteps: int = 1000) -> torch.Tensor:
    """diffusers FlowMatchEulerDiscreteScheduler() defaults (shift=1): sigmas[i] = (N - i)/N, plus a final 0."""
    ts = torch.linspace(1, num_train_timesteps, num_train_timesteps, dtype=torch.float32).flip(0)
    sig = ts / num_train_timesteps
    return torch.cat([sig, torch.zeros(1)])


def loss_weights(sigmas: torch.Tensor, scheme: str = "none") -> torch.Tensor:
    """diffusers ``compute_loss_weighting_for_sd3`` via utils/diffusion.py:117-130."""
    if scheme == "sigma_sqrt":
        return (sigmas ** -2.0).float()
    if scheme == "cosmap":
        bot = 1 - 2 * sigmas + 2 * sigmas ** 2
        return 2 / (math.pi * bot)
    return torch.ones_like(sigmas)


def spec_forward(transformer, latents, latents_mean, latents_std, encoder_hidden_states, encoder_attention_mask,
                 sigmas, noise: Optional[torch.Tensor] = None, generator=None, first_frame_sigma=None):
    """``LTXVideoModelSpecification.forward`` (base_specification.py:271-345). ``noise`` may be injected so that the
    CUDA path and the oracle see identical noise; ``first_frame_sigma`` reproduces the 10 % branch when given."""
    cfg = transformer.cfg
    B, C, Fr, H, W = latents.shape
    latents = normalize_latents(latents, latents_mean, latents_std)
    if noise is None:
        noise = torch.zeros_like(latents).normal_(generator=generator)
    if first_frame_sigma is not None:
        ff = torch.min(first_frame_sigma, sigmas.new_full(sigmas.shape, 0.25))
        noisy = torch.cat([flow_match_xt(latents[:, :, :1], noise[:, :, :1], ff),
                           flow_match_xt(latents[:, :, 1:], noise[:, :, 1:], sigmas)], dim=2)
    else:
        noisy = flow_match_xt(latents, noise, sigmas)
    lat_p = pack_latents(latents, cfg.patch_size, cfg.patch_size_t)
    noise_p = pack_latents(noise, cfg.patch_size, cfg.patch_size_t)
    noisy_p = pack_latents(noisy, cfg.patch_size, cfg.patch_size_t)
    sig = sigmas.view(-1, 1, 1).expand(-1, *noisy_p.shape[1:-1], -1)
    timesteps = (sig * 1000.0).long()
    rope_scale = [1 / (25 / 8), 32, 32]
    pred = transformer(hidden_states=noisy_p.to(lat_p), encoder_hidden_states=encoder_hidden_states,
                       timestep=timesteps, encoder_attention_mask=encoder_attention_mask, num_frames=Fr, height=H,
                       width=W, rope_interpolation_scale=rope_scale, return_dict=False)[0]
    target = flow_match_target(noise_p, lat_p)
    return pred, target, sig


def sft_loss(pred, target, sigmas, scheme: str = "none"):
    """trainer.py:463-481."""
    w = loss_weights(sigmas, scheme)
    while w.ndim < pred.ndim:
        w = w.unsqueeze(-1)
    loss = w.float() * (pred.float() - target.float()).pow(2)
    loss = loss.mean(list(range(1, loss.ndim)))
    return loss.mean()


def clip_grad_norm_(params, max_norm: float):
    """utils/torch.py:99-161 (L2, foreach semantics).  Pinned against the reference's own function by
    tests/golden/clip_golden.pt (tests/test_oracle_golden.py::test_clip_grad_norm_golden)."""
    grads = [p.grad for p in params if p.grad is not None]
    total = torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(g.float(), 2.0) for g in grads]), 2.0)
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    for g in grads:
        g.mul_(coef.to(g.dtype))
    return total


def make_synthetic_batch(cfg: LTXConfig, B: int, Fr: int, H: int, W: int, text_len: int = 128, seed: int = 1234,
                         dtype=torch.bfloat16, text_scale: float = 0.1) -> Dict[str, torch.Tensor]:
    """SURVEY §8(d) synthetic inputs (already-normalised latents; ragged text masks).  ``text_scale`` is the std of the
    text embeddings: 0.1 is the survey's throughput setting; 1.0 (T5-like magnitudes) gives the cross-attention logits
    an O(1) spread so that the attn2 q/k adapter gradients are well above bf16 rounding noise (parity tests use it)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    latents = torch.randn(B, cfg.in_channels, Fr, H, W, generator=g).to(dtype)
    ehs = (torch.randn(B, text_len, cfg.caption_channels, generator=g) * text_scale).to(dtype)
    lens = torch.randint(max(1, text_len // 8), text_len + 1, (B,), generator=g)
    mask = (torch.arange(text_len)[None, :] < lens[:, None])
    noise = torch.randn(B, cfg.in_channels, Fr, H, W, generator=g).to(dtype)
    u = torch.sigmoid(torch.randn(B, generator=g))
    sig_table = flow_match_scheduler_sigmas()
    sigmas = sig_table[(u * 1000).long()].view(B, 1, 1, 1, 1)
    return {
        "latents": latents,
        "latents_mean": torch.zeros(B, cfg.in_channels),
        "latents_std": torch.ones(B, cfg.in_channels),
        "encoder_hidden_states": ehs,
        "encoder_attention_mask": mask,
        "noise": noise,
        "sigmas": sigmas,
    }


def oracle_step(model: LTXTransformerOracle, batch: Dict[str, torch.Tensor], backward: bool = True):
    """One forward(+backward) of the restated reference step. Returns (loss, pred)."""
    dt = next(p for n, p in model.named_parameters() if "proj_in" in n).dtype
    pred, target, sig = spec_forward(
        model, batch["latents"].to(dt), batch["latents_mean"], batch["latents_std"],
        batch["encoder_hidden_states"].to(dt), batch["encoder_attention_mask"], batch["sigmas"],
        noise=batch["noise"].to(dt))
    loss = sft_loss(pred, target, sig)
    if backward:
        loss.backward()
    return loss.detach(), pred.detach()
