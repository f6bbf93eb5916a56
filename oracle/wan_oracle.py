"""CPU oracle for the Wan-2.1 T2V training step — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A plain-PyTorch restatement (CPU, fp32; autograd gives the reference gradients) of:

* diffusers ``WanTransformer3DModel`` (T2V: no image branch): Conv3d patch embedding, ``WanTimeTextImageEmbedding``
  (Timesteps(256, flip_sin_to_cos) -> time_embedder -> time_proj(silu), PixArt-style text_embedder with GELU-tanh),
  ``WanRotaryPosEmbed`` (per-head split 44 / 42 / 42 at head_dim 128, theta 10000, float64 frequencies),
  ``WanTransformerBlock`` (FP32LayerNorm norm1 / norm3 + modulation with the table added in fp32, self attention with
  RMSNorm-across-heads q/k and per-head RoPE, affine FP32LayerNorm norm2 before cross attention, GELU-tanh FFN),
  the final FP32LayerNorm + shift / scale and the unpatchify;
* peft LoRA on the attention projections (``ltx_oracle.LoraLinear``);
* the reference's Wan training forward (``finetrainers/models/wan/base_specification.py:433-493``, ``:571-576``) with
  ``compute_posterior`` forced False.

PARITY UNPINNED, as for LTX (DESIGN §2): diffusers is not vendored in the reference nor installed here, so the module
arithmetic is restated from diffusers' published source (``models/transformers/transformer_wan.py``), not run.  The
prologue functions ARE the reference's own torch code, run at fixture-generation time (tests/golden/make_wan_golden.py).
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.ltx_oracle import LoraLinear, RMSNorm, TextProjection, TimestepEmbedder, sinusoid_256

LORA_TARGETS = ("to_q", "to_k", "to_v", "to_out.0")


class WanOracleConfig:
    def __init__(self, num_attention_heads=12, attention_head_dim=128, in_channels=16, out_channels=16, text_dim=4096,
                 ffn_dim=8960, num_layers=30, eps=1e-6, rope_max_seq_len=1024):
        self.num_attention_heads, self.attention_head_dim = num_attention_heads, attention_head_dim
        self.in_channels, self.out_channels, self.text_dim = in_channels, out_channels, text_dim
        self.ffn_dim, self.num_layers, self.eps, self.rope_max_seq_len = ffn_dim, num_layers, eps, rope_max_seq_len
        self.patch_size = (1, 2, 2)

    @property
    def inner_dim(self):
        return self.num_attention_heads * self.attention_head_dim


def wan_rope_split(head_dim: int):
    """(t, h, w) dims of WanRotaryPosEmbed: h = w = 2 (head_dim // 6), t the rest."""
    hw = 2 * (head_dim // 6)
    return head_dim - 2 * hw, hw, hw


def wan_rope_freqs(head_dim: int, max_seq_len: int = 1024, theta: float = 10000.0) -> torch.Tensor:
    """WanRotaryPosEmbed.freqs: complex128 [max_seq_len, head_dim / 2], the t, h and w parts side by side
    (get_1d_rotary_pos_embed(dim, max_seq_len, theta, use_real=False, freqs_dtype=torch.float64))."""
    parts = []
    for dim in wan_rope_split(head_dim):
        freqs = 1.0 / (theta ** (torch.arange(0, dim, 2, dtype=torch.float64)[: dim // 2] / dim))
        freqs = torch.outer(torch.arange(max_seq_len), freqs)
        parts.append(torch.polar(torch.ones_like(freqs), freqs))
    return torch.cat(parts, dim=1)


def wan_rope(head_dim: int, ppf: int, pph: int, ppw: int, max_seq_len: int = 1024) -> torch.Tensor:
    """WanRotaryPosEmbed.forward on the post-patch grid: complex128 [1, 1, ppf pph ppw, head_dim / 2]."""
    t, h, _ = wan_rope_split(head_dim)
    ff, fh, fw = wan_rope_freqs(head_dim, max_seq_len).split_with_sizes([t // 2, h // 2, h // 2], dim=1)
    ff = ff[:ppf].view(ppf, 1, 1, -1).expand(ppf, pph, ppw, -1)
    fh = fh[:pph].view(1, pph, 1, -1).expand(ppf, pph, ppw, -1)
    fw = fw[:ppw].view(1, 1, ppw, -1).expand(ppf, pph, ppw, -1)
    return torch.cat([ff, fh, fw], dim=-1).reshape(1, 1, ppf * pph * ppw, -1)


def apply_rotary_emb(x: torch.Tensor, freqs: torch.Tensor) -> torch.Tensor:
    """WanAttnProcessor2_0.apply_rotary_emb: pairs (2i, 2i + 1) as complex numbers, rotated in float64."""
    xr = torch.view_as_complex(x.to(torch.float64).unflatten(3, (-1, 2)))
    return torch.view_as_real(xr * freqs).flatten(3, 4).type_as(x)


class FP32LayerNorm(nn.LayerNorm):
    def forward(self, x):
        w = self.weight.float() if self.weight is not None else None
        b = self.bias.float() if self.bias is not None else None
        return F.layer_norm(x.float(), self.normalized_shape, w, b, self.eps).to(x.dtype)


class Attention(nn.Module):
    def __init__(self, cfg: WanOracleConfig):
        super().__init__()
        d = cfg.inner_dim
        self.heads = cfg.num_attention_heads
        self.to_q, self.to_k, self.to_v = nn.Linear(d, d), nn.Linear(d, d), nn.Linear(d, d)
        self.to_out = nn.ModuleList([nn.Linear(d, d), nn.Dropout(0.0)])
        self.norm_q = RMSNorm(d, cfg.eps, True)
        self.norm_k = RMSNorm(d, cfg.eps, True)

    def forward(self, x, ctx=None, rotary_emb=None):
        ctx = x if ctx is None else ctx
        q, k, v = self.norm_q(self.to_q(x)), self.norm_k(self.to_k(ctx)), self.to_v(ctx)
        q, k, v = (t.unflatten(2, (self.heads, -1)).transpose(1, 2) for t in (q, k, v))
        if rotary_emb is not None:
            q, k = apply_rotary_emb(q, rotary_emb), apply_rotary_emb(k, rotary_emb)
        o = F.scaled_dot_product_attention(q, k, v)
        return self.to_out[0](o.transpose(1, 2).flatten(2, 3))


class _GELUProj(nn.Module):
    def __init__(self, d_in, d_out):
        super().__init__()
        self.proj = nn.Linear(d_in, d_out)

    def forward(self, x):
        return F.gelu(self.proj(x), approximate="tanh")


class FeedForward(nn.Module):
    def __init__(self, d, inner):
        super().__init__()
        self.net = nn.ModuleList([_GELUProj(d, inner), nn.Dropout(0.0), nn.Linear(inner, d)])

    def forward(self, x):
        for m in self.net:
            x = m(x)
        return x


class WanBlock(nn.Module):
    def __init__(self, cfg: WanOracleConfig):
        super().__init__()
        d = cfg.inner_dim
        self.norm1 = FP32LayerNorm(d, cfg.eps, elementwise_affine=False)
        self.attn1 = Attention(cfg)
        self.norm2 = FP32LayerNorm(d, cfg.eps, elementwise_affine=True)
        self.attn2 = Attention(cfg)
        self.ffn = FeedForward(d, cfg.ffn_dim)
        self.norm3 = FP32LayerNorm(d, cfg.eps, elementwise_affine=False)
        self.scale_shift_table = nn.Parameter(torch.randn(1, 6, d) / d ** 0.5)

    def forward(self, h, ctx, temb, rotary_emb):
        sh, sc, g, csh, csc, cg = (self.scale_shift_table + temb.float()).chunk(6, dim=1)
        n = (self.norm1(h.float()) * (1 + sc) + sh).type_as(h)
        h = (h.float() + self.attn1(n, rotary_emb=rotary_emb) * g).type_as(h)
        n = self.norm2(h.float()).type_as(h)
        h = h + self.attn2(n, ctx)
        n = (self.norm3(h.float()) * (1 + csc) + csh).type_as(h)
        return (h.float() + self.ffn(n).float() * cg).type_as(h)


class _CondEmbedder(nn.Module):
    def __init__(self, d, text_dim):
        super().__init__()
        self.time_embedder = TimestepEmbedder(d)
        self.time_proj = nn.Linear(d, 6 * d)
        self.text_embedder = TextProjection(text_dim, d)

    def forward(self, timestep, ehs):
        temb = self.time_embedder(sinusoid_256(timestep).to(ehs.dtype)).type_as(ehs)
        return temb, self.time_proj(F.silu(temb)), self.text_embedder(ehs)


class WanTransformerOracle(nn.Module):
    def __init__(self, cfg: WanOracleConfig):
        super().__init__()
        d = cfg.inner_dim
        self.cfg = cfg
        self.patch_embedding = nn.Conv3d(cfg.in_channels, d, kernel_size=cfg.patch_size, stride=cfg.patch_size)
        self.condition_embedder = _CondEmbedder(d, cfg.text_dim)
        self.blocks = nn.ModuleList([WanBlock(cfg) for _ in range(cfg.num_layers)])
        self.norm_out = FP32LayerNorm(d, cfg.eps, elementwise_affine=False)
        self.proj_out = nn.Linear(d, cfg.out_channels * 4)
        self.scale_shift_table = nn.Parameter(torch.randn(1, 2, d) / d ** 0.5)

    def forward(self, hidden_states, timestep, encoder_hidden_states):
        B, _, Fr, H, W = hidden_states.shape
        ppf, pph, ppw = Fr, H // 2, W // 2
        rotary = wan_rope(self.cfg.attention_head_dim, ppf, pph, ppw, self.cfg.rope_max_seq_len)
        h = self.patch_embedding(hidden_states).flatten(2).transpose(1, 2)
        temb, tproj, ctx = self.condition_embedder(timestep, encoder_hidden_states)
        tproj = tproj.unflatten(1, (6, -1))
        for blk in self.blocks:
            h = blk(h, ctx, tproj, rotary)
        shift, scale = (self.scale_shift_table + temb.unsqueeze(1)).chunk(2, dim=1)
        h = (self.norm_out(h.float()) * (1 + scale) + shift).type_as(h)
        h = self.proj_out(h)
        h = h.reshape(B, ppf, pph, ppw, 1, 2, 2, -1).permute(0, 7, 1, 4, 2, 5, 3, 6)
        return h.flatten(6, 7).flatten(4, 5).flatten(2, 3)


def add_lora(model: WanTransformerOracle, rank: int, alpha: float) -> None:
    """peft LoRA on blocks.*(to_q|to_k|to_v|to_out.0); every other parameter frozen."""
    for p in model.parameters():
        p.requires_grad_(False)
    for blk in model.blocks:
        for a in (blk.attn1, blk.attn2):
            for t in ("to_q", "to_k", "to_v"):
                setattr(a, t, LoraLinear(getattr(a, t), rank, alpha))
            a.to_out[0] = LoraLinear(a.to_out[0], rank, alpha)


def synthetic_init_(model: nn.Module, seed: int = 0, lora_b_std: float = 0.02) -> None:
    """Deterministic weights at the scale of a trained model: linear / conv weights U(+-1/sqrt(fan_in)), biases small,
    norm weights near 1, modulation tables N(0, 1/D), LoRA B non-zero so that every adapter gradient is non-trivial."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "lora_B" in n:
                p.copy_(torch.randn(p.shape, generator=g) * lora_b_std)
            elif "lora_A" in n:
                p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) / math.sqrt(p.shape[1]))
            elif "norm" in n and n.endswith("weight"):
                p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
            elif "norm" in n and n.endswith("bias"):
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            elif "scale_shift_table" in n:
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(p.shape[-1]))
            elif p.ndim >= 2:
                fan_in = p[0].numel()
                p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) / math.sqrt(fan_in))
            else:
                p.copy_(0.02 * torch.randn(p.shape, generator=g))


def normalize_latents(latents, latents_mean, latents_std):
    """WanModelSpecification._normalize_latents (base_specification.py:571-576); latents_std is already 1 / std."""
    mean = latents_mean.view(1, -1, 1, 1, 1).to(latents.device)
    std = latents_std.view(1, -1, 1, 1, 1).to(latents.device)
    return ((latents.float() - mean) * std).to(latents)


def prologue(moments, latents_mean, latents_std, eps, noise, sigmas):
    """The reference's Wan prologue with compute_posterior forced False (base_specification.py:446-478): normalise mean
    and logvar, sample the posterior with the given eps, noise -> (x_t, target), all [B, C, F, H, W] in moments' dtype."""
    mu, logvar = torch.chunk(moments, 2, dim=1)
    mu, logvar = normalize_latents(mu, latents_mean, latents_std), normalize_latents(logvar, latents_mean, latents_std)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    x = mu + torch.exp(0.5 * logvar) * eps
    t = sigmas.view(-1, 1, 1, 1, 1)
    return ((1.0 - t) * x + t * noise).to(x), noise - x


def oracle_step(model: WanTransformerOracle, moments, latents_mean, latents_std, eps, noise, sigmas,
                encoder_hidden_states, weights: Optional[torch.Tensor] = None):
    """fp32 forward + loss (mean over each sample, weighted, mean over the batch) + backward; -> (loss, pred)."""
    x_t, target = prologue(moments, latents_mean, latents_std, eps, noise, sigmas)
    timesteps = (sigmas.flatten() * 1000.0).long()
    pred = model(x_t.float(), timesteps, encoder_hidden_states.float())
    w = torch.ones(pred.shape[0]) if weights is None else weights
    loss = (w.view(-1, 1) * (pred.float() - target.float()).pow(2).flatten(1)).mean(1).mean()
    loss.backward()
    return loss.detach(), pred.detach()
