"""CPU oracle for the Wan-2.1 image-to-video (I2V) training step — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

``oracle.wan_oracle`` (the T2V restatement) plus what diffusers' ``WanTransformer3DModel`` adds with ``image_dim`` and
``added_kv_proj_dim`` (restated from the published ``models/transformers/transformer_wan.py``, which is not vendored in
the reference nor installed here, so this arithmetic is unpinned by upstream, as the T2V oracle's is, DESIGN §2):

* ``condition_embedder.image_embedder`` (``WanImageEmbedding`` without ``pos_embed``): ``FP32LayerNorm(image_dim)``,
  ``FeedForward(image_dim, inner_dim, mult=1, activation_fn="gelu")`` (Linear, exact GELU, Linear) and
  ``FP32LayerNorm(inner_dim)``.  Both LayerNorms are built with only the width, so they take ``nn.LayerNorm``'s default
  eps, 1e-5 (``IMAGE_NORM_EPS``; not the model's 1e-6, which is the blocks').
* The context is ``cat([image_embedder(encoder_hidden_states_image), text_embedder(encoder_hidden_states)], 1)``.
  Every block's ``attn2`` (``WanAttnProcessor2_0`` with ``add_k_proj``) splits it again at ``len - 512``; the image keys
  are ``norm_added_k(add_k_proj(img))`` (RMSNorm across heads, the model's eps, no ``norm_added_q``), the values
  ``add_v_proj(img)``; no RoPE and no mask on the image context; the output is ``to_out(sdpa(q, k_txt, v_txt)
  .type_as(q) + sdpa(q, k_img, v_img).type_as(q))`` (the two roundings are no-ops in this fp32 restatement).
* The reference's I2V prologue (``finetrainers/models/wan/base_specification.py:444-485``): the condition moments are
  normalised with the latents' statistics and replaced by their mode (the normalised mean), and the transformer input
  is ``cat([x_t, latent_condition_mask, latent_condition], dim=1)``.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import wan_oracle as O
from oracle.ltx_oracle import RMSNorm

IMAGE_NORM_EPS = 1e-5  # nn.LayerNorm's default: WanImageEmbedding builds FP32LayerNorm(in_features) / (out_features)
TEXT_LEN = 512         # WanAttnProcessor2_0: image_context_length = encoder_hidden_states.shape[1] - 512


class WanI2VOracleConfig(O.WanOracleConfig):
    def __init__(self, image_dim=1280, in_channels=36, **kw):
        super().__init__(in_channels=in_channels, **kw)
        self.image_dim = image_dim


class _GELUExact(nn.Module):
    def __init__(self, d_in, d_out):
        super().__init__()
        self.proj = nn.Linear(d_in, d_out)

    def forward(self, x):
        return F.gelu(self.proj(x))


class ImageEmbedding(nn.Module):
    def __init__(self, di, d):
        super().__init__()
        self.norm1 = O.FP32LayerNorm(di, IMAGE_NORM_EPS, elementwise_affine=True)
        self.ff = O.FeedForward(di, di)
        self.ff.net[0] = _GELUExact(di, di)
        self.ff.net[2] = nn.Linear(di, d)
        self.norm2 = O.FP32LayerNorm(d, IMAGE_NORM_EPS, elementwise_affine=True)

    def forward(self, x):
        return self.norm2(self.ff(self.norm1(x)))


class I2VAttention(O.Attention):
    def __init__(self, cfg: WanI2VOracleConfig):
        super().__init__(cfg)
        d = cfg.inner_dim
        self.add_k_proj, self.add_v_proj = nn.Linear(d, d), nn.Linear(d, d)
        self.norm_added_k = RMSNorm(d, cfg.eps, True)

    def forward(self, x, ctx=None, rotary_emb=None):
        n_img = ctx.shape[1] - TEXT_LEN
        img, txt = ctx[:, :n_img], ctx[:, n_img:]
        q, k, v = self.norm_q(self.to_q(x)), self.norm_k(self.to_k(txt)), self.to_v(txt)
        ki, vi = self.norm_added_k(self.add_k_proj(img)), self.add_v_proj(img)
        q, k, v, ki, vi = (t.unflatten(2, (self.heads, -1)).transpose(1, 2) for t in (q, k, v, ki, vi))
        o_img = F.scaled_dot_product_attention(q, ki, vi).transpose(1, 2).flatten(2, 3).type_as(q)
        o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).flatten(2, 3).type_as(q)
        return self.to_out[0](o + o_img)


class WanI2VTransformerOracle(O.WanTransformerOracle):
    def __init__(self, cfg: WanI2VOracleConfig):
        super().__init__(cfg)
        self.condition_embedder.image_embedder = ImageEmbedding(cfg.image_dim, cfg.inner_dim)
        for blk in self.blocks:
            blk.attn2 = I2VAttention(cfg)

    def forward(self, hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image):
        B, _, Fr, H, W = hidden_states.shape
        ppf, pph, ppw = Fr, H // 2, W // 2
        rotary = O.wan_rope(self.cfg.attention_head_dim, ppf, pph, ppw, self.cfg.rope_max_seq_len)
        h = self.patch_embedding(hidden_states).flatten(2).transpose(1, 2)
        temb, tproj, txt = self.condition_embedder(timestep, encoder_hidden_states)
        img = self.condition_embedder.image_embedder(encoder_hidden_states_image)
        ctx = torch.cat([img, txt], dim=1)
        tproj = tproj.unflatten(1, (6, -1))
        for blk in self.blocks:
            h = blk(h, ctx, tproj, rotary)
        shift, scale = (self.scale_shift_table + temb.unsqueeze(1)).chunk(2, dim=1)
        h = (self.norm_out(h.float()) * (1 + scale) + shift).type_as(h)
        h = self.proj_out(h)
        h = h.reshape(B, ppf, pph, ppw, 1, 2, 2, -1).permute(0, 7, 1, 4, 2, 5, 3, 6)
        return h.flatten(6, 7).flatten(4, 5).flatten(2, 3)


def i2v_prologue(moments, cond_moments, mask, latents_mean, latents_std, eps, noise, sigmas):
    """-> (hidden_states [B, 2C + Cm, F, H, W] = cat([x_t, mask, condition]), target [B, C, F, H, W]), in moments'
    dtype: the T2V prologue plus the condition's normalised mean (``DiagonalGaussianDistribution.mode()``)."""
    x_t, target = O.prologue(moments, latents_mean, latents_std, eps, noise, sigmas)
    C = x_t.shape[1]
    cond = O.normalize_latents(cond_moments[:, :C], latents_mean, latents_std)
    return torch.cat([x_t, mask.to(x_t.dtype), cond], dim=1), target


def oracle_step(model: WanI2VTransformerOracle, moments, cond_moments, mask, latents_mean, latents_std, eps, noise,
                sigmas, encoder_hidden_states, encoder_hidden_states_image, weights: Optional[torch.Tensor] = None):
    """fp32 forward + loss (mean over each sample, weighted, mean over the batch) + backward; -> (loss, pred)."""
    hidden, target = i2v_prologue(moments, cond_moments, mask, latents_mean, latents_std, eps, noise, sigmas)
    timesteps = (sigmas.flatten() * 1000.0).long()
    pred = model(hidden.float(), timesteps, encoder_hidden_states.float(), encoder_hidden_states_image.float())
    w = torch.ones(pred.shape[0]) if weights is None else weights
    loss = (w.view(-1, 1) * (pred.float() - target.float()).pow(2).flatten(1)).mean(1).mean()
    loss.backward()
    return loss.detach(), pred.detach()
