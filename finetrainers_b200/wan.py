"""Wan-2.1 text-to-video on the H100 engine: the ``torch.nn.Module`` finetrainers' ``WanModelSpecification.forward``
calls (``finetrainers/models/wan/base_specification.py:433-493``; diffusers ``WanTransformer3DModel``), trained by the
same block forward, hand-written backward, workspace plan, LoRA packing, checkpointing and CUDA graphs as LTX-Video
(``model.B200LTXTransformer``).  What differs is data (``model.ModelDesc``: LayerNorm block norms, an affine LayerNorm
before cross attention, per-head RoPE, the FFN width, the patch widths) plus the module tree and its FQNs, here.

* The Conv3d patch embedding (patch (1, 2, 2)) is a K = 64 GEMM on patchified tokens: the step prologue writes them in
  the Conv3d weight's order, so ``patch_embedding.weight`` [D, 16, 1, 2, 2] is used as [D, 64].  ``proj_out``'s output
  is unpatchified by one permute kernel (and its gradient patchified by the same kernel).
* Image-to-video (``image_dim``, ``WanConfig.wan_i2v_14b``): the 36-channel input cat([x_t, mask, condition]) is a
  K = 144 patch GEMM; the image embedder and every block's frozen image K/V (``attn2.add_k_proj`` / ``add_v_proj`` /
  ``norm_added_k``) run once per step, before the blocks; cross attention attends to the text and the image context in
  one two-context launch, and its backward takes dQ from both (no image K/V gradient: those weights are frozen).
* Layerwise fp8 storage (``enable_layerwise_casting``) follows diffusers' layer set, which includes the Conv3d patch
  embedding: the block linears, ``condition_embedder``'s linears and ``proj_out`` are cast unless a skip pattern
  matches, and the stacked text- and image-side K/V of all blocks stream through the block slots in chunks.  A pattern
  set that casts ``patch_embedding`` is refused (finetrainers' lists skip it with "patch_embed").
* Built: LoRA on to_q|to_k|to_v|to_out.0 of both attentions, keep-all / "full" / "block_skip" checkpointing, CUDA-graph
  steps, gradient accumulation, DDP, the no-grad inference plan and layerwise fp8 storage, for text-to-video and
  image-to-video.  Not built (``NotImplementedError``): the feed-forward LoRA set, LoRA on ``add_k_proj`` /
  ``add_v_proj``, fp8 storage of the patch embedding, FSDP-2, the first-last-frame variant (``pos_embed_seq_len``),
  full-rank backward.
"""
from __future__ import annotations

from dataclasses import dataclass, asdict
from typing import Dict, Optional, Tuple

import torch
import torch.nn as nn

from . import ops
from .model import B200LTXTransformer, ModelDesc, ParamLinear, _Attn, _FF, _GELUProj, _NormW, _StepFn, _base
from .specification import FlowMatchSchedulerTable


@dataclass
class WanConfig:
    """diffusers ``WanTransformer3DModel`` config of Wan-2.1 T2V 1.3B (restated from the published checkpoint config;
    DESIGN.md §2 lists such upstream facts as not vendored)."""
    patch_size: Tuple[int, int, int] = (1, 2, 2)
    num_attention_heads: int = 12
    attention_head_dim: int = 128
    in_channels: int = 16
    out_channels: int = 16
    text_dim: int = 4096
    freq_dim: int = 256
    ffn_dim: int = 8960
    num_layers: int = 30
    cross_attn_norm: bool = True
    qk_norm: Optional[str] = "rms_norm_across_heads"
    eps: float = 1e-6
    image_dim: Optional[int] = None
    added_kv_proj_dim: Optional[int] = None
    rope_max_seq_len: int = 1024
    pos_embed_seq_len: Optional[int] = None

    @property
    def inner_dim(self) -> int:
        return self.num_attention_heads * self.attention_head_dim

    def to_dict(self):
        return asdict(self)

    @classmethod
    def wan_14b(cls) -> "WanConfig":
        """Wan-2.1 T2V 14B: 40 heads x 128, FFN 13824, 40 blocks."""
        return cls(num_attention_heads=40, ffn_dim=13824, num_layers=40)

    @classmethod
    def wan_i2v_14b(cls) -> "WanConfig":
        """Wan-2.1 I2V 14B (``Wan-AI/Wan2.1-I2V-14B-480P-Diffusers``): the T2V-14B stack with a 36-channel input
        (x_t, mask, condition), a CLIP image context of width 1280 and image K/V projections from the embedded width."""
        return cls(num_attention_heads=40, ffn_dim=13824, num_layers=40, in_channels=36, out_channels=16,
                   image_dim=1280, added_kv_proj_dim=5120)


class _Conv3dParams(nn.Module):
    """Parameter container with nn.Conv3d's attribute names (weight [out, in, pt, ph, pw], bias [out])."""

    def __init__(self, cin, cout, patch, dtype, device):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, *patch, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.empty(cout, dtype=dtype, device=device))


class _AffineNorm(nn.Module):
    """FP32LayerNorm(elementwise_affine=True)'s parameters."""

    def __init__(self, d, dtype, device):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(d, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.zeros(d, dtype=dtype, device=device))


class _I2VAttn(_Attn):
    """Cross attention with diffusers' image-context projections (``added_kv_proj_dim``): add_k_proj, add_v_proj and the
    across-heads RMSNorm norm_added_k (Wan has no norm_added_q)."""

    def __init__(self, cfg: WanConfig, dtype, device):
        super().__init__(cfg, dtype, device)
        d = cfg.inner_dim
        self.add_k_proj = ParamLinear(cfg.added_kv_proj_dim, d, True, dtype, device)
        self.add_v_proj = ParamLinear(cfg.added_kv_proj_dim, d, True, dtype, device)
        self.norm_added_k = _NormW(d, dtype, device)


class _WanBlock(nn.Module):
    def __init__(self, cfg: WanConfig, dtype, device):
        super().__init__()
        d = cfg.inner_dim
        self.norm1 = nn.Identity()  # FP32LayerNorm without affine: no parameters
        self.attn1 = _Attn(cfg, dtype, device)
        self.norm2 = _AffineNorm(d, dtype, device)
        self.attn2 = (_I2VAttn if cfg.image_dim else _Attn)(cfg, dtype, device)
        self.ffn = _FF(d, cfg.ffn_dim, dtype, device)
        self.norm3 = nn.Identity()
        self.scale_shift_table = nn.Parameter(torch.empty(1, 6, d, dtype=dtype, device=device))


class _TwoLinear(nn.Module):
    def __init__(self, k, d, dtype, device):
        super().__init__()
        self.linear_1 = ParamLinear(k, d, True, dtype, device)
        self.linear_2 = ParamLinear(d, d, True, dtype, device)


class _ImageFF(nn.Module):
    """diffusers FeedForward(image_dim, d, mult=1, activation_fn="gelu"): net.0.proj, exact GELU, net.2."""

    def __init__(self, di, d, dtype, device):
        super().__init__()
        self.net = nn.ModuleList([_GELUProj(di, di, dtype, device), nn.Dropout(0.0), ParamLinear(di, d, True, dtype,
                                                                                                  device)])


class _ImageEmbedder(nn.Module):
    """diffusers WanImageEmbedding without pos_embed: FP32LayerNorm(image_dim), FeedForward, FP32LayerNorm(d)."""

    def __init__(self, di, d, dtype, device):
        super().__init__()
        self.norm1 = _AffineNorm(di, dtype, device)
        self.ff = _ImageFF(di, d, dtype, device)
        self.norm2 = _AffineNorm(d, dtype, device)


class _ConditionEmbedder(nn.Module):
    def __init__(self, d, freq_dim, text_dim, dtype, device, image_dim=None):
        super().__init__()
        self.time_embedder = _TwoLinear(freq_dim, d, dtype, device)
        self.time_proj = ParamLinear(d, 6 * d, True, dtype, device)
        self.text_embedder = _TwoLinear(text_dim, d, dtype, device)
        if image_dim:
            self.image_embedder = _ImageEmbedder(image_dim, d, dtype, device)


class _Unpatchify(torch.autograd.Function):
    """proj_out's patchified output [B, S', 4C] -> [B, C, F, H, W]; its gradient the other way (both exact permutes)."""

    @staticmethod
    def forward(ctx, pred, B, Cc, F, H, W):
        ctx.shape = (B, Cc, F, H, W)
        out = torch.empty(B, Cc, F, H, W, dtype=pred.dtype, device=pred.device)
        return ops.patch_permute(pred, out, B, Cc, F, H, W, ops.PATCH_OUT, True)

    @staticmethod
    def backward(ctx, dout):
        B, Cc, F, H, W = ctx.shape
        dp = torch.empty(B, F * (H // 2) * (W // 2), 4 * Cc, dtype=torch.bfloat16, device=dout.device)
        ops.patch_permute(dout.to(torch.bfloat16).contiguous(), dp, B, Cc, F, H, W, ops.PATCH_OUT, False)
        return dp, None, None, None, None, None


# diffusers' Wan attention splits the image context off the concatenated context at len - 512: the text encoder's length
WAN_TEXT_LEN = 512


class B200WanTransformer(B200LTXTransformer):
    """diffusers ``WanTransformer3DModel`` (T2V and I2V) FQNs and forward signature on the engine of
    ``B200LTXTransformer``."""

    def __init__(self, cfg: Optional[WanConfig] = None, dtype=torch.bfloat16, device="cuda"):
        nn.Module.__init__(self)
        cfg = cfg or WanConfig()
        if (cfg.image_dim is not None or cfg.added_kv_proj_dim is not None) and \
                (cfg.image_dim is None or cfg.added_kv_proj_dim != cfg.inner_dim):
            raise NotImplementedError(f"image_dim {cfg.image_dim} with added_kv_proj_dim {cfg.added_kv_proj_dim}: the "
                                      "image-to-video branch is built for both set, added_kv_proj_dim = inner_dim "
                                      f"({cfg.inner_dim}, the image embedder's output width)")
        if cfg.pos_embed_seq_len is not None:
            raise NotImplementedError("pos_embed_seq_len (first-last-frame-to-video, use_last_frame) is not built")
        if cfg.image_dim is not None and (cfg.image_dim <= 0 or cfg.image_dim % 8):
            raise ValueError(f"image_dim = {cfg.image_dim}: the image embedder's kernels need a positive multiple of 8")
        if tuple(cfg.patch_size) != (1, 2, 2):
            raise ValueError(f"patch_size {tuple(cfg.patch_size)}: the engine is built for Wan-2.1's (1, 2, 2)")
        if cfg.attention_head_dim not in (64, 128):
            raise ValueError(f"attention_head_dim = {cfg.attention_head_dim}: the attention and q/k-norm + RoPE kernels "
                             "are built for head dimensions 64 and 128")
        if cfg.qk_norm != "rms_norm_across_heads" or not cfg.cross_attn_norm or cfg.freq_dim != 256:
            raise ValueError("the engine is built for qk_norm='rms_norm_across_heads', cross_attn_norm=True, freq_dim=256")
        self.cfg = cfg
        self.config = cfg
        d, npatch = cfg.inner_dim, 4
        self.desc = ModelDesc(blocks="blocks", ff="ffn", in_features=cfg.in_channels * npatch,
                              out_features=cfg.out_channels * npatch, ffn_dim=cfg.ffn_dim, text_dim=cfg.text_dim,
                              norm_eps=cfg.eps, qk_eps=cfg.eps, layer_norm=True, cross_prenorm=True, rope_per_head=True,
                              lora_ffn=False, layerwise=True, fsdp=False, image_dim=cfg.image_dim or 0)
        self.patch_embedding = _Conv3dParams(cfg.in_channels, d, cfg.patch_size, dtype, device)
        self.condition_embedder = _ConditionEmbedder(d, cfg.freq_dim, cfg.text_dim, dtype, device, cfg.image_dim)
        self.blocks = nn.ModuleList([_WanBlock(cfg, dtype, device) for _ in range(cfg.num_layers)])
        self.norm_out = nn.Identity()
        self.proj_out = ParamLinear(d, cfg.out_channels * npatch, True, dtype, device)
        self.scale_shift_table = nn.Parameter(torch.empty(1, 2, d, dtype=dtype, device=device))
        self._init_engine_state(device)

    _CASTABLE = (ParamLinear, _Conv3dParams)  # diffusers' layerwise walk casts the Conv3d patch embedding too

    # the engine's names for the patch projection and the block list
    @property
    def proj_in(self):
        return self.patch_embedding

    @property
    def transformer_blocks(self):
        return self.blocks

    def _root_params(self):
        ce = self.condition_embedder
        kw, kb, kn = self._stacked_kv2()
        params = [("proj_in.w", [self.patch_embedding.weight]), ("proj_in.b", [self.patch_embedding.bias]),
                  ("t1.w", [ce.time_embedder.linear_1.weight]), ("t1.b", [ce.time_embedder.linear_1.bias]),
                  ("t2.w", [ce.time_embedder.linear_2.weight]), ("t2.b", [ce.time_embedder.linear_2.bias]),
                  ("ada.w", [ce.time_proj.weight]), ("ada.b", [ce.time_proj.bias]),
                  ("c1.w", [ce.text_embedder.linear_1.weight]), ("c1.b", [ce.text_embedder.linear_1.bias]),
                  ("c2.w", [ce.text_embedder.linear_2.weight]), ("c2.b", [ce.text_embedder.linear_2.bias]),
                  ("sst", [self.scale_shift_table]), ("proj_out.w", [self.proj_out.weight]),
                  ("proj_out.b", [self.proj_out.bias]), ("Wkv2_all", kw), ("bkv2_all", kb), ("nk2_all", kn)]
        if self.cfg.image_dim:
            ie = ce.image_embedder
            ff1, ff2 = ie.ff.net[0].proj, ie.ff.net[2]
            kw3, kb3, kn3 = [], [], []  # every block's image-side K/V, stacked as the text side's
            for blk in self.blocks:
                a2 = blk.attn2
                kw3 += [_base(a2.add_k_proj).weight, _base(a2.add_v_proj).weight]
                kb3 += [_base(a2.add_k_proj).bias, _base(a2.add_v_proj).bias]
                kn3.append(a2.norm_added_k.weight)
            params += [("img_n1.w", [ie.norm1.weight]), ("img_n1.b", [ie.norm1.bias]), ("img_ff1.w", [ff1.weight]),
                       ("img_ff1.b", [ff1.bias]), ("img_ff2.w", [ff2.weight]), ("img_ff2.b", [ff2.bias]),
                       ("img_n2.w", [ie.norm2.weight]), ("img_n2.b", [ie.norm2.bias]), ("Wkv3_all", kw3),
                       ("bkv3_all", kb3), ("nk3_all", kn3)]
        return params

    def _check_context(self, ehs, ehs_img):
        """Refuse an image context the model cannot take: one given to a text-to-video model (NotImplementedError);
        for image-to-video a missing one, one of another width or batch, or a text other than WAN_TEXT_LEN tokens, as
        diffusers' split of the concatenated context assumes (ValueError)."""
        di = self.cfg.image_dim
        if ehs_img is not None and not di:
            raise NotImplementedError("encoder_hidden_states_image given to a text-to-video model (no image_dim)")
        if not di:
            return
        if ehs_img is None:
            raise ValueError("an image-to-video model (image_dim) needs encoder_hidden_states_image")
        if ehs_img.ndim != 3 or ehs_img.shape[0] != ehs.shape[0] or ehs_img.shape[2] != di:
            raise ValueError(f"encoder_hidden_states_image must be [{ehs.shape[0]}, Li, {di}], not "
                             f"{tuple(ehs_img.shape)}")
        if ehs.shape[1] != WAN_TEXT_LEN:
            raise ValueError(f"image-to-video needs {WAN_TEXT_LEN} text tokens (diffusers splits the image context off "
                             f"at len - {WAN_TEXT_LEN}), not {ehs.shape[1]}")

    def _forward_impl(self, hidden_states, ehs, tvals, key_bias, Fr, Hh, Ww, rope_scale, ehs_img=None,
                      inference=False):
        self._check_context(ehs, ehs_img)
        return super()._forward_impl(hidden_states, ehs, tvals, key_bias, Fr, Hh, Ww, rope_scale, ehs_img, inference)

    def patchify(self, x: torch.Tensor) -> torch.Tensor:
        """[B, C, F, H, W] -> [B, F (H/2) (W/2), 4C] in the Conv3d weight's order (exact)."""
        B, Cc, F, H, W = x.shape
        out = torch.empty(B, F * (H // 2) * (W // 2), 4 * Cc, dtype=torch.bfloat16, device=x.device)
        return ops.patch_permute(x.to(torch.bfloat16).contiguous(), out, B, Cc, F, H, W, ops.PATCH_CONV, False)

    def forward(self, hidden_states, timestep, encoder_hidden_states, encoder_hidden_states_image=None,
                return_dict=False, attention_kwargs=None):
        """diffusers' signature: hidden_states [B, in_channels, F, H, W], timestep [B], encoder_hidden_states
        [B, L, text_dim], with image_dim also encoder_hidden_states_image [B, Li, image_dim] (L = 512)
        -> (prediction [B, out_channels, F, H, W],)."""
        self._check_context(encoder_hidden_states, encoder_hidden_states_image)
        if attention_kwargs:
            raise NotImplementedError(f"attention_kwargs {sorted(attention_kwargs)} are not supported")
        B, Cc, F, H, W = hidden_states.shape
        if Cc != self.cfg.in_channels or H % 2 or W % 2:
            raise ValueError(f"hidden_states must be [B, {self.cfg.in_channels}, F, H, W] with H and W even, not "
                             f"{tuple(hidden_states.shape)}")
        if timestep.numel() != B:
            raise ValueError(f"timestep has {timestep.numel()} elements: one per sample ({B}) expected")
        if not self._prepared:
            self.prepare()
        tvals = timestep.reshape(B).to(torch.float32).contiguous()
        args = (self.patchify(hidden_states), encoder_hidden_states, tvals, None, F, H // 2, W // 2, ())
        if self.cfg.image_dim:
            args += (encoder_hidden_states_image,)
        if not torch.is_grad_enabled():
            pred = self._forward_impl(*args, inference=True)
        else:
            pred = _StepFn.apply(self._anchor, self, *args)
        return (_Unpatchify.apply(pred, B, self.cfg.out_channels, F, H, W),)


def wan_moments_shape(shape, in_channels: int):
    """(B, C, F, H, W) of Wan's precomputed VAE moments [B, 2C, F, H, W]; ValueError unless dim 1 is 2 * in_channels and
    H, W are even (the (1, 2, 2) patch)."""
    if len(shape) != 5 or shape[1] != 2 * in_channels or shape[3] % 2 or shape[4] % 2:
        raise ValueError(f"Wan trains from VAE moments [B, 2 * {in_channels}, F, H, W] (mean | logvar) with H and W even, "
                         f"got shape {tuple(shape)}")
    B, C2, F, H, W = shape
    return B, C2 // 2, F, H, W


def _per_sample(v: torch.Tensor, B: int, C: int) -> torch.Tensor:
    """latents_mean / latents_std given as [C] (the VAE config's) or [B, C] -> fp32 [B, C]."""
    return v.to(torch.float32).reshape(-1, C).expand(B, C).contiguous()


class WanModelSpecification:
    """``WanModelSpecification`` hot-path mirror: the reference's ``forward`` arguments, dict mutation and return triple,
    with ``compute_posterior`` forced False as the reference forces it (the latents are always VAE moments).  The
    normalisation, posterior sample, noising, patching and target run as one libb2d launch (``b2d_wan_prep``)."""
    first_frame_conditioning_p = 0.0  # Wan has no first-frame conditioning
    latents_are_moments = True

    def __init__(self, transformer_config: Optional[WanConfig] = None, transformer_dtype=torch.bfloat16):
        self.transformer_config = transformer_config or WanConfig()
        self.transformer_dtype = transformer_dtype

    def load_diffusion_models(self, device="cuda") -> Dict[str, object]:
        """Random-init transformer; the reference's scheduler is ``FlowMatchEulerDiscreteScheduler()`` (shift 1)."""
        return {"transformer": B200WanTransformer(self.transformer_config, self.transformer_dtype, device),
                "scheduler": FlowMatchSchedulerTable()}

    def collate_conditions(self, data):
        from .data import collate
        return collate(data)

    def collate_latents(self, data):
        from .data import collate
        return collate(data)

    # -- the fused training step (trainer.SFTTrainStep) ---------------------------------------------------------------
    def packed_shape(self, C, Fr, Hh, Ww) -> Tuple[int, int]:
        """(tokens, channels) of the packed x_t / target / prediction of a [B, C, Fr, Hh, Ww] latent."""
        if Hh % 2 or Ww % 2:
            raise ValueError(f"Wan latents need even H and W (patch (1, 2, 2)), got {Hh} x {Ww}")
        return Fr * (Hh // 2) * (Ww // 2), 4 * C

    def image_inputs(self, latent_model_conditions, moments_shape, cfg: Optional[WanConfig] = None):
        """An image-to-video batch's (latent_condition [B, 2C, F, H, W], latent_condition_mask [B, Cm, F, H, W],
        encoder_hidden_states_image [B, Li, image_dim]) from ``latent_model_conditions``, shapes checked against the
        moments' and the transformer config ``cfg`` (default: the spec's) (ValueError), or None for a text-to-video
        model."""
        cfg = cfg or self.transformer_config
        if not cfg.image_dim:
            return None
        cond = latent_model_conditions.get("latent_condition")
        mask = latent_model_conditions.get("latent_condition_mask")
        img = latent_model_conditions.get("encoder_hidden_states_image")
        if cond is None or mask is None or img is None:
            raise ValueError("an image-to-video model (image_dim) trains with latent_condition, latent_condition_mask "
                             "and encoder_hidden_states_image")
        B, C2, Fr, Hh, Ww = moments_shape
        Cm = cfg.in_channels - C2
        if tuple(cond.shape) != tuple(moments_shape) or tuple(mask.shape) != (B, Cm, Fr, Hh, Ww) or Cm <= 0:
            raise ValueError(f"latent_condition {tuple(cond.shape)} must be the moments' {tuple(moments_shape)} and "
                             f"latent_condition_mask {tuple(mask.shape)} [B, in_channels - 2 C = {Cm}, F, H, W]")
        if img.ndim != 3 or img.shape[0] != B or img.shape[2] != cfg.image_dim:
            raise ValueError(f"encoder_hidden_states_image must be [{B}, Li, {cfg.image_dim}], not {tuple(img.shape)}")
        return cond, mask, img

    def step_inputs(self, key, st):
        """The prologue on the step's static buffers -> ``_forward_impl``'s arguments (capturable).  Image-to-video
        (``key[8:]`` = image tokens, image width, mask channels): x_t is written as the 36-channel input with the mask
        and the condition, and the image embeddings are the last argument."""
        B, C, Fr, Hh, Ww, L, Cc, from_moments = key[:8]
        if len(key) > 8:
            ops.wan_i2v_prep(st["moments"], st["cond"], st["cond_mask"], st["eps"], st["noise"], st["mean"], st["std"],
                             st["sig"], st["x_t"], st["target"], B, C, key[10], Fr, Hh, Ww)
        else:
            ops.wan_prep(st["moments"], st["eps"], st["noise"], st["mean"], st["std"], st["sig"], st["x_t"],
                         st["target"], B, C, Fr, Hh, Ww)
        tvals = (st["sig"] * 1000.0).long().to(torch.float32)  # base_specification.py:477
        return (st["x_t"], st["ehs"], tvals, None, Fr, Hh // 2, Ww // 2, ()) + ((st["img"],) if len(key) > 8 else ())

    # -- the reference's forward ----------------------------------------------------------------------------------------
    def forward(self, transformer: B200WanTransformer, condition_model_conditions: Dict[str, torch.Tensor],
                latent_model_conditions: Dict[str, torch.Tensor], sigmas: torch.Tensor,
                generator: Optional[torch.Generator] = None, compute_posterior: bool = True,
                noise: Optional[torch.Tensor] = None, posterior_noise: Optional[torch.Tensor] = None,
                **kwargs) -> Tuple[torch.Tensor, ...]:
        """``latents`` are VAE moments [B, 32, F, H, W]; eps is drawn from ``generator`` before the noise (or taken from
        ``posterior_noise``), as ``posterior.sample(generator)`` runs before ``normal_(generator)``.  Image-to-video:
        ``latent_condition`` (the condition's moments, of which the normalised mean is used) and
        ``latent_condition_mask`` are popped and written with x_t into the 36-channel ``hidden_states``;
        ``encoder_hidden_states_image`` passes through to the transformer.  Returns (pred, target, sigmas), pred and
        target [B, 16, F, H, W]."""
        compute_posterior = False  # noqa: F841  (the reference forces it: the latents are normalised before sampling)
        latents = latent_model_conditions.pop("latents")
        latents_mean = latent_model_conditions.pop("latents_mean")
        latents_std = latent_model_conditions.pop("latents_std")
        image = self.image_inputs(latent_model_conditions, latents.shape, transformer.cfg)
        cond = latent_model_conditions.pop("latent_condition", None)
        cond_mask = latent_model_conditions.pop("latent_condition_mask", None)
        if image is None and (cond is not None or cond_mask is not None):
            raise NotImplementedError("latent_condition given for a text-to-video model (no image_dim)")
        B, C, Fr, Hh, Ww = wan_moments_shape(latents.shape, transformer.cfg.out_channels)
        dev = latents.device
        moments = latents.to(torch.bfloat16).contiguous()
        if posterior_noise is None:
            eps = torch.randn((B, C, Fr, Hh, Ww), generator=generator, device=dev, dtype=torch.bfloat16)
        else:
            eps = posterior_noise.to(torch.bfloat16).contiguous()
        if noise is None:
            noise = torch.zeros((B, C, Fr, Hh, Ww), dtype=torch.bfloat16, device=dev).normal_(generator=generator)
        else:
            noise = noise.to(torch.bfloat16).contiguous()
        S, Cp = self.packed_shape(C, Fr, Hh, Ww)
        Cin = transformer.cfg.in_channels
        x_in = torch.empty(B, S, 4 * Cin, dtype=torch.bfloat16, device=dev)
        target = torch.empty(B, S, Cp, dtype=torch.bfloat16, device=dev)
        sig = sigmas.reshape(B).to(torch.float32).contiguous()
        mean, std = _per_sample(latents_mean, B, C).to(dev), _per_sample(latents_std, B, C).to(dev)
        if image is None:
            ops.wan_prep(moments, eps, noise, mean, std, sig, x_in, target, B, C, Fr, Hh, Ww)
        else:  # the reference's mask is a transposed view: the kernel reads dense arrays
            ops.wan_i2v_prep(moments, cond.to(torch.bfloat16).contiguous(), cond_mask.to(torch.bfloat16).contiguous(),
                             eps, noise, mean, std, sig, x_in, target, B, C, Cin - 2 * C, Fr, Hh, Ww)
        timesteps = (sig * 1000.0).long()
        x5 = torch.empty(B, Cin, Fr, Hh, Ww, dtype=torch.bfloat16, device=dev)
        latent_model_conditions["hidden_states"] = ops.patch_permute(x_in, x5, B, Cin, Fr, Hh, Ww, ops.PATCH_CONV, True)
        pred = transformer(**latent_model_conditions, **condition_model_conditions, timestep=timesteps,
                           return_dict=False)[0]
        target5 = torch.empty(B, C, Fr, Hh, Ww, dtype=torch.bfloat16, device=dev)
        ops.patch_permute(target, target5, B, C, Fr, Hh, Ww, ops.PATCH_OUT, True)
        return pred, target5, sigmas
