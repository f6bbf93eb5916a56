"""H100-native LTX-Video DiT: the ``torch.nn.Module`` finetrainers' ``LTXVideoModelSpecification.forward`` calls
(``finetrainers/models/ltx_video/base_specification.py:336-342``), re-implemented as one autograd node
whose forward AND backward are sequences of libb2d kernels (wgmma GEMMs with fused epilogues, fused norm/modulate,
q/k-norm + RoPE, wgmma attention) instead of the diffusers module graph
(``finetrainers/patches/models/ltx_video/patch.py:38-127`` + diffusers ``LTXVideoTransformerBlock``).

* Parameter FQNs are diffusers/peft compatible (``transformer_blocks.0.attn1.to_q.lora_A.default.weight`` ...), so
  ``state_dict`` / LoRA export (``base_specification.py:379-397``) keep working.  The parameters are views into packed
  device buffers (``[Wq;Wk;Wv]``, flat fp32 LoRA master / grad buffers) so the kernels see fused operands with no copies.
* By default all block activations needed by backward are kept resident (≈5.5 GB at 49x512x768, B=1, 2B model).
  ``apply_activation_checkpointing`` (the reference's ``utils/activation_checkpoint.py:24-49``) selects blocks whose
  activations are recomputed before their backward instead, keeping the block input and both attention outputs.
* The timestep embedding is evaluated on the B distinct timesteps, not on B*S rows (``patch.py:67-79`` flattens B*S);
  per-token timesteps that differ between latent frames (image-to-video: 0 on the conditioning frame) are embedded
  once per frame, on B*F rows (``timestep_values``).
* LoRA (peft semantics: ``y = Wx + b + (alpha/r) B A x``) runs in the same wgmma accumulator as the base GEMM
  (K-extension operands); master weights and gradients are fp32 (``trainer.py:130-136``), GEMM operands bf16.
* There is no fallback: without libb2d.so / an sm_90 device every call raises.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, asdict
from types import SimpleNamespace
from typing import Dict, List, NamedTuple, Optional, Tuple

import torch
import torch.nn as nn

from . import ops
from .layerwise import (DEFAULT_SKIP_MODULES_PATTERN, STORAGE_DTYPES as _STORAGE_DTYPES, LayerwiseSchedule,
                        carve, carved_numel, cast_linear_names, numel16)

LORA_TARGETS = ("to_q", "to_k", "to_v", "to_out.0")  # examples/training/sft/ltx_video/crush_smol_lora/train.sh:77
# the attention set plus both feed-forward linears: the control trainer's default (control_trainer/config.py:45,60)
LORA_FFN_TARGETS = LORA_TARGETS + ("ff.net.0.proj", "ff.net.2")
# the image embedder's two LayerNorms: diffusers WanImageEmbedding builds FP32LayerNorm(dim) with nn.LayerNorm's default
# eps (restated from the published transformer_wan.py; tests/_wan_i2v_oracle.py records the provenance)
IMAGE_NORM_EPS = 1e-5


@dataclass
class LTXConfig:
    """``tests/models/ltx_video/_test_tp.py:29-59`` (real size)."""
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
    qk_norm_eps: float = 1e-5
    ffn_mult: int = 4

    @property
    def inner_dim(self) -> int:
        return self.num_attention_heads * self.attention_head_dim

    def to_dict(self):
        return asdict(self)

    @classmethod
    def ltx_13b(cls) -> "LTXConfig":
        """The 13B LTX-Video transformer: 32 heads x 128, width 4096, 48 blocks; everything else as the default (2B)
        geometry.  Restated from the published diffusers config of the checkpoint (DESIGN.md §2 lists it among the
        upstream facts that are not vendored)."""
        return cls(num_attention_heads=32, attention_head_dim=128, cross_attention_dim=4096, num_layers=48,
                   caption_channels=4096)


@dataclass(frozen=True)
class ModelDesc:
    """What the engine needs to know about a model family beyond its width, heads and depth: the module names it packs,
    the operand widths outside the blocks, the block's norm kinds and epsilons, and which engine features it supports.
    ``_forward_impl``, ``_block_forward``, the backward, ``workspace_plan``, ``_lora_groups`` and ``prepare`` read it;
    the module tree and the root FQN map are the model class's."""
    blocks: str           # attribute of the ModuleList of DiT blocks (FQN prefix)
    ff: str               # attribute of a block's feed-forward module
    in_features: int      # proj_in's K: latent channels x patch volume
    out_features: int     # proj_out's N
    ffn_dim: int
    text_dim: int         # caption / text embedding width
    norm_eps: float       # block norms and the head's norm
    qk_eps: float         # q/k RMSNorm across heads
    layer_norm: bool      # norm1 / the FFN's norm: LayerNorm (no affine) rather than RMSNorm
    cross_prenorm: bool   # affine LayerNorm before cross attention's q projection (weight "n2w", bias "n2b")
    rope_per_head: bool   # RoPE table [S, head_dim / 2] applied per head, else [S, D / 2] over the full width
    lora_ffn: bool        # the feed-forward LoRA target set is fused
    layerwise: bool       # layerwise fp8 base-weight storage is built
    fsdp: bool            # FSDP-2 sharding is built
    # width of an image context that every block's cross attention attends to beside the text (Wan image-to-video:
    # the image embedder's input, root pieces "img_*", stacked frozen K/V "Wkv3_all"); 0: text only
    image_dim: int = 0


class ParamLinear(nn.Module):
    """Parameter container with nn.Linear's attribute names; the math happens in libb2d."""

    def __init__(self, in_features, out_features, bias=True, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty(out_features, in_features, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.empty(out_features, dtype=dtype, device=device)) if bias else None

    def forward(self, *a, **k):
        raise RuntimeError("ParamLinear holds parameters only; the b200 engine executes the fused step")


class LoraLinear(nn.Module):
    """peft-compatible naming: base_layer / lora_A.default / lora_B.default (fp32 adapters)."""

    def __init__(self, base: ParamLinear, r: int, alpha: float):
        super().__init__()
        dev = base.weight.device
        self.base_layer = base
        self.lora_A = nn.ModuleDict({"default": ParamLinear(base.in_features, r, False, torch.float32, dev)})
        self.lora_B = nn.ModuleDict({"default": ParamLinear(r, base.out_features, False, torch.float32, dev)})
        self.r, self.lora_alpha, self.scaling = r, alpha, alpha / r
        bound = 1.0 / math.sqrt(base.in_features)  # kaiming_uniform_(a=sqrt(5)) == U(-1/sqrt(fan_in), +)
        with torch.no_grad():
            self.lora_A["default"].weight.uniform_(-bound, bound)
            self.lora_B["default"].weight.zero_()


class _NormW(nn.Module):
    def __init__(self, dim, dtype, device):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim, dtype=dtype, device=device))


class _Attn(nn.Module):
    def __init__(self, cfg: LTXConfig, dtype, device):
        super().__init__()
        d = cfg.inner_dim
        self.norm_q = _NormW(d, dtype, device)
        self.norm_k = _NormW(d, dtype, device)
        self.to_q = ParamLinear(d, d, True, dtype, device)
        self.to_k = ParamLinear(d, d, True, dtype, device)
        self.to_v = ParamLinear(d, d, True, dtype, device)
        self.to_out = nn.ModuleList([ParamLinear(d, d, True, dtype, device), nn.Dropout(0.0)])


class _GELUProj(nn.Module):
    def __init__(self, d_in, d_out, dtype, device):
        super().__init__()
        self.proj = ParamLinear(d_in, d_out, True, dtype, device)


class _FF(nn.Module):
    def __init__(self, d, inner, dtype, device):
        super().__init__()
        self.net = nn.ModuleList([_GELUProj(d, inner, dtype, device), nn.Dropout(0.0),
                                  ParamLinear(inner, d, True, dtype, device)])


class _Block(nn.Module):
    def __init__(self, cfg: LTXConfig, dtype, device):
        super().__init__()
        d = cfg.inner_dim
        self.norm1 = nn.Identity()
        self.attn1 = _Attn(cfg, dtype, device)
        self.norm2 = nn.Identity()
        self.attn2 = _Attn(cfg, dtype, device)
        self.ff = _FF(d, cfg.ffn_mult * d, dtype, device)
        self.scale_shift_table = nn.Parameter(torch.empty(6, d, dtype=dtype, device=device))


class _TimestepEmbedder(nn.Module):
    def __init__(self, d, dtype, device):
        super().__init__()
        self.linear_1 = ParamLinear(256, d, True, dtype, device)
        self.linear_2 = ParamLinear(d, d, True, dtype, device)


class _Emb(nn.Module):
    def __init__(self, d, dtype, device):
        super().__init__()
        self.timestep_embedder = _TimestepEmbedder(d, dtype, device)


class _AdaSingle(nn.Module):
    def __init__(self, d, dtype, device):
        super().__init__()
        self.emb = _Emb(d, dtype, device)
        self.linear = ParamLinear(d, 6 * d, True, dtype, device)


class _TextProj(nn.Module):
    def __init__(self, c, d, dtype, device):
        super().__init__()
        self.linear_1 = ParamLinear(c, d, True, dtype, device)
        self.linear_2 = ParamLinear(d, d, True, dtype, device)


def _base(m):
    return m.base_layer if isinstance(m, LoraLinear) else m


def checkpointed_blocks(num_layers: int, checkpointing_type: str = "full", n_layer: int = 1) -> Tuple[int, ...]:
    """Indices of the blocks a checkpointing policy recomputes: every block for "full"; block i iff i % n_layer == 0 for
    "block_skip" (the reference's ``_apply_activation_checkpointing_blocks``)."""
    if checkpointing_type == "full":
        return tuple(range(num_layers))
    if checkpointing_type == "block_skip":
        if int(n_layer) < 1:
            raise ValueError(f"block_skip needs n_layer >= 1, not {n_layer}")
        return tuple(i for i in range(num_layers) if i % int(n_layer) == 0)
    if checkpointing_type == "ops":
        raise NotImplementedError("checkpointing_type 'ops' (selective recompute of single ops) is not built; "
                                  "use 'full' or 'block_skip'")
    raise ValueError(f"checkpointing type {checkpointing_type!r} not supported: 'full', 'block_skip' or 'ops'")


def timestep_values(timestep: torch.Tensor, B: int, F: int, HW: int) -> torch.Tensor:
    """The fp32 timesteps the forward embeds: ``[B]`` (one per sample) or ``[B * F]`` (one per latent frame, frame-major
    tokens at patch size 1), from the timestep the forward was given.
    * ``B`` elements, any shape: one per sample.
    * ``B * F * HW`` elements (finetrainers' per-token ``[B, S, 1]``, the image-to-video pipeline's ``[B, S]``): viewed
      as ``[B, F, HW]``.  Outside CUDA-graph capture the values are compared on the device, bit for bit, and two flags
      are read back: a frame holding more than one value raises ``ValueError`` naming the first such sample and frame;
      if every sample holds one value, it is ``[B]`` (the per-sample plan, so the training input keeps its launches);
      else ``[B * F]``.  Under capture nothing can be read back, so it is ``[B * F]`` unchecked: a timestep that varies
      within a frame then embeds each frame's first token's value.
    * Any other element count raises ``ValueError``."""
    n = timestep.numel()
    if n == B:
        return timestep.reshape(B).to(torch.float32).contiguous()
    if n != B * F * HW:
        raise ValueError(f"timestep has {n} elements: one per sample ({B}) or one per latent token ({B} x {F * HW}) "
                         f"expected, shape {tuple(timestep.shape)}")
    t = timestep.reshape(B, F, HW).to(torch.float32)
    per_frame = t[:, :, 0].reshape(B * F).contiguous()
    if timestep.is_cuda and torch.cuda.is_current_stream_capturing():
        return per_frame
    bits = t.view(torch.int32)  # exact: NaN codes compare equal, -0 and +0 do not
    within = (bits != bits[:, :, :1]).any(-1)                   # [B, F]
    across = (bits[:, :, 0] != bits[:, :1, 0]).any(-1)          # [B]
    flags = torch.stack([within.any(), across.any()]).tolist()  # the one read-back
    if flags[0]:
        b, f = (int(i) for i in within.nonzero()[0])
        raise ValueError(f"timestep varies within latent frame {f} of sample {b}: the engine takes one timestep per "
                         "latent frame")
    return t[:, 0, 0].contiguous() if not flags[1] else per_frame


class _LoraGroup(NamedTuple):
    """Adapters of a block that share their input x and their launches: A [n rp, k_in] then B [n n_out, rp] in the flat
    buffers for n = len(mods), and the workspace tensors x, dy, u = s x A^T and du = s dy B."""
    name: str
    mods: Tuple[str, ...]  # paths of the adapted linears in the block, in packing order
    k_in: int
    n_out: int
    x: str                 # workspace tensor of the adapters' input
    dy: str                # workspace tensor of their output gradient
    x_at: str = "slot"     # x kept per "block", per "slot" or "shared" by all blocks
    text: bool = False     # rows: the B*L text tokens with dy / u / du kept per block, not the B*S latent tokens in slots

    @property
    def u(self) -> str:
        return "u_" + self.name

    @property
    def du(self) -> str:
        return "du_" + self.name


# the residency schedule of a model whose base weights all stay resident: the hooks of fsdp.FSDPState and
# layerwise.LayerwiseSchedule, doing nothing
_ALL_RESIDENT = SimpleNamespace(**dict.fromkeys(
    ("begin_forward", "pre_block_forward", "post_block_forward", "begin_backward_range", "pre_block_backward",
     "post_block_backward", "end_backward"), lambda *args: None))


class _StepFn(torch.autograd.Function):
    """One autograd node for the whole 28-block stack (forward and hand-written backward)."""

    @staticmethod
    def forward(ctx, anchor, model, *args):
        """``args``: ``_forward_impl``'s positional arguments (the image context last when the model has one)."""
        ctx.model = model
        ctx.nargs = len(args)
        out = model._forward_impl(*args)
        ctx.gen = model._fwd_gen
        return out

    @staticmethod
    def backward(ctx, dpred):
        if ctx.gen != ctx.model._fwd_gen:
            raise RuntimeError("B200LTXTransformer keeps ONE set of saved activations: another forward ran between this "
                               "forward and its backward (validation pass, second micro-batch, ...); call backward first")
        ctx.model._backward_impl(dpred)
        return (None,) * (2 + ctx.nargs)


class B200LTXTransformer(nn.Module):
    def __init__(self, cfg: Optional[LTXConfig] = None, dtype=torch.bfloat16, device="cuda"):
        super().__init__()
        cfg = cfg or LTXConfig()
        if cfg.attention_head_dim not in (64, 128):
            raise ValueError(f"attention_head_dim = {cfg.attention_head_dim}: the attention and q/k-norm + RoPE kernels "
                             "are built for head dimensions 64 and 128")
        if cfg.patch_size != 1 or cfg.patch_size_t != 1:
            raise ValueError("LTX-Video uses patch_size = patch_size_t = 1")
        if cfg.cross_attention_dim != cfg.inner_dim:
            raise ValueError("cross_attention_dim must equal inner_dim (LTX-Video)")
        self.cfg = cfg
        self.config = cfg  # diffusers-style attribute
        d = cfg.inner_dim
        self.desc = ModelDesc(blocks="transformer_blocks", ff="ff", in_features=cfg.in_channels,
                              out_features=cfg.out_channels, ffn_dim=cfg.ffn_mult * d, text_dim=cfg.caption_channels,
                              norm_eps=cfg.norm_eps, qk_eps=cfg.qk_norm_eps, layer_norm=False, cross_prenorm=False,
                              rope_per_head=False, lora_ffn=True, layerwise=True, fsdp=True)
        self.proj_in = ParamLinear(cfg.in_channels, d, True, dtype, device)
        self.scale_shift_table = nn.Parameter(torch.empty(2, d, dtype=dtype, device=device))
        self.time_embed = _AdaSingle(d, dtype, device)
        self.caption_projection = _TextProj(cfg.caption_channels, d, dtype, device)
        self.transformer_blocks = nn.ModuleList([_Block(cfg, dtype, device) for _ in range(cfg.num_layers)])
        self.norm_out = nn.Identity()
        self.proj_out = ParamLinear(d, cfg.out_channels, True, dtype, device)
        self._init_engine_state(device)

    def _init_engine_state(self, device):
        self._ckpt: Tuple[int, ...] = ()  # blocks recomputed before their backward (set_activation_checkpointing)
        self.lora_rank = 0
        self.lora_scaling = 1.0
        self.lora_ffn = False  # adapters on ff.net.0.proj and ff.net.2 as well as on the attention projections
        self._prepared = False
        self._ws: Dict[Tuple, Dict[str, torch.Tensor]] = {}  # (B, S, L) -> views of that shape's workspace in the arena
        self._arena: Optional[torch.Tensor] = None  # the training arena (bytes): every training shape's workspace
        self.workspace_generation = 0  # bumped on every arena allocation: CUDA graphs of an older one must be dropped
        self._iws: Optional[Tuple[Tuple, Dict[str, torch.Tensor]]] = None  # ((B, S, L), the one inference workspace)
        self._tws: Dict[int, Dict[str, torch.Tensor]] = {}  # G -> timestep-embedding buffers of G per-frame timesteps
        self._rope: Dict[Tuple, Tuple[torch.Tensor, torch.Tensor]] = {}
        self._anchor = torch.zeros((), dtype=torch.float32, device=device, requires_grad=True)
        self._saved_key = None
        self._fsdp = None  # fsdp.FSDPState once apply_fsdp2 ran
        self._lw_cfg = None  # layerwise fp8 storage settings once enable_layerwise_casting ran
        self._lw = None      # layerwise.LayerwiseSchedule of the prepared layout (None when nothing is cast)
        self._fwd_gen = 0
        self.skip_block0_dx = True

    # ------------------------------------------------------------------------------------------------
    # adapters / packing
    # ------------------------------------------------------------------------------------------------
    def _resolve_lora_targets(self, target_modules) -> List[str]:
        """peft's matching rule (``peft.tuners.tuners_utils.check_target_module_exists``): a ``str`` is a regex that must
        FULL-match the module name, a list matches by exact name or ``.``-suffix.  Returns the matched linear FQNs."""
        import re
        names = [n for n, m in self.named_modules() if isinstance(m, ParamLinear) and ".lora_" not in n]
        names = [n[:-len(".base_layer")] if n.endswith(".base_layer") else n for n in names]
        if isinstance(target_modules, str):
            return [n for n in names if re.fullmatch(target_modules, n)]
        tm = list(target_modules)
        return [n for n in names if any(n == t or n.endswith("." + t) for t in tm)]

    def add_adapter(self, adapter_config=None, lora_alpha: Optional[float] = None, target_modules=None,
                    adapter_name: str = "default"):
        """``transformer.add_adapter(LoraConfig(r=, lora_alpha=, init_lora_weights=True, target_modules=))`` exactly as
        ``SFTTrainer._prepare_trainable_parameters`` calls it (trainer.py:120-128): the first positional argument is a
        peft-style config object (anything with ``.r``, ``.lora_alpha``, ``.target_modules`` and optionally
        ``.init_lora_weights``).  ``add_adapter(64, 64)`` (rank, alpha) is kept as a shorthand.  ``target_modules`` follows
        peft's matching rule and must select exactly one of the two sets the engine fuses, in every block:
        to_q|to_k|to_v|to_out.0 of attn1 + attn2 (the SFT default regex, config.py:26; the default here), or those plus
        ff.net.0.proj and ff.net.2 (the control trainer's default, control_trainer/config.py:45,60)."""
        init = True
        if adapter_config is None:
            rank = 64
        elif hasattr(adapter_config, "r"):
            rank = int(adapter_config.r)
            if lora_alpha is None:
                lora_alpha = getattr(adapter_config, "lora_alpha", None)
            if target_modules is None:
                target_modules = getattr(adapter_config, "target_modules", None)
            init = getattr(adapter_config, "init_lora_weights", True)
            if getattr(adapter_config, "lora_dropout", 0.0):
                raise NotImplementedError("lora_dropout > 0 is not supported (the reference never sets it)")
        else:
            rank = int(adapter_config)
        if adapter_name != "default":
            raise NotImplementedError("only the 'default' adapter name is supported")
        if self.lora_rank:
            raise ValueError("an adapter is already attached")
        if rank <= 0:
            raise ValueError("LoRA rank must be positive")
        if init not in (True, "gaussian"):
            raise NotImplementedError(f"init_lora_weights={init!r}: only True (kaiming-uniform A, zero B) and 'gaussian'")
        if target_modules is None:
            target_modules = LORA_TARGETS
        if isinstance(target_modules, (set, frozenset)):
            target_modules = sorted(target_modules)
        nb, pre, ff = len(self.transformer_blocks), self.desc.blocks, self.desc.ff
        attn_set = sorted(f"{pre}.{i}.{a}.{t}" for i in range(nb) for a in ("attn1", "attn2") for t in LORA_TARGETS)
        ffn_set = sorted(attn_set + [f"{pre}.{i}.{ff}.{t}" for i in range(nb) for t in ("net.0.proj", "net.2")])
        got = sorted(self._resolve_lora_targets(target_modules))
        if got == ffn_set and not self.desc.lora_ffn:
            raise NotImplementedError(f"{type(self).__name__}: LoRA on the feed-forward projections is not built; target "
                                      "to_q|to_k|to_v|to_out.0 of attn1 and attn2")
        if got not in (attn_set, ffn_set):
            want = ffn_set if any(".ff." in n for n in got) else attn_set
            extra = [n for n in got if n not in want][:4]
            missing = [n for n in want if n not in got][:4]
            raise NotImplementedError("b200 engine fuses LoRA on exactly one of two target sets in every block: "
                                      "to_q|to_k|to_v|to_out.0 of attn1+attn2, or those plus ff.net.0.proj and ff.net.2; "
                                      f"target_modules selects a different set (extra: {extra}, missing: {missing})")
        ffn = got == ffn_set
        alpha = float(lora_alpha if lora_alpha is not None else rank)
        for p in self.parameters():
            p.requires_grad_(False)
        self.lora_ffn = ffn
        for blk in self.transformer_blocks:
            for g in self._lora_groups().values():
                for path in g.mods:
                    parent, _, name = path.rpartition(".")
                    setattr(blk.get_submodule(parent), name, LoraLinear(blk.get_submodule(path), rank, alpha))
        if init == "gaussian":  # peft: A ~ N(0, 1/r), B = 0
            with torch.no_grad():
                for n, p in self.named_parameters():
                    if "lora_A" in n:
                        p.normal_(0.0, 1.0 / rank)
        self.lora_rank = rank
        self.lora_scaling = alpha / rank
        # kept as given for the saved config: rank * scaling does not always round back to alpha (7 * (29 / 7) != 29)
        self.lora_alpha = int(alpha) if alpha.is_integer() else alpha
        self.peft_config = {adapter_name: adapter_config if hasattr(adapter_config, "r") else None}
        self._lora_init = init
        self._lora_targets = target_modules
        self._prepared = False

    def enable_layerwise_casting(self, storage_dtype: torch.dtype = torch.float8_e4m3fn,
                                 compute_dtype: torch.dtype = torch.bfloat16,
                                 skip_modules_pattern=DEFAULT_SKIP_MODULES_PATTERN, skip_modules_classes=None,
                                 non_blocking: bool = False):
        """Store the frozen base weights of every linear layer the skip patterns leave in fp8, compute with them upcast to
        bf16 (``--layerwise_upcasting_modules transformer``, trainer.py:108-118).  The cast parameters become fp8 (the
        reference's stored state); norm weights and scale_shift_table are never cast.  Must run before ``add_adapter``
        so that the adapters stay fp32.  A pattern set that casts some but not all linear layers packed into one fused
        weight (q/k/v of self-attention; the text-side k/v of all blocks) raises NotImplementedError."""
        if storage_dtype not in _STORAGE_DTYPES:
            raise ValueError(f"layerwise casting stores float8_e4m3fn or float8_e5m2, not {storage_dtype}")
        if compute_dtype != torch.bfloat16:
            raise NotImplementedError(f"layerwise casting computes in bf16 (the engine's only GEMM operand type), "
                                      f"not {compute_dtype}")
        if skip_modules_classes is not None:
            raise NotImplementedError("skip_modules_classes is not supported; select the skipped modules by pattern")
        if skip_modules_pattern is None or isinstance(skip_modules_pattern, str) and skip_modules_pattern == "auto":
            raise NotImplementedError("give the skip patterns explicitly (finetrainers passes its "
                                      "--layerwise_upcasting_skip_modules_pattern list)")
        if self.lora_rank:
            raise ValueError("enable layerwise casting before add_adapter: the adapters must not be cast")
        if self._lw_cfg is not None:
            raise ValueError("layerwise casting is already enabled")
        if self._fsdp is not None:
            raise NotImplementedError("layerwise fp8 storage under FSDP-2 is not built; use DDP")
        if not self.desc.layerwise:
            raise NotImplementedError(f"layerwise fp8 storage is not built for {type(self).__name__}")
        patterns = (skip_modules_pattern,) if isinstance(skip_modules_pattern, str) else tuple(skip_modules_pattern)
        cast = cast_linear_names(self, patterns, ParamLinear)
        self._layerwise_plan(set(cast))  # refuses a split fused weight before anything changes
        mods = dict(self.named_modules())
        with torch.no_grad():
            for n in cast:
                for p in (mods[n].weight, mods[n].bias):
                    if p is not None:
                        p.data = p.data.to(storage_dtype)  # torch's own rounding, as module.to(storage_dtype)
        self._lw_cfg = {"storage_dtype": storage_dtype, "patterns": patterns, "cast": cast}
        self._prepared = False
        return self

    # ---- activation checkpointing -------------------------------------------------------------------------------------
    @property
    def gradient_checkpointing(self) -> bool:
        return bool(self._ckpt)

    def enable_gradient_checkpointing(self):
        """diffusers' name for checkpointing every block (``apply_activation_checkpointing(self, "full")``)."""
        self.set_activation_checkpointing(checkpointed_blocks(len(self.transformer_blocks), "full"))

    def disable_gradient_checkpointing(self):
        self.set_activation_checkpointing(())

    def set_activation_checkpointing(self, blocks):
        """Recompute the activations of the given blocks before their backward instead of keeping them.  Set before the
        first forward: the workspaces are sized by it, and captured CUDA graphs hold pointers into them."""
        nl = len(self.transformer_blocks)
        blocks = tuple(sorted(set(int(b) for b in blocks)))
        if blocks and not 0 <= blocks[0] <= blocks[-1] < nl:
            raise ValueError(f"checkpointed blocks {blocks} outside 0 .. {nl - 1}")
        if blocks != self._ckpt and self._ws:
            raise ValueError("the activation checkpointing policy must be set before the first forward: a workspace "
                             "sized by the current policy exists (and CUDA graphs may hold pointers into it)")
        self._ckpt = blocks
        return self

    def _block_slots(self, ckpt=None):
        """-> (slot of each block, slot count) in the per-block workspace tensors a checkpointed block recomputes: the
        blocks that keep their activations own one slot each, in block order, and all checkpointed blocks share one
        scratch slot after them.  With nothing checkpointed block l owns slot l."""
        ck = set(self._ckpt if ckpt is None else ckpt)
        slots, n = [], 0
        for l in range(self.cfg.num_layers):
            slots.append(None if l in ck else n)
            n += l not in ck
        return [n if s is None else s for s in slots], n + bool(ck)

    def _kept_runs(self, lo, hi):
        """Maximal runs (first block, count) of consecutive blocks in [lo, hi) that keep their activations: their slots
        are consecutive too, so each run is one block-batched launch."""
        runs = []
        for l in range(lo, hi):
            if l in self._ckpt:
                continue
            if runs and runs[-1][0] + runs[-1][1] == l:
                runs[-1] = (runs[-1][0], runs[-1][1] + 1)
            else:
                runs.append((l, 1))
        return runs

    def _layerwise_plan(self, cast):
        """-> ([cast spec keys of each block], [cast spec keys of the root unit]) for the set of cast linear FQNs.  A fused
        piece is cast iff all the linear layers packed into it are."""
        owner = {}
        for n, m in self.named_modules():
            if isinstance(m, ParamLinear) and ".lora_" not in n:
                n = n[:-len(".base_layer")] if n.endswith(".base_layer") else n
                for p in (m.weight, m.bias):
                    if p is not None:
                        owner[id(p)] = n

        def decide(key, params):
            members = sorted({owner[id(p)] for p in params if id(p) in owner})
            yes = [m for m in members if m in cast]
            if yes and len(yes) != len(members):
                no = [m for m in members if m not in cast]
                raise NotImplementedError(
                    f"layerwise casting: the skip patterns cast {yes[:3]}{' ...' if len(yes) > 3 else ''} but not "
                    f"{no[:3]}{' ...' if len(no) > 3 else ''}, which share the fused weight '{key}'")
            return bool(yes)

        blk = [[k for k, ps in self._block_params(b) if decide(k, ps)] for b in self.transformer_blocks]
        root = [k for k, ps in self._root_params() if decide(k, ps)]
        return blk, root

    def base_weight_bytes(self) -> Dict[str, int]:
        """Device bytes of the base weights in the prepared layout: bf16 resident flats, fp8 storage, bf16 slots."""
        def nb(ts):
            return sum(t.numel() * t.element_size() for t in ts if t is not None)
        lw = self._lw
        return {"bf16_resident": nb(list(self._blk_flat or []) + [self._root_flat]),
                "fp8_storage": nb(list(lw.blk_fp8) + [lw.root_fp8]) if lw else 0,
                "block_slots": nb(lw.units.slots) if (lw and lw.units) else 0,
                "root_slot": nb([lw.root_slot]) if lw else 0}

    def _apply(self, fn, recurse=True):
        """``.to()`` / ``.cuda()`` / ``.float()`` replace parameter storage when the dtype or device changes, which would
        silently detach the parameters from the packed buffers the kernels read.  Re-pack in that case (values are taken
        from the moved parameters; the fp32 LoRA masters stay fp32, the reference's own policy under DDP,
        trainer.py:130-136)."""
        was = getattr(self, "_prepared", False)
        probe = self.proj_in.weight
        probes = [self.proj_in.weight]
        if len(self.transformer_blocks):
            blk = self.transformer_blocks[0]
            probes.append(_base(getattr(blk, self.desc.ff).net[2]).weight)
            if self.lora_rank:
                probes.append(blk.attn1.to_q.lora_A["default"].weight)
        if self._lw_cfg is not None:  # a dtype cast replaces the fp8 parameters: re-pack them into fp8 storage
            probes += [p for p in self.parameters() if p.dtype in _STORAGE_DTYPES][:1]
        before = [(q.data_ptr(), q.dtype) for q in probes]
        stash = self.lora_flat.clone() if (was and self.lora_rank) else None  # a dtype cast must not round the fp32 masters
        out = super()._apply(fn, recurse)
        if self._anchor.device != probe.device:
            self._anchor = torch.zeros((), dtype=torch.float32, device=probe.device, requires_grad=True)
        if was and before != [(q.data_ptr(), q.dtype) for q in probes]:
            self._prepared = False
            self._ws.clear()
            self._arena = None
            self._iws = None
            self._tws.clear()
            self._rope.clear()
            self.prepare()
            if stash is not None:
                self.lora_flat.copy_(stash.to(self.lora_flat.device))
        return out

    def lora_parameters(self) -> List[nn.Parameter]:
        return [p for n, p in self.named_parameters() if "lora_" in n]

    def lora_state_dict(self) -> Dict[str, torch.Tensor]:
        """What ``peft.get_peft_model_state_dict`` returns for the adapters (adapter name stripped), contiguous CPU
        tensors — the ``transformer_state_dict`` finetrainers hands to ``LTXPipeline.save_lora_weights``
        (``base_specification.py:379-397``, ``trainer.py:279-306``)."""
        return {n.replace(".default.weight", ".weight"): p.detach().to("cpu").contiguous().clone()
                for n, p in self.named_parameters() if "lora_" in n}

    def save_lora_weights(self, directory: str, metadata: Optional[Dict[str, str]] = None) -> str:
        """Writes ``pytorch_lora_weights.safetensors`` with diffusers' ``transformer.`` key prefix (loadable with
        ``pipe.load_lora_weights``), plus the LoRA config as metadata like the reference's save hook."""
        import json
        import os
        from safetensors.torch import save_file
        os.makedirs(directory, exist_ok=True)
        sd = {"transformer." + k: v for k, v in self.lora_state_dict().items()}
        tm = getattr(self, "_lora_targets", LORA_TARGETS)
        # same keys, order and formatting as the reference's save hook (trainer.py:284-290)
        meta = {"format": "pt", "lora_config": json.dumps({"r": self.lora_rank, "lora_alpha": self.lora_alpha,
                                                           "init_lora_weights": getattr(self, "_lora_init", True),
                                                           "target_modules": tm if isinstance(tm, str) else list(tm)},
                                                          indent=4)}
        meta.update(metadata or {})
        path = os.path.join(directory, "pytorch_lora_weights.safetensors")
        save_file(sd, path, metadata=meta)
        return path

    # ---- flat-buffer layouts -----------------------------------------------------------------------------------------
    def _lora_groups(self) -> Dict[str, _LoraGroup]:
        """The adapter groups of every block, in the order they are packed into its slice of the flat LoRA buffers.  The
        feed-forward groups come last, so the attention-only layout is the same with or without them."""
        d, f, ff = self.cfg.inner_dim, self.desc.ffn_dim, self.desc.ff
        groups = [_LoraGroup("qkv", ("attn1.to_q", "attn1.to_k", "attn1.to_v"), d, d, "n1", "dy_qkv"),
                  _LoraGroup("o", ("attn1.to_out.0",), d, d, "ao", "dy_o", x_at="block"),
                  _LoraGroup("q2", ("attn2.to_q",), d, d, "c2n" if self.desc.cross_prenorm else "h1", "dy_q2"),
                  _LoraGroup("kv2", ("attn2.to_k", "attn2.to_v"), d, d, "enc", "dy_kv2", x_at="shared", text=True),
                  _LoraGroup("o2", ("attn2.to_out.0",), d, d, "ao2", "dy_o2", x_at="block")]
        if self.lora_ffn:  # x and dy are the FFN's input n2 / GELU output f and its gradients dwide / g
            groups += [_LoraGroup("ff1", (f"{ff}.net.0.proj",), d, f, "n2", "dwide"),
                       _LoraGroup("ff2", (f"{ff}.net.2",), f, d, "f", "g")]
        return {g.name: g for g in groups}

    def _block_specs(self):
        """(key, shape) of the tensors of ONE block's flat unit, in storage order (every size is a multiple of 8 elements,
        so every view starts 16-byte aligned as TMA requires)."""
        d, f = self.cfg.inner_dim, self.desc.ffn_dim
        specs = [("Wqkv", (3 * d, d)), ("bqkv", (3 * d,)), ("Wo", (d, d)), ("bo", (d,)), ("Wq2", (d, d)), ("bq2", (d,)),
                 ("Wo2", (d, d)), ("bo2", (d,)), ("W1", (f, d)), ("b1", (f,)), ("W2", (d, f)), ("b2", (d,)),
                 ("nq1", (d,)), ("nk1", (d,)), ("nq2", (d,)), ("sst", (6, d))]
        return specs + ([("n2w", (d,)), ("n2b", (d,))] if self.desc.cross_prenorm else [])

    def _block_params(self, blk):
        """(key, [parameters packed into that view, in order]) for one block."""
        a1, a2, ff = blk.attn1, blk.attn2, getattr(blk, self.desc.ff)
        cross = [("n2w", [blk.norm2.weight]), ("n2b", [blk.norm2.bias])] if self.desc.cross_prenorm else []
        return [("Wqkv", [_base(a1.to_q).weight, _base(a1.to_k).weight, _base(a1.to_v).weight]),
                ("bqkv", [_base(a1.to_q).bias, _base(a1.to_k).bias, _base(a1.to_v).bias]),
                ("Wo", [_base(a1.to_out[0]).weight]), ("bo", [_base(a1.to_out[0]).bias]),
                ("Wq2", [_base(a2.to_q).weight]), ("bq2", [_base(a2.to_q).bias]),
                ("Wo2", [_base(a2.to_out[0]).weight]), ("bo2", [_base(a2.to_out[0]).bias]),
                ("W1", [_base(ff.net[0].proj).weight]), ("b1", [_base(ff.net[0].proj).bias]),
                ("W2", [_base(ff.net[2]).weight]), ("b2", [_base(ff.net[2]).bias]),
                ("nq1", [a1.norm_q.weight]), ("nk1", [a1.norm_k.weight]), ("nq2", [a2.norm_q.weight]),
                ("sst", [blk.scale_shift_table])] + cross

    def _root_specs(self):
        cfg, ds = self.cfg, self.desc
        d, nl = cfg.inner_dim, cfg.num_layers
        specs = [("proj_in.w", (d, ds.in_features)), ("proj_in.b", (d,)), ("t1.w", (d, 256)), ("t1.b", (d,)),
                 ("t2.w", (d, d)), ("t2.b", (d,)), ("ada.w", (6 * d, d)), ("ada.b", (6 * d,)),
                 ("c1.w", (d, ds.text_dim)), ("c1.b", (d,)), ("c2.w", (d, d)), ("c2.b", (d,)),
                 ("sst", (2, d)), ("proj_out.w", (ds.out_features, d)), ("proj_out.b", (ds.out_features,)),
                 ("Wkv2_all", (nl, 2 * d, d)), ("bkv2_all", (nl, 2 * d)), ("nk2_all", (nl, d))]
        di = ds.image_dim
        if di:  # the image embedder (affine LayerNorm, Linear, GELU, Linear, affine LayerNorm) and every block's image K/V
            specs += [("img_n1.w", (di,)), ("img_n1.b", (di,)), ("img_ff1.w", (di, di)), ("img_ff1.b", (di,)),
                      ("img_ff2.w", (d, di)), ("img_ff2.b", (d,)), ("img_n2.w", (d,)), ("img_n2.b", (d,)),
                      ("Wkv3_all", (nl, 2 * d, d)), ("bkv3_all", (nl, 2 * d)), ("nk3_all", (nl, d))]
        return specs

    def _stacked_kv2(self):
        """The text-side K/V pieces of every block, stacked in the root unit: ([Wk2, Wv2 of each block], [biases],
        [norm_k weights])."""
        kw, kb, kn = [], [], []
        for blk in self.transformer_blocks:
            kw += [_base(blk.attn2.to_k).weight, _base(blk.attn2.to_v).weight]
            kb += [_base(blk.attn2.to_k).bias, _base(blk.attn2.to_v).bias]
            kn.append(blk.attn2.norm_k.weight)
        return kw, kb, kn

    def _root_params(self):
        te, cp = self.time_embed, self.caption_projection
        kw, kb, kn = self._stacked_kv2()
        return [("proj_in.w", [self.proj_in.weight]), ("proj_in.b", [self.proj_in.bias]),
                ("t1.w", [te.emb.timestep_embedder.linear_1.weight]), ("t1.b", [te.emb.timestep_embedder.linear_1.bias]),
                ("t2.w", [te.emb.timestep_embedder.linear_2.weight]), ("t2.b", [te.emb.timestep_embedder.linear_2.bias]),
                ("ada.w", [te.linear.weight]), ("ada.b", [te.linear.bias]),
                ("c1.w", [cp.linear_1.weight]), ("c1.b", [cp.linear_1.bias]), ("c2.w", [cp.linear_2.weight]),
                ("c2.b", [cp.linear_2.bias]), ("sst", [self.scale_shift_table]),
                ("proj_out.w", [self.proj_out.weight]), ("proj_out.b", [self.proj_out.bias]),
                ("Wkv2_all", kw), ("bkv2_all", kb), ("nk2_all", kn)]

    FLAT_ALIGN = 2048  # elements: every flat unit is padded so that it splits evenly over up to 8 ranks in 16-byte pieces
    # the root's stacked text-side [Wk2;Wv2] and biases: when cast they stream through the block slots in chunks, so they
    # have no view in the root slot and follow the slot pieces in the root's fp8 flat (LayerwiseSchedule.begin_forward
    # upcasts the slot-sized prefix of that flat)
    _STREAMED = ("Wkv2_all", "bkv2_all")

    @classmethod
    def _flat_numel(cls, specs):
        n = carved_numel(specs, 8)
        return (n + cls.FLAT_ALIGN - 1) // cls.FLAT_ALIGN * cls.FLAT_ALIGN

    @staticmethod
    def _segments(views, key_params):
        """(parameter, its segment of ``views[key]``) for every (key, [parameters]) of a unit: the parameters packed into
        one piece sit back to back in it, in order."""
        for key, params in key_params:
            v, o = views[key].reshape(-1), 0
            for prm in params:
                yield prm, v[o:o + prm.numel()].view(prm.shape)
                o += prm.numel()

    def _unit_storage(self, specs, cast, slot, dtype):
        """Storage of one flat unit: the pieces not in ``cast`` in a resident flat of ``dtype`` padded to FLAT_ALIGN, the
        cast ones in an fp8 flat whose kernel views lie at the same offsets in the bf16 ``slot`` (one upcast launch
        materialises them).  -> (resident flat, fp8 flat or None, storage views the parameters bind to, kernel views);
        with nothing cast the storage views are the kernel views."""
        dev = self.proj_in.weight.device
        keep = [(k, s) for k, s in specs if k not in cast]
        slotted = [(k, s) for k, s in specs if k in cast and k not in self._STREAMED]
        stored = slotted + [(k, s) for k, s in specs if k in cast and k in self._STREAMED]
        flat = torch.empty(self._flat_numel(keep), dtype=dtype, device=dev)
        store = carve(flat, keep, 8)
        if not stored:
            return flat, None, store, store
        f8 = torch.empty(numel16(stored), dtype=self._lw_cfg["storage_dtype"], device=dev)
        views = dict(store, **carve(slot, slotted, 16))
        store.update(carve(f8, stored, 16))
        return flat, f8, store, views

    def _bind_root_views(self, rv):
        """The kernels' views of the root unit, and every block's slices of the stacked text-side K/V pieces in it."""
        self._root_views = rv
        self._Wkv2_all, self._bkv2_all, self._nk2_all = rv.get("Wkv2_all"), rv.get("bkv2_all"), rv["nk2_all"]
        for li, e in enumerate(self._blk):
            e["nk2"] = self._nk2_all[li]
            if self._Wkv2_all is not None:
                e["Wkv2"], e["bkv2"] = self._Wkv2_all[li], self._bkv2_all[li]

    def _lora_windows(self, e, blk):
        """(lora_A, lora_B parameter, (A, B) window in the fp32 masters, (A, B) window in the gradients) of every adapter
        of a block, given its views ``e``: adapter j of a group owns A rows j rp .. j rp + r and B rows j n_out ..
        (j + 1) n_out, columns 0 .. r."""
        r, rp = self.lora_rank, self.rpad
        for g in self._groups.values():
            for j, path in enumerate(g.mods):
                m = blk.get_submodule(path)
                a, b = slice(j * rp, j * rp + r), slice(j * g.n_out, (j + 1) * g.n_out)
                yield (m.lora_A["default"].weight, m.lora_B["default"].weight,
                       (e["A_" + g.name][a], e["B_" + g.name][b, :r]), (e["gA_" + g.name][a], e["gB_" + g.name][b, :r]))

    @torch.no_grad()
    def prepare(self):
        """Pack weights into the fused layouts the kernels consume and re-point the parameters into them."""
        cfg = self.cfg
        d = cfg.inner_dim
        r = self.lora_rank
        rp = ((r + 63) // 64) * 64 if r else 0
        self.rpad = rp
        dev = self.proj_in.weight.device
        self._blk = []
        # flat fp32 LoRA master + grad (padded rank) and bf16 operand copy: per block 16 rp d elements for the attention
        # set, 26 rp d with the feed-forward adapters
        nl = cfg.num_layers
        self._groups = self._lora_groups() if r else {}
        per_blk = sum(len(g.mods) * rp * (g.k_in + g.n_out) for g in self._groups.values())
        self._per_blk = per_blk
        if r:
            self.lora_flat = torch.zeros(nl * per_blk, dtype=torch.float32, device=dev)
            self.lora_grad_flat = torch.zeros_like(self.lora_flat)
            self.lora_bf16 = torch.zeros(nl * per_blk, dtype=torch.bfloat16, device=dev)
        # ---- layerwise fp8 storage: which fused pieces are cast (none: today's layout)
        blk_cast, root_cast = self._layerwise_plan(set(self._lw_cfg["cast"])) if self._lw_cfg else ([[]] * nl, [])
        layerwise = any(blk_cast) or bool(root_cast)
        wdt = torch.bfloat16 if layerwise else self.proj_in.weight.dtype
        # ---- base weights: ONE flat buffer per DiT block (the FSDP-2 sharding unit, ptd.py:482-499) plus one "root" flat
        # buffer for everything outside the blocks; the module parameters become views of that storage.  With layerwise
        # casting a unit's cast pieces live in an fp8 flat instead, and the kernels read them from bf16 slots carved with
        # the same element offsets (one upcast launch materialises a unit)
        root_specs = self._root_specs()
        root_slot_specs = [(k, s) for k, s in root_specs if k in root_cast and k not in self._STREAMED]
        root_slot = torch.empty(numel16(root_slot_specs), dtype=torch.bfloat16, device=dev)
        self._root_flat, root_fp8, root_store, root_views = self._unit_storage(root_specs, root_cast, root_slot, wdt)
        for prm, seg in self._segments(root_store, self._root_params()):
            seg.copy_(prm.data)
            prm.data = seg
        specs = self._block_specs()
        n_slot = max([numel16([(k, s) for k, s in specs if k in bc]) for bc in blk_cast] + [0])
        slots, kv2_chunks, kv2_views = [], [], []
        # the stacked text-side [Wk2;Wv2] has no bf16 copy when cast: it streams through the block slots in chunks
        kv2_specs = lambda nb: [("W", (nb, 2 * d, d)), ("b", (nb, 2 * d))]  # noqa: E731
        if "Wkv2_all" in root_cast:
            n_slot = max(n_slot, numel16(kv2_specs(1)))
            per = max(b for b in range(1, nl + 1) if numel16(kv2_specs(b)) <= n_slot)
            kv2_chunks = [(l0, min(l0 + per, nl)) for l0 in range(0, nl, per)]
        if n_slot:
            slots = [torch.empty(n_slot, dtype=torch.bfloat16, device=dev) for _ in range(min(2, nl))]
        for c, (l0, l1) in enumerate(kv2_chunks):
            v = carve(slots[c % len(slots)], kv2_specs(l1 - l0), 16)
            kv2_views.append((v["W"], v["b"]))
        self._blk_flat, blk_fp8 = [], []
        for li, blk in enumerate(self.transformer_blocks):
            flat, f8, store, e = self._unit_storage(specs, blk_cast[li], slots[li % len(slots)] if slots else None, wdt)
            for prm, seg in self._segments(store, self._block_params(blk)):
                seg.copy_(prm.data)
                prm.data = seg
            self._blk_flat.append(flat)
            blk_fp8.append(f8)
            off = li * per_blk
            for g in self._groups.values():
                for ab, rows, cols in (("A", len(g.mods) * rp, g.k_in), ("B", len(g.mods) * g.n_out, rp)):
                    e[f"{ab}_{g.name}"], e[f"g{ab}_{g.name}"], e[f"{ab}b_{g.name}"] = (
                        t[off:off + rows * cols].view(rows, cols)
                        for t in (self.lora_flat, self.lora_grad_flat, self.lora_bf16))
                    off += rows * cols
            for pa, pb, (A, Bm), grads in self._lora_windows(e, blk):
                A.copy_(pa.data)
                Bm.copy_(pb.data)
                pa.data, pb.data = A, Bm
                pa.grad, pb.grad = grads
            self._blk.append(e)
        # the text-side K/V projection of cross attention reads only the caption embedding, so all blocks' [Wk2;Wv2], biases
        # and norm_k weights are stacked in the root unit: one batched launch per step instead of one per block
        self._bind_root_views(root_views)
        self._lw = None
        if layerwise:
            kv2_src = (root_store["Wkv2_all"], root_store["bkv2_all"]) if kv2_chunks else None
            self._lw = LayerwiseSchedule(nl, blk_fp8, slots, root_fp8, root_slot, kv2_src, kv2_chunks, kv2_views,
                                         on_cuda=dev.type == "cuda")
        self._prepared = True
        self._ws.clear()
        self._arena = None
        self._iws = None
        self._tws.clear()
        return self

    @torch.no_grad()
    def _rebind_flat_storage(self, block_flats, root_flat):
        """FSDP-2: move the base-weight views of every block onto the given full-size buffers (gather slots shared by
        several blocks) and of the root unit onto ``root_flat``, then drop the private per-block storage.  The buffers'
        contents are only valid while the owning unit is resident (fsdp.FSDPState schedules that)."""
        specs = self._block_specs()
        for e, blk, flat in zip(self._blk, self.transformer_blocks, block_flats):
            views = carve(flat, specs, 8)
            for prm, seg in self._segments(views, self._block_params(blk)):
                prm.data = seg
            e.update(views)
        rv = carve(root_flat, self._root_specs(), 8)
        for prm, seg in self._segments(rv, self._root_params()):
            prm.data = seg
        self._bind_root_views(rv)
        self._blk_flat = None
        self._root_flat = None

    def _attach_lora_grads(self):
        """(Re-)attach .grad views after an external ``zero_grad(set_to_none=True)``; returns True if any was missing."""
        missing = False
        for e, blk in zip(self._blk, self.transformer_blocks):
            for pa, pb, _, grads in self._lora_windows(e, blk):
                if pa.grad is None or pb.grad is None:
                    missing = True
                    pa.grad, pb.grad = grads
        return missing

    # ------------------------------------------------------------------------------------------------
    # workspace
    # ------------------------------------------------------------------------------------------------
    def workspace_plan(self, B, S, L, ckpt=None, sm_count=None, inference=False,
                       Li=0) -> Dict[str, Tuple[Tuple[int, ...], torch.dtype]]:
        """name -> (shape, dtype) of every workspace tensor of a step at batch B, S latent and L text tokens, under the
        checkpointing policy ``ckpt`` (block indices; default the model's).  ``sm_count`` (default: the device's) sizes
        the split-K slices of the feed-forward adapters.  ``inference``: the plan of a forward that no backward follows
        (``ckpt`` is then ignored): one slot for everything a block writes, two residual buffers, one row of attention
        outputs, and per block only the text-side k|v (and its adapters' u) that the block-batched launches write.
        ``Li``: image tokens per sample, required by (and only by) a model with an image context.  Call after
        ``prepare()`` (the padded LoRA rank sizes it)."""
        cfg = self.cfg
        d, H, nl, rp = cfg.inner_dim, cfg.num_attention_heads, cfg.num_layers, self.rpad
        hd = cfg.attention_head_dim
        R, RL = B * S, B * L
        di = self.desc.image_dim
        if bool(di) != (Li > 0):
            raise ValueError(f"{Li} image tokens for a model with image_dim {di}: an image context needs Li > 0, and "
                             "only a model with one takes it")
        # tensors a checkpointed block recomputes have one slot per block that keeps its activations plus one shared
        # scratch slot for all checkpointed blocks (nk == nl with nothing checkpointed)
        nk = 1 if inference else self._block_slots(ckpt)[1]
        nh, na = (2, 1) if inference else (nl + 1, nl)  # rows of h and of the attention outputs (_kept_rows)
        bf, f32 = torch.bfloat16, torch.float32
        ws = {}

        def z(name, *shape, kw=bf):
            ws[name] = (tuple(shape), kw)

        # embeds
        for name, shape in self._temb_specs(B).items():
            z(name, *shape)
        z("c1", RL, d); z("enc", RL, d)
        # per-block saved activations (h, both attention outputs and their lse, the text-side k|v: kept by every block)
        z("h", nh, R, d)                # training: h[l] = input of block l, h[nl] = final hidden
        z("n1", nk, R, d); z("qkv", nk, R, 3 * d)
        z("qh", nk, B, H, S, hd); z("kh", nk, B, H, S, hd); z("vh", nk, B, H, S, hd)
        z("ao", na, R, d); z("lse", na, B, H, S, kw=f32)
        z("h1", nk, R, d); z("q2", nk, R, d); z("q2h", nk, B, H, S, hd)
        z("kv2", nl, RL, 2 * d); z("k2h", nl, B, H, L, hd); z("v2h", nl, B, H, L, hd)
        z("ao2", na, R, d); z("lse2", na, B, H, S, kw=f32)
        if di:
            # the image embedder's rows (once per step), every block's image k|v (frozen: no gradient buffers) and the
            # image branch's lse, kept with the text branch's
            RLi = B * Li
            z("imn", RLi, di); z("imf", RLi, di); z("imh", RLi, d); z("img", RLi, d)
            z("kv3", nl, RLi, 2 * d); z("k3h", nl, B, H, Li, hd); z("v3h", nl, B, H, Li, hd)
            z("lse3", na, B, H, S, kw=f32)
        if self.desc.cross_prenorm:
            z("c2n", nk, R, d)         # cross attention's pre-normed input (its q projection's and adapter's x)
        F = self.desc.ffn_dim
        z("h2", nk, R, d); z("ffpre", nk, R, F)

        def lora(groups, key):  # u / dy / du of each group: per block for the text side, else per slot
            for g in groups:
                z(getattr(g, key), *((nl, RL) if g.text else (nk, R)), len(g.mods) * (g.n_out if key == "dy" else rp))

        # per-block copies of every adapter's output gradient dy and of du = s*dy*B: the weight gradients dA/dB of all
        # 28 blocks are computed at the END of backward as a handful of block-batched GEMMs (1.9 GB at B=1); a
        # checkpointed block's run right after its backward, from the scratch slot.  The feed-forward groups' dy are
        # the FFN's g / dwide below.
        att = [g for g in self._groups.values() if g.dy == "dy_" + g.name]
        ffn = [g for g in self._groups.values() if g not in att]
        bwd = [self._groups[n] for n in ("o2", "q2", "kv2", "o", "qkv")] if (att and not inference) else []
        lora(att, "u"); lora(bwd, "dy"); lora(bwd, "du")  # bwd: allocation order of dy / du
        # scratch shared by all blocks.  With feed-forward adapters the FFN's input n2, its GELU output f, its output
        # gradient g and the GELU-input gradient dwide are the adapters' x and dy, kept per block for the batched
        # weight-gradient GEMMs (3.1 GB at B=1, 2688 tokens, 28 blocks)
        ffb = (nk,) if self.lora_ffn else ()
        z("n2", *ffb, R, d); z("f", *ffb, R, F); z("y", R, d); z("pred", R, self.desc.out_features)
        if not inference:
            z("dh", R, d); z("g", *ffb, R, d); z("dwide", *ffb, R, F); z("dn", R, d); z("da", R, d)
        lora(ffn, "u")
        if not inference:
            lora(ffn, "du")
        if self.lora_ffn:
            # fp32 slices of the split-K adapter launches (u_ff2 forward, du_ff1 backward: same shape)
            s = self._ffn_splits(R, F, sm_count)
            if s > 1:
                z("splitk", s, R, rp, kw=f32)
        if inference:
            return ws
        z("dqh", B, H, S, hd); z("dkh", B, H, S, hd); z("dvh", B, H, S, hd)
        z("dk2h", nl, B, H, L, hd); z("dv2h", nl, B, H, L, hd)   # kept per block: one batched norm-bwd at the end
        if di:  # the two branch outputs the dual attention backward reads, recomputed block by block
            z("o2t", R, d); z("o2i", R, d)
        z("delta", max(ops.attn_bwd_ws_floats(B, H, S, S, head_dim=hd), ops.attn_bwd_ws_floats(B, H, S, L, head_dim=hd),
                       ops.attn_dual_bwd_ws_floats(B, H, S, L, head_dim=hd) if di else 0), kw=f32)
        return ws

    def _temb_specs(self, G) -> Dict[str, Tuple[int, ...]]:
        """name -> shape of the timestep embedding's buffers for G timesteps (bf16): its sinusoid, both MLP layers, the
        head's modulation (``embedded``) and every block's (``temb``)."""
        d = self.cfg.inner_dim
        return {"tsin": (G, 256), "t1": (G, d), "t2s": (G, d), "embedded": (G, d), "temb": (G, 6 * d)}

    def _temb_plan(self, ws, B, S, G):
        """-> (buffers of the timestep embedding, latent tokens per timestep) for G timesteps: the workspace's B-row
        buffers and S for one timestep per sample (G == B), else G-row buffers kept per G and S * B / G tokens (one
        timestep per latent frame).  The G-row buffers outlive every forward, so a captured graph replays into them,
        and they stay out of ``workspace_plan``."""
        if G == B:
            return ws, S
        bufs = self._tws.get(G)
        if bufs is None:
            dev = self.proj_in.weight.device
            bufs = {k: torch.zeros(*s, dtype=torch.bfloat16, device=dev) for k, s in self._temb_specs(G).items()}
            self._tws[G] = bufs
        return bufs, S * B // G

    def workspace_bytes(self, B, S, L, ckpt=None, sm_count=None, inference=False, Li=0) -> int:
        """Device bytes of ``workspace_plan(B, S, L, ckpt, sm_count, inference, Li)``."""
        return sum(math.prod(s) * torch.empty((), dtype=dt).element_size()
                   for s, dt in self.workspace_plan(B, S, L, ckpt, sm_count, inference, Li).values())

    @staticmethod
    def _kept_rows(l, inference=False):
        """-> (row of block l's input in the workspace's ``h``, row of its output there, row of its attention outputs
        and their lse in ``ao`` / ``lse`` / ``ao2`` / ``lse2``).  The training plans keep all of them for backward; the
        inference plan alternates between two residual rows and overwrites one row of attention outputs per block."""
        return (l % 2, (l + 1) % 2, 0) if inference else (l, l + 1, l)

    # bytes: every workspace view starts on the caching allocator's own 512-byte granularity, as a separately allocated
    # tensor would (TMA needs 16 bytes, the head_dim-128 attention output 32), so a single shape's arena takes the bytes
    # its per-tensor allocations took
    ARENA_ALIGN = 512

    @classmethod
    def arena_layout(cls, plan) -> Tuple[Dict[str, int], int]:
        """-> (name -> byte offset, bytes) of a workspace plan laid out back to back in plan order, every tensor starting
        at a multiple of ARENA_ALIGN bytes."""
        offs, o = {}, 0
        for name, (shape, dt) in plan.items():
            offs[name] = o
            o += -(-math.prod(shape) * dt.itemsize // cls.ARENA_ALIGN) * cls.ARENA_ALIGN
        return offs, o

    def _workspace(self, B, S, L, Li=0):
        """The training workspace of a step at (B, S, L) (and Li image tokens with an image context): views of
        ``workspace_plan(B, S, L, Li=Li)`` carved from the one training arena all shapes share, which holds the largest
        plan seen so far.  A plan that does not fit grows it: every shape's views and the old arena are dropped before
        the new one is allocated, so growth peaks at the new size, and ``workspace_generation`` is bumped (CUDA graphs
        captured over the old arena hold dead pointers).  A step at any shape overwrites whatever the previous step at
        any other shape left in the arena."""
        key = (B, S, L) + ((Li,) if Li else ())
        ws = self._ws.get(key)
        if ws is not None:
            return ws
        plan = self.workspace_plan(B, S, L, Li=Li)
        offs, nbytes = self.arena_layout(plan)
        if self._arena is None or self._arena.numel() < nbytes:
            self._ws.clear()
            self._arena = None
            self._arena = torch.zeros(nbytes, dtype=torch.uint8, device=self.proj_in.weight.device)
            self.workspace_generation += 1
        ws = {name: self._arena[offs[name]:offs[name] + math.prod(shape) * dt.itemsize].view(dt).view(shape)
              for name, (shape, dt) in plan.items()}
        self._ws[key] = ws
        return ws

    def _inference_workspace(self, B, S, L, Li=0):
        """The one inference workspace, for (B, S, L) (and Li image tokens): a forward at another shape frees the
        previous one before allocating its own (validation lists several resolutions).  The training workspaces in
        ``_ws`` are never touched, so CUDA graphs captured over them stay valid; a graph captured over this one must be
        dropped before a forward at another shape."""
        key = (B, S, L) + ((Li,) if Li else ())
        if self._iws is not None and self._iws[0] == key:
            return self._iws[1]
        self._iws = None
        dev = self.proj_in.weight.device
        ws = {name: torch.zeros(*shape, dtype=dt, device=dev)
              for name, (shape, dt) in self.workspace_plan(B, S, L, inference=True, Li=Li).items()}
        self._iws = (key, ws)
        return ws

    def _rope_tables(self, Fr, Hh, Ww, rope_scale):
        key = (Fr, Hh, Ww, tuple(float(x) for x in rope_scale))
        t = self._rope.get(key)
        if t is None and self.desc.rope_per_head:
            # diffusers WanRotaryPosEmbed on the post-patch grid (theta 10000), one [S, head_dim / 2] table for all heads
            hd = self.cfg.attention_head_dim
            cos = torch.empty(Fr * Hh * Ww, hd // 2, dtype=torch.float32, device=self.proj_in.weight.device)
            sin = torch.empty_like(cos)
            ops.rope_table_wan(cos, sin, Fr, Hh, Ww, hd, 10000.0)
            t = self._rope[key] = (cos, sin)
        if t is None:
            d = self.cfg.inner_dim
            dev = self.proj_in.weight.device
            cos = torch.empty(Fr * Hh * Ww, d // 2, dtype=torch.float32, device=dev)
            sin = torch.empty_like(cos)
            # diffusers LTXVideoRotaryPosEmbed: grid * scale * patch / base (base_num_frames 20, base_h = base_w = 2048)
            ops.rope_table(cos, sin, Fr, Hh, Ww, d, rope_scale[0] * self.cfg.patch_size_t / 20.0,
                           rope_scale[1] * self.cfg.patch_size / 2048.0, rope_scale[2] * self.cfg.patch_size / 2048.0)
            t = (cos, sin)
            self._rope[key] = t
        return t

    # ------------------------------------------------------------------------------------------------
    # public forward (diffusers signature; patch.py:38-51)
    # ------------------------------------------------------------------------------------------------
    def forward(self, hidden_states, encoder_hidden_states, timestep, encoder_attention_mask=None, num_frames=None,
                height=None, width=None, rope_interpolation_scale=None, return_dict=False, **kwargs):
        if not self._prepared:
            self.prepare()
        B = hidden_states.shape[0]
        # one timestep per sample, or per latent frame: finetrainers' per-token timesteps are constant per sample
        # (base_specification.py:319-320), the image-to-video pipeline's are 0 on the conditioning frame
        tvals = timestep_values(timestep, B, int(num_frames), int(height) * int(width))
        key_bias = None
        if encoder_attention_mask is not None:
            m = encoder_attention_mask
            if m.ndim == 3:
                m = m[:, 0]
            key_bias = ((1.0 - m.to(torch.float32)) * -10000.0).contiguous()  # patch.py:55-57
        if rope_interpolation_scale is None:
            rope_interpolation_scale = (1.0, 1.0, 1.0)
        args = (hidden_states, encoder_hidden_states, tvals, key_bias, int(num_frames), int(height), int(width),
                tuple(float(x) for x in rope_interpolation_scale))
        if not torch.is_grad_enabled() and self._fsdp is None:
            # no backward can follow (LTXPipeline's denoising loop): the inference plan, same kernels and arguments, so
            # the same bits, in a workspace that keeps nothing for backward.  FSDP-2's gather schedule assumes a backward
            # follows the forward, so a sharded model keeps the training plan.
            return (self._forward_impl(*args, inference=True),)
        return (_StepFn.apply(self._anchor, self, *args),)

    # ------------------------------------------------------------------------------------------------
    # forward implementation
    # ------------------------------------------------------------------------------------------------
    def refresh_lora_operands(self):
        """fp32 master -> bf16 GEMM operands (one flat cast per step)."""
        if self.lora_rank:
            ops.cast_f32_bf16(self.lora_flat, self.lora_bf16, self.lora_flat.numel(), 1.0)

    @property
    def _schedule(self):
        """FSDP-2's gathers, layerwise storage's upcasts (``FSDPState`` refuses a model with both) or no-ops."""
        return self._fsdp if self._fsdp is not None else self._lw if self._lw is not None else _ALL_RESIDENT

    def _lora_u(self, e, ws, g, a, sl, split=False):
        """u = s x A^T of group ``g``'s adapters in a block (views ``e``, workspace slot sl, row ``a`` of the inputs kept
        per block) in one launch (``split``: the deterministic split-K) -> the K-extension of the group's GEMM,
        out = x W^T + u B^T, or {} without adapters."""
        grp = self._groups.get(g)
        if grp is None:
            return {}
        rp, n_ad = self.rpad, len(grp.mods)
        x, u = ws[grp.x][a if grp.x_at == "block" else sl], ws[grp.u][sl]
        if split:
            self._lora_skinny(x, e["Ab_" + g], u, False, ws, "lora_u_splitk")
        else:
            ops.gemm(x, e["Ab_" + g], u, M=x.shape[0], N=n_ad * rp, K=grp.k_in, alpha=self.lora_scaling, tag="lora_u")
        return dict(A2=u, B2=e["Bb_" + g], K2=rp, a2_group_n=grp.n_out if n_ad > 1 else 0)

    def _lora_du(self, e, ws, g, sl, split=False):
        """du = s dy B of group ``g``'s adapters (block views ``e``, workspace slot sl) in one launch (``split``: the
        deterministic split-K) -> the K-extension of the group's dX GEMM, dx = dy W + du A, or {} without adapters."""
        grp, rp = self._groups.get(g), self.rpad
        if grp is None:
            return {}
        n_ad, n = len(grp.mods), grp.n_out
        dy, du = ws[grp.dy][sl], ws[grp.du][sl]
        if split:
            self._lora_skinny(dy, e["Bb_" + g], du, True, ws, "lora_du_splitk")
        else:
            ops.gemm(dy, e["Bb_" + g], du, M=dy.shape[0], N=rp, K=n, b_mn=True, batch=n_ad, a_boff=(0, n),
                     b_boff=(n, 0), c_boff=rp, ldc=n_ad * rp, alpha=self.lora_scaling, tag="lora_du")
        return dict(A2=du, B2=e["Ab_" + g], K2=n_ad * rp)

    def _ffn_splits(self, M, K, sm=None):
        """K slices of the two feed-forward adapter launches with a K = 4 D contraction and N = rp (u_ff2 = s f A_ff2^T,
        du_ff1 = s dwide B_ff1).  Unsplit they run one CTA per 128-row tile, 21 CTAs on 132 SMs at M = 2688, each over
        all 128 k-blocks.  Each slice must be a whole number of 64-deep k-blocks (a batch offset along K).  Measured at
        M = 2688, K = 8192, rp = 64 on an H100 80GB HBM3 at 700 W (tools/lora_ffn_bench.py: split GEMM + reduction
        replayed from a CUDA graph, 1000 calls, SM clock 1980 MHz), in us for s = 1 / 2 / 4 / 8 / 16: u_ff2 27.6 / 20.3
        / 21.7 / 25.5 / 30.3, du_ff1 27.1 / 20.2 / 21.6 / 25.3 / 30.0.  The launch reads its 44 MB operand once (13 us
        at the 3.35 TB/s data-sheet bandwidth), so beyond two slices the fp32 slice traffic and the reduction cost more
        than the added CTAs recover.  So: two slices where K splits into whole k-blocks and both slices' tiles fit on
        the SMs at once, else one."""
        sm = sm or torch.cuda.get_device_properties(self.proj_in.weight.device).multi_processor_count
        return 2 if K % 128 == 0 and 2 * -(-M // 128) <= sm else 1

    def _lora_skinny(self, x, W, out, b_mn, ws, tag):
        """out [M, rp] = bf16(s x W^T) (x [M, K], W [rp, K]; b_mn: W given as [K, rp]) over a K = 4 D contraction.
        Split-K: each slice of K stores its fp32 product into the workspace, and one reduction adds the slices in slice
        order and rounds, so the result has the same bits on every run (the atomic split-K would not)."""
        rp = self.rpad
        M, K = x.shape
        part = ws.get("splitk")
        if part is None:
            return ops.gemm(x, W, out, M=M, N=rp, K=K, b_mn=b_mn, alpha=self.lora_scaling, tag=tag)
        s = part.shape[0]
        kk = K // s
        ops.gemm(x, W, part, M=M, N=rp, K=kk, b_mn=b_mn, ldc=rp, batch=s, a_boff=(0, kk),
                 b_boff=(kk, 0) if b_mn else (0, kk), c_boff=M * rp, epi=ops.EPI_F32_STORE, tag=tag)
        return ops.splitk_reduce_bf16(part, out, s, M, rp, alpha=self.lora_scaling)

    def _forward_impl(self, hidden_states, ehs, tvals, key_bias, Fr, Hh, Ww, rope_scale, ehs_img=None,
                      inference=False):
        """The forward of the whole stack.  ``tvals``: fp32 timesteps, [B] (one per sample) or [B * Fr] (one per latent
        frame, ``timestep_values``).  ``ehs_img``: the image context [B, Li, image_dim] of a model with one (embedded
        and projected to every block's frozen image k|v once, before the blocks).  ``inference``: into the inference
        workspace (``workspace_plan(..., inference=True)``), leaving what a pending backward reads untouched; the
        launches are the same."""
        cfg = self.cfg
        d, H, nl, rp = cfg.inner_dim, cfg.num_attention_heads, cfg.num_layers, self.rpad
        hd = cfg.attention_head_dim
        B, S, Cin = hidden_states.shape
        L = ehs.shape[1]
        assert S == Fr * Hh * Ww, "sequence length must equal num_frames*height*width (patch size 1)"
        R, RL = B * S, B * L
        G = tvals.numel()
        if G not in (B, B * Fr):
            raise ValueError(f"{G} timesteps for {B} samples of {Fr} latent frames: one per sample or per frame")
        di = self.desc.image_dim
        if (ehs_img is not None) != bool(di):
            raise ValueError(f"image context {'given to a model without one' if ehs_img is not None else 'missing'}")
        if di and (ehs_img.ndim != 3 or ehs_img.shape[0] != B or ehs_img.shape[2] != di or key_bias is not None):
            raise ValueError(f"the image context must be [{B}, Li, {di}] with no text key bias, not "
                             f"{tuple(ehs_img.shape)}")
        Li = ehs_img.shape[1] if di else 0
        if inference:
            ws = self._inference_workspace(B, S, L, Li)
        else:
            ws = self._workspace(B, S, L, Li)
            self._saved_key = (B, S, L, Fr, Hh, Ww, rope_scale, G, Li)
            self._key_bias = key_bias
        temb_plan = self._temb_plan(ws, B, S, G)
        tw, rps = temb_plan
        self._fwd_gen += 1  # a backward of an earlier autograd forward now raises (_StepFn.backward)
        cos, sin = self._rope_tables(Fr, Hh, Ww, rope_scale)
        x_in = hidden_states.reshape(R, Cin).to(torch.bfloat16).contiguous()
        ehs2 = ehs.reshape(RL, self.desc.text_dim).to(torch.bfloat16).contiguous()
        self.refresh_lora_operands()
        fs = self._schedule
        # FSDP-2: all-gather the root unit and the first two blocks (communication stream); layerwise: upcast the root
        # slot, start upcasting what the block slots hold first (side stream)
        fs.begin_forward()
        rv = self._root_views  # the kernels' views of the root unit (bf16; a slot for pieces stored in fp8)
        # ---- timestep embedding on the G distinct timesteps (K2)
        ops.timestep_sinusoid(tvals, tw["tsin"], G)
        ops.gemm(tw["tsin"], rv["t1.w"], tw["t1"], M=G, N=d, K=256, bias=rv["t1.b"], epi=ops.EPI_SILU)
        ops.gemm(tw["t1"], rv["t2.w"], tw["t2s"], M=G, N=d, K=d, bias=rv["t2.b"], epi=ops.EPI_SILU, out2=tw["embedded"])
        ops.gemm(tw["t2s"], rv["ada.w"], tw["temb"], M=G, N=6 * d, K=d, bias=rv["ada.b"])
        # ---- caption projection (K3), patch embed (K1)
        ops.gemm(ehs2, rv["c1.w"], ws["c1"], M=RL, N=d, K=self.desc.text_dim, bias=rv["c1.b"], epi=ops.EPI_GELU)
        ops.gemm(ws["c1"], rv["c2.w"], ws["enc"], M=RL, N=d, K=d, bias=rv["c2.b"])
        enc = ws["enc"]
        ops.gemm(x_in, rv["proj_in.w"], ws["h"][0], M=R, N=d, K=Cin, bias=rv["proj_in.b"])
        # ---- cross-attention K/V of ALL blocks (functions of `enc` only): LoRA-down, fused [Wk2;Wv2] projection with the
        # LoRA-up K-extension, and k-norm + head split, each as ONE block-batched launch
        ops.CONTEXT = "f.kv2"
        e0, pb = self._blk[0], self._per_blk
        kv2_all = ws["kv2"].view(nl * RL, 2 * d)
        kv = self._groups.get("kv2")
        if kv:
            U = len(kv.mods) * rp
            u_all = ws[kv.u].view(nl * RL, U)
            ops.gemm(ws[kv.x], e0["Ab_kv2"], u_all, M=RL, N=U, K=kv.k_in, batch=nl, b_boff=(pb // kv.k_in, 0),
                     c_boff=RL * U, alpha=self.lora_scaling, tag="lora_u")
        if self._Wkv2_all is not None:
            kv2_parts = [(0, nl, self._Wkv2_all, self._bkv2_all)]
        else:  # stored in fp8: block-range chunks upcast through the block slots, one batched launch per chunk
            kv2_parts = [(l0, l1, None, None) for l0, l1 in self._lw.kv2_chunks]
        for c, (l0, l1, W, bkv) in enumerate(kv2_parts):
            if W is None:
                W, bkv = self._lw.kv2_wait(c)
            nb = l1 - l0
            ext = dict(A2=u_all[l0 * RL:], B2=self._blk[l0]["Bb_kv2"], K2=rp, a2_group_n=kv.n_out, a2_boff_row=RL,
                       b2_boff_row=pb // rp) if kv else {}
            ops.gemm(enc, W.view(nb * 2 * d, d), kv2_all[l0 * RL:], M=RL, N=2 * d, K=d, bias=bkv, batch=nb,
                     b_boff=(2 * d, 0), c_boff=RL * 2 * d, bias_boff=2 * d, **ext)
            if self._Wkv2_all is None:
                self._lw.kv2_release(c)
        ops.qkv_norm_rope_fwd(kv2_all, 2 * d, 0, (self._nk2_all, None), 0, None, None, (ws["k2h"], ws["v2h"]), nl * B, L, H,
                              self.desc.qk_eps, rows_per_w=RL, w_stride=d, head_dim=hd)
        if di:
            # ---- image context (frozen weights, constant input: no backward): the image embedder, then every block's
            # [Wk3;Wv3] projection and k-norm + head split, each as ONE block-batched launch
            ops.CONTEXT = "f.img"
            RLi = B * Li
            xi = ehs_img.reshape(RLi, di).to(torch.bfloat16).contiguous()
            ops.layer_norm_affine_fwd(xi, ws["imn"], rv["img_n1.w"], rv["img_n1.b"], RLi, di, IMAGE_NORM_EPS)
            ops.gemm(ws["imn"], rv["img_ff1.w"], ws["imf"], M=RLi, N=di, K=di, bias=rv["img_ff1.b"])
            ops.gelu_erf(ws["imf"], ws["imf"], RLi * di)  # exact GELU on the rounded Linear output, as F.gelu
            ops.gemm(ws["imf"], rv["img_ff2.w"], ws["imh"], M=RLi, N=d, K=di, bias=rv["img_ff2.b"])
            ops.layer_norm_affine_fwd(ws["imh"], ws["img"], rv["img_n2.w"], rv["img_n2.b"], RLi, d, IMAGE_NORM_EPS)
            kv3_all = ws["kv3"].view(nl * RLi, 2 * d)
            ops.gemm(ws["img"], rv["Wkv3_all"].view(nl * 2 * d, d), kv3_all, M=RLi, N=2 * d, K=d, bias=rv["bkv3_all"],
                     batch=nl, b_boff=(2 * d, 0), c_boff=RLi * 2 * d, bias_boff=2 * d)
            ops.qkv_norm_rope_fwd(kv3_all, 2 * d, 0, (rv["nk3_all"], None), 0, None, None, (ws["k3h"], ws["v3h"]),
                                  nl * B, Li, H, self.desc.qk_eps, rows_per_w=RLi, w_stride=d, head_dim=hd)
        slots = [0] * nl if inference else self._block_slots()[0]
        for l in range(nl):
            fs.pre_block_forward(l)
            self._block_forward(l, slots[l], ws, B, S, L, cos, sin, key_bias, temb_plan,
                                rows=self._kept_rows(l, inference))
            fs.post_block_forward(l)  # block l's weights are no longer read: its slot takes block l + 2
        ops.CONTEXT = "f.head"
        # K13: final LayerNorm + modulate (table rows 0 = shift, 1 = scale; embedded_timestep), proj_out
        t2 = rv["sst"]
        h_out = ws["h"][self._kept_rows(nl - 1, inference)[1]]
        ops.norm_modulate_fwd(h_out, ws["y"], t2[0], tw["embedded"], t2[1], tw["embedded"], d, R, d, rps, 1e-6, True)
        ops.gemm(ws["y"], rv["proj_out.w"], ws["pred"], M=R, N=self.desc.out_features, K=d, bias=rv["proj_out.b"])
        ops.CONTEXT = ""
        return ws["pred"].view(B, S, self.desc.out_features)

    def _block_forward(self, l, sl, ws, B, S, L, cos, sin, key_bias, temb_plan, recompute=False, rows=None):
        """Forward of block l, modulated by ``temb_plan`` = ``_temb_plan(...)`` (the timestep embedding's buffers and the
        latent tokens per timestep): the tensors a checkpointed block recomputes go to slot ``sl`` of the workspace, the kept
        ones to the rows ``rows`` = ``_kept_rows(l, ...)`` (block input and output in h, attention outputs and lse; by
        default the training plans' l, l + 1, l) and the text-side k|v to index l.  ``recompute`` re-runs the block
        before its backward with the same kernels and arguments, so it rewrites the same bits; it skips both attention
        forwards (their outputs are kept) and FFN down (its output h[l + 1] is kept)."""
        cfg, ds = self.cfg, self.desc
        d, H, hd = cfg.inner_dim, cfg.num_attention_heads, cfg.attention_head_dim
        F, ffn = ds.ffn_dim, self.lora_ffn
        R = B * S
        scale = 1.0 / math.sqrt(cfg.attention_head_dim)
        temb, rps = temb_plan[0]["temb"], temb_plan[1]
        ctx = "r." if recompute else "f."
        e = self._blk[l]
        sst = e["sst"]
        hi, ho, a = self._kept_rows(l) if rows is None else rows
        h_in, n1 = ws["h"][hi], ws["n1"][sl]
        # K5: RMSNorm (LayerNorm: ds.layer_norm) + modulate (shift_msa = row 0, scale_msa = row 1)
        ops.CONTEXT = ctx + "self"
        ops.norm_modulate_fwd(h_in, n1, sst[0], temb[:, 0:], sst[1], temb[:, d:], 6 * d, R, d, rps, ds.norm_eps,
                              ds.layer_norm)
        # K6: fused QKV (+LoRA)
        ops.gemm(n1, e["Wqkv"], ws["qkv"][sl], M=R, N=3 * d, K=d, bias=e["bqkv"], **self._lora_u(e, ws, "qkv", a, sl))
        # K7: q/k RMSNorm + RoPE + head split
        ops.qkv_norm_rope_fwd(ws["qkv"][sl], 3 * d, 0, (e["nq1"], e["nk1"], None), 0b011, cos, sin,
                              (ws["qh"][sl], ws["kh"][sl], ws["vh"][sl]), B, S, H, ds.qk_eps, head_dim=hd,
                              per_head=ds.rope_per_head)
        # K8: self attention
        if not recompute:
            ops.attn_fwd(ws["qh"][sl], ws["kh"][sl], ws["vh"][sl], None, ws["ao"][a], ws["lse"][a], B, H, S, S, scale,
                         head_dim=hd)
        # K9: out proj + gated residual (gate_msa = row 2)
        ops.gemm(ws["ao"][a], e["Wo"], ws["h1"][sl], M=R, N=d, K=d, bias=e["bo"], epi=ops.EPI_GATE_RES, res=h_in,
                 gate_table=sst[2], gate_temb=temb[:, 2 * d:], temb_stride=6 * d, rows_per_sample=rps,
                 **self._lora_u(e, ws, "o", a, sl))
        # K10: cross attention (no gate; an affine LayerNorm before the q projection with ds.cross_prenorm)
        ops.CONTEXT = ctx + "cross"
        h1 = ws["h1"][sl]
        xq = h1
        if ds.cross_prenorm:
            xq = ws["c2n"][sl]
            ops.layer_norm_affine_fwd(h1, xq, e["n2w"], e["n2b"], R, d, ds.norm_eps)
        ops.gemm(xq, e["Wq2"], ws["q2"][sl], M=R, N=d, K=d, bias=e["bq2"], **self._lora_u(e, ws, "q2", a, sl))
        ops.qknorm_rope_fwd(ws["q2"][sl], d, 0, e["nq2"], None, None, ws["q2h"][sl], B, S, H, True, ds.qk_eps,
                            head_dim=hd)
        if not recompute and ds.image_dim:  # two softmaxes, text then image, their bf16 outputs summed and rounded
            ops.attn_dual_fwd(ws["q2h"][sl], ws["k2h"][l], ws["v2h"][l], L, ws["k3h"][l], ws["v3h"][l],
                              ws["k3h"].shape[3], ws["ao2"][a], ws["lse2"][a], ws["lse3"][a], B, H, S, scale,
                              head_dim=hd)
        elif not recompute:
            ops.attn_fwd(ws["q2h"][sl], ws["k2h"][l], ws["v2h"][l], key_bias, ws["ao2"][a], ws["lse2"][a], B, H, S, L,
                         scale, head_dim=hd)
        ops.gemm(ws["ao2"][a], e["Wo2"], ws["h2"][sl], M=R, N=d, K=d, bias=e["bo2"], epi=ops.EPI_GATE_RES, res=h1,
                 **self._lora_u(e, ws, "o2", a, sl))
        # K11/K12: norm2 + modulate (rows 3,4), FFN with GELU epilogue, gated residual (row 5)
        # (feed-forward adapters: u_ff1 = s n2 A_ff1^T as a K-extension of FFN up; u_ff2 = s f A_ff2^T over K = 4 D by
        # the deterministic split-K, then a K-extension of FFN down)
        ops.CONTEXT = ctx + "ffn"
        h2 = ws["h2"][sl]
        n2, f = (ws["n2"][sl], ws["f"][sl]) if ffn else (ws["n2"], ws["f"])
        ops.norm_modulate_fwd(h2, n2, sst[3], temb[:, 3 * d:], sst[4], temb[:, 4 * d:], 6 * d, R, d, rps,
                              ds.norm_eps, ds.layer_norm)
        ops.gemm(n2, e["W1"], f, M=R, N=F, K=d, bias=e["b1"], epi=ops.EPI_GELU, out2=ws["ffpre"][sl], tag="ffn_up",
                 **self._lora_u(e, ws, "ff1", a, sl))
        ext = self._lora_u(e, ws, "ff2", a, sl, split=True)  # u is recomputed too: the weight gradients read it
        if not recompute:
            ops.gemm(f, e["W2"], ws["h"][ho], M=R, N=d, K=F, bias=e["b2"], epi=ops.EPI_GATE_RES,
                     res=h2, gate_table=sst[5], gate_temb=temb[:, 5 * d:], temb_stride=6 * d, rows_per_sample=rps, **ext)

    # ------------------------------------------------------------------------------------------------
    # backward implementation (LoRA: dX through every op, dW only for adapters)
    # ------------------------------------------------------------------------------------------------
    def _lora_wgrads(self, ws, lo=0, hi=None):
        """dA / dB of every adapter of blocks [lo, hi): 13 (17 with the feed-forward adapters) block-batched split-free
        GEMMs (dB_j += dy_j^T u_j ;
        dA += du^T x computed as (x^T du)^T), accumulating into the flat fp32 gradient buffer.  The whole model in one go
        at the end of backward, or one block range at a time so that the range's slice of the flat gradient is final -
        and its all-reduce can start - while earlier blocks are still in backward (trainer: DDP overlap).  Checkpointed
        blocks are left out except for the text side: theirs ran right after their backward (``_backward_blocks``)."""
        nl, rp, pb = self.cfg.num_layers, self.rpad, self._per_blk
        hi = nl if hi is None else hi
        nr = hi - lo
        kv = self._groups["kv2"]
        RL, n = ws[kv.dy].shape[1], kv.n_out
        N, U = len(kv.mods) * n, len(kv.mods) * rp
        # the text-side adapters have no dX consumer, so their du is also produced here, block-batched per adapter
        for j in range(len(kv.mods)):
            ops.gemm(ws[kv.dy].view(nl * RL, N)[lo * RL:, j * n:], self._blk[lo]["Bb_kv2"][j * n:],
                     ws[kv.du].view(nl * RL, U)[lo * RL:, j * rp:], M=RL, N=rp, K=n, lda=N, ldb=rp, ldc=U, b_mn=True,
                     batch=nr, a_boff=(RL, 0), b_boff=(pb // rp, 0), c_boff=RL * U, alpha=self.lora_scaling,
                     tag="lora_du")
        kept = self._kept_runs(lo, hi)
        for g in self._groups.values():
            self._group_wgrads(ws, g, [(lo, nr)] if g.text else kept)

    def _group_wgrads(self, ws, grp, runs):
        """dB_j += dy_j^T u_j and dA += (x^T du)^T of one adapter group for each run (first block, block count) of
        blocks with consecutive workspace slots.  The tile width is given explicitly and MN-major A never takes CTA
        pairs, so a block's launch computes the same per-element sums whatever the run length."""
        rp, pb = self.rpad, self._per_blk
        g, n_ad, k_in, n_out = grp.name, len(grp.mods), grp.k_in, grp.n_out
        slots = self._block_slots()[0]
        N = n_ad * n_out
        M = ws[grp.dy].shape[1]  # token rows of one block
        dy2, u2, du2 = ws[grp.dy].view(-1, N), ws[grp.u].view(-1, n_ad * rp), ws[grp.du].view(-1, n_ad * rp)
        x2 = ws[grp.x].view(-1, k_in)
        x_stride = 0 if grp.x_at == "shared" else M
        # the contraction runs over the M token rows of ONE block: stacking blocks along that axis is only legal when
        # M is a whole number of 64-row k-blocks (otherwise the k-tail would read the next block's rows, not zeros)
        spans = runs if M % 64 == 0 else [(l, 1) for l0, nb in runs for l in range(l0, l0 + nb)]
        for (l0, nb) in spans:
            r0 = (l0 if grp.text else slots[l0]) * M                    # block l0's first row in dy / u / du
            x0 = {"block": l0 * M, "slot": r0, "shared": 0}[grp.x_at]  # and in x
            for j in range(n_ad):
                ops.gemm(dy2[r0:, j * n_out:], u2[r0:, j * rp:], self._blk[l0]["gB_" + g][j * n_out:],
                         M=n_out, N=rp, K=M, lda=N, ldb=n_ad * rp, ldc=rp, a_mn=True, b_mn=True, batch=nb, a_boff=(M, 0),
                         b_boff=(M, 0), c_boff=pb, epi=ops.EPI_F32_ATOMIC, block_n=64 if rp == 64 else 128,
                         tag="lora_dB")
            ops.gemm(x2[x0:], du2[r0:], self._blk[l0]["gA_" + g], M=k_in, N=n_ad * rp, K=M,
                     lda=k_in, ldb=n_ad * rp, ldc=k_in, a_mn=True, b_mn=True, batch=nb, a_boff=(x_stride, 0),
                     b_boff=(M, 0), c_boff=pb, epi=ops.EPI_F32_ATOMIC_T, block_n=64, tag="lora_dA")

    def _backward_impl(self, dpred):
        """The whole backward in one call (autograd path / single graph)."""
        self._backward_head(dpred)
        self._backward_blocks(self.cfg.num_layers - 1, 0)
        self._backward_tail(0, self.cfg.num_layers)
        self._schedule.end_backward()

    def _bwd_ctx(self):
        """What the last training forward saved: its workspace, RoPE tables and timestep plan (``_temb_plan``)."""
        cfg = self.cfg
        B, S, L, Fr, Hh, Ww, rope_scale, G, Li = self._saved_key
        ws = self._workspace(B, S, L, Li)
        cos, sin = self._rope_tables(Fr, Hh, Ww, rope_scale)
        return cfg, B, S, L, ws, cos, sin, self._temb_plan(ws, B, S, G)

    def _backward_head(self, dpred):
        """proj_out / final LayerNorm+modulate backward: leaves dh (residual-stream gradient) and g (dh x gate_mlp of the
        last block) in the workspace."""
        cfg, B, S, L, ws, cos, sin, (tw, rps) = self._bwd_ctx()
        d, nl, rp = cfg.inner_dim, cfg.num_layers, self.rpad
        R = B * S
        temb = tw["temb"]
        if not rp:
            raise NotImplementedError("full-rank fine-tuning backward (base dW) is not built yet; use add_adapter()")
        if self._attach_lora_grads():
            self.lora_grad_flat.zero_()
        dp = dpred.reshape(R, self.desc.out_features).to(torch.bfloat16).contiguous()
        # head: dy = dpred Wout ; dh = LN-modulate bwd ; g = dh * gate_mlp(last block)
        ops.gemm(dp, self._root_views["proj_out.w"], ws["dn"], M=R, N=d, K=self.desc.out_features, b_mn=True)
        t2 = self._root_views["sst"]
        last = self._blk[nl - 1]["sst"]
        ops.norm_modulate_bwd(ws["dn"], ws["h"][nl], None, ws["dh"], t2[1], tw["embedded"], d, R, d, rps, 1e-6, True)
        # (embedded has stride d, temb stride 6d: the gate of the last block is applied by a separate colscale)
        ops.colscale(ws["dh"], ws["g"][self._block_slots()[0][nl - 1]] if self.lora_ffn else ws["g"], last[5],
                     temb[:, 5 * d:], 6 * d, R, d, rps)

    def _backward_blocks(self, l_hi, l_lo):
        """Backward through blocks l_hi, l_hi - 1, ..., l_lo (dX through every op; per-block dy / du of the adapters are
        stored for the batched weight-gradient GEMMs).  A checkpointed block is first re-run forward into the scratch
        slot (after its weights are resident), and its adapter weight gradients run before the next block's recompute
        overwrites that slot."""
        cfg, B, S, L, ws, cos, sin, temb_plan = self._bwd_ctx()
        d, H, hd = cfg.inner_dim, cfg.num_attention_heads, cfg.attention_head_dim
        R = B * S
        key_bias = self._key_bias
        temb, rps = temb_plan[0]["temb"], temb_plan[1]
        scale = 1.0 / math.sqrt(cfg.attention_head_dim)
        ds = self.desc
        F, ffn = ds.ffn_dim, self.lora_ffn
        dh = ws["dh"]
        slots = self._block_slots()[0]
        fs = self._schedule
        fs.begin_backward_range(l_hi, l_lo)
        for l in range(l_hi, l_lo - 1, -1):
            fs.pre_block_backward(l)
            sl = slots[l]
            ckpt = l in self._ckpt
            if ckpt:
                self._block_forward(l, sl, ws, B, S, L, cos, sin, key_bias, temb_plan, recompute=True)
            e = self._blk[l]
            sst = e["sst"]
            dh2, dq2, dyo, dqkv = (ws[self._groups[g].dy][sl] for g in ("o2", "q2", "o", "qkv"))
            g, dwide = (ws["g"][sl], ws["dwide"][sl]) if ffn else (ws["g"], ws["dwide"])
            # ---- FFN: dfp = (g W2) * gelu'(pre) ; dn2 = dfp W1 ; dh2 = dh + norm_bwd(dn2; h2, scale_mlp=row 4)
            # (feed-forward adapters: du_ff2 = s g B_ff2 extends the first, du_ff1 = s dfp B_ff1 over K = 4 D by the
            # deterministic split-K extends the second)
            ops.CONTEXT = "b.ffn"
            ops.gemm(g, e["W2"], dwide, M=R, N=F, K=d, b_mn=True, epi=ops.EPI_MUL_DGELU, aux=ws["ffpre"][sl],
                     **self._lora_du(e, ws, "ff2", sl))
            ops.gemm(dwide, e["W1"], ws["dn"], M=R, N=d, K=F, b_mn=True, **self._lora_du(e, ws, "ff1", sl, split=True))
            ops.norm_modulate_bwd(ws["dn"], ws["h2"][sl], dh, dh2, sst[4], temb[:, 4 * d:], 6 * d, R, d, rps,
                                  ds.norm_eps, ds.layer_norm)
            # ---- cross attention out-proj (no gate): da2 = dh2 W_o2 + du A
            ops.CONTEXT = "b.cross"
            ops.gemm(dh2, e["Wo2"], ws["da"], M=R, N=d, K=d, b_mn=True, **self._lora_du(e, ws, "o2", sl))
            if ds.image_dim:
                # the dual backward reads both branch outputs: the forward is re-run with them into the shared o2t / o2i,
                # rewriting the kept ao2 / lse2 / lse3 rows with the bits they hold (same kernel, same operands)
                Li = ws["k3h"].shape[3]
                ops.attn_dual_fwd(ws["q2h"][sl], ws["k2h"][l], ws["v2h"][l], L, ws["k3h"][l], ws["v3h"][l], Li,
                                  ws["ao2"][l], ws["lse2"][l], ws["lse3"][l], B, H, S, scale, out1=ws["o2t"],
                                  out2=ws["o2i"], head_dim=hd)
                ops.attn_dual_bwd(ws["q2h"][sl], ws["k2h"][l], ws["v2h"][l], L, ws["k3h"][l], ws["v3h"][l], Li,
                                  ws["o2t"], ws["o2i"], ws["da"], ws["lse2"][l], ws["lse3"][l], ws["delta"], ws["dqh"],
                                  ws["dk2h"][l], ws["dv2h"][l], B, H, S, scale, head_dim=hd)
            else:
                ops.attn_bwd(ws["q2h"][sl], ws["k2h"][l], ws["v2h"][l], key_bias, ws["ao2"][l], ws["da"], ws["lse2"][l],
                             ws["delta"], ws["dqh"], ws["dk2h"][l], ws["dv2h"][l], B, H, S, L, scale, head_dim=hd)
            ops.qknorm_rope_bwd(ws["dqh"], ws["q2"][sl], d, 0, e["nq2"], None, None, dq2, d, 0, B, S, H, True,
                                ds.qk_eps, head_dim=hd)
            # dh1 = dh2 + dq2 W_q2 + du A (through the pre-norm's backward with ds.cross_prenorm) ; gated copy (gate_msa,
            # row 2) = dy of the self-attention out-proj
            if ds.cross_prenorm:
                ops.gemm(dq2, e["Wq2"], ws["dn"], M=R, N=d, K=d, b_mn=True, **self._lora_du(e, ws, "q2", sl))
                ops.layer_norm_affine_bwd(ws["dn"], ws["h1"][sl], dh2, dh, e["n2w"], R, d, ds.norm_eps,
                                          gate2_tab=sst[2], gate2_emb=temb[:, 2 * d:], out2=dyo, emb_stride=6 * d,
                                          rows_per_sample=rps)
            else:
                ops.gemm(dq2, e["Wq2"], dh, M=R, N=d, K=d, b_mn=True, epi=ops.EPI_GATE_RES, res=dh2,
                         gate2_table=sst[2], gate2_temb=temb[:, 2 * d:], out2=dyo, temb_stride=6 * d,
                         rows_per_sample=rps, **self._lora_du(e, ws, "q2", sl))
            # ---- self attention out-proj (gated): dattn = g W_o + du A
            ops.CONTEXT = "b.self"
            ops.gemm(dyo, e["Wo"], ws["da"], M=R, N=d, K=d, b_mn=True, **self._lora_du(e, ws, "o", sl))
            ops.attn_bwd(ws["qh"][sl], ws["kh"][sl], ws["vh"][sl], None, ws["ao"][l], ws["da"], ws["lse"][l], ws["delta"],
                         ws["dqh"], ws["dkh"], ws["dvh"], B, H, S, S, scale, head_dim=hd)
            ops.qkv_norm_rope_bwd((ws["dqh"], ws["dkh"], ws["dvh"]), ws["qkv"][sl], 3 * d, 0, (e["nq1"], e["nk1"], None),
                                  0b011, cos, sin, dqkv, 3 * d, 0, B, S, H, ds.qk_eps, head_dim=hd,
                                  per_head=ds.rope_per_head)
            ext = self._lora_du(e, ws, "qkv", sl)
            if ckpt:  # its latent-side adapter weight gradients, before the next recompute overwrites the scratch slot
                ops.CONTEXT = "b.wgrad"
                for g in self._groups.values():
                    if not g.text:
                        self._group_wgrads(ws, g, [(l, 1)])
                ops.CONTEXT = "b.self"
            if l == 0 and self.skip_block0_dx:
                fs.post_block_backward(l)
                break  # nothing trainable upstream of block 0's adapters (proj_in / embeds are frozen)
            ops.gemm(dqkv, e["Wqkv"], ws["dn"], M=R, N=d, K=3 * d, b_mn=True, **ext)
            # dh0 = dh1 + norm_bwd(dn1; h_in, scale_msa=row 1) ; g = dh0 * gate_mlp of block l-1
            if l > 0:
                fs.pre_block_backward(l - 1)  # the op below reads block l-1's gate row: its all-gather must have landed
            prev = self._blk[l - 1]["sst"] if l > 0 else None
            ops.norm_modulate_bwd(ws["dn"], ws["h"][l], dh, dh, sst[1], temb[:, d:], 6 * d, R, d, rps, ds.norm_eps,
                                  ds.layer_norm, gate2_tab=prev[5] if l > 0 else None, gate2_emb=temb[:, 5 * d:] if l > 0 else None,
                                  out2=(ws["g"][slots[l - 1]] if ffn else ws["g"]) if l > 0 else None)
            fs.post_block_backward(l)
        ops.CONTEXT = ""

    def _backward_tail(self, lo, hi):
        """Adapter gradients of blocks [lo, hi): the text-side k-norm backward of those blocks in one launch (its output
        only feeds the kv2 adapter gradients), then the block-batched dA / dB GEMMs."""
        cfg, B, S, L, ws, cos, sin, _ = self._bwd_ctx()
        d, H, nl = cfg.inner_dim, cfg.num_attention_heads, cfg.num_layers
        RL = B * L
        ops.CONTEXT = "b.kv2"
        dy = ws[self._groups["kv2"].dy].view(nl * RL, 2 * d)
        ops.qkv_norm_rope_bwd((ws["dk2h"][lo:hi], ws["dv2h"][lo:hi]), ws["kv2"].view(nl * RL, 2 * d)[lo * RL:hi * RL], 2 * d, 0,
                              (self._nk2_all[lo:hi], None), 0, None, None, dy[lo * RL:hi * RL],
                              2 * d, 0, (hi - lo) * B, L, H, self.desc.qk_eps, rows_per_w=RL, w_stride=d,
                              head_dim=cfg.attention_head_dim)
        ops.CONTEXT = "b.wgrad"
        self._lora_wgrads(ws, lo, hi)
        ops.CONTEXT = ""


def apply_layerwise_casting(module: B200LTXTransformer, storage_dtype: torch.dtype, compute_dtype: torch.dtype,
                            skip_modules_pattern="auto", skip_modules_classes=None, non_blocking: bool = False):
    """diffusers' ``apply_layerwise_casting`` with the arguments finetrainers passes (trainer.py:112-118): fp8 storage of
    the frozen linear weights of a ``B200LTXTransformer``, bf16 compute.  See ``enable_layerwise_casting``."""
    if not isinstance(module, B200LTXTransformer):
        raise TypeError(f"layerwise casting is built for B200LTXTransformer, not {type(module).__name__}")
    return module.enable_layerwise_casting(storage_dtype, compute_dtype, skip_modules_pattern, skip_modules_classes,
                                           non_blocking)


def apply_activation_checkpointing(module: B200LTXTransformer, checkpointing_type: str = "full",
                                   n_layer: int = 1) -> B200LTXTransformer:
    """The reference's ``apply_activation_checkpointing`` (``utils/activation_checkpoint.py:24-49``, called by
    ``--gradient_checkpointing``) for a ``B200LTXTransformer``: "full" recomputes every block, "block_skip" block i iff
    i % n_layer == 0; "ops" is not built.  A recomputed block keeps its input, both attention outputs with their
    log-sum-exps and its text-side k|v, and re-runs everything else of its forward but FFN down before its backward
    (DESIGN §3).  Call before the first forward."""
    if not isinstance(module, B200LTXTransformer):
        raise TypeError(f"activation checkpointing is built for B200LTXTransformer, not {type(module).__name__}")
    return module.set_activation_checkpointing(checkpointed_blocks(len(module.transformer_blocks), checkpointing_type,
                                                                   n_layer))
