"""Attention-provider hook: the registry / context-manager / dispatcher API of
``finetrainers/models/attention_dispatch.py`` (``_AttentionProviderRegistry`` :295-362,
``attention_provider`` :365-402, ``attention_dispatch`` :405-447) with ONE provider, ``"b200"``: the wgmma
flash-attention forward/backward of libb2d.  The reference's ``AttentionProvider`` enum is closed, so this module ships
its own enum value with the same decorator API; a maintainer adds ``B200 = "b200"`` to the reference enum and imports
this module (see INTEGRATION.md).  No flash/flex/sage/xformers multi-backend zoo, no fallback.

Layout contract (tests/models/attention_dispatch.py:113-130): q,k,v ``[B, H, S, d]`` -> ``[B, H, S_q, d]``.
"""
from __future__ import annotations

import contextlib
import inspect
import math
from enum import Enum
from typing import Any, Callable, Dict, List, Optional

import torch

from . import ops


class AttentionProvider(str, Enum):
    B200 = "b200"


class _AttentionProviderRegistry:
    _providers: Dict[AttentionProvider, Callable] = {}
    _constraints: Dict[AttentionProvider, List[Callable]] = {}
    _supports_cp: Dict[AttentionProvider, bool] = {}
    _supported_arg_names: Dict[AttentionProvider, set] = {}
    _active_provider = AttentionProvider.B200
    _checks_enabled = False

    @classmethod
    def register(cls, provider: AttentionProvider, constraints: Optional[List[Callable]] = None,
                 supports_cp: bool = False):
        def decorator(func):
            cls._providers[provider] = func
            cls._constraints[provider] = constraints or []
            cls._supports_cp[provider] = supports_cp
            cls._supported_arg_names[provider] = set(inspect.signature(func).parameters.keys())
            return func

        return decorator

    @classmethod
    def get_active_provider(cls):
        return cls._active_provider, cls._providers[cls._active_provider]

    @classmethod
    def list_providers(cls):
        return list(cls._providers.keys())

    @classmethod
    def supports_context_parallel(cls, provider):
        if provider not in cls._providers:
            raise ValueError(f"Provider {provider} is not registered.")
        return cls._supports_cp.get(provider, False)


@contextlib.contextmanager
def attention_provider(provider: AttentionProvider = AttentionProvider.B200, *, mesh=None, **_):
    if provider not in _AttentionProviderRegistry._providers:
        raise ValueError(f"Provider {provider} is not registered.")
    if mesh is not None:
        raise ValueError(f"Provider {provider} does not support context parallelism.")
    old = _AttentionProviderRegistry._active_provider
    _AttentionProviderRegistry._active_provider = provider
    try:
        yield
    finally:
        _AttentionProviderRegistry._active_provider = old


def attention_dispatch(query, key, value, attn_mask=None, dropout_p: float = 0.0, is_causal: bool = False,
                       scale: Optional[float] = None, enable_gqa: bool = False,
                       attention_kwargs: Optional[Dict[str, Any]] = None) -> torch.Tensor:
    """Drop-in for ``F.scaled_dot_product_attention`` (patched at patches/__init__.py:55-58)."""
    attention_kwargs = attention_kwargs or {}
    name, fn = _AttentionProviderRegistry.get_active_provider()
    kwargs = {"query": query, "key": key, "value": value, "attn_mask": attn_mask, "dropout_p": dropout_p,
              "is_causal": is_causal, "scale": scale, "enable_gqa": enable_gqa, **attention_kwargs}
    if _AttentionProviderRegistry._checks_enabled:
        for check in _AttentionProviderRegistry._constraints.get(name):
            check(**kwargs)
    kwargs = {k: v for k, v in kwargs.items() if k in _AttentionProviderRegistry._supported_arg_names[name]}
    return fn(**kwargs)


HEAD_DIMS = (64, 128)  # head dimensions the kernels are built for


def _check_head_dim(query, key, value):
    d = query.shape[-1]
    if d not in HEAD_DIMS or key.shape[-1] != d or value.shape[-1] != d:
        raise ValueError(f"b200 attention supports head_dim {' or '.join(map(str, HEAD_DIMS))} with q, k and v equal; "
                         f"got q {query.shape[-1]}, k {key.shape[-1]}, v {value.shape[-1]}")


def _check_b200(query, key, value, attn_mask=None, dropout_p=0.0, is_causal=False, enable_gqa=False, **_):
    if not (query.is_cuda and key.is_cuda and value.is_cuda):
        raise ValueError("b200 attention needs CUDA tensors")
    _check_head_dim(query, key, value)
    if query.dtype != torch.bfloat16:
        raise ValueError("b200 attention computes in bf16")
    if dropout_p != 0.0 or is_causal or enable_gqa:
        raise ValueError("b200 attention: dropout / causal / gqa are not on the DiT hot path")


# Finite mask values at or below this floor mask their key like -inf.  finfo(bf16 / float32).min is how -inf is often
# spelled so that a fully masked row gives no NaN; it is also beyond what the kernel accepts (bias * log2(e) would
# overflow fp32).  A sample whose every key is at or below the floor therefore gets what a bool mask gives it: out = 0
# and zero gradients.  torch's math SDPA returns the mean of V there, because the bias absorbs the scores in rounding;
# its gradients are those of a different function, and the kernel's backward, which rebuilds P from lse, cannot follow
# them (lse has absorbed the scores and log(Sk) as well).
KEY_BIAS_FLOOR = -2.0 ** 120


def mask_to_key_bias(attn_mask: torch.Tensor, batch: int, keys: int) -> torch.Tensor:
    """A key-only SDPA mask -> the kernel's fp32 key bias [batch, keys], on the mask's device.

    The LTX cross-attention mask is an additive key bias broadcast over heads and queries: [B|1, 1|H, 1, Sk] (fewer
    dimensions are read as [B, Sk] or [Sk]).  A bool mask keeps the keys where it is True and gives the others -inf; a
    float mask is added to the scores, and its values at or below KEY_BIAS_FLOOR become -inf.

    Each sample's bias is then shifted so that its largest finite value is 0.  Softmax does not change under a constant
    shift of every key's score, but the kernel's backward does: it rebuilds P as exp(score + bias - lse), and with a
    large common offset (a sample masked everywhere with -1e9, say) lse absorbs the scores and P comes back wrong.

    The kernel takes one bias per sample, so a mask that differs between heads raises ValueError.  A mask expanded
    over heads (stride 0) is accepted without looking at its values; any other [B, H, 1, Sk] mask is compared across
    heads, which waits for the device."""
    m = attn_mask
    while m.ndim < 4:
        m = m.unsqueeze(1) if m.ndim > 1 else m.unsqueeze(0)
    if m.shape[2] != 1:
        raise ValueError("b200 attention supports key-only (query-broadcast) additive masks")
    if m.shape[1] != 1 and m.stride(1) != 0 and not bool((m == m[:, :1]).all()):
        raise ValueError("b200 attention takes one key bias per sample: the mask must be the same for every head")
    m = m[:, 0, 0, :]
    neg_inf = torch.tensor(float("-inf"), device=m.device)
    if m.dtype == torch.bool:
        kb = torch.where(m, torch.zeros((), device=m.device), neg_inf)
    else:
        kb = m.to(torch.float32)
        kb = torch.where(kb <= KEY_BIAS_FLOOR, neg_inf, kb)
        top = kb.amax(-1, keepdim=True)
        kb = kb - torch.where(torch.isinf(top), torch.zeros_like(top), top)
        kb = torch.where(kb <= KEY_BIAS_FLOOR, neg_inf, kb)
    return kb.expand(batch, keys).contiguous()


class _B200Attention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, key_bias, scale):
        B, H, Sq, d = q.shape
        Sk = k.shape[2]
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        out = torch.empty(B, Sq, H * d, dtype=torch.bfloat16, device=q.device)
        lse = torch.empty(B, H, Sq, dtype=torch.float32, device=q.device)
        ops.attn_fwd(q, k, v, key_bias, out, lse, B, H, Sq, Sk, scale, head_dim=d)
        ctx.save_for_backward(q, k, v, out, lse, key_bias if key_bias is not None else torch.empty(0, device=q.device))
        ctx.scale = scale
        ctx.has_bias = key_bias is not None
        return out.view(B, Sq, H, d).transpose(1, 2)

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse, kb = ctx.saved_tensors
        B, H, Sq, d = q.shape
        Sk = k.shape[2]
        d_tok = dout.transpose(1, 2).reshape(B, Sq, H * d).to(torch.bfloat16).contiguous()
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        delta = torch.empty(ops.attn_bwd_ws_floats(B, H, Sq, Sk, head_dim=d), dtype=torch.float32, device=q.device)
        ops.attn_bwd(q, k, v, kb if ctx.has_bias else None, out, d_tok, lse, delta, dq, dk, dv, B, H, Sq, Sk, ctx.scale,
                     head_dim=d)
        return dq, dk, dv, None, None


@_AttentionProviderRegistry.register(AttentionProvider.B200, constraints=[_check_b200], supports_cp=False)
def _b200_attention(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor,
                    attn_mask: Optional[torch.Tensor] = None, dropout_p: float = 0.0, is_causal: bool = False,
                    scale: Optional[float] = None, enable_gqa: bool = False) -> torch.Tensor:
    if dropout_p != 0.0 or is_causal or enable_gqa:
        raise ValueError("b200 attention: dropout / causal / gqa unsupported")
    _check_head_dim(query, key, value)
    key_bias = None if attn_mask is None else mask_to_key_bias(attn_mask, query.shape[0], key.shape[2])
    s = scale if scale is not None else 1.0 / math.sqrt(query.shape[-1])
    return _B200Attention.apply(query, key, value, key_bias, float(s))
