"""Thin tensor->pointer wrappers over the libb2d C ABI (include/b2d.h).  PyTorch only supplies device memory and the
current stream; all arithmetic happens in the sm_90a kernels.  No fallbacks: a missing library or a non-CUDA tensor
raises."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import lib as _l
from .lib import GemmDesc, check

EPI_STORE, EPI_GELU, EPI_SILU, EPI_GATE_RES, EPI_MUL_DGELU, EPI_F32_ATOMIC, EPI_F32_ATOMIC_T, EPI_F32_STORE = range(8)

LAUNCH_COUNT = 0  # number of libb2d kernels launched (bench.py reports it as gpu_launches)
TIMING = False    # when True every wrapper brackets its launch with CUDA events on the current stream
KERNEL_TIMES = {}  # tag -> [(start_event, end_event), ...]
CONTEXT = ""      # optional call-site label set by the model (profiling only): tags become "<CONTEXT>/<tag>"


class _Timed:
    __slots__ = ("tag", "e0")

    def __init__(self, tag):
        self.tag = tag

    def __enter__(self):
        if TIMING:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *a):
        if TIMING:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            KERNEL_TIMES.setdefault(f"{CONTEXT}/{self.tag}" if CONTEXT else self.tag, []).append((self.e0, e1))


def collect_kernel_times():
    """{tag: (total_ms, launches)} — call after torch.cuda.synchronize()."""
    return {k: (sum(a.elapsed_time(b) for a, b in v), len(v)) for k, v in KERNEL_TIMES.items()}


def _ptr(t: Optional[torch.Tensor]):
    if t is None:
        return None
    if not t.is_cuda:
        raise _l.B2DError("libb2d ops need CUDA tensors (there is no CPU fallback)")
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _count(n=1):
    global LAUNCH_COUNT
    LAUNCH_COUNT += n


def gemm(A: torch.Tensor, B: torch.Tensor, out: torch.Tensor, *, M: int, N: int, K: int, lda=None, ldb=None, ldc=None,
         a_mn=False, b_mn=False, A2=None, B2=None, K2=0, lda2=None, ldb2=None, a2_group_n=0, splits=1, batch=1,
         a_boff=(0, 0), b_boff=(0, 0), c_boff=0, epi=EPI_STORE, alpha=1.0, out2=None, ldc2=None, bias=None, res=None,
         ldres=None, aux=None, ldaux=None, gate_table=None, gate_temb=None, gate2_table=None, gate2_temb=None,
         temb_stride=0, rows_per_sample=0, block_n=0, max_ctas=0, a2_boff_row=0, b2_boff_row=0, bias_boff=0,
         cta_pair=0, tag="gemm"):
    """C = epilogue(alpha * (opA(A) opB(B)^T + A2 B2^T)).  See include/b2d.h b2d_gemm_desc."""
    d = GemmDesc()
    d.A = A.data_ptr(); d.lda = lda if lda is not None else A.stride(0)
    d.B = B.data_ptr(); d.ldb = ldb if ldb is not None else B.stride(0)
    if K2:
        d.A2 = A2.data_ptr(); d.lda2 = lda2 if lda2 is not None else A2.stride(0)
        d.B2 = B2.data_ptr(); d.ldb2 = ldb2 if ldb2 is not None else B2.stride(0)
    d.M, d.N, d.K, d.K2 = M, N, K, K2
    d.a_mn_major, d.b_mn_major = int(a_mn), int(b_mn)
    d.a2_group_n = a2_group_n
    d.splits, d.batch = splits, batch
    d.a_boff_row, d.a_boff_col = a_boff
    d.b_boff_row, d.b_boff_col = b_boff
    d.c_boff = c_boff
    d.epi = epi
    d.alpha = alpha
    d.out = out.data_ptr(); d.ldc = ldc if ldc is not None else out.stride(0)
    if out2 is not None:
        d.out2 = out2.data_ptr(); d.ldc2 = ldc2 if ldc2 is not None else out2.stride(0)
    if bias is not None:
        d.bias = bias.data_ptr()
    if res is not None:
        d.res = res.data_ptr(); d.ldres = ldres if ldres is not None else res.stride(0)
    if aux is not None:
        d.aux = aux.data_ptr(); d.ldaux = ldaux if ldaux is not None else aux.stride(0)
    # each pointer on its own: the library, not this wrapper, rejects a gate table without its temb rows
    for name, t in (("gate_table", gate_table), ("gate_temb", gate_temb), ("gate2_table", gate2_table),
                    ("gate2_temb", gate2_temb)):
        if t is not None:
            setattr(d, name, t.data_ptr())
    d.temb_stride = temb_stride
    d.rows_per_sample = rows_per_sample
    d.block_n = block_n
    d.max_ctas = max_ctas
    d.a2_boff_row, d.b2_boff_row, d.bias_boff = a2_boff_row, b2_boff_row, bias_boff
    d.cta_pair = cta_pair
    with _Timed(tag):
        check(_l.load().b2d_gemm(C.byref(d), _stream()), "gemm")
    _count()
    return out


SPLITK_MAX = 16  # B2D_SPLITK_MAX


def splitk_reduce_bf16(part, out, splits, M, N, alpha=1.0, ldc=None):
    """out[:M, :N] (bf16, leading dimension ldc, default N) = alpha * the sum of part[0..splits) (fp32 [splits, M, N])
    in slice order."""
    with _Timed("splitk_reduce"):
        check(_l.load().b2d_splitk_reduce_bf16(_ptr(part), int(splits), int(M), int(N), C.c_float(alpha), _ptr(out),
                                               C.c_int64(ldc if ldc is not None else N), _stream()),
              "splitk_reduce_bf16")
    _count()
    return out


def norm_modulate_fwd(x, y, shift_tab, shift_emb, scale_tab, scale_emb, emb_stride, rows, D, rows_per_sample, eps,
                      layer_norm=False):
    with _Timed("norm_modulate_fwd"):
        check(_l.load().b2d_norm_modulate_fwd(_ptr(x), _ptr(y), _ptr(shift_tab), _ptr(shift_emb), _ptr(scale_tab),
                                              _ptr(scale_emb), C.c_int64(emb_stride), rows, D, rows_per_sample,
                                              C.c_float(eps), int(layer_norm), _stream()), "norm_modulate_fwd")
    _count()
    return y


def norm_modulate_bwd(dy, x, dx_in, dx_out, scale_tab, scale_emb, emb_stride, rows, D, rows_per_sample, eps,
                      layer_norm=False, gate2_tab=None, gate2_emb=None, out2=None):
    with _Timed("norm_modulate_bwd"):
        check(_l.load().b2d_norm_modulate_bwd(_ptr(dy), _ptr(x), _ptr(dx_in), _ptr(dx_out), _ptr(scale_tab),
                                              _ptr(scale_emb), _ptr(gate2_tab), _ptr(gate2_emb), _ptr(out2),
                                              C.c_int64(emb_stride), rows, D, rows_per_sample, C.c_float(eps),
                                              int(layer_norm), _stream()), "norm_modulate_bwd")
    _count()
    return dx_out


def colscale(x, out, tab, emb, emb_stride, rows, D, rows_per_sample):
    with _Timed("colscale"):
        check(_l.load().b2d_colscale(_ptr(x), _ptr(out), _ptr(tab), _ptr(emb), C.c_int64(emb_stride), rows, D,
                                     rows_per_sample, _stream()), "colscale")
    _count()
    return out


def qknorm_rope_fwd(src, ld, col_off, weight, cos, sin, dst, B, S, H, norm, eps, *, head_dim=64):
    if head_dim != 64:  # the single-segment entry point is head_dim 64: use the one-segment form of the general one
        if norm and weight is None:
            raise _l.B2DError("qknorm_rope_fwd: norm needs a weight")
        qkv_norm_rope_fwd(src, ld, col_off, (weight if norm else None,), int(cos is not None), cos, sin, (dst,), B, S, H,
                          eps, head_dim=head_dim)
        return dst
    with _Timed("qknorm_rope_fwd"):
        check(_l.load().b2d_qknorm_rope_fwd(_ptr(src), C.c_int64(ld), C.c_int64(col_off), _ptr(weight), _ptr(cos),
                                            _ptr(sin), _ptr(dst), B, S, H, int(norm), C.c_float(eps), _stream()),
              "qknorm_rope_fwd")
    _count()
    return dst


def qknorm_rope_bwd(dyh, x, ld, col_off, weight, cos, sin, dx, ld_dx, dx_col_off, B, S, H, norm, eps, *, head_dim=64):
    if head_dim != 64:
        if norm and weight is None:
            raise _l.B2DError("qknorm_rope_bwd: norm needs a weight")
        return qkv_norm_rope_bwd((dyh,), x, ld, col_off, (weight if norm else None,), int(cos is not None), cos, sin, dx,
                                 ld_dx, dx_col_off, B, S, H, eps, head_dim=head_dim)
    with _Timed("qknorm_rope_bwd"):
        check(_l.load().b2d_qknorm_rope_bwd(_ptr(dyh), _ptr(x), C.c_int64(ld), C.c_int64(col_off), _ptr(weight),
                                            _ptr(cos), _ptr(sin), _ptr(dx), C.c_int64(ld_dx), C.c_int64(dx_col_off), B,
                                            S, H, int(norm), C.c_float(eps), _stream()), "qknorm_rope_bwd")
    _count()
    return dx


def _qkv_entry(direction, head_dim, per_head):
    """-> (entry point, its head-dimension argument).  head_dim 64 without per-head RoPE keeps the entry point without
    it (the same launcher behind both)."""
    if head_dim == 64 and not per_head:
        return getattr(_l.load(), "b2d_qkv_norm_rope_" + direction), ()
    return getattr(_l.load(), f"b2d_qkv_norm_rope_{'ph' if per_head else 'hd'}_{direction}"), (int(head_dim),)


def qkv_norm_rope_fwd(src, ld, col_off, weights, rope_mask, cos, sin, dsts, B, S, H, eps, rows_per_w=0, w_stride=0, *,
                      head_dim=64, per_head=False):
    """nseg = len(dsts) consecutive D-wide (D = H * head_dim) segments of src rows -> head-split dsts [B, H, S, head_dim]
    in ONE launch (b2d.h); head_dim 64 or 128.  ``per_head``: cos / sin are [S, head_dim / 2], shared by every head."""
    n = len(dsts)
    w = list(weights) + [None] * (3 - n)
    d = list(dsts) + [None] * (3 - n)
    fn, hd = _qkv_entry("fwd", head_dim, per_head)
    with _Timed("qknorm_rope_fwd"):
        check(fn(_ptr(src), C.c_int64(ld), C.c_int64(col_off), n, _ptr(w[0]), _ptr(w[1]), _ptr(w[2]), int(rope_mask),
                 _ptr(cos), _ptr(sin), _ptr(d[0]), _ptr(d[1]), _ptr(d[2]), B, S, H, *hd, C.c_float(eps), int(rows_per_w),
                 C.c_int64(w_stride), _stream()), "qkv_norm_rope_fwd")
    _count()


def qkv_norm_rope_bwd(dys, x, ld, col_off, weights, rope_mask, cos, sin, dx, ld_dx, dx_col_off, B, S, H, eps,
                      rows_per_w=0, w_stride=0, *, head_dim=64, per_head=False):
    n = len(dys)
    w = list(weights) + [None] * (3 - n)
    d = list(dys) + [None] * (3 - n)
    fn, hd = _qkv_entry("bwd", head_dim, per_head)
    with _Timed("qknorm_rope_bwd"):
        check(fn(_ptr(d[0]), _ptr(d[1]), _ptr(d[2]), _ptr(x), C.c_int64(ld), C.c_int64(col_off), n, _ptr(w[0]), _ptr(w[1]),
                 _ptr(w[2]), int(rope_mask), _ptr(cos), _ptr(sin), _ptr(dx), C.c_int64(ld_dx), C.c_int64(dx_col_off), B, S,
                 H, *hd, C.c_float(eps), int(rows_per_w), C.c_int64(w_stride), _stream()), "qkv_norm_rope_bwd")
    _count()
    return dx


def rope_table(cos, sin, F, H, W, D, sf, sh, sw):
    check(_l.load().b2d_rope_table(_ptr(cos), _ptr(sin), F, H, W, D, C.c_float(sf), C.c_float(sh), C.c_float(sw),
                                   _stream()), "rope_table")
    _count()


def rope_table_wan(cos, sin, F, H, W, head_dim, theta=10000.0):
    """Wan's per-head RoPE table (b2d.h b2d_rope_table_wan): cos, sin fp32 [F H W, head_dim / 2] on the post-patch grid."""
    check(_l.load().b2d_rope_table_wan(_ptr(cos), _ptr(sin), F, H, W, head_dim, C.c_double(theta), _stream()),
          "rope_table_wan")
    _count()


def layer_norm_affine_fwd(x, y, weight, bias, rows, D, eps):
    """y = bf16(LayerNorm(x) * weight + bias) with fp32 statistics (diffusers FP32LayerNorm, elementwise_affine)."""
    with _Timed("layer_norm_affine_fwd"):
        check(_l.load().b2d_layer_norm_affine_fwd(_ptr(x), _ptr(y), _ptr(weight), _ptr(bias), rows, D, C.c_float(eps),
                                                  _stream()), "layer_norm_affine_fwd")
    _count()
    return y


def layer_norm_affine_bwd(dy, x, dx_in, dx_out, weight, rows, D, eps, gate2_tab=None, gate2_emb=None, out2=None,
                          emb_stride=0, rows_per_sample=1):
    """dx_out = dx_in + dLayerNorm/dx (dy); optional out2 = dx_out * (gate2_tab + gate2_emb[b])."""
    with _Timed("layer_norm_affine_bwd"):
        check(_l.load().b2d_layer_norm_affine_bwd(_ptr(dy), _ptr(x), _ptr(dx_in), _ptr(dx_out), _ptr(weight),
                                                  _ptr(gate2_tab), _ptr(gate2_emb), _ptr(out2), C.c_int64(emb_stride),
                                                  rows, D, rows_per_sample, C.c_float(eps), _stream()),
              "layer_norm_affine_bwd")
    _count()
    return dx_out


def attn_fwd(q, k, v, key_bias, out, lse, B, H, Sq, Sk, scale, *, head_dim=64):
    """q [B,H,Sq,head_dim], k,v [B,H,Sk,head_dim] -> out [B,Sq,H*head_dim], lse [B,H,Sq]; head_dim 64 or 128."""
    with _Timed("attn_fwd"):
        check(_l.load().b2d_attn_fwd_hd(_ptr(q), _ptr(k), _ptr(v), _ptr(key_bias), _ptr(out), _ptr(lse), B, H, Sq, Sk,
                                        head_dim, C.c_float(scale), _stream()), "attn_fwd")
    _count()
    return out


def attn_bwd_ws_floats(B, H, Sq, Sk, *, head_dim=64):
    """fp32 elements b2d_attn_bwd_hd needs in delta_ws (include/b2d.h)."""
    return 2 * B * H * Sq + (8 * 2 * B * H * Sk * head_dim if Sk <= 512 else 0)


def attn_bwd(q, k, v, key_bias, out, dout, lse, delta_ws, dq, dk, dv, B, H, Sq, Sk, scale, *, head_dim=64):
    need = attn_bwd_ws_floats(B, H, Sq, Sk, head_dim=head_dim)
    if delta_ws.numel() < need:
        raise _l.B2DError(f"attn_bwd workspace too small: {delta_ws.numel()} < {need} floats")
    with _Timed("attn_bwd"):
        check(_l.load().b2d_attn_bwd_hd(_ptr(q), _ptr(k), _ptr(v), _ptr(key_bias), _ptr(out), _ptr(dout), _ptr(lse),
                                        _ptr(delta_ws), _ptr(dq), _ptr(dk), _ptr(dv), B, H, Sq, Sk, head_dim,
                                        C.c_float(scale), _stream()), "attn_bwd")
    if Sk <= 128:
        _count(1)  # single key tile: ONE fused delta/dQ/dK/dV kernel
    else:
        # delta + dK/dV + dQ, plus two fp32->bf16 converts when the few-key-tiles split path runs
        split = (B * H * ((Sk + 127) // 128) < 96) and Sk <= 512 and ((Sq + 63) // 64) >= 8
        _count(5 if split else 3)


def attn_dual_fwd(q, k1, v1, Sk1, k2, v2, Sk2, out, lse1, lse2, B, H, Sq, scale, *, out1=None, out2=None,
                  head_dim=128):
    """Two independent softmaxes of q over (k1, v1) and (k2, v2) in one launch (b2d.h b2d_attn_dual_fwd_hd):
    out = bf16(bf16(O1) + bf16(O2)) [B, Sq, H*head_dim], lse1 / lse2 [B, H, Sq]; out1 / out2 optionally receive the
    branch outputs bf16(O1) / bf16(O2)."""
    with _Timed("attn_dual_fwd"):
        check(_l.load().b2d_attn_dual_fwd_hd(_ptr(q), _ptr(k1), _ptr(v1), int(Sk1), _ptr(k2), _ptr(v2), int(Sk2),
                                             _ptr(out), _ptr(lse1), _ptr(lse2), _ptr(out1), _ptr(out2), B, H, Sq,
                                             head_dim, C.c_float(scale), _stream()), "attn_dual_fwd")
    _count()
    return out


def attn_dual_bwd_ws_floats(B, H, Sq, Sk1, *, head_dim=128):
    """fp32 elements b2d_attn_dual_bwd_hd needs in ws (include/b2d.h): attn_bwd's for context 1, then context 2's
    delta and -lse log2e."""
    return attn_bwd_ws_floats(B, H, Sq, Sk1, head_dim=head_dim) + 2 * B * H * Sq


def attn_dual_bwd(q, k1, v1, Sk1, k2, v2, Sk2, out1, out2, dout, lse1, lse2, ws, dq, dk1, dv1, B, H, Sq, scale, *,
                  head_dim=128):
    """dq over both contexts (one fp32 accumulator) and dk1 / dv1 (b2d.h b2d_attn_dual_bwd_hd); no dk2 / dv2."""
    need = attn_dual_bwd_ws_floats(B, H, Sq, Sk1, head_dim=head_dim)
    if ws.numel() < need:
        raise _l.B2DError(f"attn_dual_bwd workspace too small: {ws.numel()} < {need} floats")
    with _Timed("attn_dual_bwd"):
        check(_l.load().b2d_attn_dual_bwd_hd(_ptr(q), _ptr(k1), _ptr(v1), int(Sk1), _ptr(k2), _ptr(v2), int(Sk2),
                                             _ptr(out1), _ptr(out2), _ptr(dout), _ptr(lse1), _ptr(lse2), _ptr(ws),
                                             _ptr(dq), _ptr(dk1), _ptr(dv1), B, H, Sq, head_dim, C.c_float(scale),
                                             _stream()), "attn_dual_bwd")
    # delta 1, dK/dV (plus its reduce when the query range is split), delta 2, dQ
    split = (B * H * ((Sk1 + 127) // 128) < 96) and Sk1 <= 512 and ((Sq + 63) // 64) >= 8
    _count(5 if split else 4)


def prep_noise_pack(latents, noise, mean, std, sigma, sigma_ff, x_t, target, B, Cc, F, HW):
    check(_l.load().b2d_prep_noise_pack(_ptr(latents), _ptr(noise), _ptr(mean), _ptr(std), _ptr(sigma),
                                        _ptr(sigma_ff), _ptr(x_t), _ptr(target), B, Cc, F, HW, _stream()), "prep")
    _count()


def prep_posterior_noise_pack(moments, eps, noise, mean, std, sigma, sigma_ff, x_t, target, B, Cc, F, HW,
                              latents_out=None):
    """prep_noise_pack on the latent sampled from VAE moments [B, 2 Cc, F, HW] with eps [B, Cc, F, HW];
    latents_out (optional, [B, Cc, F, HW] bf16) receives that sample."""
    check(_l.load().b2d_prep_posterior_noise_pack(_ptr(moments), _ptr(eps), _ptr(noise), _ptr(mean), _ptr(std),
                                                  _ptr(sigma), _ptr(sigma_ff), _ptr(x_t), _ptr(target),
                                                  _ptr(latents_out), B, Cc, F, HW, _stream()), "prep_posterior")
    _count()


def wan_prep(moments, eps, noise, mean, std, sigma, x_t, target, B, Cc, F, H, W):
    """Wan's step prologue (b2d.h b2d_wan_prep): posterior sample of the normalised moments, x_t patchified in the
    Conv3d order, target in proj_out's order."""
    check(_l.load().b2d_wan_prep(_ptr(moments), _ptr(eps), _ptr(noise), _ptr(mean), _ptr(std), _ptr(sigma), _ptr(x_t),
                                 _ptr(target), B, Cc, F, H, W, _stream()), "wan_prep")
    _count()


def wan_i2v_prep(moments, cond_moments, cond_mask, eps, noise, mean, std, sigma, x_in, target, B, Cc, Cm, F, H, W):
    """Wan image-to-video prologue (b2d.h b2d_wan_i2v_prep): wan_prep's x_t, written with the mask and the normalised
    condition mean as the patchified transformer input cat([x_t, mask, condition]) [B, F (H/2) (W/2), 4 (2 Cc + Cm)].
    Every tensor operand must be contiguous: the kernel indexes them as dense arrays, and the reference's own mask is a
    transposed view."""
    for name, t in (("moments", moments), ("cond_moments", cond_moments), ("cond_mask", cond_mask), ("eps", eps),
                    ("noise", noise), ("mean", mean), ("std", std), ("sigma", sigma), ("x_in", x_in),
                    ("target", target)):
        if t is not None and not t.is_contiguous():
            raise _l.B2DError(f"wan_i2v_prep: {name} must be contiguous (call .contiguous())")
    check(_l.load().b2d_wan_i2v_prep(_ptr(moments), _ptr(cond_moments), _ptr(cond_mask), _ptr(eps), _ptr(noise),
                                     _ptr(mean), _ptr(std), _ptr(sigma), _ptr(x_in), _ptr(target), B, Cc, Cm, F, H, W,
                                     _stream()), "wan_i2v_prep")
    _count()


def gelu_erf(x, y, n):
    """y[:n] = bf16(exact GELU(x[:n])) in fp32 (b2d.h b2d_gelu_erf); bf16 in and out."""
    with _Timed("gelu_erf"):
        check(_l.load().b2d_gelu_erf(_ptr(x), _ptr(y), C.c_int64(n), _stream()), "gelu_erf")
    _count()
    return y


PATCH_CONV, PATCH_OUT = 0, 1  # channel orders of a patchified row: Conv3d weight's, proj_out's


def patch_permute(src, dst, B, Cc, F, H, W, order, unpatchify):
    """Exact permute between [B, Cc, F, H, W] and [B, F (H/2) (W/2), 4 Cc] (b2d.h b2d_patch_permute)."""
    with _Timed("patch_permute"):
        check(_l.load().b2d_patch_permute(_ptr(src), _ptr(dst), B, Cc, F, H, W, int(order), int(bool(unpatchify)),
                                          _stream()), "patch_permute")
    _count()
    return dst


def loss_mse(pred, target, weight, loss_scale, loss_out, dpred, partial_ws, B, per_sample):
    with _Timed("loss"):
        check(_l.load().b2d_loss_mse(_ptr(pred), _ptr(target), _ptr(weight), C.c_float(loss_scale), _ptr(loss_out),
                                     _ptr(dpred), _ptr(partial_ws), B, C.c_int64(per_sample), _stream()), "loss_mse")
    _count(2)


def timestep_sinusoid(t, out, n):
    check(_l.load().b2d_timestep_sinusoid(_ptr(t), _ptr(out), n, _stream()), "timestep_sinusoid")
    _count()


def cast_f32_bf16(src, dst, n, scale=1.0):
    with _Timed("cast"):
        check(_l.load().b2d_cast_f32_bf16(_ptr(src), _ptr(dst), C.c_int64(n), C.c_float(scale), _stream()), "cast")
    _count()


FP8_FORMATS = {torch.float8_e4m3fn: 0, torch.float8_e5m2: 1}


def upcast_fp8_bf16(src, dst, n):
    """dst[:n] (bf16) <- src[:n] (float8_e4m3fn or float8_e5m2), exactly."""
    fmt = FP8_FORMATS.get(src.dtype)
    if fmt is None or dst.dtype != torch.bfloat16:
        raise _l.B2DError(f"upcast_fp8_bf16: {src.dtype} -> {dst.dtype}; needs a float8 source and a bf16 destination")
    with _Timed("upcast"):
        check(_l.load().b2d_upcast_fp8_bf16(_ptr(src), _ptr(dst), C.c_int64(n), fmt, _stream()), "upcast_fp8_bf16")
    _count()


def cfg_euler_step(pred, latents, x_next, B, n, guided, guidance, dt):
    """One denoising step (b2d.h b2d_cfg_euler_step): latents [B, n] fp32 += dt[0] * (u + guidance (c - u)) with
    pred = [u; c] bf16 [2B, n] (``guided``) or v = pred [B, n]; x_next (bf16, as many rows as pred) = bf16(latents)."""
    with _Timed("cfg_euler_step"):
        check(_l.load().b2d_cfg_euler_step(_ptr(pred), _ptr(latents), _ptr(x_next), int(B), C.c_int64(n), int(bool(guided)),
                                           C.c_float(guidance), _ptr(dt), _stream()), "cfg_euler_step")
    _count()


def cfg_euler_step_cond(pred, latents, x_next, B, n, n_cond, guided, guidance, dt):
    """cfg_euler_step on the elements n_cond .. n of each sample (b2d.h b2d_cfg_euler_step_cond): the first n_cond, the
    conditioning frame, keep their latents and x_next, and pred is not read there."""
    with _Timed("cfg_euler_step_cond"):
        check(_l.load().b2d_cfg_euler_step_cond(_ptr(pred), _ptr(latents), _ptr(x_next), int(B), C.c_int64(n),
                                                C.c_int64(n_cond), int(bool(guided)), C.c_float(guidance), _ptr(dt),
                                                _stream()), "cfg_euler_step_cond")
    _count()


def sumsq(x, n, out, partial_ws):
    with _Timed("sumsq"):
        check(_l.load().b2d_sumsq(_ptr(x), C.c_int64(n), _ptr(out), _ptr(partial_ws), _stream()), "sumsq")
    _count(2)


def adamw_clip(p, g, m, v, n, sumsq_t, max_norm, lr, beta1, beta2, eps, wd, step, grad_div=1.0):
    with _Timed("adamw"):
        check(_l.load().b2d_adamw_clip(_ptr(p), _ptr(g), _ptr(m), _ptr(v), C.c_int64(n), _ptr(sumsq_t),
                                       C.c_float(max_norm), C.c_float(lr), C.c_float(beta1), C.c_float(beta2),
                                       C.c_float(eps), C.c_float(wd), int(step), C.c_float(grad_div), _stream()), "adamw")
    _count()
