"""GPU: attention at head_dim 128 (Wan-2.1, HunyuanVideo) against fp64 references: the reference's known-answer recipe
through the provider hook, every dispatch branch of the forward and the backward, the Wan self- and cross-attention
shapes next to torch's own bf16 SDPA, output bounds and run-to-run determinism; and the refusal of other head
dimensions."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from _util import check_sentinel, rel_err, rnd, sentinel_buffer, window

pytestmark = pytest.mark.gpu

D = 128
SHAPES = [(1, 32, 2688, 2688, False), (2, 4, 2688, 128, True), (1, 2, 200, 72, True), (1, 2, 128, 128, False),
          (1, 3, 1, 1, False), (2, 2, 130, 257, True), (1, 32, 2688, 128, True), (5, 32, 300, 128, True),
          (3, 2, 1000, 100, False), (1, 2, 1000, 300, True), (1, 1, 640, 512, False)]


def _math_sdpa(q, k, v, mask=None):
    with torch.nn.attention.sdpa_kernel(torch.nn.attention.SDPBackend.MATH):
        return F.scaled_dot_product_attention(q, k, v, attn_mask=mask)


def _key_bias(B, Sk):
    lens = torch.randint(1, Sk + 1, (B,), device="cuda")
    return ((1 - (torch.arange(Sk, device="cuda")[None] < lens[:, None]).float()) * -10000.0).contiguous()


def _ref64(q, k, v, kb, scale, dout, chunk=1024):
    """fp64 attention and its gradients, query block by query block (dK, dV accumulated over the blocks).
    q [B,H,Sq,d], k/v [B,H,Sk,d], kb [B,Sk] or None, dout [B,H,Sq,d] -> out, lse, dq, dk, dv (fp64)."""
    q, k, v, dout = q.double(), k.double(), v.double(), dout.double()
    bias = kb.double()[:, None, None, :] if kb is not None else 0.0
    out, lse, dq = torch.empty_like(q), torch.empty(q.shape[:-1], dtype=torch.float64, device=q.device), torch.empty_like(q)
    dk, dv = torch.zeros_like(k), torch.zeros_like(v)
    for i in range(0, q.shape[2], chunk):
        qi, gi = q[:, :, i:i + chunk], dout[:, :, i:i + chunk]
        s = qi @ k.transpose(-1, -2) * scale + bias
        lse[:, :, i:i + chunk] = torch.logsumexp(s, -1)
        p = torch.softmax(s, -1)
        del s
        oi = p @ v
        out[:, :, i:i + chunk] = oi
        dv += p.transpose(-1, -2) @ gi
        ds = p * (gi @ v.transpose(-1, -2) - (gi * oi).sum(-1, keepdim=True))
        del p
        dq[:, :, i:i + chunk] = ds @ k * scale
        dk += ds.transpose(-1, -2) @ qi * scale
    return out, lse, dq, dk, dv


def _run(q, k, v, kb, scale, dout_tok, head_dim=D, ws_fill=0.0):
    """fwd + bwd through ops at head_dim; returns out [B,H,Sq,d] view, lse, dq, dk, dv."""
    from finetrainers_b200 import ops
    B, H, Sq, d = q.shape
    Sk = k.shape[2]
    out = torch.zeros(B, Sq, H * d, device="cuda", dtype=torch.bfloat16)
    lse = torch.zeros(B, H, Sq, device="cuda")
    ops.attn_fwd(q, k, v, kb, out, lse, B, H, Sq, Sk, scale, head_dim=head_dim)
    dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    ws = torch.full((ops.attn_bwd_ws_floats(B, H, Sq, Sk, head_dim=head_dim),), ws_fill, device="cuda")
    ops.attn_bwd(q, k, v, kb, out, dout_tok, lse, ws, dq, dk, dv, B, H, Sq, Sk, scale, head_dim=head_dim)
    return out, lse, dq, dk, dv


def test_reference_attention_kat_d128_through_provider_hook():
    """The reference's known-answer recipe (randn bf16, torch seed 0, forward vs math SDPA at atol 5e-3, backward of
    output.mean() at atol 1e-3) at head_dim 128, with the default scale 1/sqrt(128)."""
    from finetrainers_b200.attention import attention_dispatch, attention_provider, AttentionProvider
    torch.manual_seed(0)
    q, k, v = (torch.randn(2, 8, 256, D, device="cuda", dtype=torch.bfloat16) for _ in range(3))
    ref = _math_sdpa(q, k, v)
    with attention_provider(AttentionProvider.B200):
        out = attention_dispatch(q, k, v)
    assert out.shape == ref.shape
    assert (out.float() - ref.float()).abs().max().item() < 5e-3
    grads = []
    for fn in (lambda a, b, c: _math_sdpa(a, b, c), lambda a, b, c: attention_dispatch(a, b, c)):
        qq, kk, vv = (t.clone().requires_grad_(True) for t in (q, k, v))
        fn(qq, kk, vv).mean().backward()
        grads.append((qq.grad, kk.grad, vv.grad))
    for a, b in zip(*grads):
        assert (a.float() - b.float()).abs().max().item() < 1e-3


def test_provider_d128_mask_and_gradients():
    """The provider at d = 128 with a boolean key mask [B,1,1,Sk]: output and gradients against fp64."""
    from finetrainers_b200.attention import attention_dispatch
    torch.manual_seed(3)
    B, H, Sq, Sk = 2, 4, 300, 200
    q, k, v = rnd(B, H, Sq, D), rnd(B, H, Sk, D), rnd(B, H, Sk, D)
    keep = torch.arange(Sk, device="cuda")[None] < torch.tensor([[150], [200]], device="cuda")
    qq, kk, vv = (t.clone().requires_grad_(True) for t in (q, k, v))
    out = attention_dispatch(qq, kk, vv, attn_mask=keep[:, None, None, :])
    g = rnd(B, H, Sq, D)
    out.backward(g)
    kb = torch.zeros(B, Sk, device="cuda").masked_fill(~keep, float("-inf"))
    ro, _, rdq, rdk, rdv = _ref64(q, k, v, kb, D ** -0.5, g)
    assert rel_err(out, ro) < 1e-2
    assert rel_err(qq.grad, rdq, 1e-2) < 2e-2 and rel_err(kk.grad, rdk, 1e-2) < 2e-2 and rel_err(vv.grad, rdv, 1e-2) < 2e-2


@pytest.mark.parametrize("B,H,Sq,Sk,bias", SHAPES)
def test_attention_d128_fwd_bwd_shapes(B, H, Sq, Sk, bias):
    """Every dispatch branch at d = 128: long keys (full and ragged tiles, with and without key bias), one key tile (one
    or several query tiles per head), Sq = 1, and 128 < Sk <= 512 with few heads (the split dK/dV pass)."""
    torch.manual_seed(0)
    q, k, v = rnd(B, H, Sq, D), rnd(B, H, Sk, D), rnd(B, H, Sk, D)
    kb = _key_bias(B, Sk) if bias else None
    dout = rnd(B, Sq, H * D)
    out, lse, dq, dk, dv = _run(q, k, v, kb, 0.125, dout)
    ro, rl, rdq, rdk, rdv = _ref64(q, k, v, kb, 0.125, dout.unflatten(2, (H, D)).transpose(1, 2))
    assert rel_err(out, ro.transpose(1, 2).flatten(2)) < 1e-2
    assert (lse.double() - rl).abs().max().item() < 1e-3
    assert rel_err(dq, rdq, 1e-2) < 2e-2 and rel_err(dk, rdk, 1e-2) < 2e-2 and rel_err(dv, rdv, 1e-2) < 2e-2


def _sdpa_bf16(q, k, v, scale, g):
    """torch's own bf16 attention (flash, else cuDNN) forward and backward: (backend, out, dq, dk, dv)."""
    from torch.nn.attention import SDPBackend, sdpa_kernel
    for name, be in (("flash", SDPBackend.FLASH_ATTENTION), ("cudnn", SDPBackend.CUDNN_ATTENTION)):
        try:
            qq, kk, vv = (t.clone().requires_grad_(True) for t in (q, k, v))
            with sdpa_kernel(be):
                o = F.scaled_dot_product_attention(qq, kk, vv, scale=scale)
                o.backward(g)
            return name, o.detach(), qq.grad, kk.grad, vv.grad
        except RuntimeError:
            continue
    pytest.skip("neither the flash nor the cuDNN SDPA backend is available")


@pytest.mark.parametrize("Sk,heads_checked", [(32760, 2), (512, 12)], ids=["self", "cross"])
def test_attention_d128_wan_shapes(Sk, heads_checked):
    """Wan-2.1 T2V-1.3B: 12 heads x 128 over 32760 latent tokens, self-attention and the 512-token text
    cross-attention (split dK/dV path).  Against a chunked fp64 reference on `heads_checked` heads: the fixed tolerances
    of the other tests, and a max error at most 2x that of torch's bf16 SDPA on the same inputs."""
    torch.manual_seed(4)
    B, H, Sq = 1, 12, 32760
    scale = D ** -0.5
    q, k, v = rnd(B, H, Sq, D), rnd(B, H, Sk, D), rnd(B, H, Sk, D)
    dout = rnd(B, Sq, H * D)
    out, lse, dq, dk, dv = _run(q, k, v, None, scale, dout)
    n = heads_checked
    g = dout.unflatten(2, (H, D)).transpose(1, 2)[:, :n].contiguous()
    ref = _ref64(q[:, :n], k[:, :n], v[:, :n], None, scale, g)
    got = (out.unflatten(2, (H, D)).transpose(1, 2)[:, :n], lse[:, :n], dq[:, :n], dk[:, :n], dv[:, :n])
    assert rel_err(got[0], ref[0]) < 1e-2
    assert (got[1].double() - ref[1]).abs().max().item() < 1e-3
    for a, r in zip(got[2:], ref[2:]):
        assert rel_err(a, r, 1e-2) < 2e-2
    backend, *theirs = _sdpa_bf16(q[:, :n], k[:, :n], v[:, :n], scale, g)
    for name, a, t, r in zip(("out", "dq", "dk", "dv"), got[:1] + got[2:], theirs, ref[:1] + ref[2:]):
        ours_err = (a.double() - r).abs().max().item()
        sdpa_err = (t.double() - r).abs().max().item()
        print(f"Sk={Sk} {name}: kernel max err {ours_err:.3e}, sdpa/{backend} max err {sdpa_err:.3e}")
        assert ours_err <= 2 * sdpa_err, (name, ours_err, sdpa_err, backend)


@pytest.mark.parametrize("growth", [0.02, 0.2])
def test_attention_d128_running_max_growth(growth):
    """Scores that keep growing along the key axis force the online softmax through its rescale path on every tile."""
    from finetrainers_b200 import ops
    torch.manual_seed(2)
    B, H, S = 1, 4, 1024
    q = (torch.randn(B, H, S, D, device="cuda") * 0.3 + 1.0).bfloat16()
    ramp = torch.arange(S, device="cuda", dtype=torch.float32).view(1, 1, S, 1) * growth / D
    k = (torch.randn(B, H, S, D, device="cuda") * 0.3 + ramp).bfloat16()   # q.k grows ~ growth per key
    v = rnd(B, H, S, D)
    out = torch.zeros(B, S, H * D, device="cuda", dtype=torch.bfloat16)
    lse = torch.zeros(B, H, S, device="cuda")
    ops.attn_fwd(q, k, v, None, out, lse, B, H, S, S, 0.125, head_dim=D)
    ro, rl, *_ = _ref64(q, k, v, None, 0.125, torch.zeros_like(q))
    got = out.view(B, S, H, D).transpose(1, 2)
    assert torch.isfinite(got.float()).all()
    assert rel_err(got, ro, 1e-2) < 2e-2
    assert (lse.double() - rl).abs().max().item() < 2e-2


def test_attention_d128_ones_value_gives_ones():
    """Softmax rows sum to one: V = 1 gives O = 1 (ragged key tiles, with a key bias)."""
    from finetrainers_b200 import ops
    torch.manual_seed(1)
    B, H, Sq, Sk = 2, 6, 1000, 700
    q, k = rnd(B, H, Sq, D), rnd(B, H, Sk, D)
    ones = torch.ones(B, H, Sk, D, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(B, Sq, H * D, device="cuda", dtype=torch.bfloat16)
    lse = torch.zeros(B, H, Sq, device="cuda")
    ops.attn_fwd(q, k, ones, _key_bias(B, Sk), out, lse, B, H, Sq, Sk, D ** -0.5, head_dim=D)
    assert (out.float() - 1.0).abs().max().item() < 1e-2


@pytest.mark.parametrize("B,H,Sq,Sk", [(2, 3, 200, 72), (1, 2, 1000, 300), (1, 3, 130, 700)])
def test_attention_d128_writes_only_its_outputs(B, H, Sq, Sk):
    """out, lse, dq, dk and dv sit inside NaN-patterned buffers at ragged Sq and Sk (one key tile, the split dK/dV path,
    long ragged keys): nothing outside them may change."""
    from finetrainers_b200 import ops
    torch.manual_seed(5)
    pad = 4096
    q, k, v = rnd(B, H, Sq, D), rnd(B, H, Sk, D), rnd(B, H, Sk, D)
    kb = _key_bias(B, Sk)
    dout = rnd(B, Sq, H * D)
    bufs, views = {}, {}
    for name, shape, dt in (("out", (B, Sq, H * D), torch.bfloat16), ("lse", (B, H, Sq), torch.float32),
                            ("dq", (B, H, Sq, D), torch.bfloat16), ("dk", (B, H, Sk, D), torch.bfloat16),
                            ("dv", (B, H, Sk, D), torch.bfloat16)):
        n = 1
        for s in shape:
            n *= s
        bufs[name] = sentinel_buffer(n + 2 * pad, dt)
        views[name] = bufs[name][pad:pad + n].view(shape)
    ops.attn_fwd(q, k, v, kb, views["out"], views["lse"], B, H, Sq, Sk, 0.125, head_dim=D)
    ws = torch.zeros(ops.attn_bwd_ws_floats(B, H, Sq, Sk, head_dim=D), device="cuda")
    ops.attn_bwd(q, k, v, kb, views["out"], dout, views["lse"], ws, views["dq"], views["dk"], views["dv"], B, H, Sq, Sk,
                 0.125, head_dim=D)
    torch.cuda.synchronize()
    for name, buf in bufs.items():
        n = views[name].numel()
        check_sentinel(buf, [window(buf, pad, 1, n, n)], name)
        assert torch.isfinite(views[name].float()).all(), name
    ro, rl, rdq, rdk, rdv = _ref64(q, k, v, kb, 0.125, dout.unflatten(2, (H, D)).transpose(1, 2))
    assert rel_err(views["out"], ro.transpose(1, 2).flatten(2)) < 1e-2
    assert rel_err(views["dk"], rdk, 1e-2) < 2e-2 and rel_err(views["dv"], rdv, 1e-2) < 2e-2


@pytest.mark.parametrize("B,H,Sq,Sk", [(1, 2, 1000, 300), (1, 4, 1000, 1000), (1, 12, 4096, 512)])
def test_attention_d128_bitwise_repeatable(B, H, Sq, Sk):
    """Two launches give bit-identical forward and backward results, including the split dK/dV path (the first and
    last shapes), whatever the workspace held before."""
    torch.manual_seed(6)
    q, k, v = rnd(B, H, Sq, D), rnd(B, H, Sk, D), rnd(B, H, Sk, D)
    kb = _key_bias(B, Sk)
    dout = rnd(B, Sq, H * D)
    a = _run(q, k, v, kb, 0.125, dout, ws_fill=0.0)
    b = _run(q, k, v, kb, 0.125, dout, ws_fill=float("nan"))
    for name, x, y in zip(("out", "lse", "dq", "dk", "dv"), a, b):
        assert torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32),
                           y.view(torch.int16) if y.dtype == torch.bfloat16 else y.view(torch.int32)), name


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


@pytest.mark.parametrize("d", [96, 256])
def test_attention_unsupported_head_dim_is_refused(d):
    """head_dim 96 / 256: the provider raises ValueError, ops raises B2DError, and the C entry points return
    B2D_ERR_SHAPE naming the head_dim."""
    from finetrainers_b200 import lib, ops
    from finetrainers_b200.attention import attention_dispatch
    B, H, S = 1, 2, 64
    q, k, v = rnd(B, H, S, d), rnd(B, H, S, d), rnd(B, H, S, d)
    with pytest.raises(ValueError, match="head_dim"):
        attention_dispatch(q, k, v)
    out = torch.zeros(B, S, H * d, device="cuda", dtype=torch.bfloat16)
    lse = torch.zeros(B, H, S, device="cuda")
    with pytest.raises(lib.B2DError, match=f"head_dim {d}"):
        ops.attn_fwd(q, k, v, None, out, lse, B, H, S, S, 0.125, head_dim=d)
    dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    ws = torch.zeros(ops.attn_bwd_ws_floats(B, H, S, S, head_dim=d), device="cuda")
    with pytest.raises(lib.B2DError, match=f"head_dim {d}"):
        ops.attn_bwd(q, k, v, None, out, out, lse, ws, dq, dk, dv, B, H, S, S, 0.125, head_dim=d)
    L = lib.load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    B2D_ERR_SHAPE = -1
    assert L.b2d_attn_fwd_hd(_p(q), _p(k), _p(v), None, _p(out), _p(lse), B, H, S, S, d, C.c_float(0.125), st) == \
        B2D_ERR_SHAPE
    assert f"head_dim {d}" in L.b2d_last_error().decode()
    assert L.b2d_attn_bwd_hd(_p(q), _p(k), _p(v), None, _p(out), _p(out), _p(lse), _p(ws), _p(dq), _p(dk), _p(dv), B, H,
                             S, S, d, C.c_float(0.125), st) == B2D_ERR_SHAPE
    assert (out.view(torch.int16) == 0).all() and (dq.view(torch.int16) == 0).all()
