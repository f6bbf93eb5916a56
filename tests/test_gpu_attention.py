"""GPU: the attention kernel against the reference's own known-answer recipe
(tests/models/attention_dispatch.py:41-149: q,k,v = randn[2,8,256,64] bf16, torch seed 0; forward vs
math SDPA atol 5e-3; backward of output.mean() atol 1e-3), called through the provider hook, plus LTX shapes, ragged
lengths and the masked cross-attention case."""
import pytest
import torch
import torch.nn.functional as F

from _util import rnd, rel_err

pytestmark = pytest.mark.gpu


def _math_sdpa(q, k, v, mask=None):
    with torch.nn.attention.sdpa_kernel(torch.nn.attention.SDPBackend.MATH):
        return F.scaled_dot_product_attention(q, k, v, attn_mask=mask)


def test_reference_attention_kat_through_provider_hook():
    from finetrainers_b200.attention import attention_dispatch, attention_provider, AttentionProvider
    torch.manual_seed(0)
    q, k, v = (torch.randn(2, 8, 256, 64, device="cuda", dtype=torch.bfloat16) for _ in range(3))
    ref = _math_sdpa(q, k, v)
    with attention_provider(AttentionProvider.B200):
        out = attention_dispatch(q, k, v)
    assert out.shape == ref.shape
    assert (out.float() - ref.float()).abs().max().item() < 5e-3
    # backward recipe: output.mean().backward(), compare grads at atol 1e-3.  NB: this is the reference's own recipe and it is
    # nearly vacuous (the gradients of a mean over 262k outputs are O(4e-6), far below the tolerance); it is kept because it
    # is the check the reference holds.  The backward kernels are actually held to 2 % of each gradient's scale against
    # fp32 math attention in test_attention_fwd_bwd_shapes below.
    grads = []
    for fn in (lambda a, b, c: _math_sdpa(a, b, c), lambda a, b, c: attention_dispatch(a, b, c)):
        qq, kk, vv = (t.clone().requires_grad_(True) for t in (q, k, v))
        fn(qq, kk, vv).mean().backward()
        grads.append((qq.grad, kk.grad, vv.grad))
    for a, b in zip(*grads):
        assert (a.float() - b.float()).abs().max().item() < 1e-3


@pytest.mark.parametrize("B,H,Sq,Sk,bias", [(1, 32, 2688, 2688, False), (2, 4, 2688, 128, True), (1, 2, 200, 72, True),
                                            (1, 2, 128, 128, False), (1, 3, 1, 1, False), (2, 2, 130, 257, True),
                                            (1, 32, 2688, 128, True), (5, 32, 300, 128, True), (3, 2, 1000, 100, False),
                                            (1, 2, 1000, 300, True), (1, 1, 640, 512, False)])
def test_attention_fwd_bwd_shapes(B, H, Sq, Sk, bias):
    """Covers every dispatch branch of b2d_attn_fwd_hd / b2d_attn_bwd_hd at head_dim 64: long keys (full and ragged
    tiles, with and without key bias), one key tile (one or several query tiles per head), and 128 < Sk <= 512 with
    few heads (the dK/dV pass split over gridDim.z, partials summed in a fixed order: the last two cases)."""
    from finetrainers_b200 import ops
    torch.manual_seed(0)
    q, k, v = rnd(B, H, Sq, 64), rnd(B, H, Sk, 64), rnd(B, H, Sk, 64)
    kb = None
    if bias:
        lens = torch.randint(1, Sk + 1, (B,), device="cuda")
        kb = ((1 - (torch.arange(Sk, device="cuda")[None] < lens[:, None]).float()) * -10000.0).contiguous()
    out = torch.zeros(B, Sq, H * 64, device="cuda", dtype=torch.bfloat16)
    lse = torch.zeros(B, H, Sq, device="cuda")
    ops.attn_fwd(q, k, v, kb, out, lse, B, H, Sq, Sk, 0.125)
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    am = kb[:, None, None, :] if kb is not None else None
    ref = _math_sdpa(qf, kf, vf, am)
    assert rel_err(out, ref.transpose(1, 2).flatten(2)) < 1e-2
    s = (qf @ kf.transpose(-1, -2)) * 0.125 + (am if am is not None else 0)
    assert (lse - torch.logsumexp(s, -1)).abs().max().item() < 1e-3
    dout = rnd(B, Sq, H * 64)
    ref.backward(dout.float().unflatten(2, (H, 64)).transpose(1, 2))
    dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    ws = torch.zeros(ops.attn_bwd_ws_floats(B, H, Sq, Sk), device="cuda")
    ops.attn_bwd(q, k, v, kb, out, dout, lse, ws, dq, dk, dv, B, H, Sq, Sk, 0.125)
    assert rel_err(dq, qf.grad, 1e-2) < 2e-2 and rel_err(dk, kf.grad, 1e-2) < 2e-2 and rel_err(dv, vf.grad, 1e-2) < 2e-2


def test_attention_properties_full_size():
    """Size-independent properties at the BASELINE shape: softmax rows sum to one (V = 1 => O = 1) and permuting the
    keys/values together leaves the output unchanged (up to bf16 accumulation order)."""
    from finetrainers_b200 import ops
    torch.manual_seed(1)
    B, H, S = 1, 32, 2688
    q, k = rnd(B, H, S, 64), rnd(B, H, S, 64)
    ones = torch.ones(B, H, S, 64, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(B, S, H * 64, device="cuda", dtype=torch.bfloat16)
    lse = torch.zeros(B, H, S, device="cuda")
    ops.attn_fwd(q, k, ones, None, out, lse, B, H, S, S, 0.125)
    assert (out.float() - 1.0).abs().max().item() < 1e-2
    v = rnd(B, H, S, 64)
    ops.attn_fwd(q, k, v, None, out, lse, B, H, S, S, 0.125)
    perm = torch.randperm(S, device="cuda")
    out2 = torch.zeros_like(out)
    lse2 = torch.zeros_like(lse)
    ops.attn_fwd(q, k[:, :, perm].contiguous(), v[:, :, perm].contiguous(), None, out2, lse2, B, H, S, S, 0.125)
    assert (out.float() - out2.float()).abs().max().item() < 2e-2
    assert (lse - lse2).abs().max().item() < 1e-3


@pytest.mark.parametrize("growth", [0.02, 0.2])
def test_attention_fwd_running_max_growth(growth):
    """Scores that keep growing along the key axis force the online softmax through its rescale / exact two-pass path on
    many tiles (the optimistic single pass only holds while the running maximum is stable)."""
    from finetrainers_b200 import ops
    torch.manual_seed(2)
    B, H, S = 1, 4, 1024
    q = (torch.randn(B, H, S, 64, device="cuda") * 0.3 + 1.0).bfloat16()
    ramp = torch.arange(S, device="cuda", dtype=torch.float32).view(1, 1, S, 1) * growth / 8.0
    k = (torch.randn(B, H, S, 64, device="cuda") * 0.3 + ramp / 64.0 * 8.0).bfloat16()   # q.k grows ~ growth per key
    v = rnd(B, H, S, 64)
    out = torch.zeros(B, S, H * 64, device="cuda", dtype=torch.bfloat16)
    lse = torch.zeros(B, H, S, device="cuda")
    ops.attn_fwd(q, k, v, None, out, lse, B, H, S, S, 0.125)
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float(), scale=0.125)
    ref_lse = torch.logsumexp(q.float() @ k.float().transpose(-1, -2) * 0.125, dim=-1)
    got = out.view(B, S, H, 64).transpose(1, 2).float()
    assert torch.isfinite(got).all()
    assert rel_err(got, ref, 1e-2) < 2e-2
    assert (lse - ref_lse).abs().max().item() < 2e-2
