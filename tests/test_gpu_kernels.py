"""GPU parity of every libb2d kernel, called through the C ABI (ctypes), against torch fp32 references / the oracle /
the golden vectors produced by the real reference sources.  Tolerances: bf16 outputs are compared at 1e-2 of the
reference's max magnitude (bf16 has 8 mantissa bits: ulp = 3.9e-3 relative); fp32 outputs at 2e-3; integer/byte-exact
paths (prep/pack, casts) bit-exact."""
import math

import pytest
import torch
import torch.nn.functional as F

from _util import bf16_ulp, check_bound, f32_ulp, rnd, rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from finetrainers_b200 import ops as o, lib
    lib.check(lib.load().b2d_device_check(), "device")
    return o


@pytest.mark.parametrize("M,N,K,bn", [(256, 256, 128, 64), (2688, 2048, 2048, 128), (2688, 2048, 2048, 256),
                                      (100, 72, 200, 192), (4, 2048, 256, 0), (2688, 6144, 2048, 0)])
def test_gemm_kmajor(ops, M, N, K, bn):
    torch.manual_seed(0)
    A, B = rnd(M, K), rnd(N, K, scale=0.05)
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(A, B, out, M=M, N=N, K=K, block_n=bn)
    assert rel_err(out, A.float() @ B.float().t()) < 1e-2


@pytest.mark.parametrize("M,N,K,bn,b_mn", [(2688, 2048, 2048, 256, False), (2688, 2048, 512, 160, False), (300, 520, 200, 192, False),
                                           (2688, 1024, 256, 128, False), (2688, 2048, 512, 256, True), (700, 2048, 512, 160, True),
                                           (2688, 768, 200, 192, True), (129, 128, 64, 128, True)])
def test_gemm_cta_pairs(ops, M, N, K, bn, b_mn):
    """CTA pairs (a 2-CTA cluster shares a 256 x bn tile, each CTA loading half of B and multicasting it to both) at every
    supported width, both B layouts, ragged M (an odd number of 128-row tiles leaves the last pair half empty), ragged N
    and K tails, bias + LoRA extension."""
    torch.manual_seed(0)
    A = rnd(M, K)
    Bm = rnd(K, N, scale=0.05) if b_mn else rnd(N, K, scale=0.05)
    bias = rnd(N)
    u = rnd(M, 64, scale=0.3)
    Bl = rnd(64, N, scale=0.05) if b_mn else rnd(N, 64, scale=0.05)
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(A, Bm, out, M=M, N=N, K=K, b_mn=b_mn, bias=bias, A2=u, B2=Bl, K2=64, block_n=bn, cta_pair=2)
    ref = A.float() @ (Bm.float() if b_mn else Bm.float().t()) + bias.float() + u.float() @ (Bl.float() if b_mn else Bl.float().t())
    assert rel_err(out, ref) < 1e-2
    out1 = torch.zeros_like(out)
    ops.gemm(A, Bm, out1, M=M, N=N, K=K, b_mn=b_mn, bias=bias, A2=u, B2=Bl, K2=64, block_n=bn, cta_pair=1)
    assert rel_err(out1, ref) < 1e-2
    with pytest.raises(Exception):
        ops.gemm(A[:64], Bm, out, M=64, N=N, K=K, b_mn=b_mn, block_n=bn, cta_pair=2)   # one M tile: no pair


@pytest.mark.parametrize("M,N,K", [(256, 128, 128), (2688, 2048, 8192), (200, 192, 136)])
def test_gemm_b_mn_major(ops, M, N, K):
    torch.manual_seed(0)
    A, Bt = rnd(M, K), rnd(K, N, scale=0.05)
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(A, Bt, out, M=M, N=N, K=K, b_mn=True)
    assert rel_err(out, A.float() @ Bt.float()) < 1e-2


@pytest.mark.parametrize("M,N,K,splits", [(2048, 64, 2688, 1), (2048, 192, 2688, 3), (304, 64, 1000, 2)])
def test_gemm_dw_split_k_atomic(ops, M, N, K, splits):
    torch.manual_seed(0)
    At, Bt = rnd(K, M), rnd(K, N, scale=0.05)
    ref = At.float().t() @ Bt.float()
    out = torch.zeros(M, N, device="cuda", dtype=torch.float32)
    ops.gemm(At, Bt, out, M=M, N=N, K=K, a_mn=True, b_mn=True, epi=ops.EPI_F32_ATOMIC, splits=splits, block_n=64)
    assert rel_err(out, ref) < 2e-3
    outT = torch.zeros(N, M, device="cuda", dtype=torch.float32)
    ops.gemm(At, Bt, outT, M=M, N=N, K=K, a_mn=True, b_mn=True, epi=ops.EPI_F32_ATOMIC_T, splits=splits, block_n=64,
             alpha=0.5)
    assert rel_err(outT, 0.5 * ref.t()) < 2e-3
    # accumulate semantics: a second call adds
    ops.gemm(At, Bt, out, M=M, N=N, K=K, a_mn=True, b_mn=True, epi=ops.EPI_F32_ATOMIC, splits=splits, block_n=64)
    assert rel_err(out, 2 * ref) < 2e-3


def test_gemm_epilogues(ops):
    torch.manual_seed(0)
    M, N, K = 2688, 2048, 512
    A, B, bias = rnd(M, K), rnd(N, K, scale=0.05), rnd(N)
    pre = A.float() @ B.float().t() + bias.float()
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    out2 = torch.zeros_like(out)
    ops.gemm(A, B, out, M=M, N=N, K=K, bias=bias, epi=ops.EPI_GELU, out2=out2)
    assert rel_err(out, F.gelu(pre, approximate="tanh")) < 1e-2 and rel_err(out2, pre) < 1e-2
    ops.gemm(A, B, out, M=M, N=N, K=K, bias=bias, epi=ops.EPI_SILU)
    assert rel_err(out, F.silu(pre)) < 1e-2
    res, tab, temb = rnd(M, N), rnd(6, N, scale=0.3), rnd(2, 6 * N, scale=0.3)
    ops.gemm(A, B, out, M=M, N=N, K=K, bias=bias, epi=ops.EPI_GATE_RES, res=res, gate_table=tab[2],
             gate_temb=temb[:, 2 * N:], gate2_table=tab[5], gate2_temb=temb[:, 5 * N:], out2=out2, temb_stride=6 * N,
             rows_per_sample=1344)
    gate = (tab[2].float()[None] + temb[:, 2 * N:3 * N].float()).repeat_interleave(1344, 0)
    gate2 = (tab[5].float()[None] + temb[:, 5 * N:6 * N].float()).repeat_interleave(1344, 0)
    ref = res.float() + gate * pre
    assert rel_err(out, ref) < 1e-2 and rel_err(out2, ref.bfloat16().float() * gate2) < 1e-2
    aux = rnd(M, N)
    ops.gemm(A, B, out, M=M, N=N, K=K, epi=ops.EPI_MUL_DGELU, aux=aux)
    x = aux.float().requires_grad_(True)
    F.gelu(x, approximate="tanh").sum().backward()
    assert rel_err(out, (pre - bias.float()) * x.grad) < 1e-2
    o32 = torch.zeros(M, N, device="cuda", dtype=torch.float32)
    ops.gemm(A, B, o32, M=M, N=N, K=K, bias=bias, epi=ops.EPI_F32_STORE)
    assert rel_err(o32, pre) < 2e-3


def test_gemm_lora_extension_and_batch(ops):
    torch.manual_seed(0)
    M, N, K, r = 2688, 6144, 2048, 64
    A, B, U, BL, bias = rnd(M, K), rnd(N, K, scale=0.05), rnd(M, 3 * r), rnd(N, r, scale=0.1), rnd(N)
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(A, B, out, M=M, N=N, K=K, bias=bias, A2=U, B2=BL, K2=r, a2_group_n=2048)
    ref = A.float() @ B.float().t() + bias.float()
    for j in range(3):
        ref[:, j * 2048:(j + 1) * 2048] += U[:, j * r:(j + 1) * r].float() @ BL[j * 2048:(j + 1) * 2048].float().t()
    assert rel_err(out, ref) < 1e-2
    dY, W, dU, AL = rnd(M, 6144), rnd(6144, 2048, scale=0.05), rnd(M, 192), rnd(192, 2048, scale=0.1)
    o = torch.zeros(M, 2048, device="cuda", dtype=torch.bfloat16)
    ops.gemm(dY, W, o, M=M, N=2048, K=6144, b_mn=True, A2=dU, B2=AL, K2=192)
    assert rel_err(o, dY.float() @ W.float() + dU.float() @ AL.float()) < 1e-2
    du = torch.zeros(M, 3 * r, device="cuda", dtype=torch.bfloat16)
    ops.gemm(dY, BL, du, M=M, N=r, K=2048, b_mn=True, batch=3, a_boff=(0, 2048), b_boff=(2048, 0), c_boff=r, ldc=3 * r)
    ref = torch.cat([dY[:, j * 2048:(j + 1) * 2048].float() @ BL[j * 2048:(j + 1) * 2048].float() for j in range(3)], 1)
    assert rel_err(du, ref) < 1e-2


def test_gemm_argument_errors(ops):
    from finetrainers_b200.lib import B2DError
    A, B = rnd(128, 64), rnd(64, 64)
    out = torch.zeros(128, 60, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(B2DError):
        ops.gemm(A, B, out, M=128, N=60, K=64)  # N % 8
    out = torch.zeros(128, 64, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(B2DError):
        ops.gemm(A, B, out, M=128, N=64, K=64, splits=2)  # split-K needs the atomic epilogue


@pytest.mark.parametrize("ln", [False, True])
def test_norm_modulate_fwd_bwd(ops, ln):
    torch.manual_seed(1)
    Bn, S, D = 2, 1344, 2048
    R = Bn * S
    x, tab, temb = rnd(R, D), rnd(6, D, scale=0.3), rnd(Bn, 6 * D, scale=0.3)
    y = torch.empty_like(x)
    ops.norm_modulate_fwd(x, y, tab[0], temb[:, 0:], tab[1], temb[:, D:], 6 * D, R, D, S, 1e-6, ln)
    xf = x.float().requires_grad_(True)
    shift = (tab[0].float()[None] + temb[:, :D].float()).repeat_interleave(S, 0)
    scale = (tab[1].float()[None] + temb[:, D:2 * D].float()).repeat_interleave(S, 0)
    n = F.layer_norm(xf, (D,), eps=1e-6) if ln else F.rms_norm(xf, (D,), eps=1e-6)
    ref = n * (1 + scale) + shift
    assert rel_err(y, ref) < 1e-2
    dy, dxin = rnd(R, D), rnd(R, D)
    ref.backward(dy.float())
    dx, o2 = torch.empty_like(x), torch.empty_like(x)
    ops.norm_modulate_bwd(dy, x, dxin, dx, tab[1], temb[:, D:], 6 * D, R, D, S, 1e-6, ln, gate2_tab=tab[5],
                          gate2_emb=temb[:, 5 * D:], out2=o2)
    refdx = dxin.float() + xf.grad
    g2 = (tab[5].float()[None] + temb[:, 5 * D:].float()).repeat_interleave(S, 0)
    assert rel_err(dx, refdx) < 1e-2 and rel_err(o2, refdx.bfloat16().float() * g2) < 1e-2


def test_rope_table_vs_oracle(ops):
    from oracle.ltx_oracle import ltx_rope_table
    Fr, Hh, Ww, D = 7, 16, 24, 2048
    S = Fr * Hh * Ww
    cos, sin = torch.empty(S, D // 2, device="cuda"), torch.empty(S, D // 2, device="cuda")
    ops.rope_table(cos, sin, Fr, Hh, Ww, D, (8 / 25) / 20, 32 / 2048, 32 / 2048)
    rc, rs = ltx_rope_table(Fr, Hh, Ww, D, [8 / 25, 32, 32], 1, "cpu")
    assert torch.equal(rc[0][:, 0::2], rc[0][:, 1::2])  # the reference table is pairwise constant
    # fp32 angles reach 1.6e4 rad: one ulp of the frequency is ~1e-3 rad, hence the 5e-3 absolute tolerance
    assert (cos.cpu() - rc[0][:, 0::2]).abs().max() < 5e-3 and (sin.cpu() - rs[0][:, 0::2]).abs().max() < 5e-3


@pytest.mark.parametrize("which,norm,rope", [(0, True, True), (1, True, False), (2, False, False)])
def test_qknorm_rope_fwd_bwd(ops, which, norm, rope):
    torch.manual_seed(2)
    Bq, H, S = 2, 32, 200
    D = H * 64
    ang = torch.randn(S, D // 2, device="cuda")
    cos, sin = ang.cos().repeat_interleave(2, -1).contiguous(), ang.sin().repeat_interleave(2, -1).contiguous()
    cos_p, sin_p = ang.cos().contiguous(), ang.sin().contiguous()  # kernel tables: one value per rotary pair
    qkv = rnd(Bq * S, 3 * D)
    w = (1 + 0.1 * torch.randn(D, device="cuda")).bfloat16()
    dst = torch.empty(Bq, H, S, 64, device="cuda", dtype=torch.bfloat16)
    ops.qknorm_rope_fwd(qkv, 3 * D, which * D, w, cos_p if rope else None, sin_p if rope else None, dst, Bq, S, H, norm, 1e-5)
    xf = qkv[:, which * D:(which + 1) * D].float().reshape(Bq, S, D).requires_grad_(True)
    n = F.rms_norm(xf, (D,), weight=w.float(), eps=1e-5) if norm else xf
    if rope:
        xr, xi = n.unflatten(2, (-1, 2)).unbind(-1)
        n = n * cos[None] + torch.stack([-xi, xr], dim=-1).flatten(2) * sin[None]
    ref = n.unflatten(2, (H, 64)).transpose(1, 2)
    assert rel_err(dst, ref) < 1e-2
    dyh = rnd(Bq, H, S, 64)
    ref.backward(dyh.float())
    dx = torch.zeros(Bq * S, 3 * D, device="cuda", dtype=torch.bfloat16)
    ops.qknorm_rope_bwd(dyh, qkv, 3 * D, which * D, w, cos_p if rope else None, sin_p if rope else None, dx, 3 * D, which * D,
                        Bq, S, H, norm, 1e-5)
    assert rel_err(dx[:, which * D:(which + 1) * D], xf.grad.reshape(Bq * S, D)) < 1e-2


@pytest.mark.parametrize("H,nseg", [(32, 3), (4, 3), (32, 2), (96, 3), (2, 1), (24, 2)])
def test_qkv_norm_rope_fused_segments(ops, H, nseg):
    """One launch for q|k|v (or k|v): segment i normed iff it has a weight, rotated iff its rope bit is set."""
    torch.manual_seed(3)
    Bq, S = 2, 120
    D = H * 64
    ang = torch.randn(S, D // 2, device="cuda")
    cos, sin = ang.cos().repeat_interleave(2, -1).contiguous(), ang.sin().repeat_interleave(2, -1).contiguous()
    cos_p, sin_p = ang.cos().contiguous(), ang.sin().contiguous()
    src = rnd(Bq * S, nseg * D + 64)          # packed row with a column offset
    ws = [(1 + 0.1 * torch.randn(D, device="cuda")).bfloat16() if i < nseg - 1 else None for i in range(nseg)]
    mask = 0b011 if nseg == 3 else 0b01
    dsts = [torch.empty(Bq, H, S, 64, device="cuda", dtype=torch.bfloat16) for _ in range(nseg)]
    ops.qkv_norm_rope_fwd(src, nseg * D + 64, 64, ws, mask, cos_p, sin_p, dsts, Bq, S, H, 1e-5)
    dys = [rnd(Bq, H, S, 64) for _ in range(nseg)]
    dx = torch.zeros(Bq * S, nseg * D + 64, device="cuda", dtype=torch.bfloat16)
    ops.qkv_norm_rope_bwd(dys, src, nseg * D + 64, 64, ws, mask, cos_p, sin_p, dx, nseg * D + 64, 64, Bq, S, H, 1e-5)
    for i in range(nseg):
        xf = src[:, 64 + i * D:64 + (i + 1) * D].float().reshape(Bq, S, D).requires_grad_(True)
        n = F.rms_norm(xf, (D,), weight=ws[i].float(), eps=1e-5) if ws[i] is not None else xf
        if (mask >> i) & 1:
            xr, xi = n.unflatten(2, (-1, 2)).unbind(-1)
            n = n * cos[None] + torch.stack([-xi, xr], dim=-1).flatten(2) * sin[None]
        ref = n.unflatten(2, (H, 64)).transpose(1, 2)
        assert rel_err(dsts[i], ref) < 1e-2, f"fwd seg {i}"
        ref.backward(dys[i].float())
        assert rel_err(dx[:, 64 + i * D:64 + (i + 1) * D], xf.grad.reshape(Bq * S, D)) < 1e-2, f"bwd seg {i}"
    assert dx[:, :64].abs().max() == 0


def test_golden_reference_vectors_on_gpu(ops, golden):
    """The CUDA prologue / RoPE / RMSNorm kernels against outputs of the REAL reference functions."""
    g = golden
    # prep: _normalize_latents + flow_match_xt + _pack_latents + flow_match_target, bit-exact
    lat, mean, std = g["nl_lat"].cuda(), g["nl_mean"].cuda(), g["nl_std"].cuda()
    noise, sig = g["fm_n"].cuda(), g["fm_t"].view(2).cuda()
    Bn, C, Fr, Hh, Ww = lat.shape
    xt = torch.empty(Bn, Fr * Hh * Ww, C, device="cuda", dtype=torch.bfloat16)
    tg = torch.empty_like(xt)
    ops.prep_noise_pack(lat, noise, mean, std, sig, None, xt, tg, Bn, C, Fr, Hh * Ww)
    from oracle.ltx_oracle import flow_match_xt, flow_match_target, pack_latents
    x0 = g["nl_out"]  # reference _normalize_latents output
    ref_xt = pack_latents(flow_match_xt(x0, g["fm_n"], g["fm_t"])).to(torch.bfloat16)
    ref_tg = pack_latents(flow_match_target(g["fm_n"], x0))
    assert torch.equal(xt.cpu(), ref_xt) and torch.equal(tg.cpu(), ref_tg)
    # RMSNorm (no affine) through norm_modulate with zero shift/scale, vs reference _patched_rms_norm_forward
    x = g["rms_noaffine_x"].reshape(15, 32).cuda()
    z = torch.zeros(1, 32, device="cuda", dtype=torch.bfloat16)
    y = torch.empty_like(x)
    ops.norm_modulate_fwd(x, y, z[0], z, z[0], z, 32, 15, 32, 15, g["rms_noaffine_eps"], False)
    assert (y.cpu().float() - g["rms_noaffine_out"].reshape(15, 32).float()).abs().max() < 2e-2
    # affine RMSNorm + RoPE: reference apply_rotary_emb on the reference-normalised tensor (H=1 head of 64 -> use D=64)
    torch.manual_seed(3)
    S, H = 6, 1
    xq = torch.randn(2 * S, 64).bfloat16()
    w = (1 + 0.1 * torch.randn(64)).bfloat16()
    ang = torch.randn(S, 32)
    cos, sin = ang.cos().repeat_interleave(2, -1), ang.sin().repeat_interleave(2, -1)
    from oracle.ltx_oracle import RMSNorm, apply_rotary_emb
    m = RMSNorm(64, 1e-5, True)
    m.weight.data = w.clone()
    ref = apply_rotary_emb(m(xq.view(2, S, 64)), (cos[None], sin[None]))  # oracle == reference (pinned in CPU tests)
    dst = torch.empty(2, H, S, 64, device="cuda", dtype=torch.bfloat16)
    ops.qknorm_rope_fwd(xq.cuda(), 64, 0, w.cuda(), ang.cos().cuda().contiguous(), ang.sin().cuda().contiguous(), dst, 2, S, H, True, 1e-5)
    assert (dst[:, 0].cpu().float() - ref.float()).abs().max() < 3e-2


def test_loss_sinusoid_cast_optimizer(ops):
    torch.manual_seed(4)
    Bp, S, Cc = 2, 2688, 128
    pred, tg = rnd(Bp, S, Cc), rnd(Bp, S, Cc)
    wgt = torch.tensor([1.0, 2.5], device="cuda")
    loss = torch.zeros(1, device="cuda")
    dpred, ws = torch.empty_like(pred), torch.empty(1024, device="cuda")
    ops.loss_mse(pred, tg, wgt, 1.0, loss, dpred, ws, Bp, S * Cc)
    pf = pred.float().requires_grad_(True)
    l = (wgt.view(Bp, 1, 1) * (pf - tg.float()).pow(2)).mean((1, 2)).mean()
    l.backward()
    assert abs(loss.item() - l.item()) / l.item() < 1e-5 and rel_err(dpred, pf.grad) < 1e-2
    from oracle.ltx_oracle import sinusoid_256
    t = torch.tensor([0.0, 1.0, 500.0, 999.0], device="cuda")
    so = torch.empty(4, 256, device="cuda", dtype=torch.bfloat16)
    ops.timestep_sinusoid(t, so, 4)
    assert (so.cpu().float() - sinusoid_256(t.cpu())).abs().max() < 8e-3
    n = 1000003
    src = torch.randn(n, device="cuda")
    dstb = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    ops.cast_f32_bf16(src, dstb, n, 0.5)
    assert torch.equal(dstb, (src * 0.5).bfloat16())
    # clip + AdamW vs torch.optim.AdamW + clip_grad_norm_
    p, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
    m, v, ss = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(1, device="cuda")
    pr = torch.nn.Parameter(p.clone())
    pr.grad = g.clone()
    opt = torch.optim.AdamW([pr], lr=1e-2, betas=(0.9, 0.99), weight_decay=1e-2, eps=1e-8)
    for step in (1, 2):
        ss.zero_()
        ops.sumsq(g, n, ss, ws)
        torch.nn.utils.clip_grad_norm_([pr], 1.0)
        opt.step()
        ops.adamw_clip(p, g, m, v, n, ss, 1.0, 1e-2, 0.9, 0.99, 1e-8, 1e-2, step)
        assert rel_err(p, pr.detach()) < 1e-5
        assert g.abs().max().item() == 0.0  # fused zero_grad
        g2 = torch.randn(n, device="cuda")
        g.copy_(g2)
        pr.grad = g2.clone()


# ---------------------------------------------------------------------------------------------------------------------
# argument checks of b2d_gemm / b2d_colscale that guard against silent misuse
# ---------------------------------------------------------------------------------------------------------------------
def _raises_code(code, fn):
    from finetrainers_b200.lib import B2DError
    with pytest.raises(B2DError, match=rf"\(code {code}\)"):
        fn()


def test_gemm_epilogue_argument_checks(ops):
    """gate2 without its temb rows, rows_per_sample or out2 is refused (B2D_ERR_ARG); every epilogue pointer, leading
    dimension, temb_stride and c_boff must keep rows 16-byte aligned (B2D_ERR_ALIGN); a batched launch whose batch
    offset runs along a ragged K is refused (B2D_ERR_SHAPE)."""
    M, N, K = 128, 64, 64
    A, B = rnd(M, K), rnd(N, K, scale=0.1)
    # every operand lives in storage large enough for what a launch with the rejected argument would touch (strides up
    # to N + 8, offsets up to N + 8 elements, a second batch slice), so that a check that regressed cannot reach
    # outside its allocation
    buf = torch.zeros(2 * M * (N + 8) + 64, device="cuda", dtype=torch.bfloat16)
    out2buf = torch.zeros(M * (N + 8) + 64, device="cuda", dtype=torch.bfloat16)
    res_s, aux_s = rnd(M * (N + 8) + 64), rnd(M * (N + 8) + 64)
    out, out2 = buf[:M * N].view(M, N), out2buf[:M * N].view(M, N)
    res, aux = res_s[:M * N].view(M, N), aux_s[:M * N].view(M, N)
    tab, temb = rnd(3, N), rnd(1, 3 * N)
    g = dict(res=res, epi=ops.EPI_GATE_RES, temb_stride=2 * N, rows_per_sample=M)
    run = lambda **kw: ops.gemm(A, B, kw.pop("out", out), M=M, N=N, K=K, **kw)
    run(**g, gate2_table=tab[1], gate2_temb=temb[:, N:], out2=out2)             # the accepted form
    _raises_code(-5, lambda: run(**g, gate2_table=tab[1], out2=out2))            # no gate2_temb
    _raises_code(-5, lambda: run(**dict(g, rows_per_sample=0), gate2_table=tab[1], gate2_temb=temb[:, N:], out2=out2))
    _raises_code(-5, lambda: run(**g, gate2_table=tab[1], gate2_temb=temb[:, N:]))   # no out2
    # alignment: one case per operand
    _raises_code(-2, lambda: run(ldc=N + 4))
    _raises_code(-2, lambda: run(epi=ops.EPI_GELU, out2=out2, ldc2=N + 4))
    _raises_code(-2, lambda: run(epi=ops.EPI_GELU, out2=buf[1:1 + M * N].view(M, N)))
    _raises_code(-2, lambda: run(**dict(g, res=res_s[4:]), ldres=N))
    _raises_code(-2, lambda: run(**g, ldres=N + 2))
    _raises_code(-2, lambda: run(epi=ops.EPI_MUL_DGELU, aux=aux, ldaux=N - 4))
    _raises_code(-2, lambda: run(epi=ops.EPI_MUL_DGELU, aux=aux_s[2:], ldaux=N))
    _raises_code(-2, lambda: run(bias=tab.view(-1)[1:]))
    _raises_code(-2, lambda: run(**g, gate_table=tab.view(-1)[4:], gate_temb=temb))
    _raises_code(-2, lambda: run(**g, gate_table=tab[0], gate_temb=temb.view(-1)[4:]))
    _raises_code(-2, lambda: run(**g, gate2_table=tab.view(-1)[N + 4:], gate2_temb=temb[:, N:], out2=out2))
    _raises_code(-2, lambda: run(**g, gate2_table=tab[1], gate2_temb=temb.view(-1)[N + 4:], out2=out2))
    _raises_code(-2, lambda: run(**dict(g, temb_stride=2 * N + 4), gate_table=tab[0], gate_temb=temb))
    _raises_code(-2, lambda: run(batch=2, c_boff=M * N + 4, b_boff=(0, 0)))
    o32 = torch.zeros(M, N + 4, device="cuda")
    run(out=o32, epi=ops.EPI_F32_STORE, ldc=N + 4)                                # fp32 rows: 4-element multiples
    _raises_code(-2, lambda: run(out=o32, epi=ops.EPI_F32_STORE, ldc=N + 2))
    # batched, K % 64 != 0, batch offset along K
    A2 = rnd(M, 2 * 72)
    _raises_code(-1, lambda: ops.gemm(A2, rnd(N, 72), out, M=M, N=N, K=72, batch=2, a_boff=(0, 72), c_boff=0))
    assert torch.isfinite(out.float()).all()


def test_colscale_vs_fp64(ops):
    """out = x * (tab[c] + emb[b, c]) with D = 72 (nine 8-column groups per row) and 5-row samples, against fp64; a
    non-positive rows_per_sample is refused."""
    torch.manual_seed(5)
    rps, nb, D, es = 5, 3, 72, 88
    x, tab, emb = rnd(nb * rps, D), rnd(D), rnd(nb, es)
    out = torch.empty_like(x)
    ops.colscale(x, out, tab, emb, es, nb * rps, D, rps)
    b = torch.arange(nb * rps, device="cuda") // rps
    ref = x.double() * (tab.double()[None] + emb[:, :D].double()[b])
    check_bound(out, ref, bf16_ulp(ref) + 2.0 ** -22 * ref.abs(), "colscale")
    _raises_code(-1, lambda: ops.colscale(x, out, tab, emb, es, nb * rps, D, 0))


def _norm64(x, ln, eps):
    x = x - x.mean(-1, keepdim=True) if ln else x
    return x * torch.rsqrt((x * x).mean(-1, keepdim=True) + eps)


@pytest.mark.parametrize("D", [72, 2056, 4096, 6152, 8192])
@pytest.mark.parametrize("ln", [False, True])
def test_norm_modulate_widths_vs_fp64(ops, D, ln):
    """Every ROW_DISPATCH instantiation (1, 2, 4 chunks of 2048 columns, partial last chunks), three samples, against an
    fp64 reference: forward, backward with and without the accumulated input gradient (dx_in = NULL) and the gated
    second output.  Bounds: 1 bf16 ulp + 2^-14 of the row's largest magnitude (fp32 statistics and row reductions)."""
    torch.manual_seed(D)
    S, nb, eps = 5, 3, 1e-6
    R = S * nb
    x, tab, temb = rnd(R, D), rnd(6, D, scale=0.3), rnd(nb, 6 * D, scale=0.3)
    b = torch.arange(R, device="cuda") // S
    row = lambda i: tab[i].double()[None] + temb[:, i * D:(i + 1) * D].double()[b]

    def bound(ref):
        return bf16_ulp(ref) + 2.0 ** -14 * ref.abs().amax(-1, keepdim=True)

    y = torch.empty_like(x)
    ops.norm_modulate_fwd(x, y, tab[0], temb[:, 0:], tab[1], temb[:, D:], 6 * D, R, D, S, eps, ln)
    xd = x.double().requires_grad_(True)
    ref = _norm64(xd, ln, eps) * (1 + row(1)) + row(0)
    check_bound(y, ref.detach(), bound(ref.detach()), "norm_modulate_fwd")
    dy, dxin = rnd(R, D), rnd(R, D)
    ref.backward(dy.double())
    dx, o2 = torch.empty_like(x), torch.empty_like(x)
    ops.norm_modulate_bwd(dy, x, dxin, dx, tab[1], temb[:, D:], 6 * D, R, D, S, eps, ln, gate2_tab=tab[5],
                          gate2_emb=temb[:, 5 * D:], out2=o2)
    refdx = dxin.double() + xd.grad
    check_bound(dx, refdx, bound(refdx), "norm_modulate_bwd")
    ref2 = dx.double() * row(5)
    check_bound(o2, ref2, bf16_ulp(ref2) + 2.0 ** -22 * ref2.abs(), "norm_modulate_bwd out2")
    dx0 = torch.empty_like(x)
    ops.norm_modulate_bwd(dy, x, None, dx0, tab[1], temb[:, D:], 6 * D, R, D, S, eps, ln)
    check_bound(dx0, xd.grad, bound(xd.grad), "norm_modulate_bwd dx_in = NULL")
    with pytest.raises(Exception):
        big = rnd(2, 8200)
        ops.norm_modulate_fwd(big, big, big[0], big, big[0], big, 8200, 2, 8200, 2, eps, ln)


@pytest.mark.parametrize("H", [2, 33, 128])
def test_qkv_norm_rope_stacked_weights_vs_fp64(ops, H):
    """rows_per_w > 0: the rows are two DiT blocks stacked (the text-side k|v of every block in one launch); block i's
    rows use the k-norm weight w + i * w_stride, with w_stride != D.  k is RMS-normed, v is copied; no RoPE.  Against
    fp64, forward and backward."""
    torch.manual_seed(H)
    nblk, bsz, S, eps = 2, 2, 5, 1e-5
    D, Bq = H * 64, nblk * bsz
    rows = Bq * S
    src = rnd(rows, 2 * D + 64)
    wst = D + 8
    w = (1 + 0.1 * torch.randn(nblk * wst, device="cuda")).bfloat16()
    dk, dv = (torch.empty(Bq, H, S, 64, device="cuda", dtype=torch.bfloat16) for _ in range(2))
    ops.qkv_norm_rope_fwd(src, 2 * D + 64, 64, (w, None), 0, None, None, (dk, dv), Bq, S, H, eps, rows_per_w=bsz * S,
                          w_stride=wst)
    blk = torch.arange(rows, device="cuda") // (bsz * S)
    wr = torch.stack([w[i * wst:i * wst + D] for i in range(nblk)]).double()[blk]
    xk = src[:, 64:64 + D].double().requires_grad_(True)
    k = _norm64(xk, False, eps) * wr
    heads = lambda t: t.reshape(Bq, S, H, 64).transpose(1, 2)
    check_bound(dk, heads(k.detach()), bf16_ulp(heads(k.detach())) + 2.0 ** -16 * k.detach().abs().amax(), "k fwd")
    assert torch.equal(dv, heads(src[:, 64 + D:64 + 2 * D]))
    gk, gv = rnd(Bq, H, S, 64), rnd(Bq, H, S, 64)
    k.backward(gk.double().transpose(1, 2).reshape(rows, D))
    dx = torch.zeros(rows, 2 * D + 64, device="cuda", dtype=torch.bfloat16)
    ops.qkv_norm_rope_bwd((gk, gv), src, 2 * D + 64, 64, (w, None), 0, None, None, dx, 2 * D + 64, 64, Bq, S, H, eps,
                          rows_per_w=bsz * S, w_stride=wst)
    g = xk.grad
    check_bound(dx[:, 64:64 + D], g, bf16_ulp(g) + 2.0 ** -14 * g.abs().amax(-1, keepdim=True), "k bwd")
    assert torch.equal(dx[:, 64 + D:64 + 2 * D], gv.transpose(1, 2).reshape(rows, D))
    assert dx[:, :64].abs().max() == 0


def test_prep_noise_pack_first_frame_sigma_bit_exact(ops):
    """x_t with a per-sample first-frame sigma (the first-frame conditioning branch), bit-exact against the oracle's
    spec_forward arithmetic (normalize, flow_match_xt per frame range, pack)."""
    from oracle.ltx_oracle import flow_match_target, flow_match_xt, normalize_latents, pack_latents
    torch.manual_seed(6)
    Bn, C, Fr, Hh, Ww = 3, 16, 4, 6, 5
    lat, noise = torch.randn(Bn, C, Fr, Hh, Ww).bfloat16(), torch.randn(Bn, C, Fr, Hh, Ww).bfloat16()
    mean, std = torch.randn(Bn, C), torch.rand(Bn, C) + 0.5
    sig, sff = torch.rand(Bn), torch.rand(Bn) * 0.25
    xt = torch.empty(Bn, Fr * Hh * Ww, C, device="cuda", dtype=torch.bfloat16)
    tg = torch.empty_like(xt)
    ops.prep_noise_pack(lat.cuda(), noise.cuda(), mean.cuda(), std.cuda(), sig.cuda(), sff.cuda(), xt, tg, Bn, C, Fr,
                        Hh * Ww)
    x0 = normalize_latents(lat, mean, std)
    v = lambda s: s.view(Bn, 1, 1, 1, 1)
    noisy = torch.cat([flow_match_xt(x0[:, :, :1], noise[:, :, :1], v(sff)),
                       flow_match_xt(x0[:, :, 1:], noise[:, :, 1:], v(sig))], dim=2)
    assert torch.equal(xt.cpu(), pack_latents(noisy).bfloat16())
    assert torch.equal(tg.cpu(), pack_latents(flow_match_target(noise, x0)).bfloat16())


def test_loss_mse_batch3_scaled_vs_fp64(ops):
    """loss = mean_b(w_b mean((pred - target)^2)) * loss_scale and dpred, three samples, loss_scale != 1, against fp64."""
    torch.manual_seed(7)
    Bp, per = 3, 40 * 128
    pred, tg = rnd(Bp, per), rnd(Bp, per)
    wgt, ls = torch.tensor([0.5, 1.0, 3.0], device="cuda"), 0.37
    loss, dpred, ws = torch.zeros(1, device="cuda"), torch.empty_like(pred), torch.empty(1024, device="cuda")
    ops.loss_mse(pred, tg, wgt, ls, loss, dpred, ws, Bp, per)
    d = pred.double() - tg.double()
    ref = (wgt.double()[:, None] * d * d).mean(1).mean() * ls
    assert abs(loss.item() - ref.item()) <= 1e-5 * ref.item()
    refg = 2 * wgt.double()[:, None] * d / (per * Bp) * ls
    check_bound(dpred, refg, bf16_ulp(refg) + 2.0 ** -20 * refg.abs(), "dpred")


def test_adamw_clip_grad_div_vs_fp64(ops):
    """grad_div != 1 (gradient accumulation): the step clips and applies g * grad_div, as torch's clip_grad_norm_ +
    AdamW do on the divided gradient (fp64 reference), with an n that leaves a 3-element tail.  Steps 1 and 3 have
    |g| * grad_div < max_norm < |g|, so whether they clip depends on grad_div; step 2 clips either way (where clipping
    makes grad_div cancel) and carries the earlier steps' scale forward through the moments.  Replayed in fp64, a step
    that drops grad_div, or applies it to only the gradient or only the norm, misses this bound by a factor of 300 or
    more."""
    torch.manual_seed(8)
    n, gd, lr, scales = 100003, 0.25, 1e-2, (0.005, 3.0, 0.005)
    p, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda") * scales[0]
    m, v, ss, ws = (torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(1, device="cuda"),
                    torch.empty(1024, device="cuda"))
    pr = torch.nn.Parameter(p.double())
    opt = torch.optim.AdamW([pr], lr=lr, betas=(0.9, 0.99), weight_decay=1e-2, eps=1e-8)
    for step in (1, 2, 3):
        norm = g.double().norm().item()
        assert (norm * gd < 1.0 < norm) if step != 2 else (norm * gd > 1.0)
        pr.grad = g.double() * gd
        ss.zero_()
        ops.sumsq(g, n, ss, ws)
        torch.nn.utils.clip_grad_norm_([pr], 1.0)
        opt.step()
        ops.adamw_clip(p, g, m, v, n, ss, 1.0, lr, 0.9, 0.99, 1e-8, 1e-2, step, grad_div=gd)
        check_bound(p, pr.detach(), 2 * f32_ulp(pr.detach()) + 2.0 ** -12 * lr, f"adamw step {step}")
        assert g.abs().max().item() == 0.0
        if step < 3:
            g.copy_(torch.randn(n, device="cuda") * scales[step])


def test_attn_bwd_bitwise_repeatable(ops):
    """The split dK/dV path (few heads, 128 < Sk <= 512) sums its per-range partials in a fixed order: two runs of the
    backward give the same bits."""
    torch.manual_seed(9)
    B, H, Sq, Sk = 1, 2, 1000, 300
    q, k, v = rnd(B, H, Sq, 64), rnd(B, H, Sk, 64), rnd(B, H, Sk, 64)
    out, lse = torch.zeros(B, Sq, H * 64, device="cuda", dtype=torch.bfloat16), torch.zeros(B, H, Sq, device="cuda")
    ops.attn_fwd(q, k, v, None, out, lse, B, H, Sq, Sk, 0.125)
    dout = rnd(B, Sq, H * 64)
    res = []
    for _ in range(2):
        dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
        ws = torch.zeros(ops.attn_bwd_ws_floats(B, H, Sq, Sk), device="cuda")
        ops.attn_bwd(q, k, v, None, out, dout, lse, ws, dq, dk, dv, B, H, Sq, Sk, 0.125)
        res.append((dq, dk, dv))
    for a, b in zip(*res):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
