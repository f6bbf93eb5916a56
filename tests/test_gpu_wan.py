"""GPU: Wan-2.1 T2V on the engine.

- Kernels: the step prologue bit-exact against the reference's torch ops run on the GPU; the patch permutes exact; the
  affine LayerNorm (fwd / bwd) and the per-head q/k-norm + RoPE (fwd / bwd) against fp64 with element-wise bounds; the
  per-head RoPE table against the float64 frequencies.
- Model: a 2-block full-width Wan-1.3B training step against the fp32 oracle (loss within 1e-3, every LoRA gradient
  within 5 % of its own scale); a 20-step trajectory against the oracle with torch AdamW (loss within 1e-3 on every
  step, accumulated update direction and length); CUDA-graph steps, "full" and "block_skip" checkpointing
  bit-identical to eager keep-all, with and without gradient accumulation; accumulated gradients the sum of the
  micro-steps'; two seeded 20-step runs bit-identical; a 40-step finite soak; the public forward and its autograd
  backward against the fused step.
"""
import math

import pytest
import torch

from oracle import wan_oracle as O

pytestmark = pytest.mark.gpu

D13 = dict(num_attention_heads=12, attention_head_dim=128, ffn_dim=8960)


@pytest.fixture(scope="module")
def ops():
    from finetrainers_b200 import lib, ops as o
    lib.check(lib.load().b2d_device_check(), "device")
    return o


def _same(a, b, what):
    a, b = a.reshape(-1).cpu(), b.reshape(-1).cpu()
    diff = int((a.view(torch.int16) != b.view(torch.int16)).sum())
    assert diff == 0, f"{what}: {diff} element(s) differ"


def _patchify_ref(x, out_order):
    """torch restatement: [B, C, F, H, W] -> [B, F (H/2) (W/2), 4C] in the Conv3d (c, kh, kw) or proj_out (kh, kw, c)
    channel order."""
    B, C, F, H, W = x.shape
    t = x.reshape(B, C, F, H // 2, 2, W // 2, 2)
    t = t.permute(0, 2, 3, 5, 4, 6, 1) if out_order else t.permute(0, 2, 3, 5, 1, 4, 6)
    return t.reshape(B, F * (H // 2) * (W // 2), 4 * C)


def test_wan_prologue_bitexact(ops):
    g = torch.Generator().manual_seed(0)
    B, C, F, H, W = 2, 16, 3, 6, 10
    mom = torch.cat([torch.randn(B, C, F, H, W, generator=g), torch.rand(B, C, F, H, W, generator=g) * 60 - 35], 1)
    mom.view(-1)[:4] = torch.tensor([float("nan"), float("inf"), -1e4, 1e4])
    mom = mom.to(torch.bfloat16).cuda()
    eps = torch.randn(B, C, F, H, W, generator=g).to(torch.bfloat16).cuda()
    noise = torch.randn(B, C, F, H, W, generator=g).to(torch.bfloat16).cuda()
    mean = (torch.randn(C, generator=g) * 0.3).cuda()
    std = (1.0 / (torch.rand(C, generator=g) + 0.5)).cuda()
    sig = torch.rand(B, generator=g).cuda()
    xt_ref, tg_ref = O.prologue(mom, mean, std, eps, noise, sig)
    S = F * (H // 2) * (W // 2)
    x_t = torch.empty(B, S, 4 * C, dtype=torch.bfloat16, device="cuda")
    tg = torch.empty_like(x_t)
    ops.wan_prep(mom, eps, noise, mean.expand(B, C).contiguous(), std.expand(B, C).contiguous(), sig, x_t, tg,
                 B, C, F, H, W)
    nan = torch.isnan(_patchify_ref(xt_ref, 0))
    assert torch.equal(nan.cpu(), torch.isnan(x_t).cpu())
    _same(torch.where(nan, 0, x_t), torch.where(nan, 0, _patchify_ref(xt_ref, 0)), "x_t")
    nan = torch.isnan(_patchify_ref(tg_ref, 1))
    _same(torch.where(nan, 0, tg), torch.where(nan, 0, _patchify_ref(tg_ref, 1)), "target")


@pytest.mark.parametrize("order", [0, 1])
def test_patch_permutes_exact(ops, order):
    B, C, F, H, W = 2, 16, 3, 4, 8
    x = torch.randn(B, C, F, H, W, device="cuda").to(torch.bfloat16)
    p = torch.empty(B, F * (H // 2) * (W // 2), 4 * C, dtype=torch.bfloat16, device="cuda")
    ops.patch_permute(x, p, B, C, F, H, W, order, False)
    _same(p, _patchify_ref(x, order), "patchify")
    y = torch.empty_like(x)
    ops.patch_permute(p, y, B, C, F, H, W, order, True)
    _same(y, x, "unpatchify")


def test_layer_norm_affine_fwd_bwd(ops):
    R, D, eps = 300, 1536, 1e-6
    x = (torch.randn(R, D, device="cuda") * 3 + 1).to(torch.bfloat16)
    w = (1 + 0.2 * torch.randn(D, device="cuda")).to(torch.bfloat16)
    b = (0.1 * torch.randn(D, device="cuda")).to(torch.bfloat16)
    y = torch.empty_like(x)
    ops.layer_norm_affine_fwd(x, y, w, b, R, D, eps)
    xd = x.double().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(xd, (D,), w.double(), b.double(), eps)
    err = (y.double() - ref).abs()
    assert (err <= ref.abs() * 2 ** -8 + 1e-3).all(), float(err.max())
    dy = torch.randn(R, D, device="cuda").to(torch.bfloat16)
    dx_in = torch.randn(R, D, device="cuda").to(torch.bfloat16)
    gt, ge = torch.randn(D, device="cuda").to(torch.bfloat16), torch.randn(2, 8 + D, device="cuda").to(torch.bfloat16)
    dx, out2 = torch.empty_like(x), torch.empty_like(x)
    ops.layer_norm_affine_bwd(dy, x, dx_in, dx, w, R, D, eps, gate2_tab=gt, gate2_emb=ge[:, 8:], out2=out2,
                              emb_stride=8 + D, rows_per_sample=R // 2)
    (gx,) = torch.autograd.grad(ref, xd, dy.double())
    want = dx_in.double() + gx
    scale = want.abs().amax(1, keepdim=True)
    assert ((dx.double() - want).abs() <= want.abs() * 2 ** -8 + 1e-3 * scale).all()
    gate = gt.double() + torch.repeat_interleave(ge[:, 8:].double(), R // 2, 0)
    assert ((out2.double() - dx.double() * gate).abs() <= (dx.double() * gate).abs() * 2 ** -8 + 1e-30).all()


def test_per_head_rope_table(ops):
    F, H, W, hd = 3, 5, 7, 128
    cos = torch.empty(F * H * W, hd // 2, device="cuda")
    sin = torch.empty_like(cos)
    ops.rope_table_wan(cos, sin, F, H, W, hd)
    # against the independent float64 derivation (oracle/wan_independent_constants.py): fp32 rounding only
    from oracle import wan_independent_constants as IC
    ref = torch.tensor([[IC.wan_rope_entry(f, h, w, p, hd) for p in range(hd // 2)]
                        for f in range(F) for h in range(H) for w in range(W)], dtype=torch.float64)
    assert (cos.cpu().double() - ref[..., 0]).abs().max() <= 2 ** -24
    assert (sin.cpu().double() - ref[..., 1]).abs().max() <= 2 ** -24
    # and the fp32 value nearest to it, as the one rounding of the float64 value gives
    assert torch.equal(cos.cpu(), ref[..., 0].float()) and torch.equal(sin.cpu(), ref[..., 1].float())


def test_per_head_qk_norm_rope_fwd_bwd(ops):
    B, F, H, W, heads, hd, eps = 1, 2, 4, 6, 12, 128, 1e-6
    S, D = F * H * W, heads * hd
    cos = torch.empty(S, hd // 2, device="cuda")
    sin = torch.empty_like(cos)
    ops.rope_table_wan(cos, sin, F, H, W, hd)
    qkv = torch.randn(B * S, 3 * D, device="cuda").to(torch.bfloat16)
    wq, wk = [(1 + 0.2 * torch.randn(D, device="cuda")).to(torch.bfloat16) for _ in range(2)]
    outs = [torch.empty(B, heads, S, hd, dtype=torch.bfloat16, device="cuda") for _ in range(3)]
    ops.qkv_norm_rope_fwd(qkv, 3 * D, 0, (wq, wk, None), 0b011, cos, sin, outs, B, S, heads, eps, head_dim=hd,
                          per_head=True)
    freqs = O.wan_rope(hd, F, H, W)
    x = qkv.double().view(B, S, 3, D).requires_grad_(True)

    def ref_fn(x):
        res = []
        for i, w in ((0, wq), (1, wk)):
            t = x[:, :, i]
            t = t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + eps) * w.double()
            t = t.unflatten(2, (heads, hd)).transpose(1, 2)
            tc = torch.view_as_complex(t.unflatten(3, (-1, 2)).contiguous()) * freqs.to(t.device)
            res.append(torch.view_as_real(tc).flatten(3, 4))
        res.append(x[:, :, 2].unflatten(2, (heads, hd)).transpose(1, 2))
        return res

    refs = ref_fn(x)
    for o, r, n in zip(outs, refs, "qkv"):
        assert ((o.double() - r).abs() <= r.abs() * 2 ** -8 + 2e-3).all(), (n, float((o.double() - r).abs().max()))
    dys = [torch.randn_like(o) for o in outs]
    dx = torch.empty_like(qkv)
    ops.qkv_norm_rope_bwd(dys, qkv, 3 * D, 0, (wq, wk, None), 0b011, cos, sin, dx, 3 * D, 0, B, S, heads, eps,
                          head_dim=hd, per_head=True)
    (gx,) = torch.autograd.grad(refs, x, [d.double() for d in dys])
    gx = gx.reshape(B * S, 3 * D)
    scale = gx.abs().amax(1, keepdim=True)
    assert ((dx.double() - gx).abs() <= gx.abs() * 2 ** -7 + 2e-3 * scale).all()


# ---------------------------------------------------------------------------------------------------------------------
def _pair(nl, r=32, seed=0, **geom):
    from finetrainers_b200.wan import B200WanTransformer, WanConfig
    om = O.WanTransformerOracle(O.WanOracleConfig(num_layers=nl, **geom))
    O.add_lora(om, r, r)
    O.synthetic_init_(om, seed=seed)
    with torch.no_grad():
        for n, p in om.named_parameters():
            if "lora_" not in n:
                p.copy_(p.to(torch.bfloat16).float())
    bm = B200WanTransformer(WanConfig(num_layers=nl, **geom), torch.bfloat16, "cuda")
    bm.add_adapter(r, r)
    bm.load_state_dict(om.state_dict(), strict=True)
    bm.prepare()
    bm.skip_block0_dx = False
    return om, bm


def _batch(B=1, F=3, H=16, W=24, L=512, seed=1):
    g = torch.Generator().manual_seed(seed)
    mom = torch.cat([torch.randn(B, 16, F, H, W, generator=g), torch.rand(B, 16, F, H, W, generator=g) * 4 - 8], 1)
    return dict(moments=mom.to(torch.bfloat16), mean=torch.randn(16, generator=g) * 0.2,
                std=1.0 / (torch.rand(16, generator=g) + 0.5),
                eps=torch.randn(B, 16, F, H, W, generator=g).to(torch.bfloat16),
                noise=torch.randn(B, 16, F, H, W, generator=g).to(torch.bfloat16),
                sigmas=torch.rand(B, generator=g) * 0.9 + 0.05,
                ehs=(torch.randn(B, L, 4096, generator=g)).to(torch.bfloat16))


def _micro(st, bt):
    B = bt["moments"].shape[0]
    cond = {"encoder_hidden_states": bt["ehs"].cuda()}
    lat = {"latents": bt["moments"].cuda(), "latents_mean": bt["mean"].expand(B, 16).cuda(),
           "latents_std": bt["std"].expand(B, 16).cuda()}
    return st.micro_step(cond, lat, sigmas=bt["sigmas"].cuda(), noise=bt["noise"].cuda(),
                         posterior_noise=bt["eps"].cuda())


def _grad_errors(om, bm):
    """name -> max |engine grad - oracle grad| / max |oracle grad| of every LoRA parameter."""
    og = dict(om.named_parameters())
    return {n: (p.grad.float().cpu() - og[n].grad).abs().max().item() / og[n].grad.abs().max().item()
            for n, p in bm.named_parameters() if "lora_" in n}


def test_wan13b_two_blocks_vs_oracle():
    from finetrainers_b200.trainer import SFTTrainStep
    om, bm = _pair(2, **D13)
    bt = _batch()
    loss_o, _ = O.oracle_step(om, bt["moments"], bt["mean"], bt["std"], bt["eps"], bt["noise"], bt["sigmas"],
                              bt["ehs"])
    st = SFTTrainStep(bm, flow_weighting_scheme="none")
    loss_b = _micro(st, bt).item()
    rel = abs(loss_b - loss_o.item()) / abs(loss_o.item())
    errs = _grad_errors(om, bm)
    worst = max(errs.items(), key=lambda t: t[1])
    print(f"\nWan-1.3B 2 blocks: loss rel err {rel:.2e}, worst LoRA grad err {worst[1]:.3e} ({worst[0]})")
    assert math.isfinite(loss_b) and rel < 1e-3, (loss_b, loss_o.item())
    assert worst[1] < 5e-2, worst


SMALL = dict(num_attention_heads=4, attention_head_dim=128, ffn_dim=1024)


def test_wan_twenty_step_trajectory_matches_oracle():
    """20 optimizer steps (lr 1e-3, clip 1.0, AdamW) of the engine and of the fp32 oracle with torch AdamW and the
    reference's clip, on the same data stream: the loss within 1e-3 relative on every step, and the accumulated adapter
    update keeps direction (cos > 0.98) and length (3 %).  This bounds what the bf16 LoRA operands cost over training."""
    from finetrainers_b200.trainer import SFTTrainStep
    from oracle.ltx_oracle import clip_grad_norm_
    om, bm = _pair(2, r=32, seed=3, **SMALL)
    st = SFTTrainStep(bm, flow_weighting_scheme="none", lr=1e-3, seed=5)
    params = [p for n, p in om.named_parameters() if "lora_" in n]
    opt = torch.optim.AdamW(params, lr=1e-3, betas=(0.9, 0.99), weight_decay=1e-4, eps=1e-8)
    p0 = {n: p.detach().clone() for n, p in om.named_parameters() if "lora_" in n}
    worst = 0.0
    for i in range(20):
        bt = _batch(B=2, F=2, H=8, W=12, L=32, seed=500 + i)
        loss_b = _micro(st, bt).item()
        opt.zero_grad(set_to_none=True)
        loss_o, _ = O.oracle_step(om, bt["moments"], bt["mean"], bt["std"], bt["eps"], bt["noise"], bt["sigmas"],
                                  bt["ehs"])
        rel = abs(loss_b - loss_o.item()) / abs(loss_o.item())
        worst = max(worst, rel)
        assert rel < 1e-3, (i, loss_b, loss_o.item(), rel)
        clip_grad_norm_(params, 1.0)
        opt.step()
        st.optimizer_step()
    torch.cuda.synchronize()
    og = dict(om.named_parameters())
    db = torch.cat([(p.detach().float().cpu() - p0[n]).flatten() for n, p in bm.named_parameters() if "lora_" in n])
    do = torch.cat([(og[n].detach() - p0[n]).flatten() for n, p in bm.named_parameters() if "lora_" in n])
    cos, ratio = (torch.dot(db, do) / (db.norm() * do.norm())).item(), (db.norm() / do.norm()).item()
    print(f"\nWan 20-step trajectory: worst loss rel err {worst:.2e}, update cos {cos:.5f}, length ratio {ratio:.4f}")
    assert cos > 0.98 and abs(ratio - 1) < 0.03


def _run(steps, graph=False, ckpt=None, accum=1, seed=0, shape=dict(F=2, H=8, W=12, L=64)):
    """Loss of every micro-step and the final fp32 adapter masters of ``steps`` train_step calls on one batch.
    ``ckpt``: "full" or ("block_skip", n_layer)."""
    from finetrainers_b200.model import apply_activation_checkpointing
    from finetrainers_b200.trainer import SFTTrainStep
    torch.manual_seed(seed)
    _, bm = _pair(2, r=16, seed=seed, **SMALL)
    if ckpt:
        apply_activation_checkpointing(bm, *((ckpt,) if isinstance(ckpt, str) else ckpt))
    st = SFTTrainStep(bm, flow_weighting_scheme="logit_normal", use_cuda_graph=graph, seed=seed, lr=1e-4,
                      gradient_accumulation_steps=accum)
    bt = _batch(seed=seed + 1, **shape)
    losses = []
    B = 1
    cond = {"encoder_hidden_states": bt["ehs"].cuda()}
    for _ in range(steps):
        lat = {"latents": bt["moments"].cuda(), "latents_mean": bt["mean"].expand(B, 16).cuda(),
               "latents_std": bt["std"].expand(B, 16).cuda()}
        st.train_step(cond, lat)
        losses.append(float(st.loss_buf))
    torch.cuda.synchronize()
    assert st.opt_step == steps // accum
    return losses, bm.lora_flat.detach().clone()


def test_wan_graph_checkpointing_and_seeds_bit_identical():
    """CUDA graphs, "full" and "block_skip" checkpointing and a second seeded run give the eager keep-all step's bits;
    with gradient accumulation (two micro-steps per optimizer step, clipped after each) the graph replays give the
    eager bits too."""
    base_l, base_p = _run(4)
    for kw in (dict(graph=True), dict(ckpt="full"), dict(ckpt=("block_skip", 2)), dict()):
        l, p = _run(4, **kw)
        assert l == base_l, (kw, l, base_l)
        assert torch.equal(p, base_p), kw
    acc_l, acc_p = _run(6, accum=2)
    assert not torch.equal(acc_p, base_p)
    l, p = _run(6, accum=2, graph=True)
    assert l == acc_l and torch.equal(p, acc_p)


def test_wan_grad_accumulation_sums_micro_gradients():
    """Two micro-steps with accumulation 2 leave the sum of the two micro-step gradients in the flat buffer."""
    from finetrainers_b200.trainer import SFTTrainStep
    _, bm = _pair(2, r=16, **SMALL)
    st = SFTTrainStep(bm, flow_weighting_scheme="none", gradient_accumulation_steps=2)
    gs = []
    for i in range(2):
        before = bm.lora_grad_flat.clone()
        _micro(st, _batch(F=2, H=8, W=12, L=32, seed=200 + i))
        gs.append(bm.lora_grad_flat - before)
    torch.cuda.synchronize()
    assert st.micro == 2 and gs[0].abs().max() > 0 and gs[1].abs().max() > 0
    assert torch.allclose(bm.lora_grad_flat, gs[0] + gs[1], rtol=1e-4, atol=1e-9)


def test_wan_seeded_runs_20_steps_bit_identical():
    a_l, a_p = _run(20)
    b_l, b_p = _run(20)
    assert all(math.isfinite(x) for x in a_l)
    assert a_l == b_l and torch.equal(a_p, b_p)


def test_wan_soak_40_steps():
    l, p = _run(40, graph=True, shape=dict(F=1, H=4, W=8, L=16))
    assert all(math.isfinite(x) for x in l) and torch.isfinite(p).all()


def test_wan_public_forward_matches_step():
    """spec.forward through the public forward (patchify, engine, unpatchify) computes the fused step's target and
    loss, and its autograd backward the fused step's adapter gradients bit for bit; the no-grad inference plan gives
    the same prediction."""
    from finetrainers_b200.trainer import SFTTrainStep
    from finetrainers_b200.wan import WanModelSpecification
    bt = _batch(F=2, H=8, W=12, L=64)
    _, fused = _pair(2, r=16, **SMALL)
    st = SFTTrainStep(fused, flow_weighting_scheme="none")
    loss_f = _micro(st, bt).item()
    _, bm = _pair(2, r=16, **SMALL)
    spec = WanModelSpecification(bm.cfg)
    lat = {"latents": bt["moments"].cuda(), "latents_mean": bt["mean"].cuda(), "latents_std": bt["std"].cuda()}
    pred, target, _ = spec.forward(bm, {"encoder_hidden_states": bt["ehs"].cuda()}, lat, bt["sigmas"].cuda(),
                                   noise=bt["noise"].cuda(), posterior_noise=bt["eps"].cuda())
    assert set(lat) == {"hidden_states"} and pred.shape == target.shape == (1, 16, 2, 8, 12)
    xt, tg = O.prologue(bt["moments"].cuda(), bt["mean"].cuda(), bt["std"].cuda(), bt["eps"].cuda(),
                        bt["noise"].cuda(), bt["sigmas"].cuda())
    _same(target, tg, "target")
    loss = (pred.float() - target.float()).pow(2).mean()  # the reference's loss at B = 1, weight 1
    loss.backward()
    assert abs(loss.item() - loss_f) / loss_f < 1e-5, (loss.item(), loss_f)
    # the loss gradient reaches the engine as the same bf16 dpred (2 (p - t) / n rounded once), so the adapter
    # gradients have the same bits
    gf = dict(fused.named_parameters())
    for n, p in bm.named_parameters():
        if "lora_" in n:
            assert torch.equal(p.grad, gf[n].grad), n
    with torch.no_grad():
        pred2 = bm(xt, (bt["sigmas"].cuda() * 1000.0).long(), bt["ehs"].cuda())[0]
    _same(pred2, pred.detach(), "no-grad inference plan vs training plan")
