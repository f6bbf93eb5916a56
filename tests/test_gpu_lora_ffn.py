"""GPU: LoRA on the feed-forward projections (attention set + ff.net.0.proj + ff.net.2).

(1) The split-K reduction kernel: the split product against the fp64 product element by element, the reduction alone bit
for bit against an fp32 sum in slice order, the bytes around its output window untouched, and its argument checks.
(2) The step against the fp32 oracle at SMALL size and at full width (D = 2048, S = 2688: the real split-K shape).
(3) Exact identities: a power-of-two scaling moved into B, run-to-run, CUDA graph against eager, the trainer's block-range
backward against one whole backward, and fp8-stored base weights against a bf16 model holding the fp8-rounded weights."""
import copy

import pytest
import torch

from _util import (SMALL, absmm64, bf16_ulp, check_bound, check_sentinel, mm64, rel_err, run_b200_micro,
                   sentinel_buffer, window)

pytestmark = pytest.mark.gpu

FFN_LIST = ["to_q", "to_k", "to_v", "to_out.0", "ff.net.0.proj", "ff.net.2"]
FFN_RX = "(transformer_blocks|single_transformer_blocks).*(to_q|to_k|to_v|to_out.0|ff.net.0.proj|ff.net.2)"
BATCHES = {"ragged": (2, 2, 4, 9, 24), "m64": (2, 2, 4, 8, 32)}
GAMMA = 2.0 ** -16   # fp32 accumulation error scale of the GEMM (tests/test_gpu_gemm.py)


# ---- (1) the kernel ---------------------------------------------------------------------------------------------------
def _split_product(ops, x, W, b_mn, s, part):
    """part[z] = x[:, z kk:(z+1) kk] @ W-slice^T in fp32, z < s (the model's split launch)."""
    M, K = x.shape
    N = W.shape[1] if b_mn else W.shape[0]
    kk = K // s
    ops.gemm(x, W, part, M=M, N=N, K=kk, b_mn=b_mn, ldc=N, batch=s, a_boff=(0, kk), b_boff=(kk, 0) if b_mn else (0, kk),
             c_boff=M * N, epi=ops.EPI_F32_STORE)


@pytest.mark.parametrize("b_mn", [False, True], ids=["kmajor", "mnmajor"])
@pytest.mark.parametrize("s", list(range(1, 17)))
def test_split_product_matches_fp64(s, b_mn):
    """Ragged M = 200, N = 64, K = 64 s 3 (three k-blocks per slice), alpha 0.75; out is a column window at offset 24 of
    a matrix with ldc = 136 whose other bytes hold sentinels.  Two runs are bit-identical."""
    from finetrainers_b200 import ops
    torch.manual_seed(s)
    M, N, K, alpha, off, ldc = 200, 64, 64 * s * 3, 0.75, 24, 136
    x = torch.randn(M, K, device="cuda").bfloat16()
    W = torch.randn(N, K, device="cuda").bfloat16()
    Wop = W.t().contiguous() if b_mn else W
    part = torch.empty(s, M, N, dtype=torch.float32, device="cuda")
    buf = sentinel_buffer(M * ldc + 64, torch.bfloat16)
    out = window(buf, off, M, N, ldc)
    outs = []
    for _ in range(2):
        _split_product(ops, x, Wop, b_mn, s, part)
        ops.splitk_reduce_bf16(part, out, s, M, N, alpha=alpha, ldc=ldc)
        torch.cuda.synchronize()
        outs.append(out.clone())
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
    ref = alpha * mm64(x, W)
    bound = bf16_ulp(ref) + alpha * GAMMA * absmm64(x, W)
    check_bound(out, ref, bound, f"split-K s={s}")
    check_sentinel(buf, [out], f"split-K s={s}")


@pytest.mark.parametrize("s", [1, 2, 3, 7, 16])
def test_reduction_is_the_fp32_sum_in_slice_order(s):
    """The reduction alone: bit for bit bf16_rn(alpha * (((p0 + p1) + p2) + ...)) in fp32."""
    from finetrainers_b200 import ops
    torch.manual_seed(100 + s)
    M, N = 77, 40
    part = torch.randn(s, M, N, device="cuda") * torch.logspace(-3, 3, N, device="cuda")
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    ops.splitk_reduce_bf16(part, out, s, M, N, alpha=-1.5)
    acc = part[0].clone()
    for z in range(1, s):
        acc = acc + part[z]
    want = (acc * -1.5).bfloat16()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), want.view(torch.int16))


def test_reduction_refuses_bad_arguments():
    from finetrainers_b200 import ops, lib
    part = torch.zeros(4, 64, 64, dtype=torch.float32, device="cuda")
    out = torch.zeros(64, 80, dtype=torch.bfloat16, device="cuda")
    cases = [("-5", dict(part=part, out=out, splits=0, M=64, N=64)),
             ("-5", dict(part=part, out=out, splits=ops.SPLITK_MAX + 1, M=64, N=64)),
             ("-5", dict(part=None, out=out, splits=4, M=64, N=64)),
             ("-5", dict(part=part, out=None, splits=4, M=64, N=64)),
             ("-1", dict(part=part, out=out, splits=4, M=0, N=64)),
             ("-1", dict(part=part, out=out, splits=4, M=64, N=12)),
             ("-1", dict(part=part, out=out, splits=4, M=64, N=64, ldc=56)),
             ("-2", dict(part=part, out=out, splits=4, M=64, N=64, ldc=68)),
             ("-2", dict(part=part, out=out.view(-1)[1:], splits=4, M=32, N=64, ldc=80)),
             ("-2", dict(part=part.view(-1)[2:], out=out, splits=2, M=32, N=64, ldc=80))]
    for code, kw in cases:
        with pytest.raises(lib.B2DError, match=f"code {code}"):
            ops.splitk_reduce_bf16(**kw)
    # a slice that is not a whole number of 64-deep k-blocks is refused by the split GEMM (batch offset along K)
    x = torch.zeros(64, 192, dtype=torch.bfloat16, device="cuda")
    W = torch.zeros(64, 192, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(lib.B2DError, match="code -1"):
        _split_product(ops, x, W, False, 2, part)
    torch.cuda.synchronize()
    assert out.abs().max().item() == 0


# ---- (2) against the oracle ------------------------------------------------------------------------------------------
def _ffn_pair(cfg_kwargs, rank, alpha, seed=0, lora_b_std=0.02, targets=FFN_LIST):
    """oracle (CPU, fp32 math, bf16-valued base weights) with adapters on the attention and feed-forward linears + the
    H100 model with identical parameters."""
    from oracle import ltx_oracle as O
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    om = O.LTXTransformerOracle(O.LTXConfig(**cfg_kwargs))
    O.add_lora(om, rank, alpha)
    for blk in om.transformer_blocks:
        blk.ff.net[0].proj = O.LoraLinear(blk.ff.net[0].proj, rank, alpha)
        blk.ff.net[2] = O.LoraLinear(blk.ff.net[2], rank, alpha)
    O.synthetic_init_(om, seed=seed, lora_b_std=lora_b_std)
    with torch.no_grad():
        for n, p in om.named_parameters():
            if "lora_" not in n:
                p.copy_(p.to(torch.bfloat16).float())
    bm = B200LTXTransformer(LTXConfig(**cfg_kwargs), torch.bfloat16, "cuda")
    bm.add_adapter(rank, alpha, target_modules=targets)
    assert bm.lora_ffn
    bm.load_state_dict(om.state_dict(), strict=True)
    bm.prepare()
    return O, om, bm


def _grad_errors(bm, om):
    og = dict(om.named_parameters())
    errs = {}
    for n, p in bm.named_parameters():
        if "lora_" in n:
            go = og[n].grad
            assert go is not None and go.abs().max().item() > 0, n
            errs[n] = (p.grad.float().cpu() - go).abs().max().item() / go.abs().max().item()
    return errs


@pytest.mark.parametrize("shape", list(BATCHES))
@pytest.mark.parametrize("rank,alpha", [(16, 16), (16, 64), (64, 64), (64, 32), (128, 128), (128, 256)])
def test_small_model_step_matches_oracle(rank, alpha, shape):
    O, om, bm = _ffn_pair(SMALL, rank, alpha)
    B, F, H, W, L = BATCHES[shape]
    batch = O.make_synthetic_batch(om.cfg, B, F, H, W, text_len=L, seed=7, text_scale=1.0)
    loss_o, pred_o = O.oracle_step(om, {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()})
    st, loss_b, pred_b = run_b200_micro(bm, batch)
    loss_err = abs(loss_b - loss_o.item()) / abs(loss_o.item())
    assert loss_err < 1e-3
    assert rel_err(pred_b, pred_o) < 3e-2
    og = dict(om.named_parameters())
    errs = _grad_errors(bm, om)
    assert len(errs) == 20 * SMALL["num_layers"]
    assert sum(".ff.net." in n for n in errs) == 4 * SMALL["num_layers"]
    gmax = max(p.grad.abs().max().item() for n, p in om.named_parameters() if "lora_" in n)
    for n, e in errs.items():
        assert og[n].grad.abs().max().item() > gmax / 300, (n, og[n].grad.abs().max().item(), gmax)
        assert e < 5e-2, (n, e)
    params = [p for n, p in om.named_parameters() if "lora_" in n]
    O.clip_grad_norm_(params, 1.0)
    opt = torch.optim.AdamW(params, lr=5e-5, betas=(0.9, 0.99), weight_decay=1e-4, eps=1e-8)
    opt.step()
    st.optimizer_step()
    torch.cuda.synchronize()
    for n, p in bm.named_parameters():
        if "lora_" in n:
            assert (p.detach().float().cpu() - og[n].detach()).abs().max().item() < 2e-4, n
    print(f"\nffn rank {rank} alpha {alpha} {shape}: loss err {loss_err:.2e}, worst grad err {max(errs.values()):.2e} "
          f"({max(errs, key=errs.get)})")


@pytest.mark.timeout(900)
def test_full_width_two_block_forward_backward_matches_oracle():
    """D = 2048, S = 2688 tokens, r = 64, two blocks, B = 1: the two K = 8192 adapter launches run split."""
    O, om, bm = _ffn_pair(dict(num_layers=2), 64, 64, targets=FFN_RX)
    assert "splitk" in bm._workspace(1, 2688, 128) and bm._workspace(1, 2688, 128)["splitk"].shape[0] > 1
    batch = O.make_synthetic_batch(om.cfg, 1, 7, 16, 24, seed=1234, text_scale=1.0)
    loss_o, pred_o = O.oracle_step(om, {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()})
    st, loss_b, pred_b = run_b200_micro(bm, batch)
    assert abs(loss_b - loss_o.item()) / abs(loss_o.item()) < 1e-3
    assert rel_err(pred_b, pred_o) < 3e-2
    errs = _grad_errors(bm, om)
    assert len(errs) == 2 * 20
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:4]
    print("\nfull-width ffn: grad errors (worst 4):", worst)
    for n, e in errs.items():
        assert e < 5e-2, (n, e, worst)
    og = dict(om.named_parameters())
    gb = torch.cat([p.grad.float().cpu().flatten() for n, p in bm.named_parameters() if "lora_" in n])
    go = torch.cat([og[n].grad.flatten() for n, p in bm.named_parameters() if "lora_" in n])
    assert torch.dot(gb, go) / (gb.norm() * go.norm()) > 0.999


# ---- (3) exact identities --------------------------------------------------------------------------------------------
def _state(rank, seed=0, nl=None):
    from oracle import ltx_oracle as O
    cfg = dict(SMALL, num_layers=nl) if nl else SMALL
    om = O.LTXTransformerOracle(O.LTXConfig(**cfg))
    O.add_lora(om, rank, rank)
    for blk in om.transformer_blocks:
        blk.ff.net[0].proj = O.LoraLinear(blk.ff.net[0].proj, rank, rank)
        blk.ff.net[2] = O.LoraLinear(blk.ff.net[2], rank, rank)
    O.synthetic_init_(om, seed=seed, lora_b_std=0.02)
    return {k: v.clone() for k, v in om.state_dict().items()}


def _model(sd, rank, alpha, nl=None):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    cfg = dict(SMALL, num_layers=nl) if nl else SMALL
    bm = B200LTXTransformer(LTXConfig(**cfg), torch.bfloat16, "cuda")
    bm.add_adapter(rank, alpha, target_modules=FFN_LIST)
    bm.load_state_dict(sd, strict=True)
    bm.prepare()
    return bm


def _batch(shape, seed=7, nl=None):
    from oracle import ltx_oracle as O
    B, F, H, W, L = BATCHES[shape]
    cfg = dict(SMALL, num_layers=nl) if nl else SMALL
    return O.make_synthetic_batch(O.LTXConfig(**cfg), B, F, H, W, text_len=L, seed=seed, text_scale=1.0)


def _assert_equal(got, want, what):
    if not torch.equal(got, want):
        diff = (got.float() - want.float()).abs()
        raise AssertionError(f"{what}: {int((diff != 0).sum())} element(s) differ, max |diff| {diff.max().item():.3g}")


@pytest.mark.parametrize("shape", list(BATCHES))
@pytest.mark.parametrize("c", [2.0, 0.5])
def test_power_of_two_scaling_moves_into_b(c, shape):
    """P = (A, B, alpha = c r) against Q = (A, c B, alpha = r), feed-forward adapters included: loss, pred and every dA
    bit-identical, every dB of P exactly c times Q's (tests/test_gpu_lora_ranks.py gives the argument)."""
    rank = 64
    sd = _state(rank)
    sd_q = {k: (v * c if "lora_B" in k else v) for k, v in sd.items()}
    bp, bq = _model(sd, rank, c * rank), _model(sd_q, rank, rank)
    batch = _batch(shape)
    _, loss_p, pred_p = run_b200_micro(bp, batch)
    _, loss_q, pred_q = run_b200_micro(bq, batch)
    assert loss_p == loss_q, (loss_p, loss_q)
    _assert_equal(pred_p, pred_q, "pred")
    gp = {n: p.grad.detach().clone() for n, p in bp.named_parameters() if "lora_" in n}
    gq = {n: p.grad.detach().clone() for n, p in bq.named_parameters() if "lora_" in n}
    assert len(gp) == 20 * SMALL["num_layers"]
    for n in gp:
        assert gq[n].abs().max().item() > 0, n
        _assert_equal(gp[n], gq[n] if "lora_A" in n else c * gq[n], n)


def test_step_is_bit_identical_run_to_run_and_under_a_cuda_graph():
    """Four optimizer steps of one model eager and of a second model under CUDA graphs (two eager warm-ups, capture,
    replay), and a third eager run: loss, pred, the flat gradient and the updated masters agree bit for bit."""
    from finetrainers_b200.trainer import SFTTrainStep
    sd = _state(64, seed=4)
    runs = []
    for graph in (False, True, False):
        bm = _model(sd, 64, 64)
        st = SFTTrainStep(bm, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=graph)
        st.spec.first_frame_conditioning_p = 0.0
        rec = []
        for i in range(4):
            b = _batch("ragged", seed=60 + i)
            cond = {"encoder_hidden_states": b["encoder_hidden_states"].cuda(),
                    "encoder_attention_mask": b["encoder_attention_mask"].cuda()}
            lat = {"latents": b["latents"].cuda(), "latents_mean": b["latents_mean"].cuda(),
                   "latents_std": b["latents_std"].cuda()}
            st.micro_step(cond, lat, sigmas=b["sigmas"].view(-1).cuda(), noise=b["noise"].cuda())
            torch.cuda.synchronize()
            ws = next(iter(bm._ws.values()))
            rec.append((st.loss_buf.clone(), ws["pred"].clone(), bm.lora_grad_flat.clone()))
            st.optimizer_step()
        torch.cuda.synchronize()
        if graph:
            assert len(st._graphs) == 1
        runs.append((rec, bm.lora_flat.clone()))
    for k in (1, 2):
        for i, (a, b) in enumerate(zip(runs[0][0], runs[k][0])):
            for what, x, y in zip(("loss", "pred", "grad"), a, b):
                _assert_equal(y, x, f"run {k} step {i} {what}")
        _assert_equal(runs[k][1], runs[0][1], f"run {k} masters")


def test_block_range_backward_is_bit_identical_to_one_backward():
    """Four blocks, backward in the trainer's four DDP ranges (top first): the flat gradient equals that of one whole
    backward bit for bit, and each range's slice is already final when its _backward_tail returns."""
    from finetrainers_b200.trainer import SFTTrainStep
    nl = 4
    bm = _model(_state(64, seed=9, nl=nl), 64, 64, nl=nl)
    st = SFTTrainStep(bm, flow_weighting_scheme="none", seed=5)
    st.spec.first_frame_conditioning_p = 0.0
    b = _batch("ragged", seed=3, nl=nl)
    cond = {"encoder_hidden_states": b["encoder_hidden_states"].cuda(),
            "encoder_attention_mask": b["encoder_attention_mask"].cuda()}
    lat = {"latents": b["latents"].cuda(), "latents_mean": b["latents_mean"].cuda(), "latents_std": b["latents_std"].cuda()}
    st.micro_step(cond, lat, sigmas=b["sigmas"].view(-1).cuda(), noise=b["noise"].cuda())
    torch.cuda.synchronize()
    whole = bm.lora_grad_flat.clone()
    assert whole.abs().max().item() > 0
    # the same micro-batch again from the static buffers, backward range by range
    bm.lora_grad_flat.zero_()
    (key, sbuf), = st._static.items()
    st._body_front(key, sbuf)
    pb = bm._per_blk
    snaps = []
    for lo, hi in [(3, 4), (2, 3), (1, 2), (0, 1)]:
        bm._backward_blocks(hi - 1, lo)
        bm._backward_tail(lo, hi)
        snaps.append((lo, hi, bm.lora_grad_flat[lo * pb:hi * pb].clone()))
    torch.cuda.synchronize()
    _assert_equal(bm.lora_grad_flat, whole, "flat gradient")
    for lo, hi, s in snaps:
        _assert_equal(s, whole[lo * pb:hi * pb], f"blocks [{lo}, {hi}) slice at its tail")
    # block 0's feed-forward adapter gradients exist although block 0 skips its dX
    assert bm.skip_block0_dx
    for n in ("ff.net.0.proj.lora_A", "ff.net.0.proj.lora_B", "ff.net.2.lora_A", "ff.net.2.lora_B"):
        p = dict(bm.named_parameters())[f"transformer_blocks.0.{n}.default.weight"]
        assert p.grad.abs().max().item() > 0, n


def test_fp8_ffn_base_weights_with_ffn_adapters_match_prerounded_bf16():
    """Layerwise fp8 (e4m3fn) storage of every cast linear, the feed-forward base weights included, with adapters on the
    feed-forward linears: bit-identical, eager and under CUDA graphs, to a bf16 model whose cast linears hold
    w.to(fp8).to(bf16); the FFN base weights stay fp8 and the adapters fp32."""
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig, apply_layerwise_casting
    from finetrainers_b200.trainer import SFTTrainStep
    fmt = torch.float8_e4m3fn
    skip = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]
    nl = 5
    cfg = LTXConfig(**dict(SMALL, num_layers=nl))
    torch.manual_seed(0)
    a = B200LTXTransformer(cfg, torch.bfloat16, "cuda")
    with torch.no_grad():
        for n, p in a.named_parameters():
            p.normal_(0, 0.05) if "norm_" not in n else p.normal_(1.0, 0.1)
    b = copy.deepcopy(a)
    apply_layerwise_casting(a, fmt, torch.bfloat16, skip)
    assert "transformer_blocks.0.ff.net.2" in a._lw_cfg["cast"]
    mods = dict(b.named_modules())
    with torch.no_grad():
        for n in a._lw_cfg["cast"]:
            for p in (mods[n].weight, mods[n].bias):
                p.copy_(p.to(fmt).to(torch.bfloat16))
    for m in (a, b):
        m.add_adapter(64, 64, target_modules=FFN_RX)
        m.prepare()
    with torch.no_grad():
        a.lora_flat.normal_(0, 0.05)
        b.lora_flat.copy_(a.lora_flat)
    assert a._lw is not None and b._lw is None
    blk = a.transformer_blocks[3]
    assert blk.ff.net[2].base_layer.weight.dtype == fmt and blk.ff.net[0].proj.base_layer.weight.dtype == fmt
    assert blk.ff.net[2].lora_A["default"].weight.dtype == torch.float32
    for graph in (False, True):
        sa, sb = (SFTTrainStep(m, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=graph) for m in (a, b))
        for s in (sa, sb):
            s.spec.first_frame_conditioning_p = 0.0
        for i in range(3 if graph else 1):
            bt = _batch("ragged", seed=100 + i, nl=nl)
            cond = {"encoder_hidden_states": bt["encoder_hidden_states"].cuda(),
                    "encoder_attention_mask": bt["encoder_attention_mask"].cuda()}
            lat = {"latents": bt["latents"].cuda(), "latents_mean": bt["latents_mean"].cuda(),
                   "latents_std": bt["latents_std"].cuda()}
            for s in (sa, sb):
                s.micro_step(dict(cond), dict(lat), sigmas=bt["sigmas"].view(-1).cuda(), noise=bt["noise"].cuda())
            torch.cuda.synchronize()
            assert torch.equal(sa.loss_buf, sb.loss_buf), (graph, i)
            wa, wb = next(iter(a._ws.values())), next(iter(b._ws.values()))
            _assert_equal(wa["pred"], wb["pred"], f"pred graph={graph} {i}")
            assert a.lora_grad_flat.abs().max().item() > 0
            _assert_equal(a.lora_grad_flat, b.lora_grad_flat, f"grad graph={graph} {i}")
            sa.optimizer_step()
            sb.optimizer_step()
            torch.cuda.synchronize()
            _assert_equal(a.lora_flat, b.lora_flat, f"masters graph={graph} {i}")
