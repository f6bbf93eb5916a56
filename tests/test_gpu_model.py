"""GPU: whole-step parity of the H100 DiT engine against the CPU oracle (restated reference; parity of the oracle
itself to real diffusers is unpinned — see oracle/ltx_oracle.py header), through the ModelSpecification / SFT-step API.
Tolerance from BASELINE.json north_star: per-step loss within 1e-3 relative."""
import pytest
import torch

from _util import build_pair, run_b200_micro, SMALL, rel_err

pytestmark = pytest.mark.gpu


def lora_grad_errors(bm, om):
    """{name: max|g_b200 - g_oracle| / max|g_oracle|} for every adapter tensor (per-tensor scale, no global floor)."""
    og = dict(om.named_parameters())
    errs = {}
    for n, p in bm.named_parameters():
        if "lora_" in n:
            go = og[n].grad
            assert go is not None and go.abs().max().item() > 0, n
            errs[n] = (p.grad.float().cpu() - go).abs().max().item() / go.abs().max().item()
    return errs


# (rank, lora_alpha) pairs: scaling alpha / rank and padded rank rp = 64 * ceil(rank / 64) decide every LoRA launch
#   (64, 64) and (16, 16)  scaling 1 at rp 64
#   (4, 8)                 scaling 2, almost all of the 64 padded rows zero
#   (16, 64)               scaling 4: --rank 16 with finetrainers' default --lora_alpha 64
#   (32, 32)               the reference's LTX example rank
#   (96, 64)               scaling 2/3 (not a power of two), padded inside rp 128
#   (128, 128)             the reference's LTX smoke-script rank
#   (192, 96)              scaling 1/2; the dB GEMM's second 128-wide n-tile is ragged; K2 = 3 rp = 576 in the QKV dX GEMM
#   (256, 256)             K2 = 768 in the QKV dX GEMM
RANK_ALPHA = [(64, 64), (16, 16), (4, 8), (16, 64), (32, 32), (96, 64), (128, 128), (192, 96), (256, 256)]
# batch shapes (B, F, H, W, text_len): "ragged" has R = B*S = 144 and RL = 48, not multiples of 64, so the adapter
# weight-gradient GEMMs run one block at a time; "m64" has R = 128 and RL = 64, so they run block-stacked
SMALL_BATCHES = {"ragged": (2, 2, 4, 9, 24), "m64": (2, 2, 4, 8, 32)}


def _small_cases():
    cases = []
    for shape in SMALL_BATCHES:
        for r, a in RANK_ALPHA:
            # the two configurations that predate the alpha parameter keep their ids
            pid = str(r) if (shape == "ragged" and r == a and r in (64, 16)) else f"r{r}-a{a}-{shape}"
            cases.append(pytest.param(r, a, shape, id=pid))
    return cases


@pytest.mark.parametrize("rank,alpha,shape", _small_cases())
def test_small_model_step_matches_oracle(rank, alpha, shape):
    O, om, bm = build_pair(SMALL, rank, alpha=alpha)
    assert bm.lora_scaling == alpha / rank
    # S = 72 / 64: ragged vs the 128-row tiles.  text_scale=1.0: the cross-attention logits get an O(1) spread, so the attn2
    # to_q/to_k adapter gradients are as large as the others (with the 0.1 throughput setting the text softmax is uniform
    # and those gradients cancel to rounding noise) and EVERY adapter tensor is held to the same per-tensor bound.
    B, F, H, W, L = SMALL_BATCHES[shape]
    batch = O.make_synthetic_batch(om.cfg, B, F, H, W, text_len=L, seed=7, text_scale=1.0)
    loss_o, pred_o = O.oracle_step(om, {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()})
    st, loss_b, pred_b = run_b200_micro(bm, batch)
    loss_err = abs(loss_b - loss_o.item()) / abs(loss_o.item())
    assert loss_err < 1e-3
    assert rel_err(pred_b, pred_o) < 3e-2
    og = dict(om.named_parameters())
    errs = lora_grad_errors(bm, om)
    assert len(errs) == 2 * 8 * SMALL["num_layers"]
    gmax = max(p.grad.abs().max().item() for n, p in om.named_parameters() if "lora_" in n)
    for n, e in errs.items():
        # every adapter gradient is within 300x of the largest one (nothing is rounding noise), and within 5 % of ITS OWN scale
        assert og[n].grad.abs().max().item() > gmax / 300, (n, og[n].grad.abs().max().item(), gmax)
        assert e < 5e-2, (n, e)
    # optimizer step: matches torch AdamW + clip on the oracle's gradients
    params = [p for n, p in om.named_parameters() if "lora_" in n]
    O.clip_grad_norm_(params, 1.0)
    opt = torch.optim.AdamW(params, lr=5e-5, betas=(0.9, 0.99), weight_decay=1e-4, eps=1e-8)
    opt.step()
    st.optimizer_step()
    torch.cuda.synchronize()
    pdiff = 0.0
    for n, p in bm.named_parameters():
        if "lora_" in n:
            dn = (p.detach().float().cpu() - og[n].detach()).abs().max().item()
            pdiff = max(pdiff, dn)
            assert dn < 2e-4, n
    print(f"\nrank {rank} alpha {alpha} {shape}: loss err {loss_err:.2e}, worst grad err {max(errs.values()):.2e} "
          f"({max(errs, key=errs.get)}), worst AdamW param diff {pdiff:.2e}")


def _full_width_two_block_parity(rank, alpha):
    cfgk = dict(num_layers=2)
    O, om, bm = build_pair(cfgk, rank, alpha=alpha)
    batch = O.make_synthetic_batch(om.cfg, 1, 7, 16, 24, seed=1234, text_scale=1.0)
    loss_o, pred_o = O.oracle_step(om, {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()})
    st, loss_b, pred_b = run_b200_micro(bm, batch)
    loss_err = abs(loss_b - loss_o.item()) / abs(loss_o.item())
    assert loss_err < 1e-3
    assert rel_err(pred_b, pred_o) < 3e-2
    errs = lora_grad_errors(bm, om)
    assert len(errs) == 2 * 16
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:4]
    print(f"\nfull-width rank {rank} alpha {alpha}: loss err {loss_err:.2e}, grad errors (worst 4):", worst)
    for n, e in errs.items():
        # per-tensor relative bound, no global floor; cross-attention q/k adapters included
        assert e < 5e-2, (n, e, worst)
    # cosine similarity of the whole flat gradient
    og = dict(om.named_parameters())
    gb = torch.cat([p.grad.float().cpu().flatten() for n, p in bm.named_parameters() if "lora_" in n])
    go = torch.cat([og[n].grad.flatten() for n, p in bm.named_parameters() if "lora_" in n])
    assert torch.dot(gb, go) / (gb.norm() * go.norm()) > 0.999
    assert abs(gb.norm() / go.norm() - 1) < 1e-2


@pytest.mark.timeout(600)
def test_full_width_two_block_forward_backward_matches_oracle():
    """BASELINE width (D=2048, H=32, S=2688 tokens = 21 full 128-row tiles, L=128 text keys, r=64), 2 blocks, B=1:
    forward loss AND every LoRA gradient against the fp32 oracle.  This is the shape the step's dominant kernels run
    at (wide GEMM tiles, multi-tile attention forward and backward), which the S=72 small-model tests never reach."""
    _full_width_two_block_parity(64, 64)


@pytest.mark.timeout(600)
def test_full_width_two_block_rank128_alpha256_matches_oracle():
    """The same at rank 128, lora_alpha 256: padded rank 128 (K2 = 384 in the QKV dX GEMM, 128-wide dB tiles) and
    scaling 2 on the block-stacked weight-gradient path (R = 2688 and RL = 128 are multiples of 64) at the step's real
    GEMM shapes."""
    _full_width_two_block_parity(128, 256)


def test_twenty_step_trajectory_bounds_bf16_lora_operand_drift():
    """The reference keeps the LoRA branch in fp32 under DDP (trainer.py:130-136); this engine keeps fp32 MASTER weights
    and gradients but feeds bf16 copies of A/B to the tensor cores.  20 optimizer steps (lr 1e-3, clip, AdamW) on the
    same data stream as the fp32 oracle bound what that costs: the per-step loss stays within the north_star's 1e-3
    relative on every step, and the accumulated adapter update keeps direction and length."""
    from finetrainers_b200.trainer import SFTTrainStep
    O, om, bm = build_pair(SMALL, 64, seed=3)
    st = SFTTrainStep(bm, flow_weighting_scheme="none", lr=1e-3, seed=5)
    st.spec.first_frame_conditioning_p = 0.0
    params = [p for n, p in om.named_parameters() if "lora_" in n]
    opt = torch.optim.AdamW(params, lr=1e-3, betas=(0.9, 0.99), weight_decay=1e-4, eps=1e-8)
    p0 = {n: p.detach().clone() for n, p in om.named_parameters() if "lora_" in n}
    worst = 0.0
    for i in range(20):
        batch = O.make_synthetic_batch(om.cfg, 2, 2, 4, 9, text_len=24, seed=500 + i, text_scale=1.0)
        cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(), "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}
        lat = {"latents": batch["latents"].cuda(), "latents_mean": batch["latents_mean"].cuda(), "latents_std": batch["latents_std"].cuda()}
        st.micro_step(cond, lat, sigmas=batch["sigmas"].view(-1).cuda(), noise=batch["noise"].cuda())
        torch.cuda.synchronize()
        loss_b = st.loss_buf.item()
        opt.zero_grad(set_to_none=True)
        loss_o, _ = O.oracle_step(om, {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()})
        rel = abs(loss_b - loss_o.item()) / abs(loss_o.item())
        worst = max(worst, rel)
        assert rel < 1e-3, (i, loss_b, loss_o.item(), rel)
        O.clip_grad_norm_(params, 1.0)
        opt.step()
        st.optimizer_step()
    torch.cuda.synchronize()
    print("20-step worst relative loss difference:", worst)
    og = dict(om.named_parameters())
    db = torch.cat([(p.detach().float().cpu() - p0[n]).flatten() for n, p in bm.named_parameters() if "lora_" in n])
    do = torch.cat([(og[n].detach() - p0[n]).flatten() for n, p in bm.named_parameters() if "lora_" in n])
    assert torch.dot(db, do) / (db.norm() * do.norm()) > 0.98
    assert abs(db.norm() / do.norm() - 1) < 0.03


def test_small_model_through_finetrainers_style_loss():
    """The path finetrainers' own trainer takes: pred from spec.forward, loss in torch, loss.backward()."""
    from finetrainers_b200.specification import LTXVideoModelSpecification
    O, om, bm = build_pair(SMALL, 64)
    batch = O.make_synthetic_batch(om.cfg, 1, 2, 4, 8, text_len=16, seed=3)
    loss_o, _ = O.oracle_step(om, {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()})
    spec = LTXVideoModelSpecification(bm.cfg)
    spec.first_frame_conditioning_p = 0.0
    cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(), "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}
    lat = {"latents": batch["latents"].cuda(), "latents_mean": batch["latents_mean"].cuda(), "latents_std": batch["latents_std"].cuda()}
    pred, target, sig = spec.forward(bm, cond, lat, batch["sigmas"].cuda(), noise=batch["noise"].cuda())
    loss = (pred.float() - target.float()).pow(2).mean(list(range(1, 3))).mean()  # trainer.py:474-478
    loss.backward()
    assert abs(loss.item() - loss_o.item()) / loss_o.item() < 1e-3
    og = dict(om.named_parameters())
    n = "transformer_blocks.1.attn1.to_q.lora_B.default.weight"
    g = dict(bm.named_parameters())[n].grad
    assert rel_err(g.cpu(), og[n].grad) < 5e-2
    assert "hidden_states" in lat and "latents" not in lat  # same dict mutation as the reference forward


def test_zero_lora_b_is_identity_and_deterministic():
    """Properties at the BASELINE width (D=2048, S=2688), 2 blocks: (a) B = 0 adapters change nothing (bitwise) versus
    the model without adapters, (b) forward is bitwise deterministic, (c) dA == 0 exactly when B == 0."""
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    from oracle import ltx_oracle as O
    cfg = LTXConfig(num_layers=2)
    torch.manual_seed(0)
    base = B200LTXTransformer(cfg, torch.bfloat16, "cuda")
    with torch.no_grad():
        for n, p in base.named_parameters():
            p.normal_(0, 0.02) if "norm_" not in n else p.fill_(1.0)
    sd = {k: v.clone() for k, v in base.state_dict().items()}
    base.prepare()
    lora = B200LTXTransformer(cfg, torch.bfloat16, "cuda")
    lora.load_state_dict(sd)
    lora.add_adapter(64, 64)  # B initialised to zero (peft init_lora_weights=True)
    lora.prepare()
    batch = O.make_synthetic_batch(O.LTXConfig(num_layers=2), 1, 7, 16, 24, seed=11)
    x = torch.randn(1, 2688, 128, device="cuda").bfloat16()
    args = dict(encoder_hidden_states=batch["encoder_hidden_states"].cuda(), timestep=torch.tensor([500], device="cuda"),
                encoder_attention_mask=batch["encoder_attention_mask"].cuda(), num_frames=7, height=16, width=24,
                rope_interpolation_scale=[8 / 25, 32, 32])
    with torch.no_grad():
        p0 = base(x, **args)[0].clone()
        p1 = lora(x, **args)[0].clone()
        p2 = lora(x, **args)[0].clone()
    assert torch.equal(p1, p2)
    assert torch.equal(p0, p1)
    out = lora(x, **args)[0]
    out.backward(torch.randn_like(out))
    torch.cuda.synchronize()
    for n, p in lora.named_parameters():
        if "lora_A" in n:
            assert p.grad.abs().max().item() == 0.0, n
        if "lora_B" in n:
            assert p.grad.abs().max().item() > 0.0, n


@pytest.mark.timeout(900)
def test_full_size_forward_loss_matches_oracle():
    """BASELINE config 2 (LTX-2B, 49x512x768 -> 2688 tokens, B=1, r=64): forward loss vs the fp32-math oracle on CPU."""
    from oracle import ltx_oracle as O
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    ocfg = O.LTXConfig()
    om = O.LTXTransformerOracle(ocfg)
    O.add_lora(om, 64, 64)
    O.synthetic_init_(om, seed=0, lora_b_std=0.02)
    with torch.no_grad():
        for n, p in om.named_parameters():
            if "lora_" not in n:
                p.copy_(p.to(torch.bfloat16).float())
    bm = B200LTXTransformer(LTXConfig(), torch.bfloat16, "cuda")
    bm.add_adapter(64, 64)
    bm.load_state_dict(om.state_dict(), strict=True)
    bm.prepare()
    batch = O.make_synthetic_batch(ocfg, 1, 7, 16, 24, seed=1234)
    st, loss_b, pred_b = run_b200_micro(bm, batch)
    with torch.no_grad():
        loss_o, pred_o = O.oracle_step(om, {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()},
                                       backward=False)
    assert abs(loss_b - loss_o.item()) / abs(loss_o.item()) < 1e-3
    assert rel_err(pred_b, pred_o) < 5e-2


def test_cuda_graph_step_matches_eager_and_grad_accumulation():
    """The captured step (one CUDA graph replay per micro-step) reproduces the eager step; two accumulated micro-steps
    equal one step on the concatenated batch statistics (loss averaged, gradients summed/scaled: trainer.py:479-480)."""
    from finetrainers_b200.trainer import SFTTrainStep
    from oracle import ltx_oracle as O
    losses, params = {}, {}
    for mode in ("eager", "graph"):
        _, om, bm = build_pair(SMALL, 64, seed=1)
        st = SFTTrainStep(bm, flow_weighting_scheme="none", use_cuda_graph=(mode == "graph"), seed=5)
        st.spec.first_frame_conditioning_p = 0.0
        ls = []
        for i in range(5):  # graph mode: 2 eager warm-ups, capture on the 3rd call, replays after
            batch = O.make_synthetic_batch(om.cfg, 2, 2, 4, 8, text_len=16, seed=100 + i)
            cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(), "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}
            lat = {"latents": batch["latents"].cuda(), "latents_mean": batch["latents_mean"].cuda(), "latents_std": batch["latents_std"].cuda()}
            m = st.train_step(cond, lat, sigmas=batch["sigmas"].view(-1).cuda(), noise=batch["noise"].cuda(), sync_metrics=True)
            ls.append(m["train/global_avg_loss"])
        losses[mode] = ls
        params[mode] = bm.lora_flat.clone()
    for a, b in zip(losses["eager"], losses["graph"]):
        assert abs(a - b) / abs(a) < 1e-4, (losses["eager"], losses["graph"])
    assert (params["eager"] - params["graph"]).abs().max().item() < 1e-5
    # gradient accumulation: 2 micro-steps with accum=2 leave grad = mean of the two micro-gradients
    _, om, bm = build_pair(SMALL, 64, seed=1)
    st = SFTTrainStep(bm, flow_weighting_scheme="none", gradient_accumulation_steps=2)
    st.spec.first_frame_conditioning_p = 0.0
    gs = []
    for i in range(2):
        batch = O.make_synthetic_batch(om.cfg, 1, 2, 4, 8, text_len=16, seed=200 + i)
        cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(), "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}
        lat = {"latents": batch["latents"].cuda(), "latents_mean": batch["latents_mean"].cuda(), "latents_std": batch["latents_std"].cuda()}
        before = bm.lora_grad_flat.clone()
        st.micro_step(cond, lat, sigmas=batch["sigmas"].view(-1).cuda(), noise=batch["noise"].cuda())
        gs.append(bm.lora_grad_flat - before)
    torch.cuda.synchronize()
    assert st.micro == 2 and gs[0].abs().max() > 0 and gs[1].abs().max() > 0
    assert torch.allclose(bm.lora_grad_flat, gs[0] + gs[1], rtol=1e-4, atol=1e-9)


def test_grad_accumulation_clips_after_every_micro_step_like_the_reference():
    """trainer.py:486-493 calls clip_grad_norm_ after every micro-step's backward, accumulation boundary or not: with a
    max_grad_norm far below the gradient norm the partially accumulated gradient is rescaled before the second micro-step
    adds to it.  The b200 train_step must leave the same flat gradient direction / length as torch autograd on the oracle
    run the reference's way, and the same AdamW update."""
    from finetrainers_b200.trainer import SFTTrainStep
    O, om, bm = build_pair(SMALL, 64, seed=4)
    max_norm = 1e-3
    st = SFTTrainStep(bm, flow_weighting_scheme="none", lr=1e-3, max_grad_norm=max_norm, gradient_accumulation_steps=2, seed=3)
    st.spec.first_frame_conditioning_p = 0.0
    params = [p for n, p in om.named_parameters() if "lora_" in n]
    opt = torch.optim.AdamW(params, lr=1e-3, betas=(0.9, 0.99), weight_decay=1e-4, eps=1e-8)
    p0 = {n: p.detach().clone() for n, p in om.named_parameters() if "lora_" in n}
    opt.zero_grad(set_to_none=True)
    norms = []
    for i in range(2):
        batch = O.make_synthetic_batch(om.cfg, 1, 2, 4, 8, text_len=16, seed=400 + i, text_scale=1.0)
        cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(), "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}
        lat = {"latents": batch["latents"].cuda(), "latents_mean": batch["latents_mean"].cuda(), "latents_std": batch["latents_std"].cuda()}
        if i == 0:
            st.train_step(cond, lat, sigmas=batch["sigmas"].view(-1).cuda(), noise=batch["noise"].cuda())
            torch.cuda.synchronize()
            # after the first micro-step the accumulated gradient has been clipped to max_norm
            assert abs(bm.lora_grad_flat.norm().item() - max_norm) / max_norm < 1e-3
        else:
            st.micro_step(cond, lat, sigmas=batch["sigmas"].view(-1).cuda(), noise=batch["noise"].cuda())
        fb = {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()}
        pred, target, sig = O.spec_forward(om, fb["latents"], fb["latents_mean"], fb["latents_std"], fb["encoder_hidden_states"],
                                           fb["encoder_attention_mask"], fb["sigmas"], noise=fb["noise"])
        (O.sft_loss(pred, target, sig) / 2).backward()          # trainer.py:479-480: loss / gradient_accumulation_steps
        norms.append(float(O.clip_grad_norm_(params, max_norm)))  # every micro-step
    torch.cuda.synchronize()
    # second micro-step: (clipped first gradient, norm 1e-3) + (raw second gradient): dominated by the second, as in the oracle
    g_b = bm.lora_grad_flat.norm().item()
    assert abs(g_b - norms[1]) / norms[1] < 3e-2, (g_b, norms)
    assert norms[0] > 10 * max_norm      # the first clip really was active
    opt.step()
    st.optimizer_step()
    torch.cuda.synchronize()
    og = dict(om.named_parameters())
    checked = 0
    for n, p in bm.named_parameters():
        if "lora_" in n:
            db = (p.detach().float().cpu() - p0[n]).flatten()
            do = (og[n].detach() - p0[n]).flatten()
            if do.norm() == 0:
                continue
            cos = torch.dot(db, do) / (db.norm() * do.norm())
            assert cos > 0.95 and abs(db.norm() / do.norm() - 1) < 0.05, (n, cos.item(), (db.norm() / do.norm()).item())
            checked += 1
    assert checked >= 30


def test_three_step_trajectory_first_frame_conditioning_and_lr_schedule():
    """Three optimizer steps of the b200 step against the oracle run the way the reference trainer runs them: first-frame
    conditioning branch taken (base_specification.py:298-310), sigma-dependent loss weights, clip + AdamW under a
    LambdaLR warm-up.  Per-step loss within 1e-3 (north_star); the 3-step adapter updates agree in direction and length."""
    from finetrainers_b200.lr_schedule import lr_factor_fn
    from finetrainers_b200.trainer import SFTTrainStep
    O, om, bm = build_pair(SMALL, 64, seed=2)
    st = SFTTrainStep(bm, flow_weighting_scheme="none", lr=1e-3, lr_scheduler="linear", lr_warmup_steps=2, train_steps=10, seed=11)
    st.spec.first_frame_conditioning_p = 1.0
    params = [p for n, p in om.named_parameters() if "lora_" in n]
    opt = torch.optim.AdamW(params, lr=1e-3, betas=(0.9, 0.99), weight_decay=1e-4, eps=1e-8)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lr_factor_fn("linear", num_warmup_steps=2, num_training_steps=10))
    p0 = {n: p.detach().clone() for n, p in om.named_parameters() if "lora_" in n}
    for i in range(3):
        batch = O.make_synthetic_batch(om.cfg, 2, 3, 4, 6, text_len=20, seed=300 + i, text_scale=1.0)
        cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(), "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}
        lat = {"latents": batch["latents"].cuda(), "latents_mean": batch["latents_mean"].cuda(), "latents_std": batch["latents_std"].cuda()}
        st.micro_step(cond, lat, sigmas=batch["sigmas"].view(-1).cuda(), noise=batch["noise"].cuda())
        torch.cuda.synchronize()
        loss_b = st.loss_buf.item()
        sig_ff = next(iter(st._static.values()))["sig_ff"].float().cpu()
        assert (sig_ff <= 0.25 + 1e-6).all() and (sig_ff <= batch["sigmas"].view(-1) + 1e-6).all()
        fb = {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()}
        opt.zero_grad(set_to_none=True)
        pred, target, sig = O.spec_forward(om, fb["latents"], fb["latents_mean"], fb["latents_std"], fb["encoder_hidden_states"],
                                           fb["encoder_attention_mask"], fb["sigmas"], noise=fb["noise"],
                                           first_frame_sigma=sig_ff.view(fb["sigmas"].shape))
        loss_o = O.sft_loss(pred, target, sig)
        loss_o.backward()
        assert abs(loss_b - loss_o.item()) / abs(loss_o.item()) < 1e-3, (i, loss_b, loss_o.item())
        O.clip_grad_norm_(params, 1.0)
        assert abs(st._lr_factor(i) * 1e-3 - opt.param_groups[0]["lr"]) < 1e-12
        opt.step()
        sched.step()
        st.optimizer_step()
    torch.cuda.synchronize()
    # Adam normalises every element to ~+-lr, so an element whose gradient is near zero moves by O(lr) in either
    # implementation; compare the UPDATE vector of every adapter tensor (cross-attention q/k included: the text
    # embeddings are conditioned, see test_small_model_step_matches_oracle) by direction and length.
    og = dict(om.named_parameters())
    checked = 0
    for n, p in bm.named_parameters():
        if "lora_" in n:
            db = (p.detach().float().cpu() - p0[n]).flatten()
            do = (og[n].detach() - p0[n]).flatten()
            if do.norm() == 0:
                continue
            cos = torch.dot(db, do) / (db.norm() * do.norm())
            assert cos > 0.95 and abs(db.norm() / do.norm() - 1) < 0.05, (n, cos.item(), (db.norm() / do.norm()).item())
            checked += 1
    assert checked >= 30


@pytest.mark.timeout(600)
def test_full_size_soak_gradients_stay_finite_and_sane():
    """40 optimizer steps of the full-size model (28 blocks, 2688 tokens), eager, metrics read every step: the gradient norm
    must stay finite and of order one.  This is the test that was missing when the dQ pass of the attention backward had a
    branch that produced a few rows of garbage (|dq| ~ 1e37, some inf / NaN) once every ~20 steps - invisible to every
    single-step parity test and to the bench, fatal to a real run (profiles/r2b_attention_backward_nan.md).  Before the fix
    a 40-step run failed with probability ~0.85."""
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    from finetrainers_b200.trainer import SFTTrainStep
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = B200LTXTransformer(LTXConfig(), torch.bfloat16, dev)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if "scale_shift_table" in name:
                p.normal_(0, 1.0 / p.shape[-1] ** 0.5)
            elif "norm_q" in name or "norm_k" in name:
                p.fill_(1.0)
            else:
                p.normal_(0, 0.02)
    model.add_adapter(64, 64)
    model.prepare()
    st = SFTTrainStep(model, use_cuda_graph=False, lr=1e-4, seed=7)
    g = torch.Generator(device="cpu").manual_seed(1)
    lat = torch.randn(4, 1, 128, 7, 16, 24, generator=g).bfloat16().to(dev)
    ehs = (torch.randn(4, 1, 128, 4096, generator=g) * 0.1).bfloat16().to(dev)
    mask = torch.arange(128, device=dev)[None] < 77
    mean, std = torch.zeros(1, 128, device=dev), torch.ones(1, 128, device=dev)
    for i in range(40):
        m = st.train_step({"encoder_hidden_states": ehs[i % 4], "encoder_attention_mask": mask},
                          {"latents": lat[i % 4], "latents_mean": mean, "latents_std": std}, sync_metrics=True)
        loss, gn = m["train/global_avg_loss"], m["train/grad_norm"]
        assert loss == loss and 0.5 < loss < 10.0, (i, loss)
        assert gn == gn and 1e-3 < gn < 10.0, (i, gn)
    assert torch.isfinite(model.lora_flat).all()
    del st, model
    torch.cuda.empty_cache()
