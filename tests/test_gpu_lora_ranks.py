"""GPU: exact identities of the LoRA rank and scaling.  The engine pads every adapter to rp = 64 * ceil(rank / 64) rows of
A and columns of B, and applies the scaling s = lora_alpha / rank in three kinds of launch: u = s x A^T (forward),
du = s dy B (backward), and through u in dB = dy^T u.  These tests assert bit equality, not a tolerance, so a scaling
dropped, applied twice or applied in the wrong place, or a stride that uses the rank where it should use rp, cannot hide
under rounding.

Why scaling by a power of two c moves into B exactly: u_P = bf16(c acc) = c bf16(acc) = c u_Q and bf16(c B) = c bf16(B),
so every product of the forward extension u B^T is the same fp32 value in P = (A, B, alpha = c r) and Q = (A, c B,
alpha = r).  In the backward, du_P = bf16(c acc(dy B)) = bf16(acc(dy c B)) = du_Q, so dX and dA agree, and
dB = dy^T u is c times larger in P."""
import json

import pytest
import torch

from _util import SMALL, run_b200_micro

pytestmark = pytest.mark.gpu

# (B, F, H, W, text_len): R = B*S and RL = B*L not multiples of 64 (per-block weight-gradient GEMMs), and multiples of 64
# (block-stacked weight-gradient GEMMs)
BATCHES = {"ragged": (2, 2, 4, 9, 24), "m64": (2, 2, 4, 8, 32)}
# adapter groups of one block in the order prepare() carves them: (group, module paths, number of adapters)
GROUPS = [("qkv", ["attn1.to_q", "attn1.to_k", "attn1.to_v"]), ("o", ["attn1.to_out.0"]), ("q2", ["attn2.to_q"]),
          ("kv2", ["attn2.to_k", "attn2.to_v"]), ("o2", ["attn2.to_out.0"])]


def _oracle_state(rank, seed=0):
    """A state dict (bf16-valued base weights, fp32 adapters with B != 0) for the SMALL config at `rank`."""
    from oracle import ltx_oracle as O
    om = O.LTXTransformerOracle(O.LTXConfig(**SMALL))
    O.add_lora(om, rank, rank)
    O.synthetic_init_(om, seed=seed, lora_b_std=0.02)
    return {k: v.clone() for k, v in om.state_dict().items()}


def _model(sd, rank, alpha):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    bm = B200LTXTransformer(LTXConfig(**SMALL), torch.bfloat16, "cuda")
    bm.add_adapter(rank, alpha)
    bm.load_state_dict(sd, strict=True)
    bm.prepare()
    return bm


def _batch(shape, seed=7):
    from oracle import ltx_oracle as O
    B, F, H, W, L = BATCHES[shape]
    return O.make_synthetic_batch(O.LTXConfig(**SMALL), B, F, H, W, text_len=L, seed=seed, text_scale=1.0)


def _grads(bm):
    """{name: copy of .grad} of every adapter tensor, read after micro_step (the optimizer step zeroes the buffer)."""
    return {n: p.grad.detach().clone() for n, p in bm.named_parameters() if "lora_" in n}


def _assert_equal(got, want, what):
    if not torch.equal(got, want):
        diff = (got.float() - want.float()).abs()
        raise AssertionError(f"{what}: {int((diff != 0).sum())} element(s) differ, max |diff| {diff.max().item():.3g}")


@pytest.mark.parametrize("shape", list(BATCHES))
@pytest.mark.parametrize("rank", [16, 128])
@pytest.mark.parametrize("c", [2.0, 0.5])
def test_power_of_two_scaling_moves_into_b(rank, c, shape):
    """P = (A, B, alpha = c r) against Q = (A, c B, alpha = r): loss, pred and every dA bit-identical, every dB of P
    exactly c times Q's."""
    sd = _oracle_state(rank)
    sd_q = {k: (v * c if "lora_B" in k else v) for k, v in sd.items()}
    bp, bq = _model(sd, rank, c * rank), _model(sd_q, rank, rank)
    assert bp.lora_scaling == c and bq.lora_scaling == 1.0
    batch = _batch(shape)
    _, loss_p, pred_p = run_b200_micro(bp, batch)
    _, loss_q, pred_q = run_b200_micro(bq, batch)
    gp, gq = _grads(bp), _grads(bq)
    assert loss_p == loss_q, (loss_p, loss_q)
    _assert_equal(pred_p, pred_q, "pred")
    assert len(gp) == 2 * 8 * SMALL["num_layers"]
    for n in gp:
        assert gq[n].abs().max().item() > 0, n
        if "lora_A" in n:
            _assert_equal(gp[n], gq[n], n)
        else:
            _assert_equal(gp[n], c * gq[n], n)


@pytest.mark.parametrize("shape", list(BATCHES))
def test_only_padded_rank_and_scaling_matter(shape):
    """Rank 96 and rank 128 both pad to rp = 128.  A rank-128 model whose A rows and B columns 96..127 are zero holds the
    same flat buffers as the rank-96 model, so loss, pred and the whole flat gradient must be bit-identical, and the
    rank-128 model's gradients in those rows and columns exactly zero.  Both have alpha = rank (scaling 1)."""
    sd128 = _oracle_state(128, seed=5)
    sd96 = {}
    for k, v in sd128.items():
        if "lora_A" in k:
            v[96:] = 0
            sd96[k] = v[:96].clone()
        elif "lora_B" in k:
            v[:, 96:] = 0
            sd96[k] = v[:, :96].clone()
        else:
            sd96[k] = v
    b96, b128 = _model(sd96, 96, 96), _model(sd128, 128, 128)
    assert b96.rpad == b128.rpad == 128
    _assert_equal(b96.lora_flat, b128.lora_flat, "lora_flat")
    batch = _batch(shape)
    _, loss96, pred96 = run_b200_micro(b96, batch)
    _, loss128, pred128 = run_b200_micro(b128, batch)
    assert loss96 == loss128, (loss96, loss128)
    _assert_equal(pred96, pred128, "pred")
    _assert_equal(b96.lora_grad_flat, b128.lora_grad_flat, "lora_grad_flat")
    g96, g128 = _grads(b96), _grads(b128)
    for n, g in g128.items():
        if "lora_A" in n:
            assert g[96:].abs().max().item() == 0, n
            _assert_equal(g96[n], g[:96], n)
        else:
            assert g[:, 96:].abs().max().item() == 0, n
            _assert_equal(g96[n], g[:, :96], n)
        assert g96[n].abs().max().item() > 0, n


def _layout(rank, rp, d, nl):
    """The flat LoRA layout restated from prepare(): per block, per group, A [n_ad * rp, d] then B [n_ad * d, rp]; adapter
    j owns A rows j * rp .. j * rp + rank and B rows j * d .. (j + 1) * d, columns 0 .. rank.  Returns (mask of the padded
    positions, {(block, module path, 'A' | 'B'): (offset, rows, cols, row stride)} of every real adapter tensor)."""
    per_blk = 16 * rp * d
    pad = torch.zeros(nl * per_blk, dtype=torch.bool)
    where = {}
    for li in range(nl):
        o = li * per_blk
        for _, mods in GROUPS:
            n_ad = len(mods)
            A = pad[o:o + n_ad * rp * d].view(n_ad, rp, d)
            A[:, rank:] = True
            for j, m in enumerate(mods):
                where[(li, m, "A")] = (o + j * rp * d, rank, d, d)
            o += n_ad * rp * d
            Bm = pad[o:o + n_ad * d * rp].view(n_ad * d, rp)
            Bm[:, rank:] = True
            for j, m in enumerate(mods):
                where[(li, m, "B")] = (o + j * d * rp, d, rank, rp)
            o += n_ad * d * rp
        assert o == (li + 1) * per_blk
    return pad, where


@pytest.mark.parametrize("rank,alpha", [(4, 8), (96, 64), (160, 80)])
def test_padding_stays_zero_through_training_and_export(rank, alpha, tmp_path):
    """Three optimizer steps (two accumulated micro-steps each, so both clip paths run) with the gradient clip active and
    weight decay on: every padded position of the fp32 masters, the gradient and both AdamW moments is exactly zero at
    every step.  Afterwards the exported adapters have peft's shapes and the values of the flat slices, and the saved
    metadata records the rank and lora_alpha as given."""
    from safetensors import safe_open
    from finetrainers_b200.trainer import SFTTrainStep
    sd = _oracle_state(rank, seed=2)
    bm = _model(sd, rank, alpha)
    d, nl, rp = bm.cfg.inner_dim, bm.cfg.num_layers, bm.rpad
    assert rp == 64 * -(-rank // 64) and bm.lora_flat.numel() == nl * 16 * rp * d
    pad, where = _layout(rank, rp, d, nl)
    pad = pad.cuda()
    assert int((~pad).sum()) == sum(p.numel() for n, p in bm.named_parameters() if "lora_" in n)
    max_norm = 1e-3
    st = SFTTrainStep(bm, flow_weighting_scheme="none", lr=1e-3, weight_decay=1e-2, max_grad_norm=max_norm,
                      gradient_accumulation_steps=2, seed=3)
    st.spec.first_frame_conditioning_p = 0.0

    def padded(t, what):
        nz = int((t[pad] != 0).sum())
        assert nz == 0, f"{what}: {nz} padded position(s) nonzero"
        assert t[~pad].abs().max().item() > 0, f"{what}: all real positions zero"

    for i in range(6):
        batch = _batch("ragged" if i % 2 else "m64", seed=40 + i)
        cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(),
                "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}
        lat = {"latents": batch["latents"].cuda(), "latents_mean": batch["latents_mean"].cuda(),
               "latents_std": batch["latents_std"].cuda()}
        m = st.train_step(cond, lat, sigmas=batch["sigmas"].view(-1).cuda(), noise=batch["noise"].cuda(),
                          sync_metrics=True)
        torch.cuda.synchronize()
        if m is None:   # first micro-step of the window: the accumulated gradient was clipped in place
            padded(bm.lora_grad_flat, f"step {i} lora_grad_flat")
            assert abs(bm.lora_grad_flat.norm().item() - max_norm) / max_norm < 1e-3
        else:
            assert m["train/grad_norm"] > max_norm, m     # the clip was active
            assert bm.lora_grad_flat.abs().max().item() == 0
            for what, t in (("lora_flat", bm.lora_flat), ("exp_avg", st.exp_avg), ("exp_avg_sq", st.exp_avg_sq)):
                padded(t, f"step {i} {what}")
    flat = bm.lora_flat.detach().cpu()
    exported = bm.lora_state_dict()
    assert len(exported) == 2 * 8 * nl
    for (li, mod, ab), (o, rows, cols, ld) in where.items():
        k = f"transformer_blocks.{li}.{mod}.lora_{ab}.weight"
        want = flat.as_strided((rows, cols), (ld, 1), o)
        assert exported[k].shape == ((rank, d) if ab == "A" else (d, rank)), k
        _assert_equal(exported[k], want, k)
    path = bm.save_lora_weights(str(tmp_path))
    with safe_open(path, "pt") as f:
        cfg = json.loads(f.metadata()["lora_config"])
        keys = set(f.keys())
    assert cfg["r"] == rank and cfg["lora_alpha"] == alpha, cfg
    assert keys == {"transformer." + k for k in exported}
