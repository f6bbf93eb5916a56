"""CPU: pin the oracle restatement against golden vectors produced by the REAL reference sources
(tests/golden/make_golden.py) and against the reference's own attention known-answer recipe
(tests/models/attention_dispatch.py:41-111: randn[2,8,256,64] bf16, seed 0, vs math SDPA, atol 5e-3)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import ltx_oracle as O


def test_flow_match_golden(golden):
    g = golden
    assert torch.equal(O.flow_match_xt(g["fm_x0"], g["fm_n"], g["fm_t"]), g["fm_xt"])
    assert torch.equal(O.flow_match_target(g["fm_n"], g["fm_x0"]), g["fm_target"])


def test_normalize_pack_golden(golden):
    g = golden
    assert torch.equal(O.normalize_latents(g["nl_lat"], g["nl_mean"], g["nl_std"]), g["nl_out"])
    assert torch.equal(O.pack_latents(g["nl_lat"], 1, 1), g["pack_out"])


def test_rope_apply_golden(golden):
    g = golden
    out = O.apply_rotary_emb(g["rope_x"], (g["rope_cos"], g["rope_sin"]))
    assert torch.equal(out, g["rope_out"])


def test_rmsnorm_golden(golden):
    g = golden
    for tag in ("affine", "noaffine"):
        w = g[f"rms_{tag}_w"]
        m = O.RMSNorm(32, g[f"rms_{tag}_eps"], w is not None)
        if w is not None:
            m.weight.data = w.clone()
        assert torch.equal(m(g[f"rms_{tag}_x"]), g[f"rms_{tag}_out"])


def test_prepare_sigmas_golden(golden):
    g = golden
    for scheme in ("none", "logit_normal", "mode"):
        gen = torch.Generator().manual_seed(1234)
        s = O.prepare_sigmas(g["sig_table"], 16, 1000, scheme, 0.0, 1.0, 1.29, "cpu", gen)
        assert torch.equal(s, g[f"sig_{scheme}"])
    assert torch.equal(O.flow_match_scheduler_sigmas(), g["sig_table"])


def test_attention_kat_cpu():
    """The reference's attention recipe, CPU side: default SDPA vs math SDPA (the oracle uses F.sdpa)."""
    torch.manual_seed(0)
    q, k, v = (torch.randn(2, 8, 256, 64).bfloat16() for _ in range(3))
    with torch.nn.attention.sdpa_kernel(torch.nn.attention.SDPBackend.MATH):
        ref = F.scaled_dot_product_attention(q, k, v)
    out = F.scaled_dot_product_attention(q, k, v)
    assert (out.float() - ref.float()).abs().max() < 5e-3


def test_oracle_tiny_config_two_steps_cpu():
    """BASELINE config 1: LTX dummy (tests/models/ltx_video/base_specification.py:46-63), 1 frame 64x64 -> latent
    [1,8,1,2,2], 2 SFT steps on CPU, world_size 1 — the reference's 'does not raise' smoke, plus: loss decreases."""
    torch.manual_seed(0)
    cfg = O.LTXConfig.tiny()
    m = O.LTXTransformerOracle(cfg)
    O.add_lora(m, 4, 4)
    O.synthetic_init_(m, lora_b_std=0.0)
    batch = O.make_synthetic_batch(cfg, 1, 1, 2, 2, text_len=8, dtype=torch.float32)
    opt = torch.optim.AdamW([p for p in m.parameters() if p.requires_grad], lr=1e-2)
    losses = []
    for _ in range(2):
        opt.zero_grad()
        loss, _ = O.oracle_step(m, batch)
        O.clip_grad_norm_([p for p in m.parameters() if p.requires_grad], 1.0)
        opt.step()
        losses.append(loss.item())
    assert all(map(lambda x: x == x, losses))
    assert losses[1] <= losses[0] + 1e-6
    # B == 0 at init => adapters contribute nothing: first-step gradient of lora_A is exactly zero
    m2 = O.LTXTransformerOracle(cfg)
    O.add_lora(m2, 4, 4)
    O.synthetic_init_(m2, lora_b_std=0.0)
    O.oracle_step(m2, batch)
    ga = [p.grad.abs().max().item() for n, p in m2.named_parameters() if "lora_A" in n]
    assert max(ga) == 0.0


def test_oracle_fqn_tree():
    """Parameter names follow diffusers + peft (SURVEY Appendix A; _test_tp.py:186-245)."""
    m = O.LTXTransformerOracle(O.LTXConfig.tiny())
    O.add_lora(m, 4, 4)
    names = set(n for n, _ in m.named_parameters())
    for k in ("proj_in.weight", "time_embed.emb.timestep_embedder.linear_1.weight", "time_embed.linear.bias",
              "caption_projection.linear_2.weight", "scale_shift_table", "transformer_blocks.0.scale_shift_table",
              "transformer_blocks.0.attn1.to_q.base_layer.weight", "transformer_blocks.0.attn1.to_q.lora_A.default.weight",
              "transformer_blocks.0.attn2.to_out.0.lora_B.default.weight", "transformer_blocks.0.attn1.norm_q.weight",
              "transformer_blocks.0.ff.net.0.proj.weight", "transformer_blocks.0.ff.net.2.bias", "proj_out.weight"):
        assert k in names, k
    # LoRA params: 8 adapted linears / block, 2 tensors each
    assert sum("lora_" in n for n in names) == 16


def test_clip_grad_norm_golden():
    """oracle.clip_grad_norm_ against gradients clipped by the reference's own clip_grad_norm_ / _get_total_norm /
    _clip_grads_with_norm_ (finetrainers/utils/torch.py:99-161,299-381, executed unmodified by make_clip_golden.py)."""
    import os
    from oracle import ltx_oracle as O
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "clip_golden.pt"), weights_only=True)
    for tag in ("big", "small"):
        params = [torch.nn.Parameter(torch.zeros_like(x)) for x in g[f"{tag}_grads_in"]]
        for p, x in zip(params, g[f"{tag}_grads_in"]):
            p.grad = x.clone()
        total = O.clip_grad_norm_(params, 1.0)
        assert torch.allclose(total, g[f"{tag}_total_norm"], rtol=1e-6, atol=0)
        for p, want in zip(params, g[f"{tag}_grads_out"]):
            assert torch.allclose(p.grad, want, rtol=1e-6, atol=1e-12)
    assert g["big_total_norm"] > 1.0 > g["small_total_norm"]      # one case clips, the other passes through


def test_independent_derivation_matches_oracle():
    """oracle/independent_constants.py re-derives the upstream-only constants (timestep sinusoid, LTX RoPE table incl.
    padding side and pair layout, flow-match sigma table, GELU-tanh, RMSNorm) in scalar float64 without sharing code with
    the oracle; the two must agree."""
    import math
    import torch
    import torch.nn.functional as F
    from oracle import ltx_oracle as O
    from oracle import independent_constants as I
    for t in (0.0, 1.0, 499.0, 999.0):
        a = O.sinusoid_256(torch.tensor([t]))[0].double()
        b = torch.tensor(I.sinusoid_256(t), dtype=torch.float64)
        assert (a - b).abs().max().item() < 2e-4            # fp32 exp/cos of arguments up to 999
    dim, Fr, H, W = 2048, 3, 4, 5
    scale = [8 / 25, 32, 32]
    cos, sin = O.ltx_rope_table(Fr, H, W, dim, scale)
    assert cos.shape == (1, Fr * H * W, dim)
    for (f, h, w) in ((0, 0, 0), (2, 3, 4), (1, 0, 3)):
        s = (f * H + h) * W + w
        for col in (0, 1, 2, 3, 4, 7, 8, 1000, 1001, 2046, 2047):
            c, sn = I.rope_entry(f, h, w, col, dim, *scale)
            assert abs(cos[0, s, col].item() - c) < 2e-3 and abs(sin[0, s, col].item() - sn) < 2e-3, (f, h, w, col)
    # dim % 6 == 0: no padding
    cos, sin = O.ltx_rope_table(2, 2, 2, 24, scale)
    for col in range(24):
        c, sn = I.rope_entry(1, 1, 0, col, 24, *scale)
        assert abs(cos[0, (1 * 2 + 1) * 2 + 0, col].item() - c) < 2e-3   # fp32 cos of angles up to theta * pi / 2
    assert O.flow_match_scheduler_sigmas().tolist() == pytest.approx(I.flow_match_sigmas(), abs=1e-7)
    xs = [-3.0, -0.5, 0.0, 0.7, 2.5]
    assert F.gelu(torch.tensor(xs), approximate="tanh").tolist() == pytest.approx([I.gelu_tanh(x) for x in xs], abs=1e-6)
    row = [0.5, -1.0, 2.0, 0.25]
    got = O.RMSNorm(4, 1e-5, True)(torch.tensor([row]))[0].tolist()
    assert got == pytest.approx(I.rms_norm(row, [1.0] * 4, 1e-5), abs=1e-6)
