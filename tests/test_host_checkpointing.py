"""CPU: activation checkpointing's policy and memory plan - which blocks each policy recomputes (the reference's rule),
the refused types, the refusal of a policy change once a workspace exists, and the workspace plan: keep-all is the
keep-everything layout shape for shape, and checkpointing shrinks only the tensors a block recomputes."""
import pytest
import torch

from _util import SMALL

NL = 6


def _model(nl=NL, ffn=False, rank=64, **cfg):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig, LORA_FFN_TARGETS
    m = B200LTXTransformer(LTXConfig(**dict(SMALL, num_layers=nl, **cfg)), torch.bfloat16, "cpu")
    m.add_adapter(rank, rank, target_modules=LORA_FFN_TARGETS if ffn else None)
    m.prepare()
    return m


def _reference_rule(num_layers, n_layer):
    """``_apply_activation_checkpointing_blocks``: wrap block ``index`` iff n_layer is None or index % n_layer == 0."""
    return tuple(i for i in range(num_layers) if n_layer is None or i % n_layer == 0)


@pytest.mark.parametrize("n_layer", [1, 2, 3, 5, NL, NL + 3])
def test_block_skip_selects_the_reference_rule(n_layer):
    from finetrainers_b200.model import apply_activation_checkpointing, checkpointed_blocks
    assert checkpointed_blocks(NL, "block_skip", n_layer) == _reference_rule(NL, n_layer)
    m = apply_activation_checkpointing(_model(), "block_skip", n_layer)
    assert m._ckpt == _reference_rule(NL, n_layer) and m.gradient_checkpointing


def test_full_and_the_diffusers_switches():
    from finetrainers_b200.model import apply_activation_checkpointing
    m = _model()
    assert not m.gradient_checkpointing and m._ckpt == ()
    assert apply_activation_checkpointing(m)._ckpt == _reference_rule(NL, None)
    m.disable_gradient_checkpointing()
    assert not m.gradient_checkpointing and m._ckpt == ()
    m.enable_gradient_checkpointing()
    assert m.gradient_checkpointing and m._ckpt == tuple(range(NL))


def test_ops_and_unknown_types_raise():
    from finetrainers_b200.model import apply_activation_checkpointing
    m = _model()
    with pytest.raises(NotImplementedError, match="ops"):
        apply_activation_checkpointing(m, "ops")
    with pytest.raises(ValueError, match="selective"):
        apply_activation_checkpointing(m, "selective")
    with pytest.raises(ValueError, match="n_layer"):
        apply_activation_checkpointing(m, "block_skip", 0)
    with pytest.raises(TypeError):
        apply_activation_checkpointing(torch.nn.Linear(2, 2))
    assert m._ckpt == ()


def test_policy_change_after_the_workspace_exists_raises():
    m = _model()
    m.enable_gradient_checkpointing()
    m._workspace(1, 72, 24)                 # what the first forward allocates
    m.enable_gradient_checkpointing()       # the same policy again is not a change
    with pytest.raises(ValueError, match="before the first forward"):
        m.disable_gradient_checkpointing()
    from finetrainers_b200.model import apply_activation_checkpointing
    with pytest.raises(ValueError, match="before the first forward"):
        apply_activation_checkpointing(m, "block_skip", 2)
    assert m._ckpt == tuple(range(NL))


def _keep_all_layout(m, B, S, L, splitk):
    """The keep-everything workspace restated from its definition: name -> (shape, dtype)."""
    cfg = m.cfg
    d, H, nl, rp, hd = cfg.inner_dim, cfg.num_attention_heads, cfg.num_layers, m.rpad, cfg.attention_head_dim
    R, RL, F = B * S, B * L, cfg.ffn_mult * cfg.inner_dim
    bf, f32 = torch.bfloat16, torch.float32
    hs = lambda n, s: (n, B, H, s, hd)  # noqa: E731
    ws = {"tsin": (B, 256), "t1": (B, d), "t2s": (B, d), "embedded": (B, d), "temb": (B, 6 * d), "c1": (RL, d),
          "enc": (RL, d), "h": (nl + 1, R, d), "n1": (nl, R, d), "qkv": (nl, R, 3 * d), "qh": hs(nl, S), "kh": hs(nl, S),
          "vh": hs(nl, S), "ao": (nl, R, d), "lse": (nl, B, H, S), "h1": (nl, R, d), "q2": (nl, R, d), "q2h": hs(nl, S),
          "kv2": (nl, RL, 2 * d), "k2h": hs(nl, L), "v2h": hs(nl, L), "ao2": (nl, R, d), "lse2": (nl, B, H, S),
          "h2": (nl, R, d), "ffpre": (nl, R, F),
          "u_qkv": (nl, R, 3 * rp), "u_o": (nl, R, rp), "u_q2": (nl, R, rp), "u_kv2": (nl, RL, 2 * rp), "u_o2": (nl, R, rp),
          "dy_o2": (nl, R, d), "dy_q2": (nl, R, d), "dy_kv2": (nl, RL, 2 * d), "dy_o": (nl, R, d), "dy_qkv": (nl, R, 3 * d),
          "du_o2": (nl, R, rp), "du_q2": (nl, R, rp), "du_kv2": (nl, RL, 2 * rp), "du_o": (nl, R, rp),
          "du_qkv": (nl, R, 3 * rp)}
    ffb = (nl,) if m.lora_ffn else ()
    ws.update({"n2": (*ffb, R, d), "f": (*ffb, R, F), "y": (R, d), "pred": (R, cfg.out_channels), "dh": (R, d),
               "g": (*ffb, R, d), "dwide": (*ffb, R, F), "dn": (R, d), "da": (R, d)})
    if m.lora_ffn:
        ws.update({"u_ff1": (nl, R, rp), "u_ff2": (nl, R, rp), "du_ff1": (nl, R, rp), "du_ff2": (nl, R, rp)})
        if splitk > 1:
            ws["splitk"] = (splitk, R, rp)
    ws.update({"dqh": hs(None, S)[1:], "dkh": hs(None, S)[1:], "dvh": hs(None, S)[1:], "dk2h": hs(nl, L),
               "dv2h": hs(nl, L)})
    ws["delta"] = (max(2 * B * H * S + (16 * B * H * S * hd if S <= 512 else 0), 2 * B * H * S + 16 * B * H * L * hd),)
    fp32 = {"lse", "lse2", "splitk", "delta"}
    return {k: (tuple(v), f32 if k in fp32 else bf) for k, v in ws.items()}


@pytest.mark.parametrize("ffn", [False, True], ids=["attn", "ffn"])
@pytest.mark.parametrize("hd", [64, 128])
def test_keep_all_plan_is_the_keep_everything_layout(ffn, hd):
    m = _model(ffn=ffn, num_attention_heads=256 // hd, attention_head_dim=hd)
    B, S, L = 2, 72, 24
    plan = m.workspace_plan(B, S, L, sm_count=132)
    splitk = 2 if (4 * 256) % 128 == 0 and 2 * -(-B * S // 128) <= 132 else 1
    assert plan == _keep_all_layout(m, B, S, L, splitk)
    assert list(plan) == list(_keep_all_layout(m, B, S, L, splitk))       # allocation order too
    # the allocated workspace of the default policy is that plan
    if not ffn:
        ws = m._workspace(B, S, L)
        assert {k: (tuple(v.shape), v.dtype) for k, v in ws.items()} == plan


RECOMPUTED = {"n1", "qkv", "qh", "kh", "vh", "h1", "q2", "q2h", "h2", "ffpre", "u_qkv", "u_o", "u_q2", "u_o2", "dy_o2",
              "dy_q2", "dy_o", "dy_qkv", "du_o2", "du_q2", "du_o", "du_qkv"}
RECOMPUTED_FFN = {"n2", "f", "g", "dwide", "u_ff1", "u_ff2", "du_ff1", "du_ff2"}


@pytest.mark.parametrize("ffn", [False, True], ids=["attn", "ffn"])
@pytest.mark.parametrize("policy", [("full", 1), ("block_skip", 2), ("block_skip", 4), ("block_skip", NL + 1)])
def test_checkpointed_plan_shrinks_only_the_recomputed_tensors(ffn, policy):
    from finetrainers_b200.model import checkpointed_blocks
    m = _model(ffn=ffn)
    B, S, L = 1, 72, 24
    ck = checkpointed_blocks(NL, *policy)
    keep, plan = m.workspace_plan(B, S, L, (), sm_count=132), m.workspace_plan(B, S, L, ck, sm_count=132)
    assert list(plan) == list(keep)
    slots = NL - len(ck) + 1
    shrunk = RECOMPUTED | (RECOMPUTED_FFN if ffn else set())
    for k, (shape, dt) in plan.items():
        want = (slots,) + keep[k][0][1:] if k in shrunk else keep[k][0]
        assert (shape, dt) == (want, keep[k][1]), k
    per_slot = sum(torch.Size(keep[k][0][1:]).numel() * 2 for k in shrunk)
    assert m.workspace_bytes(B, S, L, (), 132) - m.workspace_bytes(B, S, L, ck, 132) == (len(ck) - 1) * per_slot


def test_slots_and_runs():
    m = _model()
    assert m._block_slots() == (list(range(NL)), NL)
    m.set_activation_checkpointing((0, 3, 4))
    assert m._block_slots() == ([3, 0, 1, 3, 3, 2], 4)
    assert m._kept_runs(0, NL) == [(1, 2), (5, 1)]
    assert m._kept_runs(2, 4) == [(2, 1)]
    assert m._kept_runs(3, 5) == []
    with pytest.raises(ValueError, match="outside"):
        m.set_activation_checkpointing((NL,))


def test_plan_at_the_13b_width_for_a_long_clip():
    """Two blocks of the 13B geometry: per block, keep-all holds 1.2 GB at 6144 tokens, r = 64 (0.9 GB activations and
    0.3 GB of adapter dy); a checkpointed block keeps its input and two attention outputs (3 x 6144 x 4096 bf16, plus
    the lse and the text-side rows: within 10 %)."""
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    cfg = LTXConfig.ltx_13b()
    cfg.num_layers = 2
    m = B200LTXTransformer(cfg, torch.bfloat16, "cpu")
    m.add_adapter(64, 64)
    m.prepare()
    S, L = 16 * 16 * 24, 128

    def per_block(ck):
        """bytes of one block's index of the tensors stacked per block (h counted once per block)"""
        plan = m.workspace_plan(1, S, L, ck)
        return sum(torch.Size(s[1:]).numel() * torch.empty((), dtype=dt).element_size()
                   for k, (s, dt) in plan.items() if len(s) > 1 and s[0] == (3 if k == "h" else 2))

    assert 1.15e9 < per_block(()) < 1.25e9, per_block(())
    kept = 3 * S * 4096 * 2
    assert kept < per_block((0, 1)) < kept * 1.1, per_block((0, 1))
    assert m.workspace_bytes(1, S, L, ()) - m.workspace_bytes(1, S, L, (0, 1)) == per_block(()) - per_block((0, 1))
