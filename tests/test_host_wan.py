"""Host: Wan-2.1 module tree, adapter targets and refusals, packing and workspace plan, RoPE constants, spec checks."""
import math

import pytest
import torch

from finetrainers_b200.model import checkpointed_blocks
from finetrainers_b200.wan import B200WanTransformer, WanConfig, WanModelSpecification, wan_moments_shape
from oracle import wan_oracle as O


class _Lora:
    def __init__(self, r=32, lora_alpha=32, target_modules="blocks.*(to_q|to_k|to_v|to_out.0)", init_lora_weights=True):
        self.r, self.lora_alpha, self.target_modules, self.init_lora_weights = r, lora_alpha, target_modules, \
            init_lora_weights


def _tiny(nl=2):
    return WanConfig(num_attention_heads=2, attention_head_dim=128, ffn_dim=512, text_dim=64, num_layers=nl)


def test_fqns_and_shapes_match_restated_diffusers_tree():
    cfg = _tiny()
    bm = B200WanTransformer(cfg, device="cpu")
    om = O.WanTransformerOracle(O.WanOracleConfig(num_attention_heads=2, attention_head_dim=128, ffn_dim=512,
                                                  text_dim=64, num_layers=2))
    got = {k: tuple(v.shape) for k, v in bm.state_dict().items()}
    want = {k: tuple(v.shape) for k, v in om.state_dict().items()}
    assert got == want
    assert got["patch_embedding.weight"] == (256, 16, 1, 2, 2) and got["blocks.1.scale_shift_table"] == (1, 6, 256)
    assert got["scale_shift_table"] == (1, 2, 256) and got["proj_out.weight"] == (64, 256)


def test_configs():
    c = WanConfig()
    assert (c.inner_dim, c.ffn_dim, c.num_layers, c.in_channels, c.text_dim, c.eps) == (1536, 8960, 30, 16, 4096, 1e-6)
    c = WanConfig.wan_14b()
    assert (c.inner_dim, c.ffn_dim, c.num_layers) == (5120, 13824, 40)


@pytest.mark.parametrize("tm", ["blocks.*(to_q|to_k|to_v|to_out.0)", ["to_q", "to_k", "to_v", "to_out.0"]])
@pytest.mark.parametrize("init", [True, "gaussian"])
def test_lora_targets_resolve(tm, init):
    bm = B200WanTransformer(_tiny(), device="cpu")
    bm.add_adapter(_Lora(r=7, lora_alpha=29, target_modules=tm, init_lora_weights=init))
    names = [n for n, _ in bm.named_parameters() if "lora_A" in n]
    assert len(names) == 2 * 8 and "blocks.0.attn2.to_out.0.lora_A.default.weight" in names
    assert math.isclose(bm.lora_scaling, 29 / 7)
    assert all(p.requires_grad == ("lora_" in n) for n, p in bm.named_parameters())


@pytest.mark.parametrize("tm", [["to_q", "to_k", "to_v", "to_out.0", "ffn.net.0.proj", "ffn.net.2"], ["to_q"],
                                "blocks.0.*(to_q|to_k|to_v|to_out.0)"])
def test_other_target_sets_refused(tm):
    bm = B200WanTransformer(_tiny(), device="cpu")
    with pytest.raises(NotImplementedError):
        bm.add_adapter(_Lora(target_modules=tm))


def test_unbuilt_features_refused():
    with pytest.raises(NotImplementedError):
        B200WanTransformer(WanConfig(image_dim=1280, num_layers=1), device="cpu")
    bm = B200WanTransformer(_tiny(), device="cpu")
    with pytest.raises(NotImplementedError):
        bm.enable_layerwise_casting(torch.float8_e4m3fn, skip_modules_pattern=("norm",))
    from finetrainers_b200.fsdp import FSDPState
    with pytest.raises(NotImplementedError):
        FSDPState(bm)
    bm.add_adapter(_Lora())
    with pytest.raises(NotImplementedError):
        bm(torch.zeros(1, 16, 1, 2, 2), torch.zeros(1), torch.zeros(1, 4, 64), encoder_hidden_states_image=torch.zeros(1))


def _offsets(views, base):
    """Element offset of every view from the start of ``base``'s storage."""
    return {k: (v.data_ptr() - base.data_ptr()) // v.element_size() for k, v in views.items()}


def test_packing_offsets_ltx_layout_is_a_prefix():
    """A Wan block's flat unit is LTX's at the same width and FFN size, with norm2's weight and bias after the
    modulation table; the flat LoRA windows of the attention set are LTX's, block by block."""
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    cfg = _tiny()
    cfg.ffn_dim = 4 * cfg.inner_dim  # LTX's FFN width
    wan = B200WanTransformer(cfg, device="cpu")
    ltx = B200LTXTransformer(LTXConfig(num_attention_heads=2, attention_head_dim=128, cross_attention_dim=256,
                                       caption_channels=64, num_layers=2), device="cpu")
    d = 256
    for m in (wan, ltx):
        m.add_adapter(_Lora(r=16, lora_alpha=16, target_modules=["to_q", "to_k", "to_v", "to_out.0"]))
        m.prepare()
    ws, ls = wan._block_specs(), ltx._block_specs()
    assert ws[:len(ls)] == ls and ws[len(ls):] == [("n2w", (d,)), ("n2b", (d,))]
    wo = _offsets(wan._blk[1], wan._blk_flat[1])
    lo = _offsets(ltx._blk[1], ltx._blk_flat[1])
    for k, _ in ls:
        assert wo[k] == lo[k], k
    assert wo["sst"] == sum(math.prod(s) for _, s in ls[:-1])
    assert wo["n2w"] == wo["sst"] + 6 * d and wo["n2b"] == wo["n2w"] + d
    # norm2's parameters and the block table are views of the block's flat unit at those offsets
    blk = wan.blocks[1]
    assert blk.norm2.weight.data_ptr() == wan._blk[1]["n2w"].data_ptr()
    assert blk.norm2.bias.data_ptr() == wan._blk[1]["n2b"].data_ptr()
    assert blk.scale_shift_table.data_ptr() == wan._blk[1]["sst"].data_ptr()
    # LoRA: same per-block size and the same window offsets in the flat fp32 masters and gradients
    assert wan._per_blk == ltx._per_blk == 16 * 64 * d
    for l in range(2):
        keys = [k for k in wan._blk[l] if k.split("_")[0] in ("A", "B", "gA", "gB")]
        assert len(keys) == 4 * 5
        for k in keys:
            wf, lf = (wan.lora_grad_flat, ltx.lora_grad_flat) if k[0] == "g" else (wan.lora_flat, ltx.lora_flat)
            assert _offsets({k: wan._blk[l][k]}, wf) == _offsets({k: ltx._blk[l][k]}, lf), (l, k)
    assert wan.blocks[1].attn2.to_q.lora_A["default"].weight.data_ptr() == wan._blk[1]["A_q2"].data_ptr()
    # the root unit: the patch projection is the Conv3d weight as [D, 64], proj_out [64, D]
    ro = dict(wan._root_specs())
    assert ro["proj_in.w"] == (d, 64) and ro["proj_out.w"] == (64, d)
    assert wan.patch_embedding.weight.data_ptr() == wan._root_views["proj_in.w"].data_ptr()


def test_workspace_plan():
    cfg = WanConfig(num_layers=3)
    bm = B200WanTransformer(cfg, device="meta")
    bm.lora_rank, bm.rpad, bm.lora_ffn = 32, 64, False
    bm._groups = bm._lora_groups()
    d, f = 1536, 8960
    assert bm._groups["q2"].x == "c2n"
    B, S, L = 1, 20280, 512
    plan = bm.workspace_plan(B, S, L, sm_count=132)
    assert plan["c2n"] == ((3, S, d), torch.bfloat16) and plan["ffpre"] == ((3, S, f), torch.bfloat16)
    assert plan["pred"] == ((S, 64), torch.bfloat16)
    full = bm.workspace_plan(B, S, L, ckpt=checkpointed_blocks(3, "full"), sm_count=132)
    assert full["c2n"][0] == (1, S, d)
    inf = bm.workspace_plan(B, S, L, sm_count=132, inference=True)
    assert inf["c2n"][0] == (1, S, d) and "dh" not in inf


def test_rope_against_independent_derivation():
    """The oracle's WanRotaryPosEmbed restatement against oracle/wan_independent_constants.py, every entry."""
    from oracle import wan_independent_constants as IC
    assert IC.wan_rope_split(128) == O.wan_rope_split(128) == (44, 42, 42)
    F, H, W = 3, 4, 5
    rot = O.wan_rope(128, F, H, W)[0, 0]
    assert rot.shape == (F * H * W, 64) and rot.dtype == torch.complex128
    for f in range(F):
        for h in range(H):
            for w in range(W):
                tok = (f * H + h) * W + w
                for p in range(64):
                    c, s_ = IC.wan_rope_entry(f, h, w, p)
                    assert abs(rot[tok, p].real.item() - c) < 1e-12 and abs(rot[tok, p].imag.item() - s_) < 1e-12


def test_sinusoid_against_independent_derivation():
    from oracle import wan_independent_constants as IC
    from oracle.ltx_oracle import sinusoid_256
    t = torch.tensor([0.0, 1.0, 417.0, 999.0])
    got = sinusoid_256(t).double()
    for r, tv in enumerate(t.tolist()):
        assert (got[r] - torch.tensor(IC.wan_sinusoid(tv), dtype=torch.float64)).abs().max() < 1e-4


def test_patch_orders():
    """The Conv3d weight [D, 16, 1, 2, 2] viewed as [D, 64] against the derived k = c*4 + kh*2 + kw (a Conv3d on the
    latent equals the GEMM on tokens packed that way), and the torch restatement of diffusers' unpatchify against the
    derived proj_out order (kh*2 + kw)*16 + c."""
    from oracle import wan_independent_constants as IC
    w = torch.arange(3 * 64, dtype=torch.float64).view(3, 16, 1, 2, 2)
    flat = w.reshape(3, 64)
    for c in range(16):
        for kh in range(2):
            for kw in range(2):
                assert flat[1, IC.conv_k(c, kh, kw)] == w[1, c, 0, kh, kw]
    x = torch.randn(1, 16, 2, 4, 6, dtype=torch.float64)
    conv = torch.nn.Conv3d(16, 3, (1, 2, 2), (1, 2, 2)).double()
    ref = conv(x).flatten(2).transpose(1, 2)  # [1, tokens, 3]
    packed = torch.zeros(1, 2 * 2 * 3, 64, dtype=torch.float64)
    for f in range(2):
        for h in range(4):
            for ww in range(6):
                for c in range(16):
                    packed[0, IC.token(f, h, ww, 4, 6), IC.conv_k(c, h % 2, ww % 2)] = x[0, c, f, h, ww]
    assert torch.allclose(packed @ conv.weight.reshape(3, 64).T + conv.bias, ref)
    out = torch.arange(64.0).view(1, 1, 64)  # one token
    un = out.reshape(1, 1, 1, 1, 1, 2, 2, -1).permute(0, 7, 1, 4, 2, 5, 3, 6).flatten(6, 7).flatten(4, 5).flatten(2, 3)
    for c in range(16):
        for kh in range(2):
            for kw in range(2):
                assert un[0, c, 0, kh, kw] == IC.out_k(c, kh, kw)


def test_spec_value_errors():
    assert wan_moments_shape((2, 32, 3, 4, 6), 16) == (2, 16, 3, 4, 6)
    for shape in [(2, 16, 3, 4, 6), (2, 32, 3, 5, 6), (2, 32, 3, 4, 7), (2, 32, 4, 6)]:
        with pytest.raises(ValueError):
            wan_moments_shape(shape, 16)
    spec = WanModelSpecification(_tiny())
    with pytest.raises(ValueError):
        spec.packed_shape(16, 3, 5, 6)
    assert spec.packed_shape(16, 3, 4, 6) == (3 * 2 * 3, 64)
    bm = B200WanTransformer(_tiny(), device="cpu")
    with pytest.raises(ValueError):
        spec.forward(bm, {"encoder_hidden_states": torch.zeros(1, 4, 64)},
                     {"latents": torch.zeros(1, 32, 1, 3, 4), "latents_mean": torch.zeros(16),
                      "latents_std": torch.ones(16)}, torch.ones(1))


def test_golden_oracle_bit_exact():
    """The oracle's prologue against the fixture the reference's own Wan prologue functions wrote."""
    import os
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "wan_golden.pt"), weights_only=False)
    xt, tg = O.prologue(g["moments"], g["latents_mean"], g["latents_std"], g["eps"], g["noise"], g["sigmas"])
    assert torch.equal(xt.view(torch.int16), g["x_t"].view(torch.int16))
    assert torch.equal(tg.view(torch.int16), g["target"].view(torch.int16))
