"""Host: the feed-forward LoRA target set.  Which target_modules are accepted, the parameter count, names and export, the
packed layout (the attention-only layout unchanged), layerwise fp8 storage of the FFN base weights under FFN adapters,
and the C ABI declaration of the split-K reduction.  No GPU: the model is built and packed on the CPU."""
import json
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = dict(in_channels=32, out_channels=32, num_attention_heads=2, attention_head_dim=64, cross_attention_dim=128,
           num_layers=2, caption_channels=64)
CONTROL_RX = "(transformer_blocks|single_transformer_blocks).*(to_q|to_k|to_v|to_out.0|ff.net.0.proj|ff.net.2)"
FFN_LIST = ["to_q", "to_k", "to_v", "to_out.0", "ff.net.0.proj", "ff.net.2"]
ATTN = ["attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0", "attn2.to_q", "attn2.to_k", "attn2.to_v",
        "attn2.to_out.0"]


class _LoraConfig:
    def __init__(self, r, lora_alpha, init_lora_weights, target_modules):
        self.r, self.lora_alpha, self.init_lora_weights, self.target_modules = r, lora_alpha, init_lora_weights, target_modules


def _model(rank=16, alpha=32, targets=None, prepare=True):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    m = B200LTXTransformer(LTXConfig(**CFG), torch.bfloat16, "cpu")
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.02)
    m.add_adapter(_LoraConfig(rank, alpha, True, targets))
    if prepare:
        m.prepare()
    return m


@pytest.mark.parametrize("targets", [CONTROL_RX, FFN_LIST, set(FFN_LIST)], ids=["regex", "list", "set"])
@pytest.mark.parametrize("rank", [16, 64, 100])
def test_feed_forward_set_is_accepted_with_peft_names(targets, rank):
    m = _model(rank, 2 * rank, targets)
    d, f, nl = m.cfg.inner_dim, 4 * m.cfg.inner_dim, m.cfg.num_layers
    rp = 64 * -(-rank // 64)
    assert m.lora_ffn and m.rpad == rp
    trainable = {n: p for n, p in m.named_parameters() if p.requires_grad}
    assert sum(p.numel() for p in trainable.values()) == nl * 26 * rank * d
    want = set()
    for i in range(nl):
        for mod, (k_in, n_out) in [(a, (d, d)) for a in ATTN] + [("ff.net.0.proj", (d, f)), ("ff.net.2", (f, d))]:
            want.add((f"transformer_blocks.{i}.{mod}.lora_A.default.weight", (rank, k_in)))
            want.add((f"transformer_blocks.{i}.{mod}.lora_B.default.weight", (n_out, rank)))
    assert {(n, tuple(p.shape)) for n, p in trainable.items()} == want
    assert all(p.dtype == torch.float32 for p in trainable.values())
    # the packed per-block slice: 26 rp d elements, the feed-forward groups after o2
    assert m._per_blk == 26 * rp * d and m.lora_flat.numel() == nl * 26 * rp * d
    blk = m.transformer_blocks[1]
    base = m.lora_flat.data_ptr() + 1 * m._per_blk * 4
    off = lambda t: (t.data_ptr() - base) // 4  # noqa: E731
    assert off(blk.ff.net[0].proj.lora_A["default"].weight) == 16 * rp * d
    assert off(blk.ff.net[0].proj.lora_B["default"].weight) == 16 * rp * d + rp * d
    assert off(blk.ff.net[2].lora_A["default"].weight) == 16 * rp * d + rp * d + f * rp
    assert off(blk.ff.net[2].lora_B["default"].weight) == 16 * rp * d + rp * d + f * rp + rp * f
    assert blk.ff.net[2].lora_B["default"].weight.stride() == (rp, 1)
    assert blk.ff.net[2].lora_A["default"].weight.stride() == (f, 1)
    # the base layers stay visible to the packing: the FFN weights are views of the block's flat unit
    e = m._blk[1]
    assert blk.ff.net[0].proj.base_layer.weight.data_ptr() == e["W1"].data_ptr()
    assert blk.ff.net[2].base_layer.weight.data_ptr() == e["W2"].data_ptr()
    assert blk.ff.net[2].base_layer.bias.data_ptr() == e["b2"].data_ptr()
    # .grad views re-attach after zero_grad(set_to_none=True)
    for p in trainable.values():
        p.grad = None
    assert m._attach_lora_grads()
    assert blk.ff.net[2].lora_B["default"].weight.grad.data_ptr() == e["gB_ff2"].data_ptr()


def test_attention_only_layout_is_unchanged():
    """Default targets: per_blk = 16 rp d and every adapter at the offset the attention-only layout has always had
    (per block, per group qkv, o, q2, kv2, o2: A [n rp, d] then B [n d, rp])."""
    m = _model(16, 16, None)
    d, nl, rp = m.cfg.inner_dim, m.cfg.num_layers, 64
    assert not m.lora_ffn and m._per_blk == 16 * rp * d and m.lora_flat.numel() == nl * 16 * rp * d
    groups = [(["attn1.to_q", "attn1.to_k", "attn1.to_v"]), (["attn1.to_out.0"]), (["attn2.to_q"]),
              (["attn2.to_k", "attn2.to_v"]), (["attn2.to_out.0"])]
    params = dict(m.named_parameters())
    for li in range(nl):
        o = li * 16 * rp * d
        for mods in groups:
            n = len(mods)
            for j, mod in enumerate(mods):
                pa = params[f"transformer_blocks.{li}.{mod}.lora_A.default.weight"]
                pb = params[f"transformer_blocks.{li}.{mod}.lora_B.default.weight"]
                assert (pa.data_ptr() - m.lora_flat.data_ptr()) // 4 == o + j * rp * d
                assert (pb.data_ptr() - m.lora_flat.data_ptr()) // 4 == o + n * rp * d + j * d * rp
            o += 2 * n * rp * d
    assert not any(".ff." in n for n in params if "lora_" in n)


@pytest.mark.parametrize("targets", [
    ["to_q", "to_v"],
    ".*(to_q|to_k|to_v|to_out.0|proj)",                   # ff.net.0.proj without ff.net.2
    ["to_q", "to_k", "to_v", "to_out.0", "ff.net.2"],
    ["to_q", "to_k", "to_v", "to_out.0", "ff.net.0.proj"],
    ["ff.net.0.proj", "ff.net.2"],
    FFN_LIST + ["proj_out"],
    ".*(to_q|to_k|to_v|to_out.0|ff.net.0.proj|ff.net.2|proj_in)",
    "transformer_blocks.0.*(to_q|to_k|to_v|to_out.0|ff.net.0.proj|ff.net.2)",
])
def test_other_target_sets_are_refused(targets):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    m = B200LTXTransformer(LTXConfig(**CFG), torch.bfloat16, "cpu")
    with pytest.raises(NotImplementedError, match="ff.net.0.proj and ff.net.2"):
        m.add_adapter(_LoraConfig(8, 8, True, targets))
    assert m.lora_rank == 0 and not m.lora_ffn


@pytest.mark.parametrize("targets", [CONTROL_RX, FFN_LIST])
def test_export_writes_the_feed_forward_keys(targets, tmp_path):
    from safetensors import safe_open
    m = _model(16, 32, targets)
    with torch.no_grad():
        m.lora_flat.normal_(0, 0.1)
    sd = m.lora_state_dict()
    assert len(sd) == 2 * 20
    for k in ("transformer_blocks.1.ff.net.0.proj.lora_A.weight", "transformer_blocks.1.ff.net.0.proj.lora_B.weight",
              "transformer_blocks.0.ff.net.2.lora_A.weight", "transformer_blocks.0.ff.net.2.lora_B.weight"):
        assert k in sd
    assert torch.equal(sd["transformer_blocks.0.ff.net.2.lora_B.weight"],
                       m.transformer_blocks[0].ff.net[2].lora_B["default"].weight.detach())
    path = m.save_lora_weights(str(tmp_path))
    with safe_open(path, "pt") as f:
        cfg = json.loads(f.metadata()["lora_config"])
        keys = set(f.keys())
        assert torch.equal(f.get_tensor("transformer.transformer_blocks.1.ff.net.0.proj.lora_B.weight"),
                           sd["transformer_blocks.1.ff.net.0.proj.lora_B.weight"])
    assert keys == {"transformer." + k for k in sd}
    assert cfg["target_modules"] == targets and cfg["r"] == 16 and cfg["lora_alpha"] == 32


def test_layerwise_fp8_ffn_base_weights_under_ffn_adapters():
    """fp8 storage first, then adapters on the feed-forward linears: the FFN base weights are cast and packed into the
    block's fp8 storage, the adapters stay fp32, and a bf16 re-cast of the model re-packs both."""
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    m = B200LTXTransformer(LTXConfig(**CFG), torch.bfloat16, "cpu")
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.02)
    m.enable_layerwise_casting(torch.float8_e4m3fn, torch.bfloat16, ["^proj_in$", "^proj_out$", "norm"])
    assert "transformer_blocks.1.ff.net.0.proj" in m._lw_cfg["cast"]
    m.add_adapter(_LoraConfig(16, 16, True, CONTROL_RX))
    m.prepare()
    blk = m.transformer_blocks[1]
    for lin in (blk.ff.net[0].proj, blk.ff.net[2]):
        assert lin.base_layer.weight.dtype == torch.float8_e4m3fn
        assert lin.lora_A["default"].weight.dtype == torch.float32
    blk_cast, _ = m._layerwise_plan(set(m._lw_cfg["cast"]))
    assert {"W1", "b1", "W2", "b2"} <= set(blk_cast[1])
    assert m._lw is not None


def test_split_k_reduction_is_declared_in_the_abi():
    from finetrainers_b200 import lib, ops
    hdr = open(os.path.join(ROOT, "include", "b2d.h")).read()
    assert re.search(r"int b2d_splitk_reduce_bf16\(const float\* part, int32_t splits, int32_t M, int32_t N, float alpha,"
                     r"\s*void\* out, int64_t ldc,\s*void\* stream\);", hdr)
    assert int(re.search(r"#define B2D_SPLITK_MAX (\d+)", hdr).group(1)) == ops.SPLITK_MAX
    assert "b2d_splitk_reduce_bf16" in lib.EXPORTS
    src = open(os.path.join(ROOT, "finetrainers_b200", "csrc", "b2d_elem.cu")).read()
    assert "launch_k(splitk_reduce_bf16_kernel" in src
