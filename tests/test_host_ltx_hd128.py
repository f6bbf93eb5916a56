"""CPU: the head_dim-128 LTX-Video geometry (13B: 32 heads x 128, width 4096, 48 blocks) on the host side - the head_dim
q/k-norm + RoPE entry points exist and spill nothing, the preset, the flat layouts at width 4096, the oracle's RoPE
table and q/k path at head_dim 128 against second derivations, and the refusal of other head dimensions."""
import ctypes
import math
import os
import re
import shutil
import subprocess
from dataclasses import fields

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["b2d_qkv_norm_rope_hd_fwd", "b2d_qkv_norm_rope_hd_bwd"]
GEOM_13B = dict(num_attention_heads=32, attention_head_dim=128, cross_attention_dim=4096, num_layers=48,
                caption_channels=4096)


def test_library_exports_the_head_dim_qk_entry_points():
    from finetrainers_b200 import lib
    so = ctypes.CDLL(lib.build())
    header = open(os.path.join(ROOT, "include", "b2d.h")).read()
    for name in NEW:
        assert name in lib.EXPORTS, name
        assert hasattr(so, name), name
        assert re.search(r"\bint " + name + r"\(", header), name
    for name in NEW:  # the head dimension follows H in the declared argument list
        decl = re.search(name + r"\((.*?)\);", header, re.S).group(1)
        assert re.search(r"int32_t H,\s*int32_t head_dim,\s*float eps", decl), decl


def test_qkv_norm_rope_kernels_use_no_local_memory():
    """Every (chunks, head_dim) instantiation of both directions keeps its row in registers (the three-segment backward
    at two chunks - the 13B QKV row - is the one closest to the limit): no local memory, no stack."""
    tool = shutil.which("cuobjdump") or ("/usr/local/cuda/bin/cuobjdump" if os.path.exists("/usr/local/cuda/bin/cuobjdump") else None)
    if tool is None:
        pytest.skip("cuobjdump not found")
    from finetrainers_b200 import lib
    out = subprocess.run([tool, "--dump-resource-usage", lib.build()], capture_output=True, text=True, check=True).stdout
    usage = dict(re.findall(r"Function (\S*qkv_norm_rope\S*):\s*(.*)", out))
    for direction in ("fwd", "bwd"):
        for nch in (1, 2, 4):
            for hd in (64, 128):
                want = f"qkv_norm_rope_{direction}_kernelILi{nch}ELi{hd}E"
                assert any(want in name for name in usage), (want, sorted(usage))
    assert len(usage) == 12, sorted(usage)
    for name, res in usage.items():
        assert re.search(r"\bLOCAL:0\b", res) and re.search(r"\bSTACK:0\b", res), (name, res)


def test_preset_matches_the_oracle_config_field_for_field():
    from finetrainers_b200.model import LTXConfig
    from oracle import ltx_oracle as O
    cfg = LTXConfig.ltx_13b()
    assert [f.name for f in fields(cfg)] == [f.name for f in fields(O.LTXConfig)]
    ocfg = O.LTXConfig(**GEOM_13B)       # everything not named is the oracle's default (2B) value
    assert cfg.to_dict() == ocfg.to_dict()
    assert cfg.inner_dim == ocfg.inner_dim == 4096
    assert LTXConfig().to_dict() == O.LTXConfig.ltx_2b().to_dict()   # the default geometry is untouched


@pytest.mark.parametrize("head_dim", [96, 32, 256])
def test_other_head_dims_are_refused(head_dim):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    cfg = LTXConfig(in_channels=8, out_channels=8, num_attention_heads=2, attention_head_dim=head_dim,
                    cross_attention_dim=2 * head_dim, num_layers=1, caption_channels=16)
    with pytest.raises(ValueError, match=r"64 and 128"):
        B200LTXTransformer(cfg, torch.bfloat16, "cpu")


@pytest.fixture(scope="module")
def wide2():
    """The 13B width with 2 blocks on the CPU (0.5 G parameters; 48 blocks would take 26 GB)."""
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    cfg = LTXConfig(**dict(GEOM_13B, num_layers=2))
    return B200LTXTransformer(cfg, torch.bfloat16, "cpu")


def test_block_and_root_units_at_width_4096(wide2):
    from finetrainers_b200 import fsdp
    bm, D = wide2, 4096
    blk = bm.transformer_blocks[0]
    got = sum(p.numel() for p in blk.parameters())
    # q/k/v/out of both attentions (8 D^2) + the feed-forward pair (8 D^2); biases 8 D + 4 D + D; norm_q/norm_k of both
    # attentions 4 D; the 6-row table
    assert got == 16 * D * D + 13 * D + 4 * D + 6 * D
    # the block unit leaves the text-side k/v (2 D^2 + 2 D + D of norm_k) to the root unit
    specs = dict(bm._block_specs())
    raw = sum(math.prod(s) for s in specs.values())
    assert raw == 14 * D * D + 11 * D + 3 * D + 6 * D
    n_blk = bm._flat_numel(bm._block_specs())
    assert n_blk % bm.FLAT_ALIGN == 0 and 0 <= n_blk - raw < bm.FLAT_ALIGN
    n_root = bm._flat_numel(bm._root_specs())
    rraw = sum(math.prod(s) for _, s in bm._root_specs())
    assert n_root % bm.FLAT_ALIGN == 0 and 0 <= n_root - rraw < bm.FLAT_ALIGN + 8 * len(bm._root_specs())
    assert dict(bm._root_specs())["Wkv2_all"] == (2, 2 * D, D)
    for numel in (n_blk, n_root):
        for world in (2, 8):
            bounds = [fsdp.shard_bounds(numel, r, world) for r in range(world)]
            assert bounds[0][0] == 0 and bounds[-1][1] == numel
            assert all(a[1] == b[0] for a, b in zip(bounds, bounds[1:]))
            assert all((hi - lo) % 8 == 0 for lo, hi in bounds)     # 16-byte pieces
    # layerwise fp8 storage with the default skip list casts a block's linear weights and biases (14 D^2 + 11 D): that
    # is the bf16 slot the stacked text-side [Wk2;Wv2] + biases (2 D^2 + 2 D per block) stream through, 6 blocks at a
    # time, so 48 blocks make 8 chunks - the same count as 28 blocks at width 2048 make 5
    from finetrainers_b200.layerwise import numel16
    slot = numel16([(k, s) for k, s in bm._block_specs() if k[0] in "Wb"])
    per = max(b for b in range(1, 49) if numel16([("W", (b, 2 * D, D)), ("b", (b, 2 * D))]) <= slot)
    assert per == 6 and math.ceil(48 / per) == 8


@pytest.mark.parametrize("ffn", [False, True])
def test_adapters_at_width_4096(ffn):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig, LORA_FFN_TARGETS, LORA_TARGETS
    D, r, rp = 4096, 24, 64
    bm = B200LTXTransformer(LTXConfig(**dict(GEOM_13B, num_layers=2)), torch.bfloat16, "cpu")
    bm.add_adapter(r, 48, target_modules=list(LORA_FFN_TARGETS if ffn else LORA_TARGETS))
    bm.prepare()
    assert bm.rpad == rp and bm.lora_scaling == 2.0
    per = (26 if ffn else 16) * rp * D
    assert bm._per_blk == per and bm.lora_flat.numel() == 2 * per == bm.lora_grad_flat.numel()
    sd = bm.lora_state_dict()
    names = [f"transformer_blocks.{i}.{a}.{t}" for i in range(2) for a in ("attn1", "attn2") for t in LORA_TARGETS]
    if ffn:
        names += [f"transformer_blocks.{i}.ff.net.{t}" for i in range(2) for t in ("0.proj", "2")]
    assert sorted(sd) == sorted(f"{n}.lora_{x}.weight" for n in names for x in "AB")
    for n in names:
        k_in = 4 * D if n.endswith("ff.net.2") else D
        n_out = 4 * D if n.endswith("0.proj") else D
        assert sd[n + ".lora_A.weight"].shape == (r, k_in) and sd[n + ".lora_B.weight"].shape == (n_out, r)
    # every parameter and its .grad are views into the flat buffers, and no two overlap
    lo, hi = bm.lora_flat.data_ptr(), bm.lora_flat.data_ptr() + 4 * bm.lora_flat.numel()
    glo = bm.lora_grad_flat.data_ptr()
    for p in bm.lora_parameters():
        assert lo <= p.data_ptr() < hi and p.grad.data_ptr() - glo == p.data_ptr() - lo
    base_fqns = [k for k in bm.state_dict() if "lora_" not in k]
    assert "transformer_blocks.1.attn2.to_k.base_layer.weight" in base_fqns
    assert bm.state_dict()["transformer_blocks.1.ff.net.2" + (".base_layer" if ffn else "") + ".weight"].shape == (D, 4 * D)


@pytest.mark.parametrize("dim,pad,nf", [(4096, 4, 682), (768, 0, 128)])
def test_oracle_rope_table_against_the_independent_derivation(dim, pad, nf):
    """D = 4096 has D % 6 = 4 leading pad channels (cos 1, sin 0) and 682 frequencies per axis; D = 768 (6 heads x 128)
    has none.  Channel pairs share a value; the layout is frequency-major, then (f, h, w)."""
    from oracle import independent_constants as IC
    from oracle import ltx_oracle as O
    assert (dim % 6, dim // 6) == (pad, nf)
    Fr, Hh, Ww, scale = 3, 4, 5, (0.32, 32.0, 32.0)
    cos, sin = O.ltx_rope_table(Fr, Hh, Ww, dim, scale)
    assert cos.shape == sin.shape == (1, Fr * Hh * Ww, dim)
    assert torch.equal(cos[..., :pad], torch.ones(1, Fr * Hh * Ww, pad)) and not sin[..., :pad].any()
    assert torch.equal(cos[..., pad::2], cos[..., pad + 1::2]) and torch.equal(sin[..., pad::2], sin[..., pad + 1::2])
    cols = sorted({0, 1, pad, pad + 1, pad + 2, pad + 5, pad + 6, 127, 128, 129, dim // 2, dim - 7, dim - 2, dim - 1})
    worst = 0.0
    for f, h, w in [(0, 0, 0), (2, 3, 4), (1, 0, 4), (2, 1, 0)]:
        s = (f * Hh + h) * Ww + w
        for col in cols:
            c, sn = IC.rope_entry(f, h, w, col, dim, *scale)
            # fp32 angles up to 1e4 * pi/2 * |2g - 1|: the table's own rounding is ~ang * 2^-22
            x = max(0, col - pad) // 2 // 3 / (nf - 1)
            tol = 1e-6 + (1e4 ** x) * 2.0 * 2.0 ** -20
            worst = max(worst, abs(cos[0, s, col].item() - c) / tol, abs(sin[0, s, col].item() - sn) / tol)
            assert abs(cos[0, s, col].item() - c) <= tol and abs(sin[0, s, col].item() - sn) <= tol, (f, h, w, col)


def test_oracle_qk_norm_rope_head_split_at_head_dim_128():
    """The oracle's Attention at 2 heads x 128 hands SDPA q, k, v that equal a float64 restatement: RMS over all 256
    channels (across heads), the rotation of consecutive channel pairs, then channel c -> head c // 128, lane c % 128."""
    from oracle import ltx_oracle as O
    cfg = O.LTXConfig(in_channels=8, out_channels=8, num_attention_heads=2, attention_head_dim=128,
                      cross_attention_dim=256, num_layers=1, caption_channels=16)
    torch.manual_seed(3)
    att = O.Attention(cfg, cross=False).double()
    with torch.no_grad():
        att.norm_q.weight.normal_(1.0, 0.2)
        att.norm_k.weight.normal_(1.0, 0.2)
    B, Fr, Hh, Ww = 2, 1, 3, 3
    S, D = Fr * Hh * Ww, 256
    x = torch.randn(B, S, D, dtype=torch.float64)
    cos, sin = O.ltx_rope_table(Fr, Hh, Ww, D, (1.0, 1.0, 1.0), batch_size=B)
    seen = {}

    def grab(q, k, v, **kw):
        seen.update(q=q, k=k, v=v)
        return torch.zeros_like(q)

    att(x, image_rotary_emb=(cos.double(), sin.double()), sdpa=grab)
    assert seen["q"].shape == (B, 2, S, 128)
    for name, lin, nw in (("q", att.to_q, att.norm_q.weight), ("k", att.to_k, att.norm_k.weight), ("v", att.to_v, None)):
        y = x @ lin.weight.t() + lin.bias
        if nw is not None:
            y = y / torch.sqrt((y * y).sum(-1, keepdim=True) / D + cfg.qk_norm_eps) * nw
            out = torch.empty_like(y)
            for c in range(0, D, 2):
                a, b = y[..., c], y[..., c + 1]
                out[..., c] = a * cos[..., c].double() - b * sin[..., c].double()
                out[..., c + 1] = b * cos[..., c + 1].double() + a * sin[..., c + 1].double()
            y = out
        for c in (0, 1, 127, 128, 200, 255):
            # the oracle rotates in fp32 (apply_rotary_emb casts to float), values are O(1)
            assert torch.allclose(seen[name][:, c // 128, :, c % 128], y[..., c], rtol=0, atol=2e-6), (name, c)
