"""Host: layerwise fp8 weight storage for Wan-2.1 text- and image-to-video.  The cast set against diffusers'
``apply_layerwise_casting`` walk restated on the oracle trees (``nn.Linear`` and Conv layers are cast, a module whose
FQN matches a skip pattern under ``re.search`` is skipped with its subtree), the fp8 parameters that result, the
refusals (the Conv3d patch embedding, a split image-side K/V) and that they leave the model as it was, the storage bytes
after ``prepare()`` against the arithmetic from the specs, and the streamed text- and image-side K/V chunks."""
import re

import pytest
import torch

import _wan_i2v_oracle as I
from finetrainers_b200.wan import B200WanTransformer, WanConfig
from oracle import wan_oracle as O

DATACLASS_DEFAULT = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "time_embed", "^proj_in$", "^proj_out$",
                     "norm"]   # finetrainers/args.py:395
CLI_DEFAULT = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]  # :751-754
LISTS = {"dataclass": DATACLASS_DEFAULT, "cli": CLI_DEFAULT, "cli+ffn": CLI_DEFAULT + ["ffn"],
         "cli+attn2": CLI_DEFAULT + ["attn2"]}
GEOM = dict(num_attention_heads=2, attention_head_dim=64, ffn_dim=256, text_dim=64)
DI = 64  # image_dim of the image-to-video models here


def diffusers_cast(module, patterns):
    """diffusers' walk, restated independently of the engine: FQNs of the ``nn.Linear`` and Conv layers it casts."""
    conv = (torch.nn.Conv1d, torch.nn.Conv2d, torch.nn.Conv3d, torch.nn.ConvTranspose1d, torch.nn.ConvTranspose2d,
            torch.nn.ConvTranspose3d)
    out = []

    def visit(mod, fqn):
        if any(re.search(p, fqn) for p in patterns):
            return
        if isinstance(mod, (torch.nn.Linear,) + conv):
            out.append(fqn)
            return
        for name, child in mod.named_children():
            visit(child, f"{fqn}.{name}" if fqn else name)

    visit(module, "")
    return sorted(out)


def oracle(i2v, nl):
    if i2v:
        return I.WanI2VTransformerOracle(I.WanI2VOracleConfig(image_dim=DI, num_layers=nl, **GEOM))
    return O.WanTransformerOracle(O.WanOracleConfig(num_layers=nl, **GEOM))


def engine(i2v, nl=3):
    d = GEOM["num_attention_heads"] * GEOM["attention_head_dim"]
    kw = dict(in_channels=36, image_dim=DI, added_kv_proj_dim=d) if i2v else {}
    torch.manual_seed(0)
    m = B200WanTransformer(WanConfig(num_layers=nl, **GEOM, **kw), torch.bfloat16, "cpu")
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.05)
    return m


def _untouched(m, before):
    assert m._lw_cfg is None
    for n, p in m.named_parameters():
        assert p.dtype == torch.bfloat16 and torch.equal(p, before[n]), n


@pytest.mark.parametrize("which", list(LISTS))
@pytest.mark.parametrize("i2v", [False, True], ids=["t2v", "i2v"])
def test_cast_set_is_diffusers_walk_and_stored_params_are_fp8(i2v, which):
    pats = LISTS[which]
    want = diffusers_cast(oracle(i2v, 3), pats)
    m = engine(i2v)
    m.enable_layerwise_casting(torch.float8_e4m3fn, skip_modules_pattern=pats)
    assert sorted(m._lw_cfg["cast"]) == want
    # what the issue-level rule says: norms, scale_shift_table and norm_added_k never; every block linear outside the
    # extra skips, time_proj, text_embedder and the image embedder's ff under both lists; time_embedder under the CLI one
    assert not any("norm" in n or "patch_embedding" in n or n == "proj_out" for n in want)
    ce = "condition_embedder."
    assert {ce + "time_proj", ce + "text_embedder.linear_1", ce + "text_embedder.linear_2"} <= set(want)
    assert (ce + "time_embedder.linear_1" in want) == (which != "dataclass")
    assert (ce + "image_embedder.ff.net.0.proj" in want) == i2v and (ce + "image_embedder.ff.net.2" in want) == i2v
    assert ("blocks.2.ffn.net.2" in want) == (which != "cli+ffn")
    assert ("blocks.2.attn2.to_k" in want) == (which != "cli+attn2")
    assert ("blocks.1.attn2.add_v_proj" in want) == (i2v and which != "cli+attn2")
    fp8 = sorted(n for n, p in m.named_parameters() if p.dtype == torch.float8_e4m3fn)
    assert fp8 == sorted(f"{n}.{w}" for n in want for w in ("weight", "bias"))
    # after the adapter and prepare() the same parameters are fp8 (the adapted linears' under base_layer)
    m.add_adapter(16, 16)
    m.prepare()
    fp8 = sorted(n.replace(".base_layer", "") for n, p in m.named_parameters() if p.dtype == torch.float8_e4m3fn)
    assert fp8 == sorted(f"{n}.{w}" for n in want for w in ("weight", "bias"))
    assert all(p.dtype == torch.float32 for n, p in m.named_parameters() if "lora_" in n)


@pytest.mark.parametrize("i2v", [False, True], ids=["t2v", "i2v"])
@pytest.mark.parametrize("pats", [("norm",), CLI_DEFAULT[1:]])
def test_casting_the_patch_embedding_is_refused_and_changes_nothing(i2v, pats):
    """diffusers casts the Conv3d patch embedding unless a pattern skips it; the engine does not store it in fp8."""
    assert "patch_embedding" in diffusers_cast(oracle(i2v, 2), pats)
    m = engine(i2v, 2)
    before = {n: p.detach().clone() for n, p in m.named_parameters()}
    with pytest.raises(NotImplementedError, match="patch_embedding") as ei:
        m.enable_layerwise_casting(torch.float8_e4m3fn, skip_modules_pattern=pats)
    assert "patch_embed'" in str(ei.value)
    _untouched(m, before)
    m.enable_layerwise_casting(torch.float8_e4m3fn, skip_modules_pattern=CLI_DEFAULT)   # still possible afterwards


@pytest.mark.parametrize("extra,names", [
    ("add_v_proj", ["attn2.add_k_proj", "attn2.add_v_proj"]),            # k without v
    (r"blocks\.1\.attn2\.add_", ["blocks.0.attn2.add_k_proj", "blocks.1.attn2.add_k_proj"]),  # not every block
])
def test_a_split_image_side_kv_is_refused_and_changes_nothing(extra, names):
    m = engine(True)
    before = {n: p.detach().clone() for n, p in m.named_parameters()}
    with pytest.raises(NotImplementedError, match="Wkv3_all") as ei:
        m.enable_layerwise_casting(torch.float8_e4m3fn, skip_modules_pattern=CLI_DEFAULT + [extra])
    for n in names:
        assert n in str(ei.value)
    _untouched(m, before)


def _r16(n):
    return (n + 15) // 16 * 16   # fp8 pieces and their slot views start on 16-element boundaries


def _align(n):
    return (n + 2047) // 2048 * 2048   # FLAT_ALIGN of every bf16 unit


def _r8(n):
    return (n + 7) // 8 * 8


@pytest.mark.parametrize("which", ["dataclass", "cli"])
@pytest.mark.parametrize("i2v", [False, True], ids=["t2v", "i2v"])
def test_storage_bytes_after_prepare_match_the_specs(i2v, which):
    nl = 4
    m = engine(i2v, nl)
    m.enable_layerwise_casting(torch.float8_e4m3fn, skip_modules_pattern=LISTS[which])
    m.add_adapter(16, 16)
    m.prepare()
    d, f, tdim, cin, cout = 128, 256, 64, 4 * (36 if i2v else 16), 64
    blk_cast = [3 * d * d, 3 * d, d * d, d, d * d, d, d * d, d, f * d, f, d * f, d]
    time_emb = [d * 256, d, d * d, d]
    root_slot = ([] if which == "dataclass" else time_emb) + [6 * d * d, 6 * d, d * tdim, d, d * d, d]
    root_keep = [d * cin, d] + (time_emb if which == "dataclass" else []) + [2 * d, cout * d, cout, nl * d]
    kv = [nl * 2 * d * d, nl * 2 * d]
    if i2v:
        root_slot += [DI * DI, DI, d * DI, d]
        root_keep += [DI, DI, d, d, nl * d]
    fp8 = nl * sum(map(_r16, blk_cast)) + sum(map(_r16, root_slot + kv * (2 if i2v else 1)))
    got = m.base_weight_bytes()
    assert got["fp8_storage"] == fp8
    assert got["bf16_resident"] == 2 * (nl * _align(11 * d) + _align(sum(map(_r8, root_keep))))
    assert got["block_slots"] == 2 * 2 * max(sum(map(_r16, blk_cast)), _r16(2 * d * d) + _r16(2 * d))
    assert got["root_slot"] == 2 * sum(map(_r16, root_slot))
    # no persistent bf16 copy of either stacked K/V: both stream through the block slots, each in one chunk here
    assert m._Wkv2_all is None and "Wkv2_all" not in m._root_views and "Wkv3_all" not in m._root_views
    assert m._lw.kv2_chunks == [(0, nl)] and m._lw.chunks("kv3") == ([(0, nl)] if i2v else [])


def test_i2v_root_slot_holds_no_image_kv_and_chunks_cover_all_blocks(monkeypatch):
    """Feed-forward skipped: a block slot holds 6 d^2 weights, three blocks' [Wk;Wv], so five blocks take two chunks of
    each stacked K/V; they alternate over the two slots in the order kv2, kv2, kv3, kv3 and then hand the slots to
    blocks 0 and 1."""
    nl = 5
    m = engine(True, nl)
    m.enable_layerwise_casting(torch.float8_e5m2, skip_modules_pattern=CLI_DEFAULT + ["ffn"])
    m.add_adapter(16, 16)
    m.prepare()
    lw = m._lw
    for key in ("kv2", "kv3"):
        ch = lw.chunks(key)
        assert len(ch) >= 2 and ch[0][0] == 0 and ch[-1][1] == nl and all(a[1] == b[0] for a, b in zip(ch, ch[1:]))
    assert lw.kv2_chunks == lw.chunks("kv3") == [(0, 3), (3, 5)]
    # the image-side weights live in the root's fp8 flat only: no view of them in the root slot
    root = lw.root_fp8
    lo, hi = root.data_ptr(), root.data_ptr() + root.numel()
    slot_lo, slot_hi = lw.root_slot.data_ptr(), lw.root_slot.data_ptr() + 2 * lw.root_slot.numel()
    for blk in m.blocks:
        for p in (blk.attn2.add_k_proj.weight, blk.attn2.add_v_proj.bias):
            assert p.dtype == torch.float8_e5m2 and lo <= p.data_ptr() < hi
            assert not slot_lo <= p.data_ptr() < slot_hi
    # the chunk views sit in the block slots, chunk g of the streamed sequence in slot g % 2
    slots = [s.data_ptr() for s in lw.units.slots]
    seq = [v for key in ("kv2", "kv3") for v in lw.stacked[key].views]
    assert [slots.index(W.data_ptr()) for W, _ in seq] == [0, 1, 0, 1]
    # the schedule of one forward, with the upcast kernel restated on the CPU: the root slot, the four chunks, then
    # every block; each chunk is the exact upcast of its blocks' fp8 storage when it is waited for
    from finetrainers_b200 import ops
    monkeypatch.setattr(ops, "upcast_fp8_bf16", lambda src, dst, n: dst.view(-1)[:n].copy_(src.reshape(-1)[:n]))
    m._lw.begin_forward()
    for key, attr in (("kv2", "to_k"), ("kv3", "add_k_proj")):
        for c, (l0, l1) in enumerate(lw.chunks(key)):
            W, b = m._lw.chunk_wait(key, c)
            for l in range(l0, l1):
                lin = getattr(m.blocks[l].attn2, attr)
                lin = getattr(lin, "base_layer", lin)
                assert torch.equal(W[l - l0, :128], lin.weight.to(torch.bfloat16)), (key, l)
                assert torch.equal(b[l - l0, :128], lin.bias.to(torch.bfloat16)), (key, l)
            m._lw.chunk_release(key, c)
    for l in range(nl):
        m._lw.pre_block_forward(l)
        m._lw.post_block_forward(l)
    assert lw.upcasts == 1 + 4 * 2 + nl
    assert lw.units.gathers == 4 + nl


def test_fsdp2_stays_refused_with_fp8_storage():
    from finetrainers_b200.fsdp import FSDPState
    m = engine(True, 2)
    m.enable_layerwise_casting(torch.float8_e4m3fn, skip_modules_pattern=CLI_DEFAULT)
    m.add_adapter(16, 16)
    with pytest.raises(NotImplementedError):
        FSDPState(m)
