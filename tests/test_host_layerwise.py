"""Layerwise fp8 weight storage (``--layerwise_upcasting_modules transformer``), host side: which linear layers the skip
patterns cast, on the oracle's diffusers-named module tree and on the engine's module, the packed storage that results,
and every refused configuration.

The casting rule is diffusers' ``apply_layerwise_casting`` as finetrainers calls it (trainer.py:108-118); diffusers is
not installed here, so ``oracle_layerwise_cast`` below restates it from its documented behaviour, independently of the
engine: walk ``named_children()`` from the root with dotted FQNs, skip a module whose FQN matches any pattern under
``re.search`` together with its subtree, cast an ``nn.Linear``'s weight and bias and do not descend into it."""
import math
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TINY = dict(in_channels=32, out_channels=32, num_attention_heads=2, attention_head_dim=64, cross_attention_dim=128,
            num_layers=3, caption_channels=64)
DATACLASS_DEFAULT = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "time_embed", "^proj_in$", "^proj_out$",
                     "norm"]   # finetrainers/args.py:395
CLI_DEFAULT = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]  # :751-754
BLOCK_LINEARS = ["attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0", "attn2.to_q", "attn2.to_k", "attn2.to_v",
                 "attn2.to_out.0", "ff.net.0.proj", "ff.net.2"]
TIME_EMBED = ["time_embed.emb.timestep_embedder.linear_1", "time_embed.emb.timestep_embedder.linear_2", "time_embed.linear"]
CAPTION = ["caption_projection.linear_1", "caption_projection.linear_2"]


def oracle_layerwise_cast(module, patterns, storage_dtype=None):
    """The restated rule on an ``nn.Module`` tree: returns the cast ``nn.Linear`` FQNs; with ``storage_dtype`` also rounds
    their weights and biases through it in place (the values the reference computes with, bf16(fp8(w)))."""
    cast = []

    def visit(mod, fqn):
        if any(re.search(p, fqn) for p in patterns):
            return
        if isinstance(mod, torch.nn.Linear):
            cast.append(fqn)
            if storage_dtype is not None:
                with torch.no_grad():
                    for p in (mod.weight, mod.bias):
                        if p is not None:
                            p.copy_(p.to(torch.bfloat16).to(storage_dtype).to(p.dtype))
            return
        for name, child in mod.named_children():
            visit(child, f"{fqn}.{name}" if fqn else name)

    visit(module, "")
    return cast


def expected(nl, time_embed, blocks=BLOCK_LINEARS):
    return sorted((TIME_EMBED if time_embed else []) + CAPTION +
                  [f"transformer_blocks.{l}.{n}" for l in range(nl) for n in blocks])


def engine(nl=3):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    torch.manual_seed(0)
    m = B200LTXTransformer(LTXConfig(**dict(TINY, num_layers=nl)), torch.bfloat16, "cpu")
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.05)
    return m


@pytest.mark.parametrize("which", ["dataclass", "cli", "cli+attn2"])
def test_cast_set_matches_expected_on_oracle_and_engine(which):
    from oracle import ltx_oracle as O
    from finetrainers_b200.model import apply_layerwise_casting
    patterns = {"dataclass": DATACLASS_DEFAULT, "cli": CLI_DEFAULT, "cli+attn2": CLI_DEFAULT + ["attn2"]}[which]
    blocks = [b for b in BLOCK_LINEARS if not b.startswith("attn2")] if which == "cli+attn2" else BLOCK_LINEARS
    want = expected(3, which != "dataclass", blocks)
    om = O.LTXTransformerOracle(O.LTXConfig(**TINY))
    assert sorted(oracle_layerwise_cast(om, patterns)) == want
    m = engine()
    apply_layerwise_casting(m, torch.float8_e4m3fn, torch.bfloat16, patterns, non_blocking=True)
    assert sorted(m._lw_cfg["cast"]) == want
    # the stored state: exactly the cast linears' weights and biases are fp8, proj_in / proj_out never
    fp8 = sorted(n for n, p in m.named_parameters() if p.dtype == torch.float8_e4m3fn)
    assert fp8 == sorted(f"{n}.{w}" for n in want for w in ("weight", "bias"))
    assert m.proj_in.weight.dtype == m.proj_out.weight.dtype == torch.bfloat16


def test_fp8_values_are_torch_casts_and_survive_prepare_and_adapter():
    from finetrainers_b200.model import apply_layerwise_casting
    m = engine()
    w0 = {n: p.detach().clone() for n, p in m.named_parameters()}
    apply_layerwise_casting(m, torch.float8_e5m2, torch.bfloat16, CLI_DEFAULT)
    m.add_adapter(16, 16)
    m.prepare()
    for n, p in m.named_parameters():
        if "lora_" in n:
            assert p.dtype == torch.float32, n
            continue
        src = w0[n.replace(".base_layer", "")]
        want = src.to(torch.float8_e5m2) if p.dtype == torch.float8_e5m2 else src
        assert torch.equal(p.detach().view(torch.uint8) if p.dtype == torch.float8_e5m2 else p.detach(),
                           want.view(torch.uint8) if want.dtype == torch.float8_e5m2 else want), n
    # .to(dtype=bf16) keeps fp8 storage with unchanged values (the reference re-casts to storage after each forward)
    before = {n: p.detach().clone() for n, p in m.named_parameters()}
    m.to(dtype=torch.bfloat16)
    for n, p in m.named_parameters():
        assert p.dtype == before[n].dtype, n
        assert torch.equal(p.detach().float(), before[n].float()), n
    assert m._blk[0]["Wqkv"].data_ptr() == m._lw.units.slots[0].data_ptr()


def test_storage_bytes_after_prepare_match_the_specs():
    from finetrainers_b200.model import apply_layerwise_casting
    nl = 5
    m = engine(nl)
    apply_layerwise_casting(m, torch.float8_e4m3fn, torch.bfloat16, CLI_DEFAULT)
    m.add_adapter(16, 16)
    m.prepare()
    d, f, cin, cout, cap = 128, 512, 32, 32, 64
    r16 = lambda n: (n + 15) // 16 * 16  # noqa: E731  (fp8 pieces start on 16-byte boundaries)
    blk_cast = [3 * d * d, 3 * d, d * d, d, d * d, d, d * d, d, f * d, f, d * f, d]
    root_slot = [256 * d, d, d * d, d, 6 * d * d, 6 * d, cap * d, d, d * d, d]
    kv2 = [nl * 2 * d * d, nl * 2 * d]
    fp8 = nl * sum(map(r16, blk_cast)) + sum(map(r16, root_slot + kv2))
    align = lambda n: (n + 2047) // 2048 * 2048  # noqa: E731  (FLAT_ALIGN of every bf16 unit)
    bf16_blk = align(3 * d + 6 * d)                 # norm_q / norm_k / norm_q2 weights + scale_shift_table
    bf16_root = align(d * cin + d + 2 * d + cout * d + cout + nl * d)
    got = m.base_weight_bytes()
    assert got["fp8_storage"] == fp8
    assert got["bf16_resident"] == 2 * (nl * bf16_blk + bf16_root)
    assert got["block_slots"] == 2 * 2 * sum(map(r16, blk_cast))
    assert got["root_slot"] == 2 * sum(map(r16, root_slot))
    # the text-side [Wk2;Wv2] of all blocks streams through the block slots: no persistent bf16 copy
    assert m._Wkv2_all is None and m._lw.kv2_chunks == [(0, nl)]
    # nothing cast: today's layout, no schedule
    m2 = engine(nl)
    apply_layerwise_casting(m2, torch.float8_e4m3fn, torch.bfloat16, [".*"])
    m2.add_adapter(16, 16)
    m2.prepare()
    assert m2._lw is None and m2._Wkv2_all is not None and m2.base_weight_bytes()["fp8_storage"] == 0


@pytest.mark.parametrize("pattern,names", [
    ("to_k", ["attn1.to_q", "attn1.to_k"]),                      # q/k/v of self-attention share Wqkv
    (r"transformer_blocks\.1\.attn2", ["attn2.to_k"]),           # every block's text-side k/v share Wkv2_all
    (r"^transformer_blocks\.0\.attn1\.to_v$", ["attn1.to_v"]),
])
def test_a_pattern_that_splits_a_fused_weight_raises(pattern, names):
    from finetrainers_b200.model import apply_layerwise_casting
    m = engine()
    with pytest.raises(NotImplementedError) as ei:
        apply_layerwise_casting(m, torch.float8_e4m3fn, torch.bfloat16, CLI_DEFAULT + [pattern])
    for n in names:
        assert n in str(ei.value)
    assert m._lw_cfg is None and all(p.dtype == torch.bfloat16 for p in m.parameters())   # nothing changed


def test_refused_configurations():
    from finetrainers_b200.model import apply_layerwise_casting
    m = engine()
    with pytest.raises(ValueError):
        apply_layerwise_casting(m, torch.float16, torch.bfloat16, CLI_DEFAULT)
    with pytest.raises(NotImplementedError):
        apply_layerwise_casting(m, torch.float8_e4m3fn, torch.float32, CLI_DEFAULT)
    with pytest.raises(NotImplementedError):
        apply_layerwise_casting(m, torch.float8_e4m3fn, torch.bfloat16, CLI_DEFAULT, skip_modules_classes=(torch.nn.LayerNorm,))
    with pytest.raises(NotImplementedError):
        apply_layerwise_casting(m, torch.float8_e4m3fn, torch.bfloat16)   # diffusers' "auto" list
    with pytest.raises(TypeError):
        apply_layerwise_casting(torch.nn.Linear(4, 4), torch.float8_e4m3fn, torch.bfloat16, CLI_DEFAULT)
    apply_layerwise_casting(m, torch.float8_e4m3fn, torch.bfloat16, CLI_DEFAULT)
    with pytest.raises(ValueError):   # a second call
        apply_layerwise_casting(m, torch.float8_e5m2, torch.bfloat16, CLI_DEFAULT)
    m2 = engine()
    m2.add_adapter(16, 16)
    with pytest.raises(ValueError):   # after add_adapter: the adapters would be cast
        apply_layerwise_casting(m2, torch.float8_e4m3fn, torch.bfloat16, CLI_DEFAULT)


_FSDP_WORKER = r'''
import os, sys, torch
sys.path.insert(0, os.environ["B2D_ROOT"])
from finetrainers_b200.parallel import B200ParallelBackend
from finetrainers_b200.model import B200LTXTransformer, LTXConfig, apply_layerwise_casting
be = B200ParallelBackend(backend="gloo", device_type="cpu", dp_shards=2)
cfg = LTXConfig(in_channels=32, out_channels=32, num_attention_heads=2, attention_head_dim=64, cross_attention_dim=128,
                num_layers=2, caption_channels=64)
pat = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]
kw = dict(param_dtype=torch.bfloat16, reduce_dtype=torch.float32, output_dtype=None, pp_enabled=False, cpu_offload=False,
          device_mesh=be.get_mesh()[("dp_shard_cp",)])
m = B200LTXTransformer(cfg, torch.bfloat16, "cpu")
apply_layerwise_casting(m, torch.float8_e4m3fn, torch.bfloat16, pat)
m.add_adapter(16, 16)
try:
    be.apply_fsdp2(m, **kw); raise SystemExit("FSDP-2 accepted a layerwise model")
except NotImplementedError:
    pass
assert m._fsdp is None
m = B200LTXTransformer(cfg, torch.bfloat16, "cpu")
be.apply_fsdp2(m, **kw)
try:
    apply_layerwise_casting(m, torch.float8_e4m3fn, torch.bfloat16, pat); raise SystemExit("layerwise accepted under FSDP-2")
except NotImplementedError:
    pass
be.wait_for_everyone()
be.destroy()
print("LW_FSDP_OK", be.rank)
'''


def test_fsdp2_refuses_layerwise_in_either_order_world2_gloo(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_FSDP_WORKER)
    env = dict(os.environ, B2D_ROOT=ROOT, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29561", str(script)], env=env,
                       capture_output=True, text=True, timeout=240)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.count("LW_FSDP_OK") == 2
