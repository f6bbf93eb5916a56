"""CPU: host-side logic of the b200 package — C ABI surface, parameter packing / FQNs, sigma sampling, provider
registry, and the world_size-2 gloo path of the parallel backend."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_builds_and_exports_every_declared_symbol():
    from finetrainers_b200 import lib
    path = lib.build()
    so = ctypes.CDLL(path)
    header = open(os.path.join(ROOT, "include", "b2d.h")).read()
    declared = set(re.findall(r"\b(b2d_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    assert declared == set(lib.EXPORTS), declared ^ set(lib.EXPORTS)
    for name in declared:
        assert hasattr(so, name), f"{name} declared in include/b2d.h but not exported"
    so.b2d_version.restype = ctypes.c_int
    assert so.b2d_version() == 2


def test_reading_the_launch_count_does_not_load_the_library():
    """ops.LAUNCH_COUNT is 0 before anything loaded libb2d, and reading it does not load (or build) the library."""
    code = ("import sys; sys.path.insert(0, sys.argv[1]); from finetrainers_b200 import lib, ops; "
            "assert ops.LAUNCH_COUNT == 0; assert lib._lib is None; print('LAUNCH_COUNT_OK')")
    r = subprocess.run([sys.executable, "-c", code, ROOT], capture_output=True, text=True, timeout=240)
    assert r.returncode == 0 and "LAUNCH_COUNT_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def test_every_dependent_launch_kernel_waits_for_its_predecessors():
    """launch_k / launch_kc attach the programmatic-dependent-launch attribute: a kernel launched through them may start
    while its predecessor is still running, so EVERY such kernel must execute griddep_wait() before it touches global
    memory (and griddep_launch_dependents() so that the scheme has an effect).  A kernel added later without the wait would
    be a silent race; this keeps the source honest."""
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "finetrainers_b200", "csrc")
    src = {f: open(os.path.join(root, f)).read() for f in os.listdir(root) if f.endswith(".cu")}
    launched = set()
    for text in src.values():
        for m in re.finditer(r"launch_kc?\(\s*([A-Za-z_][A-Za-z0-9_]*)", text):
            launched.add(m.group(1))
    launched.discard("kern")            # launch_gemm passes the instantiated template through a local
    launched.add("gemm_kernel")
    if "KERNEL" in launched:            # ROW_DISPATCH(D, KERNEL, ...) macro: collect its instantiations
        launched.discard("KERNEL")
        for text in src.values():
            launched.update(re.findall(r"ROW_DISPATCH\([^,]+,\s*([A-Za-z_][A-Za-z0-9_]*)", text))
    launched.discard("KERNEL")
    assert len(launched) >= 10, launched
    allsrc = "\n".join(src.values())
    for k in sorted(launched):
        m = re.search(r"__global__[^;{]*\b" + k + r"\s*\(", allsrc)
        assert m, f"kernel {k} not found"
        # function body: from the first '{' after the signature to the matching '}'
        i = allsrc.index("{", allsrc.index(")", m.end()))
        depth, j = 0, i
        while True:
            c = allsrc[j]
            depth += c == "{"
            depth -= c == "}"
            if depth == 0:
                break
            j += 1
        body = allsrc[i:j]
        assert "griddep_wait()" in body, f"{k} is launched with the dependent-launch attribute but never waits"
        assert "griddep_launch_dependents()" in body, f"{k} never releases its dependents early"


def test_ops_fail_loudly_without_cuda():
    from finetrainers_b200 import ops, lib
    x = torch.zeros(8, 8, dtype=torch.bfloat16)
    with pytest.raises(lib.B2DError):
        ops.colscale(x, x, x[0], x, 8, 8, 8, 8)


def test_model_fqns_match_oracle_and_packing_is_lossless():
    from oracle import ltx_oracle as O
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    cfgk = dict(in_channels=32, out_channels=32, num_attention_heads=2, attention_head_dim=64, cross_attention_dim=128,
                num_layers=2, caption_channels=64)
    om = O.LTXTransformerOracle(O.LTXConfig(**cfgk))
    O.add_lora(om, 16, 32)
    O.synthetic_init_(om)
    bm = B200LTXTransformer(LTXConfig(**cfgk), torch.bfloat16, "cpu")
    bm.add_adapter(16, 32)
    assert [n for n, _ in bm.named_parameters()] == [n for n, _ in om.named_parameters()] or \
        set(n for n, _ in bm.named_parameters()) == set(n for n, _ in om.named_parameters())
    bm.load_state_dict(om.state_dict(), strict=True)
    before = {k: v.clone() for k, v in bm.state_dict().items()}
    bm.prepare()
    after = bm.state_dict()
    for k in before:
        assert torch.equal(before[k], after[k]), k
    # fused views: q/k/v weights are consecutive rows of one buffer; LoRA params are views of the flat fp32 buffer
    e = bm._blk[0]
    a1 = bm.transformer_blocks[0].attn1
    assert a1.to_k.base_layer.weight.data_ptr() == e["Wqkv"][128:].data_ptr()
    assert a1.to_q.lora_A["default"].weight.dtype == torch.float32
    assert bm.rpad == 64 and bm.lora_scaling == 2.0
    assert a1.to_v.lora_B["default"].weight.shape == (128, 16)
    n_lora = sum(p.numel() for p in bm.lora_parameters())
    assert n_lora == 2 * 8 * 16 * 128 * 2
    # padded entries of the flat buffer are exactly zero
    assert bm.lora_flat.abs().sum() > 0
    assert torch.count_nonzero(bm.lora_flat).item() <= n_lora
    # only adapters train
    assert all(("lora_" in n) == p.requires_grad for n, p in bm.named_parameters())


def test_sigma_sampling_matches_reference_golden(golden):
    from finetrainers_b200.trainer import prepare_sigmas, prepare_loss_weights
    from finetrainers_b200.specification import FlowMatchSchedulerTable
    sch = FlowMatchSchedulerTable()
    assert torch.equal(sch.sigmas, golden["sig_table"])
    for scheme in ("none", "logit_normal", "mode"):
        gen = torch.Generator().manual_seed(1234)
        s = prepare_sigmas(sch, sch.sigmas, 16, 1000, scheme, 0.0, 1.0, 1.29, "cpu", gen)
        assert torch.equal(s, golden[f"sig_{scheme}"])
    sig = torch.tensor([0.25, 0.5])
    assert torch.equal(prepare_loss_weights(sig, "none"), torch.ones(2))
    assert torch.allclose(prepare_loss_weights(sig, "sigma_sqrt"), torch.tensor([16.0, 4.0]))


def test_attention_provider_registry_api():
    from finetrainers_b200 import attention as A
    assert A.AttentionProvider.B200 in A._AttentionProviderRegistry.list_providers()
    name, fn = A._AttentionProviderRegistry.get_active_provider()
    assert name == A.AttentionProvider.B200
    assert {"query", "key", "value", "attn_mask", "scale"} <= A._AttentionProviderRegistry._supported_arg_names[name]
    with A.attention_provider(A.AttentionProvider.B200):
        pass
    with pytest.raises(ValueError):
        with A.attention_provider("flash"):
            pass
    assert not A._AttentionProviderRegistry.supports_context_parallel(A.AttentionProvider.B200)
    # constraint checks raise ValueError like the reference's (_check_device/_check_shape)
    q = torch.zeros(1, 2, 8, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        A._check_b200(q, q, q)


_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["B2D_ROOT"])
from finetrainers_b200.parallel import B200ParallelBackend, allreduce_flat_grads, fused_step_metrics, dist_mean, dist_max
be = B200ParallelBackend(backend="gloo", device_type="cpu")
assert be.world_size == 2 and be.data_replication_enabled and not be.data_sharding_enabled
r = be.rank
m = torch.nn.Linear(4, 4)
torch.manual_seed(r)
with torch.no_grad():
    for p in m.parameters():
        p.normal_()
be.apply_ddp(m)
w = m.weight.detach().clone()
g = [torch.zeros_like(w) for _ in range(2)]
dist.all_gather(g, w)
assert torch.equal(g[0], g[1]), "replicas must start identical"
flat = torch.full((1000,), float(r + 1))
allreduce_flat_grads(flat, chunk_bytes=1024)
assert torch.allclose(flat, torch.full((1000,), 1.5))
mt = fused_step_metrics(torch.tensor(2.0 * (r + 1)), torch.tensor(float(r)))
assert abs(mt["train/grad_norm"] - 3.0) < 1e-6 and abs(mt["train/global_avg_loss"] - 0.5) < 1e-6 and mt["train/global_max_loss"] == 1.0
assert dist_mean(torch.tensor([float(r)])) == 0.5 and dist_max(torch.tensor([float(r)])) == 1.0
be.wait_for_everyone()
be.destroy()
print("WORKER_OK", r)
'''


def test_parallel_backend_world2_gloo(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    env = dict(os.environ, B2D_ROOT=ROOT, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29531", str(script)], env=env,
                       capture_output=True, text=True, timeout=240)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert r.stdout.count("WORKER_OK") == 2


_FSDP_WORKER = r'''
import os, sys, math, torch, torch.distributed as dist
sys.path.insert(0, os.environ["B2D_ROOT"])
from finetrainers_b200.parallel import B200ParallelBackend
from finetrainers_b200.fsdp import ShardedUnits, ShardedFlatOptimizer, shard_bounds
from finetrainers_b200.model import B200LTXTransformer, LTXConfig
be = B200ParallelBackend(backend="gloo", device_type="cpu", dp_shards=2)
assert be.world_size == 2 and be.data_sharding_enabled and not be.data_replication_enabled and be._dp_degree == 1
r = be.rank
mesh = be.get_mesh()[("dp_shard_cp",)]
assert mesh.size() == 2 and mesh.get_local_rank() == r

# ---- 1. units: every rank keeps 1/W of each flat unit; gather schedule forward then backward
flats = [torch.arange(4096, dtype=torch.float32) + 10000 * i for i in range(5)]
su = ShardedUnits([f.clone() for f in flats], None)
assert su.shards[3].numel() == 2048 and torch.equal(su.shards[3], flats[3][r * 2048:(r + 1) * 2048])
su.prefetch(0); su.prefetch(1)
for l in range(5):
    assert torch.equal(su.wait(l), flats[l]), l
    if l + 2 < 5:
        su.release(l, l + 2)
assert sorted(su.resident) == [3, 4]
for l in range(4, -1, -1):
    assert torch.equal(su.wait(l), flats[l]), l
    su.release(l, l - 2)
assert sorted(su.resident) == [0, 1] and su.gathers == 5 + 3
try:
    shard_bounds(10, 0, 4); raise SystemExit("uneven split accepted")
except ValueError:
    pass

# ---- 2. sharded optimizer == AdamW + clip on the rank-averaged gradient
torch.manual_seed(0)
p0 = torch.randn(512)
g_all = [torch.randn(512) * (i + 1) for i in range(2)]
def adamw(p, g, m, v, sumsq, step=1, lr=1e-2, b1=0.9, b2=0.99, eps=1e-8, wd=1e-4, max_norm=1.0):
    coef = min(1.0, max_norm / (math.sqrt(float(sumsq)) + 1e-6))
    g = g * coef
    p.mul_(1 - lr * wd)
    m.mul_(b1).add_(g, alpha=1 - b1); v.mul_(b2).addcmul_(g, g, value=1 - b2)
    p.addcdiv_(m / (1 - b1 ** step), (v / (1 - b2 ** step)).sqrt() + eps, value=-lr)
pr, mr, vr = p0.clone(), torch.zeros(512), torch.zeros(512)
gm = (g_all[0] + g_all[1]) / 2
adamw(pr, gm, mr, vr, (gm ** 2).sum())
params = p0.clone()
opt = ShardedFlatOptimizer(params, None)
assert opt.exp_avg.numel() == 256
grad = g_all[r].clone()
ss = opt.step(grad, lambda gs: (gs ** 2).sum().reshape(1), lambda p, gs, m, v, s: adamw(p, gs, m, v, s))
assert abs(float(ss) - float((gm ** 2).sum())) < 1e-3 * float(ss)
assert torch.allclose(params, pr, atol=1e-6), (params - pr).abs().max()
assert grad.abs().max() == 0

# ---- 3. the real module: apply_fsdp2 re-binds the parameters onto gather slots; every block's weights are correct
# while it is resident, in forward order and in backward order (incl. the previous block's gate row read by block l)
cfg = LTXConfig(in_channels=32, out_channels=32, num_attention_heads=2, attention_head_dim=64, cross_attention_dim=128,
                num_layers=4, caption_channels=64)
torch.manual_seed(1)            # same weights on both ranks (apply_fsdp2 also broadcasts rank 0's)
m = B200LTXTransformer(cfg, torch.bfloat16, "cpu")
with torch.no_grad():
    for p in m.parameters():
        p.normal_(0, 0.02)
m.add_adapter(16, 16)
m.prepare()
want = {k: v.clone() for k, v in m.state_dict().items()}
total = sum(f.numel() for f in m._blk_flat) + m._root_flat.numel()
be.apply_fsdp2(m, param_dtype=torch.bfloat16, reduce_dtype=torch.float32, output_dtype=None, pp_enabled=False,
               cpu_offload=False, device_mesh=be.get_mesh()[("dp_shard_cp",)])
fs = m._fsdp
assert fs.local_param_bytes() * 2 == total * 2, (fs.local_param_bytes(), total)   # bf16: half of the elements, 2 bytes each
assert m._blk_flat is None
blk_keys = lambda l: [k for k in want if k.startswith(f"transformer_blocks.{l}.") and "lora_" not in k and "attn2.to_k" not in k
                      and "attn2.to_v" not in k and "attn2.norm_k" not in k]
sd = lambda: dict(m.named_parameters())
fs.begin_forward()
for k in want:
    if not k.startswith("transformer_blocks.") or "attn2.to_k" in k or "attn2.to_v" in k or "attn2.norm_k" in k:
        assert torch.equal(sd()[k].data, want[k]), k          # root unit resident for the whole step
for l in range(4):
    fs.pre_block_forward(l)
    for k in blk_keys(l):
        assert torch.equal(sd()[k].data, want[k]), k
    fs.post_block_forward(l)
for l in range(3, -1, -1):
    fs.pre_block_backward(l)
    for k in blk_keys(l):
        assert torch.equal(sd()[k].data, want[k]), k
    if l > 0:
        fs.pre_block_backward(l - 1)
        assert torch.equal(m._blk[l - 1]["sst"], want[f"transformer_blocks.{l - 1}.scale_shift_table"])
    fs.post_block_backward(l)
fs.end_backward()
full = fs.full_state_dict()
assert set(full) == set(want)
for k in want:
    assert torch.equal(full[k], want[k]), k
be.wait_for_everyone()
be.destroy()
print("FSDP_WORKER_OK", r)
'''


def test_fsdp2_sharding_bookkeeping_world2_gloo(tmp_path):
    """FSDP-2 (ptd.py:466-499) on the gloo backend, world 2: flat-unit sharding and the gather/release schedule, the
    ZeRO-style sharded AdamW against plain AdamW on the averaged gradient, and ``apply_fsdp2`` on the real module."""
    script = tmp_path / "f.py"
    script.write_text(_FSDP_WORKER)
    env = dict(os.environ, B2D_ROOT=ROOT, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29541", str(script)], env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert r.stdout.count("FSDP_WORKER_OK") == 2


def test_precomputed_reader_follows_reference_layout(tmp_path):
    """SURVEY §8f-2: {data_type}-{index}.pt items, rank r owns indices r*num_items + i (precomputation.py:334-341)."""
    from finetrainers_b200.data import PrecomputedReader, save_item
    for i in range(4):
        save_item({"latents": torch.full((1, 8, 1, 2, 2), float(i)), "num_frames": 1}, i, tmp_path, "latent")
    rd = PrecomputedReader(tmp_path, "latent", rank=0, world_size=1, device=None)
    assert len(rd) == 4
    vals = [int(it["latents"][0, 0, 0, 0, 0]) for it in rd]
    assert vals == [0, 1, 2, 3] and rd.requires_data


def test_resolution_sampler_and_collate_follow_reference_protocol():
    """data/sampler.py:6-58 + modeling_utils.py:156-181: bucket by the leader tensor's (F,H,W), release full buckets,
    concatenate tensors along dim 0, pass the ignore-keys through from the first item."""
    from finetrainers_b200.data import ResolutionSampler, collate
    from finetrainers_b200.specification import LTXVideoModelSpecification
    s = ResolutionSampler(batch_size=2, dim_keys={"latents": (2, 3, 4)})
    mk = lambda f, v: ({"encoder_hidden_states": torch.full((1, 4, 8), float(v)), "encoder_attention_mask": torch.ones(1, 4, dtype=torch.bool)},
                       {"latents": torch.full((1, 8, f, 2, 2), float(v)), "num_frames": f, "height": 2, "width": 2,
                        "latents_mean": torch.zeros(1, 8), "latents_std": torch.ones(1, 8)})
    s.consume(*mk(1, 0)); assert not s.is_ready
    s.consume(*mk(3, 1)); assert not s.is_ready          # different resolution: another bucket
    s.consume(*mk(1, 2)); assert s.is_ready
    cond_b, lat_b = s.get_batch()
    assert not s.is_ready and len(cond_b) == 2 and len(lat_b) == 2
    spec = LTXVideoModelSpecification()
    lat = spec.collate_latents(list(lat_b))
    cond = spec.collate_conditions(list(cond_b))
    assert lat["latents"].shape == (2, 8, 1, 2, 2) and lat["latents"][:, 0, 0, 0, 0].tolist() == [0.0, 2.0]
    assert lat["num_frames"] == 1 and lat["latents_mean"].shape == (1, 8)   # ignore-keys: first item only
    assert cond["encoder_hidden_states"].shape == (2, 4, 8)
    assert collate([{"a": "x"}, {"a": "y"}]) == {"a": ["x", "y"]}
    with pytest.raises(ValueError):
        ResolutionSampler(1, {"latents": (2,)}).consume({"foo": torch.zeros(1)})
    with pytest.raises(ValueError):
        ResolutionSampler(1, {"latents": (2,), "x": (0,)}).consume({"latents": torch.zeros(1, 1, 1)}, {"x": torch.zeros(1)})


def test_precomputed_once_reader_cycles_over_rank_slice(tmp_path):
    """precomputation.py:348-382: infinite iterator over indices rank*per_rank + i."""
    from finetrainers_b200.data import PrecomputedOnceReader, save_item
    for i in range(4):
        save_item({"latents": torch.full((1, 2), float(i))}, i, tmp_path, "latent")
    rd = PrecomputedOnceReader(tmp_path, "latent", rank=1, world_size=2, device=None)
    assert len(rd) == 2
    it = iter(rd)
    assert [int(next(it)["latents"][0, 0]) for _ in range(5)] == [2, 3, 2, 3, 2] and not rd.requires_data
    with pytest.raises(ValueError):
        PrecomputedOnceReader(tmp_path, "latent", rank=7, world_size=8)


class _LoraConfig:
    """Field-for-field what ``peft.LoraConfig(r=, lora_alpha=, init_lora_weights=, target_modules=)`` carries
    (peft is not installed here)."""

    def __init__(self, r, lora_alpha, init_lora_weights, target_modules):
        self.r, self.lora_alpha, self.init_lora_weights, self.target_modules = r, lora_alpha, init_lora_weights, target_modules
        self.lora_dropout = 0.0


def test_trainer_prepare_call_sequence_replays_on_the_b200_module():
    """Replays ``SFTTrainer._prepare_trainable_parameters`` / ``_prepare_for_training`` call for call
    (trainer.py:95-216) against the drop-in module and backend: requires_grad_(False), add_adapter(LoraConfig(...)) with
    the reference's default target regex (config.py:26), cast_training_params(fp32), get_mesh().ndim, prepare_model,
    .to(device), trainable-parameter count, parameters() for the optimizer, zero_grad."""
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    from finetrainers_b200.parallel import B200ParallelBackend
    cfg = LTXConfig(in_channels=32, out_channels=32, num_attention_heads=2, attention_head_dim=64, cross_attention_dim=128,
                    num_layers=2, caption_channels=64)
    tr = B200LTXTransformer(cfg, torch.bfloat16, "cpu")
    with torch.no_grad():
        for p in tr.parameters():
            p.normal_(0, 0.02)
    be = B200ParallelBackend(device_type="cpu")
    tr.requires_grad_(False)                                                      # utils.set_requires_grad([...], False)
    rx = "(transformer_blocks|single_transformer_blocks).*(to_q|to_k|to_v|to_out.0)"
    tr.add_adapter(_LoraConfig(r=16, lora_alpha=32, init_lora_weights=True, target_modules=rx))     # trainer.py:122-128
    assert not be.data_sharding_enabled
    for p in tr.parameters():                                                     # diffusers cast_training_params(fp32)
        if p.requires_grad:
            p.data = p.to(torch.float32)
    assert not be.context_parallel_enabled and not be.tensor_parallel_enabled and not be.pipeline_parallel_enabled
    mesh = be.get_mesh()
    assert mesh.ndim == 1
    for key in ("dp", "dp_cp", "dp_replicate", "dp_shard_cp", "pp", "cp", "tp"):  # every key the loop indexes
        assert be.get_mesh()[key].ndim == 1
    assert be.get_mesh()[("dp_replicate", "dp_shard_cp")].size() == 1
    with pytest.raises(KeyError):
        be.get_mesh()["nope"]
    be.prepare_model(tr)
    tr.prepare()
    before = {k: v.clone() for k, v in tr.state_dict().items()}
    tr.to("cpu")                                                                  # _move_components_to_device: no-op move
    tr.to(dtype=torch.bfloat16)                                                   # a cast AFTER prepare(): must re-pack
    assert tr._prepared
    a1 = tr.transformer_blocks[0].attn1
    assert a1.to_k.base_layer.weight.data_ptr() == tr._blk[0]["Wqkv"][128:].data_ptr()
    assert a1.to_q.lora_A["default"].weight.dtype == torch.float32               # fp32 masters survive the cast
    assert a1.to_q.lora_A["default"].weight.data_ptr() == tr._blk[0]["A_qkv"].data_ptr()
    for k, v in tr.state_dict().items():
        assert torch.equal(v.float(), before[k].float()), k
    trainable = [p for p in tr.parameters() if p.requires_grad]
    assert sum(p.numel() for p in trainable) == 2 * 8 * 2 * 16 * 128               # blocks * linears * (A + B) * r * d
    assert tr.lora_scaling == 2.0 and tr.lora_rank == 16
    opt = torch.optim.AdamW(trainable, lr=1e-3)
    opt.zero_grad()                                                               # set_to_none: grads re-attach lazily
    assert tr._attach_lora_grads()
    sd = {k: torch.zeros_like(v) for k, v in tr.state_dict().items()}
    tr.load_state_dict(sd)                                                        # in-place copy keeps the packed views
    assert tr._blk[0]["Wqkv"].abs().max().item() == 0.0 and tr.lora_flat.abs().max().item() == 0.0
    # list-form targets (peft suffix matching) select the same modules; anything else is refused loudly
    tr2 = B200LTXTransformer(cfg, torch.bfloat16, "cpu")
    tr2.add_adapter(_LoraConfig(8, 8, "gaussian", ["to_q", "to_k", "to_v", "to_out.0"]))
    assert tr2.lora_rank == 8
    tr3 = B200LTXTransformer(cfg, torch.bfloat16, "cpu")
    with pytest.raises(NotImplementedError):
        tr3.add_adapter(_LoraConfig(8, 8, True, ["to_q", "to_v"]))
    with pytest.raises(NotImplementedError):
        tr3.add_adapter(_LoraConfig(8, 8, True, ".*(to_q|to_k|to_v|to_out.0|proj)"))


def test_lora_export_keys_and_values(tmp_path):
    """SURVEY §8f-3: adapters export under diffusers/peft names and round-trip bit-exactly."""
    from safetensors.torch import load_file
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    cfg = LTXConfig(in_channels=32, out_channels=32, num_attention_heads=2, attention_head_dim=64, cross_attention_dim=128,
                    num_layers=1, caption_channels=64)
    m = B200LTXTransformer(cfg, torch.bfloat16, "cpu")
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.02)
    m.add_adapter(16, 16)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "lora_B" in n:
                p.normal_(0, 0.01)
    m.prepare()
    path = m.save_lora_weights(tmp_path)
    sd = load_file(path)
    k = "transformer.transformer_blocks.0.attn2.to_out.0.lora_B.weight"
    assert k in sd and sd[k].shape == (128, 16) and sd[k].dtype == torch.float32
    assert torch.equal(sd[k], m.transformer_blocks[0].attn2.to_out[0].lora_B["default"].weight.detach())
    assert len(sd) == 16


@pytest.mark.parametrize("rank,alpha", [(16, 16), (16, 64), (7, 29), (96, 64), (8, 2.5)])
def test_lora_export_metadata_records_rank_and_alpha(tmp_path, rank, alpha):
    """The saved LoRA config carries r and lora_alpha exactly as given (an integer alpha stays an integer, as in the
    reference's save hook): rank * (alpha / rank) is not always alpha again in floating point (7 * (29 / 7) = 29.000000000000004)."""
    import json
    from safetensors import safe_open
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    cfg = LTXConfig(in_channels=32, out_channels=32, num_attention_heads=2, attention_head_dim=64, cross_attention_dim=128,
                    num_layers=1, caption_channels=64)
    m = B200LTXTransformer(cfg, torch.bfloat16, "cpu")
    m.add_adapter(rank, alpha)
    assert m.lora_scaling == alpha / rank
    m.prepare()
    with safe_open(m.save_lora_weights(tmp_path), "pt") as f:
        text = f.metadata()["lora_config"]
    lc = json.loads(text)
    assert lc["r"] == rank and lc["lora_alpha"] == alpha, text
    assert isinstance(lc["lora_alpha"], int) == float(alpha).is_integer(), text


def test_lr_schedules_match_reference_lambdas():
    """finetrainers_b200.lr_schedule against the factors the reference's own lambda functions produce
    (tests/golden/make_lr_golden.py executes finetrainers/optimizer.py:250-432 unmodified)."""
    import json
    import os
    from finetrainers_b200.lr_schedule import SCHEDULES, lr_factor_fn
    cases = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "lr_golden.json")))
    assert {c["name"] for c in cases} == set(SCHEDULES)
    for c in cases:
        fn = lr_factor_fn(c["name"], **c["kwargs"])
        for step, want in zip(c["steps"], c["factors"]):
            assert fn(step) == want, (c["name"], c["kwargs"], step)
    with pytest.raises(ValueError):
        lr_factor_fn("cosine")            # needs num_training_steps
    with pytest.raises(ValueError):
        lr_factor_fn("nope")


def test_conformance_helpers_bound_and_sentinel():
    """The helpers the GPU conformance tests rest on: bf16_ulp is the spacing of bf16 numbers; check_bound accepts a
    correctly rounded result at a 1-ulp bound and rejects a 2-ulp perturbation, naming the element; check_sentinel
    flags a single changed element outside the windows and ignores writes inside them."""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from _util import bf16_ulp, check_bound, check_sentinel, f32_ulp, sentinel_buffer, window
    x = torch.tensor([1.0, 1.5, 2.0, -3.0, 0.0, 2.0 ** -130], dtype=torch.float64)
    assert bf16_ulp(x).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -6, 2.0 ** -133, 2.0 ** -133]
    assert f32_ulp(torch.tensor([1.0, 3.0], dtype=torch.float64)).tolist() == [2.0 ** -23, 2.0 ** -22]
    torch.manual_seed(0)
    ref = torch.randn(64, 48, dtype=torch.float64) * 10
    got = ref.to(torch.bfloat16)
    assert check_bound(got, ref, bf16_ulp(ref), "rounded") <= 0.5
    bad = got.clone()
    bad[5, 7] = (bad[5, 7].double() + 2 * bf16_ulp(bad[5, 7].double())).to(torch.bfloat16)
    with pytest.raises(AssertionError, match=r"\(5, 7\)"):
        check_bound(bad, ref, bf16_ulp(ref), "perturbed")
    nan = got.clone()
    nan[1, 2] = float("nan")
    with pytest.raises(AssertionError, match=r"\(1, 2\)"):
        check_bound(nan, ref, bf16_ulp(ref), "nan")
    for dtype in (torch.bfloat16, torch.float32):
        buf = sentinel_buffer(10 * 16 + 8, dtype, device="cpu")
        w = window(buf, 3, 10, 12, 16)
        w.fill_(1.0)
        check_sentinel(buf, [w], "inside only")
        buf[3 + 9 * 16 + 12] = 1.0          # one element past the last window row's end
        with pytest.raises(AssertionError, match="1 element"):
            check_sentinel(buf, [w], "outside")
