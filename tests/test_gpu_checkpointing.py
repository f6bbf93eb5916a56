"""GPU: activation checkpointing.  A recomputed block re-runs its forward with the same kernels and arguments into a
scratch slot and its adapter weight gradients run as single-block launches with the batched launches' tile schedule,
so a checkpointed model trains bit for bit like the keep-all model: every step's loss and gradient norm, the
prediction of every micro-step and the whole fp32 LoRA flat are compared with ``torch.equal`` (CUDA-graph steps,
gradient accumulation 2, first-frame conditioning on one micro-step).  The saved memory is checked against the
workspace plan, and the 13B model trains a 121-frame 768x512 clip (6144 latent tokens) on one card."""
import gc
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI_SKIP = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]
GRID, L = (7, 16, 24), 128          # 2688 latent tokens (49x512x768), 128 text tokens


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _build(cfg, policy, ffn=False, fmt=None, seed=0):
    from finetrainers_b200.model import (B200LTXTransformer, LORA_FFN_TARGETS, apply_activation_checkpointing,
                                         apply_layerwise_casting)
    torch.manual_seed(seed)
    m = B200LTXTransformer(cfg, torch.bfloat16, "cuda")
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "scale_shift_table" in n:
                p.normal_(0, 1.0 / p.shape[-1] ** 0.5)
            elif "norm_q" in n or "norm_k" in n:
                p.normal_(1.0, 0.1)
            else:
                p.normal_(0, 0.02)
    if fmt is not None:
        apply_layerwise_casting(m, fmt, torch.bfloat16, CLI_SKIP)
    m.add_adapter(64, 64, target_modules=LORA_FFN_TARGETS if ffn else None)
    if policy is not None:
        apply_activation_checkpointing(m, *policy)
    m.prepare()
    with torch.no_grad():
        m.lora_flat.normal_(0, 0.02)   # non-zero B: every adapter gradient is non-trivial
    return m


def _batches(cfg, n, grid=GRID, seed=1234):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        lat = torch.randn(1, cfg.in_channels, *grid, generator=g).bfloat16().cuda()
        ehs = (torch.randn(1, L, cfg.caption_channels, generator=g) * 0.1).bfloat16().cuda()
        mask = (torch.arange(L)[None] < 100).float().cuda()
        out.append(({"encoder_hidden_states": ehs, "encoder_attention_mask": mask},
                    {"latents": lat, "latents_mean": torch.zeros(1, cfg.in_channels, device="cuda"),
                     "latents_std": torch.ones(1, cfg.in_channels, device="cuda")}))
    return out


def _train(cfg, policy, graph=True, ffn=False, fmt=None, steps=3, accum=2, grid=GRID):
    """-> (record, max_memory_allocated) of `steps` optimizer steps from one seeded state."""
    from finetrainers_b200.trainer import SFTTrainStep
    _free()
    torch.cuda.reset_peak_memory_stats()
    m = _build(cfg, policy, ffn, fmt)
    st = SFTTrainStep(m, flow_weighting_scheme="logit_normal", lr=1e-3, seed=42, use_cuda_graph=graph,
                      gradient_accumulation_steps=accum)
    rec = {"pred": [], "metrics": []}
    for i, (cond, lat) in enumerate(_batches(cfg, steps * accum)):
        st.spec.first_frame_conditioning_p = 1.0 if i == 3 else 0.0   # first-frame conditioning on one micro-step
        st.micro_step(cond, lat)
        rec["pred"].append(next(iter(m._ws.values()))["pred"].clone())
        if st.micro % accum == 0:
            st.optimizer_step()
            rec["metrics"].append(st.metrics.clone())
        else:
            st.clip_accumulated()
    torch.cuda.synchronize()
    rec["lora"] = m.lora_flat.clone()
    rec["plan"] = m.workspace_bytes(1, grid[0] * grid[1] * grid[2], L)
    peak = torch.cuda.max_memory_allocated()
    # to the host: a record left on the device would count in the next run's peak
    rec = {k: ([t.cpu() for t in v] if isinstance(v, list) else v.cpu() if torch.is_tensor(v) else v)
           for k, v in rec.items()}
    del st, m
    _free()
    return rec, peak


def _assert_same(a, b, what):
    assert len(a["metrics"]) == len(b["metrics"]) and len(a["pred"]) == len(b["pred"])
    for i, (x, y) in enumerate(zip(a["metrics"], b["metrics"])):
        assert torch.isfinite(x).all(), (what, i, x)
        assert torch.equal(x, y), (what, "step", i, x.tolist(), y.tolist())
    for i, (x, y) in enumerate(zip(a["pred"], b["pred"])):
        assert torch.equal(x, y), (what, "prediction of micro-step", i)
    assert torch.equal(a["lora"], b["lora"]), (what, "LoRA flat", (a["lora"] - b["lora"]).abs().max().item())


def _cfg(case):
    from finetrainers_b200.model import LTXConfig
    if case == "13b":
        cfg = LTXConfig.ltx_13b()
        cfg.num_layers = 2
        return cfg
    return LTXConfig(num_layers=4)


CASES = {  # name: (config, CUDA graph, feed-forward adapters, layerwise storage)
    "attn": ("2b", True, False, None),
    "ffn": ("2b", True, True, None),
    "e4m3fn": ("2b", True, False, torch.float8_e4m3fn),
    "13b": ("13b", True, False, None),
    "eager": ("2b", False, False, None),
}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", list(CASES))
def test_checkpointed_training_is_bit_identical_and_saves_the_planned_memory(case):
    name, graph, ffn, fmt = CASES[case]
    cfg = _cfg(name)
    keep, peak_keep = _train(cfg, None, graph, ffn, fmt)
    assert keep["lora"].abs().max().item() > 0
    for policy in (("full",), ("block_skip", 2)):
        got, peak = _train(cfg, policy, graph, ffn, fmt)
        _assert_same(keep, got, (case, policy))
        planned = keep["plan"] - got["plan"]
        # one scratch slot replaces the checkpointed blocks' slots: block_skip 2 over 2 blocks saves nothing
        assert planned > 0 if cfg.num_layers > 2 or policy == ("full",) else planned == 0
        assert peak_keep - peak >= 0.8 * planned, (case, policy, peak_keep - peak, planned)


@pytest.mark.timeout(600)
def test_block_range_backward_matches_keep_all():
    """Six blocks with feed-forward adapters and e4m3fn storage, backward in the DDP segments' three block ranges (top
    first, each range filling its own layerwise slots): the flat gradient of every policy equals keep-all's one
    whole backward bit for bit, and each range's slice is final when its _backward_tail returns."""
    from finetrainers_b200.model import LTXConfig
    from finetrainers_b200.trainer import SFTTrainStep
    cfg = LTXConfig(num_layers=6)
    (cond, lat), = _batches(cfg, 1)
    whole = None
    for policy in (None, ("full",), ("block_skip", 3)):
        _free()
        m = _build(cfg, policy, ffn=True, fmt=torch.float8_e4m3fn)
        st = SFTTrainStep(m, flow_weighting_scheme="none", seed=5)
        st.spec.first_frame_conditioning_p = 0.0
        st.micro_step(cond, lat)
        torch.cuda.synchronize()
        if whole is None:
            whole = m.lora_grad_flat.clone()
            assert whole.abs().max().item() > 0
        assert torch.equal(m.lora_grad_flat, whole), policy
        m.lora_grad_flat.zero_()
        (key, sbuf), = st._static.items()
        st._body_front(key, sbuf)
        pb = m._per_blk
        for lo, hi in [(4, 6), (2, 4), (0, 2)]:
            m._backward_blocks(hi - 1, lo)
            m._backward_tail(lo, hi)
            torch.cuda.synchronize()
            assert torch.equal(m.lora_grad_flat[lo * pb:hi * pb], whole[lo * pb:hi * pb]), (policy, lo, hi)
        assert torch.equal(m.lora_grad_flat, whole), policy
        del st, m


@pytest.mark.timeout(1200)
def test_13b_trains_a_6144_token_clip_on_one_card():
    """121 frames at 768x512: 16 x 16 x 24 latent tokens, r = 64, every block checkpointed.  Keep-all is not run at this
    shape: its workspace plan alone is stated (it does not fit beside the 26 GB of bf16 weights on an 80 GB card)."""
    from finetrainers_b200.model import LTXConfig
    cfg = LTXConfig.ltx_13b()
    grid = (16, 16, 24)
    runs = []
    for _ in range(2):
        rec, peak = _train(cfg, ("full",), True, steps=3, accum=1, grid=grid)
        runs.append((rec, peak))
    (a, pa), (b, pb) = runs
    for x in a["metrics"]:
        assert torch.isfinite(x).all(), x
    _assert_same(a, b, "13b 6144 tokens, repeated")
    assert max(pa, pb) < 50e9, (pa, pb)
    print(f"13B at 6144 tokens, full: peak {max(pa, pb) / 1e9:.1f} GB, workspace plan {a['plan'] / 1e9:.1f} GB")


_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["B2D_ROOT"]); sys.path.insert(0, os.path.join(os.environ["B2D_ROOT"], "tests"))
from finetrainers_b200.model import apply_activation_checkpointing
from finetrainers_b200.parallel import B200ParallelBackend
from finetrainers_b200.trainer import SFTTrainStep
from _util import build_pair, SMALL
mode, ckpt = sys.argv[1], sys.argv[2] == "full"
be = B200ParallelBackend(backend="nccl", **({"dp_shards": 2} if mode == "fsdp" else {}))
r = be.rank
O, om, bm = build_pair(dict(SMALL, num_layers=4), 64, seed=3, device=f"cuda:{be.local_rank}")
if ckpt:
    apply_activation_checkpointing(bm, "full")
if mode == "fsdp":
    be.apply_fsdp2(bm, param_dtype=torch.bfloat16, reduce_dtype=torch.float32, output_dtype=None, pp_enabled=False,
                   cpu_offload=False, device_mesh=be.get_mesh()[("dp_shard_cp",)])
else:
    be.apply_ddp(bm, be.get_mesh())
st = SFTTrainStep(bm, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=(mode == "ddp_graph"), ddp_chunks=2)
st.spec.first_frame_conditioning_p = 0.0
losses = []
for i in range(6 if mode == "ddp_graph" else 4):
    batch = O.make_synthetic_batch(om.cfg, 2, 2, 4, 9, text_len=24, seed=900 + 10 * i + r, text_scale=1.0)
    dev = f"cuda:{be.local_rank}"
    cond = {"encoder_hidden_states": batch["encoder_hidden_states"].to(dev), "encoder_attention_mask": batch["encoder_attention_mask"].to(dev)}
    lat = {"latents": batch["latents"].to(dev), "latents_mean": batch["latents_mean"].to(dev), "latents_std": batch["latents_std"].to(dev)}
    m = st.train_step(cond, lat, sigmas=batch["sigmas"].view(-1).to(dev), noise=batch["noise"].to(dev), sync_metrics=True)
    losses.append((m["train/global_avg_loss"], m["train/grad_norm"]))
torch.cuda.synchronize()
if r == 0:
    torch.save({"losses": losses, "lora": bm.lora_flat.cpu()}, os.environ["B2D_OUT"] + f".{mode}.{sys.argv[2]}")
be.wait_for_everyone()
be.destroy()
print("MULTI_OK", mode, r)
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.timeout(900)
def test_two_ranks_checkpointed_match_keep_all(tmp_path):
    """DDP block-range segment graphs and eager FSDP-2, each with every block checkpointed against the same mode
    keeping all activations: bit for bit."""
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    out = str(tmp_path / "res")
    env = dict(os.environ, B2D_ROOT=ROOT, B2D_OUT=out, MASTER_ADDR="127.0.0.1", NCCL_DEBUG="WARN")
    port = 29571
    for mode in ("ddp_graph", "fsdp"):
        for ck in ("keep", "full"):
            r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                                "--master-addr", "127.0.0.1", "--master-port", str(port), str(script), mode, ck],
                               env=env, capture_output=True, text=True, timeout=280)
            port += 1
            assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
            assert r.stdout.count("MULTI_OK") == 2
        a, b = torch.load(f"{out}.{mode}.keep"), torch.load(f"{out}.{mode}.full")
        assert a["losses"] == b["losses"], mode
        assert torch.equal(a["lora"], b["lora"]), mode
