"""GPU: layerwise fp8 weight storage.  The upcast kernel is exact, so an fp8-stored model must compute bit for bit what
the bf16 model computes after every cast linear's weight and bias were replaced by ``w.to(fp8).to(bf16)``: pred, loss
and every LoRA gradient are compared with ``torch.equal``, eager and under CUDA graphs, through the autograd path, with
gradient accumulation, after ``load_state_dict`` into a captured model and after ``.to(dtype=bf16)``.  Five blocks, so
that both block slots are refilled in the forward and in the backward."""
import copy
import math
import os
import subprocess
import sys

import pytest
import torch

from _util import SMALL, rel_err, sentinel_buffer, check_sentinel, window

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CLI_DEFAULT = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]
DATACLASS_DEFAULT = CLI_DEFAULT[:4] + ["time_embed"] + CLI_DEFAULT[4:]
FMTS = [torch.float8_e4m3fn, torch.float8_e5m2]
NL = 5


# ---- the kernel -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS, ids=["e4m3fn", "e5m2"])
def test_upcast_every_code_matches_torch(fmt):
    from finetrainers_b200 import ops
    src = torch.arange(256, dtype=torch.uint8, device="cuda").view(fmt)
    dst = torch.empty(256, dtype=torch.bfloat16, device="cuda")
    ops.upcast_fp8_bf16(src, dst, 256)
    ref = src.to(torch.bfloat16)
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(dst), nan)
    assert int(nan.sum()) == (2 if fmt == torch.float8_e4m3fn else 6)
    # every other code bit-exact: +-0, subnormals, the largest finite values, and +-Inf for e5m2
    assert torch.equal(dst.view(torch.int16)[~nan], ref.view(torch.int16)[~nan])


@pytest.mark.parametrize("n", [1, 15, 16, 17, 4095, 14 * 2048 * 2048 + 11 * 2048])
def test_upcast_ragged_lengths_stay_in_bounds(n):
    from finetrainers_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(n)
    codes = torch.randint(0, 256, (n + 16,), dtype=torch.uint8, device="cuda", generator=g)
    src = codes[16:].view(torch.float8_e4m3fn)           # 16-byte aligned start, NaN codes included
    buf = sentinel_buffer(n + 64, torch.bfloat16)
    dst = buf[16:16 + n]
    ops.upcast_fp8_bf16(src, dst, n)
    ref = src.to(torch.bfloat16)
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(dst), nan)
    assert torch.equal(dst.view(torch.int16)[~nan], ref.view(torch.int16)[~nan])
    check_sentinel(buf, [window(buf, 16, 1, n, n)], f"upcast n={n}")


def test_upcast_refuses_misaligned_pointers():
    from finetrainers_b200 import ops, lib
    src = torch.zeros(64, dtype=torch.uint8, device="cuda").view(torch.float8_e4m3fn)
    dst = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    for s, d in ((src[1:], dst), (src, dst[1:]), (src[8:], dst)):
        with pytest.raises(lib.B2DError, match="code -2"):
            ops.upcast_fp8_bf16(s, d, 16)
    ops.upcast_fp8_bf16(src, dst, 0)       # n <= 0: no-op
    torch.cuda.synchronize()
    assert dst.abs().sum().item() == 0


# ---- model bit identity -----------------------------------------------------------------------------------------------
def _pair(fmt, patterns, nl=NL, rank=64):
    """(fp8-stored model, bf16 model with the cast linears pre-rounded through fp8), same adapters."""
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig, apply_layerwise_casting
    cfg = LTXConfig(**dict(SMALL, num_layers=nl))
    torch.manual_seed(0)
    a = B200LTXTransformer(cfg, torch.bfloat16, "cuda")
    with torch.no_grad():
        for n, p in a.named_parameters():
            p.normal_(0, 0.05) if "norm_" not in n else p.normal_(1.0, 0.1)
    b = copy.deepcopy(a)
    apply_layerwise_casting(a, fmt, torch.bfloat16, patterns)
    mods = dict(b.named_modules())
    with torch.no_grad():
        for n in a._lw_cfg["cast"]:
            for p in (mods[n].weight, mods[n].bias):
                p.copy_(p.to(fmt).to(torch.bfloat16))
    for m in (a, b):
        m.add_adapter(rank, rank)
        m.prepare()
    with torch.no_grad():
        a.lora_flat.normal_(0, 0.05)   # non-zero B: every adapter gradient is non-trivial
        b.lora_flat.copy_(a.lora_flat)
    assert a._lw is not None and b._lw is None
    return a, b


def _batch(i, B=2):
    from oracle import ltx_oracle as O
    batch = O.make_synthetic_batch(O.LTXConfig(**dict(SMALL, num_layers=NL)), B, 2, 4, 9, text_len=24, seed=100 + i,
                                   text_scale=1.0)
    cond = {"encoder_hidden_states": batch["encoder_hidden_states"].cuda(),
            "encoder_attention_mask": batch["encoder_attention_mask"].cuda()}
    lat = {"latents": batch["latents"].cuda(), "latents_mean": batch["latents_mean"].cuda(),
           "latents_std": batch["latents_std"].cuda()}
    return cond, lat, batch["sigmas"].view(-1).cuda(), batch["noise"].cuda()


def _assert_same_micro(sa, sb, what):
    torch.cuda.synchronize()
    a, b = sa.transformer, sb.transformer
    assert torch.equal(sa.loss_buf, sb.loss_buf), (what, sa.loss_buf.item(), sb.loss_buf.item())
    wa, wb = next(iter(a._ws.values())), next(iter(b._ws.values()))
    assert torch.equal(wa["pred"], wb["pred"]), what
    assert a.lora_grad_flat.abs().max().item() > 0, what
    assert torch.equal(a.lora_grad_flat, b.lora_grad_flat), what


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("fmt", FMTS, ids=["e4m3fn", "e5m2"])
@pytest.mark.parametrize("patterns", ["cli", "dataclass+ff"])
def test_fp8_model_is_bit_identical_to_prerounded_bf16(patterns, fmt, graph):
    """'dataclass+ff': time_embed and the FFN stay bf16, so one block slot holds only 6 d^2 weights and the text-side
    [Wk2;Wv2] of the five blocks streams through the two slots in two chunks."""
    from finetrainers_b200.trainer import SFTTrainStep
    pats = CLI_DEFAULT if patterns == "cli" else DATACLASS_DEFAULT + ["ff"]
    a, b = _pair(fmt, pats)
    assert len(a._lw.kv2_chunks) == (1 if patterns == "cli" else 2)
    sa, sb = (SFTTrainStep(m, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=graph) for m in (a, b))
    for s in (sa, sb):
        s.spec.first_frame_conditioning_p = 0.0
    for i in range(4):        # graph mode: 2 eager warm-ups, capture, replay
        cond, lat, sig, noise = _batch(i)
        for s in (sa, sb):
            s.micro_step(dict(cond), dict(lat), sigmas=sig, noise=noise)
        _assert_same_micro(sa, sb, f"micro {i}")
        sa.optimizer_step()
        sb.optimizer_step()
        torch.cuda.synchronize()
        assert torch.equal(a.lora_flat, b.lora_flat), i
    if graph:
        assert len(sa._graphs) == 1
    # the stored state is fp8 and unchanged by training
    assert a.transformer_blocks[3].ff.net[2].weight.dtype == (fmt if patterns == "cli" else torch.bfloat16)
    assert a.transformer_blocks[3].attn1.to_q.base_layer.weight.dtype == fmt


def test_gradient_accumulation_under_graphs_is_bit_identical():
    from finetrainers_b200.trainer import SFTTrainStep
    a, b = _pair(torch.float8_e4m3fn, CLI_DEFAULT)
    sa, sb = (SFTTrainStep(m, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=True,
                           gradient_accumulation_steps=2) for m in (a, b))
    for s in (sa, sb):
        s.spec.first_frame_conditioning_p = 0.0
    for i in range(6):        # 3 optimizer steps
        cond, lat, sig, noise = _batch(i)
        for s in (sa, sb):
            s.train_step(dict(cond), dict(lat), sigmas=sig, noise=noise)
        torch.cuda.synchronize()
        assert torch.equal(sa.loss_buf, sb.loss_buf), i
        assert torch.equal(a.lora_flat, b.lora_flat), i
    assert sa.opt_step == 3


def test_load_state_dict_after_capture_and_to_bf16_take_effect():
    """New base weights loaded into a captured model are what the next replay computes with (every forward upcasts from
    storage), and ``.to(dtype=bf16)`` keeps the fp8 storage and its values."""
    from finetrainers_b200.trainer import SFTTrainStep
    a, b = _pair(torch.float8_e4m3fn, CLI_DEFAULT)
    sa, sb = (SFTTrainStep(m, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=True) for m in (a, b))
    for s in (sa, sb):
        s.spec.first_frame_conditioning_p = 0.0

    def step(i):
        cond, lat, sig, noise = _batch(i)
        for s in (sa, sb):
            s.micro_step(dict(cond), dict(lat), sigmas=sig, noise=noise)
        _assert_same_micro(sa, sb, f"micro {i}")
        sa.optimizer_step()
        sb.optimizer_step()

    for i in range(3):
        step(i)
    assert len(sa._graphs) == 1
    # new base weights: fp8 values for the fp8 model, the same values in bf16 for the other
    torch.manual_seed(9)
    sd_a, sd_b = a.state_dict(), b.state_dict()
    new_a, new_b = {}, {}
    for n, v in sd_a.items():
        if "lora_" in n or not n.startswith("transformer_blocks.2."):
            continue
        w = (torch.randn(v.shape, device="cuda") * 0.05).to(torch.bfloat16)
        if v.dtype in FMTS:
            w = w.to(v.dtype)
        new_a[n], new_b[n] = w, w.to(sd_b[n].dtype)
    a.load_state_dict(new_a, strict=False)
    b.load_state_dict(new_b, strict=False)
    step(3)
    step(4)
    # .to(dtype=bf16) after enabling: fp8 storage, same values, same results (the model is re-packed)
    fp8_before = {n: p.detach().clone() for n, p in a.named_parameters() if p.dtype in FMTS}
    a.to(dtype=torch.bfloat16)
    b.to(dtype=torch.bfloat16)
    for n, p in a.named_parameters():
        if n in fp8_before:
            assert p.dtype == fp8_before[n].dtype and torch.equal(p.view(torch.uint8), fp8_before[n].view(torch.uint8)), n
    sa._graphs.clear(); sa._eager_runs.clear(); sb._graphs.clear(); sb._eager_runs.clear()
    for i in range(5, 8):
        step(i)


def test_autograd_path_is_bit_identical():
    """forward() + loss.backward(), the path finetrainers' own trainer takes."""
    a, b = _pair(torch.float8_e5m2, CLI_DEFAULT)
    torch.manual_seed(3)
    B, Fr, H, W, L = 1, 2, 4, 8, 16
    hs = torch.randn(B, Fr * H * W, SMALL["in_channels"], device="cuda").to(torch.bfloat16)
    ehs = torch.randn(B, L, SMALL["caption_channels"], device="cuda").to(torch.bfloat16)
    t = torch.full((B,), 500.0, device="cuda")
    mask = torch.ones(B, L, device="cuda")
    mask[:, 12:] = 0
    out = []
    for m in (a, b):
        pred = m(hs, ehs, t, mask, Fr, H, W)[0]
        loss = (pred.float() - 0.5).pow(2).mean()
        loss.backward()
        torch.cuda.synchronize()
        out.append((pred.detach().clone(), loss.detach().clone(), m.lora_grad_flat.clone()))
    (pa, la, ga), (pb, lb, gb) = out
    assert torch.equal(pa, pb) and torch.equal(la, lb) and torch.equal(ga, gb)
    assert ga.abs().max().item() > 0


# ---- against the oracle at full width --------------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_full_width_two_block_forward_backward_matches_oracle_with_fp8_storage():
    """D = 2048, S = 2688, L = 128, r = 64, two blocks, e4m3fn storage under the CLI default list: the engine against the
    fp32 oracle whose cast linears were rounded through fp8 by the restated rule, at the bf16 model's tolerances."""
    from oracle import ltx_oracle as O
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig, apply_layerwise_casting
    from _util import run_b200_micro
    from test_host_layerwise import oracle_layerwise_cast
    cfgk = dict(num_layers=2)
    om = O.LTXTransformerOracle(O.LTXConfig(**cfgk))
    O.add_lora(om, 64, 64)
    O.synthetic_init_(om, seed=0, lora_b_std=0.02)
    with torch.no_grad():
        for n, p in om.named_parameters():
            if "lora_" not in n:
                p.copy_(p.to(torch.bfloat16).float())
    # the rule runs before add_adapter in the reference: evaluate it on the adapter-free tree, round om's base layers
    names = oracle_layerwise_cast(O.LTXTransformerOracle(O.LTXConfig(**cfgk)), CLI_DEFAULT)
    mods = dict(om.named_modules())
    with torch.no_grad():
        for n in names:
            lin = getattr(mods[n], "base_layer", mods[n])
            for p in (lin.weight, lin.bias):
                p.copy_(p.to(torch.float8_e4m3fn).float())
    bm = B200LTXTransformer(LTXConfig(**cfgk), torch.bfloat16, "cuda")
    apply_layerwise_casting(bm, torch.float8_e4m3fn, torch.bfloat16, CLI_DEFAULT)
    assert sorted(bm._lw_cfg["cast"]) == sorted(names)
    bm.add_adapter(64, 64)
    bm.load_state_dict(om.state_dict(), strict=True)   # fp8-exact values: the fp8 copy is lossless
    bm.prepare()
    batch = O.make_synthetic_batch(om.cfg, 1, 7, 16, 24, seed=1234, text_scale=1.0)
    loss_o, pred_o = O.oracle_step(om, {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()})
    st, loss_b, pred_b = run_b200_micro(bm, batch)
    assert abs(loss_b - loss_o.item()) / abs(loss_o.item()) < 1e-3
    assert rel_err(pred_b, pred_o) < 3e-2
    og = dict(om.named_parameters())
    n_ad = 0
    for n, p in bm.named_parameters():
        if "lora_" in n:
            go = og[n].grad
            e = (p.grad.float().cpu() - go).abs().max().item() / go.abs().max().item()
            assert e < 5e-2, (n, e)
            n_ad += 1
    assert n_ad == 2 * 16


@pytest.mark.timeout(600)
def test_full_size_memory_matches_the_arithmetic():
    """LTX-2B, r = 64, e4m3fn under the CLI default list: device memory after prepare() is the sum of the fp8 storage,
    the bf16 weights that stay bf16, two block slots, the root slot and the LoRA buffers, within 1 %."""
    import gc
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig, apply_layerwise_casting
    gc.collect()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    m = B200LTXTransformer(LTXConfig(), torch.bfloat16, "cuda")
    apply_layerwise_casting(m, torch.float8_e4m3fn, torch.bfloat16, CLI_DEFAULT)
    m.add_adapter(64, 64)
    m.prepare()
    gc.collect()
    torch.cuda.synchronize()
    got = torch.cuda.memory_allocated() - base
    d, f, nl, cap, cin = 2048, 8192, 28, 4096, 128
    blk_cast = 3 * d * d + 3 * d + 3 * (d * d + d) + f * d + f + d * f + d
    root_cast = 256 * d + d + d * d + d + 6 * d * d + 6 * d + cap * d + d + d * d + d
    kv2 = nl * (2 * d * d + 2 * d)
    keep = nl * 9 * d + d * cin + d + 2 * d + cin * d + cin + nl * d
    want = (nl * blk_cast + root_cast + kv2) + 2 * keep + 2 * 2 * blk_cast + 2 * root_cast + nl * 2 * 8 * 64 * d * 10
    print(f"memory after prepare: {got / 1e9:.3f} GB, arithmetic {want / 1e9:.3f} GB; "
          f"base weights {m.base_weight_bytes()}")
    assert abs(got - want) <= 0.01 * want, (got, want)


# ---- DDP, 2 GPUs ------------------------------------------------------------------------------------------------------
_WORKER = r'''
import os, sys, copy, torch, torch.distributed as dist
sys.path.insert(0, os.environ["B2D_ROOT"]); sys.path.insert(0, os.path.join(os.environ["B2D_ROOT"], "tests"))
from finetrainers_b200.parallel import B200ParallelBackend
from finetrainers_b200.trainer import SFTTrainStep
import test_gpu_layerwise as T
be = B200ParallelBackend(backend="nccl")
r = be.rank
torch.cuda.set_device(be.local_rank)
a, b = T._pair(torch.float8_e4m3fn, T.CLI_DEFAULT)
for m in (a, b):
    be.apply_ddp(m, be.get_mesh())
sa, sb = (SFTTrainStep(m, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=True, ddp_chunks=2) for m in (a, b))
assert len(sa._segments) == 2
for s in (sa, sb):
    s.spec.first_frame_conditioning_p = 0.0
for i in range(5):
    cond, lat, sig, noise = T._batch(10 * i + r)                  # rank-specific data
    ma = sa.train_step(dict(cond), dict(lat), sigmas=sig, noise=noise, sync_metrics=True)
    mb = sb.train_step(dict(cond), dict(lat), sigmas=sig, noise=noise, sync_metrics=True)
    assert ma == mb, (i, ma, mb)
torch.cuda.synchronize()
assert torch.equal(a.lora_flat, b.lora_flat)
other = [torch.empty_like(a.lora_flat) for _ in range(2)]
dist.all_gather(other, a.lora_flat)
assert torch.equal(other[0], other[1]), "ranks diverged"
be.wait_for_everyone()
be.destroy()
print("LW_DDP_OK", r)
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.timeout(600)
def test_ddp_graph_segments_are_bit_identical_on_two_gpus(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    env = dict(os.environ, B2D_ROOT=ROOT, MASTER_ADDR="127.0.0.1", NCCL_DEBUG="WARN")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29571", str(script)], env=env,
                       capture_output=True, text=True, timeout=500)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert r.stdout.count("LW_DDP_OK") == 2
