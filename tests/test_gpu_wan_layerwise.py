"""GPU: layerwise fp8 weight storage for Wan-2.1 text- and image-to-video.

- The upcast is exact, so an fp8-stored Wan model computes bit for bit what its bf16 twin computes after every cast
  linear was rounded through fp8: loss, prediction, every LoRA gradient and the LoRA masters after each of 4 optimizer
  steps, with ``torch.equal``.  T2V at head_dim 64 and 128 and I2V, e4m3fn and e5m2, eager and CUDA graphs, keep-all /
  "full" / "block_skip", and a skip list that makes both stacked K/V stream in two chunks each.  The same identity for
  graph-replayed gradient accumulation, for interleaved buckets on a NaN-filled arena, for the no-grad inference
  forward and for ``load_state_dict`` into a captured model.
- I2V at the 14B width, 2 blocks, e4m3fn, against the fp32 oracle whose cast linears were rounded through fp8, at the
  bars of tests/test_gpu_wan_i2v.py.
- T2V-14B, all 40 blocks, 81 x 480 x 832, "full": one step is finite and its peak memory is the arithmetic's.
- DDP on two GPUs: segment graphs bit-identical to the bf16 twin's.
"""
import copy
import math
import os
import subprocess
import sys

import pytest
import torch

import _wan_i2v_oracle as I
import test_gpu_wan as TW
import test_gpu_wan_i2v as TI
from oracle import wan_oracle as O
from test_host_wan_layerwise import CLI_DEFAULT, DATACLASS_DEFAULT, diffusers_cast

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4, E5 = torch.float8_e4m3fn, torch.float8_e5m2
MULTI = CLI_DEFAULT + ["ffn"]   # a block slot holds 6 d^2: five blocks' stacked K/V stream in two chunks each


def _cfg(i2v, hd, nl):
    from finetrainers_b200.wan import WanConfig
    heads = 256 // hd
    kw = dict(in_channels=36, image_dim=128, added_kv_proj_dim=256) if i2v else {}
    return WanConfig(num_attention_heads=heads, attention_head_dim=hd, ffn_dim=512, num_layers=nl, **kw)


def _pair(i2v, fmt, pats, hd=64, nl=3, ckpt=None, r=16):
    """(fp8-stored model, bf16 model with the cast linears pre-rounded through fp8), same adapters."""
    from finetrainers_b200.model import apply_activation_checkpointing
    from finetrainers_b200.wan import B200WanTransformer
    torch.manual_seed(0)
    a = B200WanTransformer(_cfg(i2v, hd, nl), torch.bfloat16, "cuda")
    with torch.no_grad():
        for n, p in a.named_parameters():
            p.normal_(1.0, 0.1) if "norm" in n and n.endswith("weight") else p.normal_(0, 0.05)
    b = copy.deepcopy(a)
    a.enable_layerwise_casting(fmt, skip_modules_pattern=pats)
    mods = dict(b.named_modules())
    with torch.no_grad():
        for n in a._lw_cfg["cast"]:
            for p in (mods[n].weight, mods[n].bias):
                p.copy_(p.to(fmt).to(torch.bfloat16))
    for m in (a, b):
        m.add_adapter(r, r)
        if ckpt:
            apply_activation_checkpointing(m, *ckpt)
        m.prepare()
        m.skip_block0_dx = False
    with torch.no_grad():
        a.lora_flat.normal_(0, 0.05)   # non-zero B: every adapter gradient is non-trivial
        b.lora_flat.copy_(a.lora_flat)
    assert a._lw is not None and b._lw is None
    return a, b


def _bt(i2v, seed, F=2, H=8, W=12):
    return TI._batch(F=F, H=H, W=W, seed=seed) if i2v else TW._batch(F=F, H=H, W=W, seed=seed)


def _micro(i2v, st, bt):
    return TI._micro(st, bt) if i2v else TW._micro(st, bt)


def _assert_same_micro(sa, sb, what):
    torch.cuda.synchronize()
    a, b = sa.transformer, sb.transformer
    assert torch.isfinite(sa.loss_buf).all(), what
    assert torch.equal(sa.loss_buf, sb.loss_buf), (what, sa.loss_buf.item(), sb.loss_buf.item())
    key = a._saved_key[:3] + (a._saved_key[8],)
    assert torch.equal(a._workspace(*key)["pred"], b._workspace(*key)["pred"]), what
    assert a.lora_grad_flat.abs().max().item() > 0, what
    assert torch.equal(a.lora_grad_flat, b.lora_grad_flat), what


def _trainers(a, b, graph, accum=1):
    from finetrainers_b200.trainer import SFTTrainStep
    return (SFTTrainStep(m, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=graph,
                         gradient_accumulation_steps=accum) for m in (a, b))


CASES = {  # id: (i2v, head_dim, storage, CUDA graph, checkpointing, skip list)
    "t2v64-e4m3fn-eager-keep": (False, 64, E4, False, None, CLI_DEFAULT),
    "t2v128-e5m2-graph-full": (False, 128, E5, True, ("full",), CLI_DEFAULT),
    "t2v64-e4m3fn-graph-blockskip-2chunks": (False, 64, E4, True, ("block_skip", 2), MULTI),
    "i2v64-e4m3fn-graph-keep-dataclass": (True, 64, E4, True, None, DATACLASS_DEFAULT),
    "i2v64-e5m2-eager-full-2chunks": (True, 64, E5, False, ("full",), MULTI),
    "i2v128-e4m3fn-graph-blockskip-2chunks": (True, 128, E4, True, ("block_skip", 2), MULTI),
}


@pytest.mark.parametrize("case", list(CASES))
def test_fp8_wan_is_bit_identical_to_prerounded_bf16(case):
    i2v, hd, fmt, graph, ckpt, pats = CASES[case]
    nl = 5 if pats is MULTI else 3
    a, b = _pair(i2v, fmt, pats, hd=hd, nl=nl, ckpt=ckpt)
    if pats is MULTI:
        assert len(a._lw.kv2_chunks) == 2 and len(a._lw.chunks("kv3")) == (2 if i2v else 0)
    sa, sb = _trainers(a, b, graph)
    for i in range(4):        # graph mode: 2 eager warm-ups, capture, replay
        bt = _bt(i2v, 10 + i)
        for s in (sa, sb):
            _micro(i2v, s, bt)
        _assert_same_micro(sa, sb, (case, i))
        sa.optimizer_step()
        sb.optimizer_step()
        torch.cuda.synchronize()
        assert torch.equal(a.lora_flat, b.lora_flat), (case, i)
    if graph:
        assert len(sa._graphs) == 1
    assert a.blocks[1].attn1.to_q.base_layer.weight.dtype == fmt
    if i2v:
        assert a.blocks[1].attn2.add_k_proj.weight.dtype == fmt


def test_graph_replayed_gradient_accumulation_is_bit_identical():
    a, b = _pair(True, E4, MULTI, nl=5)
    sa, sb = _trainers(a, b, True, accum=2)
    for i in range(6):        # 3 optimizer steps
        bt = _bt(True, 20 + i)
        lat = TI._lat(bt)
        for s in (sa, sb):
            s.train_step({"encoder_hidden_states": bt["ehs"].cuda()}, dict(lat), sigmas=bt["sigmas"].cuda(),
                         noise=bt["noise"].cuda(), posterior_noise=bt["eps"].cuda())
        torch.cuda.synchronize()
        assert torch.equal(sa.loss_buf, sb.loss_buf), i
        assert torch.equal(a.lora_flat, b.lora_flat), i
    assert sa.opt_step == 3 and len(sa._graphs) == 1


@pytest.mark.parametrize("i2v", [False, True], ids=["t2v", "i2v"])
def test_interleaved_buckets_on_a_poisoned_arena_are_bit_identical(i2v):
    """Three resolutions in one shared arena, NaN-filled before every step, under CUDA graphs."""
    a, b = _pair(i2v, E4, MULTI, nl=5)
    sa, sb = _trainers(a, b, True)
    grids = [(2, 8, 12), (1, 8, 8), (3, 4, 8)]           # 48, 16 and 24 latent tokens
    a._workspace(1, 48, 512, 257 if i2v else 0)   # the largest bucket first: the arena holds every one
    for i, (F, H, W) in enumerate(grids * 4):
        bt = _bt(i2v, 30 + i, F, H, W)
        a._arena.fill_(0xFF)   # NaN in every bf16 and fp32 view
        for s in (sa, sb):
            _micro(i2v, s, bt)
        _assert_same_micro(sa, sb, (i, F, H, W))
        sa.optimizer_step()
        sb.optimizer_step()
        torch.cuda.synchronize()
        assert torch.equal(a.lora_flat, b.lora_flat), i
    assert len(sa._graphs) == 3


@pytest.mark.parametrize("i2v", [False, True], ids=["t2v", "i2v"])
def test_no_grad_inference_forward_is_bit_identical(i2v):
    a, b = _pair(i2v, E5, MULTI, nl=5)
    bt = _bt(i2v, 40)
    torch.manual_seed(1)
    x = torch.randn(1, 36 if i2v else 16, 2, 8, 12, device="cuda").to(torch.bfloat16)
    t = torch.full((1,), 700, device="cuda")
    kw = dict(encoder_hidden_states_image=bt["img"].cuda()) if i2v else {}
    with torch.no_grad():
        pa = a(x, t, bt["ehs"].cuda(), **kw)[0].clone()
        pb = b(x, t, bt["ehs"].cuda(), **kw)[0].clone()
    TI._same(pa, pb, "inference prediction")
    assert torch.isfinite(pa.float()).all()


def test_load_state_dict_after_capture_takes_effect():
    """New base weights of one block and of its image-side K/V, loaded into a captured I2V model, are what the next
    replay computes with: every forward upcasts from storage, the streamed chunks included."""
    a, b = _pair(True, E4, MULTI, nl=5)
    sa, sb = _trainers(a, b, True)

    def step(i):
        bt = _bt(True, 50 + i)
        for s in (sa, sb):
            _micro(True, s, bt)
        _assert_same_micro(sa, sb, i)
        sa.optimizer_step()
        sb.optimizer_step()

    for i in range(3):
        step(i)
    assert len(sa._graphs) == 1
    torch.manual_seed(9)
    sd_a, sd_b = a.state_dict(), b.state_dict()
    new_a, new_b = {}, {}
    for n, v in sd_a.items():
        if "lora_" in n or not n.startswith("blocks.4."):
            continue
        w = (torch.randn(v.shape, device="cuda") * 0.05).to(torch.bfloat16)
        if v.dtype in (E4, E5):
            w = w.to(v.dtype)
        new_a[n], new_b[n] = w, w.to(sd_b[n].dtype)
    assert "blocks.4.attn2.add_v_proj.weight" in new_a and new_a["blocks.4.attn2.add_v_proj.weight"].dtype == E4
    a.load_state_dict(new_a, strict=False)
    b.load_state_dict(new_b, strict=False)
    step(3)
    step(4)
    assert len(sa._graphs) == 1


# ---- against the oracle at the 14B width ----------------------------------------------------------------------------
@pytest.mark.timeout(1200)
def test_i2v_14b_width_two_blocks_fp8_vs_oracle():
    from finetrainers_b200.wan import B200WanTransformer, WanConfig
    c = WanConfig.wan_i2v_14b()
    geom = dict(num_attention_heads=c.num_attention_heads, attention_head_dim=c.attention_head_dim, ffn_dim=c.ffn_dim)
    ocfg = lambda: I.WanI2VOracleConfig(image_dim=c.image_dim, num_layers=2, **geom)  # noqa: E731
    om = I.WanI2VTransformerOracle(ocfg())
    O.add_lora(om, 32, 32)
    O.synthetic_init_(om, seed=0)
    with torch.no_grad():
        for n, p in om.named_parameters():
            if "lora_" not in n:
                p.copy_(p.to(torch.bfloat16).float())
    # the rule runs before add_adapter in the reference: evaluate it on the adapter-free tree, round om's base layers
    names = diffusers_cast(I.WanI2VTransformerOracle(ocfg()), CLI_DEFAULT)
    mods = dict(om.named_modules())
    with torch.no_grad():
        for n in names:
            lin = getattr(mods[n], "base_layer", mods[n])
            for p in (lin.weight, lin.bias):
                p.copy_(p.to(E4).float())
    d = c.inner_dim
    bm = B200WanTransformer(WanConfig(num_layers=2, in_channels=36, image_dim=c.image_dim, added_kv_proj_dim=d, **geom),
                            torch.bfloat16, "cuda")
    bm.enable_layerwise_casting(E4, skip_modules_pattern=CLI_DEFAULT)
    assert sorted(bm._lw_cfg["cast"]) == names
    bm.add_adapter(32, 32)
    bm.load_state_dict(om.state_dict(), strict=True)   # fp8-exact values: the fp8 copy is lossless
    bm.prepare()
    bm.skip_block0_dx = False
    assert bm.blocks[1].attn2.add_k_proj.weight.dtype == E4 and "Wkv3_all" not in bm._root_views
    TI._compare(om, bm, TI._batch(F=2, H=30, W=52, image_dim=c.image_dim), "Wan I2V 14B width, 2 blocks, e4m3fn")


# ---- full size --------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(1800)
def test_t2v_14b_81_frames_full_checkpointing_fits_with_fp8_storage():
    """T2V-14B, 40 blocks, 81 x 480 x 832 (21 x 60 x 104 latents, 32 760 tokens), B = 1, r = 32, "full", e4m3fn under
    the CLI list.  The step's peak allocation is the base weights + the workspace + the LoRA state (fp32 master and
    gradient, bf16 operand copy, two AdamW moments) within 1.5 GiB, and under 80 GB."""
    import gc
    from finetrainers_b200.model import apply_activation_checkpointing
    from finetrainers_b200.trainer import SFTTrainStep
    from finetrainers_b200.wan import B200WanTransformer, WanConfig
    gc.collect()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    m = B200WanTransformer(WanConfig.wan_14b(), torch.bfloat16, "cuda")
    with torch.no_grad():
        for n, p in m.named_parameters():
            p.fill_(1.0) if "norm" in n and n.endswith("weight") else p.normal_(0, 0.02)
    m.enable_layerwise_casting(E4, skip_modules_pattern=CLI_DEFAULT)
    m.add_adapter(32, 32)
    apply_activation_checkpointing(m, "full")
    m.prepare()
    st = SFTTrainStep(m, flow_weighting_scheme="logit_normal")
    Fl, Hl, Wl = 21, 60, 104
    S = Fl * (Hl // 2) * (Wl // 2)
    g = torch.Generator(device="cuda").manual_seed(0)
    lat = {"latents": torch.randn(1, 32, Fl, Hl, Wl, device="cuda", generator=g).to(torch.bfloat16),
           "latents_mean": torch.zeros(1, 16, device="cuda"), "latents_std": torch.ones(1, 16, device="cuda")}
    cond = {"encoder_hidden_states": torch.randn(1, 512, 4096, device="cuda", generator=g).to(torch.bfloat16)}
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    st.train_step(cond, lat)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    loss = float(st.loss_buf)
    bw = m.base_weight_bytes()
    ws = m.workspace_bytes(1, S, 512)
    lora = m.lora_flat.numel() * (4 + 4 + 2 + 8)
    want = sum(bw.values()) + ws + lora
    print(f"\nT2V-14B 81x480x832 full e4m3fn: peak {peak / 2**30:.2f} GiB; base weights {sum(bw.values()) / 2**30:.2f} "
          f"GiB {bw}, workspace {ws / 2**30:.2f} GiB, LoRA state {lora / 2**30:.2f} GiB, sum {want / 2**30:.2f} GiB; "
          f"loss {loss}")
    assert math.isfinite(loss)
    assert peak < 80e9
    assert want <= peak <= want + 1.5 * 2**30, (peak, want)


# ---- DDP, 2 GPUs ------------------------------------------------------------------------------------------------------
_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["B2D_ROOT"]); sys.path.insert(0, os.path.join(os.environ["B2D_ROOT"], "tests"))
from finetrainers_b200.parallel import B200ParallelBackend
import test_gpu_wan_layerwise as T
be = B200ParallelBackend(backend="nccl")
r = be.rank
torch.cuda.set_device(be.local_rank)
a, b = T._pair(True, torch.float8_e4m3fn, T.MULTI, nl=5)
for m in (a, b):
    be.apply_ddp(m, be.get_mesh())
from finetrainers_b200.trainer import SFTTrainStep
sa, sb = (SFTTrainStep(m, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=True, ddp_chunks=2) for m in (a, b))
assert len(sa._segments) == 2
for i in range(5):
    bt = T._bt(True, 10 * i + r)                                  # rank-specific data
    lat = T.TI._lat(bt)
    kw = dict(sigmas=bt["sigmas"].cuda(), noise=bt["noise"].cuda(), posterior_noise=bt["eps"].cuda(), sync_metrics=True)
    ma = sa.train_step({"encoder_hidden_states": bt["ehs"].cuda()}, dict(lat), **kw)
    mb = sb.train_step({"encoder_hidden_states": bt["ehs"].cuda()}, dict(lat), **kw)
    assert ma == mb, (i, ma, mb)
torch.cuda.synchronize()
assert torch.equal(a.lora_flat, b.lora_flat)
other = [torch.empty_like(a.lora_flat) for _ in range(2)]
dist.all_gather(other, a.lora_flat)
assert torch.equal(other[0], other[1]), "ranks diverged"
be.wait_for_everyone()
be.destroy()
print("WAN_LW_DDP_OK", r)
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.timeout(600)
def test_ddp_graph_segments_are_bit_identical_on_two_gpus(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    env = dict(os.environ, B2D_ROOT=ROOT, MASTER_ADDR="127.0.0.1", NCCL_DEBUG="WARN")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29573", str(script)], env=env,
                       capture_output=True, text=True, timeout=500)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert r.stdout.count("WAN_LW_DDP_OK") == 2
