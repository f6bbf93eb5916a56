"""GPU: multi-resolution training in one shared training arena.  A model that trains interleaved resolution buckets
reuses one arena for every bucket's workspace, so a step starts on another bucket's bytes: here the whole arena is
filled with NaN before every step, and every micro-step's loss, prediction and flat gradient, every optimizer step's
gradient norm and the whole fp32 LoRA flat after AdamW must equal those of a model that only ever trained that step's
bucket, from the same state and inputs, bit for bit.  Growth under CUDA graphs re-captures every graph, the peak of an
interleaved run is the largest bucket's, and the 13B model trains three buckets on one card."""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu
CLI_SKIP = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]
L = 128
# latent grids: 49x512x768 (2688 tokens), 49x480x704 (2310), one 512x768 image (384), 25x512x768 (1536)
G2688, G2310, G384, G1536 = (7, 16, 24), (7, 15, 22), (1, 16, 24), (4, 16, 24)


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _build(cfg, policy=None, ffn=False, fmt=None, seed=0):
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


def _trainer(m, graph, accum):
    from finetrainers_b200.trainer import SFTTrainStep
    st = SFTTrainStep(m, flow_weighting_scheme="logit_normal", lr=1e-3, seed=42, use_cuda_graph=graph,
                      gradient_accumulation_steps=accum)
    st.spec.first_frame_conditioning_p = 0.0
    return st


def _inputs(cfg, grid, i, moments=False):
    """Micro-step i's inputs at one latent grid, drawn on the host from seed i: conditions, latents (VAE moments with
    ``moments``) and the explicit sigmas, noise and posterior noise, so that no generator state is involved."""
    g = torch.Generator().manual_seed(1000 + i)
    C = cfg.in_channels
    lat = torch.randn(1, 2 * C if moments else C, *grid, generator=g)
    if moments:
        lat[:, C:] = lat[:, C:] * 0.5 - 2.0   # log-variances
    ehs = torch.randn(1, L, cfg.caption_channels, generator=g) * 0.1
    mask = (torch.arange(L)[None] < 100).float()
    kw = dict(sigmas=torch.rand(1, generator=g).cuda(), noise=torch.randn(1, C, *grid, generator=g).bfloat16().cuda())
    if moments:
        kw.update(compute_posterior=False, posterior_noise=torch.randn(1, C, *grid, generator=g).bfloat16().cuda())
    cond = {"encoder_hidden_states": ehs.bfloat16().cuda(), "encoder_attention_mask": mask.cuda()}
    latc = {"latents": lat.bfloat16().cuda(), "latents_mean": torch.zeros(1, C, device="cuda"),
            "latents_std": torch.ones(1, C, device="cuda")}
    return cond, latc, kw


def _state_from(dst, src):
    """Give trainer ``dst`` (and its model) the optimizer-visible state of ``src``: LoRA masters, accumulated gradient,
    AdamW moments, step counters and the accumulated loss."""
    for a, b in ((dst.transformer.lora_flat, src.transformer.lora_flat),
                 (dst.transformer.lora_grad_flat, src.transformer.lora_grad_flat), (dst.exp_avg, src.exp_avg),
                 (dst.exp_avg_sq, src.exp_avg_sq), (dst.loss_acc, src.loss_acc)):
        a.copy_(b)
    dst.opt_step, dst.micro = src.opt_step, src.micro


def _pred(m, grid):
    return m._workspace(1, grid[0] * grid[1] * grid[2], L)["pred"]


def _finish(st):
    """Optimizer step at the end of an accumulation window, else the reference's clip after the micro-step."""
    if st.micro % st.grad_accum == 0:
        st.optimizer_step()
        return True
    st.clip_accumulated()
    return False


def _cfg(name):
    from finetrainers_b200.model import LTXConfig
    if name == "13b":
        cfg = LTXConfig.ltx_13b()
        cfg.num_layers = 2
        return cfg
    return LTXConfig(num_layers=3)


POISON = {  # name: (config, CUDA graph, checkpointing, FFN adapters, layerwise storage, moments input, accumulation)
    "keep_all": ("2b", True, None, False, None, False, 1),
    "eager": ("2b", False, None, False, None, False, 1),
    "full": ("2b", True, ("full",), False, None, False, 1),
    "full_eager": ("2b", False, ("full",), False, None, False, 1),
    "block_skip2": ("2b", True, ("block_skip", 2), False, None, False, 1),
    "ffn": ("2b", True, None, True, None, False, 1),
    "e4m3fn": ("2b", True, None, False, torch.float8_e4m3fn, False, 1),
    "moments": ("2b", True, None, False, None, True, 1),
    "accum2": ("2b", True, None, False, None, False, 2),
    "13b": ("13b", True, None, False, None, False, 1),
}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", list(POISON))
def test_poisoned_arena_trains_each_bucket_like_a_single_bucket_model(case):
    name, graph, policy, ffn, fmt, moments, accum = POISON[case]
    cfg = _cfg(name)
    _free()
    grids = [G2688, G2310, G384]
    m = _build(cfg, policy, ffn, fmt)
    st = _trainer(m, graph, accum)
    refs = {}
    for grid in grids:   # one model per bucket that never sees another shape
        rm = _build(cfg, policy, ffn, fmt)
        refs[grid] = _trainer(rm, graph, accum)
    order = grids * 4    # each bucket: two eager warm-ups, then capture and replay under CUDA graphs
    m._workspace(1, 2688, L)   # the arena exists before the first step, so that step starts on poison too
    for i, grid in enumerate(order):
        ref = refs[grid]
        _state_from(ref, st)
        cond, lat, kw = _inputs(cfg, grid, i, moments)
        m._arena.fill_(0xFF)   # NaN in every bf16 and fp32 view
        st.micro_step(cond, lat, **kw)
        ref.micro_step(cond, lat, **kw)
        torch.cuda.synchronize()
        what = (case, i, grid)
        assert torch.isfinite(st.loss_buf).all(), what
        assert torch.equal(st.loss_buf, ref.loss_buf), (what, "loss")
        assert torch.equal(_pred(m, grid), _pred(ref.transformer, grid)), (what, "pred")
        assert torch.equal(m.lora_grad_flat, ref.transformer.lora_grad_flat), (what, "gradient")
        if _finish(st):
            assert _finish(ref)
            torch.cuda.synchronize()
            assert torch.isfinite(st.metrics).all(), what
            assert torch.equal(st.metrics, ref.metrics), (what, st.metrics.tolist(), ref.metrics.tolist())
            assert torch.equal(m.lora_flat, ref.transformer.lora_flat), (what, "LoRA flat")
        else:
            assert not _finish(ref)
    assert m.workspace_generation == 1   # largest bucket first: the arena never grew
    if graph:
        assert len(st._graphs) == len(grids)
    del st, m, refs
    _free()


def _run(cfg, graph, order, policy=None):
    """-> (per step (metrics, pred) on the host, final LoRA flat, trainer) of one model over ``order``."""
    m = _build(cfg, policy)
    st = _trainer(m, graph, 1)
    out = []
    for i, grid in enumerate(order):
        cond, lat, kw = _inputs(cfg, grid, i)
        st.micro_step(cond, lat, **kw)
        st.optimizer_step()
        out.append((st.metrics.cpu(), _pred(m, grid).cpu()))
    torch.cuda.synchronize()
    return out, m.lora_flat.cpu(), st


@pytest.mark.timeout(600)
def test_growth_recaptures_every_graph_and_matches_eager():
    """small -> large -> small: the large bucket grows the arena, so the small bucket's graph (captured over the old
    arena) is dropped and re-captured; every step equals the eager run's."""
    cfg = _cfg("2b")
    order = [G384] * 3 + [G2688] * 3 + [G384] * 3
    _free()
    eager, eager_lora, _ = _run(cfg, False, order)
    m = _build(cfg)
    st = _trainer(m, True, 1)
    got, small_graph = [], None
    for i, grid in enumerate(order):
        cond, lat, kw = _inputs(cfg, grid, i)
        st.micro_step(cond, lat, **kw)
        st.optimizer_step()
        got.append((st.metrics.cpu(), _pred(m, grid).cpu()))
        if i == 2:
            (gkey, small_graph), = st._graphs.items()
            assert m.workspace_generation == 1
    torch.cuda.synchronize()
    assert m.workspace_generation == 2 and st._graph_gen == 2
    assert st._graphs[gkey] is not small_graph, "the small bucket replayed a graph of the old arena"
    assert len(st._graphs) == 2
    for i, ((a, pa), (b, pb)) in enumerate(zip(got, eager)):
        assert torch.isfinite(a).all(), (i, a)
        assert torch.equal(a, b), (i, a.tolist(), b.tolist())
        assert torch.equal(pa, pb), ("pred", i)
    assert torch.equal(m.lora_flat.cpu(), eager_lora)
    del st, m, small_graph
    _free()


def _static_bytes(cfg, grid):
    """Device bytes a shape adds besides its workspace: the trainer's static input buffers and the RoPE tables, each
    allocation rounded up to the caching allocator's 512 bytes (plus the key bias the model keeps for backward)."""
    B, C, S = 1, cfg.in_channels, grid[0] * grid[1] * grid[2]
    r = lambda n: -(-n // 512) * 512  # noqa: E731
    static = [2 * B * C * S] * 2 + [4 * B * C] * 2 + [2 * B * L * cfg.caption_channels, 4 * B * L] + [4 * B] * 2
    static += [2 * B * S * C] * 3
    rope = [4 * S * cfg.inner_dim // 2] * 2
    return sum(r(n) for n in static + rope + [4 * B * L])


def _peak(cfg, order):
    _free()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m = _build(cfg)
    st = _trainer(m, True, 1)
    for i, grid in enumerate(order):
        cond, lat, kw = _inputs(cfg, grid, i)
        st.micro_step(cond, lat, **kw)
        st.optimizer_step()
        del cond, lat, kw
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    arena = m._arena.numel()
    del st, m
    _free()
    return peak, arena


@pytest.mark.timeout(600)
def test_interleaved_peak_is_the_largest_bucket_peak():
    cfg = _cfg("2b")
    buckets = [G2310, G2688, G384]   # a smaller bucket first: the run also grows the arena once
    single, arena1 = _peak(cfg, [G2688] * 4)
    multi, arena3 = _peak(cfg, buckets * 4)
    extra = sum(_static_bytes(cfg, g) for g in buckets if g != G2688)
    # the caching allocator hands out a cached block whole when splitting it would leave less than 1 MiB, so each of the
    # smaller buckets' allocations may count up to that much more than its size: 2 MiB per bucket covers it (one
    # bucket's workspace, what a per-shape workspace would add, is hundreds of MB here)
    slack = 2 * 2 ** 20 * (len(buckets) - 1)
    assert arena3 == arena1
    print(f"\nsingle bucket peak {single / 1e9:.3f} GB, three interleaved {multi / 1e9:.3f} GB, "
          f"per-shape extra {extra / 1e6:.1f} MB")
    assert multi <= single + extra + slack, (multi, single, extra)


@pytest.mark.timeout(1500)
def test_13b_trains_three_buckets_in_one_arena():
    """The 13B model keeping all activations over 2688-, 2310- and 1536-token buckets, interleaved, two CUDA-graph
    steps per bucket after two eager warm-ups: finite and repeatable bit for bit."""
    from finetrainers_b200.model import LTXConfig
    cfg = LTXConfig.ltx_13b()
    buckets = [G2688, G2310, G1536]
    runs = []
    for _ in range(2):
        _free()
        torch.cuda.reset_peak_memory_stats()
        out, lora, st = _run(cfg, True, buckets * 4)
        m = st.transformer
        plans = [m.arena_layout(m.workspace_plan(1, g[0] * g[1] * g[2], L))[1] for g in buckets]
        arena = m._arena.numel()
        del st, m
        _free()
        runs.append((out, lora, torch.cuda.max_memory_allocated(), arena, plans))
    (a, la, pa, arena, plans), (b, lb, pb, _, _) = runs
    for i, ((x, px), (y, py)) in enumerate(zip(a, b)):
        assert torch.isfinite(x).all(), (i, x)
        assert torch.equal(x, y) and torch.equal(px, py), i
    assert torch.equal(la, lb)
    assert arena == max(plans)
    print(f"\n13B keep-all, 3 buckets interleaved: peak {max(pa, pb) / 1e9:.1f} GB, arena {arena / 1e9:.2f} GB "
          f"(per-bucket workspaces {', '.join(f'{p / 1e9:.2f}' for p in plans)} GB, sum {sum(plans) / 1e9:.1f} GB)")
