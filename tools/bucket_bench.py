"""Multi-resolution training: per-bucket step time and peak memory of CUDA-graph steps interleaved over several
resolution buckets, against each bucket trained alone, on one GPU.

    python tools/bucket_bench.py --out DIR [--model 2b|13b] [--buckets 2688,2310,1536,384] [--steps 5] [--warmup 3]

B = 1, LoRA r = 64 on the attention projections, keep-all activations, 128 text tokens, one optimizer step per
micro-step.  Buckets are latent token counts: 2688 (49x512x768), 2310 (49x480x704), 1536 (25x512x768) and 384 (one
512x768 image).  The interleaved arm runs ``warmup`` rounds (one step per bucket each; the first two of every bucket are
eager, then its graph is captured) and then ``steps`` timed rounds; every step is timed on its own with CUDA events
around it.  Each bucket alone: a fresh model, ``warmup`` steps, ``steps`` timed steps.  ``max_memory_allocated`` covers
each arm from the model's construction on; an arm that runs out of device memory is reported as such.  Writes
DIR/buckets_<model>.json and prints a table headed by the card name, its enforced power limit and the SM clock read
through NVML in the same run (queries only).  There is no CPU path: without a CUDA device the script fails.
"""
import argparse
import gc
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

RANK, L = 64, 128
GRIDS = {2688: (7, 16, 24), 2310: (7, 15, 22), 1536: (4, 16, 24), 384: (1, 16, 24)}


def _free():
    import torch
    gc.collect()
    torch.cuda.empty_cache()


def _model(cfg):
    import torch
    from finetrainers_b200.model import B200LTXTransformer
    from finetrainers_b200.trainer import SFTTrainStep
    torch.manual_seed(0)
    m = B200LTXTransformer(cfg, torch.bfloat16, "cuda")
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "scale_shift_table" in n:
                p.normal_(0, 1.0 / p.shape[-1] ** 0.5)
            elif "norm_q" in n or "norm_k" in n:
                p.fill_(1.0)
            else:
                p.normal_(0, 0.02)
    m.add_adapter(RANK, RANK)
    m.prepare()
    return m, SFTTrainStep(m, flow_weighting_scheme="logit_normal", seed=42, use_cuda_graph=True)


def _step_fn(cfg, st, tokens):
    """One training step at a bucket, on fixed seeded inputs -> () -> ms of that step (CUDA events around it)."""
    import torch
    g = torch.Generator().manual_seed(tokens)
    grid = GRIDS[tokens]
    lat = torch.randn(1, cfg.in_channels, *grid, generator=g).bfloat16().cuda()
    cond = {"encoder_hidden_states": (torch.randn(1, L, cfg.caption_channels, generator=g) * 0.1).bfloat16().cuda(),
            "encoder_attention_mask": (torch.arange(L)[None] < 100).cuda()}
    latc = {"latents": lat, "latents_mean": torch.zeros(1, cfg.in_channels, device="cuda"),
            "latents_std": torch.ones(1, cfg.in_channels, device="cuda")}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def step():
        e0.record()
        st.train_step(cond, latc)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)
    return step


def _arm(cfg, buckets, warmup, steps):
    """Steps over ``buckets`` in rounds (one step per bucket each) -> {ms per bucket, max allocated, losses} or
    {"oom": message}."""
    import torch
    _free()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m = st = None
    try:
        m, st = _model(cfg)
        fns = {t: _step_fn(cfg, st, t) for t in buckets}
        for _ in range(warmup):
            for t in buckets:
                fns[t]()
        times = {t: [] for t in buckets}
        for _ in range(steps):
            for t in buckets:
                times[t].append(fns[t]())
        loss = st.metrics[1].item()
        out = {"ms_per_step": {t: statistics.median(v) for t, v in times.items()},
               "ms_all": {t: v for t, v in times.items()},
               "max_allocated_gb": (torch.cuda.max_memory_allocated() - base) / 1e9,
               "workspace_plans_gb": {t: m.workspace_bytes(1, t, L) / 1e9 for t in buckets},
               "last_loss": loss}
        if not loss == loss or abs(loss) == float("inf"):
            raise SystemExit(f"non-finite loss {loss}")
    except torch.cuda.OutOfMemoryError as e:
        out = {"oom": str(e).split("\n")[0], "max_allocated_gb": (torch.cuda.max_memory_allocated() - base) / 1e9}
    del m, st
    _free()
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="output directory (buckets_<model>.json is written there)")
    ap.add_argument("--model", choices=("2b", "13b"), default="2b")
    ap.add_argument("--buckets", default="2688,2310,1536,384", help="comma list of " + ",".join(map(str, GRIDS)))
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args(argv)
    buckets = [int(b) for b in args.buckets.split(",")]
    for b in buckets:
        if b not in GRIDS:
            ap.error(f"unknown bucket {b}: one of {sorted(GRIDS)}")
    if args.warmup < 3:
        ap.error("--warmup must be at least 3: two eager steps and the capture per bucket")
    from ltx13b_bench import card, card_line
    from finetrainers_b200.model import LTXConfig
    info = card()
    cfg = LTXConfig.ltx_13b() if args.model == "13b" else LTXConfig()
    res = dict(info, model=args.model, text_tokens=L, rank=RANK, buckets=buckets, steps=args.steps, warmup=args.warmup)
    res["interleaved"] = _arm(cfg, buckets, args.warmup, args.steps)
    res["alone"] = {t: _arm(cfg, [t], args.warmup, args.steps) for t in buckets}
    try:
        import pynvml as nv
        h = nv.nvmlDeviceGetHandleByIndex(0)
        res["sm_mhz_after"] = nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)
    except Exception as e:  # noqa: BLE001
        res["sm_mhz_after"] = f"unavailable: {e!r}"
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, f"buckets_{args.model}.json")
    with open(path, "w") as fh:
        json.dump(res, fh, indent=1)
    it = res["interleaved"]
    print(f"\n{args.model}, B = 1, r = {RANK}, keep-all, CUDA-graph steps, median of {args.steps} "
          f"{card_line(info)}, SM clock after the timed work {res['sm_mhz_after']} MHz")
    print(f"{'bucket':>7} {'interleaved ms':>15} {'alone ms':>9} {'ratio':>6} {'alone max alloc GB':>19}")
    for t in buckets:
        a = res["alone"][t]
        x, y = it.get("ms_per_step", {}).get(t), a.get("ms_per_step", {}).get(t)
        print(f"{t:>7} {x if x else float('nan'):>15.2f} {y if y else float('nan'):>9.2f} "
              f"{(x / y) if (x and y) else float('nan'):>6.3f} {a['max_allocated_gb']:>19.2f}{'  (oom)' if 'oom' in a else ''}")
    print(f"interleaved max allocated {it['max_allocated_gb']:.2f} GB{'  (oom: ' + it['oom'] + ')' if 'oom' in it else ''}")
    print(json.dumps({"wrote": path}))


if __name__ == "__main__":
    main()
