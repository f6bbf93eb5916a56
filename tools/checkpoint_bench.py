"""Activation checkpointing: step time and peak memory per policy, on one GPU.

    python tools/checkpoint_bench.py --out DIR [--rounds 3] [--steps 10] [--warmup 3] [--parts 2b,13b,13b_long]

B = 1, LoRA r = 64 on the attention projections, CUDA-graph training step, 128 text tokens.  Writes
DIR/checkpoint.json and prints the tables; every table carries the card name, enforced power limit and max SM clock read
through NVML (queries only).  There is no CPU path: without a CUDA device the script fails.

  2b        the default geometry at 2688 tokens (49x512x768): keep-all, "full" and "block_skip" n_layer = 2, each first
            alone for its peak memory, then all three resident and alternated round by round.
  13b       the 13B geometry at 2688 tokens: keep-all and "full", one model at a time (rounds back to back).
  13b_long  the 13B geometry at 6144 tokens (121x512x768): "full" alone; keep-all's workspace plan is stated, not run.

Beside each measurement: the workspace plan's bytes, and for "full" / block_skip the recompute's share of the step's
GEMM FLOPs (``recompute_flops``), the estimate the measured time ratio is read against.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

RANK, L = 64, 128
GRID_2688, GRID_6144 = (7, 16, 24), (16, 16, 24)
POLICIES = {"keep-all": None, "full": ("full",), "block_skip2": ("block_skip", 2)}


def gemm_flops_per_token(cfg, rank=RANK):
    """(forward GEMM FLOPs per latent token of one block, the part a recomputed block runs again): QKV, out, cross q,
    cross out, FFN up and down with the attention-set LoRA down/up products; the recompute skips FFN down.  The
    training step is counted as forward + 2 x forward (dX and, for the adapters only, dW)."""
    d, f, r = cfg.inner_dim, cfg.ffn_mult * cfg.inner_dim, rank
    qkv = 2 * d * 3 * d + 2 * d * 3 * r + 2 * 3 * r * d
    o = q2 = o2 = 2 * d * d + 2 * d * r + 2 * r * d
    up, down = 2 * d * f, 2 * f * d
    fwd = qkv + o + q2 + o2 + up + down
    return fwd, fwd - down


def recompute_share(cfg, n_ckpt):
    """recompute FLOPs over the keep-all step's GEMM FLOPs (3 x forward), counting the checkpointed blocks only"""
    fwd, rec = gemm_flops_per_token(cfg)
    return n_ckpt * rec / (cfg.num_layers * 3 * fwd)


def run(cfg, policy, grid, warmup):
    import torch
    from finetrainers_b200.model import B200LTXTransformer, apply_activation_checkpointing
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
    if policy is not None:
        apply_activation_checkpointing(m, *policy)
    m.prepare()
    st = SFTTrainStep(m, flow_weighting_scheme="logit_normal", seed=42, use_cuda_graph=True)
    g = torch.Generator().manual_seed(1234)
    lat = torch.randn(1, cfg.in_channels, *grid, generator=g).bfloat16().cuda()
    ehs = (torch.randn(1, L, cfg.caption_channels, generator=g) * 0.1).bfloat16().cuda()
    mask = (torch.arange(L)[None] < 100).cuda()
    mean, std = torch.zeros(1, cfg.in_channels, device="cuda"), torch.ones(1, cfg.in_channels, device="cuda")

    def step():
        st.train_step({"encoder_hidden_states": ehs, "encoder_attention_mask": mask},
                      {"latents": lat, "latents_mean": mean, "latents_std": std})
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    loss = st.metrics[1].item()
    if not loss == loss or abs(loss) == float("inf"):
        raise SystemExit(f"non-finite loss {loss} after warm-up")
    S = grid[0] * grid[1] * grid[2]
    info = {"workspace_plan_gb": m.workspace_bytes(1, S, L) / 1e9,
            "keep_all_plan_gb": m.workspace_bytes(1, S, L, ()) / 1e9,
            "checkpointed_blocks": len(m._ckpt), "loss_after_warmup": loss}
    if m._ckpt:
        info["recompute_flops"] = recompute_share(cfg, len(m._ckpt))
    return m, st, step, info


def _free():
    import gc
    import torch
    gc.collect()
    torch.cuda.empty_cache()


def alone(cfg, policy, grid, args, timed_rounds):
    """build, warm up, peak memory; with timed_rounds, time them back to back"""
    import torch
    from ltx13b_bench import timed
    _free()
    torch.cuda.reset_peak_memory_stats()
    m, st, step, info = run(cfg, policy, grid, args.warmup)
    info["max_allocated_gb"] = torch.cuda.max_memory_allocated() / 1e9
    if timed_rounds:
        r = [timed(step, args.steps) for _ in range(args.rounds)]
        info.update(ms_per_step_median=statistics.median(r), rounds=r, schedule="alone on the card, rounds back to back")
    del m, st, step
    _free()
    return info


def table(title, res, info):
    from ltx13b_bench import card_line
    print(f"\n{title} {card_line(info)}")
    print(f"{'policy':<12} {'ms/step':>9} {'x keep-all':>10} {'recompute':>9} {'max alloc GB':>12} {'plan GB':>8}  rounds")
    base = res.get("keep-all", {}).get("ms_per_step_median")
    for k, r in res.items():
        ms = r.get("ms_per_step_median")
        print(f"{k:<12} {ms if ms else float('nan'):>9.2f} {(ms / base) if (ms and base) else float('nan'):>10.3f} "
              f"{r.get('recompute_flops', 0.0):>9.3f} {r['max_allocated_gb']:>12.2f} {r['workspace_plan_gb']:>8.2f}  "
              + " ".join(f"{x:.2f}" for x in r.get("rounds", [])))


def part_2b(args, info):
    from ltx13b_bench import timed
    from finetrainers_b200.model import LTXConfig
    cfg = LTXConfig()
    res = {k: alone(cfg, p, GRID_2688, args, False) for k, p in POLICIES.items()}
    arms = {k: run(cfg, p, GRID_2688, args.warmup) for k, p in POLICIES.items()}
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, (_, _, step, _) in arms.items():
            times[k].append(timed(step, args.steps))
    for k, v in times.items():
        res[k].update(ms_per_step_median=statistics.median(v), rounds=v,
                      schedule="all three models resident, alternated round by round")
    del arms
    _free()
    table(f"2B, B = 1, 2688 tokens, r = {RANK}, CUDA-graph step, {args.rounds} x {args.steps} steps", res, info)
    return res


def part_13b(args, info):
    from finetrainers_b200.model import LTXConfig
    cfg = LTXConfig.ltx_13b()
    res = {k: alone(cfg, POLICIES[k], GRID_2688, args, True) for k in ("keep-all", "full")}
    table(f"13B, B = 1, 2688 tokens, r = {RANK}, CUDA-graph step, {args.rounds} x {args.steps} steps", res, info)
    return res


def part_13b_long(args, info):
    from finetrainers_b200.model import LTXConfig
    cfg = LTXConfig.ltx_13b()
    res = {"full": alone(cfg, ("full",), GRID_6144, args, True)}
    table(f"13B, B = 1, 6144 tokens, r = {RANK}, CUDA-graph step, {args.rounds} x {args.steps} steps (keep-all: plan "
          f"{res['full']['keep_all_plan_gb']:.1f} GB of workspace, not run)", res, info)
    return res


PARTS = {"2b": part_2b, "13b": part_13b, "13b_long": part_13b_long}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="output directory (checkpoint.json is written there)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--parts", default="2b,13b,13b_long", help="comma list of " + ",".join(PARTS))
    args = ap.parse_args(argv)
    parts = args.parts.split(",")
    for p in parts:
        if p not in PARTS:
            ap.error(f"unknown part {p!r}")
    from ltx13b_bench import card
    info = card()
    os.makedirs(args.out, exist_ok=True)
    out = dict(info, text_tokens=L, rank=RANK)
    for p in parts:
        out[p] = PARTS[p](args, info)
        with open(os.path.join(args.out, "checkpoint.json"), "w") as fh:   # after every part: a later failure keeps it
            json.dump(out, fh, indent=1)
    print(json.dumps({"wrote": os.path.join(args.out, "checkpoint.json")}))


if __name__ == "__main__":
    main()
