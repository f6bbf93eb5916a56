"""The 13B LTX-Video geometry (32 heads x 128, width 4096, 48 blocks) on one GPU, beside the 2B geometry in the same call.

    python tools/ltx13b_bench.py --out DIR [--rounds 3] [--steps 10] [--warmup 3] [--iters 30] [--parts step,gemm,attn,qk]

B = 1, 49x512x768 (2688 latent tokens, 128 text tokens), LoRA r = 64 on the attention projections.  Writes DIR/ltx13b.json
and prints the same tables; every table carries the card name, enforced power limit and max SM clock read through NVML
(queries only).  There is no CPU path: without a CUDA device the script fails.

  step  CUDA-graph training step, bf16 weights and layerwise e4m3fn storage (CLI skip list): median ms/step over
        --rounds rounds of --steps steps after --warmup steps, memory_allocated after prepare() and max_memory_allocated.
        The two 2B models are resident together and alternate round by round.  The two 13B models do not fit one 80 GB
        card together, so they are built and timed one after the other (rounds back to back, not alternated).
  gemm  the twelve step GEMMs at M = 2688, D = 4096 by tools/gemm_bench.py's method (CUDA events over --iters launches on
        rotated operand sets): the library's automatic tile choice, then block_n 64 / 128 x single CTA / CTA pair.
        TFLOP/s counts 2 M N (K + K2).
  attn  self- and cross-attention forward / backward at 32 x 128, S = 2688 (L = 128 keys for cross attention): TFLOP/s
        counts 4 Sq Sk d H forward and 2.5 x that backward.
  qk    the q/k-norm + RoPE + head-split launches of one block: bytes moved per token (segments in and out at 2 bytes, one
        (cos, sin) row of D / 2 fp32 pairs when a segment is rotated, the norm weights once) over time, against the
        3.35 TB/s data-sheet HBM bandwidth.
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

M, L, RANK = 2688, 128, 64
GRID = (7, 16, 24)                      # latent frames x height x width of 49x512x768
CLI_SKIP = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]
HBM_GBS = 3350.0


def attn_flops(H, Sq, Sk, d):
    """forward FLOPs of one attention call (QK^T and PV); the backward counts 2.5 x this"""
    return 4.0 * Sq * Sk * d * H


def qk_bytes(D, nseg, rope, n_norm):
    """bytes one token row moves through a q/k-norm + RoPE launch: nseg segments read and written as bf16, one table row
    (cos and sin, D / 2 fp32 each) when a segment is rotated; plus, once per launch, the norm weights (returned second)"""
    return 2 * nseg * D * 2 + (D * 4 if rope else 0), n_norm * D * 2


def card():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/ltx13b_bench.py measures on a CUDA device; none is visible")
    info = {"card": torch.cuda.get_device_name(0)}
    try:
        import pynvml as nv
        nv.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "").split(",")[0].strip()
        h = nv.nvmlDeviceGetHandleByIndex(int(vis) if vis.isdigit() else 0)
        info["power_limit_w"] = nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        info["max_sm_mhz"] = nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)
    except Exception as e:  # noqa: BLE001
        info["nvml"] = f"unavailable: {e!r}"
    return info


def card_line(info):
    return (f"[{info['card']}, power limit {info.get('power_limit_w', 'n/a')} W, max SM clock "
            f"{info.get('max_sm_mhz', 'n/a')} MHz]")


def build(cfg, fmt):
    import torch
    from finetrainers_b200.model import B200LTXTransformer, apply_layerwise_casting
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
    if fmt is not None:
        apply_layerwise_casting(m, fmt, torch.bfloat16, CLI_SKIP)
    m.add_adapter(RANK, RANK)
    m.prepare()
    after_prepare = torch.cuda.memory_allocated()
    st = SFTTrainStep(m, flow_weighting_scheme="logit_normal", seed=42, use_cuda_graph=True)
    g = torch.Generator().manual_seed(1234)
    lat = torch.randn(1, cfg.in_channels, *GRID, generator=g).bfloat16().cuda()
    ehs = (torch.randn(1, L, cfg.caption_channels, generator=g) * 0.1).bfloat16().cuda()
    mask = (torch.arange(L)[None] < 100).cuda()
    mean, std = torch.zeros(1, cfg.in_channels, device="cuda"), torch.ones(1, cfg.in_channels, device="cuda")

    def step():
        st.train_step({"encoder_hidden_states": ehs, "encoder_attention_mask": mask},
                      {"latents": lat, "latents_mean": mean, "latents_std": std})
    return m, st, step, after_prepare


def timed(step, n):
    import torch
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def part_step(args, info):
    import torch
    from finetrainers_b200.model import LTXConfig
    fp8 = torch.float8_e4m3fn
    res = {}

    def free():
        gc.collect()
        torch.cuda.empty_cache()

    def arm(cfg, fmt):
        free()
        torch.cuda.reset_peak_memory_stats()
        m, st, step, after = build(cfg, fmt)
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        loss = st.metrics[1].item()
        if not loss == loss or abs(loss) == float("inf"):
            raise SystemExit(f"non-finite loss {loss} after warm-up")
        return m, step, {"after_prepare_gb": after / 1e9, "max_allocated_gb": torch.cuda.max_memory_allocated() / 1e9,
                         "loss_after_warmup": loss}

    # 13B: one model at a time
    cfg = LTXConfig.ltx_13b()
    for name, fmt in (("bf16", None), ("e4m3fn", fp8)):
        m, step, mem = arm(cfg, fmt)
        rounds = [timed(step, args.steps) for _ in range(args.rounds)]
        res[f"13b_{name}"] = dict(mem, ms_per_step_median=statistics.median(rounds), rounds=rounds,
                                  schedule="alone on the card, rounds back to back")
        del m, step
    free()
    # 2B: each arm's memory alone, then both resident and alternated
    cfg = LTXConfig()
    for name, fmt in (("bf16", None), ("e4m3fn", fp8)):
        m, step, mem = arm(cfg, fmt)
        res[f"2b_{name}"] = mem
        del m, step
    free()
    arms = {"bf16": build(cfg, None)[2], "e4m3fn": build(cfg, fp8)[2]}
    for step in arms.values():
        for _ in range(args.warmup):
            step()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, step in arms.items():
            times[k].append(timed(step, args.steps))
    for k, v in times.items():
        res[f"2b_{k}"].update(ms_per_step_median=statistics.median(v), rounds=v,
                              schedule="both models resident, alternated round by round")
    del arms
    free()
    res["ratio_13b_over_2b_bf16"] = res["13b_bf16"]["ms_per_step_median"] / res["2b_bf16"]["ms_per_step_median"]
    res["ratio_13b_over_2b_e4m3fn"] = res["13b_e4m3fn"]["ms_per_step_median"] / res["2b_e4m3fn"]["ms_per_step_median"]
    print(f"\nstep time, B = 1, {M} tokens, r = {RANK}, CUDA-graph step, {args.rounds} x {args.steps} steps "
          f"{card_line(info)}")
    print(f"{'model':<12} {'ms/step':>9} {'after prepare GB':>17} {'max allocated GB':>17}  rounds")
    for k in ("13b_bf16", "13b_e4m3fn", "2b_bf16", "2b_e4m3fn"):
        r = res[k]
        print(f"{k:<12} {r['ms_per_step_median']:>9.2f} {r['after_prepare_gb']:>17.2f} {r['max_allocated_gb']:>17.2f}  "
              + " ".join(f"{x:.2f}" for x in r["rounds"]))
    print(f"13B / 2B: bf16 {res['ratio_13b_over_2b_bf16']:.2f}, e4m3fn {res['ratio_13b_over_2b_e4m3fn']:.2f}")
    return res


def part_gemm(args, info):
    import torch
    import gemm_bench as gb
    gb.set_width(4096)
    clock = gb.Clock()
    rows = []
    configs = [(0, 0)] + [(bn, cp) for bn in (64, 128) for cp in (1, 2)]
    print(f"\nstep GEMMs at M = {M}, D = 4096, K2 = LoRA extension {card_line(info)}")
    print(f"{'shape':<12} {'N':>6} {'K':>6} {'K2':>4} {'epi':<9} {'bn':>4} {'pair':>4} {'fused us':>9} {'TF/s':>6} {'store us':>9}")
    for (name, N, K, b_mn, epi, K2, gn) in gb.SHAPES:
        sets = gb.make_sets(N, K, b_mn, epi, K2, gn)
        flop = 2.0 * M * N * (K + K2)
        for bn, cp in configs:
            try:
                f = gb.time_ms(gb.launcher(sets, N, K, b_mn, epi, K2, gn, True, bn, cp), args.iters, clock)
                s = gb.time_ms(gb.launcher(sets, N, K, b_mn, epi, K2, gn, False, bn, cp), args.iters, clock)
            except Exception as e:  # noqa: BLE001  (a tile choice the library rejects for this shape)
                print(f"{name:<12} bn={bn} pair={cp}: {str(e).splitlines()[0]}")
                continue
            rows.append({"shape": name, "N": N, "K": K, "K2": K2, "epi": epi, "block_n": bn, "cta_pair": cp,
                         "fused_us": f * 1e3, "fused_tflops": flop / f / 1e9, "store_us": s * 1e3})
            print(f"{name:<12} {N:>6} {K:>6} {K2:>4} {epi:<9} {bn or 'auto':>4} {cp or 'auto':>4} {f * 1e3:>9.1f} "
                  f"{flop / f / 1e9:>6.0f} {s * 1e3:>9.1f}", flush=True)
        del sets
        torch.cuda.empty_cache()
    auto = sum(r["fused_us"] for r in rows if r["block_n"] == 0)
    print(f"sum over the twelve shapes, automatic choice: {auto / 1e3:.3f} ms; x 48 blocks {48 * auto / 1e3:.1f} ms")
    return {"rows": rows, "sum_auto_ms": auto / 1e3, "sm_mhz_median": clock.finish()}


def _events(fn, iters):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters          # us


def part_attn(args, info):
    import torch
    from finetrainers_b200 import ops
    H, d, rows = 32, 128, []
    print(f"\nattention at {H} x {d}, S = {M} {card_line(info)}")
    print(f"{'call':<8} {'Sk':>5} {'fwd us':>8} {'TF/s':>6} {'bwd us':>8} {'TF/s':>6}")
    for name, Sk in (("self", M), ("cross", L)):
        r = lambda *s: torch.randn(*s, device="cuda").bfloat16()  # noqa: E731
        q, k, v = r(1, H, M, d), r(1, H, Sk, d), r(1, H, Sk, d)
        out, dout = torch.empty(1, M, H * d, device="cuda", dtype=torch.bfloat16), r(1, M, H * d)
        lse = torch.empty(1, H, M, device="cuda", dtype=torch.float32)
        kb = None
        if name == "cross":
            kb = torch.zeros(1, Sk, device="cuda")
            kb[:, 100:] = -10000.0
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        ws = torch.empty(ops.attn_bwd_ws_floats(1, H, M, Sk, head_dim=d), device="cuda", dtype=torch.float32)
        scale = d ** -0.5
        tf = _events(lambda: ops.attn_fwd(q, k, v, kb, out, lse, 1, H, M, Sk, scale, head_dim=d), args.iters)
        tb = _events(lambda: ops.attn_bwd(q, k, v, kb, out, dout, lse, ws, dq, dk, dv, 1, H, M, Sk, scale, head_dim=d),
                     args.iters)
        fl = attn_flops(H, M, Sk, d)
        rows.append({"call": name, "Sk": Sk, "fwd_us": tf, "fwd_tflops": fl / tf / 1e6, "bwd_us": tb,
                     "bwd_tflops": 2.5 * fl / tb / 1e6})
        print(f"{name:<8} {Sk:>5} {tf:>8.1f} {fl / tf / 1e6:>6.0f} {tb:>8.1f} {2.5 * fl / tb / 1e6:>6.0f}")
    return {"rows": rows}


def part_qk(args, info):
    import torch
    from finetrainers_b200 import ops
    H, d, D, nl = 32, 128, 4096, 48
    r = lambda *s: torch.randn(*s, device="cuda").bfloat16()  # noqa: E731
    ang = torch.randn(M, D // 2, device="cuda")
    cos, sin = ang.cos(), ang.sin()
    w = [torch.ones(D, device="cuda", dtype=torch.bfloat16) for _ in range(2)]
    wk = torch.ones(nl, D, device="cuda", dtype=torch.bfloat16)
    qkv, dqkv = r(M, 3 * D), torch.empty(M, 3 * D, device="cuda", dtype=torch.bfloat16)
    hs = [r(1, H, M, d) for _ in range(3)]
    q2, dq2 = r(M, D), torch.empty(M, D, device="cuda", dtype=torch.bfloat16)
    kv2, dkv2 = r(nl * L, 2 * D), torch.empty(nl * L, 2 * D, device="cuda", dtype=torch.bfloat16)
    k2h = [r(nl, H, L, d) for _ in range(2)]
    eps = 1e-5
    # name, token rows, segments, rotated, normed segments, forward launch, backward launch
    calls = [
        ("self q|k|v", M, 3, True, 2,
         lambda: ops.qkv_norm_rope_fwd(qkv, 3 * D, 0, (w[0], w[1], None), 0b011, cos, sin, hs, 1, M, H, eps, head_dim=d),
         lambda: ops.qkv_norm_rope_bwd(hs, qkv, 3 * D, 0, (w[0], w[1], None), 0b011, cos, sin, dqkv, 3 * D, 0, 1, M, H,
                                       eps, head_dim=d)),
        ("cross q", M, 1, False, 1,
         lambda: ops.qknorm_rope_fwd(q2, D, 0, w[0], None, None, hs[0], 1, M, H, True, eps, head_dim=d),
         lambda: ops.qknorm_rope_bwd(hs[0], q2, D, 0, w[0], None, None, dq2, D, 0, 1, M, H, True, eps, head_dim=d)),
        ("text k|v x48", nl * L, 2, False, nl,
         lambda: ops.qkv_norm_rope_fwd(kv2, 2 * D, 0, (wk, None), 0, None, None, k2h, nl, L, H, eps, rows_per_w=L,
                                       w_stride=D, head_dim=d),
         lambda: ops.qkv_norm_rope_bwd(k2h, kv2, 2 * D, 0, (wk, None), 0, None, None, dkv2, 2 * D, 0, nl, L, H, eps,
                                       rows_per_w=L, w_stride=D, head_dim=d)),
    ]
    rows = []
    print(f"\nq/k-norm + RoPE + head split at {H} x {d} (D = {D}); bytes / time against {HBM_GBS / 1e3:.2f} TB/s "
          f"{card_line(info)}")
    print(f"{'launch':<14} {'rows':>6} {'MB':>7} {'fwd us':>8} {'GB/s':>6} {'of peak':>8} {'bwd us':>8} {'GB/s':>6} {'of peak':>8}")
    for name, n_rows, nseg, rope, n_norm, fwd, bwd in calls:
        per_row, once = qk_bytes(D, nseg, rope, n_norm)
        # the backward also reads the source segments it renormalises: one more bf16 read per normed segment
        b_f = n_rows * per_row + once
        b_b = b_f + n_rows * (2 if name.startswith("self") else 1) * D * 2
        tf, tb = _events(fwd, args.iters), _events(bwd, args.iters)
        rows.append({"launch": name, "rows": n_rows, "fwd_bytes": b_f, "bwd_bytes": b_b, "fwd_us": tf, "bwd_us": tb,
                     "fwd_gbs": b_f / tf / 1e3, "bwd_gbs": b_b / tb / 1e3})
        print(f"{name:<14} {n_rows:>6} {b_f / 1e6:>7.1f} {tf:>8.1f} {b_f / tf / 1e3:>6.0f} {b_f / tf / 1e3 / HBM_GBS:>8.2f} "
              f"{tb:>8.1f} {b_b / tb / 1e3:>6.0f} {b_b / tb / 1e3 / HBM_GBS:>8.2f}")
    return {"rows": rows, "hbm_peak_gbs": HBM_GBS}


PARTS = {"step": part_step, "gemm": part_gemm, "attn": part_attn, "qk": part_qk}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="output directory (ltx13b.json is written there)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=30, help="launches per isolated kernel timing")
    ap.add_argument("--parts", default="qk,attn,gemm,step", help="comma list of " + ",".join(PARTS))
    args = ap.parse_args(argv)
    parts = args.parts.split(",")
    for p in parts:
        if p not in PARTS:
            ap.error(f"unknown part {p!r}")
    info = card()
    os.makedirs(args.out, exist_ok=True)
    out = dict(info, tokens=M, text_tokens=L, rank=RANK)
    for p in parts:
        out[p] = PARTS[p](args, info)
        with open(os.path.join(args.out, "ltx13b.json"), "w") as fh:     # after every part: a later failure keeps it
            json.dump(out, fh, indent=1)
    print(json.dumps({"wrote": os.path.join(args.out, "ltx13b.json")}))


if __name__ == "__main__":
    main()
