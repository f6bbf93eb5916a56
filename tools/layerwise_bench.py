"""Layerwise fp8 weight storage at LTX-2B size: the bf16 model against fp8 storage, alternated in one session.

    python tools/layerwise_bench.py [--rounds 3] [--steps 10] [--warmup 3] [--fmt e4m3fn]

B = 1, 49x512x768 (2688 latent tokens), LoRA r = 64, CUDA-graph step, CLI default skip list.  Prints one JSON line:
median ms/step per arm (each round times both arms back to back), max_memory_allocated of each arm built alone, the
base-weight bytes, the upcast kernel on one block's fp8 flat (CUDA events, mean of --launches launches) against the
3.35 TB/s data-sheet HBM bandwidth, and the card name, enforced power limit and median SM clock (NVML)."""
import argparse
import gc
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import ClockSampler, F_LAT, H_LAT, W_LAT, TEXT_LEN, RANK_LORA  # noqa: E402

CLI_SKIP = ["patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$", "norm"]
HBM_GBS = 3350.0


def build(fmt):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig, apply_layerwise_casting
    from finetrainers_b200.trainer import SFTTrainStep
    torch.manual_seed(0)
    m = B200LTXTransformer(LTXConfig(), torch.bfloat16, "cuda")
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
    m.add_adapter(RANK_LORA, RANK_LORA)
    m.prepare()
    st = SFTTrainStep(m, flow_weighting_scheme="logit_normal", seed=42, use_cuda_graph=True)
    g = torch.Generator().manual_seed(1234)
    lat = torch.randn(1, 128, F_LAT, H_LAT, W_LAT, generator=g).bfloat16().cuda()
    ehs = (torch.randn(1, TEXT_LEN, 4096, generator=g) * 0.1).bfloat16().cuda()
    mask = (torch.arange(TEXT_LEN)[None] < 100).cuda()
    mean, std = torch.zeros(1, 128, device="cuda"), torch.ones(1, 128, device="cuda")

    def step():
        st.train_step({"encoder_hidden_states": ehs, "encoder_attention_mask": mask},
                      {"latents": lat, "latents_mean": mean, "latents_std": std})
    return m, st, step


def timed(step, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--fmt", choices=["e4m3fn", "e5m2"], default="e4m3fn")
    args = ap.parse_args()
    fmt = {"e4m3fn": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}[args.fmt]
    from finetrainers_b200 import ops
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    out = {"card": torch.cuda.get_device_name(), "fmt": args.fmt}
    try:
        out["power_limit_w"] = sampler.nv.nvmlDeviceGetEnforcedPowerLimit(sampler.h) / 1000.0
    except Exception as e:  # noqa: BLE001
        out["power_limit_w"] = f"unavailable: {e!r}"

    # ---- memory: each arm built alone, peak over build + warm-up (graph capture included)
    for name, f in (("bf16", None), (args.fmt, fmt)):
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        m, st, step = build(f)
        after_prepare = torch.cuda.memory_allocated()
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        out[f"{name}_memory"] = {"after_prepare_gb": after_prepare / 1e9,
                                 "max_allocated_gb": torch.cuda.max_memory_allocated() / 1e9,
                                 "base_weights": {k: v / 1e9 for k, v in m.base_weight_bytes().items()}}
        if f is not None:
            # the upcast kernel on one block: read n fp8 bytes, write 2n bf16 bytes
            lw = m._lw
            src, dst = lw.blk_fp8[0], lw.units.slots[0]
            n = src.numel()
            for _ in range(3):
                ops.upcast_fp8_bf16(src, dst, n)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.launches):
                ops.upcast_fp8_bf16(src, dst, n)
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / args.launches
            out["upcast_one_block"] = {"elements": n, "us": us, "gbs": 3 * n / us / 1e3, "hbm_peak_gbs": HBM_GBS,
                                       "fraction_of_peak": 3 * n / us / 1e3 / HBM_GBS, "launches": args.launches,
                                       "upcasts_per_step": lw.upcasts // max(1, args.warmup)}
        del m, st, step
    gc.collect()
    torch.cuda.empty_cache()

    # ---- step time: both arms resident, alternated round by round
    arms = {"bf16": build(None)[2], args.fmt: build(fmt)[2]}
    for step in arms.values():
        for _ in range(args.warmup):
            step()
    mark0 = sampler.mark()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, step in arms.items():
            times[k].append(timed(step, args.steps))
    clocks = sampler.finish(mark0, sampler.mark())
    out["ms_per_step"] = {k: {"median": statistics.median(v), "rounds": v} for k, v in times.items()}
    out["ratio_fp8_over_bf16"] = out["ms_per_step"][args.fmt]["median"] / out["ms_per_step"]["bf16"]["median"]
    out["clocks"] = clocks
    print(json.dumps(out))


if __name__ == "__main__":
    main()
