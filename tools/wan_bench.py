"""Wan-2.1 1.3B LoRA training step on one GPU: ms/step, latent tokens/s and peak allocated memory per shape and
checkpointing policy (B = 1, r = 32, 512 text tokens, CUDA-graph steps).  Prints one JSON line per configuration and the
card's name, power limit and SM clock read in the same run.

    python tools/wan_bench.py [--steps 10 --warmup 3] [--shapes 49x480x832,81x832x480] [--layers 30]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def run(frames, height, width, ckpt, steps, warmup, layers):
    from finetrainers_b200.model import apply_activation_checkpointing
    from finetrainers_b200.trainer import SFTTrainStep
    from finetrainers_b200.wan import B200WanTransformer, WanConfig
    Fl, Hl, Wl = (frames - 1) // 4 + 1, height // 8, width // 8  # Wan VAE: 4x temporal, 8x spatial
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    m = B200WanTransformer(WanConfig(num_layers=layers), torch.bfloat16, "cuda")
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.02)
    m.add_adapter(32, 32)
    if ckpt:
        apply_activation_checkpointing(m, "full")
    st = SFTTrainStep(m, use_cuda_graph=True, flow_weighting_scheme="logit_normal")
    g = torch.Generator(device="cuda").manual_seed(0)
    lat = {"latents": torch.randn(1, 32, Fl, Hl, Wl, device="cuda", generator=g).to(torch.bfloat16),
           "latents_mean": torch.zeros(1, 16, device="cuda"), "latents_std": torch.ones(1, 16, device="cuda")}
    cond = {"encoder_hidden_states": torch.randn(1, 512, 4096, device="cuda", generator=g).to(torch.bfloat16)}
    for _ in range(warmup):
        st.train_step(cond, lat)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        st.train_step(cond, lat)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    tokens = Fl * (Hl // 2) * (Wl // 2)
    out = dict(shape=f"{frames}x{height}x{width}", latent_tokens=tokens, checkpointing="full" if ckpt else "keep-all",
               layers=layers, ms_per_step=round(ms, 2), latent_tokens_per_s=round(tokens * 1e3 / ms, 1),
               max_memory_allocated_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
               loss=float(st.metrics[1]))
    del st, m
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--layers", type=int, default=30)
    ap.add_argument("--shapes", default="49x480x832,81x832x480")
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    for shp in a.shapes.split(","):
        f, h, w = (int(x) for x in shp.split("x"))
        for ckpt in (False, True):
            try:
                print(json.dumps(run(f, h, w, ckpt, a.steps, a.warmup, a.layers)), flush=True)
            except torch.cuda.OutOfMemoryError:
                print(json.dumps(dict(shape=shp, checkpointing="full" if ckpt else "keep-all", result="out of memory")),
                      flush=True)
                torch.cuda.empty_cache()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
