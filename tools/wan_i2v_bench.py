"""Wan-2.1 I2V-14B LoRA training step on one GPU, with the T2V-14B step at the same shape for the image context's cost:
ms/step, latent tokens/s and peak allocated memory per clip (B = 1, r = 32, 512 text + 257 image tokens, CUDA-graph
steps, "full" checkpointing; an out-of-memory run is reported as a row).  ``--storage`` lists the base-weight storage
dtypes to compare: bf16, or layerwise fp8 (e4m3fn / e5m2) under finetrainers' CLI skip list; the storage dtypes and
models alternate within each of ``--repeat`` rounds, so that a spread shows beside each number.  Prints one JSON line
per configuration (with ``base_weight_bytes()``) and the card's name, power limit and SM clock read in the same run.

    python tools/wan_i2v_bench.py [--steps 3 --warmup 3] [--shapes 49x480x832,81x480x832] [--layers 40]
                                  [--storage bf16,e4m3fn] [--models i2v,t2v] [--repeat 2]
"""
import argparse
import gc
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from wan_bench import card  # noqa: E402


STORAGE = {"bf16": None, "e4m3fn": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}


def run(model, frames, height, width, steps, warmup, layers, storage="bf16"):
    from finetrainers_b200.layerwise import CLI_SKIP_MODULES_PATTERN
    from finetrainers_b200.model import apply_activation_checkpointing
    from finetrainers_b200.trainer import SFTTrainStep
    from finetrainers_b200.wan import B200WanTransformer, WanConfig
    Fl, Hl, Wl = (frames - 1) // 4 + 1, height // 8, width // 8  # Wan VAE: 4x temporal, 8x spatial
    i2v = model == "i2v"
    cfg = WanConfig.wan_i2v_14b() if i2v else WanConfig.wan_14b()
    cfg.num_layers = layers
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    m = B200WanTransformer(cfg, torch.bfloat16, "cuda")
    with torch.no_grad():
        for n, p in m.named_parameters():
            p.fill_(1.0) if "norm" in n and n.endswith("weight") else p.normal_(0, 0.02)
    if STORAGE[storage] is not None:
        m.enable_layerwise_casting(STORAGE[storage], skip_modules_pattern=CLI_SKIP_MODULES_PATTERN)
    m.add_adapter(32, 32)
    apply_activation_checkpointing(m, "full")
    st = SFTTrainStep(m, use_cuda_graph=True, flow_weighting_scheme="logit_normal")
    g = torch.Generator(device="cuda").manual_seed(0)
    lat = {"latents": torch.randn(1, 32, Fl, Hl, Wl, device="cuda", generator=g).to(torch.bfloat16),
           "latents_mean": torch.zeros(1, 16, device="cuda"), "latents_std": torch.ones(1, 16, device="cuda")}
    if i2v:
        mask = torch.zeros(1, 4, Fl, Hl, Wl, dtype=torch.bfloat16, device="cuda")
        mask[:, :, 0] = 1
        lat.update(latent_condition=torch.randn(1, 32, Fl, Hl, Wl, device="cuda", generator=g).to(torch.bfloat16),
                   latent_condition_mask=mask,
                   encoder_hidden_states_image=torch.randn(1, 257, 1280, device="cuda", generator=g).to(torch.bfloat16))
    cond = {"encoder_hidden_states": torch.randn(1, 512, 4096, device="cuda", generator=g).to(torch.bfloat16)}
    gc.collect()  # the trainer packed the weights: nothing of the unpacked (or bf16, before the cast) copies is left
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()  # the step's peak, not the bf16 weights before they were cast
    for _ in range(warmup):  # two eager steps, then the capture
        st.train_step(cond, lat)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        st.train_step(cond, lat)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    tokens = Fl * (Hl // 2) * (Wl // 2)
    return dict(model=model, storage=storage, shape=f"{frames}x{height}x{width}", latent_tokens=tokens,
                checkpointing="full", layers=layers, ms_per_step=round(ms, 1),
                latent_tokens_per_s=round(tokens * 1e3 / ms, 1),
                max_memory_allocated_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                base_weight_gib={k: round(v / 2 ** 30, 3) for k, v in m.base_weight_bytes().items()},
                loss=float(st.metrics[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--shapes", default="49x480x832,81x480x832")
    ap.add_argument("--storage", default="bf16", help="comma-separated: bf16, e4m3fn, e5m2")
    ap.add_argument("--models", default="i2v,t2v")
    ap.add_argument("--repeat", type=int, default=1)
    a = ap.parse_args()
    storages = a.storage.split(",")
    if any(s not in STORAGE for s in storages):
        raise SystemExit(f"--storage takes {sorted(STORAGE)}, not {a.storage}")
    print(json.dumps({"card": card()}), flush=True)
    for shp in a.shapes.split(","):
        f, h, w = (int(x) for x in shp.split("x"))
        for rep in range(a.repeat):
            for storage in storages:
                for model in a.models.split(","):
                    try:
                        row = run(model, f, h, w, a.steps, a.warmup, a.layers, storage)
                    except torch.cuda.OutOfMemoryError:
                        row = dict(model=model, storage=storage, shape=shp, checkpointing="full",
                                   result="out of memory")
                    print(json.dumps(dict(row, round=rep)), flush=True)
                    gc.collect()
                    torch.cuda.empty_cache()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
