"""Validation sampling at the 2B and 13B LTX-Video geometries on one GPU.

    python tools/sample_bench.py --out DIR [--steps 50] [--warmup 5] [--models 2b,13b]

B = 1 prompt with classifier-free guidance (a batch of 2 rows), 49x512x768 (2688 latent tokens), 128 text tokens, LoRA
r = 64 on the attention projections, random weights.  For each model:

  step    the denoising step (no-grad forward in the inference plan + the guided Euler launch) captured in one CUDA graph
          and replayed --steps times after --warmup replays, timed with CUDA events: ms per step, and ms per sample of
          --steps steps;
  plan    workspace_bytes of the inference plan and of the training plan (keep-all) at the same shape (B = 2 rows);
  memory  13B only, on the freshly built model before anything else ran on it: max_memory_allocated over 3 training
          steps with CUDA graphs (the third a replay), then over a --steps step sample through generate_latents, then
          over one more training step, each phase's peak on its own; and memory_allocated before and after the sample
          (the inference workspace stays allocated for the next sample at that shape).

Writes DIR/sample_bench.json and prints it, with the card name, its enforced power limit and its maximum and current SM
clock (NVML, queries only).  There is no CPU path: without a CUDA device the script fails.
"""
import argparse
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

S, L, GRID = 2688, 128, (7, 16, 24)


def card():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/sample_bench.py measures on a CUDA device; none is visible")
    info = {"card": torch.cuda.get_device_name(0)}
    try:
        import pynvml as nv
        nv.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "").split(",")[0].strip()
        h = nv.nvmlDeviceGetHandleByIndex(int(vis) if vis.isdigit() else 0)
        info["power_limit_w"] = nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        info["sm_clock_max_mhz"] = nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)
        info["sm_clock_mhz"] = nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)
    except Exception as e:  # noqa: BLE001
        info["nvml"] = f"not read ({type(e).__name__})"
    return info


def build(cfg):
    import torch
    from finetrainers_b200.model import B200LTXTransformer
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
    m.add_adapter(64, 64)
    m.prepare()
    with torch.no_grad():
        m.lora_flat.normal_(0, 0.01)
    return m


def prompts(m):
    import torch
    g = torch.Generator().manual_seed(5)
    pe = (torch.randn(1, L, m.cfg.caption_channels, generator=g) * 0.1).bfloat16().cuda()
    ne = (torch.randn(1, L, m.cfg.caption_channels, generator=g) * 0.1).bfloat16().cuda()
    pm = (torch.arange(L)[None] < 100).float().cuda()
    nm = (torch.arange(L)[None] < 3).float().cuda()
    return pe, pm, ne, nm


def time_step(m, steps, warmup):
    """ms per denoising step from CUDA-graph replays (the step generate_latents replays)."""
    import torch
    from finetrainers_b200 import ops
    pe, pm, ne, nm = prompts(m)
    ehs, mask = torch.cat([ne, pe]), torch.cat([nm, pm])
    lat = torch.randn(1, S, 128, device="cuda")
    x_in = lat.bfloat16().repeat(2, 1, 1)
    t = torch.full((2,), 987.5, device="cuda")
    dt = torch.full((1,), -1e-6, device="cuda")  # tiny steps: the latents stay in range over many replays

    def step():
        pred = m(x_in, ehs, t, mask, *GRID, (8 / 25, 32, 32))[0]
        ops.cfg_euler_step(pred, lat, x_in, 1, S * 128, True, 3.0, dt)

    with torch.no_grad():
        step()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        for _ in range(warmup):
            g.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    assert torch.isfinite(lat).all()
    del g
    return ms


def memory_13b(m, steps):
    import random
    import torch
    from finetrainers_b200.specification import LTXVideoModelSpecification
    from finetrainers_b200.trainer import SFTTrainStep
    random.seed(0)
    st = SFTTrainStep(m, flow_weighting_scheme="logit_normal", seed=42, use_cuda_graph=True)
    g = torch.Generator().manual_seed(1234)
    lat = torch.randn(1, 128, *GRID, generator=g).bfloat16().cuda()
    ehs = (torch.randn(1, L, 4096, generator=g) * 0.1).bfloat16().cuda()
    cond = {"encoder_hidden_states": ehs, "encoder_attention_mask": (torch.arange(L)[None] < 100).cuda()}
    latc = {"latents": lat, "latents_mean": torch.zeros(1, 128, device="cuda"),
            "latents_std": torch.ones(1, 128, device="cuda")}
    assert m._iws is None, "the training-only peak needs a model that has not sampled yet"
    gb = 1e9
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(3):
        st.train_step(cond, latc)
    torch.cuda.synchronize()
    r = {"train_peak_gb": torch.cuda.max_memory_allocated() / gb,
         "allocated_before_sample_gb": torch.cuda.memory_allocated() / gb}
    pe, pm, ne, nm = prompts(m)
    torch.cuda.reset_peak_memory_stats()
    out = LTXVideoModelSpecification(m.cfg).generate_latents(m, pe, pm, ne, nm, num_frames=49, height=512, width=768,
                                                             num_inference_steps=steps,
                                                             generator=torch.Generator().manual_seed(1))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    del out
    r["sample_peak_gb"] = torch.cuda.max_memory_allocated() / gb
    r["allocated_after_sample_gb"] = torch.cuda.memory_allocated() / gb
    torch.cuda.reset_peak_memory_stats()
    st.train_step(cond, latc)
    torch.cuda.synchronize()
    r["train_after_sample_peak_gb"] = torch.cuda.max_memory_allocated() / gb
    del st
    return r


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--models", default="2b,13b")
    a = ap.parse_args()
    import torch
    from finetrainers_b200.model import LTXConfig
    res = {"device": card(), "shape": {"B": 1, "rows": 2, "tokens": S, "text_tokens": L, "rank": 64},
           "steps": a.steps, "warmup": a.warmup}
    for name in a.models.split(","):
        cfg = LTXConfig() if name == "2b" else LTXConfig.ltx_13b()
        m = build(cfg)
        r = {"inference_workspace_gb": m.workspace_bytes(2, S, L, inference=True) / 1e9,
             "training_workspace_gb": m.workspace_bytes(2, S, L) / 1e9}
        if name == "13b":
            r.update(memory_13b(m, a.steps))  # first: nothing has sampled on this model yet
            gc.collect()
        ms = time_step(m, a.steps, a.warmup)
        r.update({"ms_per_step": ms, "ms_per_sample": ms * a.steps})
        res[name] = r
        print(name, json.dumps(r), flush=True)
        del m
        gc.collect()
        torch.cuda.empty_cache()
    res["device_at_end"] = card()  # the SM clock after the timed work
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "sample_bench.json"), "w") as f:
        json.dump(res, f, indent=2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
