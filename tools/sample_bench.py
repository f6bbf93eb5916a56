"""Validation sampling at the 2B and 13B LTX-Video geometries on one GPU.

    python tools/sample_bench.py --out DIR [--steps 50] [--warmup 5] [--models 2b,13b]

B = 1 prompt with classifier-free guidance (a batch of 2 rows), 49x512x768 (2688 latent tokens), 128 text tokens, LoRA
r = 64 on the attention projections, random weights.  For each model:

  step    the denoising step (no-grad forward in the inference plan + the guided Euler launch) captured in one CUDA graph
          and replayed --steps times after --warmup replays, timed with CUDA events: ms per step, and ms per sample of
          --steps steps;
  i2v     the same for image-to-video (LTXImageToVideoPipeline's step): per-token timesteps 0 on latent frame 0, so the
          forward embeds one timestep per latent frame, and the conditioned Euler launch;
  frames  the no-grad forward alone at 704x480 (7 x 15 x 22 = 2310 latent tokens, H W = 330), B = 1 with guidance,
          one timestep per sample against one per latent frame (frame 0 at 0), each from CUDA-graph replays, the two
          alternated in rounds: at H W = 330 the per-frame gate epilogues run the cooperative schedule;
  readback  2B only: forward + backward of the public training forward at 2688 tokens, eager, with finetrainers'
          per-token [B, S, 1] timesteps (one device-to-host read-back of two flags per call) against one timestep per
          sample, alternated in rounds;
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


def frame_timesteps(grid, t=987.5):
    """The I2V pipeline's per-token timesteps for 2 rows: 0 on latent frame 0, t elsewhere."""
    import torch
    hw = grid[1] * grid[2]
    ts = torch.full((2, grid[0] * hw), t, device="cuda")
    ts[:, :hw] = 0.0
    return ts


def replay_ms(fn, steps, warmup):
    """fn captured in one CUDA graph (after one eager call) -> ms per replay over `steps` replays after `warmup`."""
    import torch
    with torch.no_grad():
        fn()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        for _ in range(warmup):
            g.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
    del g
    return e0.elapsed_time(e1) / steps


def time_step(m, steps, warmup, i2v=False):
    """ms per denoising step from CUDA-graph replays (the step generate_latents replays); ``i2v``: the image-to-video
    step, frame 0 conditioned."""
    import torch
    from finetrainers_b200 import ops
    pe, pm, ne, nm = prompts(m)
    ehs, mask = torch.cat([ne, pe]), torch.cat([nm, pm])
    lat = torch.randn(1, S, 128, device="cuda")
    x_in = lat.bfloat16().repeat(2, 1, 1)
    t = frame_timesteps(GRID) if i2v else torch.full((2,), 987.5, device="cuda")
    dt = torch.full((1,), -1e-6, device="cuda")  # tiny steps: the latents stay in range over many replays
    n_cond = GRID[1] * GRID[2] * 128

    def step():
        pred = m(x_in, ehs, t, mask, *GRID, (8 / 25, 32, 32))[0]
        if i2v:
            ops.cfg_euler_step_cond(pred, lat, x_in, 1, S * 128, n_cond, True, 3.0, dt)
        else:
            ops.cfg_euler_step(pred, lat, x_in, 1, S * 128, True, 3.0, dt)

    ms = replay_ms(step, steps, warmup)
    assert torch.isfinite(lat).all()
    return ms


def time_frames(m, steps, warmup, rounds=3):
    """ms per no-grad forward at 704x480 with one timestep per sample and per latent frame, alternated in rounds."""
    import torch
    grid = (7, 15, 22)
    pe, pm, ne, nm = prompts(m)
    ehs, mask = torch.cat([ne, pe]), torch.cat([nm, pm])
    x_in = torch.randn(2, grid[0] * grid[1] * grid[2], 128, device="cuda").bfloat16()
    ts = {"per_sample": torch.full((2,), 987.5, device="cuda"), "per_frame": frame_timesteps(grid)}
    out = {k: [] for k in ts}
    for _ in range(rounds):
        for k, t in ts.items():
            out[k].append(replay_ms(lambda: m(x_in, ehs, t, mask, *grid, (8 / 25, 32, 32)), steps, warmup))
    return {f"{k}_ms": sorted(v)[len(v) // 2] for k, v in out.items()} | {"rounds": out}


def time_readback(m, iters, rounds=3):
    """ms per eager public forward + backward at 2688 tokens, B = 1: per-token [B, S, 1] timesteps (constant, so the
    per-sample plan after one read-back) against 1-D [B] timesteps, alternated in rounds."""
    import torch
    pe, pm, _, _ = prompts(m)
    x = torch.randn(1, S, 128, device="cuda").bfloat16()
    dp = torch.randn(1, S, 128, device="cuda").bfloat16()
    ts = {"per_token": torch.full((1, S, 1), 987, device="cuda", dtype=torch.long),
          "per_sample": torch.full((1,), 987, device="cuda", dtype=torch.long)}

    def run(t, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            m(x, pe, t, pm, *GRID, (8 / 25, 32, 32))[0].backward(dp)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    out = {k: [] for k in ts}
    for t in ts.values():
        run(t, 2)  # warm-up
    for _ in range(rounds):
        for k, t in ts.items():
            out[k].append(run(t, iters))
    return {f"{k}_ms": sorted(v)[len(v) // 2] for k, v in out.items()} | {"rounds": out}


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
        ms = time_step(m, a.steps, a.warmup, i2v=True)
        r.update({"i2v_ms_per_step": ms, "i2v_ms_per_sample": ms * a.steps})
        r["frames_704x480"] = time_frames(m, a.steps, a.warmup)
        if name == "2b":
            r["readback_2688"] = time_readback(m, 10)
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
