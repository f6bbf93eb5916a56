"""Training from precomputed VAE moments at LTX-2B size: the step fed latents against the step fed moments
(compute_posterior=False), alternated in one session.

    python tools/posterior_bench.py [--rounds 3] [--steps 10] [--warmup 3] [--launches 2000]

B = 1, 49x512x768 (2688 latent tokens), LoRA r = 64, CUDA-graph step; one model and one SFTTrainStep serve both inputs
(they get separate static buffers and graphs).  Prints one JSON line: median ms/step of each input over --rounds rounds of
--steps steps and their ratio; the isolated prologue (b2d_prep_noise_pack against b2d_prep_posterior_noise_pack at the
step's shape, mean of --launches launches replayed from CUDA graphs, CUDA events); the card name, enforced power limit
and median SM clock (NVML) of each timed window."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import ClockSampler, F_LAT, H_LAT, W_LAT, TEXT_LEN, RANK_LORA  # noqa: E402

C_LAT = 128
GRAPH_CALLS = 100


def build():
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
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
    m.add_adapter(RANK_LORA, RANK_LORA)
    with torch.no_grad():  # B != 0, so that the adapters change the step's numbers
        for n, p in m.named_parameters():
            if "lora_B" in n:
                p.normal_(0, 0.01)
    m.prepare()
    st = SFTTrainStep(m, flow_weighting_scheme="logit_normal", seed=42, use_cuda_graph=True)
    g = torch.Generator().manual_seed(1234)
    shp = (1, C_LAT, F_LAT, H_LAT, W_LAT)
    lat = torch.randn(shp, generator=g).bfloat16().cuda()
    moments = torch.cat([torch.randn(shp, generator=g), torch.rand(shp, generator=g) * 4.0 - 5.0], 1).bfloat16().cuda()
    ehs = (torch.randn(1, TEXT_LEN, 4096, generator=g) * 0.1).bfloat16().cuda()
    mask = (torch.arange(TEXT_LEN)[None] < 100).cuda()
    mean, std = torch.zeros(1, C_LAT, device="cuda"), torch.ones(1, C_LAT, device="cuda")
    cond = {"encoder_hidden_states": ehs, "encoder_attention_mask": mask}

    def step_latents():
        st.train_step(cond, {"latents": lat, "latents_mean": mean, "latents_std": std})

    def step_moments():
        st.train_step(cond, {"latents": moments, "latents_mean": mean, "latents_std": std}, compute_posterior=False)
    return {"latents": step_latents, "moments": step_moments}


def timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def prologue_us(launches):
    """us per launch of the two prologue kernels at the step's shape (B = 1, C = 128, S = 2688)."""
    from finetrainers_b200 import ops
    B, C, F, HW = 1, C_LAT, F_LAT, H_LAT * W_LAT
    g = torch.Generator(device="cuda").manual_seed(0)
    bf = dict(dtype=torch.bfloat16, device="cuda")
    lat = torch.randn(B, C, F, HW, device="cuda", generator=g).bfloat16()
    moments = torch.randn(B, 2 * C, F, HW, device="cuda", generator=g).bfloat16()
    eps = torch.randn(B, C, F, HW, device="cuda", generator=g).bfloat16()
    noise = torch.randn(B, C, F, HW, device="cuda", generator=g).bfloat16()
    mean, std = torch.zeros(B, C, device="cuda"), torch.ones(B, C, device="cuda")
    sig, sff = torch.full((B,), 0.5, device="cuda"), torch.full((B,), 0.1, device="cuda")
    x_t, target = torch.empty(B, F * HW, C, **bf), torch.empty(B, F * HW, C, **bf)
    runs = {
        "prep_noise_pack": lambda: ops.prep_noise_pack(lat, noise, mean, std, sig, sff, x_t, target, B, C, F, HW),
        "prep_posterior_noise_pack": lambda: ops.prep_posterior_noise_pack(moments, eps, noise, mean, std, sig, sff,
                                                                           x_t, target, B, C, F, HW),
    }
    graphs = {}
    for k, run in runs.items():
        for _ in range(5):
            run()
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            for _ in range(GRAPH_CALLS):
                run()
        gr.replay()
        graphs[k] = gr
    res = {k: [] for k in graphs}
    for _ in range(3):  # alternated
        for k, gr in graphs.items():
            res[k].append(timed(gr.replay, max(1, launches // GRAPH_CALLS)) * 1e3 / GRAPH_CALLS)
    return {k: {"mean_us": statistics.mean(v), "rounds_us": v} for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--launches", type=int, default=2000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("posterior_bench needs a CUDA device")
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    out = {"card": torch.cuda.get_device_name()}
    try:
        out["power_limit_w"] = sampler.nv.nvmlDeviceGetEnforcedPowerLimit(sampler.h) / 1000.0
    except Exception as e:  # noqa: BLE001
        out["power_limit_w"] = f"unavailable: {e!r}"

    m0 = sampler.mark()
    out["prologue"] = prologue_us(args.launches)
    m1 = sampler.mark()

    arms = build()
    for step in arms.values():
        for _ in range(args.warmup):
            step()
    m2 = sampler.mark()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, step in arms.items():
            times[k].append(timed(step, args.steps))
    m3 = sampler.mark()
    out["ms_per_step"] = {k: {"median": statistics.median(v), "rounds": v} for k, v in times.items()}
    out["ratio_moments_over_latents"] = out["ms_per_step"]["moments"]["median"] / out["ms_per_step"]["latents"]["median"]
    out["clocks_prologue"] = sampler.finish(m0, m1)
    out["clocks_step"] = sampler.finish(m2, m3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
