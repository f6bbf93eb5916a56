"""LoRA on the feed-forward projections at LTX-2B size: the attention target set against attention + ff.net.0.proj +
ff.net.2, alternated in one session.

    python tools/lora_ffn_bench.py [--rounds 3] [--steps 10] [--warmup 3] [--launches 1000]

B = 1, 49x512x768 (2688 latent tokens), LoRA r = 64, CUDA-graph step.  Prints one JSON line: median ms/step per target
set (each round times both back to back) and their ratio, max_memory_allocated of each set built alone, CUDA-event
times (mean of --launches, replayed from CUDA graphs) of the two K = 4 D adapter launches (u_ff2 = s f A_ff2^T,
du_ff1 = s dwide B_ff1) at every split count against the unsplit launch, with the count the model picks, and the card name, enforced power limit and
median SM clock (NVML)."""
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

FFN_RX = "(transformer_blocks|single_transformer_blocks).*(to_q|to_k|to_v|to_out.0|ff.net.0.proj|ff.net.2)"
SETS = {"attn": None, "attn_ffn": FFN_RX}
GRAPH_CALLS = 50


def build(targets):
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
    m.add_adapter(RANK_LORA, RANK_LORA, target_modules=targets)
    with torch.no_grad():  # B != 0, so that the adapters change the step's numbers
        for n, p in m.named_parameters():
            if "lora_B" in n:
                p.normal_(0, 0.01)
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


def timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def skinny_launches(launches):
    """us per call of the two K = 4 D adapter launches at M = 2688, N = rp = 64, for each split count."""
    from finetrainers_b200 import ops
    M, K, rp = F_LAT * H_LAT * W_LAT, 4 * 2048, 64
    x = (torch.randn(M, K, device="cuda") * 0.1).bfloat16()
    A = (torch.randn(rp, K, device="cuda") * 0.01).bfloat16()      # A_ff2 [rp, 4D]
    Bm = (torch.randn(K, rp, device="cuda") * 0.01).bfloat16()     # B_ff1 [4D, rp]
    out = torch.empty(M, rp, dtype=torch.bfloat16, device="cuda")
    part = torch.empty(ops.SPLITK_MAX, M, rp, dtype=torch.float32, device="cuda")
    res = {}
    for name, W, b_mn in (("u_ff2", A, False), ("du_ff1", Bm, True)):
        res[name] = {}
        for s in (1, 2, 4, 8, 16):
            kk = K // s

            def run():
                if s == 1:
                    ops.gemm(x, W, out, M=M, N=rp, K=K, b_mn=b_mn, alpha=0.5)
                else:
                    ops.gemm(x, W, part, M=M, N=rp, K=kk, b_mn=b_mn, ldc=rp, batch=s, a_boff=(0, kk),
                             b_boff=(kk, 0) if b_mn else (0, kk), c_boff=M * rp, epi=ops.EPI_F32_STORE)
                    ops.splitk_reduce_bf16(part, out, s, M, rp, alpha=0.5)
            for _ in range(5):
                run()
            # replayed from a CUDA graph (as in the step): a Python loop of launches would time the host's enqueue rate
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(GRAPH_CALLS):
                    run()
            g.replay()
            res[name][s] = timed(g.replay, max(1, launches // GRAPH_CALLS)) * 1e3 / GRAPH_CALLS
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--launches", type=int, default=1000)
    args = ap.parse_args()
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    out = {"card": torch.cuda.get_device_name()}
    try:
        out["power_limit_w"] = sampler.nv.nvmlDeviceGetEnforcedPowerLimit(sampler.h) / 1000.0
    except Exception as e:  # noqa: BLE001
        out["power_limit_w"] = f"unavailable: {e!r}"

    # ---- the two split-K launches, every split count
    mark0 = sampler.mark()
    out["skinny_us"] = skinny_launches(args.launches)
    out["skinny_clocks"] = sampler.finish(mark0, sampler.mark())

    # ---- memory: each target set built alone, peak over build + warm-up (graph capture included)
    for name, tm in SETS.items():
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        m, st, step = build(tm)
        after_prepare = torch.cuda.memory_allocated()
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        out[f"{name}_memory"] = {"after_prepare_gb": after_prepare / 1e9,
                                 "max_allocated_gb": torch.cuda.max_memory_allocated() / 1e9,
                                 "trainable_params": sum(p.numel() for p in m.parameters() if p.requires_grad)}
        if m.lora_ffn:
            out["splits_chosen"] = m._ffn_splits(F_LAT * H_LAT * W_LAT, 4 * m.cfg.inner_dim)
        del m, st, step
    gc.collect()
    torch.cuda.empty_cache()
    out["memory_delta_gb"] = (out["attn_ffn_memory"]["max_allocated_gb"] - out["attn_memory"]["max_allocated_gb"])

    # ---- step time: both target sets resident, alternated round by round
    arms = {k: build(tm)[2] for k, tm in SETS.items()}
    for step in arms.values():
        for _ in range(args.warmup):
            step()
    mark0 = sampler.mark()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, step in arms.items():
            times[k].append(timed(step, args.steps))
    out["clocks"] = sampler.finish(mark0, sampler.mark())
    out["ms_per_step"] = {k: {"median": statistics.median(v), "rounds": v} for k, v in times.items()}
    out["ratio_ffn_over_attn"] = out["ms_per_step"]["attn_ffn"]["median"] / out["ms_per_step"]["attn"]["median"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
