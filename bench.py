"""bench.py — the DiT training-step benchmark (BASELINE.json: LTX-Video-2B T2V LoRA SFT, 49x512x768, bf16).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl b200|reference|reference-gpu] [--batch B] [--dump-outputs DIR]
  (N > 1: python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...)

One "step" = one full SFT step of the hot path on one batch of synthetic latents per GPU: noising/packing, DiT forward
(28 blocks), flow-match MSE loss, hand-written backward, gradient all-reduce (N>1), clip + AdamW.
`value`  = latent tokens/s over the whole job with the batch already resident in HBM (K steps between two CUDA events,
           max over ranks); the per-step event pairs give `ms_per_step_median` beside it.
`e2e`    = the same step through the public API (SFTTrainStep.train_step) with the batch in pinned HOST memory: per
           step H2D of latents + text embeddings + mask, and a D2H read of the step's loss/grad-norm metrics.
`--impl reference` times the CPU restatement of the reference step (oracle/ltx_oracle.py; the reference itself cannot
be installed here: diffusers/peft are absent, no network) on the host cores: each timed "step" is ONE bounded sample =
forward+loss+backward of `n` of the 28 blocks at full width, `n` sized so the K+W samples finish within a few minutes;
`ms_per_step` is the time of that sample and `value` the tokens/s it extrapolates to (x 28/n), both stated in the line.
`--dump-outputs DIR` writes what the last timed step computed as DIR/<name>.npy (see dump_outputs).
`--impl reference-gpu` (informational): the same oracle moved to cuda:0 in bf16 with
PyTorch SDPA and per-block activation checkpointing - the "PyTorch eager on the same box" bar of SURVEY section 0.
"""
import argparse
import json
import math
import os
import random
import statistics
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "latent_tokens_per_sec"
UNIT = "tokens/s"
F_LAT, H_LAT, W_LAT = 7, 16, 24          # 49x512x768 -> (49-1)/8+1, 512/32, 768/32
S_TOK = F_LAT * H_LAT * W_LAT            # 2688 latent tokens per sample
TEXT_LEN = 128
RANK_LORA = 64
N_BLOCKS = 28
FLOP_PER_TOKEN_ALG = 8.88e9              # SURVEY §8(d): 2G + 3.5A, no recompute counted


def workload_config(B, world, parallelism="ddp"):
    """The `config` object of BOTH arms (the reference arm reports on the b200 arm's config)."""
    return {"workload": f"LTX-Video-2B T2V LoRA r={RANK_LORA} SFT step, 49x512x768 (2688 latent tokens/sample), "
                        f"B={B}/GPU, AdamW+clip, logit_normal sigmas", "global_batch": B * world,
            "parallelism": f"{parallelism}{world}",
            "l2": "working set (3.8 GB weights + 5.5 GB activations per step) >> 50 MB L2; no flush needed",
            "random_init": True}


def read_peaks():
    """Dense BF16 tensor and HBM3 peaks of the H100 SXM data sheet (700 W part); a power-capped card reaches less."""
    return {"burst": 989.0, "sustained": 989.0, "hbm": 3350.0, "src": "H100 SXM data sheet"}


DUMP_PARAM_SAMPLE = 2_000_000   # seeded sample of the trained LoRA parameters written by --dump-outputs (8 MB fp32)


def dump_outputs(d, model, step, B):
    """What a caller of the timed step receives after its last call: the step metrics (gradient norm, loss), the
    prediction of the last forward and the updated LoRA parameters (a fixed, seeded sample of the flat fp32 buffer)."""
    import numpy as np
    import torch
    os.makedirs(d, exist_ok=True)
    torch.cuda.synchronize()
    np.save(os.path.join(d, "metrics.npy"), step.metrics[0:2].double().cpu().numpy())
    pred = model._workspace(B, S_TOK, TEXT_LEN)["pred"]
    np.save(os.path.join(d, "pred.npy"), pred.float().view(B, S_TOK, -1).cpu().numpy())
    flat = model.lora_flat.detach()
    g = torch.Generator().manual_seed(0)
    idx = torch.randint(0, flat.numel(), (min(DUMP_PARAM_SAMPLE, flat.numel()),), generator=g)
    np.save(os.path.join(d, "lora_params_sample.npy"), flat.float().cpu()[idx].numpy())


class ClockSampler:
    """SM clock / throttle reasons sampled IN-PROCESS through NVML every 100 ms (no fork: forking `nvidia-smi` from a
    process that holds a CUDA context stalled the first timed loop of round 1 by seconds)."""
    _REASONS = (("hw_slowdown", 0x8), ("hw_thermal_slowdown", 0x40), ("sw_thermal_slowdown", 0x20), ("sw_power_cap", 0x4))

    def __init__(self, idx):
        self.rows, self.stop, self.h, self.mx = [], False, None, None
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            # honour CUDA_VISIBLE_DEVICES: NVML enumerates physical devices
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = idx
            if vis:
                ent = [v.strip() for v in vis.split(",") if v.strip()]
                if idx < len(ent) and ent[idx].isdigit():
                    phys = int(ent[idx])
            self.h = pynvml.nvmlDeviceGetHandleByIndex(phys)
            self.mx = float(pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM))
        except Exception as e:  # noqa: BLE001
            self.err = repr(e)
        self.t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        nv = self.nv
        while not self.stop:
            try:
                sm = float(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
                try:
                    rs = int(nv.nvmlDeviceGetCurrentClocksEventReasons(self.h))
                except Exception:  # noqa: BLE001
                    rs = int(nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h))
                util = float(nv.nvmlDeviceGetUtilizationRates(self.h).gpu)
                self.rows.append((sm, rs, util))
            except Exception:  # noqa: BLE001
                pass
            time.sleep(0.1)

    def start(self):
        if self.h is not None:
            self.t.start()

    def mark(self):
        return len(self.rows)

    def finish(self, lo=0, hi=None):
        self.stop = True
        if self.h is not None:
            self.t.join(timeout=3)
        rows = self.rows[lo:hi]
        load = [r for r in rows if r[2] >= 50.0] or rows
        reasons = set()
        for _, rs, _ in load:
            for nme, bit in self._REASONS:
                if rs & bit:
                    reasons.add(nme)
        sm = [r[0] for r in load]
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": self.mx, "reasons": sorted(reasons),
                "samples": len(sm), "source": "nvml in-process, 100 ms" if self.h is not None else f"unavailable: {getattr(self, 'err', '')}"}


# ----------------------------------------------------------------------------------------------------------------------
# reference arm: the CPU restatement of the reference step on the host cores
# ----------------------------------------------------------------------------------------------------------------------
def physical_cores():
    """Physical cores this process may run on (SMT siblings counted once): oversubscribing the hyperthreads made the
    fp32 oracle ~10x slower on the 128-thread GPU hosts."""
    try:
        allowed = os.sched_getaffinity(0)
        seen, cur = set(), {}
        for line in open("/proc/cpuinfo"):
            if ":" in line:
                k, v = [x.strip() for x in line.split(":", 1)]
                cur[k] = v
            elif not line.strip() and cur:
                if int(cur.get("processor", -1)) in allowed:
                    seen.add((cur.get("physical id", "0"), cur.get("core id", cur.get("processor"))))
                cur = {}
        return max(1, len(seen)) if seen else max(1, len(allowed) // 2)
    except Exception:  # noqa: BLE001
        return max(1, (os.cpu_count() or 2) // 2)


class CpuReference:
    """Oracle (fp32) with `layers` of the 28 blocks at full width (D=2048, S=2688, L=128, r=64, B=1); one sample = one
    forward + loss + backward.  Built once, sampled many times."""

    def __init__(self, layers, threads=None):
        import torch
        from oracle import ltx_oracle as O
        # torchrun exports OMP_NUM_THREADS=1; this leg runs on rank 0 alone, so it takes every core the box gives us
        n = threads or physical_cores()
        torch.set_num_threads(n)
        self.cores = torch.get_num_threads()
        self.layers = layers
        self.O = O
        cfg = O.LTXConfig(num_layers=layers)
        self.m = O.LTXTransformerOracle(cfg)
        O.add_lora(self.m, RANK_LORA, RANK_LORA)
        O.synthetic_init_(self.m, seed=0, lora_b_std=0.02)
        self.batch = O.make_synthetic_batch(cfg, 1, F_LAT, H_LAT, W_LAT, TEXT_LEN, seed=1234, dtype=torch.float32)

    def sample(self):
        """-> seconds for fwd+loss+bwd of `layers` blocks."""
        for p in self.m.parameters():
            p.grad = None
        t0 = time.perf_counter()
        self.O.oracle_step(self.m, self.batch)
        return time.perf_counter() - t0

    def describe(self):
        return (f"oracle (CPU restatement of the reference step, plain PyTorch) fwd+loss+bwd fp32, {self.layers} of "
                f"{N_BLOCKS} blocks at full width (D=2048, S=2688, L=128, r=64, B=1) per sample; tokens/s = 2688 / "
                f"(sample_seconds x {N_BLOCKS}/{self.layers})")


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    n_samples = args.steps + args.warmup
    # ~1.2 s per block and sample on a 64-core host: size the sample so the whole run stays near four minutes
    layers = max(1, min(N_BLOCKS, int(240.0 / (max(1, n_samples) * 1.2))))
    ref = CpuReference(layers)
    times = []
    for i in range(n_samples):
        t = ref.sample()
        if i >= args.warmup:
            times.append(t)
    t_sample = sum(times) / len(times)
    full = t_sample * N_BLOCKS / layers
    v = S_TOK / full
    world = int(os.environ.get("WORLD_SIZE", "1"))
    line = {
        "impl": "reference", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": t_sample * 1e3, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": workload_config(args.batch, world),
        "cpu_baseline": {"value": v, "unit": UNIT, "cores": ref.cores, "kind": "port", "sample": ref.describe(),
                         "sample_seconds": t_sample, "extrapolated_full_step_seconds": full},
        "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "note": "each timed step is ONE bounded sample (ms_per_step = its wall time); value extrapolates the sample to "
                "the full 28-block step, so value != tokens_per_step / ms_per_step by the factor 28/blocks_in_sample; "
                "device=cpu, runs on rank 0 only",
    }
    print(json.dumps(line))


def run_reference_gpu(args):
    """Informational: the oracle itself on cuda:0 (bf16 base weights, fp32 adapters as trainer.py:130-136, PyTorch SDPA,
    per-block activation checkpointing as --gradient_checkpointing, torch.optim.AdamW + clip) - eager PyTorch on the box."""
    import torch
    from torch.utils.checkpoint import checkpoint
    from oracle import ltx_oracle as O
    dev = torch.device("cuda", 0)
    cfg = O.LTXConfig()
    m = O.LTXTransformerOracle(cfg)
    O.add_lora(m, RANK_LORA, RANK_LORA)
    O.synthetic_init_(m, seed=0, lora_b_std=0.02)
    for n, p in m.named_parameters():
        p.data = p.data.to(dev, torch.float32 if "lora_" in n else torch.bfloat16)
    for blk in m.transformer_blocks:
        fwd = blk.forward
        blk.forward = (lambda f: (lambda *a, **k: checkpoint(f, *a, use_reentrant=False, **k)))(fwd)
    params = [p for n, p in m.named_parameters() if "lora_" in n]
    opt = torch.optim.AdamW(params, lr=5e-5, betas=(0.9, 0.99), weight_decay=1e-4, eps=1e-8)
    batch = O.make_synthetic_batch(cfg, args.batch, F_LAT, H_LAT, W_LAT, TEXT_LEN, seed=1234)
    batch = {k: v.to(dev) for k, v in batch.items()}

    def step(_):
        opt.zero_grad(set_to_none=True)
        O.oracle_step(m, batch)
        O.clip_grad_norm_(params, 1.0)
        opt.step()

    for i in range(max(args.warmup, 3)):
        step(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        step(i)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    v = args.batch * S_TOK / (ms * 1e-3)
    print(json.dumps({"impl": "reference-gpu", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": 1, "steps": args.steps,
                      "warmup": max(args.warmup, 3), "ms_per_step": ms, "higher_is_better": True, "dtype": "bf16",
                      "data": "synthetic", "config": workload_config(args.batch, 1),
                      "note": "informational: oracle/ltx_oracle.py (restated reference step) in eager PyTorch on cuda:0, bf16 "
                              "weights, fp32 LoRA, F.scaled_dot_product_attention, per-block checkpointing, torch AdamW"}))


# ----------------------------------------------------------------------------------------------------------------------
# b200 arm
# ----------------------------------------------------------------------------------------------------------------------
def run_b200(args):
    import torch
    import torch.distributed as dist
    from finetrainers_b200 import ops
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    from finetrainers_b200.trainer import SFTTrainStep
    from finetrainers_b200.parallel import B200ParallelBackend

    os.environ.setdefault("NCCL_DEBUG", "WARN")  # keep NCCL's version banner off stdout: rank 0 prints ONE JSON line
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != args.gpus:
        raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={world}: launch with torch.distributed.run --nproc-per-node {args.gpus}")
    local = int(os.environ.get("LOCAL_RANK", "0"))
    rank = int(os.environ.get("RANK", "0"))
    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()               # before CUDA work and warm-up: nothing is forked or started inside a timed region
    fsdp = args.parallelism == "fsdp"
    if fsdp and world < 2:
        raise SystemExit("--parallelism fsdp needs --gpus >= 2 (torchrun)")
    be = B200ParallelBackend(backend="nccl", **({"dp_shards": world} if fsdp else {})) if world > 1 else None
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    B = args.batch

    # ---- model: LTX-2B architecture, random init (no checkpoints offline), LoRA r=64 on to_q|to_k|to_v|to_out.0
    torch.manual_seed(0)
    # the step draws its first-frame-conditioning decision from Python's global `random`, as the reference does: seeded
    # so that the same arguments give the same inputs on every run
    random.seed(1234 + rank)
    model = B200LTXTransformer(LTXConfig(), torch.bfloat16, dev)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "scale_shift_table" in n:
                p.normal_(0, 1.0 / p.shape[-1] ** 0.5)
            elif "norm_q" in n or "norm_k" in n:
                p.fill_(1.0)
            else:
                p.normal_(0, 0.02)
    model.add_adapter(RANK_LORA, RANK_LORA)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "lora_B" in n:
                p.normal_(0, 0.01)
    model.prepare()
    if be is not None:
        if fsdp:
            be.apply_fsdp2(model, param_dtype=torch.bfloat16, reduce_dtype=torch.float32, output_dtype=None,
                           pp_enabled=False, cpu_offload=False, device_mesh=be.get_mesh()[("dp_shard_cp",)])
        else:
            be.apply_ddp(model)
    # optimiser settings of the reference example (examples/training/sft/ltx_video/crush_smol_lora/train.sh:88-98)
    step = SFTTrainStep(model, flow_weighting_scheme="logit_normal", seed=42 + rank, use_cuda_graph=not args.no_graph,
                        lr=5e-5, beta1=0.9, beta2=0.99, weight_decay=1e-4, eps=1e-8, max_grad_norm=1.0,
                        lr_scheduler="constant_with_warmup", lr_warmup_steps=1000, ddp_chunks=args.ddp_chunks)

    # ---- synthetic data: a small pool of pinned host batches (SURVEY §8d), plus one device-resident copy
    g = torch.Generator().manual_seed(1234 + rank)
    pool = []
    for _ in range(4):
        lat = torch.randn(B, 128, F_LAT, H_LAT, W_LAT, generator=g).bfloat16().pin_memory()
        ehs = (torch.randn(B, TEXT_LEN, 4096, generator=g) * 0.1).bfloat16().pin_memory()
        lens = torch.randint(16, TEXT_LEN + 1, (B,), generator=g)
        mask = (torch.arange(TEXT_LEN)[None] < lens[:, None]).pin_memory()
        pool.append((lat, ehs, mask))
    mean = torch.zeros(B, 128, device=dev)
    std = torch.ones(B, 128, device=dev)
    dev_pool = [(a.to(dev), b.to(dev), c.to(dev)) for a, b, c in pool]
    h2d_bytes = sum(t.numel() * t.element_size() for t in pool[0])

    def step_resident(i):
        lat, ehs, mask = dev_pool[i % len(dev_pool)]
        step.train_step({"encoder_hidden_states": ehs, "encoder_attention_mask": mask},
                        {"latents": lat, "latents_mean": mean, "latents_std": std})

    last_metrics = {}

    def step_e2e(i):
        lat, ehs, mask = pool[i % len(pool)]
        lat_d = lat.to(dev, non_blocking=True)
        ehs_d = ehs.to(dev, non_blocking=True)
        mask_d = mask.to(dev, non_blocking=True)
        m = step.train_step({"encoder_hidden_states": ehs_d, "encoder_attention_mask": mask_d},
                            {"latents": lat_d, "latents_mean": mean, "latents_std": std}, sync_metrics=True)
        last_metrics.update(m)
        # a throughput measured on garbage is not a measurement: stop at the first non-finite loss / gradient norm
        if not (math.isfinite(m["train/global_avg_loss"]) and math.isfinite(m["train/grad_norm"])):
            raise SystemExit(f"bench: non-finite training metrics at e2e step {i}: {m}")
        return m

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, n):
        """n calls between a barrier+sync on both sides; an event after every call.  -> (total ms [max over ranks],
        per-call ms list of this rank)."""
        barrier()
        evs = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
        evs[0].record()
        for i in range(n):
            fn(i)
            evs[i + 1].record()
        barrier()
        ms = evs[0].elapsed_time(evs[n])
        per = [evs[i].elapsed_time(evs[i + 1]) for i in range(n)]
        if world > 1:
            t = torch.tensor([ms], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = t.item()
        return ms, per

    n_before = ops.LAUNCH_COUNT
    step_resident(0)                       # eager: also counts the kernels one step launches
    launches_per_step = ops.LAUNCH_COUNT - n_before
    warm = max(args.warmup, 3)
    for i in range(warm + 2):              # +2: eager warm-ups before the CUDA graph is captured
        step_resident(i)
    mark0 = sampler.mark() if sampler else 0
    ms_total, per_step = timed(step_resident, args.steps)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, model, step, B)
    for i in range(2):
        step_e2e(i)
    ms_e2e, per_e2e = timed(step_e2e, args.steps)
    remeasured = False
    if abs(ms_total - ms_e2e) / ms_total > 0.05:
        # the two loops run the same graph; >5 % apart means one of them was disturbed (host stall, clock ramp): redo both once
        remeasured = True
        ms_total, per_step = timed(step_resident, args.steps)
        ms_e2e, per_e2e = timed(step_e2e, args.steps)
    mark1 = sampler.mark() if sampler else 0
    launches = launches_per_step * args.steps

    # ---- dominant kernel measured live, twice:
    # (a) isolated: the FFN up-projection GEMM launch of the step (2688 x 8192 x 2048, GELU epilogue, two outputs), CUDA
    #     events on the launching stream, operands rotated over 3 buffer sets (> 50 MB L2 in total)  -> vs BURST peak
    # (b) in-step: one eager step with an event pair around every libb2d launch                       -> vs SUSTAINED peak
    R_, D_ = B * S_TOK, 2048
    sets = [(torch.randn(R_, D_, device=dev).bfloat16(), torch.empty(R_, 4 * D_, device=dev, dtype=torch.bfloat16),
             torch.empty(R_, 4 * D_, device=dev, dtype=torch.bfloat16)) for _ in range(3)]
    e_blk = model._blk[0]

    def ffn_up(i):
        x_, f_, pre_ = sets[i % 3]
        ops.gemm(x_, e_blk["W1"], f_, M=R_, N=4 * D_, K=D_, bias=e_blk["b1"], epi=ops.EPI_GELU, out2=pre_)

    for i in range(3):
        ffn_up(i)
    n_k = 30
    ms_k, _ = timed(ffn_up, n_k)
    del sets
    # every rank runs the eager step (it contains the gradient exchange); rank 0's event pairs are the ones reported
    graph_flag = step.use_cuda_graph
    step.use_cuda_graph = False
    ops.KERNEL_TIMES.clear()
    ops.TIMING = rank == 0
    step_resident(0)
    torch.cuda.synchronize()
    ops.TIMING = False
    step.use_cuda_graph = graph_flag
    in_step = None
    if rank == 0:
        kt = ops.collect_kernel_times()
        tot = sum(v[0] for v in kt.values())
        gemm_ms = sum(v[0] for k, v in kt.items() if k.split("/")[-1] in ("gemm", "ffn_up", "lora_u", "lora_du", "lora_dA", "lora_dB"))
        attn_ms = sum(v[0] for k, v in kt.items() if k.split("/")[-1] in ("attn_fwd", "attn_bwd"))
        up = [v for k, v in kt.items() if k.endswith("ffn_up")]
        in_step = {"eager_step_kernel_ms": tot, "gemm_ms": gemm_ms, "attention_ms": attn_ms,
                   "other_ms": tot - gemm_ms - attn_ms,
                   "ffn_up_avg_us": (sum(v[0] for v in up) / max(1, sum(v[1] for v in up))) * 1e3 if up else None}
    if world > 1:
        dist.barrier()
    clocks = sampler.finish(mark0, mark1) if sampler else None

    ms_step = ms_total / args.steps
    tokens_per_step = B * S_TOK * world
    value = tokens_per_step / (ms_step * 1e-3)
    e2e_value = tokens_per_step / (ms_e2e / args.steps * 1e-3)
    if rank != 0:
        if be is not None:
            be.destroy()
        return
    peaks = read_peaks()
    avg_ms = ms_k / n_k
    flops = 2.0 * (B * S_TOK) * 8192 * 2048
    ach = flops / (avg_ms * 1e-3) / 1e12
    roof = {"bound": "tensor", "kernel": "b2d GEMM, FFN up-projection 2688x8192x2048 + bias + GELU epilogue, two bf16 outputs",
            "achieved": ach, "peak": peaks["burst"], "unit": "TFLOP/s", "frac": ach / peaks["burst"], "traffic": None,
            "peak_source": f"{peaks['src']} bf16 dense TFLOP/s (the kernel is timed alone, {n_k} back-to-back launches)",
            "avg_launch_us": avg_ms * 1e3, "launches_timed": n_k,
            "frac_of_sustained_peak": ach / peaks["sustained"],
            "step_frac_of_alg_roofline": (value / world) * FLOP_PER_TOKEN_ALG / (peaks["sustained"] * 1e12)}
    if in_step and in_step.get("ffn_up_avg_us"):
        a2 = flops / (in_step["ffn_up_avg_us"] * 1e-6) / 1e12
        roof["in_step"] = {"avg_launch_us": in_step["ffn_up_avg_us"], "achieved": a2, "peak": peaks["sustained"],
                           "frac": a2 / peaks["sustained"], "how": "event pair around each of the 28 launches in one eager step"}
        roof["step_breakdown_ms"] = {k: in_step[k] for k in ("eager_step_kernel_ms", "gemm_ms", "attention_ms", "other_ms")}
    cpu = None
    if world == 1 and not args.no_cpu_baseline:
        ref = CpuReference(4)
        ref.sample()
        t = ref.sample()
        full = t * N_BLOCKS / ref.layers
        cpu = {"value": S_TOK / full, "unit": UNIT, "cores": ref.cores, "kind": "port", "sample": ref.describe(),
               "sample_seconds": t, "extrapolated_full_step_seconds": full}
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": warm,
        "ms_per_step": ms_step, "ms_per_step_median": statistics.median(per_step), "ms_per_step_max": max(per_step),
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
        "data": "synthetic", "tokens_per_sec_per_gpu": value / world,
        "config": workload_config(B, world, args.parallelism),
        "e2e": {"value": e2e_value, "unit": UNIT, "h2d_bytes_per_step": h2d_bytes, "d2h_bytes_per_step": 12,
                "ms_per_step": ms_e2e / args.steps, "ms_per_step_median": statistics.median(per_e2e)},
        "consistency": {"value_vs_e2e_rel_diff": abs(ms_total - ms_e2e) / ms_total, "remeasured": remeasured},
        "gpu_launches": launches, "clocks": clocks, "roofline": roof, "cpu_baseline": cpu,
        "final_metrics": {"loss": last_metrics.get("train/global_avg_loss"), "grad_norm": last_metrics.get("train/grad_norm")},
        "cuda_graph": step.use_cuda_graph,
    }
    if fsdp:
        fs = model._fsdp
        line["fsdp"] = {"local_param_bytes": fs.local_param_bytes(), "full_bytes_per_block": fs.full_bytes_per_block,
                        "allgathers_per_step": (2 * (fs.nl - 2) + 1), "note": "per-block bf16 all-gather prefetched one block "
                        "ahead on a communication stream; fp32 reduce-scatter of the flat LoRA gradient; sharded AdamW"}
    print(json.dumps(line))
    if be is not None:
        be.destroy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference", "reference-gpu"])
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-graph", action="store_true", help="launch every kernel from Python instead of replaying a CUDA graph")
    ap.add_argument("--ddp-chunks", type=int, default=4, help="N > 1, ddp: block-range chunks of the overlapped gradient exchange (1 = one serial all-reduce)")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the last timed step's metrics, prediction and a seeded sample of the LoRA parameters as .npy")
    ap.add_argument("--parallelism", default="ddp", choices=["ddp", "fsdp"],
                    help="N > 1: ddp = replicas + flat gradient all-reduce (default); fsdp = FSDP-2 per-block sharding")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    elif args.impl == "reference-gpu":
        run_reference_gpu(args)
    else:
        run_b200(args)


if __name__ == "__main__":
    main()
