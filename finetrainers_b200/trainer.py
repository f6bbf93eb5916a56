"""The SFT train-step body of finetrainers' ``SFTTrainer._train``
(``finetrainers/trainer/sft_trainer/trainer.py:397-529``) rebuilt around the H100 engine.

Kept from the reference: sigma sampling (``utils/diffusion.py:38-63,84-114``), loss weighting (``:117-130``), the
loss definition (``trainer.py:474-481``), clip-then-AdamW ordering (``:488-503``), gradient accumulation (including the
reference's clip after EVERY micro-step, ``train_step`` -> ``clip_accumulated``), and the per-step metrics (``global_avg_loss``, ``global_max_loss``, ``grad_norm``; ``:507-520``).

Changed here: loss + dloss/dpred is one kernel; LoRA gradients land in one flat fp32 buffer that is all-reduced in
place (DDP) and consumed by one fused clip+AdamW kernel; the three scalar reductions are one 3-float all-reduce; the
host never synchronises inside a step unless the caller asks for the metrics (``sync_metrics``).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from . import ops
from .model import B200LTXTransformer
from .specification import LTXVideoModelSpecification, FlowMatchSchedulerTable, moments_channels
from .lr_schedule import lr_factor_fn
from .parallel import allreduce_flat_grads, fused_step_metrics


def compute_density_for_timestep_sampling(weighting_scheme: str, batch_size: int, logit_mean: float = 0.0,
                                          logit_std: float = 1.0, mode_scale: float = 1.29, device="cpu",
                                          generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """utils/diffusion.py:38-63."""
    if weighting_scheme == "logit_normal":
        u = torch.normal(mean=logit_mean, std=logit_std, size=(batch_size,), device=device, generator=generator)
        u = torch.nn.functional.sigmoid(u)
    elif weighting_scheme == "mode":
        u = torch.rand(size=(batch_size,), device=device, generator=generator)
        u = 1 - u - mode_scale * (torch.cos(math.pi * u / 2) ** 2 - 1 + u)
    else:
        u = torch.rand(size=(batch_size,), device=device, generator=generator)
    return u


def prepare_sigmas(scheduler, sigmas: torch.Tensor, batch_size: int, num_train_timesteps: int,
                   flow_weighting_scheme: str = "none", flow_logit_mean: float = 0.0, flow_logit_std: float = 1.0,
                   flow_mode_scale: float = 1.29, device="cpu", generator=None) -> torch.Tensor:
    """utils/diffusion.py:84-114 (flow-match branch)."""
    w = compute_density_for_timestep_sampling(flow_weighting_scheme, batch_size, flow_logit_mean, flow_logit_std,
                                              flow_mode_scale, device, generator)
    indices = (w * num_train_timesteps).long()
    return sigmas[indices]


def prepare_loss_weights(sigmas: torch.Tensor, flow_weighting_scheme: str = "none") -> torch.Tensor:
    """utils/diffusion.py:117-130 -> diffusers compute_loss_weighting_for_sd3."""
    if flow_weighting_scheme == "sigma_sqrt":
        return (sigmas ** -2.0).float()
    if flow_weighting_scheme == "cosmap":
        bot = 1 - 2 * sigmas + 2 * sigmas ** 2
        return 2 / (math.pi * bot)
    return torch.ones_like(sigmas)


def expand_tensor_dims(t: torch.Tensor, ndim: int) -> torch.Tensor:
    """utils/torch.py:219-221."""
    while t.ndim < ndim:
        t = t.unsqueeze(-1)
    return t


class SFTTrainStep:
    """One optimizer step = ``gradient_accumulation_steps`` micro-steps of forward/loss/backward, then
    all-reduce (DDP) + clip + AdamW on the flat LoRA buffers.

    ``use_cuda_graph=True`` captures prologue + forward + loss + backward of a micro-step (≈1.6k kernel launches) into
    one CUDA graph per input shape: the reference step is launch/host-bound at B=1 (SURVEY §3.2), and so is any
    per-kernel Python dispatch; replaying a graph removes the host from the critical path.  Inputs are copied into static
    device buffers; sigma / noise / first-frame decisions are drawn outside the graph with the same torch calls as the
    reference and handed over through those buffers."""

    def __init__(self, transformer: B200LTXTransformer, spec: Optional[LTXVideoModelSpecification] = None, *,
                 lr: float = 5e-5, beta1: float = 0.9, beta2: float = 0.99, weight_decay: float = 1e-4,
                 eps: float = 1e-8, max_grad_norm: float = 1.0, gradient_accumulation_steps: int = 1,
                 flow_weighting_scheme: str = "logit_normal", flow_logit_mean: float = 0.0,
                 flow_logit_std: float = 1.0, flow_mode_scale: float = 1.29, seed: int = 42,
                 process_group=None, use_cuda_graph: bool = False, lr_scheduler: str = "constant",
                 lr_warmup_steps: int = 0, train_steps: Optional[int] = None, lr_num_cycles: float = 1,
                 lr_power: float = 1.0, ddp_chunks: int = 4):
        self.transformer = transformer
        if spec is None:
            from .wan import B200WanTransformer, WanModelSpecification
            spec = (WanModelSpecification if isinstance(transformer, B200WanTransformer)
                    else LTXVideoModelSpecification)(transformer.cfg)
        self.spec = spec
        self.scheduler = FlowMatchSchedulerTable()
        self.lr, self.beta1, self.beta2, self.wd, self.eps = lr, beta1, beta2, weight_decay, eps
        self.max_grad_norm = max_grad_norm
        # LambdaLR semantics (finetrainers/optimizer.py:191-229): optimizer step k (1-based) runs at lr * factor(k - 1)
        self._lr_factor = lr_factor_fn(lr_scheduler, num_warmup_steps=lr_warmup_steps, num_training_steps=train_steps,
                                       num_cycles=lr_num_cycles, power=lr_power, lr_init=lr)
        self.last_lr = lr * self._lr_factor(0)
        self.grad_accum = gradient_accumulation_steps
        self.scheme = flow_weighting_scheme
        self.flow_logit_mean, self.flow_logit_std, self.flow_mode_scale = flow_logit_mean, flow_logit_std, flow_mode_scale
        if not transformer._prepared:
            transformer.prepare()
        dev = transformer.proj_in.weight.device
        self.device = dev
        self.generator = torch.Generator(device=dev).manual_seed(seed)
        self.scheduler_sigmas = self.scheduler.sigmas.to(dev)
        n = transformer.lora_flat.numel()
        self.fsdp = getattr(transformer, "_fsdp", None)
        if self.fsdp is not None:
            # FSDP-2: optimizer state only for this rank's 1/W slice of the flat trainable buffer (fsdp.ShardedFlatOptimizer)
            from .fsdp import ShardedFlatOptimizer
            self.sharded_opt = ShardedFlatOptimizer(transformer.lora_flat, self.fsdp.group)
            self.exp_avg, self.exp_avg_sq = self.sharded_opt.exp_avg, self.sharded_opt.exp_avg_sq
            process_group = self.fsdp.group
            use_cuda_graph = False  # the step interleaves NCCL all-gathers on a second stream: launched eagerly
        else:
            self.exp_avg = torch.zeros(n, dtype=torch.float32, device=dev)
            self.exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=dev)
        self.sumsq = torch.zeros(1, dtype=torch.float32, device=dev)
        self.loss_buf = torch.zeros(1, dtype=torch.float32, device=dev)
        self.loss_acc = torch.zeros(1, dtype=torch.float32, device=dev)
        self.partial = torch.zeros(1024, dtype=torch.float32, device=dev)
        self.metrics = torch.zeros(3, dtype=torch.float32, device=dev)
        self.opt_step = 0
        self.micro = 0
        self.pg = process_group
        self.world = torch.distributed.get_world_size(process_group) if (
            torch.distributed.is_available() and torch.distributed.is_initialized()) else 1
        self.use_cuda_graph = use_cuda_graph
        # DDP exchange overlap: backward is cut into `ddp_chunks` block ranges; as soon as a range's adapter gradients are
        # final (its batched dA/dB GEMMs ran) their slice of the flat buffer is all-reduced on NCCL's stream while the
        # next range is still in backward - the role of replicate(bucket_cap_mb=100)'s bucketed reducer (ptd.py:462-463)
        nl = transformer.cfg.num_layers
        n_chunks = min(ddp_chunks, nl) if (self.world > 1 and self.fsdp is None) else 1
        self._segments = [(nl * c // n_chunks, nl * (c + 1) // n_chunks) for c in range(n_chunks)][::-1]  # top blocks first
        self._pending_ar = []
        self._comm = torch.cuda.Stream(dev) if (n_chunks > 1 and dev.type == "cuda") else None
        self._static: Dict[tuple, Dict[str, torch.Tensor]] = {}
        self._graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}
        self._eager_runs: Dict[tuple, int] = {}
        # every graph is captured into one memory pool, so their temporaries do not multiply with shapes x segments.  They
        # replay one at a time on one stream, and what a captured segment allocates is read at most by the later segments
        # of the same step (the key bias the backward reads), which replay right after it
        self._pool = None
        self._graph_gen = transformer.workspace_generation  # the training arena the graphs in _graphs point into

    # -- static buffers per input shape ---------------------------------------------------------------------------
    def _buffers(self, B, C, Fr, Hh, Ww, L, Cc, from_moments: bool = False, image=()):
        """Static buffers per (input shape, input kind): a moments input and a latents input never share buffers or a
        graph, whatever their shapes.  ``image``: (image tokens, image width, mask channels) of an image-to-video input,
        part of the key, so a graph captured for one image context shape never replays for another."""
        key = (B, C, Fr, Hh, Ww, L, Cc, from_moments) + tuple(image)
        st = self._static.get(key)
        if st is None:
            dev = self.device
            S, Cp = self.spec.packed_shape(C, Fr, Hh, Ww)
            bf = dict(dtype=torch.bfloat16, device=dev)
            if from_moments:  # VAE moments [mean | logvar] and the posterior draw eps
                inp = {"moments": torch.zeros(B, 2 * C, Fr, Hh, Ww, **bf), "eps": torch.zeros(B, C, Fr, Hh, Ww, **bf)}
            else:
                inp = {"latents": torch.zeros(B, C, Fr, Hh, Ww, **bf)}
            st = {
                **inp, "noise": torch.zeros(B, C, Fr, Hh, Ww, **bf),
                "mean": torch.zeros(B, C, dtype=torch.float32, device=dev),
                "std": torch.ones(B, C, dtype=torch.float32, device=dev),
                "ehs": torch.zeros(B, L, Cc, **bf), "mask": torch.ones(B, L, dtype=torch.float32, device=dev),
                "sig": torch.zeros(B, dtype=torch.float32, device=dev),
                "sig_ff": torch.zeros(B, dtype=torch.float32, device=dev),
                "x_t": torch.zeros(B, S, Cp, **bf), "target": torch.zeros(B, S, Cp, **bf),
                "dpred": torch.zeros(B, S, Cp, **bf),
            }
            if image:  # the condition moments, its mask, the image embeddings; x_t is the wider transformer input
                Li, Di, Cm = image
                st.update(cond=torch.zeros(B, 2 * C, Fr, Hh, Ww, **bf), cond_mask=torch.zeros(B, Cm, Fr, Hh, Ww, **bf),
                          img=torch.zeros(B, Li, Di, **bf),
                          x_t=torch.zeros(B, S, self.spec.packed_shape(2 * C + Cm, Fr, Hh, Ww)[1], **bf))
            self._static[key] = st
        return key, st

    def _body_front(self, key, st):
        """prologue + forward + loss + head backward on the static buffers (capturable: no host sync, no data-dependent
        Python control flow)."""
        B = key[0]
        tr = self.transformer
        inputs = self.spec.step_inputs(key, st)                               # the spec's prologue
        weights = prepare_loss_weights(st["sig"], self.scheme).contiguous()   # trainer.py:463-470
        pred = tr._forward_impl(*inputs)
        ops.loss_mse(pred, st["target"], weights, 1.0 / self.grad_accum, self.loss_buf, st["dpred"], self.partial, B,
                     pred.shape[1] * pred.shape[2])
        tr._backward_head(st["dpred"])
        self.loss_acc += self.loss_buf

    def _body_segment(self, key, st, seg: int, segments):
        """Segment `seg` of the step: (front part for seg 0) + backward through its block range + that range's adapter
        gradients."""
        tr = self.transformer
        lo, hi = segments[seg]
        if seg == 0:
            self._body_front(key, st)
        tr._backward_blocks(hi - 1, lo)
        tr._backward_tail(lo, hi)
        if seg == len(segments) - 1 and tr._fsdp is not None:
            tr._fsdp.end_backward()

    def _drop_stale_graphs(self):
        """The model's training arena grew (a larger shape's first step): every graph, of every shape and segment,
        holds pointers into the freed arena, so all are dropped and re-warmed and re-captured like a new shape's."""
        gen = self.transformer.workspace_generation
        if gen != self._graph_gen:
            self._graphs.clear()
            self._eager_runs.clear()
            self._pool = None
            self._graph_gen = gen

    def _run_segment(self, key, st, seg: int, segments):
        """Eager, or one CUDA-graph replay per (shape, segmentation, segment)."""
        if not self.use_cuda_graph:
            self._body_segment(key, st, seg, segments)
            return
        self._drop_stale_graphs()
        gkey = (key, len(segments), seg)
        g = self._graphs.get(gkey)
        if g is None:
            n = self._eager_runs.get(gkey, 0)
            if n < 2:  # warm-up eagerly (lazy one-time work: rope tables, func attributes, workspace allocation)
                self._body_segment(key, st, seg, segments)
                self._drop_stale_graphs()  # this run grew the arena: it is the first warm-up in the new one
                self._eager_runs[gkey] = n + 1
                return
            torch.cuda.synchronize()
            if self._pool is None:
                self._pool = torch.cuda.graph_pool_handle()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self._pool):
                self._body_segment(key, st, seg, segments)
            self._graphs[gkey] = g
        g.replay()

    def _allreduce_range_async(self, lo: int, hi: int):
        """Average blocks [lo, hi)'s slice of the flat gradient buffer across ranks on NCCL's stream, ordered after the
        work issued so far on the compute stream."""
        tr = self.transformer
        sl = tr.lora_grad_flat[lo * tr._per_blk:hi * tr._per_blk]
        ev = torch.cuda.Event()
        ev.record()
        with torch.cuda.stream(self._comm):
            self._comm.wait_event(ev)
            self._pending_ar.append(allreduce_flat_grads(sl, self.pg, async_op=True))

    # -- forward + loss + backward of one micro-batch (trainer.py:436-483) ---------------------------------------
    @torch.no_grad()
    def micro_step(self, condition_model_conditions: Dict[str, torch.Tensor],
                   latent_model_conditions: Dict[str, torch.Tensor], sigmas: Optional[torch.Tensor] = None,
                   noise: Optional[torch.Tensor] = None, compute_posterior: bool = True,
                   posterior_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``compute_posterior=False`` (the reference's precomputed path): ``latents`` holds VAE moments
        ``[B, 2C, F, H, W]``; the latent is sampled from them in the prologue kernel with eps drawn from ``self.generator``
        after the sigmas and before the noise, or taken from ``posterior_noise`` when given."""
        import random as _random
        latents = latent_model_conditions["latents"]
        compute_posterior = compute_posterior and not self.spec.latents_are_moments  # Wan: always moments
        if compute_posterior:
            B, C, Fr, Hh, Ww = latents.shape
        else:
            # the latent's channels are the prediction's: an image-to-video model's input is wider (x_t, mask, condition)
            C = moments_channels(latents.shape, self.transformer.cfg.out_channels)
            B, _, Fr, Hh, Ww = latents.shape
        ehs = condition_model_conditions["encoder_hidden_states"]
        mask = condition_model_conditions.get("encoder_attention_mask")
        image = self.spec.image_inputs(latent_model_conditions, latents.shape, self.transformer.cfg)
        ikey = (image[2].shape[1], image[2].shape[2], image[1].shape[1]) if image is not None else ()
        key, st = self._buffers(B, C, Fr, Hh, Ww, ehs.shape[1], ehs.shape[2], not compute_posterior, ikey)
        if not self.transformer._prepared:
            self.transformer.prepare()
        # ---- host-side sampling, identical calls to the reference (utils/diffusion.py:84-114, base_specification.py:296-305)
        if sigmas is None:
            sigmas = prepare_sigmas(self.scheduler, self.scheduler_sigmas, B, self.scheduler.config.num_train_timesteps,
                                    self.scheme, self.flow_logit_mean, self.flow_logit_std, self.flow_mode_scale,
                                    self.device, self.generator)
        st["sig"].copy_(sigmas.reshape(B), non_blocking=True)
        if compute_posterior:
            st["latents"].copy_(latents, non_blocking=True)
        else:
            st["moments"].copy_(latents, non_blocking=True)
            if posterior_noise is None:  # models/utils.py:23-29: drawn before the flow-match noise
                st["eps"].normal_(generator=self.generator)
            else:
                st["eps"].copy_(posterior_noise, non_blocking=True)
        if noise is None:
            st["noise"].normal_(generator=self.generator)
        else:
            st["noise"].copy_(noise, non_blocking=True)
        if "latents_mean" in latent_model_conditions:
            st["mean"].copy_(latent_model_conditions["latents_mean"].reshape(B, C), non_blocking=True)
            st["std"].copy_(latent_model_conditions["latents_std"].reshape(B, C), non_blocking=True)
        else:  # already-normalised latents: do not keep a previous batch's statistics in the static buffers
            st["mean"].zero_()
            st["std"].fill_(1.0)
        st["ehs"].copy_(ehs, non_blocking=True)
        if image is not None:  # copy_ also makes the reference's transposed mask view dense
            for name, t in zip(("cond", "cond_mask", "img"), image):
                st[name].copy_(t, non_blocking=True)
        if mask is not None:
            st["mask"].copy_(mask, non_blocking=True)
        else:
            st["mask"].fill_(1.0)
        if _random.random() < self.spec.first_frame_conditioning_p:
            ff = torch.rand(B, device=self.device, generator=self.generator) * st["sig"]
            st["sig_ff"].copy_(torch.clamp(ff, max=self.spec.min_first_frame_sigma))
        else:
            st["sig_ff"].copy_(st["sig"])  # first latent frame uses the same sigma: identical to the plain branch
        # ---- the step body: eager, or CUDA-graph replays.  On the micro-step that completes an accumulation window under
        # DDP the backward runs in block-range segments with each range's gradient all-reduce issued behind it.
        last_micro = (self.micro + 1) % self.grad_accum == 0
        nl = self.transformer.cfg.num_layers
        segments = self._segments if (len(self._segments) > 1 and last_micro) else [(0, nl)]
        for seg in range(len(segments)):
            self._run_segment(key, st, seg, segments)
            if len(segments) > 1:
                self._allreduce_range_async(*segments[seg])
        self.micro += 1
        return self.loss_buf

    # -- clip + AdamW (+ DDP all-reduce) (trainer.py:486-520) ---------------------------------------------------
    @torch.no_grad()
    def optimizer_step(self, sync_metrics: bool = False):
        tr = self.transformer
        g = tr.lora_grad_flat
        self.opt_step += 1
        self.last_lr = self.lr * self._lr_factor(self.opt_step - 1)
        if self.fsdp is not None:
            # FSDP-2: fp32 reduce-scatter(AVG) -> global-norm clip + AdamW on the local slice -> in-place all-gather
            def sumsq_fn(gs):
                self.sumsq.zero_()
                ops.sumsq(gs, gs.numel(), self.sumsq, self.partial)
                return self.sumsq

            def update_fn(p, gs, m, v, ss):
                ops.adamw_clip(p, gs, m, v, gs.numel(), ss, self.max_grad_norm, self.last_lr, self.beta1, self.beta2,
                               self.eps, self.wd, self.opt_step, 1.0)

            self.sharded_opt.step(g, sumsq_fn, update_fn)
        else:
            if self._pending_ar:
                for w in self._pending_ar:   # the chunked exchange was issued behind each backward segment
                    if w is not None:
                        w.wait()
                self._pending_ar.clear()
            elif self.world > 1:
                # DDP: average the flat fp32 gradient buffer in place over NVLink (ptd.py:462-463 replicate(bucket_cap_mb=100))
                allreduce_flat_grads(g, self.pg)
            self.sumsq.zero_()
            ops.sumsq(g, g.numel(), self.sumsq, self.partial)
            ops.adamw_clip(tr.lora_flat, g, self.exp_avg, self.exp_avg_sq, g.numel(), self.sumsq, self.max_grad_norm,
                           self.last_lr, self.beta1, self.beta2, self.eps, self.wd, self.opt_step, 1.0)
        self.metrics[0:1] = self.sumsq.sqrt()
        self.metrics[1:2] = self.loss_acc
        self.metrics[2:3] = self.loss_acc
        self.loss_acc.zero_()
        self.micro = 0
        if not sync_metrics:
            return None
        return fused_step_metrics(self.metrics[0], self.metrics[1], self.pg)

    @torch.no_grad()
    def clip_accumulated(self):
        """The reference clips after EVERY micro-step's backward (``trainer.py:486-493`` sits outside the
        ``step % gradient_accumulation_steps`` test), so inside an accumulation window the PARTIALLY accumulated gradient is
        rescaled to ``max_grad_norm`` before the next micro-step adds to it.  Under DDP / FSDP-2 the reference's gradient
        is already averaged over ranks at that point; the buffer holds (previous, identical on every rank) + (this rank's
        micro-gradient), so averaging the whole buffer gives exactly that."""
        g = self.transformer.lora_grad_flat
        if self._pending_ar:
            for w in self._pending_ar:
                if w is not None:
                    w.wait()
            self._pending_ar.clear()
        elif self.world > 1:
            allreduce_flat_grads(g, self.pg)
        if self.max_grad_norm is not None and self.max_grad_norm > 0:
            self.sumsq.zero_()
            ops.sumsq(g, g.numel(), self.sumsq, self.partial)
            g.mul_(torch.clamp(self.max_grad_norm / (self.sumsq.sqrt() + 1e-6), max=1.0))

    def train_step(self, condition_model_conditions, latent_model_conditions, sigmas=None, noise=None,
                   sync_metrics=False, compute_posterior=True, posterior_noise=None):
        self.micro_step(condition_model_conditions, latent_model_conditions, sigmas, noise, compute_posterior,
                        posterior_noise)
        if self.micro % self.grad_accum == 0:
            return self.optimizer_step(sync_metrics)
        self.clip_accumulated()
        return None
