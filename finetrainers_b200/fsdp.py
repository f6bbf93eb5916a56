"""FSDP-2 for the H100 engine: what ``apply_fsdp2`` / ``fully_shard`` do in the reference
(``finetrainers/parallel/ptd.py:466-499``, call site ``trainer/sft_trainer/trainer.py:163-184``:
``fully_shard`` per transformer block + the root module, ``MixedPrecisionPolicy(param_dtype=bf16, reduce_dtype=fp32)``,
``reshard_after_forward`` for every block but the last), rebuilt for a model whose parameters already live in flat buffers.

Sharding unit = one DiT block's flat bf16 buffer (``B200LTXTransformer._blk_flat[l]``, 134 MB at LTX-2B) or the root
buffer (embeds / head / the stacked text-side K/V weights).  Rank ``r`` of ``W`` permanently stores elements
``[r*n/W, (r+1)*n/W)`` of every unit.  A unit is materialised by ONE ``all_gather_into_tensor`` into one of two
full-size *slots* (block ``l`` always uses slot ``l % 2``, so the kernels' weight views are fixed at set-up time):

    forward :  AG(root) AG(0) AG(1) | wait 0, compute 0, release -> AG(2) | wait 1, compute 1, release -> AG(3) | ...
    backward:  blocks nl-1, nl-2 are still resident (the last block is not resharded, as in the reference);
               wait l, backward l, release -> AG(l-2)

The all-gathers run on a communication stream one block ahead of compute (134 MB over NVLink 5 at ~700 GB/s is
~0.2 ms against ~0.5 ms of block compute), ordered against compute with CUDA events; nothing is copied or cast
(parameters are stored in the compute dtype).  Trainable state is sharded ZeRO-style on the flat fp32 LoRA buffers:
gradients are reduce-scattered in fp32 (AVG), each rank clips with the global norm and runs AdamW on its 1/W slice
(optimizer state exists only for that slice) and the updated fp32 masters are all-gathered in place.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import torch
import torch.distributed as dist


def _backend(group) -> str:
    return dist.get_backend(group)


def shard_bounds(numel: int, rank: int, world: int):
    """[lo, hi) of rank's slice of a flat unit whose length divides evenly (units are padded to FLAT_ALIGN)."""
    if numel % world:
        raise ValueError(f"flat unit of {numel} elements does not split evenly over {world} ranks")
    n = numel // world
    return rank * n, (rank + 1) * n


def all_gather_flat(full: torch.Tensor, shard: torch.Tensor, group=None, async_op: bool = False):
    """full[r*n:(r+1)*n] <- rank r's shard (in-place form allowed: ``shard`` may alias its slice of ``full``)."""
    return dist.all_gather_into_tensor(full, shard, group=group, async_op=async_op)


def reduce_scatter_avg(shard_out: torch.Tensor, full: torch.Tensor, group=None):
    """shard_out <- mean over ranks of full[r*n:(r+1)*n] (fp32 reduce, ``reduce_dtype=torch.float32`` in the reference).
    gloo has no reduce-scatter: all-reduce then slice (CPU tests only)."""
    world = dist.get_world_size(group)
    if _backend(group) == "nccl":
        dist.reduce_scatter_tensor(shard_out, full, op=dist.ReduceOp.AVG, group=group)
    else:
        tmp = full.clone()
        dist.all_reduce(tmp, op=dist.ReduceOp.SUM, group=group)
        lo, hi = shard_bounds(full.numel(), dist.get_rank(group), world)
        shard_out.copy_(tmp[lo:hi] / world)
    return shard_out


class UnitSlots:
    """The slot schedule shared by FSDP-2 and layerwise casting: ``n`` units take turns in a few full-size slots (unit
    ``u`` always in slot ``slot_of(u)``, ``u % n_slots`` by default, so the kernels' weight views are fixed at set-up
    time), and a unit is materialised by ``fill(unit, slot)`` on a side stream one unit ahead of compute.  ``fill`` runs
    with the side stream current and returns an object whose ``wait()`` makes the then-current stream wait for it (a
    collective's work handle, an event) or ``None`` (synchronous, CPU).

    ``fork=True`` additionally makes every fill wait for all work issued so far on the current stream: a fill then never
    depends on a previous graph replay or step, which is what CUDA-graph capture of the side stream needs."""

    def __init__(self, n: int, slots: List[torch.Tensor], fill: Callable, stream=None, fork: bool = False,
                 slot_of: Optional[Callable[[int], int]] = None):
        self.n = n
        self.slots = slots
        self.n_slots = len(slots)
        self.fill = fill
        self.comm = stream
        self.cuda = stream is not None
        self.fork = fork
        self._slot_of = slot_of
        self.resident = [-1] * self.n_slots        # unit currently (being) materialised into each slot
        self.work = [None] * self.n_slots          # outstanding fill of each slot
        self.free_ev = [None] * self.n_slots       # compute-stream event: the slot's previous tenant is no longer read
        self.gathers = 0                           # number of fills (tests / bench)

    def slot_of(self, unit: int) -> int:
        return self._slot_of(unit) if self._slot_of is not None else unit % self.n_slots

    def slot_tensor(self, unit: int) -> torch.Tensor:
        return self.slots[self.slot_of(unit)]

    def reset(self) -> None:
        """Forget every slot's tenant: the next wait() of any unit fills it again."""
        self.resident = [-1] * self.n_slots
        self.work = [None] * self.n_slots
        self.free_ev = [None] * self.n_slots

    def prefetch(self, unit: int) -> None:
        """Start filling ``unit``'s slot (no-op if it is already resident or in flight)."""
        if unit < 0 or unit >= self.n:
            return
        s = self.slot_of(unit)
        if self.resident[s] == unit:
            return
        self.gathers += 1
        if self.cuda:
            fork_ev = None
            if self.fork:
                fork_ev = torch.cuda.Event()
                fork_ev.record(torch.cuda.current_stream())
            with torch.cuda.stream(self.comm):
                if self.free_ev[s] is not None:
                    self.comm.wait_event(self.free_ev[s])   # the previous tenant's last reader has been issued and finishes first
                if fork_ev is not None:
                    self.comm.wait_event(fork_ev)
                self.work[s] = self.fill(unit, self.slots[s])
        else:
            self.fill(unit, self.slots[s])
        self.resident[s] = unit

    def wait(self, unit: int) -> torch.Tensor:
        """Make the current stream wait until ``unit`` is resident; returns its slot."""
        s = self.slot_of(unit)
        if self.resident[s] != unit:
            self.prefetch(unit)
        if self.cuda and self.work[s] is not None:
            self.work[s].wait()            # current stream waits on the fill's completion
            self.work[s] = None
        return self.slots[s]

    def release(self, unit: int, then_prefetch: int = -1) -> None:
        """The current stream is done reading ``unit``: its slot may be overwritten (by ``then_prefetch``)."""
        s = self.slot_of(unit)
        if self.cuda:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            self.free_ev[s] = ev
        if then_prefetch >= 0 and self.slot_of(then_prefetch) == s:
            self.prefetch(then_prefetch)


class ShardedUnits(UnitSlots):
    """Shards + slots + the prefetch schedule for a list of equally sized flat units (the DiT blocks); a slot is filled
    by one all-gather of the unit's shards."""

    def __init__(self, flats: List[torch.Tensor], group=None, n_slots: int = 2, on_cuda: Optional[bool] = None):
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.numel = flats[0].numel()
        assert all(f.numel() == self.numel for f in flats)
        lo, hi = shard_bounds(self.numel, self.rank, self.world)
        self.shards = [f[lo:hi].clone() for f in flats]
        dev, dt = flats[0].device, flats[0].dtype
        slots = [torch.empty(self.numel, dtype=dt, device=dev) for _ in range(min(n_slots, len(flats)))]
        cuda = flats[0].is_cuda if on_cuda is None else on_cuda
        super().__init__(len(flats), slots, self._gather, torch.cuda.Stream(dev) if cuda else None)

    def _gather(self, unit: int, slot: torch.Tensor):
        return all_gather_flat(slot, self.shards[unit], self.group, async_op=self.cuda)

    def gather_full(self, unit: int) -> torch.Tensor:
        """A private full copy of ``unit`` (state_dict / export paths; not used by the step)."""
        out = torch.empty(self.numel, dtype=self.slots[0].dtype, device=self.slots[0].device)
        all_gather_flat(out, self.shards[unit], self.group)
        return out


class ShardedFlatOptimizer:
    """ZeRO-style step on ONE flat fp32 parameter buffer: reduce-scatter(AVG) the flat gradient, global-norm clip, update
    the local slice with ``update_fn(p, g, m, v, sumsq_tensor, step)`` and all-gather the parameters in place."""

    def __init__(self, params: torch.Tensor, group=None):
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.numel = params.numel()
        self.lo, self.hi = shard_bounds(self.numel, self.rank, self.world)
        n = self.hi - self.lo
        self.params = params
        self.g_shard = torch.zeros(n, dtype=torch.float32, device=params.device)
        self.exp_avg = torch.zeros(n, dtype=torch.float32, device=params.device)
        self.exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=params.device)

    def step(self, grad_flat: torch.Tensor, sumsq_fn: Callable[[torch.Tensor], torch.Tensor],
             update_fn: Callable[..., None]) -> torch.Tensor:
        """-> global sum of squares of the averaged gradient (a 1-element tensor, identical on every rank)."""
        reduce_scatter_avg(self.g_shard, grad_flat, self.group)
        sumsq = sumsq_fn(self.g_shard)
        dist.all_reduce(sumsq, op=dist.ReduceOp.SUM, group=self.group)
        update_fn(self.params[self.lo:self.hi], self.g_shard, self.exp_avg, self.exp_avg_sq, sumsq)
        all_gather_flat(self.params, self.params[self.lo:self.hi], self.group)
        grad_flat.zero_()
        return sumsq


class FSDPState:
    """Attached to a prepared ``B200LTXTransformer`` by ``B200ParallelBackend.apply_fsdp2``."""

    def __init__(self, model, group=None):
        if getattr(model, "_lw_cfg", None) is not None:
            # the reference's FSDP path casts the whole transformer to one dtype (trainer.py:132-133)
            raise NotImplementedError("FSDP-2 of a model with layerwise fp8 weight storage is not built; "
                                      "use DDP (apply_ddp) with layerwise casting")
        if not getattr(model, "_prepared", False):
            model.prepare()
        self.model = model
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        # replicas must agree before they are cut into shards
        for f in list(model._blk_flat) + [model._root_flat]:
            dist.broadcast(f, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        if model.lora_rank:
            dist.broadcast(model.lora_flat, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        self.blocks = ShardedUnits(model._blk_flat, group)
        self.root = ShardedUnits([model._root_flat], group, n_slots=1)
        self.full_bytes_per_block = model._blk_flat[0].numel() * model._blk_flat[0].element_size()
        model._rebind_flat_storage([self.blocks.slot_tensor(l) for l in range(len(model._blk_flat))], self.root.slots[0])
        self.nl = len(model.transformer_blocks)

    # ---- schedule hooks called by the model --------------------------------------------------------------------
    def begin_forward(self):
        self.root.prefetch(0)
        self.blocks.prefetch(0)
        self.blocks.prefetch(1)
        self.root.wait(0)

    def pre_block_forward(self, l: int):
        self.blocks.wait(l)

    def post_block_forward(self, l: int):
        nxt = l + self.blocks.n_slots
        if nxt < self.nl:                       # the last n_slots blocks stay resident for the start of backward
            self.blocks.release(l, nxt)

    def begin_backward_range(self, l_hi: int, l_lo: int):
        pass  # pre_block_backward gathers any block of the range that is not resident

    def pre_block_backward(self, l: int):
        self.blocks.wait(l)

    def post_block_backward(self, l: int):
        self.blocks.release(l, l - self.blocks.n_slots)

    def end_backward(self):
        # root: resharded after backward (its slot is rewritten by the next step's all-gather); blocks 0/1 are resident and
        # are exactly what the next forward starts with
        if self.root.cuda:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            self.root.free_ev[0] = ev
        self.root.resident[0] = -1

    def local_param_bytes(self) -> int:
        b = sum(s.numel() * s.element_size() for s in self.blocks.shards)
        return b + self.root.shards[0].numel() * self.root.shards[0].element_size()

    def full_state_dict(self):
        """Full (unsharded) base-weight tensors keyed like ``state_dict()``, gathered unit by unit (export / tests)."""
        from .layerwise import carve  # layerwise imports this module
        m = self.model
        out = {}
        names = {id(p): n for n, p in m.named_parameters()}
        for l, blk in enumerate(m.transformer_blocks):
            views = carve(self.blocks.gather_full(l), m._block_specs(), 8)
            out.update((names[id(prm)], seg.clone()) for prm, seg in m._segments(views, m._block_params(blk)))
        views = carve(self.root.gather_full(0), m._root_specs(), 8)
        out.update((names[id(prm)], seg.clone()) for prm, seg in m._segments(views, m._root_params()))
        for n, p in m.named_parameters():
            if "lora_" in n:
                out[n] = p.detach().clone()
        return out
