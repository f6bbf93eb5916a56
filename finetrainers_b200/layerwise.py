"""Layerwise fp8 weight storage for LoRA training: ``--layerwise_upcasting_modules transformer``
(``finetrainers/trainer/sft_trainer/trainer.py:108-118``, ``finetrainers/args.py:149-156,392-395,743-756``).

The reference calls diffusers' ``apply_layerwise_casting`` on the transformer before ``add_adapter``: every
``nn.Linear`` and Conv layer whose module FQN no skip pattern matches (``re.search``; a match skips the module's whole subtree) stores
its weight and bias in fp8, and a hook upcasts them to the compute dtype around that layer's forward.  This engine keeps
the same stored state (the module's cast parameters are fp8 tensors) and computes with the same values, bf16(fp8(W)),
but materialises the bf16 copies itself: the cast pieces of a DiT block live in one fp8 flat buffer, and one upcast
kernel per block fills one of two bf16 *slots* one block ahead of compute on a side stream (``fsdp.UnitSlots``, the
schedule FSDP-2 fills with all-gathers).  The upcast is exact, so the result is bit-identical to a bf16 model whose cast
weights were rounded through fp8.
"""
from __future__ import annotations

import math
import re
from typing import Dict, Iterable, List, NamedTuple, Optional, Sequence, Tuple

import torch

from . import ops
from .fsdp import UnitSlots

STORAGE_DTYPES = (torch.float8_e4m3fn, torch.float8_e5m2)

# finetrainers' two default skip lists: the BaseArgs dataclass default (args.py:395) and the train.py CLI default
# (args.py:751-754), which does not skip time_embed
DEFAULT_SKIP_MODULES_PATTERN = ("patch_embed", "pos_embed", "x_embedder", "context_embedder", "time_embed", "^proj_in$",
                                "^proj_out$", "norm")
CLI_SKIP_MODULES_PATTERN = ("patch_embed", "pos_embed", "x_embedder", "context_embedder", "^proj_in$", "^proj_out$",
                            "norm")


def cast_linear_names(root: torch.nn.Module, patterns: Sequence[str], linear_types) -> List[str]:
    """FQNs of the layers the walk casts: ``named_children()`` from the root with dotted FQNs; a module whose FQN (the
    root's is ``""``) matches a pattern under ``re.search`` is skipped with its subtree; a layer of ``linear_types`` (the
    engine's stand-ins for diffusers' ``nn.Linear`` and Conv layers) is cast and not descended into."""
    out: List[str] = []

    def walk(mod, fqn):
        if any(re.search(p, fqn) for p in patterns):
            return
        if isinstance(mod, linear_types):
            out.append(fqn)
            return
        for name, child in mod.named_children():
            walk(child, f"{fqn}.{name}" if fqn else name)

    walk(root, "")
    return out


def carve(flat: torch.Tensor, specs: Iterable[Tuple[str, tuple]], align: int):
    """Views of ``specs`` in ``flat``, each starting at a multiple of ``align`` elements: 8 in the resident flat units
    (16 bytes in bf16, as TMA requires), 16 in fp8 storage (16 bytes) and in the bf16 slots carved with its offsets."""
    out, o = {}, 0
    for key, shape in specs:
        n = math.prod(shape)
        out[key] = flat[o:o + n].view(shape)
        o += (n + align - 1) // align * align
    return out


def carved_numel(specs, align: int) -> int:
    return sum((math.prod(shape) + align - 1) // align * align for _, shape in specs)


def numel16(specs) -> int:
    """Elements of the fp8 storage of ``specs``, and of the bf16 slot carved with the same offsets."""
    return carved_numel(specs, 16)


class _EventWork:
    """Completion of work issued on the side stream: ``wait()`` orders the current stream after it."""
    __slots__ = ("ev",)

    def __init__(self, stream):
        self.ev = torch.cuda.Event()
        self.ev.record(stream)

    def wait(self):
        torch.cuda.current_stream().wait_event(self.ev)


class Stacked(NamedTuple):
    """One stacked root piece of every block that streams through the block slots when cast (the text-side
    ``[Wk2;Wv2]``, the image-side ``[Wk3;Wv3]``): its fp8 storage, its block-range chunks and their views in the slots."""
    src: Tuple[torch.Tensor, torch.Tensor]               # (W fp8 [nl, 2d, d], b fp8 [nl, 2d])
    chunks: List[Tuple[int, int]]                        # [(l0, l1)] block ranges
    views: List[Tuple[torch.Tensor, torch.Tensor]]       # per chunk: (W view [nb, 2d, d], b view [nb, 2d]) in its slot


class LayerwiseSchedule:
    """Upcast schedule of one prepared model (built by ``B200LTXTransformer.prepare``); the model calls the same hooks it
    calls for FSDP-2.

    Units of the block slots: blocks ``0 .. nl-1`` (block ``l`` in slot ``l % 2``), then the chunks of the stacked
    pieces ``stacked`` in order (the text-side ``[Wk2;Wv2]`` of all blocks, then the image-side ``[Wk3;Wv3]``; chunk
    ``g`` of that sequence in slot ``g % 2``), which stream through the block slots before block 0 is materialised, so
    that they never need a persistent bf16 copy.

    Every forward materialises from storage (the root slot and every block), and a backward block range that does not
    directly follow the forward in the same launch sequence materialises its blocks again: no CUDA-graph replay and no
    eager segment reads a slot filled by another replay or step, and every side-stream fill is waited for inside the
    graph or segment that issued it.  ``load_state_dict``, ``.to()`` and DDP segment graphs are correct by construction."""

    def __init__(self, nl: int, blk_fp8: List[torch.Tensor], slots: List[torch.Tensor], root_fp8: torch.Tensor,
                 root_slot: torch.Tensor, stacked: Optional[Dict[str, Stacked]] = None, on_cuda: bool = True):
        self.nl = nl
        self.blk_fp8 = blk_fp8            # per block: fp8 flat (None when nothing of that block is cast)
        self.root_fp8, self.root_slot = root_fp8, root_slot
        self.stacked = dict(stacked or {})  # "kv2" / "kv3" -> Stacked, in streaming order
        # the streamed chunks in order: (stacked key, chunk index); unit nl + g is the g-th of them
        self._chunk_units = [(k, c) for k, st in self.stacked.items() for c in range(len(st.chunks))]
        self._first = {}
        for g, (k, c) in enumerate(self._chunk_units):
            self._first.setdefault(k, g)
        self.upcasts = 0
        stream = torch.cuda.Stream(slots[0].device) if (on_cuda and slots) else None
        nc = len(self._chunk_units)
        ns = max(1, len(slots))
        self.units = UnitSlots(nl + nc, slots, self._fill, stream, fork=True,
                               slot_of=lambda u: (u if u < nl else u - nl) % ns) if slots else None
        self._continues = False           # the next backward block range directly follows a forward
        self.lo = 0

    @property
    def kv2_chunks(self) -> List[Tuple[int, int]]:
        """Block ranges of the text-side ``[Wk2;Wv2]`` chunks ([] when that piece is not cast)."""
        return self.chunks("kv2")

    def chunks(self, key: str) -> List[Tuple[int, int]]:
        st = self.stacked.get(key)
        return list(st.chunks) if st is not None else []

    def _upcast(self, src, dst, n):
        ops.upcast_fp8_bf16(src, dst, n)
        self.upcasts += 1

    def _fill(self, unit: int, slot: torch.Tensor):
        if unit < self.nl:
            f8 = self.blk_fp8[unit]
            if f8 is not None:
                self._upcast(f8, slot, f8.numel())
        else:
            k, c = self._chunk_units[unit - self.nl]
            st = self.stacked[k]
            (l0, l1), (Wv, bv) = st.chunks[c], st.views[c]
            W8, b8 = st.src
            self._upcast(W8[l0:l1], Wv, Wv.numel())
            self._upcast(b8[l0:l1], bv, bv.numel())
        return _EventWork(torch.cuda.current_stream()) if self.units.cuda else None

    def _has_block(self, l: int) -> bool:
        return self.units is not None and self.blk_fp8[l] is not None

    # ---- hooks called by the model ----------------------------------------------------------------------------------
    def begin_forward(self):
        if self.root_slot.numel():  # the slot part is the prefix of the root's fp8 flat (same element offsets)
            self._upcast(self.root_fp8, self.root_slot, self.root_slot.numel())
        if self.units is None:
            return
        self.units.reset()
        # slot s first takes streamed chunk s, or block s when there are fewer chunks than slots
        nc = len(self._chunk_units)
        for s in range(self.units.n_slots):
            self.units.prefetch(self.nl + s if s < nc else s)
        self._continues = True

    def chunk_wait(self, key: str, c: int):
        """Block the current stream until chunk ``c`` of the stacked piece ``key`` is in its slot -> (W, b)."""
        self.units.wait(self.nl + self._first[key] + c)
        return self.stacked[key].views[c]

    def chunk_release(self, key: str, c: int):
        """Chunk ``c`` of ``key`` is no longer read: its slot takes the streamed chunk two further on, or, after the last
        chunk in that slot, the block that owns the slot (block s for slot s)."""
        u = self.nl + self._first[key] + c
        nxt = u + self.units.n_slots
        if nxt >= self.nl + len(self._chunk_units):
            nxt = self.units.slot_of(u)
        self.units.release(u, nxt)

    def pre_block_forward(self, l: int):
        if self._has_block(l):
            self.units.wait(l)

    def post_block_forward(self, l: int):
        if self._has_block(l) and l + self.units.n_slots < self.nl:   # the last blocks stay resident for backward
            self.units.release(l, l + self.units.n_slots)

    def begin_backward_range(self, l_hi: int, l_lo: int):
        """Blocks ``l_hi`` down to ``l_lo`` are about to run backward.  Only the range that directly follows the forward
        keeps what the forward left resident; any other range (a separate DDP segment or graph) fills its own slots."""
        self.lo = l_lo
        if self.units is not None and not (self._continues and l_hi == self.nl - 1):
            self.units.reset()
            for l in range(l_hi, max(l_lo, l_hi - self.units.n_slots + 1) - 1, -1):
                self.units.prefetch(l)
        self._continues = False

    def pre_block_backward(self, l: int):
        # the model also calls this for block l - 1 below the range, for its gate row; scale_shift_table is never cast
        if l >= self.lo and self._has_block(l):
            self.units.wait(l)

    def post_block_backward(self, l: int):
        if self._has_block(l):
            nxt = l - self.units.n_slots
            self.units.release(l, nxt if nxt >= self.lo else -1)

    def end_backward(self):
        pass
