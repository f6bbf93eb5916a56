"""Precomputed latent / condition feed — the step immediately BEFORE the hot path (SURVEY §8f-2).

On-disk format and index arithmetic are the reference's (``finetrainers/data/precomputation.py``):
``{data_type}-{index}.pt`` written with ``torch.save(dict)`` and read with ``torch.load(weights_only=True)``
(``:413-420``); ``PrecomputedDataIterable`` gives rank ``r`` the indices ``r*num_items + i`` and raises ``requires_data``
on its last item (``:319-345``); ``PrecomputedOnceDataIterable`` cycles forever over ``r*per_rank + i`` (``:348-382``).
``ResolutionSampler`` (``data/sampler.py:6-58``) and the collate functions (``models/modeling_utils.py:156-181``) are the
host logic between the iterables and ``ModelSpecification.forward``.

What changes here: the reference deserialises every item ON the training thread straight onto the GPU
(``map_location=torch.device(rank)``: a synchronous ``torch.load`` + pageable H2D per item).  At > 70 k tokens/s a step
is 37 ms, so here a BACKGROUND THREAD runs ``torch.load`` to CPU, stages the tensors in a ring of pinned host buffers
and issues the H2D copy on a side stream, ``prefetch`` items ahead of the consumer; the training thread only pops a
ready item and makes its stream wait on the copy's event.  Device tensors are allocated on the side stream and handed
over with ``record_stream`` so the caching allocator cannot recycle them while the consumer's (possibly graph-replayed,
many steps deep) work is still queued.
"""
from __future__ import annotations

import pathlib
import queue
import threading
from typing import Any, Dict, Iterator, List, Optional, Tuple

import torch

# models/modeling_utils.py:22
IGNORE_KEYS_FOR_COLLATION = {"height", "width", "num_frames", "frame_rate", "rope_interpolation_scale", "return_dict",
                             "attention_kwargs", "cross_attention_kwargs", "joint_attention_kwargs", "latents_mean",
                             "latents_std"}


def save_item(item: Dict[str, Any], index: int, directory, data_type: str) -> None:
    """precomputation.py:413-415."""
    directory = pathlib.Path(directory)
    directory.mkdir(parents=True, exist_ok=True)
    torch.save(item, (directory / f"{data_type}-{index}.pt").as_posix())


def load_item(index: int, directory, data_type: str, map_location=None) -> Dict[str, Any]:
    """precomputation.py:418-420."""
    return torch.load((pathlib.Path(directory) / f"{data_type}-{index}.pt").as_posix(), map_location=map_location,
                      weights_only=True)


class _AsyncStager:
    """Background loader: index stream -> (device item, copy-done event).  One thread, one side stream, a pinned ring."""
    _END = object()

    def __init__(self, directory, data_type: str, indices: Iterator[Tuple[int, bool]], device: torch.device, depth: int):
        self.dir, self.data_type, self.device, self.depth = directory, data_type, torch.device(device), max(1, depth)
        self.indices = indices
        self.q: "queue.Queue" = queue.Queue(maxsize=self.depth)
        self.stream = torch.cuda.Stream(self.device)
        self.slots: List[Dict[str, torch.Tensor]] = [dict() for _ in range(self.depth + 2)]
        self.slot_ev: List[Optional[torch.cuda.Event]] = [None] * (self.depth + 2)
        self.stop = threading.Event()
        self.err: Optional[BaseException] = None
        self.thread = threading.Thread(target=self._run, daemon=True, name=f"b200-feed-{data_type}")
        self.thread.start()

    def _run(self):
        try:
            torch.cuda.set_device(self.device)
            n = 0
            for index, last in self.indices:
                if self.stop.is_set():
                    break
                item = load_item(index, self.dir, self.data_type, map_location="cpu")
                slot = n % len(self.slots)
                if self.slot_ev[slot] is not None:
                    self.slot_ev[slot].synchronize()  # the H2D copy that last read this pinned slot has finished
                out: Dict[str, Any] = {}
                with torch.cuda.stream(self.stream):
                    for k, v in item.items():
                        if not torch.is_tensor(v):
                            out[k] = v
                            continue
                        pin = self.slots[slot].get(k)
                        if pin is None or pin.shape != v.shape or pin.dtype != v.dtype:
                            pin = torch.empty(v.shape, dtype=v.dtype, pin_memory=True)
                            self.slots[slot][k] = pin
                        pin.copy_(v)
                        out[k] = pin.to(self.device, non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(self.stream)
                self.slot_ev[slot] = ev
                n += 1
                while not self.stop.is_set():
                    try:
                        self.q.put((out, ev, last), timeout=0.1)
                        break
                    except queue.Full:
                        continue
        except BaseException as e:  # noqa: BLE001  (re-raised on the consumer thread)
            self.err = e
        finally:
            while True:
                try:
                    self.q.put(self._END, timeout=0.1)
                    break
                except queue.Full:
                    if self.stop.is_set():
                        break

    def get(self):
        x = self.q.get()
        if x is self._END:
            if self.err is not None:
                raise self.err
            return None
        return x

    def close(self):
        self.stop.set()
        try:
            while True:
                self.q.get_nowait()
        except queue.Empty:
            pass
        self.thread.join(timeout=5)


class PrecomputedReader:
    """``PrecomputedDataIterable`` (precomputation.py:319-345): one pass over this rank's ``num_items`` items;
    ``requires_data`` turns True when the last item is handed out."""

    def __init__(self, save_dir, data_type: str, rank: int = 0, world_size: int = 1,
                 device: Optional[torch.device] = None, prefetch: int = 2):
        self.dir = pathlib.Path(save_dir)
        self.data_type = data_type
        self.rank, self.world_size = rank, world_size
        self.device = torch.device(device) if device is not None else None
        self.num_items = len(list(self.dir.glob(f"{data_type}-*.pt")))
        self.prefetch = int(prefetch) if (self.device is not None and self.device.type == "cuda") else 0
        self.requires_data = False

    def __len__(self) -> int:
        return self.num_items

    def _indices(self) -> Iterator[Tuple[int, bool]]:
        for i in range(self.num_items):
            yield self.rank * self.num_items + i, i == self.num_items - 1

    def __iter__(self) -> Iterator[Dict[str, Any]]:
        if not self.prefetch:
            for index, last in self._indices():
                if last:
                    self.requires_data = True
                yield load_item(index, self.dir, self.data_type, map_location=self.device)
            return
        stager = _AsyncStager(self.dir, self.data_type, self._indices(), self.device, self.prefetch)
        try:
            while True:
                got = stager.get()
                if got is None:
                    return
                item, ev, last = got
                cur = torch.cuda.current_stream(self.device)
                cur.wait_event(ev)
                for v in item.values():
                    if torch.is_tensor(v):
                        v.record_stream(cur)
                if last:
                    self.requires_data = True
                yield item
        finally:
            stager.close()


class PrecomputedOnceReader(PrecomputedReader):
    """``PrecomputedOnceDataIterable`` (precomputation.py:348-382): cycles forever over this rank's slice; never asks
    for more data."""

    def __init__(self, save_dir, data_type: str, rank: int = 0, world_size: int = 1,
                 device: Optional[torch.device] = None, prefetch: int = 2):
        super().__init__(save_dir, data_type, rank, world_size, device, prefetch)
        if self.num_items <= rank:
            raise ValueError(f"Precomputed data directory is empty or does not contain enough items (required {rank + 1}, "
                             f"found {self.num_items}).")
        self.num_items_per_rank = max(1, self.num_items // world_size)

    def __len__(self) -> int:
        return self.num_items_per_rank

    def _indices(self) -> Iterator[Tuple[int, bool]]:
        i = 0
        while True:
            yield self.rank * self.num_items_per_rank + i, False
            i = (i + 1) % self.num_items_per_rank


class ResolutionSampler:
    """Buckets items by the leader tensor's sizes along ``dim_keys[leader]`` and releases a batch when a bucket holds
    ``batch_size`` items (data/sampler.py:6-58: same ``consume`` / ``is_ready`` / ``get_batch`` protocol and errors)."""

    def __init__(self, batch_size: int = 1, dim_keys: Optional[Dict[str, Tuple[int, ...]]] = None) -> None:
        if dim_keys is None:
            raise AssertionError("dim_keys must be provided")
        self.batch_size, self.dim_keys = batch_size, dim_keys
        self._leader: Optional[str] = None
        self._open: Dict[Tuple[int, ...], List[tuple]] = {}
        self._ready: List[List[tuple]] = []

    @property
    def is_ready(self) -> bool:
        return bool(self._ready)

    def _pick_leader(self, items) -> None:
        found = [k for it in items for k in self.dim_keys if k in it]
        if len(found) > 1:
            raise ValueError(f"Only one leader key is allowed in provided list of data dictionaries. Found {len(found)} leader keys")
        if not found:
            raise ValueError("No leader key found in provided list of data dictionaries")
        holder = next(it for it in items if found[0] in it)
        if not torch.is_tensor(holder[found[0]]):
            raise ValueError(f"Leader key {found[0]} must be a tensor")
        self._leader = found[0]

    def consume(self, *dict_items: Dict[Any, Any]) -> None:
        if self._leader is None:
            self._pick_leader(dict_items)
        holder = next((it for it in dict_items if self._leader in it), None)
        if holder is None:
            raise ValueError(f"Leader key {self._leader} not found in provided list of data dictionaries")
        t = holder[self._leader]
        dims = tuple(t.size(d) for d in self.dim_keys[self._leader])
        bucket = self._open.setdefault(dims, [])
        bucket.append(dict_items)
        if len(bucket) == self.batch_size:
            self._ready.append(self._open.pop(dims))

    def get_batch(self) -> List[Tuple[Dict[str, Any], ...]]:
        """-> one tuple per consumed stream (conditions, latents), each holding ``batch_size`` item dicts."""
        return list(zip(*self._ready.pop()))


def collate(data: List[Dict[str, Any]]) -> Dict[str, Any]:
    """``collate_conditions`` / ``collate_latents`` (modeling_utils.py:156-181): tensors are concatenated along dim 0,
    the keys in ``IGNORE_KEYS_FOR_COLLATION`` are taken from the first item, everything else becomes a list."""
    out: Dict[str, Any] = {}
    for key in data[0].keys():
        if key in IGNORE_KEYS_FOR_COLLATION:
            out[key] = data[0][key]
            continue
        vals = [d[key] for d in data]
        out[key] = torch.cat(vals) if torch.is_tensor(vals[0]) else vals
    return out
