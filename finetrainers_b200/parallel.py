"""Parallel backend for the data-parallel hot path: the subset of finetrainers' ``BaseParallelBackend``
(``finetrainers/parallel/base.py:9-115``) that ``SFTTrainer`` touches for DDP training, one process per
GPU over NCCL/NVLink (``parallel/ptd.py:41-279``; DDP = ``replicate(bucket_cap_mb=100)`` ``ptd.py:462-463``).

Design: the LoRA gradients already live in ONE flat fp32 buffer written by the backward kernels, so "DDP" is a
single in-place all-reduce (AVG) of that buffer on the NVSwitch fabric (235 MB at r=64: ~0.5 ms, NVLS-capable) issued
right after backward — no reducer hooks, no per-parameter buckets — and the three scalar metrics reductions
(``parallel/utils.py:6-19``, ``trainer.py:512-518``) fold into one 3-float all-reduce.  The path shards over independent
samples; there is no activation traffic (SURVEY §8e).  FSDP-2 / HSDP / CP / TP / PP are outside round 1.
"""
from __future__ import annotations

import datetime
import os
from contextlib import contextmanager
from typing import Any, Dict, Optional

import torch
import torch.distributed as dist


def _avg_all_reduce(t: torch.Tensor, group=None, async_op: bool = False):
    """AVG all-reduce that also works on the gloo backend (CPU tests): SUM then divide.  ``async_op`` (NCCL only) returns
    the work handle instead of the tensor."""
    group = _group_of(group)
    if group is _UNIT_GROUP or not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return None if async_op else t
    if dist.get_backend(group) == "nccl":
        w = dist.all_reduce(t, op=dist.ReduceOp.AVG, group=group, async_op=async_op)
        if async_op:
            return w
    else:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
        t.div_(dist.get_world_size(group))
    return None if async_op else t   # gloo: completed synchronously, nothing to wait for


def dist_mean(x: torch.Tensor, group=None) -> float:
    """parallel/utils.py:17-19."""
    assert x.numel() == 1
    return _avg_all_reduce(x.clone(), group).item()


def dist_max(x: torch.Tensor, group=None) -> float:
    """parallel/utils.py:13-15."""
    assert x.numel() == 1
    y = x.clone()
    group = _group_of(group)
    if group is not _UNIT_GROUP and dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(y, op=dist.ReduceOp.MAX, group=group)
    return y.item()


def fused_step_metrics(grad_norm: torch.Tensor, loss: torch.Tensor, group=None) -> Dict[str, float]:
    """grad_norm AVG, loss AVG, loss MAX over the data-parallel group (trainer.py:507-520: three collectives and up to
    five ``.item()`` syncs there) as ONE all-gather of two floats per rank and ONE host sync."""
    mine = torch.stack([grad_norm.reshape(()).float(), loss.reshape(()).float()])
    group = _group_of(group)
    if group is not _UNIT_GROUP and dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        allv = torch.empty(dist.get_world_size(group) * 2, dtype=torch.float32, device=mine.device)
        dist.all_gather_into_tensor(allv, mine, group=group)
        rows = allv.view(-1, 2).tolist()
    else:
        rows = [mine.tolist()]
    n = len(rows)
    return {"train/grad_norm": sum(r[0] for r in rows) / n, "train/global_avg_loss": sum(r[1] for r in rows) / n,
            "train/global_max_loss": max(r[1] for r in rows)}


def allreduce_flat_grads(flat_grad: torch.Tensor, group=None, chunk_bytes: int = 0, async_op: bool = False):
    """Average the flat gradient buffer in place.  ``chunk_bytes`` > 0 issues several collectives (bucket_cap_mb-style);
    ``async_op`` issues ONE collective and returns its work handle (None when there is nothing to exchange)."""
    group = _group_of(group)
    if async_op:
        return _avg_all_reduce(flat_grad, group, async_op=True)
    if group is _UNIT_GROUP or not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return flat_grad
    if chunk_bytes <= 0:
        return _avg_all_reduce(flat_grad, group)
    n = max(1, chunk_bytes // flat_grad.element_size())
    for s in range(0, flat_grad.numel(), n):
        _avg_all_reduce(flat_grad[s:s + n], group)
    return flat_grad


class B200Mesh:
    """Stand-in for the ``torch.distributed.DeviceMesh`` the reference builds (ptd.py:182-219) restricted to what this
    backend supports: ONE data-parallel dimension (replicated = DDP, or sharded = FSDP-2); pp / cp / tp have size 1.
    ``mesh[name]`` (a name or a tuple of names, as trainer.py:166-183 builds them) returns a sub-mesh with
    ``get_group()`` / ``size()`` / ``get_local_rank()`` / ``ndim``; the data-parallel names all map to the world group."""
    _DP_NAMES = ("dp", "dp_cp", "dp_replicate", "dp_shard", "dp_shard_cp")
    _UNIT_NAMES = ("pp", "cp", "tp")

    def __init__(self, world: int, rank: int, sharded: bool, names=None, group="world"):
        self._world, self._rank, self._sharded = world, rank, sharded
        self.mesh_dim_names = tuple(names) if names is not None else (("dp_shard_cp",) if sharded else ("dp_replicate",))
        self._group = group

    @property
    def ndim(self) -> int:
        return 1

    def size(self, mesh_dim: Optional[int] = None) -> int:
        return self._world if self._group == "world" else 1

    def get_local_rank(self, mesh_dim=None) -> int:
        return self._rank if self._group == "world" else 0

    def get_group(self, mesh_dim=None):
        """None = the default (world) process group for the data-parallel views; unit meshes have no peers."""
        if self._group != "world":
            return _UNIT_GROUP
        return dist.group.WORLD if dist.is_initialized() else None

    def __getitem__(self, name):
        names = (name,) if isinstance(name, str) else tuple(name)
        for n in names:
            if n not in self._DP_NAMES + self._UNIT_NAMES:
                raise KeyError(f"mesh dimension {n!r} does not exist (have {self._DP_NAMES + self._UNIT_NAMES})")
        unit = all(n in self._UNIT_NAMES for n in names)
        return B200Mesh(self._world, self._rank, self._sharded, names, "unit" if unit else "world")

    def __repr__(self):
        return f"B200Mesh({self.mesh_dim_names}, size={self.size()})"


_UNIT_GROUP = object()  # marker: a mesh dimension of size 1 (no collective is ever issued on it)


def _group_of(mesh_or_group):
    """Accept what the reference passes (a mesh, ``parallel/utils.py:6-19``) or a raw process group / None."""
    if isinstance(mesh_or_group, B200Mesh):
        return mesh_or_group.get_group()
    return mesh_or_group


class B200ParallelBackend:
    """Same surface as ``PytorchDTensorParallelBackend`` for the calls the SFT loop makes (ptd.py:41-279)."""

    def __init__(self, world_size: Optional[int] = None, dp_degree: Optional[int] = None, dp_shards: int = 1,
                 backend: str = "nccl", timeout: int = 180, device_type: str = "cuda", **other_degrees):
        """Same keyword names as ``PytorchDTensorParallelBackend.__init__`` (ptd.py:41-57).  Supported layouts: pure
        replication (``dp_degree == world``, DDP) or pure sharding (``dp_shards == world``, FSDP-2); pp / cp / tp must be 1
        and HSDP (both > 1) is not built (SURVEY section 2.2: out of scope for the LTX path)."""
        for k, v in other_degrees.items():
            if k in ("pp_degree", "cp_degree", "tp_degree"):
                if v not in (None, 1):
                    raise NotImplementedError(f"{k}={v}: only data parallelism is built (SURVEY section 2.2)")
            elif k not in ("logging_dir", "output_dir", "gradient_accumulation_steps"):
                raise TypeError(f"unexpected argument {k!r}")
        self._device_type = device_type
        if not dist.is_initialized() and int(os.environ.get("WORLD_SIZE", "1")) > 1:
            dist.init_process_group(backend=backend, timeout=datetime.timedelta(seconds=timeout))
        self._world = dist.get_world_size() if dist.is_initialized() else 1
        self._rank = dist.get_rank() if dist.is_initialized() else 0
        self._local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        if world_size is not None and world_size != self._world:
            raise ValueError(f"world_size {world_size} != launched world {self._world}")
        dp_shards = 1 if dp_shards in (None, -1) else int(dp_shards)
        if dp_shards > 1:
            if dp_degree not in (None, 1):
                raise NotImplementedError("HSDP (dp_degree > 1 together with dp_shards > 1) is not built")
            if dp_shards != self._world:
                raise ValueError(f"dp_shards {dp_shards} must equal world_size {self._world}")
            self._dp_degree, self._dp_shards = 1, dp_shards
        else:
            self._dp_degree, self._dp_shards = dp_degree or self._world, 1
            if self._dp_degree != self._world:
                raise ValueError("the b200 backend is pure data parallel: dp_degree (or dp_shards) must equal world_size")
        if device_type == "cuda":
            torch.cuda.set_device(self._local_rank)
        self.tracker = None
        self._mesh = None

    # --- model / optimizer preparation -------------------------------------------------------------------------
    def apply_ddp(self, model: torch.nn.Module, device_mesh=None) -> torch.nn.Module:
        """Replicas start identical (broadcast from rank 0); gradient averaging is done on the flat buffer by
        ``SFTTrainStep.optimizer_step`` / ``allreduce_flat_grads``."""
        if self._world > 1:
            with torch.no_grad():
                if hasattr(model, "lora_flat") and getattr(model, "_prepared", False):
                    dist.broadcast(model.lora_flat, src=0)
                else:
                    for p in model.parameters():
                        dist.broadcast(p.data, src=0)
        model._b200_ddp = True
        return model

    def apply_fsdp2(self, model: torch.nn.Module, param_dtype: torch.dtype = torch.bfloat16,
                    reduce_dtype: torch.dtype = torch.float32, output_dtype: Optional[torch.dtype] = None,
                    pp_enabled: bool = False, cpu_offload: bool = False, device_mesh=None) -> torch.nn.Module:
        """``PytorchDTensorParallelBackend.apply_fsdp2`` (ptd.py:100-113 -> ``apply_fsdp2`` ptd.py:466-499), same argument
        names.  Every DiT block and the root become sharding units (``fsdp.FSDPState``); parameters are stored and
        gathered in ``param_dtype`` (must be the model's dtype: nothing is cast), gradients are reduced in fp32."""
        from .fsdp import FSDPState
        if pp_enabled:
            raise NotImplementedError("pipeline parallelism is not built (the reference's SFT loop refuses it too, trainer.py:90-93)")
        if cpu_offload:
            raise NotImplementedError("cpu_offload is not built (the reference passes False, trainer.py:181)")
        if reduce_dtype not in (None, torch.float32):
            raise NotImplementedError("gradients are reduced in fp32 (MixedPrecisionPolicy(reduce_dtype=torch.float32), trainer.py:178)")
        wdt = next(p for n, p in model.named_parameters() if "lora_" not in n).dtype
        if param_dtype is not None and param_dtype != wdt:
            raise ValueError(f"param_dtype {param_dtype} != parameter dtype {wdt}: call model.to(dtype=...) first (trainer.py:133)")
        group = device_mesh.get_group() if isinstance(device_mesh, B200Mesh) else device_mesh
        if group is _UNIT_GROUP:
            group = None
        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError("apply_fsdp2 needs an initialised process group")
        model._fsdp = FSDPState(model, group)
        return model

    def apply_context_parallel(self, *args, **kwargs):
        raise NotImplementedError("context parallelism is out of scope: LTX has no CP plan in the reference either")

    def prepare_model(self, model):
        return model

    def prepare_optimizer(self, optimizer):
        return optimizer

    def prepare_dataset(self, dataset):
        return dataset

    def prepare_dataloader(self, dataset, batch_size=1, num_workers=0, pin_memory=True):
        return torch.utils.data.DataLoader(dataset, batch_size=batch_size, num_workers=num_workers, pin_memory=pin_memory)

    def get_mesh(self, name: Optional[str] = None):
        """``get_mesh()`` / ``get_mesh()[name]`` as the SFT loop indexes it (trainer.py:144,150,183,186,492,512,595): a
        1-D data-parallel mesh whose every named view the loop asks for resolves to a process group."""
        if self._mesh is None:
            self._mesh = B200Mesh(self._world, self._rank, self._dp_shards > 1)
        return self._mesh[name] if name is not None else self._mesh

    def get_checkpointer(self, *args, **kwargs):
        raise NotImplementedError("checkpointing stays with the caller (parameter FQNs are diffusers/peft compatible)")

    def wait_for_everyone(self):
        if self._world > 1:
            dist.barrier()

    @contextmanager
    def main_process_first(self):
        if not self.is_main_process:
            self.wait_for_everyone()
        yield
        if self.is_main_process:
            self.wait_for_everyone()

    def destroy(self):
        if dist.is_initialized():
            dist.destroy_process_group()

    def log(self, metrics: Dict[str, Any], step: int) -> None:
        if self.is_main_process and self.tracker is not None:
            self.tracker.log(metrics, step)

    # --- properties ---------------------------------------------------------------------------------------------
    @property
    def world_size(self):
        return self._world

    @property
    def rank(self):
        return self._rank

    @property
    def local_rank(self):
        return self._local_rank

    @property
    def is_main_process(self):
        return self._rank == 0

    @property
    def is_local_main_process(self):
        return self._local_rank == 0

    @property
    def device(self):
        return torch.device(self._device_type, self._local_rank) if self._device_type == "cuda" else torch.device("cpu")

    @property
    def pipeline_parallel_enabled(self):
        return False

    @property
    def data_parallel_enabled(self):
        return self._world > 1

    @property
    def data_replication_enabled(self):
        return self._dp_degree > 1

    @property
    def data_sharding_enabled(self):
        return self._dp_shards > 1

    @property
    def context_parallel_enabled(self):
        return False

    @property
    def tensor_parallel_enabled(self):
        return False
