"""B200Group: the ``BaseGroup`` backend (boundary B1) over libb200_collective.so.

Drop-in for the reference's ``NCCLGroup`` (python/ray/util/collective/collective_group/
nccl_collective_group.py:128-412): same constructor, same list-wrapped operands, same
error behaviour, results in place, kernels enqueued on the caller's current CUDA stream
with no host synchronisation.  Register it with

    register_collective_backend("B200", B200Group)

in the driver and every actor (backend_registry.py:55-58), then use
``init_collective_group(..., backend="B200")`` and the usual ``collective.allreduce`` calls.
"""
from __future__ import annotations

import os
from typing import List, Optional

import torch

from .. import _native as N
from ..comm import B200Comm, dtype_code
from ..store import Store, default_store
from . import types
from .base_group import BaseGroup
from .types import ReduceOp

# ray.util.collective.types.ReduceOp -> b200_op_t (identical numbering, types.py:55-59)
_REDUCE_OP = {ReduceOp.SUM: N.SUM, ReduceOp.PRODUCT: N.PROD, ReduceOp.MIN: N.MIN, ReduceOp.MAX: N.MAX}


def _op_code(op) -> int:
    if isinstance(op, ReduceOp):
        return _REDUCE_OP[op]
    # a ReduceOp enum from the real ray.util.collective.types compares unequal to ours;
    # fall back to its name / value
    name = getattr(op, "name", None)
    if name in ("SUM", "PRODUCT", "MIN", "MAX"):
        return _REDUCE_OP[ReduceOp[name]]
    raise RuntimeError(f"Unsupported reduce op {op!r}")


def _as_cuda_tensor(t) -> torch.Tensor:
    """Accepts what NCCLGroup accepts on the GPU (nccl_util.py:162-179): torch CUDA tensors
    and objects exposing ``__cuda_array_interface__`` (cupy arrays), zero-copy."""
    if isinstance(t, torch.Tensor):
        if not t.is_cuda:
            raise RuntimeError("Torch tensor must be on GPU when using B200 collectives.")
        return t
    if hasattr(t, "__cuda_array_interface__"):
        return torch.as_tensor(t, device="cuda")
    raise ValueError(
        "Unsupported tensor type. Got: {}. Supported GPU tensor types are: torch.Tensor, "
        "cupy.ndarray.".format(type(t)))


def _unwrap_one(wrapped) -> torch.Tensor:
    if not isinstance(wrapped, list) or len(wrapped) != 1:
        raise RuntimeError("The B200 backend drives one GPU per process: expected a 1-element tensor list, "
                           f"got {type(wrapped)} of length {len(wrapped) if isinstance(wrapped, list) else '?'}")
    return _as_cuda_tensor(wrapped[0])


def _check_same_shape_dtype(single: torch.Tensor, many: List[torch.Tensor]) -> None:
    # nccl_collective_group.py:729-770: every list member must match dtype and exact shape
    for t in many:
        if t.dtype != single.dtype:
            raise RuntimeError(
                "All tensor operands to scatter/gather must have the same dtype. "
                f"Got '{t.dtype}' and '{single.dtype}'.")
        if tuple(t.shape) != tuple(single.shape):
            raise RuntimeError(
                "All tensor operands to scatter/gather must have the same shape. "
                f"Got '{tuple(t.shape)}' and '{tuple(single.shape)}'.")


class B200Group(BaseGroup):
    """One process (one GPU) in a B200 collective group."""

    #: rendezvous store used by groups created without an explicit one
    store: Optional[Store] = None

    def __init__(self, world_size: int, rank: int, group_name: str, store: Optional[Store] = None,
                 device: Optional[int] = None, **comm_kwargs):
        super().__init__(world_size, rank, group_name)
        if not torch.cuda.is_available():
            raise RuntimeError("B200 backend requires a CUDA device")
        self._device = torch.cuda.current_device() if device is None else int(device)
        store = store or type(self).store or default_store()
        for key, env in (("staging_bytes", "B200_STAGING_BYTES"), ("heap_bytes", "B200_HEAP_BYTES"),
                         ("inbox_bytes", "B200_INBOX_BYTES"), ("timeout_ms", "B200_TIMEOUT_MS")):
            if key not in comm_kwargs and os.environ.get(env):
                comm_kwargs[key] = int(os.environ[env])
        self._comm = B200Comm(world_size, rank, self._device, store=store, group_name=group_name, **comm_kwargs)

    # ------------------------------------------------------------------ metadata
    @classmethod
    def backend(cls):
        return types.Backend.B200

    @classmethod
    def check_backend_availability(cls) -> bool:
        try:
            N.load()
        except (ImportError, OSError, AttributeError):
            return False
        return torch.cuda.is_available()

    @property
    def comm(self) -> B200Comm:
        return self._comm

    def destroy_group(self):
        if self._comm is not None:
            self._comm.destroy()
            self._comm = None

    def _live(self) -> B200Comm:
        if self._comm is None:
            raise RuntimeError(f"The collective group '{self._group_name}' has been destroyed.")
        return self._comm

    # ------------------------------------------------------------------ collectives
    def allreduce(self, tensors, allreduce_options=types.AllReduceOptions()):
        t = _unwrap_one(tensors)
        self._live().allreduce(t, _op_code(allreduce_options.reduceOp))

    def barrier(self, barrier_options=types.BarrierOptions()):
        """Blocks until all processes reach this barrier (nccl_collective_group.py:211-229
        all-reduces a 1-element array; here a flag-only kernel, then a host wait)."""
        comm = self._live()
        comm.barrier()
        torch.cuda.current_stream(self._device).synchronize()
        comm.check_status()

    def reduce(self, tensors, reduce_options=types.ReduceOptions()):
        t = _unwrap_one(tensors)
        # legacy multi-GPU root index: len(tensors) * root_rank + root_tensor (:242) -- with one
        # tensor per process this is root_rank
        root = len(tensors) * reduce_options.root_rank + reduce_options.root_tensor
        self._live().reduce(t, root, _op_code(reduce_options.reduceOp))

    def broadcast(self, tensors, broadcast_options=types.BroadcastOptions()):
        t = _unwrap_one(tensors)
        root = len(tensors) * broadcast_options.root_rank + broadcast_options.root_tensor
        self._live().broadcast(t, root)

    def broadcast_multi(self, tensors, src_rank: int = 0):
        """Extension beyond the reference API (weight sync): broadcast a whole list of tensors, any
        dtypes, from ``src_rank`` in place -- one launch per staging slot of packed data instead of
        one ``broadcast`` per tensor.  Every rank passes tensors of the same byte sizes in order."""
        if not isinstance(tensors, list):
            raise RuntimeError("The input must be a list of tensors. Got '{}'.".format(type(tensors)))
        if src_rank < 0 or src_rank >= self._world_size:
            raise ValueError("rank '{}' is out of range for world size '{}'".format(src_rank, self._world_size))
        self._live().broadcast_multi([_as_cuda_tensor(t) for t in tensors], src_rank)

    def allgather(self, tensor_lists, tensors, allgather_options=types.AllGatherOptions()):
        t = _unwrap_one(tensors)
        if not isinstance(tensor_lists, list) or len(tensor_lists) != 1:
            raise RuntimeError("expected one output tensor list per process")
        outs = [_as_cuda_tensor(o) for o in tensor_lists[0]]
        if len(outs) != self._world_size:
            raise RuntimeError("The length of the tensor list operands to allgather must be equal to world_size.")
        _check_same_shape_dtype(t, outs)
        self._live().allgather(outs, t)

    def reducescatter(self, tensors, tensor_lists, reducescatter_options=types.ReduceScatterOptions()):
        out = _unwrap_one(tensors)
        if not isinstance(tensor_lists, list) or len(tensor_lists) != 1:
            raise RuntimeError("expected one input tensor list per process")
        ins = [_as_cuda_tensor(i) for i in tensor_lists[0]]
        if len(ins) != self._world_size:
            raise RuntimeError("The length of the tensor list operands to reducescatter must be equal to world_size.")
        _check_same_shape_dtype(out, ins)
        self._live().reducescatter(out, ins, _op_code(reducescatter_options.reduceOp))

    def allgatherv(self, tensor_list, tensor):
        """Extension beyond the reference API, whose ``allgather`` requires equal shapes:
        ``tensor_list[p]`` receives rank p's ``tensor``, whose size may differ per rank.  Every rank
        passes outputs of the same sizes; ``tensor_list[this rank]`` has this rank's size."""
        if not isinstance(tensor_list, list):
            raise RuntimeError("The output must be a list of tensors. Got '{}'.".format(type(tensor_list)))
        t = _as_cuda_tensor(tensor)
        outs = [_as_cuda_tensor(o) for o in tensor_list]
        if len(outs) != self._world_size:
            raise RuntimeError("The length of the tensor list operands to allgather must be equal to world_size.")
        self._live().allgatherv(outs, t)

    def reducescatterv(self, tensor, tensor_list, op=ReduceOp.SUM):
        """Extension beyond the reference API, whose ``reducescatter`` requires equal shapes:
        ``tensor`` = op over ranks of that rank's ``tensor_list[this rank]``; ``tensor_list[q]`` has
        rank q's output size, the same on every rank."""
        if not isinstance(tensor_list, list):
            raise RuntimeError("The input must be a list of tensors. Got '{}'.".format(type(tensor_list)))
        out = _as_cuda_tensor(tensor)
        ins = [_as_cuda_tensor(i) for i in tensor_list]
        if len(ins) != self._world_size:
            raise RuntimeError("The length of the tensor list operands to reducescatter must be equal to world_size.")
        self._live().reducescatterv(out, ins, _op_code(op))

    def allgather_multi(self, tensor_lists, tensors):
        """Extension beyond the reference API: ``allgather`` of a whole list of tensors (any dtypes)
        -- ``tensor_lists[i][p]`` receives rank p's ``tensors[i]`` -- in one launch per staging slot
        of packed data instead of one per tensor.  Every rank passes the same sizes in order."""
        if not isinstance(tensors, list) or not isinstance(tensor_lists, list):
            raise RuntimeError("The inputs must be lists of tensors. Got '{}' and '{}'.".format(
                type(tensor_lists), type(tensors)))
        if len(tensor_lists) != len(tensors):
            raise RuntimeError("expected one output tensor list per input tensor")
        ins = [_as_cuda_tensor(t) for t in tensors]
        out_lists = []
        for lst, t in zip(tensor_lists, ins):
            outs = [_as_cuda_tensor(o) for o in lst]
            if len(outs) != self._world_size:
                raise RuntimeError("The length of the tensor list operands to allgather must be equal to world_size.")
            _check_same_shape_dtype(t, outs)
            out_lists.append(outs)
        self._live().allgather_multi(out_lists, ins)

    def reducescatter_multi(self, tensors, tensor_lists, op=ReduceOp.SUM):
        """Extension beyond the reference API: ``reducescatter`` of a whole list of tensors of one
        dtype -- ``tensors[i]`` = op over ranks of that rank's ``tensor_lists[i][this rank]`` -- in
        one launch per window of packed data, bit-identical to one ``reducescatter`` per tensor."""
        if not isinstance(tensors, list) or not isinstance(tensor_lists, list):
            raise RuntimeError("The inputs must be lists of tensors. Got '{}' and '{}'.".format(
                type(tensors), type(tensor_lists)))
        if len(tensor_lists) != len(tensors):
            raise RuntimeError("expected one input tensor list per output tensor")
        outs = [_as_cuda_tensor(t) for t in tensors]
        in_lists = []
        for out, lst in zip(outs, tensor_lists):
            ins = [_as_cuda_tensor(i) for i in lst]
            if len(ins) != self._world_size:
                raise RuntimeError("The length of the tensor list operands to reducescatter must be equal to world_size.")
            _check_same_shape_dtype(out, ins)
            in_lists.append(ins)
        self._live().reducescatter_multi(outs, in_lists, _op_code(op))

    def send(self, tensors, send_options=types.SendOptions()):
        t = _unwrap_one(tensors)
        self._check_peer(send_options.dst_rank)
        t = self._slice(t, send_options.n_elements)
        self._live().send(t, send_options.dst_rank)

    def recv(self, tensors, recv_options=types.RecvOptions()):
        t = _unwrap_one(tensors)
        self._check_peer(recv_options.src_rank)
        t = self._slice(t, recv_options.n_elements)
        self._live().recv(t, recv_options.src_rank)

    # ------------------------------------------------------------------ helpers
    def _check_peer(self, peer: int) -> None:
        if peer == self._rank:
            raise RuntimeError("The peer rank '{}' is self.".format(peer))
        if peer < 0 or peer >= self._world_size:
            raise ValueError("rank '{}' is out of range for world size '{}'".format(peer, self._world_size))

    @staticmethod
    def _slice(t: torch.Tensor, n_elements: int) -> torch.Tensor:
        # n_elements > 0 sends a prefix (nccl_collective_group.py:374-381)
        if n_elements and n_elements > 0:
            if not t.is_contiguous():
                raise RuntimeError("tensor must be contiguous")
            return t.view(-1)[:n_elements]
        return t


__all__ = ["B200Group", "dtype_code"]
