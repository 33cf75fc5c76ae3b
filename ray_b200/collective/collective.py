"""Functional collective API -- the calls a Ray actor makes.

API-compatible with ``ray.util.collective`` (python/ray/util/collective/collective.py): the
same function names, argument order, defaults, validation and exceptions, so an actor
written against the reference only changes its import (or, with Ray installed, keeps
``ray.util.collective`` and registers ``B200Group`` as a backend -- INTEGRATION.md).

Differences that follow from running without Ray's control plane in this repository:
  * the declarative path (``create_collective_group``) records the membership in the
    rendezvous ``Store`` instead of a detached ``Info`` actor (collective.py:188-261,
    util.py:55-85); lazy creation in ``get_group_handle`` reads it back, then falls back to
    the ``collective_*`` environment variables exactly like the reference (:760-770);
  * "inside an actor" (:795-804) cannot be checked; each *process or rank thread* owns one
    ``GroupManager`` (see ``use_manager``).
"""
from __future__ import annotations

import contextlib
import json
import logging
import os
import threading
from typing import Dict, List, Optional

import numpy as np
import torch

from ..store import Store, default_store
from . import types
from .registry import _global_registry

logger = logging.getLogger(__name__)


class GroupManager:
    """Per-process table of the collective groups this process belongs to
    (collective.py:65-133)."""

    def __init__(self, store: Optional[Store] = None):
        self._groups: Dict[str, object] = {}
        self._store = store
        self.lock = threading.Lock()

    @property
    def store(self) -> Store:
        return self._store if self._store is not None else default_store()

    def create_collective_group(self, backend, world_size, rank, group_name, gloo_timeout=None):
        key = str(backend).upper()
        cls = _global_registry.get(key)
        if not cls.check_backend_availability():
            raise RuntimeError(f"Backend {key} is not available. Please check the installation.")
        if key == "GLOO":
            group = cls(world_size, rank, group_name, gloo_timeout)
        elif self._store is not None and key == "B200":
            group = cls(world_size, rank, group_name, store=self._store)
        else:
            group = cls(world_size, rank, group_name)
        self._groups[group_name] = group
        return group

    def is_group_exist(self, group_name) -> bool:
        return group_name in self._groups

    def get_group_by_name(self, group_name):
        if group_name not in self._groups:
            logger.warning("The group '%s' is not initialized.", group_name)
            return None
        return self._groups[group_name]

    def destroy_collective_group(self, group_name) -> None:
        group = self._groups.pop(group_name, None)
        if group is None:
            logger.warning("The group '%s' does not exist.", group_name)
            return
        group.destroy_group()
        # the declarative record plays the role of the detached ``info_<name>`` actor
        try:
            self.store.delete(_info_key(group_name))
        except Exception:
            pass


_process_mgr = GroupManager()
_tls = threading.local()


def _mgr() -> GroupManager:
    return getattr(_tls, "mgr", None) or _process_mgr


@contextlib.contextmanager
def use_manager(mgr: GroupManager):
    """Bind ``mgr`` to the calling thread: lets several ranks live in one process (the
    single-GPU test harness) the way several actors live in several processes."""
    prev = getattr(_tls, "mgr", None)
    _tls.mgr = mgr
    try:
        yield mgr
    finally:
        _tls.mgr = prev


def _info_key(group_name: str) -> str:
    return f"b200/info_{group_name}"


# --------------------------------------------------------------------------- lifecycle
def is_group_initialized(group_name: str) -> bool:
    m = _mgr()
    with m.lock:
        return m.is_group_exist(group_name)


def init_collective_group(world_size: int, rank: int, backend=types.Backend.B200,
                          group_name: str = "default", gloo_timeout: int = 30000) -> None:
    """Imperative group creation inside a worker (collective.py:149-185)."""
    if not group_name:
        raise ValueError("group_name '{}' needs to be a string.".format(group_name))
    m = _mgr()
    with m.lock:
        if m.is_group_exist(group_name):
            raise RuntimeError("Trying to initialize a group a second time.")
        assert world_size > 0
        assert rank >= 0
        assert rank < world_size
        m.create_collective_group(backend, world_size, rank, group_name, gloo_timeout)


def create_collective_group(members: List[str], world_size: int, ranks: List[int],
                            backend=types.Backend.B200, group_name: str = "default",
                            gloo_timeout: int = 30000, store: Optional[Store] = None) -> None:
    """Declarative creation from the driver (collective.py:188-261).  ``members`` are the
    workers' identifiers (actor ids in Ray; any unique strings here); each worker later
    resolves its own rank through ``get_group_handle`` with ``member_id`` set via
    ``set_member_id``."""
    if len(ranks) != len(members):
        raise RuntimeError("Each actor should correspond to one rank. Got '{}' ranks but '{}' actors".format(
            len(ranks), len(members)))
    if set(ranks) != set(range(len(ranks))):
        raise RuntimeError("Ranks must be a permutation from 0 to '{}'. Got '{}'.".format(
            len(ranks), "".join(str(r) for r in ranks)))
    if world_size <= 0:
        raise RuntimeError("World size must be greater than zero. Got '{}'.".format(world_size))
    if any(r < 0 for r in ranks):
        raise RuntimeError("Ranks must be non-negative.")
    if any(r >= world_size for r in ranks):
        raise RuntimeError("Ranks cannot be greater than world_size.")
    key = str(backend).upper()
    if not _global_registry.is_registered(key):
        raise RuntimeError(f"Backend {key} is not registered. Please register it using "
                           f"register_collective_backend('{key}', YourBackendClass).")
    if not _global_registry.check(key):
        raise RuntimeError(f"Backend {key} is registered but not available.")
    st = store or _mgr().store
    try:
        st.get(_info_key(group_name), timeout_s=0.0)
        raise RuntimeError("Trying to initialize a group twice.")
    except TimeoutError:
        pass
    record = {"members": list(members), "world_size": world_size, "ranks": list(ranks),
              "backend": key, "gloo_timeout": gloo_timeout}
    st.set(_info_key(group_name), json.dumps(record).encode())


def set_member_id(member_id: str) -> None:
    """Identify this worker for declarative groups (Ray: the actor id, collective.py:752-753)."""
    _tls.member_id = member_id


def destroy_collective_group(group_name: str = "default") -> None:
    m = _mgr()
    with m.lock:
        m.destroy_collective_group(group_name)


def get_rank(group_name: str = "default") -> int:
    """Rank of this process in the group, -1 if it is not a member (collective.py:274-293)."""
    m = _mgr()
    with m.lock:
        return m.get_group_by_name(group_name).rank if m.is_group_exist(group_name) else -1


def get_collective_group_size(group_name: str = "default") -> int:
    m = _mgr()
    with m.lock:
        return m.get_group_by_name(group_name).world_size if m.is_group_exist(group_name) else -1


def get_group_handle(group_name: str = "default"):
    """Return the group, creating it lazily from the declarative record or from the
    ``collective_*`` environment variables (collective.py:729-777)."""
    m = _mgr()
    with m.lock:
        if not m.is_group_exist(group_name):
            created = False
            member = getattr(_tls, "member_id", None)
            if member is not None:
                try:
                    rec = json.loads(m.store.get(_info_key(group_name), timeout_s=0.0).decode())
                    rank = rec["ranks"][rec["members"].index(member)]
                    m.create_collective_group(rec["backend"], rec["world_size"], rank, group_name,
                                              rec["gloo_timeout"])
                    created = True
                except (TimeoutError, ValueError):
                    created = False
            if not created:
                if os.environ.get("collective_group_name") == group_name:
                    m.create_collective_group(
                        os.environ["collective_backend"], int(os.environ["collective_world_size"]),
                        int(os.environ["collective_rank"]), group_name,
                        int(os.getenv("collective_gloo_timeout", 30000)))
                else:
                    raise RuntimeError(
                        "The collective group '{}' is not initialized in the process.".format(group_name))
        return m.get_group_by_name(group_name)


# --------------------------------------------------------------------------- operations
def allreduce(tensor, group_name: str = "default", op=types.ReduceOp.SUM) -> None:
    """In-place all-reduce (collective.py:316-331).  Passes the options *class* with the op
    set on it, as the reference does (SURVEY Q1)."""
    _check_single_tensor_input(tensor)
    g = get_group_handle(group_name)
    opts = types.AllReduceOptions
    opts.reduceOp = op
    g.allreduce([tensor], opts)


def barrier(group_name: str = "default") -> None:
    get_group_handle(group_name).barrier()


def reduce(tensor, dst_rank: int = 0, group_name: str = "default", op=types.ReduceOp.SUM) -> None:
    _check_single_tensor_input(tensor)
    g = get_group_handle(group_name)
    _check_rank_valid(g, dst_rank)
    opts = types.ReduceOptions()
    opts.reduceOp, opts.root_rank, opts.root_tensor = op, dst_rank, 0
    g.reduce([tensor], opts)


def broadcast(tensor, src_rank: int = 0, group_name: str = "default") -> None:
    _check_single_tensor_input(tensor)
    g = get_group_handle(group_name)
    _check_rank_valid(g, src_rank)
    opts = types.BroadcastOptions()
    opts.root_rank, opts.root_tensor = src_rank, 0
    g.broadcast([tensor], opts)


def broadcast_multi(tensors: list, src_rank: int = 0, group_name: str = "default") -> None:
    """Broadcast a list of tensors (any dtypes) from ``src_rank`` in place, as one call: an
    extension beyond ``ray.util.collective`` for weight sync, where a loop of ``broadcast`` pays one
    launch per parameter.  Every rank passes tensors of the same byte sizes in the same order; the
    group's backend must provide ``broadcast_multi`` (``B200Group`` does)."""
    _check_tensor_list_input(tensors)
    g = get_group_handle(group_name)
    _check_rank_valid(g, src_rank)
    if not hasattr(g, "broadcast_multi"):
        raise RuntimeError("The collective group '{}' ({}) has no list broadcast.".format(
            group_name, type(g).__name__))
    g.broadcast_multi(tensors, src_rank)


def allgather(tensor_list: list, tensor, group_name: str = "default") -> None:
    _check_single_tensor_input(tensor)
    _check_tensor_list_input(tensor_list)
    g = get_group_handle(group_name)
    if len(tensor_list) != g.world_size:
        raise RuntimeError("The length of the tensor list operands to allgather must be equal to world_size.")
    g.allgather([tensor_list], [tensor], types.AllGatherOptions())


def reducescatter(tensor, tensor_list: list, group_name: str = "default", op=types.ReduceOp.SUM) -> None:
    _check_single_tensor_input(tensor)
    _check_tensor_list_input(tensor_list)
    g = get_group_handle(group_name)
    opts = types.ReduceScatterOptions()
    opts.reduceOp = op
    if len(tensor_list) != g.world_size:
        raise RuntimeError("The length of the tensor list operands to reducescatter must be equal to world_size.")
    g.reducescatter([tensor], [tensor_list], opts)


def allgatherv(tensor_list: list, tensor, group_name: str = "default") -> None:
    """``allgather`` with a size per rank: ``tensor_list[p]`` receives rank p's ``tensor``.  An
    extension beyond ``ray.util.collective``, whose ``allgather`` requires equal shapes, for
    variable-length results (eval outputs, per-rank token counts, a sharded buffer whose last rank
    holds the remainder).  Every rank passes outputs of the same sizes; the group's backend must
    provide ``allgatherv`` (``B200Group`` does)."""
    _check_single_tensor_input(tensor)
    _check_tensor_list_input(tensor_list)
    g = get_group_handle(group_name)
    if len(tensor_list) != g.world_size:
        raise RuntimeError("The length of the tensor list operands to allgather must be equal to world_size.")
    if not hasattr(g, "allgatherv"):
        raise RuntimeError("The collective group '{}' ({}) has no uneven all-gather.".format(
            group_name, type(g).__name__))
    g.allgatherv(tensor_list, tensor)


def reducescatterv(tensor, tensor_list: list, group_name: str = "default", op=types.ReduceOp.SUM) -> None:
    """``reducescatter`` with a size per rank: ``tensor`` = op over ranks of that rank's
    ``tensor_list[this rank]``, where ``tensor_list[q]`` has rank q's output size on every rank.  The
    mirror image of ``allgatherv``; the group's backend must provide ``reducescatterv``
    (``B200Group`` does)."""
    _check_single_tensor_input(tensor)
    _check_tensor_list_input(tensor_list)
    g = get_group_handle(group_name)
    if len(tensor_list) != g.world_size:
        raise RuntimeError("The length of the tensor list operands to reducescatter must be equal to world_size.")
    if not hasattr(g, "reducescatterv"):
        raise RuntimeError("The collective group '{}' ({}) has no uneven reduce-scatter.".format(
            group_name, type(g).__name__))
    g.reducescatterv(tensor, tensor_list, op)


def _check_list_of_lists(tensor_lists, tensors, world_size: int, what: str) -> None:
    if not isinstance(tensor_lists, list):
        raise RuntimeError("The input must be a list of tensor lists. Got '{}'.".format(type(tensor_lists)))
    if len(tensor_lists) != len(tensors):
        raise RuntimeError("Got {} tensor lists for {} tensors.".format(len(tensor_lists), len(tensors)))
    for lst in tensor_lists:
        _check_tensor_list_input(lst)
        if len(lst) != world_size:
            raise RuntimeError(
                "The length of the tensor list operands to {} must be equal to world_size.".format(what))


def allgather_multi(tensor_lists: list, tensors: list, group_name: str = "default") -> None:
    """``allgather`` of a list of tensors (any dtypes) as one call: ``tensor_lists[i][p]`` receives
    rank p's ``tensors[i]``.  An extension beyond ``ray.util.collective`` for sharded parameters,
    where a loop of ``allgather`` pays one launch per tensor.  Every rank passes tensors of the same
    byte sizes in the same order; the group's backend must provide ``allgather_multi``
    (``B200Group`` does)."""
    _check_tensor_list_input(tensors)
    g = get_group_handle(group_name)
    _check_list_of_lists(tensor_lists, tensors, g.world_size, "allgather")
    if not hasattr(g, "allgather_multi"):
        raise RuntimeError("The collective group '{}' ({}) has no list all-gather.".format(
            group_name, type(g).__name__))
    g.allgather_multi(tensor_lists, tensors)


def reducescatter_multi(tensors: list, tensor_lists: list, group_name: str = "default",
                        op=types.ReduceOp.SUM) -> None:
    """``reducescatter`` of a list of tensors of one dtype as one call: ``tensors[i]`` = op over ranks
    of that rank's ``tensor_lists[i][this rank]``.  The mirror image of ``allgather_multi``; the
    group's backend must provide ``reducescatter_multi`` (``B200Group`` does)."""
    _check_tensor_list_input(tensors)
    g = get_group_handle(group_name)
    _check_list_of_lists(tensor_lists, tensors, g.world_size, "reducescatter")
    if not hasattr(g, "reducescatter_multi"):
        raise RuntimeError("The collective group '{}' ({}) has no list reduce-scatter.".format(
            group_name, type(g).__name__))
    g.reducescatter_multi(tensors, tensor_lists, op)


def send(tensor, dst_rank: int, group_name: str = "default") -> None:
    _check_single_tensor_input(tensor)
    g = get_group_handle(group_name)
    _check_rank_valid(g, dst_rank)
    if dst_rank == g.rank:
        raise RuntimeError("The destination rank '{}' is self.".format(dst_rank))
    opts = types.SendOptions()
    opts.dst_rank = dst_rank
    g.send([tensor], opts)


def recv(tensor, src_rank: int, group_name: str = "default") -> None:
    _check_single_tensor_input(tensor)
    g = get_group_handle(group_name)
    _check_rank_valid(g, src_rank)
    if src_rank == g.rank:
        raise RuntimeError("The destination rank '{}' is self.".format(src_rank))
    opts = types.RecvOptions()
    opts.src_rank = src_rank
    g.recv([tensor], opts)


def synchronize(gpu_id: int) -> None:
    """Wait for all work on a device (collective.py:713-726 uses cupy; torch here)."""
    torch.cuda.synchronize(gpu_id)


# --------------------------------------------------------------------------- validation
def _check_single_tensor_input(tensor) -> None:
    """np.ndarray, torch.Tensor and CUDA-array-interface objects (cupy) pass the API check
    (collective.py:780-793); whether the *backend* accepts them is the backend's business."""
    if isinstance(tensor, (np.ndarray, torch.Tensor)) or hasattr(tensor, "__cuda_array_interface__"):
        return
    raise RuntimeError("Unrecognized tensor type '{}'. Supported types are: np.ndarray, torch.Tensor, "
                       "cupy.ndarray.".format(type(tensor)))


def _check_rank_valid(g, rank: int) -> None:
    if rank < 0:
        raise ValueError("rank '{}' is negative.".format(rank))
    if rank >= g.world_size:
        raise ValueError("rank '{}' must be less than world size '{}'".format(rank, g.world_size))


def _check_tensor_list_input(tensor_list) -> None:
    if not isinstance(tensor_list, list):
        raise RuntimeError("The input must be a list of tensors. Got '{}'.".format(type(tensor_list)))
    if not tensor_list:
        raise RuntimeError("Got an empty list of tensors.")
    for t in tensor_list:
        _check_single_tensor_input(t)
