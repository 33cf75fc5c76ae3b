"""``B200Communicator``: the Compiled-Graph ``Communicator`` (boundary B2) over the C ABI.

Implements the abstract interface at python/ray/experimental/channel/communicator.py:18-199
with the behaviour of the reference's ``_NcclGroup`` (experimental/channel/nccl_group.py:
21-374): out-of-place collectives on raw CUDA streams, ``recv`` that allocates through the
caller's allocator and returns a tensor that is safe to read from any stream, idempotent
``destroy()`` callable from another thread that unblocks pending device waits, and
``RayChannelError`` once the group is closed.

Use it as ``with_tensor_transport(transport=B200Communicator(...))``,
``allreduce.bind(nodes, transport=comm)``, ``experimental_compile(_default_communicator=comm)``
or class-register it with ``register_accelerator_context("cuda", B200Communicator)`` (it
accepts the constructor arguments of torch_tensor_accelerator_channel.py:673-680).
"""
from __future__ import annotations

import uuid
from typing import Callable, List, Optional, Tuple

import torch

from .. import _native as N
from ..comm import B200Comm
from ..store import Store, default_store

try:  # pragma: no cover - Ray is not installable in the build environment
    from ray.exceptions import RayChannelError  # type: ignore
    from ray.experimental.channel.communicator import Communicator  # type: ignore

    HAVE_RAY_COMMUNICATOR = True
except Exception:
    import abc

    HAVE_RAY_COMMUNICATOR = False

    class RayChannelError(Exception):
        """Stand-in for ray.exceptions.RayChannelError: the channel / communicator is closed."""

    class Communicator(abc.ABC):
        """Method-for-method restatement of the reference ABC (communicator.py:18-199)."""

        @abc.abstractmethod
        def initialize(self, rank: int) -> None: ...

        @abc.abstractmethod
        def get_actor_handles(self) -> list: ...

        @abc.abstractmethod
        def get_rank(self, actor) -> int: ...

        @abc.abstractmethod
        def get_self_rank(self) -> Optional[int]: ...

        def get_world_size(self) -> int:
            raise NotImplementedError

        @abc.abstractmethod
        def send(self, value: torch.Tensor, peer_rank: int) -> None: ...

        @abc.abstractmethod
        def recv(self, shape, dtype, peer_rank: int, allocator=None) -> torch.Tensor: ...

        @property
        @abc.abstractmethod
        def recv_stream(self): ...

        @property
        @abc.abstractmethod
        def send_stream(self): ...

        @abc.abstractmethod
        def allgather(self, send_buf, recv_buf) -> None: ...

        @abc.abstractmethod
        def allreduce(self, send_buf, recv_buf, op) -> None: ...

        @abc.abstractmethod
        def reducescatter(self, send_buf, recv_buf, op) -> None: ...

        @abc.abstractmethod
        def destroy(self) -> None: ...

        @abc.abstractmethod
        def get_transport_name(self) -> str: ...

        @classmethod
        @abc.abstractmethod
        def generate_communicator_id(cls) -> str: ...


TorchTensorAllocator = Callable[[Tuple[int], torch.dtype], torch.Tensor]

# ray.experimental.util.types.ReduceOp numbering (experimental/util/types.py:11-17) ->
# b200_op_t.  NOTE: MAX and MIN are swapped relative to ray.util.collective (SURVEY Q2).
_CGRAPH_OP = {0: N.SUM, 1: N.PROD, 2: N.MAX, 3: N.MIN, 4: N.AVG}
_CGRAPH_OP_BY_NAME = {"SUM": N.SUM, "PRODUCT": N.PROD, "MAX": N.MAX, "MIN": N.MIN, "AVG": N.AVG}


def _cgraph_op_code(op) -> int:
    name = getattr(op, "name", None)
    if name in _CGRAPH_OP_BY_NAME:
        return _CGRAPH_OP_BY_NAME[name]
    if isinstance(op, int) and op in _CGRAPH_OP:
        return _CGRAPH_OP[op]
    raise ValueError(f"Operation {op} not supported")


def _actor_key(actor):
    return getattr(actor, "_ray_actor_id", actor)


class B200Communicator(Communicator):
    """One actor's endpoint of a Compiled-Graph accelerator group.

    The object is created on the driver (rank unknown), pickled into every actor, and
    ``initialize(rank)`` is called there (torch_tensor_accelerator_channel.py:652-680); the
    native communicator is only built at that point.
    """

    def __init__(self, world_size: int, comm_id: Optional[str] = None, rank: Optional[int] = None,
                 actor_handles: Optional[list] = None, cuda_stream: Optional[torch.cuda.Stream] = None,
                 use_communication_streams: bool = False, store: Optional[Store] = None,
                 device: Optional[int] = None, host_sync: bool = False, **comm_kwargs):
        #: False (default): no host synchronisation per op.  Every op is enqueued and the tensor it
        #: produces is guarded by a CUDA event that the caller's current stream waits on -- the
        #: GPUFuture contract of the reference's overlap mode (dag/dag_operation_future.py:101-133,
        #: nccl_group.py:168-174) applied to every mode.  True: block the host after every recv /
        #: collective like the reference's non-overlap path (nccl_group.py:232-240,262-266).
        self._host_sync = host_sync
        self._world_size = world_size
        self._comm_id = comm_id or self.generate_communicator_id()
        self._rank: Optional[int] = None
        self._actor_handles = list(actor_handles or [])
        self._use_communication_streams = use_communication_streams
        self._store = store
        self._device = device
        self._comm_kwargs = comm_kwargs
        self._comm: Optional[B200Comm] = None
        self._cuda_stream = cuda_stream
        self._send_stream = self._recv_stream = None
        self._closed = False
        if rank is not None:
            self.initialize(rank)

    # pickling: only the description travels, never the native handle
    def __getstate__(self):
        return {"world_size": self._world_size, "comm_id": self._comm_id, "actor_handles": self._actor_handles,
                "use_communication_streams": self._use_communication_streams, "host_sync": self._host_sync,
                "comm_kwargs": self._comm_kwargs,
                "store": self._store if _is_picklable_store(self._store) else None}

    def __setstate__(self, st):
        self.__init__(st["world_size"], st["comm_id"], None, st["actor_handles"], None,
                      st["use_communication_streams"], st.get("store"), None, st.get("host_sync", False),
                      **st.get("comm_kwargs", {}))

    # ------------------------------------------------------------------ membership
    def initialize(self, rank: int) -> None:
        if self._comm is not None:
            return
        if not (0 <= rank < self._world_size):
            raise ValueError(f"rank {rank} out of range for world size {self._world_size}")
        self._rank = rank
        dev = torch.cuda.current_device() if self._device is None else self._device
        self._device = dev
        self._comm = B200Comm(self._world_size, rank, dev, store=self._store or default_store(),
                              group_name=f"cgraph-{self._comm_id}", **self._comm_kwargs)
        if self._cuda_stream is None:
            self._cuda_stream = torch.cuda.current_stream(dev)
        if self._use_communication_streams:
            self._send_stream = torch.cuda.Stream(device=dev)
            self._recv_stream = torch.cuda.Stream(device=dev)
        else:
            self._send_stream = self._recv_stream = self._cuda_stream

    def get_actor_handles(self) -> list:
        return self._actor_handles

    def get_rank(self, actor) -> int:
        keys = [_actor_key(a) for a in self._actor_handles]
        try:
            return keys.index(_actor_key(actor))
        except ValueError:
            raise ValueError("Actor is not in the B200 group.") from None

    def get_self_rank(self) -> Optional[int]:
        return self._rank

    def get_world_size(self) -> int:
        return self._world_size

    @property
    def comm(self) -> Optional[B200Comm]:
        return self._comm

    # ------------------------------------------------------------------ p2p
    def _check_open(self, what: str = "B200 group has been destroyed.") -> B200Comm:
        if self._closed or self._comm is None:
            raise RayChannelError(what)
        return self._comm

    def _raise_if_failed(self, comm: B200Comm, what: str = "B200 group has been destroyed.") -> None:
        """Non-blocking health check: the kernels mirror their sticky status into host-mapped memory,
        so this is a plain load -- no CUDA call, no synchronisation."""
        if self._closed or comm.status() != 0:
            raise RayChannelError(what)

    def send(self, buf: torch.Tensor, peer_rank: int) -> None:
        comm = self._check_open()
        self._raise_if_failed(comm)
        try:
            cur = torch.cuda.current_stream(self._device)
            if self._send_stream is not cur and self._send_stream.cuda_stream != cur.cuda_stream:
                # the tensor was produced on the caller's stream: order the send after it on the
                # device (the reference blocks the host here instead, nccl_group.py:167-174)
                self._send_stream.wait_stream(cur)
                buf.record_stream(self._send_stream)
            comm.send(buf, peer_rank, stream=self._send_stream)
        except N.B200AbortedError as e:
            raise RayChannelError(str(e)) from e

    def recv(self, shape: Tuple[int], dtype: torch.dtype, peer_rank: int,
             allocator: Optional[TorchTensorAllocator] = None) -> torch.Tensor:
        comm = self._check_open()
        assert allocator is not None, "B200 group requires a tensor allocator"
        self._raise_if_failed(comm)
        buf = allocator(shape, dtype)
        try:
            cur = torch.cuda.current_stream(self._device)
            same = self._recv_stream is cur or self._recv_stream.cuda_stream == cur.cuda_stream
            if not same:
                self._recv_stream.wait_stream(cur)  # the allocation may recycle memory still in use on `cur`
                buf.record_stream(self._recv_stream)
            comm.recv(buf, peer_rank, stream=self._recv_stream)
            if self._host_sync:
                # Buffer contents are undefined if the op was aborted: wait and re-check
                # (nccl_group.py:232-240).
                self._recv_stream.synchronize()
                self._raise_if_failed(comm)
            else:
                ev = torch.cuda.Event()
                ev.record(self._recv_stream)
                if not same:
                    cur.wait_event(ev)  # safe to read on the caller's stream; other streams wait on the event
                buf._b200_ready = ev  # noqa: SLF001 - the GPUFuture-style handle of this tensor
                self._last_recv_event = ev
        except N.B200AbortedError as e:
            raise RayChannelError(str(e)) from e
        if self._closed:
            raise RayChannelError("B200 group has been destroyed.")
        return buf

    def send_multi(self, bufs: List[torch.Tensor], peer_rank: int) -> None:
        """``send`` for a list of tensors: one message, one launch per table of tensors."""
        comm = self._check_open()
        self._raise_if_failed(comm)
        try:
            cur = torch.cuda.current_stream(self._device)
            if self._send_stream is not cur and self._send_stream.cuda_stream != cur.cuda_stream:
                self._send_stream.wait_stream(cur)
                for b in bufs:
                    b.record_stream(self._send_stream)
            comm.send_multi(bufs, peer_rank, stream=self._send_stream)
        except N.B200AbortedError as e:
            raise RayChannelError(str(e)) from e

    def recv_multi(self, metas: List[Tuple[Tuple[int], torch.dtype]], peer_rank: int,
                   allocator: Optional[TorchTensorAllocator] = None) -> List[torch.Tensor]:
        """``recv`` for a list of (shape, dtype): the peer's ``send_multi`` in one message.  Every
        returned tensor carries the ``_b200_ready`` event of the receive."""
        comm = self._check_open()
        assert allocator is not None, "B200 group requires a tensor allocator"
        self._raise_if_failed(comm)
        bufs = [allocator(shape, dtype) for shape, dtype in metas]
        try:
            cur = torch.cuda.current_stream(self._device)
            same = self._recv_stream is cur or self._recv_stream.cuda_stream == cur.cuda_stream
            if not same:
                self._recv_stream.wait_stream(cur)  # the allocations may recycle memory still in use on `cur`
                for b in bufs:
                    b.record_stream(self._recv_stream)
            comm.recv_multi(bufs, peer_rank, stream=self._recv_stream)
            if self._host_sync:
                self._recv_stream.synchronize()
                self._raise_if_failed(comm)
            else:
                ev = torch.cuda.Event()
                ev.record(self._recv_stream)
                if not same:
                    cur.wait_event(ev)
                for b in bufs:
                    b._b200_ready = ev  # noqa: SLF001
                self._last_recv_event = ev
        except N.B200AbortedError as e:
            raise RayChannelError(str(e)) from e
        if self._closed:
            raise RayChannelError("B200 group has been destroyed.")
        return bufs

    def wait(self, tensor: Optional[torch.Tensor] = None) -> None:
        """Block the host until ``tensor`` (default: the most recent recv) has arrived, then raise
        ``RayChannelError`` if the group was destroyed / aborted meanwhile -- what the reference's
        non-overlap recv does implicitly on every call."""
        ev = getattr(tensor, "_b200_ready", None) if tensor is not None else getattr(self, "_last_recv_event", None)
        if ev is not None:
            ev.synchronize()
        if self._comm is not None:
            self._raise_if_failed(self._comm)
        elif self._closed:
            raise RayChannelError("B200 group has been destroyed.")

    @property
    def recv_stream(self):
        return torch.cuda.StreamContext(self._recv_stream)

    @property
    def send_stream(self):
        return torch.cuda.StreamContext(self._send_stream)

    # ------------------------------------------------------------------ collectives
    def _collective(self, send_buf, recv_buf, fn) -> None:
        comm = self._check_open()
        assert send_buf.dtype == recv_buf.dtype, (
            "Ray Compiled Graph derived the dtype of recv_buf from send_buf, so send_buf and recv_buf must "
            "have the same dtype.")
        what = ("B200 group has been destroyed during a collective operation. There may "
                "be a dtype mismatch between input tensors from different ranks.")
        self._raise_if_failed(comm, what)
        try:
            cur = torch.cuda.current_stream(self._device)
            same = self._cuda_stream is cur or self._cuda_stream.cuda_stream == cur.cuda_stream
            if not same:
                self._cuda_stream.wait_stream(cur)
            with torch.cuda.stream(self._cuda_stream):
                fn(comm)
            if self._host_sync:
                self._cuda_stream.synchronize()  # nccl_group.py:262-266
                self._raise_if_failed(comm, what)
            elif not same:
                cur.wait_stream(self._cuda_stream)  # device-side ordering only
                send_buf.record_stream(self._cuda_stream)
                recv_buf.record_stream(self._cuda_stream)
        except N.B200AbortedError as e:
            raise RayChannelError(str(e)) from e

    def allgather(self, send_buf: torch.Tensor, recv_buf: torch.Tensor) -> None:
        self._collective(send_buf, recv_buf, lambda c: c.allgather_into(recv_buf, send_buf))

    def allreduce(self, send_buf: torch.Tensor, recv_buf: torch.Tensor, op=0) -> None:
        code = _cgraph_op_code(op)
        self._collective(send_buf, recv_buf, lambda c: c.allreduce(send_buf, code, out=recv_buf))

    def reducescatter(self, send_buf: torch.Tensor, recv_buf: torch.Tensor, op=0) -> None:
        code = _cgraph_op_code(op)
        self._collective(send_buf, recv_buf, lambda c: c.reducescatter_from(recv_buf, send_buf, code))

    def allreduce_multi(self, tensors, op=0) -> None:
        """In-place all-reduce of a list of same-dtype tensors as ONE message in ONE launch (the
        multi-tensor ``allreduce.bind`` case, dag/collective_node.py:212-232)."""
        code = _cgraph_op_code(op)
        comm = self._check_open()
        if len({t.dtype for t in tensors}) > 1:
            raise ValueError(f"Expected all input tensors to have the same dtype, but got {[t.dtype for t in tensors]}")
        self._raise_if_failed(comm)
        try:
            cur = torch.cuda.current_stream(self._device)
            same = self._cuda_stream is cur or self._cuda_stream.cuda_stream == cur.cuda_stream
            if not same:
                self._cuda_stream.wait_stream(cur)
            with torch.cuda.stream(self._cuda_stream):
                comm.allreduce_multi(list(tensors), code)
            if self._host_sync:
                self._cuda_stream.synchronize()
                self._raise_if_failed(comm, "B200 group has been destroyed during a collective operation.")
            elif not same:
                cur.wait_stream(self._cuda_stream)
        except N.B200AbortedError as e:
            raise RayChannelError(str(e)) from e

    # ------------------------------------------------------------------ lifecycle
    def broadcast(self, tensor: torch.Tensor, root_rank: int) -> None:
        """In-place broadcast over the WHOLE group (NVLS multimem.st when the multicast mapping
        exists): the multi-reader fast path of the tensor channel -- the reference loops send per
        reader and carries a TODO for exactly this (torch_tensor_accelerator_channel.py:587-590)."""
        self._collective(tensor, tensor, lambda c: c.broadcast(tensor, root_rank))

    def destroy(self) -> None:
        if self._closed:
            return
        self._closed = True  # set before the abort so unblocked ops observe it (nccl_group.py:356-364)
        if self._comm is not None:
            self._comm.abort()
            self._comm.destroy()

    def get_transport_name(self) -> str:
        return "accelerator"

    @classmethod
    def generate_communicator_id(cls) -> str:
        return str(uuid.uuid4())


def _is_picklable_store(store) -> bool:
    from ..store import FileStore

    return isinstance(store, FileStore)
