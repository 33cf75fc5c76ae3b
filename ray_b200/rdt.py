"""RDT tensor transport (boundary B3): ``@ray.method(tensor_transport="B200")``.

Implements ``TensorTransportManager`` (python/ray/experimental/rdt/tensor_transport_manager.py:
37-224) the way the reference's ``CollectiveTensorTransport`` does for NCCL / GLOO
(python/ray/experimental/rdt/collective_tensor_transport.py:34-203): a two-sided transport whose
``__ray_send__`` / ``__ray_recv__`` halves (run on the ``_ray_system`` concurrency-group thread,
rdt_manager.py:655-681) map to ``collective.send`` / ``collective.recv`` of a collective group
that contains both actors -- here a B200 group, so the payload moves through the
sender-push NVLink kernel.  Three differences from the NCCL transport:

* the tensors of an object travel as ONE message (``b200_send_multi`` / ``b200_recv_multi``): one
  launch per side per 256 tensors instead of one per tensor;

* ``can_abort_transport()`` is True: the device-side waits poll an abort word, so a stuck
  transfer is cancelled instead of Ray having to kill both actors (tensor_transport_manager.py:
  75-92);
* sends are eager up to the inbox ring size, so the sender does not block on the receiver
  having posted its recv.

Register with ``register_tensor_transport("B200", ["cuda"], B200TensorTransport, torch.Tensor)``
(python/ray/experimental/rdt/util.py:46-84).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, List, Optional, Tuple

import torch

try:  # pragma: no cover - Ray is not installable in the build environment
    import ray.util.collective as _collective  # type: ignore
    from ray.experimental.rdt.tensor_transport_manager import (  # type: ignore
        CommunicatorMetadata,
        TensorTransportManager,
        TensorTransportMetadata,
    )

    HAVE_RAY_RDT = True
except Exception:
    import abc

    from . import collective as _collective

    HAVE_RAY_RDT = False

    @dataclass
    class CommunicatorMetadata:
        """Metadata for the communicator."""

    @dataclass
    class TensorTransportMetadata:
        """(shape, dtype) per tensor plus the common device type."""

        tensor_meta: List[Tuple[Any, Any]] = field(default_factory=list)
        tensor_device: Optional[str] = None

    class TensorTransportManager(abc.ABC):
        @abc.abstractmethod
        def tensor_transport_backend(self) -> str: ...

        @staticmethod
        @abc.abstractmethod
        def is_one_sided() -> bool: ...

        @staticmethod
        @abc.abstractmethod
        def can_abort_transport() -> bool: ...

        @abc.abstractmethod
        def actor_has_tensor_transport(self, actor) -> bool: ...

        @abc.abstractmethod
        def extract_tensor_transport_metadata(self, obj_id, rdt_object): ...

        @abc.abstractmethod
        def get_communicator_metadata(self, src_actor, dst_actor, backend=None): ...

        @abc.abstractmethod
        def recv_multiple_tensors(self, obj_id, tensor_transport_metadata, communicator_metadata,
                                  target_buffers=None): ...

        @abc.abstractmethod
        def send_multiple_tensors(self, tensors, tensor_transport_metadata, communicator_metadata): ...

        @abc.abstractmethod
        def garbage_collect(self, obj_id, tensor_transport_meta, tensors): ...

        @abc.abstractmethod
        def abort_transport(self, obj_id, communicator_metadata): ...


@dataclass
class B200CommunicatorMetadata(CommunicatorMetadata):
    """Which group and which ranks a transfer uses (collective_tensor_transport.py:19-31)."""

    communicator_name: str = ""
    src_rank: Optional[int] = None
    dst_rank: Optional[int] = None


@dataclass
class B200TransportMetadata(TensorTransportMetadata):
    pass


class B200TensorTransport(TensorTransportManager):
    """Two-sided RDT transport over a B200 collective group."""

    #: resolves (src_actor, dst_actor) -> (group name, src rank, dst rank) on the driver; with Ray
    #: this is ray.experimental.collective.get_collective_groups, injected here for harnesses
    group_resolver = None

    def tensor_transport_backend(self) -> str:
        return "B200"

    @staticmethod
    def is_one_sided() -> bool:
        return False

    @staticmethod
    def can_abort_transport() -> bool:
        return True

    def actor_has_tensor_transport(self, actor) -> bool:
        if HAVE_RAY_RDT:  # pragma: no cover
            from ray.experimental.collective import get_collective_groups

            return len(get_collective_groups([actor], backend=self.tensor_transport_backend())) > 0
        return self.group_resolver is not None

    def extract_tensor_transport_metadata(self, obj_id: str, rdt_object: List[torch.Tensor]) -> B200TransportMetadata:
        meta, device = [], None
        for t in rdt_object or []:
            device = device or t.device
            if t.device.type != device.type:
                raise ValueError("All tensors in an RDT object must have the same device type.")
            meta.append((t.shape, t.dtype))
        return B200TransportMetadata(tensor_meta=meta, tensor_device=device.type if device else None)

    def get_communicator_metadata(self, src_actor, dst_actor, backend: Optional[str] = None) -> B200CommunicatorMetadata:
        if HAVE_RAY_RDT:  # pragma: no cover
            from ray.experimental.collective import get_collective_groups

            groups = get_collective_groups([src_actor, dst_actor], backend=backend)
            if len(groups) == 0:
                raise ValueError(f"No communicators found for actors {src_actor} and {dst_actor}. Create a "
                                 "communicator with `ray.experimental.collective.create_collective_group` before "
                                 "calling actor tasks. with non-default tensor_transport.")
            if len(groups) > 1:
                raise ValueError(f"There are {len(groups)} possible communicators that contain actors {src_actor} "
                                 f"and {dst_actor}. Currently, RDT objects only support one communicator.")
            g = groups[0]
            name, src, dst = g.name, g.get_rank(src_actor), g.get_rank(dst_actor)
        else:
            if self.group_resolver is None:
                raise ValueError(f"No communicators found for actors {src_actor} and {dst_actor}.")
            name, src, dst = self.group_resolver(src_actor, dst_actor)
        if src == -1 or dst == -1:
            raise ValueError("Sender and receiver must be in the same communicator.")
        return B200CommunicatorMetadata(communicator_name=name, src_rank=src, dst_rank=dst)

    def recv_multiple_tensors(self, obj_id, tensor_transport_metadata, communicator_metadata,
                              target_buffers: Optional[List[torch.Tensor]] = None) -> List[torch.Tensor]:
        assert isinstance(communicator_metadata, B200CommunicatorMetadata)
        tensors = target_buffers or [torch.empty(tuple(shape), dtype=dtype, device="cuda")
                                     for shape, dtype in tensor_transport_metadata.tensor_meta]
        # the whole object is one message: one launch per table of tensors, not one per tensor
        self._comm_of(communicator_metadata.communicator_name).recv_multi(tensors, communicator_metadata.src_rank)
        return tensors

    def send_multiple_tensors(self, tensors, tensor_transport_metadata, communicator_metadata) -> None:
        assert isinstance(communicator_metadata, B200CommunicatorMetadata)
        device = tensors[0].device if tensors else None
        for t in tensors:
            if t.device.type != device.type:
                raise ValueError(f"tensor device {t.device} does not match device {device}")
        self._comm_of(communicator_metadata.communicator_name).send_multi(tensors, communicator_metadata.dst_rank)

    def _comm_of(self, group_name: str):
        """The native endpoint (B200Comm) of a B200 collective group."""
        group = _collective.get_group_handle(group_name)
        comm = getattr(group, "comm", None)
        if comm is None:
            raise RuntimeError(f"collective group {group_name!r} is not a B200 group")
        return comm

    def garbage_collect(self, obj_id, tensor_transport_meta, tensors) -> None:
        """Nothing is registered per object: the inbox ring is owned by the communicator."""

    def abort_transport(self, obj_id, communicator_metadata) -> None:
        group = _collective.get_group_handle(communicator_metadata.communicator_name)
        comm = getattr(group, "comm", None)
        if comm is not None:
            comm.abort()


# --------------------------------------------------------------------------------------------
# One-sided transport (SURVEY 8f row 4; pattern: experimental/rdt/cuda_ipc_transport.py:57-186)
# --------------------------------------------------------------------------------------------
@dataclass
class B200IpcTransportMetadata(TensorTransportMetadata):
    """What the receiver needs to pull the object by itself: where every tensor sits in the
    owner's symmetric heap, which rank owns it, and the event that orders the pull after the
    owner's writes."""

    communicator_name: str = ""
    src_rank: int = -1
    heap_offsets: List[int] = field(default_factory=list)
    nbytes: List[int] = field(default_factory=list)
    event_ipc_handle: Optional[bytes] = None
    src_pid: int = -1
    obj_id: str = ""


class _HeapArena:
    """First-fit allocator over the part of a rank's symmetric heap reserved for RDT objects.
    Unlike b200_symm_alloc it is LOCAL: peers never need to agree on it, because any offset of the
    owner's heap is readable through the peer mapping that already exists."""

    def __init__(self, start: int, size: int, align: int = 256):
        self._free = [(start, size)]
        self._align = align
        self._used = {}

    def alloc(self, nbytes: int) -> int:
        need = max((nbytes + self._align - 1) // self._align * self._align, self._align)
        for i, (off, size) in enumerate(self._free):
            if size >= need:
                self._free[i] = (off + need, size - need)
                if self._free[i][1] == 0:
                    del self._free[i]
                self._used[off] = need
                return off
        raise MemoryError(f"RDT arena of the symmetric heap is exhausted ({nbytes} bytes requested); raise heap_bytes")

    def free(self, off: int) -> None:
        size = self._used.pop(off)
        self._free.append((off, size))
        self._free.sort()
        merged = []
        for o, s in self._free:
            if merged and merged[-1][0] + merged[-1][1] == o:
                merged[-1] = (merged[-1][0], merged[-1][1] + s)
            else:
                merged.append((o, s))
        self._free = merged


class B200IpcTransport(B200TensorTransport):
    """One-sided RDT transport: ``extract_tensor_transport_metadata`` (sender, right after the task
    returns) places the object in the sender's symmetric heap and returns (heap offsets, event);
    ``recv_multiple_tensors`` pulls it with a receiver-side kernel (``b200_get``: bulk loads over
    NVLink) straight into ``target_buffers`` -- no kernel, no thread and no call on the sender.
    Where the reference's ``CudaIpcTransport`` only works when both actors were given the SAME GPU
    (cuda_ipc_transport.py:131-153), this works between any two GPUs of the NVSwitch domain.

    A tensor that already lives in the heap (created under ``comm.mem_pool()`` /
    ``symm_empty``) is published in place; any other tensor is copied once into an arena of the
    heap on the sender's stream (its lifetime ends in ``garbage_collect``)."""

    #: fraction of the heap (from the top) used as the RDT arena
    arena_fraction = 0.5
    _same_process_events = {}

    def __init__(self):
        self._arenas = {}
        self._staged = {}  # obj_id -> list of (group, offset)
        self._ipc_events = {}

    def tensor_transport_backend(self) -> str:
        return "B200_IPC"

    @staticmethod
    def is_one_sided() -> bool:
        return True

    def _arena(self, group_name: str, comm) -> "_HeapArena":
        if group_name not in self._arenas:
            _, size = comm.heap_range()
            if size == 0:
                raise RuntimeError("the B200 group was created without a symmetric heap: set heap_bytes "
                                   "(B200_HEAP_BYTES) to use the one-sided transport")
            start = int(size * (1.0 - self.arena_fraction)) // 4096 * 4096
            self._arenas[group_name] = _HeapArena(start, size - start)
        return self._arenas[group_name]

    #: which group / rank an actor publishes through; with Ray this comes from
    #: ray.experimental.collective.get_collective_groups, harnesses set it per thread
    publish_resolver = None

    def extract_tensor_transport_metadata(self, obj_id: str, rdt_object: List[torch.Tensor]) -> B200IpcTransportMetadata:
        import os

        base = super().extract_tensor_transport_metadata(obj_id, rdt_object)
        meta = B200IpcTransportMetadata(tensor_meta=base.tensor_meta, tensor_device=base.tensor_device, obj_id=obj_id,
                                        src_pid=os.getpid())
        if not rdt_object:
            return meta
        if self.publish_resolver is None:
            raise ValueError("B200IpcTransport.publish_resolver is not set: no group to publish through")
        group_name, src_rank = self.publish_resolver()
        comm = self._comm_of(group_name)
        meta.communicator_name, meta.src_rank = group_name, src_rank
        heap_base, heap_size = comm.heap_range()
        device = rdt_object[0].device
        staged = []
        for t in rdt_object:
            if t.device != device:
                raise ValueError("All tensors in an RDT object must be on the same GPU.")
            t = t.contiguous()
            nbytes = t.numel() * t.element_size()
            ptr = t.data_ptr()
            if heap_base <= ptr and ptr + nbytes <= heap_base + heap_size:
                off = ptr - heap_base  # already symmetric: publish in place
            else:
                off = self._arena(group_name, comm).alloc(nbytes)
                staged.append((group_name, off))
                comm.heap_view(off, nbytes).copy_(t.view(-1).view(torch.uint8), non_blocking=True)
            meta.heap_offsets.append(int(off))
            meta.nbytes.append(int(nbytes))
        self._staged[obj_id] = staged
        # the receiver's pull must come after everything the sender enqueued so far
        stream = torch.cuda.current_stream(device)
        plain = torch.cuda.Event()  # consumers in this process (thread actors) wait on this one:
        plain.record(stream)        # an IPC handle cannot be opened by the process that created it
        B200IpcTransport._same_process_events[(meta.src_pid, obj_id)] = plain
        try:
            shared = torch.cuda.Event(interprocess=True)
            shared.record(stream)
            meta.event_ipc_handle = shared.ipc_handle()
            self._ipc_events[obj_id] = shared  # keep it alive until garbage_collect
        except Exception:  # pragma: no cover - e.g. a driver that cannot export events
            plain.synchronize()
        return meta

    def get_communicator_metadata(self, src_actor, dst_actor, backend: Optional[str] = None) -> B200CommunicatorMetadata:
        return super().get_communicator_metadata(src_actor, dst_actor, backend if backend != "B200_IPC" else "B200")

    def recv_multiple_tensors(self, obj_id, tensor_transport_metadata, communicator_metadata,
                              target_buffers: Optional[List[torch.Tensor]] = None) -> List[torch.Tensor]:
        import os

        m = tensor_transport_metadata
        assert isinstance(m, B200IpcTransportMetadata), "metadata must come from B200IpcTransport"
        if not m.tensor_meta:
            return []
        comm = self._comm_of(m.communicator_name)
        device = torch.device("cuda", comm.device)
        tensors = target_buffers or [torch.empty(tuple(shape), dtype=dtype, device=device) for shape, dtype in m.tensor_meta]
        stream = torch.cuda.current_stream(device)
        local = B200IpcTransport._same_process_events.get((m.src_pid, m.obj_id)) if m.src_pid == os.getpid() else None
        if local is not None:
            stream.wait_event(local)  # same process (thread actors): IPC handles cannot be opened by their creator
        elif m.event_ipc_handle is not None:
            stream.wait_event(torch.cuda.Event.from_ipc_handle(device=device, handle=m.event_ipc_handle))
        for t, nbytes in zip(tensors, m.nbytes):
            if t.numel() * t.element_size() != nbytes:
                raise ValueError("target buffer size does not match the published tensor")
        comm.get_multi(tensors, m.src_rank, m.heap_offsets)  # the whole object in one launch
        return tensors

    def send_multiple_tensors(self, tensors, tensor_transport_metadata, communicator_metadata) -> None:
        raise NotImplementedError("B200_IPC is one-sided: the receiver pulls, nothing runs on the sender.")

    def garbage_collect(self, obj_id, tensor_transport_meta, tensors) -> None:
        """The object was consumed everywhere: release its arena slots and its event."""
        import os

        for group_name, off in self._staged.pop(obj_id, []):
            arena = self._arenas.get(group_name)
            if arena is not None:
                arena.free(off)
        B200IpcTransport._same_process_events.pop((os.getpid(), obj_id), None)
        self._ipc_events.pop(obj_id, None)
