"""B200Comm: one rank's communicator -- a thin torch.Tensor <-> C-ABI adapter.

All arithmetic and data movement happens in libb200_collective.so; this file only turns
tensors into (pointer, count, dtype, stream) tuples, mirrors the argument checks of the
reference backends, and performs the one-time handle exchange through a ``Store``.
"""
from __future__ import annotations

import ctypes
import threading
from typing import List, Optional, Sequence

import torch

from . import _native as N
from .store import Store, default_store

# torch dtype -> b200_dtype_t.  Same coverage as the reference's TORCH_NCCL_DTYPE_MAP
# (util/collective/collective_group/nccl_util.py:51-71); torch.bool travels as int8 there.
TORCH_DTYPE_MAP = {
    torch.bool: N.I8,
    torch.uint8: N.U8,
    torch.int8: N.I8,
    torch.int32: N.I32,
    torch.int64: N.I64,
    torch.float16: N.F16,
    torch.bfloat16: N.BF16,
    torch.float32: N.F32,
    torch.float64: N.F64,
}
for _name, _code in (("uint32", N.U32), ("uint64", N.U64)):
    if hasattr(torch, _name):
        TORCH_DTYPE_MAP[getattr(torch, _name)] = _code


def dtype_code(dtype: torch.dtype) -> int:
    try:
        return TORCH_DTYPE_MAP[dtype]
    except KeyError:
        raise ValueError(f"dtype {dtype} is not supported by the B200 collective backend") from None


def _check_cuda_contiguous(t: torch.Tensor, what: str = "tensor") -> None:
    if not isinstance(t, torch.Tensor):
        raise RuntimeError(f"{what} must be a torch.Tensor, got {type(t)}")
    if not t.is_cuda:
        # same wording as nccl_util.get_tensor_ptr (nccl_util.py:170-173)
        raise RuntimeError("Torch tensor must be on GPU when using B200 collectives.")
    if not t.is_contiguous():
        raise RuntimeError(f"{what} must be contiguous")


def _tensor_list(tensors: Sequence[torch.Tensor]):
    """(pointer array, byte-size array) of a list of contiguous CUDA tensors."""
    ptrs = (ctypes.c_void_p * max(len(tensors), 1))()
    sizes = (ctypes.c_size_t * max(len(tensors), 1))()
    for i, t in enumerate(tensors):
        _check_cuda_contiguous(t, f"tensor {i}")
        ptrs[i] = t.data_ptr()
        sizes[i] = t.numel() * t.element_size()
    return ptrs, sizes


PREMUL_DTYPES = (torch.float16, torch.bfloat16, torch.float32, torch.float64)


class PremulSum:
    """c10d's ``PREMUL_SUM(factor)``, usable as the ``op`` of every reducing ``B200Comm`` method:
    SUM over ``round_T(x_r * factor)``, each rank's input scaled as the kernel reads it.

    ``factor`` is a float or a one-element tensor.  A CPU tensor is read now, with ``.item()``.  A
    CUDA tensor must have the operand's dtype and is read by the kernels when they run, so the host
    never synchronises and a captured CUDA graph replays with the value it holds at replay time.
    A float factor is rounded to the operand's dtype, as ProcessGroupNCCL does."""

    def __init__(self, factor):
        if isinstance(factor, torch.Tensor):
            if factor.numel() != 1:
                raise RuntimeError(f"PREMUL_SUM factor must have exactly one element, got {factor.numel()}")
            if not factor.is_cuda:
                factor = float(factor.item())
        elif isinstance(factor, (int, float)) and not isinstance(factor, bool):
            factor = float(factor)
        else:
            raise RuntimeError(f"PREMUL_SUM factor must be a float or a one-element tensor, got {type(factor)}")
        self.factor = factor

    @property
    def device_factor(self) -> Optional[torch.Tensor]:
        """The CUDA factor tensor the kernels read, or None for a host factor."""
        return self.factor if isinstance(self.factor, torch.Tensor) else None

    def __repr__(self) -> str:
        return f"PremulSum({self.factor!r})"


class SymmetricTensorHolder:
    """Exposes a slice of the symmetric heap through __cuda_array_interface__."""

    def __init__(self, ptr: int, nbytes: int, owner):
        self._owner = owner  # keeps the communicator alive
        self.__cuda_array_interface__ = {
            "shape": (nbytes,),
            "typestr": "|u1",
            "data": (ptr, False),
            "version": 3,
            "strides": None,
        }


class B200Comm:
    """One rank of a B200 collective group.

    Args:
        world_size, rank: group geometry (<= 8 ranks: one NVSwitch domain).
        device: CUDA device ordinal of this rank in this process.
        store: rendezvous store shared by all ranks (default: ``default_store()``).
        group_name: namespaces the store keys, so several groups can coexist
            (the reference tests create 5 at once, SURVEY Q4).
        staging_bytes / heap_bytes / inbox_bytes / enable_multicast / timeout_ms:
            see ``b200_config_t`` in include/b200_collective.h.
    """

    def __init__(
        self,
        world_size: int,
        rank: int,
        device: int,
        store: Optional[Store] = None,
        group_name: str = "default",
        staging_bytes: int = 0,
        heap_bytes: int = 0,
        inbox_bytes: int = 0,
        enable_multicast: bool = True,
        timeout_ms: int = 0,
        rendezvous_timeout_s: float = 180.0,
    ):
        self._lib = N.load()
        self._h = ctypes.c_void_p()
        self.world_size = int(world_size)
        self.rank = int(rank)
        self.device = int(device)
        self.group_name = group_name
        self._closed = False
        self._lock = threading.Lock()
        cfg = N.B200Config(int(staging_bytes), int(heap_bytes), int(inbox_bytes),
                           1 if enable_multicast else 0, int(timeout_ms))
        N.check(self._lib.b200_comm_create(self.world_size, self.rank, self.device,
                                           ctypes.byref(cfg), ctypes.byref(self._h)))
        try:
            store = store if store is not None else default_store()
            blob = ctypes.create_string_buffer(N.HANDLE_BYTES)
            N.check(self._lib.b200_comm_export_handle(self._h, blob))
            prefix = f"b200/{group_name}/handle/"
            store.set(prefix + str(self.rank), blob.raw)
            blobs = b"".join(store.get(prefix + str(p), rendezvous_timeout_s) for p in range(self.world_size))
            N.check(self._lib.b200_comm_connect(self._h, blobs))
            # every rank has read every handle once connect() returned on all ranks; the
            # owner removes its key so the name can be reused (destroy / re-init, SURVEY Q4)
            store.delete(prefix + str(self.rank))
        except BaseException:
            self._lib.b200_comm_destroy(self._h)
            self._h = ctypes.c_void_p()
            self._closed = True
            raise

    # ------------------------------------------------------------------ helpers
    def _stream(self, stream: Optional[torch.cuda.Stream] = None) -> int:
        """Raw handle of the stream an op is enqueued on (default: this device's current stream).

        The kernels read the communicator's launch counter at entry and rely on STREAM ORDER for
        their epoch and slot parity (include/b200_collective.h: "collectives of one communicator
        must be stream-ordered").  A caller that switches streams between two ops of the same
        communicator (ADVICE r01) is therefore ordered here on the device: the new stream waits for
        an event recorded at the tail of the previous one.  Costs nothing while the stream stays
        the same."""
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        last = getattr(self, "_last_stream", None)
        if last is not None and last.cuda_stream != st.cuda_stream:
            ev = torch.cuda.Event()
            ev.record(last)
            st.wait_event(ev)
        self._last_stream = st
        return st.cuda_stream

    @property
    def has_multicast(self) -> bool:
        return bool(self._lib.b200_comm_has_multicast(self._h))

    @property
    def launch_count(self) -> int:
        return int(self._lib.b200_comm_launch_count(self._h))

    def set_blocks(self, nblocks: int) -> None:
        N.check(self._lib.b200_comm_set_blocks(self._h, int(nblocks)))

    def set_param(self, param: int, value: int) -> None:
        """Tuning knob (``N.PARAM_*``); must be set identically on every rank."""
        N.check(self._lib.b200_comm_set_param(self._h, int(param), int(value)))

    def trace_enable(self, capacity: int) -> None:
        """Profiling aid: let instrumented kernels record up to ``capacity`` timestamped events."""
        N.check(self._lib.b200_comm_trace_enable(self._h, int(capacity)))

    def trace_read(self, max_events: int = 1 << 20, reset: bool = True):
        """-> list of (ns, cta, event, arg) recorded since the last reset (synchronises the device)."""
        buf = (ctypes.c_ulonglong * (2 * max_events))()
        n = self._lib.b200_comm_trace_read(self._h, buf, max_events, 1 if reset else 0)
        if n < 0:
            N.check(n)
        return [(buf[2 * i], buf[2 * i + 1] >> 40, (buf[2 * i + 1] >> 32) & 0xFF, buf[2 * i + 1] & 0xFFFFFFFF)
                for i in range(n)]

    def status(self) -> int:
        return int(self._lib.b200_comm_status(self._h))

    def check_status(self) -> None:
        """Raise if a kernel of this communicator gave up (abort / watchdog).  Only
        meaningful after the stream was synchronised."""
        st = self.status()
        if st == N.ERR_ABORTED:
            raise N.B200AbortedError(st, "communicator aborted")
        if st == N.ERR_TIMEOUT:
            raise N.B200TimeoutError(st, "a peer did not arrive before the device watchdog expired")
        if st != 0:
            raise N.B200Error(st, N.last_error())

    # ------------------------------------------------------------------ symmetric heap
    def symm_empty(self, shape, dtype=torch.float32) -> torch.Tensor:
        """Collectively allocate a tensor in the symmetric heap (zero-copy operand)."""
        shape = tuple(int(s) for s in (shape if isinstance(shape, (tuple, list, torch.Size)) else (shape,)))
        numel = 1
        for s in shape:
            numel *= s
        nbytes = max(numel * torch.empty((), dtype=dtype).element_size(), 1)
        ptr = ctypes.c_void_p()
        N.check(self._lib.b200_symm_alloc(self._h, nbytes, ctypes.byref(ptr)))
        holder = SymmetricTensorHolder(ptr.value, nbytes, self)
        raw = torch.as_tensor(holder, device=torch.device("cuda", self.device))
        t = raw.view(dtype)[:numel].view(shape)
        t._b200_holder = holder  # noqa: SLF001 - keep the mapping alive with the tensor
        return t

    def mem_pool(self):
        """A ``torch.cuda.MemPool`` whose memory is this communicator's symmetric heap: tensors
        created under ``with torch.cuda.use_mem_pool(comm.mem_pool()):`` are ordinary torch
        tensors, yet collectives reduce them in place with no staging copies (what
        ``ncclMemAlloc`` + buffer registration buys on the NCCL side).  Every rank must create
        the same tensors in the same order.  One communicator per process can back the pool."""
        if getattr(self, "_pool", None) is None:
            from torch.cuda.memory import CUDAPluggableAllocator

            N.check(self._lib.b200_pool_bind(self._h))
            self._allocator = CUDAPluggableAllocator(str(N.LIB_PATH), "b200_pool_alloc", "b200_pool_free")
            self._pool = torch.cuda.MemPool(self._allocator.allocator())
        return self._pool

    def symm_reset(self) -> None:
        N.check(self._lib.b200_symm_reset(self._h))

    def symm_contains(self, t: torch.Tensor) -> bool:
        return bool(self._lib.b200_symm_contains(self._h, t.data_ptr(), t.numel() * t.element_size()))

    def _with_op(self, op, dtype: torch.dtype, enqueue) -> None:
        """``enqueue(op_code)``.  A ``PremulSum`` becomes a native op for ``dtype`` that lives for this
        call only: the kernels copy the factor (or its device address) into their arguments."""
        if not isinstance(op, PremulSum):
            enqueue(int(op))
            return
        if dtype not in PREMUL_DTYPES:
            # ProcessGroupNCCL's refusal for an integer (or bool) operand
            raise RuntimeError(f"Cannot use ReduceOp.PREMUL_SUM with {dtype}: "
                               "PreMulSum Data type must be half, float, bfloat16 or double")
        f = op.device_factor
        handle = ctypes.c_int()
        if f is not None:
            if f.dtype != dtype or f.numel() != 1:
                raise RuntimeError(f"PREMUL_SUM factor tensor must hold one {dtype} element, got "
                                   f"{f.numel()} of {f.dtype}")
            N.check(self._lib.b200_op_create_premul(self._h, f.data_ptr(), dtype_code(dtype), N.PREMUL_DEVICE,
                                                    ctypes.byref(handle)))
        else:
            host = torch.tensor([op.factor], dtype=dtype)
            N.check(self._lib.b200_op_create_premul(self._h, host.data_ptr(), dtype_code(dtype), N.PREMUL_HOST,
                                                    ctypes.byref(handle)))
        try:
            enqueue(handle.value)
        finally:
            self._lib.b200_op_destroy(self._h, handle.value)
        if f is not None:
            f.record_stream(torch.cuda.current_stream(self.device))

    # ------------------------------------------------------------------ collectives
    def allreduce(self, tensor: torch.Tensor, op: int = N.SUM, out: Optional[torch.Tensor] = None,
                  algo: int = N.ALGO_AUTO) -> None:
        _check_cuda_contiguous(tensor)
        out = tensor if out is None else out
        if out is not tensor:
            _check_cuda_contiguous(out, "output tensor")
            if out.dtype != tensor.dtype or out.numel() != tensor.numel():
                raise RuntimeError("allreduce output must match the input's dtype and size")
        self._with_op(op, tensor.dtype, lambda code: N.check(self._lib.b200_allreduce(
            self._h, tensor.data_ptr(), out.data_ptr(), tensor.numel(), dtype_code(tensor.dtype), code, int(algo),
            self._stream())))

    def allgather(self, outs: Sequence[torch.Tensor], tensor: torch.Tensor) -> None:
        _check_cuda_contiguous(tensor)
        if len(outs) != self.world_size:
            raise RuntimeError("The length of the tensor list operands to allgather must be equal to world_size.")
        arr = (ctypes.c_void_p * N.MAX_RANKS)()
        for i, o in enumerate(outs):
            _check_cuda_contiguous(o, "output tensor")
            if o.dtype != tensor.dtype or o.numel() != tensor.numel():
                raise RuntimeError("All tensor operands to allgather must have the same dtype and size.")
            arr[i] = o.data_ptr()
        N.check(self._lib.b200_allgather(self._h, tensor.data_ptr(), arr, tensor.numel(),
                                         dtype_code(tensor.dtype), self._stream()))

    def allgather_into(self, out: torch.Tensor, tensor: torch.Tensor) -> None:
        """out = concat over ranks along dim 0 (the Compiled-Graph layout, collective_node.py:198-206)."""
        _check_cuda_contiguous(tensor)
        _check_cuda_contiguous(out, "output tensor")
        if out.dtype != tensor.dtype or out.numel() != tensor.numel() * self.world_size:
            raise RuntimeError("allgather output must hold world_size copies of the input")
        arr = (ctypes.c_void_p * N.MAX_RANKS)()
        step = tensor.numel() * tensor.element_size()
        for p in range(self.world_size):
            arr[p] = out.data_ptr() + p * step
        N.check(self._lib.b200_allgather(self._h, tensor.data_ptr(), arr, tensor.numel(),
                                         dtype_code(tensor.dtype), self._stream()))

    def reducescatter(self, out: torch.Tensor, ins: Sequence[torch.Tensor], op: int = N.SUM) -> None:
        _check_cuda_contiguous(out, "output tensor")
        if len(ins) != self.world_size:
            raise RuntimeError("The length of the tensor list operands to reducescatter must be equal to world_size.")
        arr = (ctypes.c_void_p * N.MAX_RANKS)()
        for i, t in enumerate(ins):
            _check_cuda_contiguous(t)
            if t.dtype != out.dtype or t.numel() != out.numel():
                raise RuntimeError("All tensor operands to reducescatter must have the same dtype and size.")
            arr[i] = t.data_ptr()
        self._with_op(op, out.dtype, lambda code: N.check(self._lib.b200_reducescatter(
            self._h, arr, out.data_ptr(), out.numel(), dtype_code(out.dtype), code, self._stream())))

    def reducescatter_from(self, out: torch.Tensor, tensor: torch.Tensor, op: int = N.SUM) -> None:
        """out = reduce over ranks of this rank's 1/world slice of ``tensor`` along dim 0
        (the Compiled-Graph layout, collective_node.py:207-219)."""
        _check_cuda_contiguous(tensor)
        _check_cuda_contiguous(out, "output tensor")
        if out.dtype != tensor.dtype or out.numel() * self.world_size != tensor.numel():
            raise RuntimeError("reducescatter input must hold world_size slices of the output size")
        arr = (ctypes.c_void_p * N.MAX_RANKS)()
        step = out.numel() * out.element_size()
        for p in range(self.world_size):
            arr[p] = tensor.data_ptr() + p * step
        self._with_op(op, out.dtype, lambda code: N.check(self._lib.b200_reducescatter(
            self._h, arr, out.data_ptr(), out.numel(), dtype_code(out.dtype), code, self._stream())))

    def _uneven_parts(self, parts: Sequence[torch.Tensor], own: torch.Tensor, what: str, own_what: str):
        """(pointer array, count array) of the world_size parts of an uneven all-gather or
        reduce-scatter; the counts are the parts' numels and must match ``own`` at this rank."""
        if len(parts) != self.world_size:
            raise RuntimeError(f"The length of the tensor list operands to {what} must be equal to world_size.")
        ptrs, counts = (ctypes.c_void_p * N.MAX_RANKS)(), (ctypes.c_size_t * N.MAX_RANKS)()
        for p, t in enumerate(parts):
            _check_cuda_contiguous(t, f"tensor {p}")
            if t.dtype != own.dtype:
                raise RuntimeError(f"All tensor operands to {what} must have the same dtype.")
            ptrs[p] = t.data_ptr()
            counts[p] = t.numel()
        if parts[self.rank].numel() != own.numel():
            raise RuntimeError(f"{what}: tensor {self.rank} (this rank's part) has {parts[self.rank].numel()} "
                               f"elements, the {own_what} {own.numel()}")
        return ptrs, counts

    def allgatherv(self, outs: Sequence[torch.Tensor], tensor: torch.Tensor) -> None:
        """``allgather`` with a size per rank: ``outs[p]`` receives rank p's ``tensor``, whose size
        may differ per rank.  Every rank passes outputs of the same sizes, and ``outs[this rank]``
        has this rank's size (it may be ``tensor`` itself).  Equal sizes run ``allgather``'s
        launches; otherwise one launch per window of staging_bytes / 16 units of the largest part."""
        _check_cuda_contiguous(tensor)
        ptrs, counts = self._uneven_parts(outs, tensor, "allgatherv", "input has")
        N.check(self._lib.b200_allgatherv(self._h, tensor.data_ptr(), counts, ptrs, dtype_code(tensor.dtype),
                                          self._stream()))

    def reducescatterv(self, out: torch.Tensor, ins: Sequence[torch.Tensor], op: int = N.SUM) -> None:
        """``reducescatter`` with a size per rank: ``out`` = op over ranks of that rank's
        ``ins[this rank]``, reduced rank-ascending; ``ins[q]`` has rank q's output size, the same on
        every rank, and ``ins[this rank]`` may be ``out`` itself.  Equal sizes run
        ``reducescatter``'s launches."""
        _check_cuda_contiguous(out, "output tensor")
        ptrs, counts = self._uneven_parts(ins, out, "reducescatterv", "output has")
        self._with_op(op, out.dtype, lambda code: N.check(self._lib.b200_reducescatterv(
            self._h, ptrs, counts, out.data_ptr(), dtype_code(out.dtype), code, self._stream())))

    def allgather_multi(self, out_lists: Sequence[Sequence[torch.Tensor]], tensors: Sequence[torch.Tensor]) -> None:
        """``allgather`` of a list of tensors (any dtypes): ``out_lists[i][p]`` receives rank p's
        ``tensors[i]``.  One launch per staging slot of packed data (per ``N.P2P_TABLE_MAX``
        non-empty tensors at most) instead of one per tensor.  Every rank passes tensors of the same
        byte sizes in the same order; ``out_lists[i][this rank]`` may be ``tensors[i]`` itself."""
        n = self.world_size
        if len(out_lists) != len(tensors):
            raise RuntimeError(f"allgather_multi got {len(out_lists)} output lists for {len(tensors)} tensors")
        ptrs, sizes = _tensor_list(tensors)
        outs = (ctypes.c_void_p * max(len(tensors) * n, 1))()
        for i, (lst, t) in enumerate(zip(out_lists, tensors)):
            if len(lst) != n:
                raise RuntimeError("The length of the tensor list operands to allgather must be equal to world_size.")
            for p, o in enumerate(lst):
                _check_cuda_contiguous(o, "output tensor")
                if o.dtype != t.dtype or o.numel() != t.numel():
                    raise RuntimeError("All tensor operands to allgather must have the same dtype and size.")
                outs[i * n + p] = o.data_ptr()
        if not tensors:
            return
        N.check(self._lib.b200_allgather_multi(self._h, ptrs, sizes, len(tensors), outs, self._stream()))

    def allgather_into_multi(self, outs: Sequence[torch.Tensor], tensors: Sequence[torch.Tensor]) -> None:
        """``allgather_into`` of a list of tensors (any dtypes) in one ``b200_allgather_multi`` call:
        ``outs[i]`` is the rank-major concatenation of every rank's ``tensors[i]`` (the
        ``all_gather_into_tensor`` layout)."""
        n = self.world_size
        if len(outs) != len(tensors):
            raise RuntimeError(f"allgather_into_multi got {len(outs)} outputs for {len(tensors)} tensors")
        ptrs, sizes = _tensor_list(tensors)
        arr = (ctypes.c_void_p * max(len(tensors) * n, 1))()
        for i, (o, t) in enumerate(zip(outs, tensors)):
            _check_cuda_contiguous(o, "output tensor")
            if o.dtype != t.dtype or o.numel() != t.numel() * n:
                raise RuntimeError("allgather output must hold world_size copies of the input")
            for p in range(n):
                arr[i * n + p] = o.data_ptr() + p * sizes[i]
        if not tensors:
            return
        N.check(self._lib.b200_allgather_multi(self._h, ptrs, sizes, len(tensors), arr, self._stream()))

    def _reducescatter_multi(self, outs: Sequence[torch.Tensor], ins, op: int) -> None:
        """outs[i] = reduce over ranks of (that rank's ins[i * world_size + this rank]); ``ins`` is a
        flat pointer array."""
        ptrs = (ctypes.c_void_p * max(len(outs), 1))()
        counts = (ctypes.c_size_t * max(len(outs), 1))()
        for i, o in enumerate(outs):
            ptrs[i] = o.data_ptr()
            counts[i] = o.numel()
        if not outs:
            return
        self._with_op(op, outs[0].dtype, lambda code: N.check(self._lib.b200_reducescatter_multi(
            self._h, ins, ptrs, counts, len(outs), dtype_code(outs[0].dtype), code, self._stream())))

    def _check_rs_outputs(self, outs: Sequence[torch.Tensor], n_in: int) -> None:
        if len(outs) != n_in:
            raise RuntimeError(f"reducescatter list got {len(outs)} outputs for {n_in} inputs")
        for i, o in enumerate(outs):
            _check_cuda_contiguous(o, f"output tensor {i}")
            if o.dtype != outs[0].dtype:
                raise RuntimeError("All tensor operands to a list reducescatter must have the same dtype.")

    def reducescatter_multi(self, outs: Sequence[torch.Tensor], in_lists: Sequence[Sequence[torch.Tensor]],
                            op: int = N.SUM) -> None:
        """``reducescatter`` of a list of tensors of one dtype: ``outs[i]`` = op over ranks of that
        rank's ``in_lists[i][this rank]``, bit-identical to one ``reducescatter`` per tensor, in one
        launch per window of packed data.  ``outs[i]`` may be ``in_lists[i][this rank]`` itself."""
        n = self.world_size
        self._check_rs_outputs(outs, len(in_lists))
        arr = (ctypes.c_void_p * max(len(outs) * n, 1))()
        for i, (o, lst) in enumerate(zip(outs, in_lists)):
            if len(lst) != n:
                raise RuntimeError("The length of the tensor list operands to reducescatter must be equal to world_size.")
            for q, t in enumerate(lst):
                _check_cuda_contiguous(t)
                if t.dtype != o.dtype or t.numel() != o.numel():
                    raise RuntimeError("All tensor operands to reducescatter must have the same dtype and size.")
                arr[i * n + q] = t.data_ptr()
        self._reducescatter_multi(outs, arr, op)

    def reducescatter_from_multi(self, outs: Sequence[torch.Tensor], tensors: Sequence[torch.Tensor],
                                 op: int = N.SUM) -> None:
        """``reducescatter_from`` of a list of tensors of one dtype in one ``b200_reducescatter_multi``
        call: ``outs[i]`` = op over ranks of this rank's 1/world slice of ``tensors[i]`` (the
        ``reduce_scatter_tensor`` layout)."""
        n = self.world_size
        self._check_rs_outputs(outs, len(tensors))
        arr = (ctypes.c_void_p * max(len(outs) * n, 1))()
        for i, (o, t) in enumerate(zip(outs, tensors)):
            _check_cuda_contiguous(t, f"tensor {i}")
            if t.dtype != o.dtype or o.numel() * n != t.numel():
                raise RuntimeError("reducescatter input must hold world_size slices of the output size")
            step = o.numel() * o.element_size()
            for q in range(n):
                arr[i * n + q] = t.data_ptr() + q * step
        self._reducescatter_multi(outs, arr, op)

    def broadcast(self, tensor: torch.Tensor, root: int = 0) -> None:
        _check_cuda_contiguous(tensor)
        N.check(self._lib.b200_broadcast(self._h, tensor.data_ptr(), tensor.numel(),
                                         dtype_code(tensor.dtype), int(root), self._stream()))

    def broadcast_multi(self, tensors: Sequence[torch.Tensor], root: int = 0,
                        stream: Optional[torch.cuda.Stream] = None) -> None:
        """In-place broadcast of a list of tensors (any dtypes) from ``root``: one launch per
        staging slot of packed data (per ``N.P2P_TABLE_MAX`` non-empty tensors at most) instead of
        one per tensor.  Every rank passes tensors of the same byte sizes in the same order."""
        ptrs, sizes = _tensor_list(tensors)
        if not tensors:
            return
        N.check(self._lib.b200_broadcast_multi(self._h, ptrs, sizes, len(tensors), int(root),
                                               stream.cuda_stream if stream is not None else self._stream()))

    def reduce(self, tensor: torch.Tensor, root: int = 0, op: int = N.SUM) -> None:
        _check_cuda_contiguous(tensor)
        self._with_op(op, tensor.dtype, lambda code: N.check(self._lib.b200_reduce(
            self._h, tensor.data_ptr(), tensor.numel(), dtype_code(tensor.dtype), code, int(root), self._stream())))

    def barrier(self) -> None:
        N.check(self._lib.b200_barrier(self._h, self._stream()))

    def alltoall(self, outs: Sequence[Optional[torch.Tensor]], ins: Sequence[Optional[torch.Tensor]]) -> None:
        """All-to-all(v) in one launch: ``ins[p]`` goes to rank p, ``outs[p]`` receives rank p's
        ``ins[this rank]``.  ``None`` means nothing moves in that direction with that peer; sizes
        may differ per peer, but every rank must agree on the size of each pair's message."""
        n = self.world_size
        if len(outs) != n or len(ins) != n:
            raise RuntimeError("The length of the tensor list operands to alltoall must be equal to world_size.")
        in_ptrs, out_ptrs = (ctypes.c_void_p * n)(), (ctypes.c_void_p * n)()
        send_counts, recv_counts = (ctypes.c_size_t * n)(), (ctypes.c_size_t * n)()
        dtype = None
        for tensors, ptrs, counts, what in ((ins, in_ptrs, send_counts, "input tensor"),
                                           (outs, out_ptrs, recv_counts, "output tensor")):
            for p, t in enumerate(tensors):
                if t is None:
                    continue
                _check_cuda_contiguous(t, what)
                if dtype is None:
                    dtype = t.dtype
                elif t.dtype != dtype:
                    raise RuntimeError("All tensor operands to alltoall must have the same dtype.")
                ptrs[p] = t.data_ptr()
                counts[p] = t.numel()
        if dtype is None:
            return
        N.check(self._lib.b200_alltoall(self._h, in_ptrs, send_counts, out_ptrs, recv_counts, dtype_code(dtype),
                                        self._stream()))

    def send(self, tensor: torch.Tensor, peer: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Enqueue a send on ``stream`` (default: the current stream of this rank's device)."""
        _check_cuda_contiguous(tensor)
        st = self._lib.b200_send(self._h, tensor.data_ptr(), tensor.numel() * tensor.element_size(), int(peer),
                                 stream.cuda_stream if stream is not None else self._stream())
        if st:
            N.check(st)

    def recv(self, tensor: torch.Tensor, peer: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        _check_cuda_contiguous(tensor)
        st = self._lib.b200_recv(self._h, tensor.data_ptr(), tensor.numel() * tensor.element_size(), int(peer),
                                 stream.cuda_stream if stream is not None else self._stream())
        if st:
            N.check(st)

    def send_multi(self, tensors: Sequence[torch.Tensor], peer: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Send a list of tensors (any dtypes) as one message: one launch per ``N.P2P_TABLE_MAX``
        non-empty tensors instead of one per tensor.  The peer's ``recv_multi`` must pass tensors
        of the same byte sizes in the same order."""
        ptrs, sizes = _tensor_list(tensors)
        if not tensors:
            return
        N.check(self._lib.b200_send_multi(self._h, ptrs, sizes, len(tensors), int(peer),
                                          stream.cuda_stream if stream is not None else self._stream()))

    def recv_multi(self, tensors: Sequence[torch.Tensor], peer: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Receive what the peer's ``send_multi`` sent into ``tensors`` (same byte sizes, same order)."""
        ptrs, sizes = _tensor_list(tensors)
        if not tensors:
            return
        N.check(self._lib.b200_recv_multi(self._h, ptrs, sizes, len(tensors), int(peer),
                                          stream.cuda_stream if stream is not None else self._stream()))

    def p2p_batch(self, ops: Sequence, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Run a list of sends and receives as one launch (``ncclGroupStart/End`` of sends and
        receives).  ``ops`` holds ``(is_send, tensor, peer)`` triples; tensors are contiguous CUDA
        tensors of any dtype and move as raw bytes.  Each op is the message ``send`` / ``recv`` would
        make, so it pairs with a plain ``send`` / ``recv`` on the peer or with an op of the peer's
        batch; ops to one (peer, direction) are consecutive messages in list order.  A bidirectional
        or ring exchange larger than the inbox completes here, where plain calls in the wrong order
        would wait on each other.  At most ``N.P2P_TABLE_MAX`` ops per batch."""
        ops = list(ops)
        if not ops:
            return
        n = len(ops)
        bufs, sizes = (ctypes.c_void_p * n)(), (ctypes.c_size_t * n)()
        peers, sends = (ctypes.c_int * n)(), (ctypes.c_int * n)()
        for i, (is_send, t, peer) in enumerate(ops):
            _check_cuda_contiguous(t, f"tensor {i}")
            bufs[i] = t.data_ptr()
            sizes[i] = t.numel() * t.element_size()
            peers[i] = int(peer)
            sends[i] = 1 if is_send else 0
        N.check(self._lib.b200_p2p_batch(self._h, bufs, sizes, peers, sends, n,
                                         stream.cuda_stream if stream is not None else self._stream()))

    def send_ptr(self, ptr: int, nbytes: int, peer: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """send() from a raw device-visible address (e.g. pinned host memory under unified
        addressing: the Compiled-Graph channel keeps its metadata header there)."""
        st = self._lib.b200_send(self._h, ptr, int(nbytes), int(peer),
                                 stream.cuda_stream if stream is not None else self._stream())
        if st:
            N.check(st)

    def recv_ptr(self, ptr: int, nbytes: int, peer: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        st = self._lib.b200_recv(self._h, ptr, int(nbytes), int(peer),
                                 stream.cuda_stream if stream is not None else self._stream())
        if st:
            N.check(st)

    # ------------------------------------------------------------------ one-sided get
    def heap_range(self):
        """(base address, bytes) of this rank's symmetric heap."""
        base, nbytes = ctypes.c_void_p(), ctypes.c_size_t()
        N.check(self._lib.b200_symm_base(self._h, ctypes.byref(base), ctypes.byref(nbytes)))
        return int(base.value or 0), int(nbytes.value)

    def heap_view(self, offset: int, nbytes: int) -> torch.Tensor:
        """uint8 tensor over [offset, offset+nbytes) of this rank's heap (no allocation bookkeeping)."""
        base, size = self.heap_range()
        if offset < 0 or offset + nbytes > size:
            raise ValueError("range outside the symmetric heap")
        holder = SymmetricTensorHolder(base + offset, max(nbytes, 1), self)
        t = torch.as_tensor(holder, device=torch.device("cuda", self.device))[:nbytes]
        t._b200_holder = holder  # noqa: SLF001
        return t

    def get(self, dst: torch.Tensor, src_rank: int, src_heap_offset: int,
            stream: Optional[torch.cuda.Stream] = None) -> None:
        """Pull ``dst.nbytes`` bytes from ``src_rank``'s symmetric heap into ``dst``; only this rank
        runs a kernel."""
        _check_cuda_contiguous(dst)
        if src_heap_offset < 0:
            raise ValueError("range outside the symmetric heap")
        N.check(self._lib.b200_get(self._h, dst.data_ptr(), int(src_rank), int(src_heap_offset),
                                   dst.numel() * dst.element_size(),
                                   stream.cuda_stream if stream is not None else self._stream()))

    def get_multi(self, dsts: Sequence[torch.Tensor], src_rank: int, src_heap_offsets: Sequence[int],
                  stream: Optional[torch.cuda.Stream] = None) -> None:
        """``get`` for a list: ``dsts[i]`` receives ``dsts[i].nbytes`` bytes from ``src_heap_offsets[i]``
        of ``src_rank``'s heap, one launch per ``N.P2P_TABLE_MAX`` non-empty tensors."""
        if len(dsts) != len(src_heap_offsets):
            raise ValueError(f"get_multi got {len(dsts)} destination tensors but {len(src_heap_offsets)} offsets")
        ptrs, sizes = _tensor_list(dsts)
        if not dsts:
            return
        offs = (ctypes.c_size_t * len(dsts))(*[int(o) for o in src_heap_offsets])
        N.check(self._lib.b200_get_multi(self._h, ptrs, int(src_rank), offs, sizes, len(dsts),
                                         stream.cuda_stream if stream is not None else self._stream()))

    def grad_allreduce(self, grad: torch.Tensor, scale: float, wire_dtype: torch.dtype = torch.bfloat16) -> None:
        """Fused ``grad = sum_r wire(grad_r * scale)`` on a flat fp32 bucket (SURVEY K8)."""
        _check_cuda_contiguous(grad)
        if grad.dtype != torch.float32:
            raise RuntimeError("grad_allreduce expects a float32 bucket")
        N.check(self._lib.b200_grad_allreduce(self._h, grad.data_ptr(), grad.numel(), float(scale),
                                              dtype_code(wire_dtype), self._stream()))

    def grad_reducescatter(self, out: torch.Tensor, grad: torch.Tensor, scale: float,
                           wire_dtype: torch.dtype = torch.bfloat16) -> None:
        """Fused sharded gradient sync (the FSDP / ZeRO counterpart of ``grad_allreduce``):
        ``out = sum_r wire(grad_r[this rank's 1/world slice] * scale)``, cast back to fp32.
        ``out`` may be this rank's own slice of ``grad`` (in place), but no other part of it."""
        _check_cuda_contiguous(grad)
        _check_cuda_contiguous(out, "output tensor")
        if grad.dtype != torch.float32 or out.dtype != torch.float32:
            raise RuntimeError("grad_reducescatter expects float32 gradient and output tensors")
        if grad.numel() != out.numel() * self.world_size:
            raise RuntimeError("grad_reducescatter input must hold world_size slices of the output size")
        N.check(self._lib.b200_grad_reducescatter(self._h, grad.data_ptr(), out.data_ptr(), out.numel(),
                                                  float(scale), dtype_code(wire_dtype), self._stream()))

    def allreduce_multi(self, tensors: List[torch.Tensor], op: int = N.SUM) -> None:
        if not tensors:
            return
        dt = tensors[0].dtype
        ptrs = (ctypes.c_void_p * len(tensors))()
        counts = (ctypes.c_size_t * len(tensors))()
        for i, t in enumerate(tensors):
            _check_cuda_contiguous(t)
            if t.dtype != dt:
                raise ValueError("Expected all input tensors to have the same dtype")
            ptrs[i] = t.data_ptr()
            counts[i] = t.numel()
        self._with_op(op, dt, lambda code: N.check(self._lib.b200_allreduce_multi(
            self._h, ptrs, counts, len(tensors), dtype_code(dt), code, self._stream())))

    # ------------------------------------------------------------------ lifecycle
    def abort(self) -> None:
        if self._h:
            self._lib.b200_comm_abort(self._h)

    def destroy(self) -> None:
        with self._lock:
            if self._closed:
                return
            self._closed = True
        self._lib.b200_comm_destroy(self._h)
        self._h = ctypes.c_void_p()

    @property
    def closed(self) -> bool:
        return self._closed

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass
