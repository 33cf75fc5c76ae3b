"""c10d process group backed by libb200_collective.so (boundary B4).

``TorchTrainer`` and RLlib's ``LearnerGroup`` never call ``ray.util.collective``: they run
``dist.init_process_group(backend=...)`` on every worker (python/ray/train/torch/config.py:
144) and wrap the model in ``DistributedDataParallel`` (train_loop_utils.py:456-480;
rllib/core/learner/torch/torch_learner.py:535-563), so gradient all-reduce, the initial
parameter broadcast and the per-forward buffer broadcasts all go through the *c10d*
process group.  ``register_b200_backend()`` makes ``backend="b200"`` (or
``"cpu:gloo,cuda:b200"``) a valid choice there; every CUDA collective the DDP reducer and
user code issue then lands in the hand-written kernels, with no NCCL communicator created.

Stream semantics follow ProcessGroupNCCL: each op runs on a dedicated communication stream
ordered after the caller's current stream; ``Work.wait()`` and the returned CUDA-aware
``Future`` order the caller's stream after the op without blocking the host, which is what
lets DDP overlap bucket all-reduces with the rest of the backward pass.
"""
from __future__ import annotations

import datetime
import threading
from typing import List, Optional

import torch
import torch.distributed as dist

from .. import _native as N
from ..comm import B200Comm, PremulSum
from ..store import TorchDistStore

BACKEND_NAME = "b200"

_group_counter = 0
_counter_lock = threading.Lock()


def _op_code(reduce_op):
    """The B200Comm op of a c10d ReduceOp: an ``N.*`` code, or a ``PremulSum`` carrying the factor of
    ``dist._make_nccl_premul_sum(factor)`` (a float or a one-element tensor)."""
    if reduce_op == dist.ReduceOp.PREMUL_SUM:
        return PremulSum(reduce_op.__getstate__()[1])
    table = ((dist.ReduceOp.SUM, N.SUM), (dist.ReduceOp.PRODUCT, N.PROD), (dist.ReduceOp.MIN, N.MIN),
             (dist.ReduceOp.MAX, N.MAX), (dist.ReduceOp.AVG, N.AVG))
    for torch_op, code in table:
        if reduce_op == torch_op:
            return code
    raise RuntimeError(f"ReduceOp {reduce_op} is not supported by the b200 backend")


class B200Work(dist._Work):
    """Completion handle of one enqueued op (c10d::Work).

    Error model (ProcessGroupNCCL's async error handling, which the reference's TorchConfig relies
    on -- python/ray/train/torch/config.py:123-150): a kernel that gives up on a peer (device
    watchdog / abort) writes a sticky status word that the host can read without a CUDA call.
    ``wait()`` / ``is_success()`` / ``exception()`` surface it, and the native layer refuses every
    later launch on that communicator, so a late or dead rank produces an exception on its peers
    instead of silently diverging replicas.
    """

    def __init__(self, result, device: Optional[torch.device], done_event: Optional[torch.cuda.Event],
                 comm_stream: Optional[torch.cuda.Stream], comm: Optional[B200Comm] = None,
                 default_timeout: Optional[datetime.timedelta] = None):
        super().__init__()
        self._result = result
        self._device = device
        self._event = done_event
        self._comm = comm
        self._default_timeout = default_timeout
        if device is not None and device.type == "cuda":
            self._future = torch.futures.Future(devices=[device])
            # set_result records the completion on the *current* stream: make that the comm stream
            with torch.cuda.stream(comm_stream):
                self._future.set_result(result)
        else:
            self._future = torch.futures.Future()
            self._future.set_result(result)

    def _error(self) -> Optional[BaseException]:
        if self._comm is None or self._comm.closed:
            return None
        st = self._comm.status()
        if st == 0:
            return None
        if st == N.ERR_TIMEOUT:
            return N.B200TimeoutError(st, "a b200 collective timed out waiting for a peer (device watchdog)")
        if st == N.ERR_ABORTED:
            return N.B200AbortedError(st, "the b200 communicator was aborted")
        return N.B200Error(st, N.last_error())

    def wait(self, timeout=None) -> bool:
        """Stream-ordered like ProcessGroupNCCL: the caller's current stream waits for the op, the
        host does not -- unless a ``timeout`` is given, in which case the host blocks until the op
        finished or the timeout expired (c10d raises in that case; so does this)."""
        if self._event is None:
            return True
        if timeout is not None and timeout != datetime.timedelta(0):
            import time

            secs = timeout.total_seconds() if isinstance(timeout, datetime.timedelta) else float(timeout)
            start = time.monotonic()
            deadline = start + secs
            while not self._event.query():
                now = time.monotonic()
                if now - start > 2e-3:
                    time.sleep(0.0002)  # busy-poll the first 2 ms (barriers stay fast), then yield
                if now > deadline:
                    if self._comm is not None:
                        self._comm.abort()  # peers blocked on this rank fail too instead of hanging
                    raise N.B200TimeoutError(N.ERR_TIMEOUT, f"b200 collective did not complete within {secs:.1f} s")
        torch.cuda.current_stream(self._device).wait_event(self._event)
        if self._event.query():
            err = self._error()
            if err is not None:
                raise err
        return True

    def synchronize(self) -> None:
        self.wait()

    def is_completed(self) -> bool:
        return self._event is None or self._event.query()

    def is_success(self) -> bool:
        return self.is_completed() and self._error() is None

    def exception(self):
        return self._error() if self.is_completed() else None

    def get_future(self):
        return self._future

    def result(self):
        return self._result if isinstance(self._result, list) else [self._result]


class _CoalescedP2PWork(dist._Work):
    """What ``send`` / ``recv`` return inside a coalescing block: it completes with the block's one
    batch launch, so it can only be waited for once the block has ended."""

    def __init__(self, result):
        super().__init__()
        self._result = result
        self._batch: Optional[B200Work] = None

    def _work(self) -> B200Work:
        if self._batch is None:
            raise RuntimeError("this send / recv runs when its coalescing block ends; wait for it after the block")
        return self._batch

    def wait(self, timeout=None) -> bool:
        return self._work().wait(timeout)

    def synchronize(self) -> None:
        self.wait()

    def is_completed(self) -> bool:
        return self._batch is not None and self._batch.is_completed()

    def is_success(self) -> bool:
        return self._work().is_success()

    def exception(self):
        return self._batch.exception() if self._batch is not None else None

    def get_future(self):
        return self._work().get_future()

    def result(self):
        return self._result


class B200ProcessGroup(dist.ProcessGroup):
    """One rank's c10d process group.  CUDA tensors go to the B200 kernels; CPU tensors (rare:
    object collectives, barriers issued before any GPU work) go to an internal gloo group."""

    def __init__(self, store, rank: int, size: int, timeout: Optional[datetime.timedelta] = None,
                 comm_kwargs: Optional[dict] = None):
        super().__init__(rank, size)
        global _group_counter
        with _counter_lock:
            _group_counter += 1
            self._serial = _group_counter
        self._store = store
        self._rank, self._size = rank, size
        self._timeout = timeout or datetime.timedelta(seconds=1800)
        self._comm_kwargs = dict(comm_kwargs or {})
        self._comm: Optional[B200Comm] = None
        self._device: Optional[torch.device] = None
        self._stream: Optional[torch.cuda.Stream] = None
        self._gloo = None
        self._lock = threading.Lock()
        #: when True every op appends (start_event, end_event, first_tensor_bytes, tag) to ``timings``;
        #: tag is "grad" for the fused gradient-bucket launches, "op" for everything else
        self.record_timings = False
        self.timings = []

    # ------------------------------------------------------------------ plumbing
    def getBackendName(self) -> str:  # noqa: N802 - c10d virtual
        return BACKEND_NAME

    @property
    def comm(self) -> Optional[B200Comm]:
        return self._comm

    def _engine(self, device: torch.device) -> B200Comm:
        """The communicator is created on the first CUDA op (like ProcessGroupNCCL), because
        Ray Train binds the worker's device after the process group exists."""
        with self._lock:
            if self._comm is None:
                idx = device.index if device.index is not None else torch.cuda.current_device()
                self._device = torch.device("cuda", idx)
                # `self._store` is already scoped to this process group by torch (a PrefixStore per
                # group), so the keys must NOT depend on per-process counters: ranks that are not
                # members of every subgroup would otherwise disagree on the names.
                st = TorchDistStore(dist.PrefixStore("b200comm/", self._store))
                kwargs = dict(self._comm_kwargs)
                # the process group's collective timeout IS the device watchdog (NCCL blocks for
                # the same period and then raises): a rank that is late by a checkpoint or an
                # evaluation pass must not trip it
                kwargs.setdefault("timeout_ms", int(min(self._timeout.total_seconds() * 1000, 2**31 - 1)))
                self._comm = B200Comm(self._size, self._rank, idx, store=st, group_name="pg", **kwargs)
                # highest priority: when the bucket all-reduce overlaps the backward pass its CTAs
                # are placed ahead of the queued compute CTAs as SMs free up
                prio = torch.cuda.Stream.priority_range()[1] if hasattr(torch.cuda.Stream, "priority_range") else -1
                self._stream = torch.cuda.Stream(device=self._device, priority=prio)
            elif device.index is not None and device.index != self._device.index:
                raise RuntimeError(f"b200 process group is bound to {self._device}, got a tensor on {device}")
            return self._comm

    def _cpu_group(self):
        with self._lock:
            if self._gloo is None:
                self._gloo = dist.ProcessGroupGloo(dist.PrefixStore("b200gloo/", self._store),
                                                   self._rank, self._size, self._timeout)
            return self._gloo

    @staticmethod
    def _with_factor(tensors, op):
        """``tensors`` plus a ``PremulSum`` op's CUDA factor, which the kernels read on the
        communication stream and ``_run`` therefore records there; ``tensors`` itself otherwise."""
        if isinstance(op, PremulSum) and op.device_factor is not None:
            return list(tensors) + [op.device_factor]
        return tensors

    def _run(self, tensors: List[torch.Tensor], fn, result, tag: str = "op") -> B200Work:
        """Enqueue ``fn(comm)`` on the communication stream, ordered after the caller's stream."""
        dev = tensors[0].device
        comm = self._engine(dev)
        cur = torch.cuda.current_stream(self._device)
        self._stream.wait_stream(cur)
        with torch.cuda.device(self._device), torch.cuda.stream(self._stream):
            if self.record_timings:
                start = torch.cuda.Event(enable_timing=True)
                done = torch.cuda.Event(enable_timing=True)
                start.record(self._stream)
                fn(comm)
                done.record(self._stream)
                self.timings.append((start, done, tensors[0].numel() * tensors[0].element_size(), tag))
            else:
                fn(comm)
                done = torch.cuda.Event()
                done.record(self._stream)
        for t in tensors:
            t.record_stream(self._stream)
        return B200Work(result, self._device, done, self._stream, comm, self._timeout)

    @staticmethod
    def _all_cuda(tensors) -> bool:
        return all(t.is_cuda for t in tensors)

    @staticmethod
    def _contig(t: torch.Tensor) -> torch.Tensor:
        if not t.is_contiguous():
            raise RuntimeError("b200 backend requires contiguous tensors")
        return t

    # ------------------------------------------------------------------ collectives
    def allreduce(self, tensors, opts=None):
        if not self._all_cuda(tensors):
            return self._cpu_group().allreduce(tensors, opts) if opts is not None else self._cpu_group().allreduce(tensors)
        op = _op_code(opts.reduceOp) if opts is not None else N.SUM

        def fn(comm):
            for t in tensors:
                comm.allreduce(self._contig(t), op)

        return self._run(self._with_factor(tensors, op), fn, tensors)

    def allreduce_coalesced(self, tensors, opts=None):
        if not self._all_cuda(tensors):
            return self._cpu_group().allreduce_coalesced(tensors, opts)
        op = _op_code(opts.reduceOp) if opts is not None else N.SUM
        return self._run(self._with_factor(tensors, op),
                         lambda comm: comm.allreduce_multi([self._contig(t) for t in tensors], op), tensors)

    def broadcast(self, tensors, opts=None):
        if not self._all_cuda(tensors):
            return self._cpu_group().broadcast(tensors, opts)
        root = opts.rootRank if opts is not None else 0

        def fn(comm):
            for t in tensors:
                comm.broadcast(self._contig(t), root)

        return self._run(tensors, fn, tensors)

    def broadcast_multi(self, tensors: List[torch.Tensor], root: int) -> B200Work:
        """In-place broadcast of a list of contiguous CUDA tensors (any dtypes) from ``root`` in one
        ``b200_broadcast_multi`` call: DDP's per-forward buffer sync without the flatten, the
        per-dtype broadcasts and the per-tensor copy-out of c10d's ``_broadcast_coalesced``."""
        return self._run(tensors, lambda comm: comm.broadcast_multi([self._contig(t) for t in tensors], root),
                         tensors)

    @staticmethod
    def _cpu_each(calls):
        """gloo ops one after another (gloo has no coalesced form of them): the host waits for all
        but the last, whose work is returned."""
        work = None
        for call in calls:
            if work is not None:
                work.wait()
            work = call()
        return work

    @staticmethod
    def _by_dtype(outputs, inputs):
        """[(outputs, inputs)] per dtype of the outputs, in order of first appearance: a list
        reduce-scatter takes one dtype per call, and every rank passes the same list."""
        groups = {}
        for o, i in zip(outputs, inputs):
            outs, ins = groups.setdefault(o.dtype, ([], []))
            outs.append(o)
            ins.append(i)
        return list(groups.values())

    @staticmethod
    def _refuse_uneven_lists(what: str, pairs) -> None:
        """The list forms have no uneven variant: every (tensor, per-rank tensors) pair must agree in
        size.  One tensor of uneven parts goes through all_gather / reduce_scatter instead."""
        for i, (t, per_rank) in enumerate(pairs):
            if any(x.numel() != t.numel() for x in per_rank):
                raise RuntimeError(f"b200 process group: {what} of a tensor list needs equal sizes on every rank "
                                   f"(tensor {i} differs); uneven sizes are supported for a single tensor only")

    def _allgather_lists(self, output_lists, inputs) -> B200Work:
        """output_lists[i][p] receives rank p's inputs[i], in one b200_allgather_multi call; an output
        list that is not contiguous receives through temporaries and a copy."""
        self._refuse_uneven_lists("all_gather", zip(inputs, output_lists))

        def fn(comm):
            lists = [list(outs) if all(o.is_contiguous() for o in outs) else [torch.empty_like(t) for _ in outs]
                     for outs, t in zip(output_lists, inputs)]
            comm.allgather_multi(lists, [self._contig(t) for t in inputs])
            for outs, got in zip(output_lists, lists):
                for o, s in zip(outs, got):
                    if o is not s:
                        o.copy_(s)

        flat = [o for outs in output_lists for o in outs] + list(inputs)
        return self._run(flat, fn, output_lists)

    def allgather(self, output_tensors, input_tensors, opts=None):
        if not self._all_cuda(input_tensors):
            return self._cpu_group().allgather(output_tensors, input_tensors, opts)
        if len(input_tensors) > 1:
            return self._allgather_lists(output_tensors, input_tensors)

        def fn(comm):
            for outs, t in zip(output_tensors, input_tensors):
                # parts of a different size per rank: one b200_allgatherv call where ProcessGroupNCCL
                # falls back to a coalesced broadcast per rank
                uneven = any(o.numel() != t.numel() for o in outs)
                if all(o.is_contiguous() for o in outs):
                    if uneven:
                        comm.allgatherv(list(outs), self._contig(t))
                    else:
                        comm.allgather(list(outs), self._contig(t))
                elif uneven:
                    tmp = [torch.empty(o.shape, dtype=o.dtype, device=o.device) for o in outs]
                    comm.allgatherv(tmp, self._contig(t))
                    for o, s in zip(outs, tmp):
                        o.copy_(s)
                else:
                    tmp = [torch.empty_like(t) for _ in outs]
                    comm.allgather(tmp, self._contig(t))
                    for o, s in zip(outs, tmp):
                        o.copy_(s)

        flat = [o for outs in output_tensors for o in outs] + list(input_tensors)
        return self._run(flat, fn, output_tensors)

    def _allgather_base(self, output, input, opts=None):  # noqa: A002 - c10d signature
        if not input.is_cuda:
            return self._cpu_group()._allgather_base(output, input, opts)
        return self._run([output, input],
                         lambda comm: comm.allgather_into(self._contig(output), self._contig(input)), output)

    def allgather_coalesced(self, output_lists, input_list, opts=None):
        """``dist.all_gather_coalesced``: ``output_lists[p][i]`` receives rank p's ``input_list[i]``,
        in one ``b200_allgather_multi`` call."""
        if not self._all_cuda(input_list):
            return self._cpu_group().allgather_coalesced(output_lists, input_list, opts)
        if len(output_lists) != self._size or any(len(outs) != len(input_list) for outs in output_lists):
            raise RuntimeError("allgather_coalesced expects world_size output lists, each as long as the input list")
        return self._allgather_lists([[outs[i] for outs in output_lists] for i in range(len(input_list))],
                                     input_list)

    def allgather_into_tensor_coalesced(self, outputs, inputs, opts=None):
        """The fast path of ``_coalescing_manager`` around ``all_gather_into_tensor`` calls: one
        ``b200_allgather_multi`` call for the whole block."""
        if not self._all_cuda(inputs):
            gloo = self._cpu_group()
            return self._cpu_each([lambda o=o, i=i: gloo._allgather_base(o, i) for o, i in zip(outputs, inputs)])
        return self._run(list(outputs) + list(inputs),
                         lambda comm: comm.allgather_into_multi([self._contig(o) for o in outputs],
                                                                [self._contig(i) for i in inputs]), outputs)

    def reduce_scatter(self, output_tensors, input_tensors, opts=None):
        if not self._all_cuda(output_tensors):
            return self._cpu_group().reduce_scatter(output_tensors, input_tensors, opts)
        op = _op_code(opts.reduceOp) if opts is not None else N.SUM
        if len(output_tensors) > 1:
            self._refuse_uneven_lists("reduce_scatter", zip(output_tensors, input_tensors))

            def fn_multi(comm):
                for outs, ins in self._by_dtype(output_tensors, input_tensors):
                    comm.reducescatter_multi([self._contig(o) for o in outs],
                                             [[self._contig(i) for i in lst] for lst in ins], op)

            flat = list(output_tensors) + [i for ins in input_tensors for i in ins]
            return self._run(self._with_factor(flat, op), fn_multi, output_tensors)

        def fn(comm):
            for out, ins in zip(output_tensors, input_tensors):
                # parts of a different size per rank: one b200_reducescatterv call where
                # ProcessGroupNCCL falls back to a coalesced reduce per rank
                if any(i.numel() != out.numel() for i in ins):
                    comm.reducescatterv(self._contig(out), [self._contig(i) for i in ins], op)
                else:
                    comm.reducescatter(self._contig(out), [self._contig(i) for i in ins], op)

        flat = list(output_tensors) + [i for ins in input_tensors for i in ins]
        return self._run(self._with_factor(flat, op), fn, output_tensors)

    def _reduce_scatter_base(self, output, input, opts=None):  # noqa: A002
        op = _op_code(opts.reduceOp) if opts is not None else N.SUM
        return self._run(self._with_factor([output, input], op),
                         lambda comm: comm.reducescatter_from(self._contig(output), self._contig(input), op), output)

    def reduce_scatter_tensor_coalesced(self, outputs, inputs, opts=None):
        """The fast path of ``_coalescing_manager`` around ``reduce_scatter_tensor`` calls: one
        ``b200_reducescatter_multi`` call per dtype, in order of first appearance."""
        if not self._all_cuda(outputs):
            gloo = self._cpu_group()
            rs_opts = opts if opts is not None else dist.ReduceScatterOptions()
            return self._cpu_each([lambda o=o, i=i: gloo._reduce_scatter_base(o, i, rs_opts) for o, i in
                                   zip(outputs, inputs)])
        op = _op_code(opts.reduceOp) if opts is not None else N.SUM

        def fn(comm):
            for outs, ins in self._by_dtype(outputs, inputs):
                comm.reducescatter_from_multi([self._contig(o) for o in outs], [self._contig(i) for i in ins], op)

        return self._run(self._with_factor(list(outputs) + list(inputs), op), fn, outputs)

    def reduce(self, tensors, opts=None):
        if not self._all_cuda(tensors):
            return self._cpu_group().reduce(tensors, opts)
        op = _op_code(opts.reduceOp) if opts is not None else N.SUM
        root = opts.rootRank if opts is not None else 0

        def fn(comm):
            for t in tensors:
                comm.reduce(self._contig(t), root, op)

        return self._run(self._with_factor(tensors, op), fn, tensors)

    def barrier(self, opts=None):
        if self._comm is None or not torch.cuda.is_available():
            # nothing has touched the GPU yet: a host barrier is all that is needed
            return self._cpu_group().barrier(opts) if opts is not None else self._cpu_group().barrier()
        dummy = torch.empty(0, device=self._device)
        work = self._run([dummy], lambda comm: comm.barrier(), None)
        work.wait(self._timeout)  # dist.barrier() is host-blocking for NCCL as well; raises on a dead peer
        self._comm.check_status()
        return work

    def send(self, tensors, dst_rank, tag=0):
        if not self._all_cuda(tensors):
            return self._cpu_group().send(tensors, dst_rank, tag)
        if self._p2p_block is not None:
            return self._defer_p2p(True, tensors, dst_rank)

        def fn(comm):
            for t in tensors:
                comm.send(self._contig(t), dst_rank)

        return self._run(tensors, fn, tensors)

    def recv(self, tensors, src_rank, tag=0):
        if not self._all_cuda(tensors):
            return self._cpu_group().recv(tensors, src_rank, tag)
        if self._p2p_block is not None:
            return self._defer_p2p(False, tensors, src_rank)

        def fn(comm):
            for t in tensors:
                comm.recv(self._contig(t), src_rank)

        return self._run(tensors, fn, tensors)

    # ------------------------------------------------------------------ grouped point-to-point
    #: (is_send, tensor, peer) of the CUDA sends / receives recorded since _start_coalescing, and
    #: their Work handles; None outside a coalescing block
    _p2p_block = None

    def _defer_p2p(self, is_send: bool, tensors, peer: int) -> "_CoalescedP2PWork":
        ops, works = self._p2p_block
        ops.extend((is_send, self._contig(t), peer) for t in tensors)
        work = _CoalescedP2PWork(tensors)
        works.append(work)
        return work

    def _start_coalescing(self, device):  # noqa: D401 - c10d virtual, called by dist._coalescing_manager
        """Open a coalescing block: CUDA sends and receives are recorded until ``_end_coalescing``
        issues them as one ``b200_p2p_batch`` launch (``ncclGroupStart``).  CPU tensors still go to
        gloo at once, and other ops run as usual: torch issues its coalesced collectives itself."""
        if self._p2p_block is not None:
            raise RuntimeError("b200 process group: a coalescing block is already open")
        self._p2p_block = ([], [])

    def _end_coalescing(self, device):
        """Close the block (``ncclGroupEnd``): every recorded send and receive runs as one launch,
        whose Work is returned; the Work each ``send`` / ``recv`` returned completes with it."""
        block, self._p2p_block = self._p2p_block, None
        if block is None:
            raise RuntimeError("b200 process group: no coalescing block is open")
        ops, works = block
        if not ops:
            return None
        tensors = [t for _, t, _ in ops]
        work = self._run(tensors, lambda comm: comm.p2p_batch(ops), tensors)
        for w in works:
            w._batch = work
        return work

    # ------------------------------------------------------------------ rooted / all-to-all ops
    # gather, scatter and both all-to-all forms are one b200_alltoall launch each
    def gather(self, output_tensors, input_tensors, opts=None):
        """Root receives every rank's tensor (c10d ``gather``): an all-to-all in which every rank
        sends only to the root."""
        if not self._all_cuda(input_tensors):
            return self._cpu_group().gather(output_tensors, input_tensors, opts)
        root = opts.rootRank if opts is not None else 0

        def fn(comm):
            for i, t in enumerate(input_tensors):
                ins = [None] * self._size
                ins[root] = self._contig(t)
                outs = [self._contig(o) for o in output_tensors[i]] if self._rank == root else [None] * self._size
                comm.alltoall(outs, ins)

        flat = list(input_tensors) + [o for outs in output_tensors for o in outs]
        return self._run(flat, fn, output_tensors)

    def scatter(self, output_tensors, input_tensors, opts=None):
        """Mirror image of ``gather``: the root sends ``input_tensors[i][p]`` to rank p."""
        if not self._all_cuda(output_tensors):
            return self._cpu_group().scatter(output_tensors, input_tensors, opts)
        root = opts.rootRank if opts is not None else 0

        def fn(comm):
            for i, out in enumerate(output_tensors):
                outs = [None] * self._size
                outs[root] = self._contig(out)
                ins = [self._contig(t) for t in input_tensors[i]] if self._rank == root else [None] * self._size
                comm.alltoall(outs, ins)

        flat = list(output_tensors) + [t for ins in input_tensors for t in ins]
        return self._run(flat, fn, output_tensors)

    def alltoall_base(self, output, input, output_split_sizes, input_split_sizes, opts=None):  # noqa: A002
        if not input.is_cuda:
            return self._cpu_group().alltoall_base(output, input, output_split_sizes, input_split_sizes, opts)

        def splits(t, sizes, what):
            if not sizes:
                if t.size(0) % self._size:
                    raise RuntimeError("alltoall_base: dim 0 must be divisible by the world size")
                sizes = [t.size(0) // self._size] * self._size
            sizes = list(sizes)
            if len(sizes) != self._size:
                raise RuntimeError(f"alltoall_base: {len(sizes)} {what} split sizes for world size {self._size}")
            if sum(sizes) != t.size(0):
                raise RuntimeError(f"alltoall_base: {what} split sizes sum to {sum(sizes)}, dim 0 is {t.size(0)}")
            return list(torch.split(t, sizes, dim=0))

        sends = [self._contig(x) for x in splits(input, input_split_sizes, "input")]
        recvs = [self._contig(x) for x in splits(output, output_split_sizes, "output")]
        return self._run([output, input], lambda comm: comm.alltoall(recvs, sends), output)

    def alltoall(self, output_tensors, input_tensors, opts=None):
        if not self._all_cuda(input_tensors):
            return self._cpu_group().alltoall(output_tensors, input_tensors, opts)
        sends = [self._contig(t) for t in input_tensors]
        recvs = [self._contig(t) for t in output_tensors]
        return self._run(list(output_tensors) + list(input_tensors), lambda comm: comm.alltoall(recvs, sends),
                         output_tensors)

    # ------------------------------------------------------------------ fused gradient path
    def grad_allreduce(self, bucket: torch.Tensor, scale: float, wire_dtype: torch.dtype) -> torch.futures.Future:
        """Fused scale + wire cast + all-reduce + cast back on a flat fp32 bucket; returns the
        CUDA-aware future a DDP communication hook must return."""
        work = self._run([bucket], lambda comm: comm.grad_allreduce(bucket, scale, wire_dtype), bucket, tag="grad")
        return work.get_future()

    def grad_reducescatter(self, out: torch.Tensor, grad: torch.Tensor, scale: float,
                           wire_dtype: torch.dtype) -> B200Work:
        """Fused scale + wire cast + reduce-scatter + cast back: ``out`` receives this rank's shard
        of the scaled sum of the flat fp32 ``grad`` (world_size * out.numel() elements)."""
        return self._run([out, grad], lambda comm: comm.grad_reducescatter(out, grad, scale, wire_dtype), out,
                         tag="grad")

    # ------------------------------------------------------------------ lifecycle
    def abort(self):
        if self._comm is not None:
            self._comm.abort()

    def shutdown(self):
        if self._comm is not None:
            self._comm.destroy()
            self._comm = None

    def __del__(self):
        try:
            self.shutdown()
        except Exception:
            pass


def batch_isend_irecv(p2p_op_list):
    """Drop-in for ``dist.batch_isend_irecv`` that pipeline-parallel and ring-exchange code must call
    on the b200 backend.  torch coalesces the list only for a plain ``ProcessGroup``; on a b200 group
    it would issue one send or receive after another, and an exchange whose messages exceed the
    receiver's inbox would then wait forever.  Here a list of CUDA tensors on a b200 group runs inside
    ``dist._coalescing_manager`` -- torch's own NCCL branch -- as one ``b200_p2p_batch`` launch, and
    the one Work of that launch is returned.  Any other list goes to ``dist.batch_isend_irecv``."""
    if p2p_op_list:
        dist.distributed_c10d._check_p2p_op_list(p2p_op_list)
        group = p2p_op_list[0].group or dist.distributed_c10d._get_default_group()
        if isinstance(group, B200ProcessGroup) and all(op.tensor.is_cuda for op in p2p_op_list):
            with dist._coalescing_manager(group, p2p_op_list[0].tensor.device, async_ops=True) as cm:
                for op in p2p_op_list:
                    peer = {"group_dst" if op.op is dist.isend else "group_src": op.group_peer}
                    op.op(op.tensor, group=op.group, tag=op.tag, **peer)
            return cm.works
    return dist.batch_isend_irecv(p2p_op_list)


_registered = False


def _create_backend(store, rank, size, timeout):
    # `timeout` is init_process_group(timeout=...): TorchConfig.timeout_s in Ray Train (config.py:140-150)
    return B200ProcessGroup(store, rank, size, timeout)


def register_b200_backend() -> None:
    """Make ``dist.init_process_group(backend="b200")`` available in this process.  Must run
    on every worker before the process group is created (Ray Train: from the backend's
    ``on_start``, see ``ray_b200.train.torch_config``)."""
    global _registered
    if _registered:
        return
    dist.Backend.register_backend(BACKEND_NAME, _create_backend, devices=["cuda", "cpu"])
    _registered = True
