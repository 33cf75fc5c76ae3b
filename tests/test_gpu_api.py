"""API-level tests: ``ray_b200.collective`` driven the way the reference's tests drive
``ray.util.collective`` (python/ray/util/collective/tests/single_node_gpu_tests/*.py):
two or more workers, ``ones * k`` buffers, exact equality, group lifecycle and error
behaviour.  Workers are threads that each own a ``GroupManager`` (the stand-in for one actor
process each), a CUDA stream, and -- when the box has enough GPUs -- their own device.
"""
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu


class Workers:
    """n worker threads; ``run(fn)`` executes fn(rank) on every worker concurrently."""

    def __init__(self, n):
        from ray_b200 import collective as col
        from ray_b200.store import DictStore

        self.n = n
        self.col = col
        self.store = DictStore()
        ndev = torch.cuda.device_count()
        self.devices = [r % ndev for r in range(n)] if ndev < n else list(range(n))
        self.mgrs = [col.GroupManager(self.store) for _ in range(n)]
        self.streams = [torch.cuda.Stream(device=d) for d in self.devices]
        self.shared = len(set(self.devices)) < n

    def run(self, fn):
        results, errors = [None] * self.n, [None] * self.n

        def body(r):
            try:
                # operands are produced on the device's default stream by the test body
                self.streams[r].wait_stream(torch.cuda.default_stream(self.devices[r]))
                with torch.cuda.device(self.devices[r]), torch.cuda.stream(self.streams[r]), \
                        self.col.use_manager(self.mgrs[r]):
                    results[r] = fn(r)
                    self.streams[r].synchronize()
            except BaseException as e:  # noqa: BLE001
                errors[r] = e

        ts = [threading.Thread(target=body, args=(r,)) for r in range(self.n)]
        for t in ts:
            t.start()
        for t in ts:
            t.join(120)
        for e in errors:
            if e is not None:
                raise e
        return results

    def init(self, group_name="default", **kw):
        def f(r):
            self.col.init_collective_group(self.n, r, backend="b200", group_name=group_name)
            if self.shared:
                g = self.col.get_group_handle(group_name)
                sms = torch.cuda.get_device_properties(self.devices[0]).multi_processor_count
                g.comm.set_blocks(max(1, (sms - 8) // self.n))

        self.run(f)

    def destroy(self, group_name="default"):
        self.run(lambda r: self.col.destroy_collective_group(group_name))

    def dev(self, r):
        return torch.device("cuda", self.devices[r])


@pytest.fixture()
def workers(native_lib):
    made = []

    def make(n):
        w = Workers(n)
        made.append(w)
        return w

    yield make
    for w in made:
        for m in w.mgrs:
            for name in list(m._groups):
                try:
                    m._groups[name].comm.abort()
                except Exception:
                    pass
        for m in w.mgrs:
            for name in list(m._groups):
                m.destroy_collective_group(name)


@pytest.mark.parametrize("group_name", ["default", "test", "123?34!"])
@pytest.mark.parametrize("world", [2, 4])
def test_allreduce_different_name_and_ops(workers, group_name, world):
    """test_allreduce.py:11-29 (names) and :91-124 (ops)."""
    w = workers(world)
    col = w.col
    w.init(group_name)
    assert w.run(lambda r: col.get_rank(group_name)) == list(range(world))
    assert w.run(lambda r: col.get_collective_group_size(group_name)) == [world] * world
    for size in (2, 2 ** 5, 2 ** 10, 2 ** 15, 2 ** 20):
        bufs = [torch.ones(size, device=w.dev(r)) for r in range(world)]
        w.run(lambda r: col.allreduce(bufs[r], group_name))
        for b in bufs:
            assert torch.all(b == world)
    for op, want in ((col.ReduceOp.SUM, sum(range(2, world + 2))), (col.ReduceOp.MIN, 2),
                     (col.ReduceOp.MAX, world + 1), (col.ReduceOp.PRODUCT, None)):
        bufs = [torch.ones(10, device=w.dev(r)) * (r + 2) for r in range(world)]
        w.run(lambda r: col.allreduce(bufs[r], group_name, op))
        if want is None:
            want = 1
            for r in range(world):
                want *= r + 2
        for b in bufs:
            assert torch.all(b == want), op


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float16, torch.float32, torch.float64, torch.int64])
def test_allreduce_different_dtype(workers, dtype):
    """test_allreduce.py:79-88."""
    w = workers(2)
    w.init()
    bufs = [torch.ones(10, dtype=dtype, device=w.dev(r)) for r in range(2)]
    w.run(lambda r: w.col.allreduce(bufs[r]))
    for b in bufs:
        assert torch.all(b == 2) and b.dtype == dtype


def test_group_lifecycle_destroy_reinit_multiple_groups(workers):
    """test_allreduce.py:32-76 and test_basic_apis.py: destroy, use-after-destroy, re-init,
    double init, several groups at once."""
    w = workers(2)
    col = w.col
    w.init("default")
    bufs = [torch.ones(10, device=w.dev(r)) for r in range(2)]
    w.run(lambda r: col.allreduce(bufs[r]))
    assert torch.all(bufs[0] == 2)
    with pytest.raises(RuntimeError, match="second time"):
        w.run(lambda r: col.init_collective_group(2, r, backend="b200", group_name="default"))
    w.destroy("default")
    assert w.run(lambda r: col.is_group_initialized("default")) == [False, False]
    assert w.run(lambda r: col.get_rank("default")) == [-1, -1]
    with pytest.raises(RuntimeError, match="not initialized"):
        w.run(lambda r: col.allreduce(bufs[r]))
    w.init("default")  # same name again
    w.run(lambda r: col.allreduce(bufs[r]))
    assert torch.all(bufs[1] == 4)
    names = [str(i) for i in range(5)]
    for nme in names:
        w.init(nme)
    for i, nme in enumerate(names):
        w.run(lambda r: col.allreduce(bufs[r], nme))
        assert torch.all(bufs[0] == 4 * 2 ** (i + 1))
    for nme in names:
        w.destroy(nme)


def test_argument_validation_matches_reference(workers):
    """Q6/Q7/Q8 of SURVEY appendix A: list length, shapes, ranks, CPU tensors, bad types."""
    w = workers(2)
    col = w.col
    w.init()
    dev = w.dev(0)

    def on_rank0(fn):
        with torch.cuda.device(w.devices[0]), col.use_manager(w.mgrs[0]):
            fn()

    t = torch.ones(4, device=dev)
    with pytest.raises(RuntimeError, match="world_size"):
        on_rank0(lambda: col.allgather([t.clone()], t))
    with pytest.raises(RuntimeError, match="world_size"):
        on_rank0(lambda: col.reducescatter(t, [t.clone()] * 3))
    with pytest.raises(RuntimeError, match="same shape"):
        on_rank0(lambda: col.allgather([t.clone(), torch.ones(5, device=dev)], t))
    with pytest.raises(RuntimeError, match="same dtype"):
        on_rank0(lambda: col.allgather([t.clone(), torch.ones(4, device=dev, dtype=torch.float16)], t))
    with pytest.raises(ValueError):
        on_rank0(lambda: col.send(t, 5))
    with pytest.raises(ValueError):
        on_rank0(lambda: col.broadcast(t, -1))
    with pytest.raises(RuntimeError, match="is self"):
        on_rank0(lambda: col.send(t, 0))
    with pytest.raises(RuntimeError, match="is self"):
        on_rank0(lambda: col.recv(t, 0))
    with pytest.raises(RuntimeError, match="must be on GPU"):
        on_rank0(lambda: col.allreduce(torch.ones(4)))
    with pytest.raises(RuntimeError, match="Unrecognized tensor type"):
        on_rank0(lambda: col.allreduce([1, 2, 3]))
    with pytest.raises(RuntimeError, match="empty list"):
        on_rank0(lambda: col.allgather([], t))
    with pytest.raises(ValueError, match="Unrecognized backend"):
        col.Backend("mpi")


def test_reduce_broadcast_allgather_reducescatter_sendrecv_via_api(workers):
    """test_reduce.py:18-20, test_broadcast.py, test_allgather.py, test_reducescatter.py,
    test_sendrecv.py -- the ones*k patterns."""
    world = 4
    w = workers(world)
    col = w.col
    w.init()
    for root in range(world):
        bufs = [torch.ones(33, device=w.dev(r)) * (r + 1) for r in range(world)]
        w.run(lambda r: col.reduce(bufs[r], root))
        for r in range(world):
            assert torch.all(bufs[r] == (10 if r == root else r + 1))
        bufs = [torch.ones(33, device=w.dev(r)) * (r + 1) for r in range(world)]
        w.run(lambda r: col.broadcast(bufs[r], root))
        for r in range(world):
            assert torch.all(bufs[r] == root + 1)
    ins = [torch.ones(8, 3, device=w.dev(r)) * (r + 1) for r in range(world)]
    lists = [[torch.zeros(8, 3, device=w.dev(r)) for _ in range(world)] for r in range(world)]
    w.run(lambda r: col.allgather(lists[r], ins[r]))
    for r in range(world):
        for p in range(world):
            assert torch.all(lists[r][p] == p + 1)
    outs = [torch.zeros(8, 3, device=w.dev(r)) for r in range(world)]
    lists = [[torch.ones(8, 3, device=w.dev(r)) * (r + 1) * (i + 1) for i in range(world)] for r in range(world)]
    w.run(lambda r: col.reducescatter(outs[r], lists[r]))
    for r in range(world):
        assert torch.all(outs[r] == 10 * (r + 1))
    shape = [5, 9, 10, 85]
    a = torch.ones(*shape, device=w.dev(1)) * 7
    b = torch.zeros(*shape, device=w.dev(3))
    w.run(lambda r: col.send(a, 3) if r == 1 else (col.recv(b, 1) if r == 3 else None))
    assert torch.all(b == 7)
    w.run(lambda r: col.barrier())


def test_declarative_group_and_env_var_creation(workers, monkeypatch):
    """collective.py:188-261 (driver declares the group) and :760-770 (env-var fallback)."""
    w = workers(2)
    col = w.col
    col.create_collective_group(["actor-a", "actor-b"], 2, [1, 0], backend="b200", group_name="decl",
                                store=w.store)
    with pytest.raises(RuntimeError, match="twice"):
        col.create_collective_group(["actor-a", "actor-b"], 2, [1, 0], backend="b200", group_name="decl",
                                    store=w.store)
    with pytest.raises(RuntimeError, match="permutation"):
        col.create_collective_group(["a", "b"], 2, [0, 0], backend="b200", group_name="bad", store=w.store)
    bufs = [torch.ones(10, device=w.dev(r)) for r in range(2)]

    def f(r):
        col.set_member_id("actor-a" if r == 0 else "actor-b")
        if w.shared:
            col.get_group_handle("decl").comm.set_blocks(64)
        col.allreduce(bufs[r], "decl")  # lazily creates the group from the record
        return col.get_rank("decl")

    assert w.run(f) == [1, 0]
    assert torch.all(bufs[0] == 2)
    w.destroy("decl")


def test_rdt_tensor_transport_over_b200_group(workers):
    """Boundary B3: TensorTransportManager contract (python/ray/experimental/rdt/
    tensor_transport_manager.py:37-224) mapped onto send/recv of a B200 group, as the reference's
    CollectiveTensorTransport does for NCCL (collective_tensor_transport.py:124-176)."""
    from ray_b200.rdt import B200CommunicatorMetadata, B200TensorTransport

    w = workers(2)
    w.init("rdt-group")
    tr = B200TensorTransport()
    assert tr.tensor_transport_backend() == "B200" and not tr.is_one_sided() and tr.can_abort_transport()
    B200TensorTransport.group_resolver = staticmethod(
        lambda src, dst: ("rdt-group", int(src[-1]), int(dst[-1])))
    try:
        assert tr.actor_has_tensor_transport("actor0")
        meta_c = tr.get_communicator_metadata("actor0", "actor1", "B200")
        assert isinstance(meta_c, B200CommunicatorMetadata) and (meta_c.src_rank, meta_c.dst_rank) == (0, 1)
        payload = [torch.randn(17, 3), torch.arange(1000, dtype=torch.float32), torch.randn(5).to(torch.float16)]
        sent = [t.to(w.dev(0)) for t in payload]
        meta_t = tr.extract_tensor_transport_metadata("obj-1", sent)
        assert meta_t.tensor_device == "cuda" and len(meta_t.tensor_meta) == 3
        with pytest.raises(ValueError, match="same device type"):
            tr.extract_tensor_transport_metadata("obj-2", [sent[0], torch.ones(1)])

        def f(r):
            if r == 0:
                tr.send_multiple_tensors(sent, meta_t, meta_c)
                return None
            got = tr.recv_multiple_tensors("obj-1", meta_t, meta_c)
            torch.cuda.current_stream().synchronize()
            return [g.cpu() for g in got]

        got = w.run(f)[1]
        assert all(torch.equal(g, p) for g, p in zip(got, payload))
        tr.garbage_collect("obj-1", meta_t, sent)
    finally:
        B200TensorTransport.group_resolver = None


def test_rdt_one_sided_transport_pulls_without_the_sender(workers, monkeypatch):
    """SURVEY 8f row 4: RDT one-sided ``B200_IPC`` transport.  extract_tensor_transport_metadata
    publishes (heap offset, event); recv_multiple_tensors pulls with a receiver-side kernel into
    target_buffers; the sender's communicator launches nothing (cuda_ipc_transport.py:57-186 is the
    pattern, without its same-GPU restriction)."""
    import threading

    from ray_b200.rdt import B200IpcTransport, B200IpcTransportMetadata

    monkeypatch.setenv("B200_HEAP_BYTES", str(64 << 20))
    w = workers(2)
    w.init("ipc-group")
    tr = B200IpcTransport()
    assert tr.tensor_transport_backend() == "B200_IPC" and tr.is_one_sided() and tr.can_abort_transport()
    B200IpcTransport.group_resolver = staticmethod(lambda src, dst: ("ipc-group", int(src[-1]), int(dst[-1])))
    B200IpcTransport.publish_resolver = staticmethod(lambda: ("ipc-group", 0))
    box, ready, done = {}, threading.Event(), threading.Event()
    payload = [torch.randn(1 << 20), torch.arange(1003, dtype=torch.int32), torch.randn(7, 9).to(torch.float16)]
    try:
        meta_c = tr.get_communicator_metadata("actor0", "actor1", "B200_IPC")

        def f(r):
            comm = w.col.get_group_handle("ipc-group").comm
            if r == 0:
                sent = [t.to(w.dev(0)) for t in payload]
                in_heap = comm.symm_empty((4096,), torch.float32)  # already symmetric: published in place
                in_heap.copy_(torch.arange(4096, dtype=torch.float32))
                before = comm.launch_count
                box["meta"] = tr.extract_tensor_transport_metadata("obj-9", sent + [in_heap])
                ready.set()
                done.wait(60)
                launches = comm.launch_count - before
                tr.garbage_collect("obj-9", box["meta"], sent)
                return launches
            ready.wait(60)
            meta = box["meta"]
            assert isinstance(meta, B200IpcTransportMetadata) and meta.src_rank == 0 and len(meta.heap_offsets) == 4
            targets = [torch.zeros(tuple(s), dtype=d, device=w.dev(1)) for s, d in meta.tensor_meta]
            got = tr.recv_multiple_tensors("obj-9", meta, meta_c, target_buffers=targets)
            torch.cuda.current_stream().synchronize()
            assert all(g.data_ptr() == t.data_ptr() for g, t in zip(got, targets)), "must land in target_buffers"
            out = [g.cpu() for g in got]
            again = tr.recv_multiple_tensors("obj-9", meta, meta_c)  # a second consumer allocates its own
            torch.cuda.current_stream().synchronize()
            done.set()
            return out, [a.cpu() for a in again]

        res = w.run(f)
        assert res[0] == 0, "the sender must not launch a single kernel of the library"
        for got in res[1]:
            assert all(torch.equal(g, p) for g, p in zip(got[:3], payload))
            assert torch.equal(got[3], torch.arange(4096, dtype=torch.float32))
        with pytest.raises(NotImplementedError):
            tr.send_multiple_tensors([], None, None)
        assert tr._staged == {}
    finally:
        done.set()
        B200IpcTransport.group_resolver = None
        B200IpcTransport.publish_resolver = None
