"""Host-side logic of grouped point-to-point that needs no GPU: B200Comm.p2p_batch's argument checks
and the arrays it hands to b200_p2p_batch, the recording of CUDA sends and receives inside a c10d
coalescing block of B200ProcessGroup, and ray_b200.train.batch_isend_irecv's choice of path."""
import types

import pytest
import torch
import torch.distributed as dist

from ray_b200 import train as T
from ray_b200.comm import B200Comm
from ray_b200.train import process_group as PG
from ray_b200.train.process_group import B200ProcessGroup


class _CudaLooking(torch.Tensor):
    """A CPU tensor that reports is_cuda, to reach the checks behind the device check."""

    @property
    def is_cuda(self):
        return True


def _cl(*shape, dtype=torch.float32):
    return torch.ones(*shape, dtype=dtype).as_subclass(_CudaLooking)


# ---- B200Comm.p2p_batch ---------------------------------------------------------------------------

class _RecordingLib:
    def __init__(self):
        self.calls = []

    def b200_p2p_batch(self, h, bufs, sizes, peers, sends, n, stream):
        self.calls.append(([bufs[i] for i in range(n)], [sizes[i] for i in range(n)], [peers[i] for i in range(n)],
                           [sends[i] for i in range(n)], n, stream))
        return 0


def _comm():
    # no native communicator: the library is a recorder
    c = B200Comm.__new__(B200Comm)
    c.world_size, c._h, c._lib = 4, None, _RecordingLib()
    c._stream = lambda: 77
    return c


def test_comm_p2p_batch_empty_is_a_no_op():
    c = _comm()
    assert c.p2p_batch([]) is None
    assert c.p2p_batch(iter(())) is None
    assert c._lib.calls == []


def test_comm_p2p_batch_checks():
    c = _comm()
    with pytest.raises(RuntimeError, match="must be on GPU"):
        c.p2p_batch([(True, _cl(2), 1), (False, torch.ones(2), 2)])
    with pytest.raises(RuntimeError, match="tensor 1 must be contiguous"):
        c.p2p_batch([(True, _cl(2), 1), (False, torch.ones(2, 2).t().as_subclass(_CudaLooking), 2)])
    with pytest.raises(RuntimeError, match="must be a torch.Tensor"):
        c.p2p_batch([(True, [1, 2], 1)])
    assert c._lib.calls == []


def test_comm_p2p_batch_passes_bytes_peers_and_directions_in_order():
    c = _comm()
    a, b, z = _cl(3, dtype=torch.float16), _cl(5, dtype=torch.int64), _cl(0)
    c.p2p_batch([(True, a, 1), (0, b, 3), (1, z, 2), (False, a, 1)])
    (bufs, sizes, peers, sends, n, stream), = c._lib.calls
    assert n == 4 and stream == 77
    assert bufs[:2] == [a.data_ptr(), b.data_ptr()]
    assert sizes == [6, 40, 0, 6] and peers == [1, 3, 2, 1] and sends == [1, 0, 1, 0]


# ---- B200ProcessGroup coalescing block --------------------------------------------------------------

class _RecComm:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        return lambda *args: self.calls.append((name,) + args)


class _FakeGloo:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return lambda *args: self.calls.append((name,) + args) or "gloo-work"


class _BatchWork:
    def __init__(self):
        self.waited = 0

    def wait(self, timeout=None):
        self.waited += 1
        return True

    def is_completed(self):
        return True


@pytest.fixture()
def pg(monkeypatch):
    """A B200ProcessGroup of world 3 whose communicator and gloo group record calls; ops run inline and
    _run returns a fresh _BatchWork."""
    p = B200ProcessGroup.__new__(B200ProcessGroup)
    p._size, p._rank = 3, 0
    p._comm, p._gloo = _RecComm(), _FakeGloo()
    p.runs = []

    def run(self, tensors, fn, result, tag="op"):
        fn(self._comm)
        self.runs.append(list(tensors))
        return _BatchWork()

    monkeypatch.setattr(B200ProcessGroup, "_run", run)
    monkeypatch.setattr(B200ProcessGroup, "_cpu_group", lambda self: self._gloo)
    return p


def test_block_records_sends_and_receives_in_issue_order(pg):
    a, b, c, d = _cl(4), _cl(2, dtype=torch.int64), _cl(8), _cl(1, dtype=torch.bfloat16)
    pg._start_coalescing(torch.device("cuda", 0))
    w1 = pg.send([a], 1)
    w2 = pg.recv([b], 2)
    w3 = pg.send([c, d], 2)
    assert pg._comm.calls == [] and pg.runs == []
    work = pg._end_coalescing(torch.device("cuda", 0))
    (name, ops), = pg._comm.calls
    assert name == "p2p_batch"
    assert [(s, p) for s, _, p in ops] == [(True, 1), (False, 2), (True, 2), (True, 2)]
    assert all(got is want for (_, got, _), want in zip(ops, [a, b, c, d]))
    assert pg.runs == [[a, b, c, d]]
    assert isinstance(work, _BatchWork)
    # the Work each call returned completes with the batch
    for w in (w1, w2, w3):
        assert w.wait() and w.is_completed()
    assert work.waited == 3
    assert w3.result() == [c, d]


def test_wait_inside_the_block_raises(pg):
    pg._start_coalescing(torch.device("cuda", 0))
    w = pg.send([_cl(4)], 1)
    assert not w.is_completed() and w.exception() is None
    with pytest.raises(RuntimeError, match="runs when its coalescing block ends"):
        w.wait()
    with pytest.raises(RuntimeError, match="runs when its coalescing block ends"):
        w.get_future()
    pg._end_coalescing(torch.device("cuda", 0))
    assert w.wait()


def test_block_without_sends_launches_nothing(pg):
    pg._start_coalescing(torch.device("cuda", 0))
    assert pg._end_coalescing(torch.device("cuda", 0)) is None
    assert pg._comm.calls == [] and pg.runs == []


def test_blocks_do_not_nest_and_must_be_open_to_end(pg):
    pg._start_coalescing(torch.device("cuda", 0))
    with pytest.raises(RuntimeError, match="already open"):
        pg._start_coalescing(torch.device("cuda", 0))
    pg._end_coalescing(torch.device("cuda", 0))
    with pytest.raises(RuntimeError, match="no coalescing block is open"):
        pg._end_coalescing(torch.device("cuda", 0))


def test_cpu_tensors_go_to_gloo_inside_a_block(pg):
    pg._start_coalescing(torch.device("cuda", 0))
    assert pg.send([torch.ones(2)], 1) == "gloo-work"
    assert pg.recv([torch.ones(3)], 2) == "gloo-work"
    assert [c[0] for c in pg._gloo.calls] == ["send", "recv"]
    assert pg._end_coalescing(torch.device("cuda", 0)) is None
    assert pg._comm.calls == []


def test_send_and_recv_outside_a_block_run_at_once(pg):
    a, b = _cl(4), _cl(2)
    assert isinstance(pg.send([a], 1), _BatchWork)
    assert isinstance(pg.recv([b], 2), _BatchWork)
    assert pg._comm.calls == [("send", a, 1), ("recv", b, 2)]


def test_non_contiguous_tensor_is_refused_when_recorded(pg):
    pg._start_coalescing(torch.device("cuda", 0))
    with pytest.raises(RuntimeError, match="contiguous"):
        pg.send([torch.ones(2, 2).t().as_subclass(_CudaLooking)], 1)
    pg._end_coalescing(torch.device("cuda", 0))


# ---- ray_b200.train.batch_isend_irecv ------------------------------------------------------------------

def _op(fn, tensor, peer, group):
    return types.SimpleNamespace(op=fn, tensor=tensor, group_peer=peer, group=group, tag=0)


def test_batch_isend_irecv_delegates_for_other_groups(monkeypatch):
    seen = []
    monkeypatch.setattr(dist.distributed_c10d, "_check_p2p_op_list", lambda ops: None)
    monkeypatch.setattr(dist, "batch_isend_irecv", lambda ops: seen.append(ops) or ["torch-works"])
    other = object()
    ops = [_op(dist.isend, _cl(2), 1, other), _op(dist.irecv, _cl(2), 1, other)]
    assert T.batch_isend_irecv(ops) == ["torch-works"] and seen == [ops]
    assert T.batch_isend_irecv([]) == ["torch-works"] and seen[-1] == []


def test_batch_isend_irecv_delegates_cpu_tensors_on_a_b200_group(monkeypatch, pg):
    seen = []
    monkeypatch.setattr(dist.distributed_c10d, "_check_p2p_op_list", lambda ops: None)
    monkeypatch.setattr(dist, "batch_isend_irecv", lambda ops: seen.append(ops) or ["torch-works"])
    ops = [_op(dist.isend, _cl(2), 1, pg), _op(dist.irecv, torch.ones(2), 1, pg)]
    assert T.batch_isend_irecv(ops) == ["torch-works"] and seen == [ops]
    assert pg._comm.calls == []


def test_batch_isend_irecv_runs_one_batch_on_a_b200_group(monkeypatch, pg):
    monkeypatch.setattr(dist.distributed_c10d, "_check_p2p_op_list", lambda ops: None)

    def fail(ops):
        raise AssertionError("must not delegate")

    monkeypatch.setattr(dist, "batch_isend_irecv", fail)
    calls = []
    monkeypatch.setattr(PG.dist, "isend", lambda t, group, tag, group_dst: calls.append(("isend", group_dst))
                        or group.send([t], group_dst, tag))
    monkeypatch.setattr(PG.dist, "irecv", lambda t, group, tag, group_src: calls.append(("irecv", group_src))
                        or group.recv([t], group_src, tag))
    a, b, c = _cl(4), _cl(4), _cl(3)
    ops = [_op(PG.dist.isend, a, 1, pg), _op(PG.dist.irecv, b, 2, pg), _op(PG.dist.isend, c, 2, pg)]
    works = T.batch_isend_irecv(ops)
    assert calls == [("isend", 1), ("irecv", 2), ("isend", 2)]
    (name, batch), = pg._comm.calls
    assert name == "p2p_batch" and [(s, p) for s, _, p in batch] == [(True, 1), (False, 2), (True, 2)]
    assert len(works) == 1 and isinstance(works[0], _BatchWork)
    assert pg._p2p_block is None
