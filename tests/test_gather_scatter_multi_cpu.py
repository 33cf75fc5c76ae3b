"""Host-side logic of the tensor-list all-gather and reduce-scatter that needs no GPU: the argument
checks of the four B200Comm methods, B200Group.allgather_multi / reducescatter_multi and
ray_b200.collective.allgather_multi / reducescatter_multi, and how B200ProcessGroup routes c10d's
coalesced and list collectives."""
import numpy as np
import pytest
import torch

from ray_b200 import _native as N
from ray_b200 import collective as col
from ray_b200.collective.b200_group import B200Group
from ray_b200.comm import B200Comm
from ray_b200.train.process_group import B200ProcessGroup


class _CudaLooking(torch.Tensor):
    """A CPU tensor that reports is_cuda, to reach the checks behind the device check."""

    @property
    def is_cuda(self):
        return True


def _cl(*shape, dtype=torch.float32):
    return torch.ones(*shape, dtype=dtype).as_subclass(_CudaLooking)


# ---- B200Comm -------------------------------------------------------------------------------------

def _comm(world=2):
    # no native communicator: every call below must be decided in Python
    c = B200Comm.__new__(B200Comm)
    c.world_size = world
    return c


def test_comm_empty_lists_are_no_ops():
    c = _comm()
    assert c.allgather_multi([], []) is None
    assert c.allgather_into_multi([], []) is None
    assert c.reducescatter_multi([], []) is None
    assert c.reducescatter_from_multi([], []) is None


def test_comm_allgather_multi_checks():
    c = _comm()
    with pytest.raises(RuntimeError, match="2 output lists for 1 tensors"):
        c.allgather_multi([[_cl(2), _cl(2)], [_cl(2), _cl(2)]], [_cl(2)])
    with pytest.raises(RuntimeError, match="must be on GPU"):
        c.allgather_multi([[_cl(2), _cl(2)]], [torch.ones(2)])
    with pytest.raises(RuntimeError, match="equal to world_size"):
        c.allgather_multi([[_cl(2)]], [_cl(2)])
    with pytest.raises(RuntimeError, match="same dtype and size"):
        c.allgather_multi([[_cl(2), _cl(3)]], [_cl(2)])
    with pytest.raises(RuntimeError, match="same dtype and size"):
        c.allgather_multi([[_cl(2), _cl(2, dtype=torch.float16)]], [_cl(2)])
    with pytest.raises(RuntimeError, match="output tensor must be contiguous"):
        c.allgather_multi([[_cl(2, 2), torch.ones(2, 2).t().as_subclass(_CudaLooking)]], [_cl(2, 2)])


def test_comm_allgather_into_multi_checks():
    c = _comm(3)
    with pytest.raises(RuntimeError, match="1 outputs for 2 tensors"):
        c.allgather_into_multi([_cl(6)], [_cl(2), _cl(2)])
    with pytest.raises(RuntimeError, match="world_size copies"):
        c.allgather_into_multi([_cl(4)], [_cl(2)])
    with pytest.raises(RuntimeError, match="world_size copies"):
        c.allgather_into_multi([_cl(6, dtype=torch.int64)], [_cl(2)])
    with pytest.raises(RuntimeError, match="tensor 0 must be contiguous"):
        c.allgather_into_multi([_cl(12)], [torch.ones(2, 2).t().as_subclass(_CudaLooking)])


def test_comm_reducescatter_multi_checks():
    c = _comm()
    with pytest.raises(RuntimeError, match="1 outputs for 2 inputs"):
        c.reducescatter_multi([_cl(2)], [[_cl(2), _cl(2)], [_cl(2), _cl(2)]])
    with pytest.raises(RuntimeError, match="same dtype"):
        c.reducescatter_multi([_cl(2), _cl(2, dtype=torch.int64)], [[_cl(2)] * 2, [_cl(2, dtype=torch.int64)] * 2])
    with pytest.raises(RuntimeError, match="equal to world_size"):
        c.reducescatter_multi([_cl(2)], [[_cl(2)]])
    with pytest.raises(RuntimeError, match="same dtype and size"):
        c.reducescatter_multi([_cl(2)], [[_cl(2), _cl(5)]])
    with pytest.raises(RuntimeError, match="output tensor 0 must be contiguous"):
        c.reducescatter_multi([torch.ones(2, 2).t().as_subclass(_CudaLooking)], [[_cl(2, 2)] * 2])
    with pytest.raises(RuntimeError, match="must be on GPU"):
        c.reducescatter_multi([_cl(2)], [[_cl(2), torch.ones(2)]])


def test_comm_reducescatter_from_multi_checks():
    c = _comm(4)
    with pytest.raises(RuntimeError, match="2 outputs for 1 inputs"):
        c.reducescatter_from_multi([_cl(2), _cl(2)], [_cl(8)])
    with pytest.raises(RuntimeError, match="world_size slices"):
        c.reducescatter_from_multi([_cl(2)], [_cl(6)])
    with pytest.raises(RuntimeError, match="world_size slices"):
        c.reducescatter_from_multi([_cl(2)], [_cl(8, dtype=torch.float64)])
    with pytest.raises(RuntimeError, match="same dtype"):
        c.reducescatter_from_multi([_cl(2), _cl(1, dtype=torch.int32)], [_cl(8), _cl(4, dtype=torch.int32)])


# ---- B200Group ------------------------------------------------------------------------------------

class _RecordingComm:
    def __init__(self):
        self.calls = []

    def allgather_multi(self, out_lists, tensors):
        self.calls.append(("ag", out_lists, tensors))

    def reducescatter_multi(self, outs, in_lists, op):
        self.calls.append(("rs", outs, in_lists, op))


def _group(world=2):
    g = B200Group.__new__(B200Group)
    g._world_size, g._rank, g._group_name = world, 0, "g"
    g._comm = _RecordingComm()
    return g


def test_group_allgather_multi_checks_and_forwards():
    g = _group()
    with pytest.raises(RuntimeError, match="must be lists of tensors"):
        g.allgather_multi([[_cl(2), _cl(2)]], (_cl(2),))
    with pytest.raises(RuntimeError, match="one output tensor list per input tensor"):
        g.allgather_multi([], [_cl(2)])
    with pytest.raises(RuntimeError, match="equal to world_size"):
        g.allgather_multi([[_cl(2)]], [_cl(2)])
    with pytest.raises(RuntimeError, match="same shape"):
        g.allgather_multi([[_cl(2), _cl(1, 2)]], [_cl(2)])
    with pytest.raises(ValueError, match="Unsupported tensor type"):
        g.allgather_multi([[_cl(2), _cl(2)]], [np.ones(2)])
    assert g._comm.calls == []
    ts, outs = [_cl(2), _cl(3)], [[_cl(2), _cl(2)], [_cl(3), _cl(3)]]
    g.allgather_multi(outs, ts)
    (kind, got_outs, got_ts), = g._comm.calls
    assert kind == "ag" and all(a is b for a, b in zip(got_ts, ts))
    assert all(a is b for la, lb in zip(got_outs, outs) for a, b in zip(la, lb))


def test_group_reducescatter_multi_checks_and_forwards():
    g = _group()
    with pytest.raises(RuntimeError, match="must be lists of tensors"):
        g.reducescatter_multi(_cl(2), [[_cl(2), _cl(2)]])
    with pytest.raises(RuntimeError, match="one input tensor list per output tensor"):
        g.reducescatter_multi([_cl(2)], [])
    with pytest.raises(RuntimeError, match="equal to world_size"):
        g.reducescatter_multi([_cl(2)], [[_cl(2), _cl(2), _cl(2)]])
    with pytest.raises(RuntimeError, match="same dtype"):
        g.reducescatter_multi([_cl(2)], [[_cl(2), _cl(2, dtype=torch.int64)]])
    assert g._comm.calls == []
    g.reducescatter_multi([_cl(2)], [[_cl(2), _cl(2)]], col.ReduceOp.MAX)
    assert g._comm.calls[0][0] == "rs" and g._comm.calls[0][3] == N.MAX
    g.reducescatter_multi([_cl(2)], [[_cl(2), _cl(2)]])
    assert g._comm.calls[1][3] == N.SUM


# ---- ray_b200.collective ----------------------------------------------------------------------------

class _FakeGroup:
    world_size, rank = 2, 0

    def __init__(self):
        self.calls = []

    def allgather_multi(self, tensor_lists, tensors):
        self.calls.append(("ag", tensor_lists, tensors))

    def reducescatter_multi(self, tensors, tensor_lists, op):
        self.calls.append(("rs", tensors, tensor_lists, op))


def _with_group(group):
    mgr = col.GroupManager()
    mgr._groups["g"] = group
    return col.use_manager(mgr)


def test_functional_allgather_multi_validates():
    fake = _FakeGroup()
    t = torch.ones(2)
    with _with_group(fake):
        with pytest.raises(RuntimeError, match="must be a list of tensors"):
            col.allgather_multi([[t, t]], t, group_name="g")
        with pytest.raises(RuntimeError, match="empty list"):
            col.allgather_multi([], [], group_name="g")
        with pytest.raises(RuntimeError, match="list of tensor lists"):
            col.allgather_multi((t, t), [t], group_name="g")
        with pytest.raises(RuntimeError, match="2 tensor lists for 1 tensors"):
            col.allgather_multi([[t, t], [t, t]], [t], group_name="g")
        with pytest.raises(RuntimeError, match="equal to world_size"):
            col.allgather_multi([[t]], [t], group_name="g")
        with pytest.raises(RuntimeError, match="Unrecognized tensor type"):
            col.allgather_multi([[t, "x"]], [t], group_name="g")
        assert fake.calls == []
        lists, ts = [[t, np.zeros(2)]], [t]
        col.allgather_multi(lists, ts, group_name="g")
        assert fake.calls == [("ag", lists, ts)]
    with pytest.raises(RuntimeError, match="not initialized"):
        col.allgather_multi([[t, t]], [t], group_name="no-such-group")


def test_functional_reducescatter_multi_validates():
    fake = _FakeGroup()
    t = torch.ones(2)
    with _with_group(fake):
        with pytest.raises(RuntimeError, match="must be a list of tensors"):
            col.reducescatter_multi(t, [[t, t]], group_name="g")
        with pytest.raises(RuntimeError, match="1 tensor lists for 2 tensors"):
            col.reducescatter_multi([t, t], [[t, t]], group_name="g")
        with pytest.raises(RuntimeError, match="equal to world_size"):
            col.reducescatter_multi([t], [[t, t, t]], group_name="g")
        assert fake.calls == []
        col.reducescatter_multi([t], [[t, t]], group_name="g", op=col.ReduceOp.MIN)
        assert fake.calls == [("rs", [t], [[t, t]], col.ReduceOp.MIN)]


def test_functional_api_refuses_a_group_without_list_gather_or_scatter():
    class Plain:
        world_size, rank = 2, 0

    t = torch.ones(2)
    with _with_group(Plain()):
        with pytest.raises(RuntimeError, match="has no list all-gather"):
            col.allgather_multi([[t, t]], [t], group_name="g")
        with pytest.raises(RuntimeError, match="has no list reduce-scatter"):
            col.reducescatter_multi([t], [[t, t]], group_name="g")


# ---- B200ProcessGroup routing ------------------------------------------------------------------------

class _RecComm:
    """Records the B200Comm calls a process-group method makes."""

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

        def call(*args):
            self.calls.append((name,) + args)

            class Work:
                waited = 0

                def wait(self):
                    Work.waited += 1
                    return True

            return Work()

        return call


@pytest.fixture()
def pg(monkeypatch):
    """A B200ProcessGroup of world 2 whose communicator and gloo group record calls; ops run inline."""
    p = B200ProcessGroup.__new__(B200ProcessGroup)
    p._size, p._rank = 2, 0
    p._comm, p._gloo = _RecComm(), _FakeGloo()
    monkeypatch.setattr(B200ProcessGroup, "_run", lambda self, tensors, fn, result, tag="op": fn(self._comm))
    monkeypatch.setattr(B200ProcessGroup, "_cpu_group", lambda self: self._gloo)
    return p


def _names(calls):
    return [c[0] for c in calls]


def test_coalesced_allgather_is_one_list_call(pg):
    outs = [_cl(4), _cl(6, dtype=torch.int64), _cl(2, dtype=torch.float16)]
    ins = [_cl(2), _cl(3, dtype=torch.int64), _cl(1, dtype=torch.float16)]
    pg.allgather_into_tensor_coalesced(outs, ins)
    assert _names(pg._comm.calls) == ["allgather_into_multi"]
    _, got_outs, got_ins = pg._comm.calls[0]
    assert all(a is b for a, b in zip(got_outs, outs)) and all(a is b for a, b in zip(got_ins, ins))


def test_coalesced_reducescatter_is_one_call_per_dtype_in_first_appearance_order(pg):
    import torch.distributed as dist

    outs = [_cl(2, dtype=torch.int64), _cl(2), _cl(3, dtype=torch.int64), _cl(1, dtype=torch.bfloat16), _cl(5)]
    ins = [_cl(2 * o.numel(), dtype=o.dtype) for o in outs]
    opts = dist.ReduceScatterOptions()
    opts.reduceOp = dist.ReduceOp.MAX
    pg.reduce_scatter_tensor_coalesced(outs, ins, opts)
    assert _names(pg._comm.calls) == ["reducescatter_from_multi"] * 3
    order = [[o.dtype for o in call[1]] for call in pg._comm.calls]
    assert order == [[torch.int64, torch.int64], [torch.float32, torch.float32], [torch.bfloat16]]
    assert pg._comm.calls[0][1][0] is outs[0] and pg._comm.calls[0][1][1] is outs[2]
    assert pg._comm.calls[0][2][0] is ins[0] and pg._comm.calls[0][2][1] is ins[2]
    assert all(call[3] == N.MAX for call in pg._comm.calls)
    pg._comm.calls.clear()
    pg.reduce_scatter_tensor_coalesced([_cl(2)], [_cl(4)])
    assert pg._comm.calls[0][0] == "reducescatter_from_multi" and pg._comm.calls[0][3] == N.SUM


def test_allgather_coalesced_transposes_into_one_list_call(pg):
    ins = [_cl(2), _cl(3)]
    output_lists = [[_cl(2), _cl(3)], [_cl(2), _cl(3)]]  # output_lists[p][i]
    pg.allgather_coalesced(output_lists, ins)
    (name, lists, got_ins), = pg._comm.calls
    assert name == "allgather_multi" and all(a is b for a, b in zip(got_ins, ins))
    for i in range(2):
        assert all(lists[i][p] is output_lists[p][i] for p in range(2))
    with pytest.raises(RuntimeError, match="world_size output lists"):
        pg.allgather_coalesced([[_cl(2), _cl(3)]], ins)


def test_list_allgather_and_reduce_scatter_take_the_list_entry(pg):
    a, b = _cl(2), _cl(3, dtype=torch.int64)
    outs_a, outs_b = [_cl(2), _cl(2)], [_cl(3, dtype=torch.int64), _cl(3, dtype=torch.int64)]
    pg.allgather([outs_a, outs_b], [a, b])
    assert _names(pg._comm.calls) == ["allgather_multi"]
    pg._comm.calls.clear()
    pg.allgather([outs_a], [a])  # one input: the single-tensor path as before
    assert _names(pg._comm.calls) == ["allgather"]
    pg._comm.calls.clear()
    o1, o2, o3 = _cl(2), _cl(2, dtype=torch.int64), _cl(4)
    pg.reduce_scatter([o1, o2, o3], [[_cl(2)] * 2, [_cl(2, dtype=torch.int64)] * 2, [_cl(4)] * 2])
    assert _names(pg._comm.calls) == ["reducescatter_multi", "reducescatter_multi"]
    assert pg._comm.calls[0][1] == [o1, o3] and pg._comm.calls[1][1] == [o2]
    pg._comm.calls.clear()
    pg.reduce_scatter([o1], [[_cl(2)] * 2])
    assert _names(pg._comm.calls) == ["reducescatter"]


def test_non_contiguous_outputs_receive_through_temporaries(pg):
    received = []

    def allgather_multi(lists, ins):
        received.append(lists)
        for lst in lists:
            for t in lst:
                t.fill_(7)

    pg._comm.allgather_multi = allgather_multi
    a, b = torch.zeros(2).as_subclass(_CudaLooking), torch.zeros(3).as_subclass(_CudaLooking)
    strided = [torch.zeros(6)[::2], torch.zeros(6)[1::2]]
    plain = [torch.zeros(2), torch.zeros(2)]
    pg.allgather([plain, strided], [a, b])
    assert received[0][0][0] is plain[0] and received[0][1][0] is not strided[0]
    assert all(torch.all(t == 7) for t in plain + strided)


def test_cpu_tensors_go_to_gloo(pg):
    outs, ins = [torch.zeros(4), torch.zeros(2)], [torch.ones(2), torch.ones(1)]
    pg.allgather_into_tensor_coalesced(outs, ins)
    assert _names(pg._gloo.calls) == ["_allgather_base", "_allgather_base"]
    pg._gloo.calls.clear()
    pg.reduce_scatter_tensor_coalesced(ins, outs)
    assert _names(pg._gloo.calls) == ["_reduce_scatter_base", "_reduce_scatter_base"]
    pg._gloo.calls.clear()
    pg.allgather_coalesced([[torch.zeros(2)], [torch.zeros(2)]], [torch.ones(2)])
    assert _names(pg._gloo.calls) == ["allgather_coalesced"]
    pg._gloo.calls.clear()
    pg.allgather([[torch.zeros(2)] * 2, [torch.zeros(1)] * 2], [torch.ones(2), torch.ones(1)])
    pg.reduce_scatter([torch.zeros(2), torch.zeros(1)], [[torch.ones(2)] * 2, [torch.ones(1)] * 2])
    assert _names(pg._gloo.calls) == ["allgather", "reduce_scatter"]
    assert pg._comm.calls == []
