"""Host-side logic of the uneven all-gather and reduce-scatter that needs no GPU: the argument checks
of B200Comm.allgatherv / reducescatterv, B200Group.allgatherv / reducescatterv and
ray_b200.collective.allgatherv / reducescatterv, how B200ProcessGroup routes c10d's all_gather and
reduce_scatter by size, and the launch formulas."""
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


def _strided():
    return torch.ones(2, 2).t().as_subclass(_CudaLooking)


# ---- B200Comm -------------------------------------------------------------------------------------

class _NoLib:
    """Any native call fails the test: every case below must be decided in Python."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} reached the native library")


def _comm(world=2, rank=0):
    c = B200Comm.__new__(B200Comm)
    c.world_size, c.rank = world, rank
    c._lib = _NoLib()
    return c


def test_comm_allgatherv_checks():
    c = _comm(3, rank=1)
    with pytest.raises(RuntimeError, match="must be on GPU"):
        c.allgatherv([_cl(2), _cl(3), _cl(4)], torch.ones(3))
    with pytest.raises(RuntimeError, match="tensor must be contiguous"):
        c.allgatherv([_cl(2), _cl(4), _cl(4)], _strided())
    with pytest.raises(RuntimeError, match="equal to world_size"):
        c.allgatherv([_cl(2), _cl(3)], _cl(3))
    with pytest.raises(RuntimeError, match="tensor 2 must be contiguous"):
        c.allgatherv([_cl(2), _cl(3), _strided()], _cl(3))
    with pytest.raises(RuntimeError, match="must be on GPU"):
        c.allgatherv([_cl(2), _cl(3), torch.ones(4)], _cl(3))
    with pytest.raises(RuntimeError, match="same dtype"):
        c.allgatherv([_cl(2), _cl(3), _cl(4, dtype=torch.int64)], _cl(3))
    with pytest.raises(RuntimeError, match=r"tensor 1 \(this rank's part\) has 4 elements, the input has 3"):
        c.allgatherv([_cl(2), _cl(4), _cl(4)], _cl(3))


def test_comm_reducescatterv_checks():
    c = _comm(2, rank=0)
    with pytest.raises(RuntimeError, match="output tensor must be contiguous"):
        c.reducescatterv(_strided(), [_cl(4), _cl(1)])
    with pytest.raises(RuntimeError, match="equal to world_size"):
        c.reducescatterv(_cl(2), [_cl(2)])
    with pytest.raises(RuntimeError, match="same dtype"):
        c.reducescatterv(_cl(2), [_cl(2), _cl(5, dtype=torch.float16)])
    with pytest.raises(RuntimeError, match="tensor 1 must be contiguous"):
        c.reducescatterv(_cl(2), [_cl(2), _strided()])
    with pytest.raises(RuntimeError, match=r"tensor 0 \(this rank's part\) has 3 elements, the output has 2"):
        c.reducescatterv(_cl(2), [_cl(3), _cl(2)])


class _RecordingLib:
    def __init__(self):
        self.calls = []

    def b200_allgatherv(self, h, in_ptr, counts, outs, dtype, stream):
        self.calls.append(("ag", in_ptr, list(counts[:3]), list(outs[:3]), dtype))
        return N.OK

    def b200_reducescatterv(self, h, ins, counts, out, dtype, op, stream):
        self.calls.append(("rs", list(ins[:3]), list(counts[:3]), out, dtype, op))
        return N.OK


def test_comm_passes_numels_as_counts(monkeypatch):
    c = _comm(3, rank=2)
    c._lib, c._h = _RecordingLib(), None
    monkeypatch.setattr(B200Comm, "_stream", lambda self: 0)
    outs = [_cl(5, dtype=torch.int32), _cl(0, dtype=torch.int32), _cl(2, 3, dtype=torch.int32)]
    t = _cl(6, dtype=torch.int32)
    c.allgatherv(outs, t)
    kind, in_ptr, counts, ptrs, dtype = c._lib.calls[0]
    assert kind == "ag" and counts == [5, 0, 6] and dtype == N.I32 and in_ptr == t.data_ptr()
    assert ptrs[0] == outs[0].data_ptr() and ptrs[2] == outs[2].data_ptr()
    out = _cl(6, dtype=torch.bfloat16)
    ins = [_cl(1, dtype=torch.bfloat16), _cl(7, dtype=torch.bfloat16), _cl(6, dtype=torch.bfloat16)]
    c.reducescatterv(out, ins, N.AVG)
    kind, ptrs, counts, out_ptr, dtype, op = c._lib.calls[1]
    assert kind == "rs" and counts == [1, 7, 6] and dtype == N.BF16 and op == N.AVG and out_ptr == out.data_ptr()


# ---- B200Group ------------------------------------------------------------------------------------

class _RecordingComm:
    def __init__(self):
        self.calls = []

    def allgatherv(self, outs, tensor):
        self.calls.append(("ag", outs, tensor))

    def reducescatterv(self, out, ins, op):
        self.calls.append(("rs", out, ins, op))


def _group(world=2):
    g = B200Group.__new__(B200Group)
    g._world_size, g._rank, g._group_name = world, 0, "g"
    g._comm = _RecordingComm()
    return g


def test_group_allgatherv_checks_and_forwards():
    g = _group()
    with pytest.raises(RuntimeError, match="output must be a list of tensors"):
        g.allgatherv((_cl(2), _cl(3)), _cl(2))
    with pytest.raises(RuntimeError, match="equal to world_size"):
        g.allgatherv([_cl(2)], _cl(2))
    with pytest.raises(ValueError, match="Unsupported tensor type"):
        g.allgatherv([_cl(2), np.ones(3)], _cl(2))
    with pytest.raises(RuntimeError, match="must be on GPU"):
        g.allgatherv([_cl(2), _cl(3)], torch.ones(2))
    assert g._comm.calls == []
    outs, t = [_cl(2), _cl(1, 3)], _cl(2)  # shapes may differ per rank
    g.allgatherv(outs, t)
    (kind, got_outs, got_t), = g._comm.calls
    assert kind == "ag" and got_t is t and all(a is b for a, b in zip(got_outs, outs))


def test_group_reducescatterv_checks_and_forwards():
    g = _group()
    with pytest.raises(RuntimeError, match="input must be a list of tensors"):
        g.reducescatterv(_cl(2), (_cl(2), _cl(3)))
    with pytest.raises(RuntimeError, match="equal to world_size"):
        g.reducescatterv(_cl(2), [_cl(2), _cl(3), _cl(4)])
    assert g._comm.calls == []
    g.reducescatterv(_cl(2), [_cl(2), _cl(5)], col.ReduceOp.MAX)
    assert g._comm.calls[0][0] == "rs" and g._comm.calls[0][3] == N.MAX
    g.reducescatterv(_cl(2), [_cl(2), _cl(5)])
    assert g._comm.calls[1][3] == N.SUM


# ---- ray_b200.collective ----------------------------------------------------------------------------

class _FakeGroup:
    world_size, rank = 2, 0

    def __init__(self):
        self.calls = []

    def allgatherv(self, tensor_list, tensor):
        self.calls.append(("ag", tensor_list, tensor))

    def reducescatterv(self, tensor, tensor_list, op):
        self.calls.append(("rs", tensor, tensor_list, op))


def _with_group(group):
    mgr = col.GroupManager()
    mgr._groups["g"] = group
    return col.use_manager(mgr)


def test_functional_allgatherv_validates():
    fake = _FakeGroup()
    t, u = torch.ones(2), torch.ones(5)
    with _with_group(fake):
        with pytest.raises(RuntimeError, match="must be a list of tensors"):
            col.allgatherv((t, u), t, group_name="g")
        with pytest.raises(RuntimeError, match="empty list"):
            col.allgatherv([], t, group_name="g")
        with pytest.raises(RuntimeError, match="Unrecognized tensor type"):
            col.allgatherv([t, u], "x", group_name="g")
        with pytest.raises(RuntimeError, match="equal to world_size"):
            col.allgatherv([t], t, group_name="g")
        assert fake.calls == []
        col.allgatherv([t, u], t, group_name="g")
        assert fake.calls == [("ag", [t, u], t)]
    with pytest.raises(RuntimeError, match="not initialized"):
        col.allgatherv([t, u], t, group_name="no-such-group")


def test_functional_reducescatterv_validates():
    fake = _FakeGroup()
    t, u = torch.ones(2), torch.ones(5)
    with _with_group(fake):
        with pytest.raises(RuntimeError, match="must be a list of tensors"):
            col.reducescatterv(t, (t, u), group_name="g")
        with pytest.raises(RuntimeError, match="equal to world_size"):
            col.reducescatterv(t, [t, u, u], group_name="g")
        with pytest.raises(RuntimeError, match="Unrecognized tensor type"):
            col.reducescatterv(None, [t, u], group_name="g")
        assert fake.calls == []
        col.reducescatterv(t, [t, u], group_name="g", op=col.ReduceOp.MIN)
        assert fake.calls == [("rs", t, [t, u], col.ReduceOp.MIN)]


def test_functional_api_refuses_a_group_without_uneven_gather_or_scatter():
    class Plain:
        world_size, rank = 2, 0

    t = torch.ones(2)
    with _with_group(Plain()):
        with pytest.raises(RuntimeError, match="has no uneven all-gather"):
            col.allgatherv([t, t], t, group_name="g")
        with pytest.raises(RuntimeError, match="has no uneven reduce-scatter"):
            col.reducescatterv(t, [t, t], group_name="g")


def test_ray_allgather_and_reducescatter_keep_the_equal_shape_rule():
    g = _group()
    with pytest.raises(RuntimeError, match="same shape"):
        g.allgather([[_cl(2), _cl(3)]], [_cl(2)])
    with pytest.raises(RuntimeError, match="same shape"):
        g.reducescatter([_cl(2)], [[_cl(2), _cl(3)]])
    assert g._comm.calls == []


# ---- B200ProcessGroup routing ------------------------------------------------------------------------

class _RecComm:
    """Records the B200Comm calls a process-group method makes."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        return lambda *args: self.calls.append((name,) + args)


@pytest.fixture()
def pg(monkeypatch):
    """A B200ProcessGroup of world 2 whose communicator records calls; ops run inline."""
    p = B200ProcessGroup.__new__(B200ProcessGroup)
    p._size, p._rank = 2, 0
    p._comm = _RecComm()
    monkeypatch.setattr(B200ProcessGroup, "_run", lambda self, tensors, fn, result, tag="op": fn(self._comm))
    return p


def _names(calls):
    return [c[0] for c in calls]


def test_uneven_all_gather_takes_the_v_form(pg):
    t = _cl(2)
    outs = [_cl(2), _cl(5)]
    pg.allgather([outs], [t])
    (name, got_outs, got_t), = pg._comm.calls
    assert name == "allgatherv" and got_t is t and all(a is b for a, b in zip(got_outs, outs))


def test_even_all_gather_keeps_todays_call(pg):
    pg.allgather([[_cl(3), _cl(3)]], [_cl(3)])
    pg.allgather([[_cl(1, 3), _cl(3, 1)]], [_cl(3)])  # same numel, other shapes
    assert _names(pg._comm.calls) == ["allgather", "allgather"]


def test_uneven_reduce_scatter_takes_the_v_form(pg):
    import torch.distributed as dist

    opts = dist.ReduceScatterOptions()
    opts.reduceOp = dist.ReduceOp.AVG
    out, ins = _cl(3), [_cl(3), _cl(8)]
    pg.reduce_scatter([out], [ins], opts)
    (name, got_out, got_ins, op), = pg._comm.calls
    assert name == "reducescatterv" and got_out is out and op == N.AVG
    assert all(a is b for a, b in zip(got_ins, ins))
    pg._comm.calls.clear()
    pg.reduce_scatter([_cl(4)], [[_cl(4), _cl(4)]])
    assert _names(pg._comm.calls) == ["reducescatter"] and pg._comm.calls[0][3] == N.SUM


def test_uneven_all_gather_into_non_contiguous_outputs_goes_through_temporaries(pg):
    received = []

    def allgatherv(outs, t):
        received.append(outs)
        for p, o in enumerate(outs):
            o.fill_(p + 1)

    pg._comm.allgatherv = allgatherv
    t = torch.zeros(2).as_subclass(_CudaLooking)
    plain, strided = torch.zeros(2), torch.zeros(3, 3)[:, 0]
    pg.allgather([[plain, strided]], [t])
    got = received[0]
    assert got[1] is not strided and got[1].is_contiguous() and got[1].shape == strided.shape
    assert torch.all(plain == 1) and torch.all(strided == 2)


def test_uneven_lists_keep_refusing(pg):
    a, b = _cl(2), _cl(3)
    with pytest.raises(RuntimeError, match="all_gather of a tensor list needs equal sizes.*tensor 1 differs"):
        pg.allgather([[_cl(2), _cl(2)], [_cl(3), _cl(4)]], [a, b])
    with pytest.raises(RuntimeError, match="all_gather of a tensor list needs equal sizes.*tensor 0 differs"):
        pg.allgather_coalesced([[_cl(2)], [_cl(5)]], [a])
    with pytest.raises(RuntimeError, match="reduce_scatter of a tensor list needs equal sizes.*tensor 0 differs"):
        pg.reduce_scatter([a, b], [[_cl(2), _cl(1)], [_cl(3), _cl(3)]])
    assert pg._comm.calls == []
    # equal lists still take the list entries
    pg.allgather([[_cl(2), _cl(2)], [_cl(3), _cl(3)]], [a, b])
    pg.reduce_scatter([a, b], [[_cl(2), _cl(2)], [_cl(3), _cl(3)]])
    assert _names(pg._comm.calls) == ["allgather_multi", "reducescatter_multi"]


# ---- launch formulas -------------------------------------------------------------------------------

def ag_launches(nbytes, staging):
    """ceil(max_p U_p / W), W = staging_bytes / 16 and U_p = ceil(bytes_p / 16)."""
    return -(-max(-(-b // 16) for b in nbytes) // (staging // 16))


def rs_launches(nbytes, staging):
    """ceil(max_q U_q / W), W = floor(staging_bytes / (16 n))."""
    return -(-max(-(-b // 16) for b in nbytes) // (staging // (16 * len(nbytes))))


def test_launch_formulas():
    S = 2 << 20
    assert ag_launches([0, 0], S) == 0 and rs_launches([0, 0, 0], S) == 0
    assert ag_launches([1, 0], S) == 1 and ag_launches([S, 3], S) == 1 and ag_launches([5, S + 1], S) == 2
    assert ag_launches([S + 15, 0], S) == 2  # a 15-byte tail is one more unit
    assert ag_launches([3 * S - 16, 17, 0, 5], S) == 3
    assert rs_launches([S // 2, 1], S) == 1 and rs_launches([S // 2 + 1, 0], S) == 2
    assert rs_launches([S // 8] + [0] * 7, S) == 1 and rs_launches([S // 8 + 1] + [1] * 7, S) == 2
    # three ranks: W = floor(S / 48) units is not a whole divisor of the slot
    w3 = S // 48
    assert rs_launches([16 * w3, 0, 1], S) == 1 and rs_launches([16 * w3 + 1, 0, 1], S) == 2
