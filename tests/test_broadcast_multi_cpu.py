"""Host-side logic of the tensor-list broadcast that needs no GPU: the argument checks of
B200Comm.broadcast_multi, B200Group.broadcast_multi and ray_b200.collective.broadcast_multi, and
B200DistributedDataParallel's choice between the one-launch path and torch's own buffer sync."""
import numpy as np
import pytest
import torch
from torch.nn.parallel import DistributedDataParallel

from ray_b200 import collective as col
from ray_b200.collective.b200_group import B200Group
from ray_b200.comm import B200Comm
from ray_b200.train import train_loop_utils as tlu


class _CudaLooking(torch.Tensor):
    """A CPU tensor that reports is_cuda, to reach the checks behind the device check."""

    @property
    def is_cuda(self):
        return True


def _cuda_looking(*shape):
    return torch.ones(*shape).as_subclass(_CudaLooking)


# ---- B200Comm -------------------------------------------------------------------------------------

def _comm():
    # no native communicator: every call below must be decided in Python
    return B200Comm.__new__(B200Comm)


def test_comm_empty_list_is_a_no_op():
    assert _comm().broadcast_multi([], 0) is None


def test_comm_refuses_cpu_non_contiguous_and_non_tensors():
    with pytest.raises(RuntimeError, match="must be on GPU"):
        _comm().broadcast_multi([torch.ones(4)], 0)
    with pytest.raises(RuntimeError, match="tensor 1 must be contiguous"):
        _comm().broadcast_multi([_cuda_looking(4), torch.ones(4, 4).t().as_subclass(_CudaLooking)], 0)
    with pytest.raises(RuntimeError, match="must be a torch.Tensor"):
        _comm().broadcast_multi([[1, 2]], 0)


# ---- B200Group ------------------------------------------------------------------------------------

class _RecordingComm:
    def __init__(self):
        self.calls = []

    def broadcast_multi(self, tensors, root):
        self.calls.append((tensors, root))


def _group(world=3):
    g = B200Group.__new__(B200Group)
    g._world_size, g._rank, g._group_name = world, 0, "g"
    g._comm = _RecordingComm()
    return g


def test_group_checks_list_rank_and_tensor_types():
    g = _group()
    with pytest.raises(RuntimeError, match="must be a list of tensors"):
        g.broadcast_multi((_cuda_looking(2),), 0)
    for bad in (-1, 3):
        with pytest.raises(ValueError, match="out of range for world size '3'"):
            g.broadcast_multi([_cuda_looking(2)], bad)
    with pytest.raises(RuntimeError, match="must be on GPU"):
        g.broadcast_multi([torch.ones(2)], 0)
    with pytest.raises(ValueError, match="Unsupported tensor type"):
        g.broadcast_multi([np.ones(2)], 0)
    assert g._comm.calls == []
    ts = [_cuda_looking(2), _cuda_looking(3)]
    g.broadcast_multi(ts, 2)
    assert len(g._comm.calls) == 1 and g._comm.calls[0][1] == 2
    assert all(a is b for a, b in zip(g._comm.calls[0][0], ts))


# ---- ray_b200.collective.broadcast_multi ----------------------------------------------------------

class _FakeGroup:
    world_size, rank = 2, 0

    def __init__(self):
        self.calls = []

    def broadcast_multi(self, tensors, src_rank):
        self.calls.append((tensors, src_rank))


def _with_group(group):
    mgr = col.GroupManager()
    mgr._groups["g"] = group
    return col.use_manager(mgr)


def test_functional_api_validates_like_broadcast():
    fake = _FakeGroup()
    with _with_group(fake):
        with pytest.raises(RuntimeError, match="must be a list of tensors"):
            col.broadcast_multi(torch.ones(2), 0, group_name="g")
        with pytest.raises(RuntimeError, match="empty list"):
            col.broadcast_multi([], 0, group_name="g")
        with pytest.raises(RuntimeError, match="Unrecognized tensor type"):
            col.broadcast_multi([torch.ones(2), "x"], 0, group_name="g")
        with pytest.raises(ValueError, match="negative"):
            col.broadcast_multi([torch.ones(2)], -1, group_name="g")
        with pytest.raises(ValueError, match="must be less than world size"):
            col.broadcast_multi([torch.ones(2)], 2, group_name="g")
        assert fake.calls == []
        ts = [torch.ones(2), np.zeros(3)]
        col.broadcast_multi(ts, 1, group_name="g")
        assert fake.calls == [(ts, 1)]
    with pytest.raises(RuntimeError, match="not initialized"):
        col.broadcast_multi([torch.ones(2)], 0, group_name="no-such-group")


def test_functional_api_refuses_a_group_without_list_broadcast():
    class Plain:
        world_size, rank = 2, 0

    with _with_group(Plain()):
        with pytest.raises(RuntimeError, match="has no list broadcast"):
            col.broadcast_multi([torch.ones(2)], 0, group_name="g")


# ---- B200DistributedDataParallel ------------------------------------------------------------------

class _FakePG:
    """Stands in for B200ProcessGroup (patched into train_loop_utils)."""

    def __init__(self):
        self.calls, self.waits = [], 0

    def broadcast_multi(self, tensors, root):
        pg = self

        class Work:
            def wait(self):
                pg.waits += 1
                return True

        self.calls.append((tensors, root))
        return Work()


@pytest.fixture()
def ddp(monkeypatch):
    """(model, native calls, torch calls): a B200DistributedDataParallel shell on a fake group."""
    monkeypatch.setattr(tlu, "B200ProcessGroup", _FakePG)
    fallback = []
    monkeypatch.setattr(DistributedDataParallel, "_distributed_broadcast_coalesced",
                        lambda self, tensors, size, rank=0: fallback.append((tensors, size, rank)))
    m = tlu.B200DistributedDataParallel.__new__(tlu.B200DistributedDataParallel)
    torch.nn.Module.__init__(m)
    m.process_group = _FakePG()
    m.device = torch.device("cpu")  # what _CudaLooking tensors report
    return m, m.process_group, fallback


def test_override_takes_one_native_call_for_contiguous_cuda_tensors(ddp):
    m, pg, fallback = ddp
    bufs = [_cuda_looking(3), torch.zeros(2, dtype=torch.int64).as_subclass(_CudaLooking)]
    m._distributed_broadcast_coalesced(bufs, 250 << 20, 1)
    assert len(pg.calls) == 1 and pg.calls[0][1] == 1 and pg.waits == 1 and fallback == []
    assert all(a is b for a, b in zip(pg.calls[0][0], bufs))
    m._distributed_broadcast_coalesced([], 250 << 20, 0)
    assert len(pg.calls) == 1 and fallback == []


@pytest.mark.parametrize("case", ["non_contiguous", "cpu_tensor", "other_device", "other_group"])
def test_override_falls_back_to_torch(ddp, case):
    m, pg, fallback = ddp
    bufs = [_cuda_looking(3), _cuda_looking(4, 4)]
    if case == "non_contiguous":
        bufs[1] = torch.ones(4, 4).t().as_subclass(_CudaLooking)
    elif case == "cpu_tensor":
        bufs[1] = torch.ones(4)
    elif case == "other_device":
        m.device = torch.device("cuda", 1)
    else:
        m.process_group = object()
    m._distributed_broadcast_coalesced(bufs, 123, 2)
    assert pg.calls == [] and len(fallback) == 1
    assert fallback[0][1:] == (123, 2) and all(a is b for a, b in zip(fallback[0][0], bufs))


def test_prepare_model_builds_the_subclass(monkeypatch):
    built = []

    class Recorder(tlu.B200DistributedDataParallel):
        def __init__(self, module, **kwargs):
            torch.nn.Module.__init__(self)
            built.append(kwargs)

    monkeypatch.setattr(tlu, "B200DistributedDataParallel", Recorder)
    monkeypatch.setattr(tlu.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(tlu.dist, "get_world_size", lambda: 2)
    out = tlu.prepare_model(torch.nn.Linear(2, 2), move_to_device=torch.device("cpu"),
                            parallel_strategy_kwargs={"broadcast_buffers": False})
    assert isinstance(out, DistributedDataParallel) and built == [{"broadcast_buffers": False}]
