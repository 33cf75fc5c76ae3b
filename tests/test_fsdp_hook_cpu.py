"""The FSDP communication hook's dispatch (CPU only): which process-group call it makes for sharded and
NO_SHARD gradients, with which scale and wire type, against a fake group that records the calls."""
import torch

from ray_b200.train import b200_fsdp_grad_hook


class _Work:
    def __init__(self, calls):
        self.calls = calls

    def wait(self):
        self.calls.append(("wait",))
        return True


class _FakeGroup:
    def __init__(self, n):
        self.n, self.calls = n, []

    def size(self):
        return self.n

    def grad_reducescatter(self, out, grad, scale, wire_dtype):
        self.calls.append(("grad_reducescatter", out, grad, scale, wire_dtype))
        return _Work(self.calls)

    def grad_allreduce(self, grad, scale, wire_dtype):
        self.calls.append(("grad_allreduce", grad, scale, wire_dtype))
        return _Work(self.calls)

    def _reduce_scatter_base(self, out, grad):
        self.calls.append(("_reduce_scatter_base", out, grad.clone()))
        return _Work(self.calls)

    def allreduce(self, tensors):
        self.calls.append(("allreduce", tensors[0].clone()))
        return _Work(self.calls)


def test_sharded_fp32_gradient_is_one_fused_reduce_scatter():
    pg = _FakeGroup(4)
    grad, out = torch.ones(12), torch.empty(3)
    b200_fsdp_grad_hook(torch.bfloat16)(pg, grad, out)
    (name, o, g, scale, wire), wait = pg.calls
    assert (name, scale, wire) == ("grad_reducescatter", 0.25, torch.bfloat16)
    assert o is out and g is grad and wait == ("wait",)
    assert torch.equal(grad, torch.ones(12))  # no pre-division: the kernel scales


def test_no_shard_fp32_gradient_is_one_fused_allreduce():
    pg = _FakeGroup(2)
    grad = torch.ones(5)
    b200_fsdp_grad_hook(torch.float16)(pg, grad)
    (name, g, scale, wire), wait = pg.calls
    assert (name, scale, wire) == ("grad_allreduce", 0.5, torch.float16)
    assert g is grad and wait == ("wait",)


def test_low_precision_gradients_pre_divide_and_fall_back():
    pg = _FakeGroup(2)
    grad, out = torch.full((4,), 3.0, dtype=torch.bfloat16), torch.empty(2, dtype=torch.bfloat16)
    b200_fsdp_grad_hook(torch.bfloat16)(pg, grad, out)
    (name, o, sent), wait = pg.calls
    assert name == "_reduce_scatter_base" and o is out and wait == ("wait",)
    assert torch.equal(sent, torch.full((4,), 1.5, dtype=torch.bfloat16))

    pg = _FakeGroup(4)
    grad = torch.full((3,), 2.0, dtype=torch.float16)
    b200_fsdp_grad_hook(torch.bfloat16)(pg, grad)
    (name, sent), wait = pg.calls
    assert name == "allreduce" and wait == ("wait",)
    assert torch.equal(sent, torch.full((3,), 0.5, dtype=torch.float16))


def test_explicit_process_group_wins_over_the_hook_state():
    mine, other = _FakeGroup(2), _FakeGroup(8)
    b200_fsdp_grad_hook(torch.float32, process_group=mine)(other, torch.ones(4), torch.empty(2))
    assert mine.calls[0][0] == "grad_reducescatter" and mine.calls[0][3] == 0.5 and not other.calls
