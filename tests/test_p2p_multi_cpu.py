"""Argument checks of the tensor-list point-to-point calls (B200Comm.send_multi / recv_multi /
get_multi) that need no GPU: they raise before anything reaches the library."""
import pytest
import torch

from ray_b200.comm import B200Comm


class _CudaLooking(torch.Tensor):
    """A CPU tensor that reports is_cuda, to reach the checks behind the device check."""

    @property
    def is_cuda(self):
        return True


def _comm():
    # no native communicator: every call below must be decided in Python
    return B200Comm.__new__(B200Comm)


@pytest.mark.parametrize("method", ["send_multi", "recv_multi"])
def test_empty_list_is_a_no_op(method):
    assert getattr(_comm(), method)([], 1) is None


def test_get_multi_empty_list_is_a_no_op():
    assert _comm().get_multi([], 1, []) is None


@pytest.mark.parametrize("method", ["send_multi", "recv_multi"])
def test_cpu_tensor_is_refused(method):
    with pytest.raises(RuntimeError, match="must be on GPU"):
        getattr(_comm(), method)([torch.ones(4)], 1)


@pytest.mark.parametrize("method", ["send_multi", "recv_multi"])
def test_non_contiguous_tensor_is_refused(method):
    t = torch.ones(4, 4).t().as_subclass(_CudaLooking)
    ok = torch.ones(4).as_subclass(_CudaLooking)
    with pytest.raises(RuntimeError, match="tensor 1 must be contiguous"):
        getattr(_comm(), method)([ok, t], 1)


def test_non_tensor_is_refused():
    with pytest.raises(RuntimeError, match="must be a torch.Tensor"):
        _comm().send_multi([[1, 2]], 1)


def test_get_multi_checks_tensors_and_list_lengths():
    with pytest.raises(ValueError, match="2 destination tensors but 1 offsets"):
        _comm().get_multi([torch.ones(4), torch.ones(4)], 1, [0])
    with pytest.raises(RuntimeError, match="must be on GPU"):
        _comm().get_multi([torch.ones(4)], 1, [0])
    with pytest.raises(RuntimeError, match="must be contiguous"):
        _comm().get_multi([torch.ones(4, 4).t().as_subclass(_CudaLooking)], 1, [0])
