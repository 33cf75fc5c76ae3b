"""PREMUL_SUM's host side without a GPU: the factor c10d hands over in each options type, the
``PremulSum`` value, the refusal of integer operands, and which B200Comm call each c10d entry makes
with which op, against a fake communicator."""

import pytest
import torch
import torch.distributed as dist

from ray_b200 import _native as N
from ray_b200.comm import B200Comm, PremulSum
from ray_b200.train import process_group as P


@pytest.mark.parametrize("opts_type", [dist.AllreduceOptions, dist.ReduceOptions, dist.ReduceScatterOptions,
                                       dist.AllreduceCoalescedOptions])
@pytest.mark.parametrize("factor", [0.25, torch.tensor([0.5])])
def test_factor_is_read_from_every_options_type(opts_type, factor):
    opts = opts_type()
    opts.reduceOp = dist._make_nccl_premul_sum(factor)
    op = P._op_code(opts.reduceOp)
    assert isinstance(op, PremulSum)
    assert op.factor == (0.25 if isinstance(factor, float) else 0.5)
    assert op.device_factor is None  # a CPU tensor is read with .item()


def test_plain_ops_keep_their_codes():
    assert [P._op_code(o) for o in (dist.ReduceOp.SUM, dist.ReduceOp.PRODUCT, dist.ReduceOp.MIN,
                                    dist.ReduceOp.MAX, dist.ReduceOp.AVG)] == [N.SUM, N.PROD, N.MIN, N.MAX, N.AVG]
    with pytest.raises(RuntimeError, match="not supported by the b200 backend"):
        P._op_code(dist.ReduceOp.BAND)


class _FakeCuda(torch.Tensor):
    """A one-element float tensor that reports itself as a CUDA tensor (no GPU here)."""

    @property
    def is_cuda(self):
        return True


def test_premul_factor_forms():
    assert PremulSum(2).factor == 2.0 and PremulSum(torch.tensor(3.0)).factor == 3.0
    dev = torch.tensor([0.5]).as_subclass(_FakeCuda)
    op = PremulSum(dev)
    assert op.device_factor is dev
    with pytest.raises(RuntimeError, match="exactly one element"):
        PremulSum(torch.ones(2))
    with pytest.raises(RuntimeError, match="float or a one-element tensor"):
        PremulSum("0.5")


class _Lib:
    """Records b200_op_create_premul / b200_op_destroy and the reducing calls' op argument."""

    def __init__(self):
        self.calls = []

    def b200_op_create_premul(self, h, scalar, dtype, residence, out):
        self.calls.append(("create", scalar, dtype, residence))
        out._obj.value = 0x100
        return 0

    def b200_op_destroy(self, h, op):
        self.calls.append(("destroy", op))
        return 0

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name,) + args)
            return 0
        return call


def _comm():
    c = B200Comm.__new__(B200Comm)
    c._lib, c._h, c.device = _Lib(), None, 0
    c._stream = lambda stream=None: 0
    return c


def test_with_op_creates_uses_and_destroys_a_native_op():
    c = _comm()
    seen = []
    c._with_op(PremulSum(0.25), torch.bfloat16, seen.append)
    (create, scalar, dtype, residence), (destroy, op) = c._lib.calls
    assert (create, dtype, residence, destroy) == ("create", N.BF16, N.PREMUL_HOST, "destroy")
    assert seen == [0x100] and op == 0x100
    c._lib.calls.clear()
    c._with_op(N.MAX, torch.int32, seen.append)  # plain ops pass straight through
    assert seen[-1] == N.MAX and not c._lib.calls


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64, torch.uint8, torch.int8, torch.bool])
def test_integer_operands_are_refused_before_anything_is_created(dtype):
    c = _comm()
    with pytest.raises(RuntimeError, match="Cannot use ReduceOp.PREMUL_SUM"):
        c._with_op(PremulSum(0.5), dtype, lambda code: pytest.fail("enqueued"))
    assert not c._lib.calls


def test_device_factor_must_match_the_operand():
    c = _comm()
    with pytest.raises(RuntimeError, match="factor tensor must hold one torch.float32"):
        c._with_op(PremulSum(torch.tensor([0.5], dtype=torch.float64).as_subclass(_FakeCuda)), torch.float32,
                   lambda code: pytest.fail("enqueued"))
    assert not c._lib.calls


# ---- c10d routing -------------------------------------------------------------------------------

class _FakeComm:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args, **kwargs):
            self.calls.append((name, args))
        return call


class _Cuda(torch.Tensor):
    @property
    def is_cuda(self):
        return True

    def record_stream(self, stream):
        pass


def _group():
    pg = P.B200ProcessGroup.__new__(P.B200ProcessGroup)
    comm = _FakeComm()
    recorded = []

    def run(tensors, fn, result, tag="op"):
        recorded.append(list(tensors))
        fn(comm)

    pg._run = run
    pg._size = 2
    return pg, comm, recorded


def _t(n=4):
    return torch.zeros(n).as_subclass(_Cuda)


def _opts(cls, factor):
    o = cls()
    o.reduceOp = dist._make_nccl_premul_sum(factor)
    return o


def _routes():
    x, y = _t(8), _t(4)
    return {
        "allreduce": (lambda pg, f: pg.allreduce([x], _opts(dist.AllreduceOptions, f)), "allreduce"),
        "allreduce_coalesced": (lambda pg, f: pg.allreduce_coalesced([x, y], _opts(dist.AllreduceCoalescedOptions, f)),
                                "allreduce_multi"),
        "reduce": (lambda pg, f: pg.reduce([x], _opts(dist.ReduceOptions, f)), "reduce"),
        "reduce_scatter": (lambda pg, f: pg.reduce_scatter([y], [[y, y]], _opts(dist.ReduceScatterOptions, f)),
                           "reducescatter"),
        "reduce_scatter uneven": (lambda pg, f: pg.reduce_scatter([y], [[y, _t(6)]],
                                                                  _opts(dist.ReduceScatterOptions, f)),
                                  "reducescatterv"),
        "reduce_scatter list": (lambda pg, f: pg.reduce_scatter([y, y], [[y, y], [y, y]],
                                                                _opts(dist.ReduceScatterOptions, f)),
                                "reducescatter_multi"),
        "_reduce_scatter_base": (lambda pg, f: pg._reduce_scatter_base(y, x, _opts(dist.ReduceScatterOptions, f)),
                                 "reducescatter_from"),
        "reduce_scatter_tensor_coalesced": (
            lambda pg, f: pg.reduce_scatter_tensor_coalesced([y], [x], _opts(dist.ReduceScatterOptions, f)),
            "reducescatter_from_multi"),
    }


@pytest.mark.parametrize("entry", list(_routes()))
@pytest.mark.parametrize("kind", ["float", "cuda tensor"])
def test_every_reducing_entry_passes_the_factor(entry, kind):
    call, method = _routes()[entry]
    factor = 0.125 if kind == "float" else torch.tensor([0.125]).as_subclass(_Cuda)
    pg, comm, recorded = _group()
    call(pg, factor)
    (name, args), = comm.calls
    assert name == method
    op = args[-1]
    assert isinstance(op, PremulSum)
    if kind == "float":
        assert op.factor == 0.125 and op.device_factor is None
        assert all(t is not factor for t in recorded[0])
    else:
        # the CUDA factor is read by the kernels: it is recorded on the communication stream
        assert op.device_factor is not None and recorded[0][-1] is op.device_factor
