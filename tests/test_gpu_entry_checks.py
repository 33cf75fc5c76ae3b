"""Argument contract of the C entry points, called through the raw binding so that no Python-side
check runs first: for every invalid argument the status, the error text and that nothing was
launched; the zero-count and world-1 shortcuts succeed without a launch.  Also the per-launch cap
of the pull all-gather, which must follow the all-gather's own chunk size."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

MiB = 1 << 20
BAD = 99  # neither a dtype, an op nor a wire dtype


@pytest.fixture(scope="module")
def groups(native_lib):
    from ray_b200.testing import LocalGroup

    gs = {1: LocalGroup(1, timeout_ms=20000, staging_bytes=2 * MiB, inbox_bytes=2 * MiB),
          2: LocalGroup(2, timeout_ms=20000, staging_bytes=2 * MiB, heap_bytes=MiB, inbox_bytes=2 * MiB,
                        enable_multicast=False)}
    yield gs
    for g in gs.values():
        g.destroy()


def _ptrs(*xs):
    return (ctypes.c_void_p * 8)(*xs)


def _counts(*xs):
    return (ctypes.c_size_t * 8)(*xs)


def test_entry_points_reject_invalid_arguments_without_launching(groups):
    from ray_b200 import _native as N

    lib = N.load()
    g1, g2 = groups[1], groups[2]
    h1, h = g1.comms[0]._h, g2.comms[0]._h
    dev = g2.device(0)
    x = torch.zeros(64, device=dev)
    y = torch.zeros(64, device=dev)
    x1 = torch.ones(64, device=g1.device(0))
    y1 = torch.zeros(64, device=g1.device(0))
    X, Y = x.data_ptr(), y.data_ptr()
    heap = g2.comms[0].heap_range()[1]
    F32, SUM, S = N.F32, N.SUM, None
    INV, UNS, OK = N.ERR_INVALID, N.ERR_UNSUPPORTED, N.OK

    cases = [
        # (what, call, status, substring of b200_last_error() or None)
        # every entry point checks the communicator first
        ("allreduce null comm", lambda: lib.b200_allreduce(None, X, X, 64, BAD, BAD, 0, S), INV, "null communicator"),
        ("multi null comm", lambda: lib.b200_allreduce_multi(None, None, None, 0, F32, SUM, S), INV, "null communicator"),
        ("allgather null comm", lambda: lib.b200_allgather(None, X, None, 64, F32, S), INV, "null communicator"),
        ("broadcast null comm", lambda: lib.b200_broadcast(None, X, 64, F32, 0, S), INV, "null communicator"),
        ("barrier null comm", lambda: lib.b200_barrier(None, S), INV, "null communicator"),
        ("reducescatter null comm", lambda: lib.b200_reducescatter(None, None, X, 64, F32, SUM, S), INV,
         "null communicator"),
        ("reduce null comm", lambda: lib.b200_reduce(None, X, 64, F32, SUM, 0, S), INV, "null communicator"),
        ("send null comm", lambda: lib.b200_send(None, X, 16, 1, S), INV, "null communicator"),
        ("recv null comm", lambda: lib.b200_recv(None, X, 16, 1, S), INV, "null communicator"),
        ("alltoall null comm", lambda: lib.b200_alltoall(None, None, None, None, None, F32, S), INV,
         "null communicator"),
        ("symm_base null comm", lambda: lib.b200_symm_base(None, None, None), INV, "null communicator"),
        ("get null comm", lambda: lib.b200_get(None, X, 0, 0, 16, S), INV, "null communicator"),
        ("grad null comm", lambda: lib.b200_grad_allreduce(None, X, 64, 1.0, F32, S), INV, "null communicator"),
        # all-reduce
        ("allreduce dtype", lambda: lib.b200_allreduce(h, X, X, 64, BAD, SUM, 0, S), UNS, f"unsupported dtype {BAD}"),
        ("allreduce dtype before op", lambda: lib.b200_allreduce(h, X, X, 64, BAD, BAD, 0, S), UNS,
         f"unsupported dtype {BAD}"),
        ("allreduce op", lambda: lib.b200_allreduce(h, X, X, 64, F32, BAD, 0, S), UNS, f"unsupported reduce op {BAD}"),
        ("allreduce negative op", lambda: lib.b200_allreduce(h, X, X, 64, F32, -1, 0, S), UNS,
         "unsupported reduce op -1"),
        ("allreduce zero count", lambda: lib.b200_allreduce(h, None, None, 0, F32, SUM, 0, S), OK, None),
        ("allreduce null in", lambda: lib.b200_allreduce(h, None, X, 64, F32, SUM, 0, S), INV, "null tensor pointer"),
        ("allreduce null out", lambda: lib.b200_allreduce(h, X, None, 64, F32, SUM, 0, S), INV, "null tensor pointer"),
        ("allreduce NVLS without multicast", lambda: lib.b200_allreduce(h, X, X, 64, F32, SUM, N.ALGO_NVLS, S), UNS,
         "multicast mapping is not active"),
        ("allreduce PIPE misaligned", lambda: lib.b200_allreduce(h, X + 4, X + 4, 60, F32, SUM, N.ALGO_PIPE, S), UNS,
         "needs 16-byte aligned operands"),
        ("allreduce world 1", lambda: lib.b200_allreduce(h1, x1.data_ptr(), y1.data_ptr(), 64, F32, SUM, 0, S), OK,
         None),
        # multi-tensor all-reduce
        ("multi dtype", lambda: lib.b200_allreduce_multi(h, _ptrs(X), _counts(64), 1, BAD, SUM, S), UNS,
         f"unsupported dtype {BAD}"),
        ("multi op", lambda: lib.b200_allreduce_multi(h, _ptrs(X), _counts(64), 1, F32, BAD, S), UNS,
         f"unsupported reduce op {BAD}"),
        ("multi negative count", lambda: lib.b200_allreduce_multi(h, _ptrs(X), _counts(64), -1, F32, SUM, S), INV,
         "invalid tensor list"),
        ("multi null list", lambda: lib.b200_allreduce_multi(h, None, _counts(64), 1, F32, SUM, S), INV,
         "invalid tensor list"),
        ("multi null tensor", lambda: lib.b200_allreduce_multi(h, _ptrs(None, X), _counts(64, 64), 2, F32, SUM, S),
         INV, "tensor 0 is null"),
        ("multi empty tensors", lambda: lib.b200_allreduce_multi(h, _ptrs(None), _counts(0), 1, F32, SUM, S), OK, None),
        ("multi world 1", lambda: lib.b200_allreduce_multi(h1, _ptrs(x1.data_ptr()), _counts(64), 1, F32, SUM, S), OK,
         None),
        # all-gather
        ("allgather dtype", lambda: lib.b200_allgather(h, X, _ptrs(X, Y), 64, BAD, S), UNS, f"unsupported dtype {BAD}"),
        ("allgather zero count", lambda: lib.b200_allgather(h, None, None, 0, F32, S), OK, None),
        ("allgather null in", lambda: lib.b200_allgather(h, None, _ptrs(X, Y), 64, F32, S), INV, "null tensor pointer"),
        ("allgather null outs", lambda: lib.b200_allgather(h, X, None, 64, F32, S), INV, "null tensor pointer"),
        ("allgather null output", lambda: lib.b200_allgather(h, X, _ptrs(Y, None), 64, F32, S), INV,
         "output tensor 1 is null"),
        ("allgather world 1", lambda: lib.b200_allgather(h1, x1.data_ptr(), _ptrs(y1.data_ptr()), 64, F32, S), OK,
         None),
        # broadcast: the world-1 shortcut comes before the null check
        ("broadcast dtype", lambda: lib.b200_broadcast(h, X, 64, BAD, 0, S), UNS, f"unsupported dtype {BAD}"),
        ("broadcast root", lambda: lib.b200_broadcast(h, X, 64, F32, 2, S), INV,
         "root rank 2 out of range for world size 2"),
        ("broadcast negative root", lambda: lib.b200_broadcast(h, X, 64, F32, -1, S), INV,
         "root rank -1 out of range for world size 2"),
        ("broadcast root before zero count", lambda: lib.b200_broadcast(h, X, 0, F32, 5, S), INV,
         "root rank 5 out of range"),
        ("broadcast zero count", lambda: lib.b200_broadcast(h, None, 0, F32, 0, S), OK, None),
        ("broadcast null buf", lambda: lib.b200_broadcast(h, None, 64, F32, 0, S), INV, "null tensor pointer"),
        ("broadcast world 1 null buf", lambda: lib.b200_broadcast(h1, None, 64, F32, 0, S), OK, None),
        # barrier
        ("barrier world 1", lambda: lib.b200_barrier(h1, S), OK, None),
        # reduce-scatter
        ("reducescatter dtype", lambda: lib.b200_reducescatter(h, _ptrs(X, Y), X, 64, BAD, SUM, S), UNS,
         f"unsupported dtype {BAD}"),
        ("reducescatter op", lambda: lib.b200_reducescatter(h, _ptrs(X, Y), X, 64, F32, BAD, S), UNS,
         f"unsupported reduce op {BAD}"),
        ("reducescatter zero count", lambda: lib.b200_reducescatter(h, None, None, 0, F32, SUM, S), OK, None),
        ("reducescatter null ins", lambda: lib.b200_reducescatter(h, None, X, 64, F32, SUM, S), INV,
         "null tensor pointer"),
        ("reducescatter null out", lambda: lib.b200_reducescatter(h, _ptrs(X, Y), None, 64, F32, SUM, S), INV,
         "null tensor pointer"),
        ("reducescatter null input", lambda: lib.b200_reducescatter(h, _ptrs(X, None), Y, 64, F32, SUM, S), INV,
         "input tensor 1 is null"),
        ("reducescatter world 1",
         lambda: lib.b200_reducescatter(h1, _ptrs(x1.data_ptr()), y1.data_ptr(), 64, F32, SUM, S), OK, None),
        # reduce: the null check comes before the world-1 shortcut
        ("reduce dtype", lambda: lib.b200_reduce(h, X, 64, BAD, SUM, 0, S), UNS, f"unsupported dtype {BAD}"),
        ("reduce op", lambda: lib.b200_reduce(h, X, 64, F32, BAD, 0, S), UNS, f"unsupported reduce op {BAD}"),
        ("reduce root", lambda: lib.b200_reduce(h, X, 64, F32, SUM, 2, S), INV,
         "root rank 2 out of range for world size 2"),
        ("reduce root before zero count", lambda: lib.b200_reduce(h, X, 0, F32, SUM, -3, S), INV,
         "root rank -3 out of range"),
        ("reduce zero count", lambda: lib.b200_reduce(h, None, 0, F32, SUM, 0, S), OK, None),
        ("reduce null buf", lambda: lib.b200_reduce(h, None, 64, F32, SUM, 0, S), INV, "null tensor pointer"),
        ("reduce world 1 null buf", lambda: lib.b200_reduce(h1, None, 64, F32, SUM, 0, S), INV, "null tensor pointer"),
        ("reduce world 1", lambda: lib.b200_reduce(h1, x1.data_ptr(), 64, F32, SUM, 0, S), OK, None),
        # send / recv
        ("send peer", lambda: lib.b200_send(h, X, 16, 2, S), INV, "peer rank 2 out of range for world size 2"),
        ("recv negative peer", lambda: lib.b200_recv(h, X, 16, -1, S), INV, "peer rank -1 out of range"),
        ("send peer before zero count", lambda: lib.b200_send(h, X, 0, 7, S), INV, "peer rank 7 out of range"),
        ("send to self", lambda: lib.b200_send(h, X, 16, 0, S), INV, "peer rank 0 is this rank"),
        ("recv from self", lambda: lib.b200_recv(h, X, 16, 0, S), INV, "peer rank 0 is this rank"),
        ("send zero count", lambda: lib.b200_send(h, None, 0, 1, S), OK, None),
        ("recv null buf", lambda: lib.b200_recv(h, None, 16, 1, S), INV, "null tensor pointer"),
        # all-to-all
        ("alltoall dtype", lambda: lib.b200_alltoall(h, _ptrs(X, Y), _counts(4, 4), _ptrs(X, Y), _counts(4, 4), BAD, S),
         UNS, f"unsupported dtype {BAD}"),
        ("alltoall null arrays", lambda: lib.b200_alltoall(h, None, _counts(4, 4), _ptrs(X, Y), _counts(4, 4), F32, S),
         INV, "null argument array"),
        ("alltoall null input",
         lambda: lib.b200_alltoall(h, _ptrs(X, None), _counts(0, 4), _ptrs(Y, Y + 64), _counts(0, 4), F32, S),
         INV, "input 1 is null but has 4 elements"),
        ("alltoall null output",
         lambda: lib.b200_alltoall(h, _ptrs(X, X + 64), _counts(0, 4), _ptrs(Y, None), _counts(0, 4), F32, S),
         INV, "output 1 is null but has 4 elements"),
        ("alltoall own segment",
         lambda: lib.b200_alltoall(h, _ptrs(X, X + 64), _counts(4, 4), _ptrs(Y, Y + 64), _counts(8, 4), F32, S),
         INV, "own segment: 4 elements sent but 8 received"),
        ("alltoall overlap",
         lambda: lib.b200_alltoall(h, _ptrs(X, X + 64), _counts(4, 4), _ptrs(Y, X + 64), _counts(4, 4), F32, S),
         INV, "output 1 overlaps input 1"),
        ("alltoall nothing to move",
         lambda: lib.b200_alltoall(h, _ptrs(None, None), _counts(0, 0), _ptrs(None, None), _counts(0, 0), F32, S),
         OK, None),
        ("alltoall world 1",
         lambda: lib.b200_alltoall(h1, _ptrs(x1.data_ptr()), _counts(64), _ptrs(y1.data_ptr()), _counts(64), F32, S),
         OK, None),
        # one-sided get: the heap range is checked before the zero count
        ("get source", lambda: lib.b200_get(h, Y, 2, 0, 16, S), INV, "source rank 2 out of range for world size 2"),
        ("get negative source", lambda: lib.b200_get(h, Y, -1, 0, 16, S), INV, "source rank -1 out of range"),
        ("get outside heap", lambda: lib.b200_get(h, Y, 1, heap - 16, 32, S), INV,
         f"[{heap - 16}, {heap + 16}) is outside the {heap}-byte symmetric heap"),
        ("get outside heap before zero count", lambda: lib.b200_get(h, Y, 1, heap + 16, 0, S), INV,
         f"is outside the {heap}-byte symmetric heap"),
        ("get zero count", lambda: lib.b200_get(h, None, 1, 0, 0, S), OK, None),
        ("get null dst", lambda: lib.b200_get(h, None, 1, 0, 16, S), INV, "null tensor pointer"),
        # fused gradient all-reduce
        ("grad wire dtype", lambda: lib.b200_grad_allreduce(h, X, 64, 1.0, BAD, S), UNS,
         f"wire dtype must be f32, bf16 or f16 (got {BAD})"),
        ("grad integer wire dtype", lambda: lib.b200_grad_allreduce(h, X, 64, 1.0, N.I32, S), UNS,
         f"(got {N.I32})"),
        ("grad zero count", lambda: lib.b200_grad_allreduce(h, None, 0, 1.0, F32, S), OK, None),
        ("grad null grad", lambda: lib.b200_grad_allreduce(h, None, 64, 1.0, F32, S), INV, "null gradient pointer"),
        # symmetric heap base
        ("symm_base", lambda: lib.b200_symm_base(h, None, None), OK, None),
    ]
    comms = g1.comms + g2.comms
    for what, call, status, text in cases:
        before = [c.launch_count for c in comms]
        got = call()
        assert got == status, (what, got, N.last_error())
        if text is not None:
            assert text in N.last_error(), (what, N.last_error())
        assert [c.launch_count for c in comms] == before, what
    g1.synchronize()
    g2.synchronize()
    assert torch.equal(y1, x1)  # the world-1 shortcuts copied in -> out


def test_pull_allgather_launch_takes_at_most_max_pipe_chunks_of_its_own_chunk(native_lib):
    """A 640 MiB staging slot holds 640 chunks of the all-gather's default 1 MiB, but the per-chunk
    flags and counters have room for 512: a 600 MiB all-gather must take two launches (512 + 88
    chunks) and still be bit exact."""
    from ray_b200.testing import LocalGroup

    world, nbytes = 3, 600 * MiB
    numel = nbytes // 4
    with LocalGroup(world, timeout_ms=60000, staging_bytes=640 * MiB, inbox_bytes=2 * MiB) as g:
        xs = [torch.randn(numel, device=g.device(r), generator=torch.Generator(device=g.device(r)).manual_seed(r))
              for r in range(world)]
        outs = [[torch.empty(numel, device=g.device(r)) for _ in range(world)] for r in range(world)]
        before = [c.launch_count for c in g.comms]
        g.run(lambda c, r: c.allgather(outs[r], xs[r]))
        assert [c.launch_count - b for c, b in zip(g.comms, before)] == [2] * world
        for r in range(world):
            for p in range(world):
                assert torch.equal(outs[r][p], xs[p].to(g.device(r))), (r, p)
