"""Tensor-list broadcast in one launch per staging slot: b200_broadcast_multi
(B200Comm.broadcast_multi, B200Group.broadcast_multi, ray_b200.collective.broadcast_multi).

Every byte each rank ends up with is compared with the root's tensors.  The tensors of every rank
are views into one buffer with guard bytes around each of them, and the guard bytes must come back
unchanged: the padding of a tensor's last 16-byte unit goes through the staging slot but must never
be stored.  The launch count of every call is checked against the plan: one launch per window of at
most one staging slot of each table's packed stream.
"""
import ctypes

import numpy as np
import pytest
import torch

from ray_b200 import _native as N

pytestmark = pytest.mark.gpu

TABLE = N.P2P_TABLE_MAX
GUARD = 0x5A
STAGING = 2 << 20  # the library's smallest staging slot: lists of a few MiB span several windows


@pytest.fixture(scope="module")
def groups(native_lib):
    from ray_b200.testing import LocalGroup

    cache = {}

    def get(n):
        if n not in cache:
            cache[n] = LocalGroup(n, timeout_ms=15000, staging_bytes=STAGING)
        return cache[n]

    yield get
    for g in cache.values():
        g.destroy()


def planned_launches(sizes, staging=STAGING):
    """Sum over tables of ceil(16 * units / staging_bytes)."""
    nonempty = [s for s in sizes if s]
    launches = 0
    for i in range(0, len(nonempty), TABLE):
        units = sum(-(-s // 16) for s in nonempty[i:i + TABLE])
        launches += -(-16 * units // staging)
    return launches


def _layout(sizes, misalign):
    """Offsets of tensors of `sizes` bytes in one buffer: tensor i starts misalign(i) bytes past a
    16-byte boundary, with at least 32 guard bytes on both sides."""
    offs, pos = [], 32
    for i, s in enumerate(sizes):
        pos = (pos + 15) // 16 * 16 + misalign(i)
        offs.append(pos)
        pos += s + 32
    return offs, pos


def _bcast(g, root, sizes, misalign=lambda r, i: 0, seed=0):
    """broadcast_multi of a list of `sizes` bytes from `root`; checks every byte of every rank, the
    guard bytes and the launch count of every rank."""
    n = g.world_size
    rng = np.random.default_rng(seed)
    data = [torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in sizes]
    bufs, views, wants = [], [], []
    for r in range(n):
        offs, total = _layout(sizes, lambda i: misalign(r, i))
        buf = torch.full((total,), GUARD, dtype=torch.uint8)
        want = buf.clone()
        for o, s, d in zip(offs, sizes, data):
            want[o:o + s] = d
            # the root holds the data; every other rank starts with different bytes
            buf[o:o + s] = d if r == root else torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8))
        buf = buf.to(g.device(r))
        bufs.append(buf)
        views.append([buf[o:o + s] for o, s in zip(offs, sizes)])
        wants.append(want)
    before = [c.launch_count for c in g.comms]
    g.run(lambda c, r: c.broadcast_multi(views[r], root))
    launches = [c.launch_count - b for c, b in zip(g.comms, before)]
    assert launches == [planned_launches(sizes) if n > 1 else 0] * n, launches
    for r in range(n):
        assert torch.equal(bufs[r].cpu(), wants[r]), f"rank {r}: payload or guard bytes differ (root {root})"


LISTS = {
    "one": [100_000],
    "bytes_1_to_15": list(range(1, 16)),
    "zeros_scattered": [0, 100, 0, 0, 4096, 0, 17, 33, 0],
    "tiny": [1, 2, 3, 4097, 5],
    "several_slots": [(1 << 20) + 16 * i + (i % 3) for i in range(7)],
    "larger_than_slot": [3, (5 << 20) + 7, 11],
    "table_max_plus_one": [16 + (i % 37) for i in range(TABLE + 1)],
    "tables_spanning_slots": [9000 + i for i in range(2 * TABLE + 10)],
}


def test_plan_formula():
    assert planned_launches([]) == 0 and planned_launches([0, 0]) == 0
    assert planned_launches([1]) == 1 and planned_launches([STAGING]) == 1 and planned_launches([STAGING + 1]) == 2
    assert planned_launches(LISTS["several_slots"]) == 4
    assert planned_launches(LISTS["larger_than_slot"]) == 3
    assert planned_launches(LISTS["table_max_plus_one"]) == 2
    assert planned_launches(LISTS["tables_spanning_slots"]) == 2 + 2 + 1


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("name", list(LISTS))
def test_lists_byte_for_byte_every_root(groups, world, name):
    g = groups(world)
    for root in range(world):
        _bcast(g, root, LISTS[name], seed=root)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_views_misaligned_by_1_to_15_bytes(groups, world):
    g = groups(world)
    sizes = [(i * 977) % 5000 + 1 for i in range(40)] + [300_000, 70_001, (2 << 20) + 9]
    for root in range(world):
        _bcast(g, root, sizes, misalign=lambda r, i: (i * (r + 3) + root) % 15 + 1, seed=10 + root)
    # aligned root, misaligned receivers and the other way round
    _bcast(g, 0, sizes, misalign=lambda r, i: 0 if r == 0 else i % 15 + 1, seed=20)
    _bcast(g, world - 1, sizes, misalign=lambda r, i: 0 if r != world - 1 else (7 * i) % 15 + 1, seed=21)


def test_empty_lists_launch_nothing(groups):
    g = groups(2)
    before = [c.launch_count for c in g.comms]
    g.run(lambda c, r: c.broadcast_multi([], 0))
    g.run(lambda c, r: c.broadcast_multi([torch.empty(0, device=g.device(r)),
                                          torch.empty(0, dtype=torch.int64, device=g.device(r))], 1))
    assert [c.launch_count for c in g.comms] == before


def test_world_one_launches_nothing(native_lib):
    from ray_b200.testing import LocalGroup

    with LocalGroup(1, staging_bytes=STAGING) as g:
        x = torch.arange(1000, dtype=torch.float32, device=g.device(0))
        before = g.comms[0].launch_count
        g.run(lambda c, r: c.broadcast_multi([x, x[:7]], 0))
        assert g.comms[0].launch_count == before
        assert torch.equal(x.cpu(), torch.arange(1000, dtype=torch.float32))


@pytest.mark.parametrize("world", [2, 3])
def test_mixed_dtypes(groups, world):
    g = groups(world)
    rng = np.random.default_rng(5)
    sent = [torch.from_numpy(rng.standard_normal((17, 3)).astype(np.float32)),
            torch.from_numpy(rng.standard_normal(1001)).to(torch.float16),
            torch.arange(-50, 77, dtype=torch.int64), torch.from_numpy(rng.random(13) < 0.5),
            torch.from_numpy(rng.standard_normal(2049)).to(torch.bfloat16), torch.zeros(0, dtype=torch.float64),
            torch.from_numpy(rng.integers(0, 256, 7, dtype=np.uint8)), torch.tensor(3, dtype=torch.int64)]
    root = world - 1
    tensors = [[t.to(g.device(r)) if r == root else torch.zeros_like(t, device=g.device(r)) for t in sent]
               for r in range(world)]
    g.run(lambda c, r: c.broadcast_multi(tensors[r], root))
    for r in range(world):
        for t, s in zip(tensors[r], sent):
            assert t.dtype == s.dtype and torch.equal(t.cpu(), s), (r, s.dtype)


@pytest.mark.parametrize("world", [2, 4])
def test_interleaves_with_broadcast_and_allreduce_in_stream_order(groups, world):
    """broadcast, broadcast_multi, allreduce, broadcast_multi, broadcast: the launch counter and the
    staging-slot parity carry on from one call to the next."""
    g = groups(world)
    rng = np.random.default_rng(9)
    a = torch.from_numpy(rng.standard_normal(300_000).astype(np.float32))
    lst = [torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in (5, 70_000, 0, 3 << 20, 3)]
    lst2 = [torch.from_numpy(rng.standard_normal(s).astype(np.float32)) for s in (1, 1000, 600_000)]
    b = torch.from_numpy(rng.standard_normal(123).astype(np.float32))
    for rep in range(2):
        ra, rl, rl2 = rep % world, (rep + 1) % world, world - 1
        xa = [a.to(g.device(r)) if r == ra else torch.zeros_like(a, device=g.device(r)) for r in range(world)]
        xl = [[t.to(g.device(r)) if r == rl else torch.zeros_like(t, device=g.device(r)) for t in lst]
              for r in range(world)]
        xl2 = [[t.to(g.device(r)) if r == rl2 else torch.zeros_like(t, device=g.device(r)) for t in lst2]
               for r in range(world)]
        xs = [torch.full((5000,), float(r + 1), device=g.device(r)) for r in range(world)]
        xb = [b.to(g.device(r)) if r == 0 else torch.zeros_like(b, device=g.device(r)) for r in range(world)]

        def f(c, r):
            c.broadcast(xa[r], ra)
            c.broadcast_multi(xl[r], rl)
            c.allreduce(xs[r], N.SUM)
            c.broadcast_multi(xl2[r], rl2)
            c.broadcast(xb[r], 0)

        g.run(f)
        for r in range(world):
            assert torch.equal(xa[r].cpu(), a) and torch.equal(xb[r].cpu(), b)
            assert all(torch.equal(o.cpu(), t) for o, t in zip(xl[r], lst))
            assert all(torch.equal(o.cpu(), t) for o, t in zip(xl2[r], lst2))
            assert torch.all(xs[r].cpu() == world * (world + 1) / 2)


def test_cuda_graph_replay_matches_eager(groups):
    g = groups(3)
    sizes = [3, 4096, 100_001, (2 << 20) + 5] + [40 + i for i in range(TABLE)]
    root = 1
    lists = [[torch.zeros(s, dtype=torch.uint8, device=g.device(r)) for s in sizes] for r in range(3)]

    def f(c, r):
        c.broadcast_multi(lists[r], root, stream=g.streams[r])

    g.run(f)  # eager first, outside capture
    graphs = []
    for r, c in enumerate(g.comms):
        torch.cuda.set_device(g.devices[r])
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=g.streams[r]):
            f(c, r)
        graphs.append(gr)
    for rep in range(2):
        rng = np.random.default_rng(100 + rep)
        fresh = [torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in sizes]
        for r in range(3):
            for t, d in zip(lists[r], fresh):
                if r == root:
                    t.copy_(d)
                else:
                    t.zero_()
        for d in set(g.devices):
            torch.cuda.synchronize(d)
        for r in range(3):
            torch.cuda.set_device(g.devices[r])
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        g.synchronize()
        graph_out = [[t.cpu() for t in lists[r]] for r in range(3)]
        for r in range(3):
            assert all(torch.equal(o, d) for o, d in zip(graph_out[r], fresh)), r
        for r in range(3):
            if r != root:
                for t in lists[r]:
                    t.zero_()
        g.run(f)
        for r in range(3):
            assert all(torch.equal(t.cpu(), e) for t, e in zip(lists[r], graph_out[r])), "eager and replay differ"


def _arr(ctype, vals):
    return (ctype * max(len(vals), 1))(*vals)


def test_refused_calls_launch_nothing(groups):
    g = groups(2)
    lib, c = N.load(), g.comms[0]
    h, dev = c._h, g.device(0)
    x = torch.zeros(64, dtype=torch.uint8, device=dev)
    P = _arr(ctypes.c_void_p, [x.data_ptr(), x.data_ptr() + 32])
    S = _arr(ctypes.c_size_t, [16, 16])
    cases = [
        ("root negative", lambda: lib.b200_broadcast_multi(h, P, S, 2, -1, None),
         "root rank -1 out of range for world size 2"),
        ("root too large", lambda: lib.b200_broadcast_multi(h, P, S, 2, 2, None),
         "root rank 2 out of range for world size 2"),
        ("negative count", lambda: lib.b200_broadcast_multi(h, P, S, -1, 0, None), "ntensors -1 is negative"),
        ("null pointer array", lambda: lib.b200_broadcast_multi(h, None, S, 2, 0, None), "null argument array"),
        ("null size array", lambda: lib.b200_broadcast_multi(h, P, None, 2, 0, None), "null argument array"),
        ("null entry", lambda: lib.b200_broadcast_multi(h, _arr(ctypes.c_void_p, [x.data_ptr(), None]), S, 2, 0,
                                                        None), "tensor 1 is null but has 16 bytes"),
    ]
    before = c.launch_count
    with torch.cuda.device(dev):
        for name, call, text in cases:
            assert call() == N.ERR_INVALID, name
            assert text in N.last_error(), (name, N.last_error())
        # allowed: no arrays with no tensors, and NULL pointers of empty entries
        assert lib.b200_broadcast_multi(h, None, None, 0, 0, None) == N.OK
    torch.cuda.synchronize(dev)
    assert c.launch_count == before


@pytest.mark.parametrize("world", [3, 4])
def test_nvls_windows_byte_for_byte(groups, world):
    """From 3 ranks on, windows of at least 64 KiB take the multicast store when the NVLS mapping
    exists (the root writes each unit once, the switch replicates it)."""
    g = groups(world)
    if not g.has_multicast:
        pytest.skip("no NVLS multicast mapping on this system")
    sizes = [(1 << 20) + 3, 5, 64 << 10, (3 << 20) + 16] + [1000 + i for i in range(300)]
    for root in range(world):
        _bcast(g, root, sizes, misalign=lambda r, i: (i + r) % 16, seed=root)


# ---- integration --------------------------------------------------------------------------------

def test_collective_api_broadcast_multi(native_lib):
    """ray_b200.collective.broadcast_multi through a B200 group of three workers."""
    from tests.test_gpu_api import Workers

    w = Workers(3)
    w.init("bcast-multi")
    try:
        payload = [torch.randn(17, 3), torch.arange(1000, dtype=torch.int64), torch.randn(5).to(torch.float16)]

        def f(r):
            ts = [t.to(w.dev(r)) if r == 2 else torch.zeros_like(t, device=w.dev(r)) for t in payload]
            comm = w.col.get_group_handle("bcast-multi").comm
            before = comm.launch_count
            w.col.broadcast_multi(ts, src_rank=2, group_name="bcast-multi")
            torch.cuda.current_stream().synchronize()
            return comm.launch_count - before, [t.cpu() for t in ts]

        res = w.run(f)
        for launches, got in res:
            assert launches == 1
            assert all(torch.equal(a, b) for a, b in zip(got, payload))
    finally:
        w.destroy("bcast-multi")
