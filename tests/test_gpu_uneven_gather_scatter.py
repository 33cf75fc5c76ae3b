"""All-gather and reduce-scatter with a size per rank: b200_allgatherv and b200_reducescatterv
(B200Comm.allgatherv / reducescatterv, c10d's all_gather / reduce_scatter of uneven parts).

All-gather: every byte every rank receives is compared with what its owner sent, and the guard
bytes around every output must come back unchanged.  Reduce-scatter: every output is bit-identical
to the rank-ascending oracle, and with equal sizes to b200_reducescatter.  The launch count of
every rank is checked against the window formula, and equal sizes must make exactly the launches
of b200_allgather / b200_reducescatter.
"""
import ctypes
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from oracle import collective_oracle as O
from ray_b200 import _native as N
from tests.test_gpu_reduction_matrix import DTYPES, HALF, OPS, Operand, make_inputs, same_bits
from tests.test_uneven_gather_scatter_cpu import ag_launches, rs_launches

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GUARD = 0x5A
STAGING = 2 << 20  # the library's smallest staging slot: parts of a few MiB span several windows
WORLDS = [2, 3, 4, 8]


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


def _launches(g, fn):
    before = [c.launch_count for c in g.comms]
    g.run(fn)
    return [c.launch_count - b for c, b in zip(g.comms, before)]


def _layout(sizes, misalign):
    """Offsets of parts of `sizes` bytes in one buffer: part p starts misalign(p) bytes past a 16-byte
    boundary, with at least 32 guard bytes on both sides."""
    offs, pos = [], 32
    for p, s in enumerate(sizes):
        pos = (pos + 15) // 16 * 16 + misalign(p)
        offs.append(pos)
        pos += s + 32
    return offs, pos


# ---- all-gather ---------------------------------------------------------------------------------

def _agv(g, sizes, misalign=lambda r, p: 0, seed=0, in_place=False):
    """allgatherv of parts of `sizes` bytes (rank p sends sizes[p]): every output byte of every rank,
    the guard bytes around every output and every rank's launch count.  Output p of rank r starts
    misalign(r, p) bytes past a 16-byte boundary; the input of rank r is its own output r when
    `in_place`, else a view with its own misalignment.  Returns the launch counts."""
    n = g.world_size
    rng = np.random.default_rng(seed)
    data = [torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in sizes]
    bufs, wants, outs, ins = [], [], [], []
    for r in range(n):
        offs, total = _layout(sizes, lambda p: misalign(r, p))
        want = torch.full((total,), GUARD, dtype=torch.uint8)
        buf = want.clone()
        for p, s in enumerate(sizes):
            want[offs[p]:offs[p] + s] = data[p]
            buf[offs[p]:offs[p] + s] = data[r] if (in_place and p == r) else GUARD ^ 0xFF
        buf = buf.to(g.device(r))
        bufs.append(buf)
        wants.append(want)
        outs.append([buf[o:o + s] for o, s in zip(offs, sizes)])
        if in_place:
            ins.append(outs[r][r])
        else:
            front = 32 + misalign(r, 7 * r + 3)
            ibuf = torch.full((front + sizes[r] + 32,), GUARD, dtype=torch.uint8)
            ibuf[front:front + sizes[r]] = data[r]
            ins.append(ibuf.to(g.device(r))[front:front + sizes[r]])
    launches = _launches(g, lambda c, r: c.allgatherv(outs[r], ins[r]))
    for r in range(n):
        assert torch.equal(bufs[r].cpu(), wants[r]), f"rank {r}: payload or guard bytes differ"
    return launches


S = STAGING
AG_SIZES = {
    # name -> sizes(n): bytes of each rank's part
    "tails_1_to_15": lambda n: [100 * p + (p % 15) + 1 for p in range(n)],
    "first_empty": lambda n: [0] + [4096 + 3 * p for p in range(1, n)],
    "last_shorter": lambda n: [70_000 + p for p in range(n - 1)] + [70_000 // 3],
    "larger_than_slot": lambda n: [3 + p if p != 1 else 2 * S + S // 2 + 7 for p in range(n)],
    "skew_several_windows": lambda n: [((3 * S) >> p) + p for p in range(n)],
    "one_byte_and_slot": lambda n: [1] + [S + 16 * p for p in range(1, n)],
}


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", list(AG_SIZES))
def test_allgatherv_byte_for_byte(groups, world, name):
    sizes = AG_SIZES[name](world)
    launches = _agv(groups(world), sizes, seed=world)
    assert launches == [ag_launches(sizes, STAGING)] * world, launches


@pytest.mark.parametrize("world", [2, 3, 4])
def test_allgatherv_views_misaligned_by_1_to_15_bytes(groups, world):
    g = groups(world)
    sizes = [(S + 999) * (p % 2) + 77 * p + 5 for p in range(world)]
    _agv(g, sizes, misalign=lambda r, p: (p * (r + 3) + r) % 15 + 1, seed=10)
    # aligned on some ranks, misaligned on the others
    _agv(g, sizes, misalign=lambda r, p: 0 if r == 0 else p % 15 + 1, seed=11)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_allgatherv_in_place(groups, world):
    g = groups(world)
    _agv(g, AG_SIZES["larger_than_slot"](world), misalign=lambda r, p: (p + r) % 16, seed=20, in_place=True)
    _agv(g, AG_SIZES["first_empty"](world), seed=21, in_place=True)


@pytest.mark.parametrize("world", [2, 4])
def test_allgatherv_all_empty_launches_nothing(groups, world):
    assert _agv(groups(world), [0] * world) == [0] * world


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("part", [4097, 5 << 20])  # the staged kernel; the pull kernel (aligned, >= 4 MiB)
def test_allgatherv_equal_sizes_make_allgathers_launches(groups, world, part):
    g = groups(world)
    launches = _agv(g, [part] * world, seed=30)
    outs = [[torch.empty(part, dtype=torch.uint8, device=g.device(r)) for _ in range(world)] for r in range(world)]
    ins = [torch.zeros(part, dtype=torch.uint8, device=g.device(r)) for r in range(world)]
    assert launches == _launches(g, lambda c, r: c.allgather(outs[r], ins[r]))


# ---- reduce-scatter -----------------------------------------------------------------------------

RS_SMALL = [0, 13, 1003, 65_537, 7, 1, 4097]


def _rs_bytes(n):
    """Rank 0's part spans two windows; the others cycle through small sizes, mostly not a multiple
    of 16 bytes, and an empty one."""
    return [S // n + 999 if q == 0 else RS_SMALL[q % len(RS_SMALL)] for q in range(n)]


def _rsv(g, dname, op, byte_sizes, seed=0, in_place=False):
    """reducescatterv of one dtype over misaligned operands with guard bytes: every output against
    the rank-ascending oracle, guards, unchanged inputs and every rank's launch count.  Returns the
    outputs (numpy) and the launch counts."""
    n = g.world_size
    tdt, ndt = DTYPES[dname]
    es = ndt.itemsize
    counts = [max(b // es, 1) if b else 0 for b in byte_sizes]
    # vals[q][r]: rank r's contribution to rank q's output
    vals = [make_inputs(dname, op, n, k, seed + 31 * q) if k else [np.zeros(0, ndt)] * n
            for q, k in enumerate(counts)]
    ins = [[Operand(vals[q][r], dname, g.device(r), (q + r) % 3, seed=r * 1000 + q) for q in range(n)]
           for r in range(n)]
    outs = [ins[r][r] if in_place else Operand(np.zeros(counts[r], ndt), dname, g.device(r), (2 * r) % 3,
                                               seed=7 + r * 100) for r in range(n)]
    launches = _launches(g, lambda c, r: c.reducescatterv(outs[r].view, [x.view for x in ins[r]], op))
    got = []
    for r in range(n):
        val, guards = outs[r].read()
        assert guards, (dname, op, r, "guard bytes changed")
        if counts[r]:
            want = O.reduce_rank_ascending([vals[r][p] for p in range(n)], op,
                                           accumulate="fp32" if dname in HALF else "native")
            assert same_bits(val, want), (dname, op, r, "differs from the oracle")
        for q in range(n):
            if not (in_place and q == r):
                assert ins[r][q].unchanged(), (dname, op, r, q, "input changed")
        got.append(val.copy())
    return got, launches, counts


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("dname", list(DTYPES))
def test_reducescatterv_against_oracle(groups, dname, op, world):
    g = groups(world)
    _, launches, counts = _rsv(g, dname, OPS[op], _rs_bytes(world), seed=world)
    es = DTYPES[dname][1].itemsize
    assert launches == [rs_launches([k * es for k in counts], STAGING)] * world, launches


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("dname,op", [("float32", "SUM"), ("bfloat16", "AVG"), ("int64", "MAX")])
def test_reducescatterv_several_windows(groups, dname, op, world):
    g = groups(world)
    sizes = [3 * S // world + 5, 0] + [S // world + 16 * q + 3 for q in range(2, world)]
    sizes = sizes[::-1]  # the largest part on the last rank
    _, launches, counts = _rsv(g, dname, OPS[op], sizes, seed=50)
    es = DTYPES[dname][1].itemsize
    assert launches == [rs_launches([k * es for k in counts], STAGING)] * world
    assert launches[0] >= 3


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("dname", ["uint8", "bfloat16", "float32", "float64"])
def test_reducescatterv_in_place(groups, dname, world):
    _rsv(groups(world), dname, O.SUM, _rs_bytes(world), seed=40, in_place=True)
    _rsv(groups(world), dname, O.AVG, [S // world + 7 * q for q in range(world)], seed=41, in_place=True)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("dname,op", [("float32", "SUM"), ("float16", "AVG"), ("int32", "PROD"), ("uint8", "MIN")])
def test_reducescatterv_equal_sizes_match_reducescatter(groups, dname, op, world):
    """Equal counts: bit-identical to b200_reducescatter on the same inputs, with its launches."""
    g = groups(world)
    nbytes = S // world + 1003  # two windows
    _, launches, counts = _rsv(g, dname, OPS[op], [nbytes] * world, seed=60)
    tdt, ndt = DTYPES[dname]
    k = counts[0]
    ins = [[torch.from_numpy(x).to(g.device(r)) for x in make_inputs(dname, OPS[op], world, k, 60 + r)]
           for r in range(world)]
    outs_v = [torch.empty(k, dtype=tdt, device=g.device(r)) for r in range(world)]
    outs = [torch.empty(k, dtype=tdt, device=g.device(r)) for r in range(world)]
    lv = _launches(g, lambda c, r: c.reducescatterv(outs_v[r], ins[r], OPS[op]))
    le = _launches(g, lambda c, r: c.reducescatter(outs[r], ins[r], OPS[op]))
    assert launches == lv == le, (launches, lv, le)
    for r in range(world):
        assert same_bits(outs_v[r].cpu().view(torch.uint8).numpy().view(ndt),
                         outs[r].cpu().view(torch.uint8).numpy().view(ndt)), r


# ---- ordering, graphs, refusals, world 1 --------------------------------------------------------

@pytest.mark.parametrize("world", [2, 4])
def test_interleaves_with_other_collectives_on_two_streams(groups, world):
    """allreduce, allgatherv, broadcast, reducescatterv, allgather and send / recv, alternating between
    two streams of every rank: every result is right and the status stays 0."""
    g = groups(world)
    side = [torch.cuda.Stream(device=d) for d in g.devices]
    rng = np.random.default_rng(12)
    ag_sizes = [(S + 5) if p == 0 else 3 * p for p in range(world)]
    ag_data = [torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in ag_sizes]
    rs_counts = [1, 300_000] + [999 * q for q in range(2, world)]
    rs_host = [[rng.integers(-100, 100, k).astype(np.float32) for k in rs_counts] for _ in range(world)]
    bc = torch.from_numpy(rng.standard_normal(600_000).astype(np.float32))
    p2p = torch.from_numpy(rng.standard_normal(12345).astype(np.float32))
    for rep in range(2):
        xs = [torch.full((5000,), float(r + 1), device=g.device(r)) for r in range(world)]
        ag_in = [ag_data[r].to(g.device(r)) for r in range(world)]
        ag_out = [[torch.empty(s, dtype=torch.uint8, device=g.device(r)) for s in ag_sizes] for r in range(world)]
        even_out = [[torch.empty(7, device=g.device(r)) for _ in range(world)] for r in range(world)]
        bl = [bc.to(g.device(r)) if r == rep else torch.zeros_like(bc, device=g.device(r)) for r in range(world)]
        rs_in = [[torch.from_numpy(h).to(g.device(r)) for h in rs_host[r]] for r in range(world)]
        rs_out = [torch.empty(rs_counts[r], device=g.device(r)) for r in range(world)]
        rx = torch.zeros_like(p2p, device=g.device(1))
        tx = p2p.to(g.device(0))

        def f(c, r):
            c.allreduce(xs[r], N.SUM)
            with torch.cuda.stream(side[r]):
                c.allgatherv(ag_out[r], ag_in[r])
            c.broadcast(bl[r], rep)
            with torch.cuda.stream(side[r]):
                c.reducescatterv(rs_out[r], rs_in[r], N.SUM)
            c.allgather(even_out[r], torch.full((7,), float(r), device=g.device(r)))
            if r == 0:
                c.send(tx, 1)
            elif r == 1:
                c.recv(rx, 0)

        g.run(f)
        for s in side:
            s.synchronize()
        g.synchronize()
        for r in range(world):
            assert torch.all(xs[r].cpu() == world * (world + 1) / 2)
            assert all(torch.equal(ag_out[r][p].cpu(), ag_data[p]) for p in range(world)), r
            assert torch.equal(bl[r].cpu(), bc)
            assert np.array_equal(rs_out[r].cpu().numpy(), sum(rs_host[p][r] for p in range(world))), r
            assert all(torch.all(even_out[r][p].cpu() == p) for p in range(world))
            assert g.comms[r].status() == 0
        assert torch.equal(rx.cpu(), p2p)


def test_cuda_graph_replay(groups):
    """One capture of an allgatherv plus a reducescatterv per rank, replayed twice with new inputs in
    between."""
    n = 3
    g = groups(n)
    ag_sizes = [3, (2 * S) + 5, 0]
    rs_counts = [7001, 0, S // 4]  # float32: the last part spans two windows
    ag_in = [torch.zeros(ag_sizes[r], dtype=torch.uint8, device=g.device(r)) for r in range(n)]
    ag_out = [[torch.zeros(s, dtype=torch.uint8, device=g.device(r)) for s in ag_sizes] for r in range(n)]
    rs_in = [[torch.zeros(k, dtype=torch.float32, device=g.device(r)) for k in rs_counts] for r in range(n)]
    rs_out = [torch.zeros(rs_counts[r], dtype=torch.float32, device=g.device(r)) for r in range(n)]

    def f(c, r):
        c.allgatherv(ag_out[r], ag_in[r])
        c.reducescatterv(rs_out[r], rs_in[r], N.MAX)

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
        fresh_ag = [torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in ag_sizes]
        fresh_rs = [[torch.from_numpy(rng.standard_normal(k).astype(np.float32)) for k in rs_counts]
                    for _ in range(n)]
        for r in range(n):
            ag_in[r].copy_(fresh_ag[r])
            for t, d in zip(rs_in[r], fresh_rs[r]):
                t.copy_(d)
        for d in set(g.devices):
            torch.cuda.synchronize(d)
        for r in range(n):
            torch.cuda.set_device(g.devices[r])
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        g.synchronize()
        for r in range(n):
            assert all(torch.equal(ag_out[r][p].cpu(), fresh_ag[p]) for p in range(n)), (rep, r)
            want = O.reduce_rank_ascending([fresh_rs[p][r].numpy() for p in range(n)], O.MAX)
            assert same_bits(rs_out[r].cpu().numpy(), want), (rep, r)


def _arr(ctype, vals):
    return (ctype * max(len(vals), 1))(*vals)


def test_refused_calls_launch_nothing(groups):
    g = groups(2)
    lib, c = N.load(), g.comms[0]
    h, dev = c._h, g.device(0)
    x = torch.zeros(256, dtype=torch.uint8, device=dev)
    p = x.data_ptr()
    PTRS = _arr(ctypes.c_void_p, [p, p + 64])
    C = _arr(ctypes.c_size_t, [4, 2])  # rank 0's part: 4 elements
    ag, rs = lib.b200_allgatherv, lib.b200_reducescatterv
    F32 = N.F32
    cases = [
        ("ag null count array", lambda: ag(h, p, None, PTRS, F32, None), N.ERR_INVALID, "null argument array"),
        ("ag null output array", lambda: ag(h, p, C, None, F32, None), N.ERR_INVALID, "null argument array"),
        ("ag null output", lambda: ag(h, p, C, _arr(ctypes.c_void_p, [p, None]), F32, None), N.ERR_INVALID,
         "tensor 1 is null but has 8 bytes"),
        ("ag null input", lambda: ag(h, None, C, PTRS, F32, None), N.ERR_INVALID, "null tensor pointer"),
        ("ag bad dtype", lambda: ag(h, p, C, PTRS, 99, None), N.ERR_UNSUPPORTED, "unsupported dtype 99"),
        ("rs null input array", lambda: rs(h, None, C, p, F32, N.SUM, None), N.ERR_INVALID, "null argument array"),
        ("rs null count array", lambda: rs(h, PTRS, None, p, F32, N.SUM, None), N.ERR_INVALID,
         "null argument array"),
        ("rs null input", lambda: rs(h, _arr(ctypes.c_void_p, [None, p]), C, p, F32, N.SUM, None), N.ERR_INVALID,
         "tensor 0 is null but has 16 bytes"),
        ("rs null output", lambda: rs(h, PTRS, C, None, F32, N.SUM, None), N.ERR_INVALID, "null tensor pointer"),
        ("rs bad dtype", lambda: rs(h, PTRS, C, p, 99, N.SUM, None), N.ERR_UNSUPPORTED, "unsupported dtype 99"),
        ("rs bad op", lambda: rs(h, PTRS, C, p, F32, 7, None), N.ERR_UNSUPPORTED, "unsupported reduce op 7"),
    ]
    before = c.launch_count
    with torch.cuda.device(dev):
        for name, call, status, text in cases:
            assert call() == status, name
            assert text in N.last_error(), (name, N.last_error())
        # allowed: NULL pointers of zero counts; all counts zero launches nothing
        Z = _arr(ctypes.c_size_t, [0, 0])
        nulls = _arr(ctypes.c_void_p, [None, None])
        assert ag(h, None, Z, nulls, F32, None) == N.OK
        assert rs(h, nulls, Z, None, F32, N.AVG, None) == N.OK
    torch.cuda.synchronize(dev)
    assert c.launch_count == before
    assert c.status() == 0


def test_world_one_copies_without_launching(native_lib):
    from ray_b200.testing import LocalGroup

    with LocalGroup(1, staging_bytes=STAGING) as g:
        c, dev = g.comms[0], g.device(0)
        a = torch.arange(1000, dtype=torch.float32, device=dev)
        oa = torch.zeros_like(a)
        before = c.launch_count
        g.run(lambda c, r: c.allgatherv([oa], a))
        assert torch.equal(oa, a)
        g.run(lambda c, r: c.allgatherv([a], a))  # in place
        x, ox = torch.randn(513, device=dev), torch.zeros(513, device=dev)
        g.run(lambda c, r: c.reducescatterv(ox, [x], N.AVG))  # AVG over one rank: the identity
        assert torch.equal(ox, x)
        assert c.launch_count == before


# ---- c10d in worker processes -------------------------------------------------------------------

def _c10d_worker(rank, world, init_file, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist

    from ray_b200 import train as T

    ndev = torch.cuda.device_count()
    os.environ["LOCAL_RANK"] = str(rank if ndev >= world else 0)
    device = T.get_device()
    torch.cuda.set_device(device)
    T.setup_torch_process_group("cpu:gloo,cuda:b200", rank, world, f"file://{init_file}", timeout_s=120)
    pg = dist.distributed_c10d._get_default_group()
    assert isinstance(pg, T.B200ProcessGroup)
    x = torch.zeros(1, device=device)
    dist.all_reduce(x)
    if ndev < world:
        pg.comm.set_blocks(32)  # co-resident grids when the workers share one GPU
    staging = 256 << 20  # the default staging slot

    def launches(fn):
        torch.cuda.synchronize()
        before = pg.comm.launch_count
        fn()
        torch.cuda.synchronize()
        return pg.comm.launch_count - before

    # all_gather of variable-length results: the last rank holds the remainder, rank 1 nothing
    lengths = [1000 + 3 * p for p in range(world - 1)] + [377]
    lengths[1] = 0
    for dt in (torch.int64, torch.float32):
        mine = (torch.arange(lengths[rank], device=device) * (rank + 1)).to(dt)
        outs = [torch.full((k,), -1, dtype=dt, device=device) for k in lengths]
        n = launches(lambda: dist.all_gather(outs, mine))
        assert n == ag_launches([k * outs[0].element_size() for k in lengths], staging), n
        for p, k in enumerate(lengths):
            assert torch.equal(outs[p], (torch.arange(k, device=device) * (p + 1)).to(dt)), (dt, p)
    # non-contiguous outputs receive through temporaries
    strided = [torch.zeros(2 * k, device=device)[::2] for k in lengths]
    dist.all_gather(strided, torch.full((lengths[rank],), float(rank), device=device))
    assert all(torch.all(strided[p] == p) for p in range(world))

    # reduce_scatter onto uneven shards: SUM of int64, AVG and SUM of float32
    shards = [5000 + 7 * q for q in range(world - 1)] + [1234]
    out_i = torch.empty(shards[rank], dtype=torch.int64, device=device)
    ins_i = [torch.arange(k, device=device) + 1000 * rank + q for q, k in enumerate(shards)]
    n = launches(lambda: dist.reduce_scatter(out_i, ins_i))
    assert n == rs_launches([k * 8 for k in shards], staging), n
    assert torch.equal(out_i, sum(torch.arange(shards[rank], device=device) + 1000 * p + rank for p in range(world)))
    out_f = torch.empty(shards[rank], device=device)
    ins_f = [torch.full((k,), float(world * (rank + 1)), device=device) for k in shards]
    dist.reduce_scatter(out_f, ins_f, op=dist.ReduceOp.AVG)
    assert torch.all(out_f == world * (world + 1) / 2)
    dist.reduce_scatter(out_f, ins_f, op=dist.ReduceOp.SUM)
    assert torch.all(out_f == world * world * (world + 1) / 2)

    # equal sizes keep today's launches: one staged all-gather / reduce-scatter each
    eq = [torch.empty(4, device=device) for _ in range(world)]
    assert launches(lambda: dist.all_gather(eq, torch.full((4,), float(rank), device=device))) == 1
    assert all(torch.all(eq[p] == p) for p in range(world))
    rs_out = torch.empty(6, device=device)
    assert launches(lambda: dist.reduce_scatter(rs_out, [torch.full((6,), float(q + rank), device=device)
                                                         for q in range(world)])) == 1
    assert torch.all(rs_out == sum(rank + p for p in range(world)))

    torch.cuda.synchronize()
    pg.comm.check_status()
    dist.barrier()
    dist.destroy_process_group()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as f:
        f.write("ok")


@pytest.mark.parametrize("world", [2, 3])
def test_c10d_uneven_all_gather_and_reduce_scatter(native_lib, world):
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_c10d_worker, args=(world, os.path.join(d, "rdzv"), d), nprocs=world, join=True)
        assert all(os.path.exists(os.path.join(d, f"ok{r}")) for r in range(world))
