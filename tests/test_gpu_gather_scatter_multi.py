"""Tensor-list all-gather and reduce-scatter in one launch per window: b200_allgather_multi and
b200_reducescatter_multi (B200Comm.allgather_multi / allgather_into_multi / reducescatter_multi /
reducescatter_from_multi, the c10d coalesced collectives, ray_b200.collective).

All-gather: every byte every rank receives is compared with what its peers sent, and the guard
bytes around every output must come back unchanged (the padding of a tensor's last 16-byte unit
goes through the staging slot but is never stored).  Reduce-scatter: every output is bit-identical
to a per-tensor b200_reducescatter of the same inputs and to the rank-ascending oracle.  The launch
count of every call is checked against the plan.
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

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE = N.P2P_TABLE_MAX
GUARD = 0x5A
STAGING = 2 << 20  # the library's smallest staging slot: lists of a few MiB span several windows
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


def _planned(sizes, window_units):
    launches = 0
    nonempty = [s for s in sizes if s]
    for i in range(0, len(nonempty), TABLE):
        units = sum(-(-s // 16) for s in nonempty[i:i + TABLE])
        launches += -(-units // window_units)
    return launches


def ag_planned(sizes, staging=STAGING):
    """Sum over tables of ceil(16 * units / staging_bytes)."""
    return _planned(sizes, staging // 16)


def rs_planned(sizes, world, staging=STAGING):
    """Sum over tables of ceil(units / floor(staging_bytes / (16 * world)))."""
    return _planned(sizes, staging // (16 * world))


def test_plan_formulas():
    assert ag_planned([]) == 0 and ag_planned([0, 0]) == 0 and ag_planned([STAGING + 1]) == 2
    assert ag_planned([16 + i for i in range(TABLE + 1)]) == 2
    assert rs_planned([STAGING // 2], 2) == 1 and rs_planned([STAGING // 2 + 1], 2) == 2
    assert rs_planned([STAGING], 8) == 8 and rs_planned([1] * (TABLE + 1), 8) == 2


def _layout(sizes, misalign):
    """Offsets of tensors of `sizes` bytes in one buffer: tensor i starts misalign(i) bytes past a
    16-byte boundary, with at least 32 guard bytes on both sides."""
    offs, pos = [], 32
    for i, s in enumerate(sizes):
        pos = (pos + 15) // 16 * 16 + misalign(i)
        offs.append(pos)
        pos += s + 32
    return offs, pos


LISTS = {
    "one": [100_000],
    "bytes_1_to_15": list(range(1, 16)),
    "zeros_scattered": [0, 100, 0, 0, 4096, 0, 17, 33, 0],
    "tiny": [1, 2, 3, 4097, 5],
    "several_windows": [(1 << 20) + 16 * i + (i % 3) for i in range(5)],
    "larger_than_slot": [3, (5 << 20) + 7, 11],
    "table_max_plus_one": [16 + (i % 37) for i in range(TABLE + 1)],
    "tables_spanning_slots": [9000 + i for i in range(2 * TABLE + 10)],
}


# ---- all-gather ---------------------------------------------------------------------------------

def _ag(g, sizes, misalign=lambda r, j: 0, seed=0, in_place=False):
    """allgather_multi of a list of `sizes` bytes: every output byte of every rank, the guard bytes
    around every output, and the launch count of every rank.  Output j = i * n + p of rank r starts
    misalign(r, j) bytes past a 16-byte boundary; the input of rank r is its own output i * n + r
    when `in_place`, else a view with its own misalignment."""
    n = g.world_size
    rng = np.random.default_rng(seed)
    data = [[torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in sizes] for _ in range(n)]
    flat_sizes = [s for s in sizes for _ in range(n)]
    bufs, wants, out_lists, ins = [], [], [], []
    for r in range(n):
        offs, total = _layout(flat_sizes, lambda j: misalign(r, j))
        want = torch.full((total,), GUARD, dtype=torch.uint8)
        buf = want.clone()
        for i, s in enumerate(sizes):
            for p in range(n):
                o = offs[i * n + p]
                want[o:o + s] = data[p][i]
                buf[o:o + s] = data[r][i] if (in_place and p == r) else GUARD ^ 0xFF
        buf = buf.to(g.device(r))
        bufs.append(buf)
        wants.append(want)
        out_lists.append([[buf[offs[i * n + p]:offs[i * n + p] + s] for p in range(n)] for i, s in enumerate(sizes)])
        if in_place:
            ins.append([out_lists[r][i][r] for i in range(len(sizes))])
        else:
            ioffs, itotal = _layout(sizes, lambda i: misalign(r, i * 7 + 3))
            ibuf = torch.full((itotal,), GUARD, dtype=torch.uint8)
            for o, s, d in zip(ioffs, sizes, data[r]):
                ibuf[o:o + s] = d
            ibuf = ibuf.to(g.device(r))
            ins.append([ibuf[o:o + s] for o, s in zip(ioffs, sizes)])
    before = [c.launch_count for c in g.comms]
    g.run(lambda c, r: c.allgather_multi(out_lists[r], ins[r]))
    launches = [c.launch_count - b for c, b in zip(g.comms, before)]
    assert launches == [ag_planned(sizes) if n > 1 else 0] * n, launches
    for r in range(n):
        assert torch.equal(bufs[r].cpu(), wants[r]), f"rank {r}: payload or guard bytes differ"


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", list(LISTS))
def test_allgather_lists_byte_for_byte(groups, world, name):
    _ag(groups(world), LISTS[name], seed=world)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_allgather_views_misaligned_by_1_to_15_bytes(groups, world):
    g = groups(world)
    sizes = [(i * 977) % 5000 + 1 for i in range(40)] + [300_000, 70_001, (2 << 20) + 9]
    _ag(g, sizes, misalign=lambda r, j: (j * (r + 3) + r) % 15 + 1, seed=10)
    # aligned on some ranks, misaligned on the others
    _ag(g, sizes, misalign=lambda r, j: 0 if r == 0 else j % 15 + 1, seed=11)


@pytest.mark.parametrize("world", [2, 3])
def test_allgather_in_place(groups, world):
    g = groups(world)
    _ag(g, LISTS["tiny"] + LISTS["several_windows"], misalign=lambda r, j: (j + r) % 16, seed=20, in_place=True)
    _ag(g, LISTS["table_max_plus_one"], seed=21, in_place=True)


@pytest.mark.parametrize("world", [2, 4])
def test_allgather_into_multi_mixed_dtypes(groups, world):
    """The all_gather_into_tensor layout (rank-major outputs) with one list of several dtypes."""
    g = groups(world)
    rng = np.random.default_rng(3)
    sent = [[torch.from_numpy(rng.standard_normal((17, 3)).astype(np.float32)),
             torch.arange(-50, 77, dtype=torch.int64) * (r + 1),
             torch.from_numpy(rng.standard_normal(2049)).to(torch.bfloat16), torch.zeros(0, dtype=torch.float64),
             torch.from_numpy(rng.random(13) < 0.5)] for r in range(world)]
    ins = [[t.to(g.device(r)) for t in sent[r]] for r in range(world)]
    outs = [[torch.empty((world * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=g.device(r))
             for t in sent[r]] for r in range(world)]
    g.run(lambda c, r: c.allgather_into_multi(outs[r], ins[r]))
    for r in range(world):
        for i, o in enumerate(outs[r]):
            assert torch.equal(o.cpu(), torch.cat([sent[p][i] for p in range(world)])), (r, i)


# ---- reduce-scatter -----------------------------------------------------------------------------

RS_BYTES = [1, 7, 0, 13, 1003, 65_537, (1 << 20) + 27]  # most byte sizes not a multiple of 16


def _rs(g, dname, op, byte_sizes, seed=0, in_place=False):
    """reducescatter_multi of one dtype over padded, misaligned operands: outputs bit-identical to a
    per-tensor reducescatter of the same inputs and to the oracle; guards, launch count."""
    n = g.world_size
    tdt, ndt = DTYPES[dname]
    es = ndt.itemsize
    counts = [max(b // es, 1) if b else 0 for b in byte_sizes]
    # vals[i][r * n + q]: rank r's contribution to rank q's output i
    vals = [make_inputs(dname, op, n * n, k, seed + 31 * i) if k else [np.zeros(0, ndt)] * (n * n)
            for i, k in enumerate(counts)]
    ins = [[[Operand(vals[i][r * n + q], dname, g.device(r), (i + q + r) % 3, seed=r * 1000 + i * 10 + q)
             for q in range(n)] for i in range(len(counts))] for r in range(n)]
    if in_place:
        outs = [[ins[r][i][r] for i in range(len(counts))] for r in range(n)]
    else:
        outs = [[Operand(np.zeros(k, ndt), dname, g.device(r), (i + 2 * r) % 3, seed=7 + r * 100 + i)
                 for i, k in enumerate(counts)] for r in range(n)]
    refs = [[torch.empty(k, dtype=tdt, device=g.device(r)) for k in counts] for r in range(n)]
    # the per-tensor reference first: in place, the list call overwrites this rank's own input
    g.run(lambda c, r: [c.reducescatter(refs[r][i], [ins[r][i][q].view for q in range(n)], op)
                        for i, k in enumerate(counts) if k])
    before = [c.launch_count for c in g.comms]
    g.run(lambda c, r: c.reducescatter_multi([o.view for o in outs[r]],
                                             [[x.view for x in ins[r][i]] for i in range(len(counts))], op))
    launches = [c.launch_count - b for c, b in zip(g.comms, before)]
    assert launches == [rs_planned([k * es for k in counts], n)] * n, launches
    for r in range(n):
        for i, k in enumerate(counts):
            got, guards = outs[r][i].read()
            assert guards, (dname, op, r, i, "guard bytes changed")
            assert same_bits(got, refs[r][i].cpu().view(torch.uint8).numpy().view(ndt)), \
                (dname, op, r, i, "differs from per-tensor reducescatter")
            want = O.reduce_rank_ascending([vals[i][p * n + r] for p in range(n)], op,
                                           accumulate="fp32" if dname in HALF else "native")
            assert same_bits(got, want), (dname, op, r, i, "differs from the oracle")
            if not in_place:
                for q in range(n):
                    assert ins[r][i][q].unchanged(), (dname, op, r, i, q, "input changed")


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("dname", list(DTYPES))
def test_reducescatter_against_oracle(groups, dname, op, world):
    _rs(groups(world), dname, OPS[op], RS_BYTES, seed=world)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("dname", ["uint8", "bfloat16", "float32", "float64"])
def test_reducescatter_in_place(groups, dname, world):
    _rs(groups(world), dname, O.SUM, RS_BYTES, seed=40, in_place=True)
    _rs(groups(world), dname, O.AVG, [40 + (i % 7) for i in range(TABLE + 3)], seed=41, in_place=True)


@pytest.mark.parametrize("world", [2, 4])
def test_reducescatter_from_multi(groups, world):
    """The reduce_scatter_tensor layout: rank-major inputs, one output per tensor."""
    g = groups(world)
    counts = [3, 1000, 0, 70_001]
    rng = np.random.default_rng(8)
    host = [[rng.standard_normal(world * k).astype(np.float32) for k in counts] for _ in range(world)]
    ins = [[torch.from_numpy(h).to(g.device(r)) for h in host[r]] for r in range(world)]
    outs = [[torch.empty(k, device=g.device(r)) for k in counts] for r in range(world)]
    g.run(lambda c, r: c.reducescatter_from_multi(outs[r], ins[r], N.SUM))
    for r in range(world):
        for i, k in enumerate(counts):
            want = O.reduce_rank_ascending([host[p][i][r * k:(r + 1) * k] for p in range(world)], O.SUM)
            assert same_bits(outs[r][i].cpu().numpy(), want), (r, i)


# ---- ordering, graphs, refusals, world 1 --------------------------------------------------------

@pytest.mark.parametrize("world", [2, 4])
def test_interleaves_with_other_collectives_on_two_streams(groups, world):
    """allreduce, allgather_multi, broadcast_multi, reducescatter_multi, send / recv, alternating
    between two streams of every rank: every result is right and the status stays 0."""
    g = groups(world)
    side = [torch.cuda.Stream(device=d) for d in g.devices]
    rng = np.random.default_rng(12)
    ag_sizes = [5, 70_000, 0, 3 << 20, 3]
    ag_data = [[torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in ag_sizes] for _ in range(world)]
    bc = [torch.from_numpy(rng.standard_normal(s).astype(np.float32)) for s in (1, 1000, 600_000)]
    rs_counts = [1, 999, 300_000]
    rs_host = [[[rng.integers(-100, 100, k).astype(np.float32) for _ in range(world)] for k in rs_counts]
               for _ in range(world)]
    p2p = torch.from_numpy(rng.standard_normal(12345).astype(np.float32))
    for rep in range(2):
        xs = [torch.full((5000,), float(r + 1), device=g.device(r)) for r in range(world)]
        ag_in = [[t.to(g.device(r)) for t in ag_data[r]] for r in range(world)]
        ag_out = [[[torch.empty_like(t, device=g.device(r)) for _ in range(world)] for t in ag_data[r]]
                  for r in range(world)]
        bl = [[t.to(g.device(r)) if r == rep else torch.zeros_like(t, device=g.device(r)) for t in bc]
              for r in range(world)]
        rs_in = [[[torch.from_numpy(h).to(g.device(r)) for h in lst] for lst in rs_host[r]] for r in range(world)]
        rs_out = [[torch.empty(k, device=g.device(r)) for k in rs_counts] for r in range(world)]
        rx = torch.zeros_like(p2p, device=g.device(1))
        tx = p2p.to(g.device(0))

        def f(c, r):
            c.allreduce(xs[r], N.SUM)
            with torch.cuda.stream(side[r]):
                c.allgather_multi(ag_out[r], ag_in[r])
            c.broadcast_multi(bl[r], rep)
            with torch.cuda.stream(side[r]):
                c.reducescatter_multi(rs_out[r], rs_in[r], N.SUM)
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
            for i, t in enumerate(ag_data[r]):
                assert all(torch.equal(ag_out[r][i][p].cpu(), ag_data[p][i]) for p in range(world)), (r, i)
            assert all(torch.equal(t.cpu(), b) for t, b in zip(bl[r], bc))
            for i in range(len(rs_counts)):
                want = sum(rs_host[p][i][r] for p in range(world))
                assert np.array_equal(rs_out[r][i].cpu().numpy(), want), (r, i)
            assert g.comms[r].status() == 0
        assert torch.equal(rx.cpu(), p2p)


def test_cuda_graph_replay(groups):
    """One capture of a list all-gather plus a list reduce-scatter per rank, replayed twice with
    new inputs in between."""
    n = 3
    g = groups(n)
    ag_sizes = [3, 4096, 100_001, (2 << 20) + 5] + [40 + i for i in range(TABLE)]
    rs_counts = [5, 7001, 400_000]
    ag_in = [[torch.zeros(s, dtype=torch.uint8, device=g.device(r)) for s in ag_sizes] for r in range(n)]
    ag_out = [[[torch.zeros(s, dtype=torch.uint8, device=g.device(r)) for _ in range(n)] for s in ag_sizes]
              for r in range(n)]
    rs_in = [[[torch.zeros(k, dtype=torch.float32, device=g.device(r)) for _ in range(n)] for k in rs_counts]
             for r in range(n)]
    rs_out = [[torch.zeros(k, dtype=torch.float32, device=g.device(r)) for k in rs_counts] for r in range(n)]

    def f(c, r):
        c.allgather_multi(ag_out[r], ag_in[r])
        c.reducescatter_multi(rs_out[r], rs_in[r], N.MAX)

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
        fresh_ag = [[torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in ag_sizes] for _ in range(n)]
        fresh_rs = [[[torch.from_numpy(rng.standard_normal(k).astype(np.float32)) for _ in range(n)]
                     for k in rs_counts] for _ in range(n)]
        for r in range(n):
            for t, d in zip(ag_in[r], fresh_ag[r]):
                t.copy_(d)
            for lst, dl in zip(rs_in[r], fresh_rs[r]):
                for t, d in zip(lst, dl):
                    t.copy_(d)
        for d in set(g.devices):
            torch.cuda.synchronize(d)
        for r in range(n):
            torch.cuda.set_device(g.devices[r])
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        g.synchronize()
        for r in range(n):
            for i in range(len(ag_sizes)):
                assert all(torch.equal(ag_out[r][i][p].cpu(), fresh_ag[p][i]) for p in range(n)), (rep, r, i)
            for i in range(len(rs_counts)):
                want = O.reduce_rank_ascending([fresh_rs[p][i][r].numpy() for p in range(n)], O.MAX)
                assert same_bits(rs_out[r][i].cpu().numpy(), want), (rep, r, i)


def _arr(ctype, vals):
    return (ctype * max(len(vals), 1))(*vals)


def test_refused_calls_launch_nothing(groups):
    g = groups(2)
    lib, c = N.load(), g.comms[0]
    h, dev = c._h, g.device(0)
    x = torch.zeros(256, dtype=torch.uint8, device=dev)
    p = x.data_ptr()
    IN = _arr(ctypes.c_void_p, [p, p + 16])
    OUT = _arr(ctypes.c_void_p, [p + 64, p + 80, p + 96, p + 112])
    S = _arr(ctypes.c_size_t, [16, 16])
    ag, rs = lib.b200_allgather_multi, lib.b200_reducescatter_multi
    F32 = N.F32
    cases = [
        ("ag negative count", lambda: ag(h, IN, S, -1, OUT, None), N.ERR_INVALID, "ntensors -1 is negative"),
        ("ag null input array", lambda: ag(h, None, S, 2, OUT, None), N.ERR_INVALID, "null argument array"),
        ("ag null size array", lambda: ag(h, IN, None, 2, OUT, None), N.ERR_INVALID, "null argument array"),
        ("ag null output array", lambda: ag(h, IN, S, 2, None, None), N.ERR_INVALID, "null argument array"),
        ("ag null input", lambda: ag(h, _arr(ctypes.c_void_p, [p, None]), S, 2, OUT, None), N.ERR_INVALID,
         "tensor 1 is null but has 16 bytes"),
        ("ag null output", lambda: ag(h, IN, S, 2, _arr(ctypes.c_void_p, [p + 64, p + 80, p + 96, None]), None),
         N.ERR_INVALID, "output 1 of tensor 1 is null but has 16 bytes"),
        ("rs negative count", lambda: rs(h, OUT, IN, S, -1, F32, N.SUM, None), N.ERR_INVALID,
         "ntensors -1 is negative"),
        ("rs null input array", lambda: rs(h, None, IN, S, 2, F32, N.SUM, None), N.ERR_INVALID,
         "null argument array"),
        ("rs null output array", lambda: rs(h, OUT, None, S, 2, F32, N.SUM, None), N.ERR_INVALID,
         "null argument array"),
        ("rs null count array", lambda: rs(h, OUT, IN, None, 2, F32, N.SUM, None), N.ERR_INVALID,
         "null argument array"),
        ("rs null output", lambda: rs(h, OUT, _arr(ctypes.c_void_p, [None, p]), S, 2, F32, N.SUM, None),
         N.ERR_INVALID, "tensor 0 is null but has 64 bytes"),
        ("rs null input", lambda: rs(h, _arr(ctypes.c_void_p, [p, None, p, p]), IN, S, 2, F32, N.SUM, None),
         N.ERR_INVALID, "input 1 of tensor 0 is null but has 64 bytes"),
        ("rs bad dtype", lambda: rs(h, OUT, IN, S, 2, 99, N.SUM, None), N.ERR_UNSUPPORTED, "unsupported dtype 99"),
        ("rs bad op", lambda: rs(h, OUT, IN, S, 2, F32, 7, None), N.ERR_UNSUPPORTED, "unsupported reduce op 7"),
    ]
    before = c.launch_count
    with torch.cuda.device(dev):
        for name, call, status, text in cases:
            assert call() == status, name
            assert text in N.last_error(), (name, N.last_error())
        # allowed: no arrays with no tensors, and NULL pointers of empty entries
        assert ag(h, None, None, 0, None, None) == N.OK
        assert rs(h, None, None, None, 0, F32, N.SUM, None) == N.OK
        Z = _arr(ctypes.c_size_t, [0, 0])
        nulls = _arr(ctypes.c_void_p, [None] * 4)
        assert ag(h, nulls, Z, 2, nulls, None) == N.OK
        assert rs(h, nulls, nulls, Z, 2, F32, N.SUM, None) == N.OK
    torch.cuda.synchronize(dev)
    assert c.launch_count == before
    assert c.status() == 0


def test_world_one_copies_without_launching(native_lib):
    from ray_b200.testing import LocalGroup

    with LocalGroup(1, staging_bytes=STAGING) as g:
        c, dev = g.comms[0], g.device(0)
        a = torch.arange(1000, dtype=torch.float32, device=dev)
        b = torch.arange(77, dtype=torch.int64, device=dev)
        oa, ob = torch.zeros_like(a), torch.zeros_like(b)
        before = c.launch_count
        g.run(lambda c, r: c.allgather_multi([[oa], [b]], [a, b]))  # b in place
        assert torch.equal(oa, a) and torch.equal(b.cpu(), torch.arange(77))
        x = torch.randn(513, device=dev)
        y = torch.randn(9, device=dev)
        ox = torch.zeros_like(x)
        g.run(lambda c, r: c.reducescatter_multi([ox, y], [[x], [y]], N.AVG))  # AVG over one rank: identity
        assert torch.equal(ox, x)
        g.run(lambda c, r: c.reducescatter_from_multi([ox], [x * 2], N.SUM))
        assert torch.equal(ox, x * 2)
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

    def launches(fn):
        torch.cuda.synchronize()
        before = pg.comm.launch_count
        fn()
        torch.cuda.synchronize()
        return pg.comm.launch_count - before

    def val(k, dtype, p, i):
        return (torch.arange(k, device=device) * (p + 1) + 10 * i).to(dtype)

    # k all_gather_into_tensor calls in a coalescing block, the last two in place
    shapes = [(5, torch.float32), (1000, torch.bfloat16), (3, torch.int64), (70_001, torch.float32),
              (17, torch.float16), (2049, torch.float32)]
    k = len(shapes)
    ag_outs = [torch.full((world * n,), -1, dtype=dt, device=device) for n, dt in shapes]
    ag_ins = [val(n, dt, rank, i) for i, (n, dt) in enumerate(shapes[:-2])]
    ag_ins += [ag_outs[i][rank * n:(rank + 1) * n] for i, (n, _) in enumerate(shapes) if i >= k - 2]
    for i in range(k - 2, k):
        ag_ins[i].copy_(val(shapes[i][0], shapes[i][1], rank, i))

    def coalesced_ag():
        with dist._coalescing_manager(group=pg):
            for o, t in zip(ag_outs, ag_ins):
                dist.all_gather_into_tensor(o, t, group=pg)

    assert launches(coalesced_ag) == 1
    for i, (n, dt) in enumerate(shapes):
        assert torch.equal(ag_outs[i], torch.cat([val(n, dt, p, i) for p in range(world)])), i

    # k reduce_scatter_tensor calls in a coalescing block: two dtypes, the last one in place
    rs_shapes = [(5, torch.float32), (1000, torch.int64), (70_001, torch.float32), (3, torch.int64)]
    rs_ins = [val(world * n, dt, rank, i) for i, (n, dt) in enumerate(rs_shapes)]
    rs_outs = [torch.empty(n, dtype=dt, device=device) for n, dt in rs_shapes[:-1]]
    rs_outs.append(rs_ins[-1][rank * rs_shapes[-1][0]:(rank + 1) * rs_shapes[-1][0]])

    def coalesced_rs():
        with dist._coalescing_manager(group=pg):
            for o, t in zip(rs_outs, rs_ins):
                dist.reduce_scatter_tensor(o, t, group=pg)

    assert launches(coalesced_rs) == 2  # one per dtype
    for i, (n, dt) in enumerate(rs_shapes):
        want = sum(val(world * n, dt, p, i)[rank * n:(rank + 1) * n] for p in range(world))
        assert torch.equal(rs_outs[i], want), i

    # dist.all_gather_coalesced (one dtype): output_lists[p][i] receives rank p's inputs[i]
    lengths = [5, 1000, 3, 70_001]
    inputs = [val(n, torch.float32, rank, i) for i, n in enumerate(lengths)]
    output_lists = [[torch.empty_like(t) for t in inputs] for _ in range(world)]
    assert launches(lambda: dist.all_gather_coalesced(output_lists, inputs, group=pg)) == 1
    for p in range(world):
        for i, n in enumerate(lengths):
            assert torch.equal(output_lists[p][i], val(n, torch.float32, p, i)), (p, i)

    # all_gather / reduce_scatter with tensor lists, and the process group's list forms
    outs = [torch.empty(4, device=device) for _ in range(world)]
    dist.all_gather(outs, torch.full((4,), float(rank), device=device), group=pg)
    assert all(torch.all(outs[p] == p) for p in range(world))
    rs_out = torch.empty(6, device=device)
    dist.reduce_scatter(rs_out, [torch.full((6,), float(q + rank), device=device) for q in range(world)], group=pg)
    assert torch.all(rs_out == sum(rank + p for p in range(world)))
    a, b = val(9, torch.float32, rank, 0), val(300, torch.int64, rank, 1)
    la = [torch.empty_like(a) for _ in range(world)]
    lb = [torch.empty(600, dtype=torch.int64, device=device)[::2] for _ in range(world)]  # not contiguous
    assert launches(lambda: pg.allgather([la, lb], [a, b]).wait()) == 1
    for p in range(world):
        assert torch.equal(la[p], val(9, torch.float32, p, 0)) and torch.equal(lb[p], val(300, torch.int64, p, 1))
    o1, o2 = torch.empty(7, device=device), torch.empty(11, device=device)
    l1 = [val(7, torch.float32, rank, q) for q in range(world)]
    l2 = [val(11, torch.float32, rank, 5 + q) for q in range(world)]
    assert launches(lambda: pg.reduce_scatter([o1, o2], [l1, l2]).wait()) == 1
    assert torch.equal(o1, sum(val(7, torch.float32, p, rank) for p in range(world)))
    assert torch.equal(o2, sum(val(11, torch.float32, p, 5 + rank) for p in range(world)))

    torch.cuda.synchronize()
    pg.comm.check_status()
    dist.barrier()
    dist.destroy_process_group()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as f:
        f.write("ok")


@pytest.mark.parametrize("world", [2, 3])
def test_c10d_coalesced_collectives(native_lib, world):
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_c10d_worker, args=(world, os.path.join(d, "rdzv"), d), nprocs=world, join=True)
        assert all(os.path.exists(os.path.join(d, f"ok{r}")) for r in range(world))


def test_collective_api_list_gather_and_scatter(native_lib):
    """ray_b200.collective.allgather_multi / reducescatter_multi through a B200 group of three workers."""
    from tests.test_gpu_api import Workers

    w = Workers(3)
    w.init("ag-rs-multi")
    try:
        def f(r):
            dev = w.dev(r)
            ts = [torch.full((17, 3), float(r), device=dev), torch.arange(1000, dtype=torch.int64, device=dev) + r]
            lists = [[torch.empty_like(t) for _ in range(3)] for t in ts]
            comm = w.col.get_group_handle("ag-rs-multi").comm
            before = comm.launch_count
            w.col.allgather_multi(lists, ts, group_name="ag-rs-multi")
            outs = [torch.empty(5, device=dev), torch.empty(999, device=dev)]
            ins = [[torch.full((5,), float(r + q), device=dev) for q in range(3)],
                   [torch.full((999,), float(r * q), device=dev) for q in range(3)]]
            w.col.reducescatter_multi(outs, ins, group_name="ag-rs-multi")
            torch.cuda.current_stream().synchronize()
            return (comm.launch_count - before, [[t.cpu() for t in lst] for lst in lists], [o.cpu() for o in outs])

        res = w.run(f)
        for r, (launches, lists, outs) in enumerate(res):
            assert launches == 2
            for p in range(3):
                assert torch.all(lists[0][p] == p) and torch.equal(lists[1][p], torch.arange(1000) + p)
            assert torch.all(outs[0] == sum(p + r for p in range(3)))
            assert torch.all(outs[1] == sum(p * r for p in range(3)))
    finally:
        w.destroy("ag-rs-multi")
