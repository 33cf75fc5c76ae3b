"""Grouped point-to-point: b200_p2p_batch (B200Comm.p2p_batch), B200ProcessGroup's coalescing block and
ray_b200.train.batch_isend_irecv.

The inbox here is 8 MiB per source, and several exchanges move 2.5 times that per direction.  Issued as
plain sends ahead of their receives on both sides, those exchanges could not complete; these tests
only ever run them as batches, or as plain calls in an order that cannot wait on itself, and show
that every byte arrives.  Every destination and every source sits in a buffer of random bytes with
at least 32 guard bytes on each side, and the whole buffer is compared on the device.  The device
watchdog is 15 s, so a defect fails as B200TimeoutError instead of stalling the suite.
"""
import ctypes
import os
import sys
import tempfile

import pytest
import torch
import torch.multiprocessing as mp

from ray_b200 import _native as N

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INBOX = 8 << 20
CHUNK = 16 << 10  # one chunk: the smallest p2p chunk
SIZES = [1, 13, CHUNK, INBOX, INBOX * 5 // 2]


@pytest.fixture(scope="module")
def groups(native_lib):
    from ray_b200.testing import LocalGroup

    cache = {}

    def get(n):
        if n not in cache:
            cache[n] = LocalGroup(n, timeout_ms=15000, staging_bytes=8 << 20, inbox_bytes=INBOX)
        return cache[n]

    yield get
    for g in cache.values():
        g.destroy()


class _Arena:
    """A tensor of `size` bytes at byte offset 32 + mis of a buffer of random bytes (guards included)."""

    def __init__(self, dev, size, mis, gen):
        self.buf = torch.randint(0, 256, (size + mis + 80,), dtype=torch.uint8, device=dev, generator=gen)
        self.lo, self.size = 32 + mis, size
        self.view = self.buf[self.lo:self.lo + size]
        self.before = self.buf.clone()


def _exchange(g, plan, seed=0, plain=(), stream_calls=None):
    """Run plan[r] = [(is_send, peer, size, mis), ...] on every rank: as one p2p_batch, or, for the ranks
    in `plain`, as plain send / recv calls in list order.  The k-th send of a directed pair meets the
    k-th receive.  Checks every byte of every buffer and the launch count of every rank."""
    n = g.world_size
    arenas = []
    for r in range(n):
        gen = torch.Generator(device=g.device(r)).manual_seed(seed * 131 + r)
        arenas.append([_Arena(g.device(r), size, mis, gen) for _, _, size, mis in plan[r]])
    before = [c.launch_count for c in g.comms]

    def f(c, r):
        ops = [(s, a.view, p) for (s, p, _, _), a in zip(plan[r], arenas[r])]
        if r in plain:
            for s, t, p in ops:
                (c.send if s else c.recv)(t, p)
        else:
            c.p2p_batch(ops)

    g.run(f)
    for r in range(n):
        live = sum(1 for op in plan[r] if op[2])
        want = live if r in plain else min(live, 1)
        assert g.comms[r].launch_count - before[r] == want, (r, g.comms[r].launch_count - before[r], want)
    # pair the k-th send of (a -> b) with the k-th receive of b from a
    sends, recvs = {}, {}
    for r in range(n):
        for (s, p, _, _), a in zip(plan[r], arenas[r]):
            (sends if s else recvs).setdefault((r, p) if s else (p, r), []).append(a)
    assert sends.keys() == recvs.keys()
    for key in sends:
        assert len(sends[key]) == len(recvs[key]), key
        for src, dst in zip(sends[key], recvs[key]):
            assert src.size == dst.size, key
            dst.before[dst.lo:dst.lo + dst.size] = src.before[src.lo:src.lo + src.size].to(dst.buf.device)
    for r in range(n):
        for k, a in enumerate(arenas[r]):
            assert torch.equal(a.buf, a.before), f"rank {r} op {k} {plan[r][k]}: payload or guard bytes differ"


def _restore_blocks(g):
    """The grid cap LocalGroup gave its communicators."""
    sms = torch.cuda.get_device_properties(g.devices[0]).multi_processor_count
    for c in g.comms:
        c.set_blocks(max(1, (sms - 4) // g.world_size) if g.shared_gpu else 0)


def _ring(n, size, mis=lambda r, s: 0):
    """Every rank sends `size` bytes to r+1 and receives from r-1 (at world 2: a bidirectional exchange)."""
    return [[(True, (r + 1) % n, size, mis(r, True)), (False, (r - 1) % n, size, mis(r, False))] for r in range(n)]


@pytest.mark.parametrize("size", SIZES, ids=["1B", "13B", "chunk", "inbox", "2.5inbox"])
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_ring_exchange(groups, world, size):
    g = groups(world)
    _exchange(g, _ring(world, size), seed=world)
    # receives first in the list: the batch does not care
    _exchange(g, [ops[::-1] for ops in _ring(world, size)], seed=world + 1)


def test_several_ops_to_one_peer_keep_their_order(groups):
    g = groups(2)
    sizes = [INBOX + 48, 0, 13, 3 * INBOX // 2, CHUNK + 1, 0, 1, 2 * INBOX, 4096]
    # the sender's views are misaligned where the receiver's are aligned and the reverse, so the large
    # messages meet bulk copies on one side and ld/st on the other
    plan = [[(True, 1, s, (k % 2) * 5) for k, s in enumerate(sizes)] + [(False, 1, 777_777, 0)],
            [(False, 0, s, ((k + 1) % 2) * 9) for k, s in enumerate(sizes)] + [(True, 0, 777_777, 3)]]
    _exchange(g, plan, seed=7)
    # the same on both directions at once, with receives interleaved between the sends
    both = [[op for k, s in enumerate(sizes) for op in ((True, 1 - r, s, (k + r) % 3 * 7),
                                                        (False, 1 - r, s, (k + r) % 2 * 11))]
            for r in range(2)]
    _exchange(g, both, seed=8)


def test_mixed_dtypes(groups):
    g = groups(3)
    gen = torch.Generator().manual_seed(11)
    sent = [torch.randn(17, 3, generator=gen), torch.randn(1001, generator=gen).to(torch.float16),
            torch.arange(-50, 77, dtype=torch.int64), torch.rand(13, generator=gen) < 0.5,
            torch.randn(3 << 20, generator=gen).to(torch.bfloat16), torch.zeros(0, dtype=torch.float64),
            torch.randint(0, 256, (7,), dtype=torch.uint8, generator=gen)]
    ins = [t.to(g.device(0)) for t in sent]
    outs = [[torch.empty_like(t, device=g.device(r)) for t in sent] for r in range(3)]

    def f(c, r):
        if r == 0:
            c.p2p_batch([(True, t, p) for t in ins for p in (1, 2)])
        else:
            c.p2p_batch([(False, o, 0) for o in outs[r]])

    g.run(f)
    for r in (1, 2):
        for o, s in zip(outs[r], sent):
            assert o.dtype == s.dtype and torch.equal(o.cpu(), s)


@pytest.mark.parametrize("batch_rank", [0, 1])
def test_batch_pairs_with_plain_calls(groups, batch_rank):
    g = groups(2)
    other = 1 - batch_rank
    big = INBOX * 5 // 2
    # the plain side in either order: its peer's ops all run at once
    for order in (1, -1):
        plan = _ring(2, big, mis=lambda r, s: 3 if (r == other and s) else 0)
        plan[other] = plan[other][::order]
        _exchange(g, plan, seed=20 + order, plain=(other,))
    # several messages each way against plain calls: the plain side's order matches the batch's per pair
    plan = [[(True, 1, big, 0), (False, 1, 13, 0), (True, 1, CHUNK, 1), (False, 1, INBOX, 0)],
            [(False, 0, big, 0), (True, 0, 13, 0), (False, 0, CHUNK, 0), (True, 0, INBOX, 5)]]
    _exchange(g, plan, seed=30, plain=(other,))


@pytest.mark.parametrize("batch_send", [True, False])
def test_folded_role_against_plain_16_cta_peer(groups, batch_send):
    """Grid cap 2(n-1): one CTA per role serves all 16 sub-rings of a 2.5-inbox message, in order,
    while the peer's plain send / recv runs 16 CTAs, one per sub-ring."""
    g = groups(2)
    for c in g.comms:
        c.set_blocks(2)
    try:
        big = INBOX * 5 // 2
        plan = [[(batch_send, 1, big, 0), (batch_send, 1, 1000, 0), (not batch_send, 1, big, 0)],
                [(not batch_send, 0, big, 0), (not batch_send, 0, 1000, 0), (batch_send, 0, big, 4)]]
        # rank 1 plain; its order keeps the directions independent: both messages to rank 0 first
        _exchange(g, plan, seed=40, plain=(1,))
        plan[1] = [plan[1][2], plan[1][0], plan[1][1]]
        _exchange(g, plan, seed=41, plain=(1,))
        _exchange(g, plan, seed=42)  # both folded
    finally:
        _restore_blocks(g)


def test_interleaves_with_send_recv_and_alltoall(groups):
    """send/recv, batch, alltoall, batch, send/recv on the same pairs in one stream: the persistent
    sequence numbers stay consistent across all three kinds of launch."""
    g = groups(3)
    n = 3
    gen = torch.Generator().manual_seed(50)

    def rnd(k):
        return torch.randint(0, 256, (k,), dtype=torch.uint8, generator=gen)

    s1 = rnd(300_001)
    b1 = [[rnd(INBOX + 17 * (r + 1)), rnd(64)] for r in range(n)]  # rank r's two sends to r+1
    a2a = [[rnd(5000 * (1 + r + 2 * p)) for p in range(n)] for r in range(n)]  # rank r -> rank p
    b2 = [rnd(2 * INBOX + r) for r in range(n)]  # rank r -> r-1
    s2 = rnd(CHUNK * 3)
    dev = [g.device(r) for r in range(n)]
    s1d, s2d = s1.to(dev[0]), s2.to(dev[2])
    b1d = [[t.to(dev[r]) for t in b1[r]] for r in range(n)]
    a2ad = [[t.to(dev[r]) for t in a2a[r]] for r in range(n)]
    b2d = [b2[r].to(dev[r]) for r in range(n)]
    r_s1, r_s2 = torch.empty_like(s1, device=dev[1]), torch.empty_like(s2, device=dev[0])
    r_b1 = [[torch.empty_like(t, device=dev[r]) for t in b1[(r - 1) % n]] for r in range(n)]
    r_a2a = [[torch.empty_like(a2a[p][r], device=dev[r]) for p in range(n)] for r in range(n)]
    r_b2 = [torch.empty_like(b2[(r + 1) % n], device=dev[r]) for r in range(n)]
    before = [c.launch_count for c in g.comms]

    def f(c, r):
        if r == 0:
            c.send(s1d, 1)
        elif r == 1:
            c.recv(r_s1, 0)
        c.p2p_batch([(True, b1d[r][0], (r + 1) % n), (False, r_b1[r][0], (r - 1) % n),
                     (True, b1d[r][1], (r + 1) % n), (False, r_b1[r][1], (r - 1) % n)])
        c.alltoall(r_a2a[r], a2ad[r])
        c.p2p_batch([(False, r_b2[r], (r + 1) % n), (True, b2d[r], (r - 1) % n)])
        if r == 2:
            c.send(s2d, 0)
        elif r == 0:
            c.recv(r_s2, 2)

    g.run(f)
    assert [c.launch_count - b for c, b in zip(g.comms, before)] == [5, 4, 4]
    assert torch.equal(r_s1.cpu(), s1) and torch.equal(r_s2.cpu(), s2)
    for r in range(n):
        assert all(torch.equal(o.cpu(), t) for o, t in zip(r_b1[r], b1[(r - 1) % n])), r
        assert all(torch.equal(r_a2a[r][p].cpu(), a2a[p][r]) for p in range(n)), r
        assert torch.equal(r_b2[r].cpu(), b2[(r + 1) % n]), r


def test_cuda_graph_replay_matches_eager(groups):
    g = groups(2)
    sizes = [INBOX * 5 // 2, 13, CHUNK]
    srcs = [[torch.empty(s, dtype=torch.uint8, device=g.device(r)) for s in sizes] for r in range(2)]
    dsts = [[torch.empty(s, dtype=torch.uint8, device=g.device(r)) for s in sizes] for r in range(2)]

    def call(c, r):
        c.p2p_batch([op for k in range(len(sizes)) for op in ((True, srcs[r][k], 1 - r), (False, dsts[r][k], 1 - r))])

    def fill(seed):
        for r in range(2):
            gen = torch.Generator(device=g.device(r)).manual_seed(seed + r)
            for t in srcs[r] + dsts[r]:
                t.copy_(torch.randint(0, 256, t.shape, dtype=torch.uint8, device=g.device(r), generator=gen))

    fill(60)
    g.run(call)
    eager = [[t.clone() for t in dsts[r]] for r in range(2)]
    assert all(torch.equal(eager[r][k], srcs[1 - r][k].to(g.device(r))) for r in range(2) for k in range(3))
    graphs = []
    for r, c in enumerate(g.comms):
        torch.cuda.set_device(g.devices[r])
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=g.streams[r]):
            call(c, r)
        graphs.append(gr)
    for seed in (60, 70):
        fill(seed)
        want = [[t.clone() for t in srcs[1 - r]] for r in range(2)]
        torch.cuda.synchronize()
        for r in range(2):
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        g.synchronize()
        for r in range(2):
            for k in range(3):
                assert torch.equal(dsts[r][k], want[r][k].to(g.device(r))), (seed, r, k)
        if seed == 60:
            assert all(torch.equal(dsts[r][k], eager[r][k]) for r in range(2) for k in range(3))


def test_launch_counts_and_refusals(groups):
    g = groups(3)
    c = g.comms[0]
    dev = g.device(0)
    t = torch.zeros(64, dtype=torch.uint8, device=dev)
    before = c.launch_count

    def refused(fn, match=None):
        with pytest.raises(N.B200Error, match=match):
            fn()
        assert c.launch_count == before

    c.p2p_batch([])
    c.p2p_batch([(True, t[:0], 1), (False, t[:0], 2)])
    assert c.launch_count == before
    refused(lambda: c.p2p_batch([(True, t[:0], 1)] * (N.P2P_TABLE_MAX + 1)), "at most 256")
    refused(lambda: c.p2p_batch([(True, t, 3)]), "out of range")
    refused(lambda: c.p2p_batch([(True, t, -1)]), "out of range")
    refused(lambda: c.p2p_batch([(False, t, 1), (True, t, 0)]), "is this rank")
    refused(lambda: c.p2p_batch([(True, t[:0], 0)]), "is this rank")  # an empty op's peer is checked too
    lib, h = c._lib, c._h
    stream = torch.cuda.current_stream(dev).cuda_stream
    one = (ctypes.c_void_p * 1)(t.data_ptr())
    size = (ctypes.c_size_t * 1)(64)
    peer, send = (ctypes.c_int * 1)(1), (ctypes.c_int * 1)(1)
    assert lib.b200_p2p_batch(h, one, size, peer, send, -1, stream) == N.ERR_INVALID
    assert lib.b200_p2p_batch(h, None, size, peer, send, 1, stream) == N.ERR_INVALID
    assert lib.b200_p2p_batch(h, one, size, None, send, 1, stream) == N.ERR_INVALID
    assert lib.b200_p2p_batch(h, one, size, peer, None, 1, stream) == N.ERR_INVALID
    assert lib.b200_p2p_batch(h, (ctypes.c_void_p * 1)(None), size, peer, send, 1, stream) == N.ERR_INVALID
    assert lib.b200_p2p_batch(h, None, None, None, None, 0, stream) == N.OK
    c.set_blocks(2 * (3 - 1) - 1)
    try:
        refused(lambda: c.p2p_batch([(True, t, 1)]), "co-resident CTAs")
        # checked against the world size, whatever the batch holds, so every rank refuses alike
        assert lib.b200_p2p_batch(h, None, None, None, None, 0, stream) == N.ERR_INVALID
    finally:
        _restore_blocks(g)
    assert c.launch_count == before
    # one launch per batch, whatever it holds
    plan = [[(True, 1, 13, 0), (True, 2, CHUNK, 0), (False, 1, 5, 0), (False, 2, 0, 0)],
            [(False, 0, 13, 0), (True, 0, 5, 0)],
            [(False, 0, CHUNK, 0), (True, 0, 0, 0)]]
    _exchange(g, plan, seed=80)


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

    nxt, prv = (rank + 1) % world, (rank - 1) % world

    def payload(src, k, dtype=torch.float32):
        return (torch.arange(k, device=device) % 9973 + 7 * src).to(dtype)

    # a ring exchange of 40 MiB per direction through the default 32 MiB inbox
    k = (40 << 20) // 4
    out = torch.full((k,), -1.0, device=device)
    ops = [dist.P2POp(dist.isend, payload(rank, k), nxt), dist.P2POp(dist.irecv, out, prv)]
    works = []
    assert launches(lambda: works.extend(T.batch_isend_irecv(ops))) == 1
    assert len(works) == 1
    for w in works:
        w.wait()
    assert torch.equal(out, payload(prv, k))

    # isend / irecv in a coalescing block: one launch, the Works complete with it
    a_out = torch.zeros(1000, dtype=torch.int64, device=device)
    b_out = torch.zeros(33, dtype=torch.bfloat16, device=device)
    got = {}

    def block():
        with dist._coalescing_manager(pg, device, async_ops=True) as cm:
            w1 = dist.irecv(a_out, prv)
            w2 = dist.isend(payload(rank, 1000, torch.int64), nxt)
            w3 = dist.isend(payload(rank, 33, torch.bfloat16), nxt)
            w4 = dist.irecv(b_out, prv)
            try:
                w1.wait()
            except RuntimeError:
                got["early"] = True
        got["works"] = [w1, w2, w3, w4]
        cm.wait()

    assert launches(block) == 1
    assert got["early"] and len(got["works"]) == 4
    for w in got["works"]:
        w.wait()
    assert torch.equal(a_out, payload(prv, 1000, torch.int64)) and torch.equal(b_out, payload(prv, 33, torch.bfloat16))

    # plain send / recv outside any block: one launch each, as before
    small = torch.zeros(17, device=device)
    if rank == 0:
        assert launches(lambda: dist.send(payload(0, 17), 1)) == 1
    elif rank == 1:
        assert launches(lambda: dist.recv(small, 0)) == 1
        assert torch.equal(small, payload(0, 17))

    torch.cuda.synchronize()
    pg.comm.check_status()
    dist.barrier()
    dist.destroy_process_group()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as f:
        f.write("ok")


@pytest.mark.parametrize("world", [2, 3])
def test_c10d_batch_isend_irecv(native_lib, world):
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_c10d_worker, args=(world, os.path.join(d, "rdzv"), d), nprocs=world, join=True)
        assert all(os.path.exists(os.path.join(d, f"ok{r}")) for r in range(world))
