"""Tensor lists point to point in one launch: b200_send_multi / b200_recv_multi / b200_get_multi
(B200Comm.send_multi / recv_multi / get_multi) and the paths built on them (RDT two-sided and
one-sided transports, the tensor channel's point-to-point payload).

Every received byte is compared with what was sent.  Received tensors are views into one buffer
with guard bytes around each of them, and the guard bytes must come back unchanged: the padding of
a tensor's last 16-byte unit travels on the wire but must never be stored.
"""
import ctypes

import numpy as np
import pytest
import torch

from ray_b200 import _native as N

pytestmark = pytest.mark.gpu

TABLE = N.P2P_TABLE_MAX
GUARD = 0x5A
PAIRS = {2: [(0, 1), (1, 0)], 3: [(0, 2), (2, 0)], 4: [(1, 3), (3, 0)]}


@pytest.fixture(scope="module")
def groups(native_lib):
    from ray_b200.testing import LocalGroup

    cache = {}

    def get(n):
        if n not in cache:
            # 8 MiB inbox: 64 KiB ring slots, so aligned lists of large tensors take the bulk path
            cache[n] = LocalGroup(n, timeout_ms=15000, staging_bytes=8 << 20, inbox_bytes=8 << 20,
                                  heap_bytes=64 << 20)
        return cache[n]

    yield get
    for g in cache.values():
        g.destroy()


def _layout(sizes, misalign):
    """Offsets of tensors of `sizes` bytes in one buffer: tensor i starts misalign(i) bytes past a
    16-byte boundary, with at least 32 guard bytes on both sides."""
    offs, pos = [], 32
    for i, s in enumerate(sizes):
        pos = (pos + 15) // 16 * 16 + misalign(i)
        offs.append(pos)
        pos += s + 32
    return offs, pos


def _list(dev, sizes, misalign, fill):
    offs, total = _layout(sizes, misalign)
    buf = torch.full((total,), fill, dtype=torch.uint8, device=dev)
    return buf, offs, [buf[o:o + s] for o, s in zip(offs, sizes)]


def _transfer(g, src, dst, sizes, s_mis=lambda i: 0, r_mis=lambda i: 0, seed=0):
    """src send_multi -> dst recv_multi of a list of `sizes` bytes; checks every byte, the guard
    bytes and the launch count of both sides."""
    rng = np.random.default_rng(seed)
    data = [torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in sizes]
    sbuf, soffs, sviews = _list(g.device(src), sizes, s_mis, 0xA5)
    for v, d in zip(sviews, data):
        v.copy_(d)
    sent = sbuf.cpu()
    rbuf, roffs, rviews = _list(g.device(dst), sizes, r_mis, GUARD)
    want = torch.full_like(rbuf, GUARD, device="cpu")
    for o, d in zip(roffs, data):
        want[o:o + d.numel()] = d
    before = [c.launch_count for c in g.comms]

    def f(c, r):
        if r == src:
            c.send_multi(sviews, dst)
        elif r == dst:
            c.recv_multi(rviews, src)

    g.run(f)
    tables = -(-sum(1 for s in sizes if s) // TABLE)
    launches = [c.launch_count - b for c, b in zip(g.comms, before)]
    assert launches[src] == tables and launches[dst] == tables, launches
    assert torch.equal(rbuf.cpu(), want), "payload or guard bytes differ"
    assert torch.equal(sbuf.cpu(), sent), "the sent tensors changed"


LISTS = {
    "one": [100_000],
    "bytes_1_to_15": list(range(1, 16)),
    "zeros_scattered": [0, 100, 0, 0, 4096, 0, 17, 33, 0],
    "below_one_chunk": [1000, 2000, 3000, 5],
    "larger_than_inbox": [(1 << 20) + 16 * i + (i % 3) for i in range(20)],
    "larger_than_inbox_aligned": [1 << 20] * 20,
    "table_max_plus_one": [16 + (i % 37) for i in range(TABLE + 1)],
    "large_aligned": [64 << 10] * 12,
}


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("name", list(LISTS))
def test_lists_byte_for_byte(groups, world, name):
    g = groups(world)
    for k, (src, dst) in enumerate(PAIRS[world]):
        _transfer(g, src, dst, LISTS[name], seed=k)


@pytest.mark.parametrize("world", [2, 4])
def test_views_misaligned_by_1_to_15_bytes(groups, world):
    g = groups(world)
    sizes = [(i * 977) % 5000 + 1 for i in range(40)] + [300_000, 70_001]
    src, dst = PAIRS[world][0]
    _transfer(g, src, dst, sizes, s_mis=lambda i: i % 15 + 1, r_mis=lambda i: (7 * i) % 15 + 1, seed=3)
    _transfer(g, dst, src, sizes, s_mis=lambda i: 0, r_mis=lambda i: i % 15 + 1, seed=4)


def test_empty_list_launches_nothing(groups):
    g = groups(2)
    before = [c.launch_count for c in g.comms]
    g.run(lambda c, r: c.send_multi([], 1) if r == 0 else c.recv_multi([], 0))
    g.run(lambda c, r: c.send_multi([torch.empty(0, device=g.device(0))], 1) if r == 0 else
          c.recv_multi([torch.empty(0, device=g.device(1))], 0))
    assert [c.launch_count for c in g.comms] == before


def test_mixed_dtypes(groups):
    g = groups(2)
    rng = np.random.default_rng(5)
    sent = [torch.from_numpy(rng.standard_normal((17, 3)).astype(np.float32)),
            torch.from_numpy(rng.standard_normal(1001)).to(torch.float16),
            torch.arange(-50, 77, dtype=torch.int64), torch.from_numpy(rng.random(13) < 0.5),
            torch.from_numpy(rng.standard_normal(2049)).to(torch.bfloat16), torch.zeros(0, dtype=torch.float64),
            torch.from_numpy(rng.integers(0, 256, 7, dtype=np.uint8))]
    ins = [t.to(g.device(0)) for t in sent]
    outs = [torch.empty_like(t, device=g.device(1)) for t in sent]
    g.run(lambda c, r: c.send_multi(ins, 1) if r == 0 else c.recv_multi(outs, 0))
    for o, s in zip(outs, sent):
        assert o.dtype == s.dtype and torch.equal(o.cpu(), s)


@pytest.mark.parametrize("sender,receiver", [("ldst", "ldst"), ("bulk", "bulk"), ("bulk", "ldst"),
                                             ("ldst", "bulk")])
def test_each_mechanism_pairing(groups, sender, receiver):
    """Large 16-byte aligned whole-unit tensors take the bulk-copy unit; a side with one misaligned
    view, or with B200_PARAM_P2P_BULK_MIN_CHUNK = 0, moves its bytes with ld/st.  The wire layout is
    the same either way."""
    g = groups(2)
    sizes = [64 << 10] * 10 + [48 << 10, 1 << 20]
    forced = []
    try:
        if sender == "ldst" and receiver == "ldst":
            for c in g.comms:
                c.set_param(N.PARAM_P2P_BULK_MIN_CHUNK, 0)
                forced.append(c)
            _transfer(g, 0, 1, sizes, seed=11)
            return
        s_mis = (lambda i: 0) if sender == "bulk" else (lambda i: 1 if i == 3 else 0)
        r_mis = (lambda i: 0) if receiver == "bulk" else (lambda i: 9 if i == 5 else 0)
        _transfer(g, 0, 1, sizes, s_mis=s_mis, r_mis=r_mis, seed=12)
    finally:
        for c in forced:
            c.set_param(N.PARAM_P2P_BULK_MIN_CHUNK, -1)


def test_interleaves_with_send_recv_in_stream_order(groups):
    """send, send_multi, send against recv, recv_multi, recv: the sequence numbers carry on."""
    g = groups(2)
    rng = np.random.default_rng(9)
    a = torch.from_numpy(rng.standard_normal(30_000).astype(np.float32))
    lst = [torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in (5, 70_000, 0, 1 << 20, 3)]
    b = torch.from_numpy(rng.standard_normal(123).astype(np.float32))
    ins = [a.to(g.device(0)), [t.to(g.device(0)) for t in lst], b.to(g.device(0))]
    outs = [torch.zeros_like(a, device=g.device(1)), [torch.zeros_like(t, device=g.device(1)) for t in lst],
            torch.zeros_like(b, device=g.device(1))]
    for _ in range(2):
        def f(c, r):
            if r == 0:
                c.send(ins[0], 1)
                c.send_multi(ins[1], 1)
                c.send(ins[2], 1)
            else:
                c.recv(outs[0], 0)
                c.recv_multi(outs[1], 0)
                c.recv(outs[2], 0)

        g.run(f)
        assert torch.equal(outs[0].cpu(), a) and torch.equal(outs[2].cpu(), b)
        assert all(torch.equal(o.cpu(), t) for o, t in zip(outs[1], lst))


def test_cuda_graph_replay_matches_eager(groups):
    g = groups(2)
    sizes = [3, 4096, 100_001, 64 << 10]
    ins = [torch.zeros(s, dtype=torch.uint8, device=g.device(0)) for s in sizes]
    outs = [torch.zeros(s, dtype=torch.uint8, device=g.device(1)) for s in sizes]

    def f(c, r):
        if r == 0:
            c.send_multi(ins, 1, stream=g.streams[0])
        else:
            c.recv_multi(outs, 0, stream=g.streams[1])

    g.run(f)  # eager first: kernel attributes are set outside capture
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
        for t, d in zip(ins, fresh):
            t.copy_(d)
        for o in outs:
            o.zero_()
        for d in set(g.devices):
            torch.cuda.synchronize(d)
        for r in range(2):
            torch.cuda.set_device(g.devices[r])
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        g.synchronize()
        graph_out = [o.cpu() for o in outs]
        assert all(torch.equal(o, d) for o, d in zip(graph_out, fresh))
        for o in outs:
            o.zero_()
        g.run(f)
        assert all(torch.equal(o.cpu(), e) for o, e in zip(outs, graph_out)), "eager and replay differ"


def _arr(ctype, vals):
    return (ctype * max(len(vals), 1))(*vals)


def test_refused_calls_launch_nothing(groups):
    g = groups(2)
    lib, c = N.load(), g.comms[0]
    h, dev = c._h, g.device(0)
    x = torch.zeros(64, dtype=torch.uint8, device=dev)
    P = _arr(ctypes.c_void_p, [x.data_ptr(), x.data_ptr() + 32])
    S = _arr(ctypes.c_size_t, [16, 16])
    _, heap = c.heap_range()
    cases = [
        ("send null entry", lambda: lib.b200_send_multi(h, _arr(ctypes.c_void_p, [x.data_ptr(), None]), S, 2, 1, None),
         "tensor 1 is null but has 16 bytes"),
        ("recv null entry", lambda: lib.b200_recv_multi(h, _arr(ctypes.c_void_p, [None, None]), S, 2, 1, None),
         "tensor 0 is null but has 16 bytes"),
        ("send self", lambda: lib.b200_send_multi(h, P, S, 2, 0, None), "peer rank 0 is this rank"),
        ("recv bad rank", lambda: lib.b200_recv_multi(h, P, S, 2, 2, None), "peer rank 2 out of range for world size 2"),
        ("negative count", lambda: lib.b200_send_multi(h, P, S, -1, 1, None), "ntensors -1 is negative"),
        ("null arrays", lambda: lib.b200_recv_multi(h, None, S, 2, 1, None), "null argument array"),
        ("get bad rank", lambda: lib.b200_get_multi(h, P, 5, _arr(ctypes.c_size_t, [0, 0]), S, 2, None),
         "source rank 5 out of range"),
        ("get outside heap", lambda: lib.b200_get_multi(h, P, 1, _arr(ctypes.c_size_t, [0, heap - 8]), S, 2, None),
         f"tensor 1: [{heap - 8}, {heap + 8}) is outside the {heap}-byte symmetric heap"),
        ("get null entry", lambda: lib.b200_get_multi(h, _arr(ctypes.c_void_p, [None, None]), 1,
                                                      _arr(ctypes.c_size_t, [0, 0]), S, 2, None),
         "tensor 0 is null but has 16 bytes"),
    ]
    before = c.launch_count
    with torch.cuda.device(dev):
        for name, call, text in cases:
            assert call() == N.ERR_INVALID, name
            assert text in N.last_error(), (name, N.last_error())
    torch.cuda.synchronize(dev)
    assert c.launch_count == before


def _publish(g, owner, sizes, misalign, seed):
    """Writes random bytes for each size into the owner's heap; returns (offsets, host data)."""
    rng = np.random.default_rng(seed)
    offs, total = _layout(sizes, misalign)
    data = [torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in sizes]
    view = g.comms[owner].heap_view(0, total)
    for o, d in zip(offs, data):
        view[o:o + d.numel()].copy_(d)
    torch.cuda.synchronize(g.devices[owner])
    return offs, data


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("case", ["small_misaligned", "large_aligned", "table_max_plus_one"])
def test_get_multi_byte_for_byte(groups, world, case):
    g = groups(world)
    if case == "small_misaligned":
        sizes, smis, dmis = [1, 15, 0, 4096, 3, 70_001, 0, 100], (lambda i: i % 15), (lambda i: (3 * i) % 16)
    elif case == "large_aligned":
        sizes, smis, dmis = [512 << 10] * 6 + [256 << 10], (lambda i: 0), (lambda i: 0)
    else:
        sizes, smis, dmis = [16 + i % 5 for i in range(TABLE + 1)], (lambda i: i % 2), (lambda i: 0)
    owner, me = PAIRS[world][0]
    offs, data = _publish(g, owner, sizes, smis, seed=world)
    buf, doffs, views = _list(g.device(me), sizes, dmis, GUARD)
    want = torch.full_like(buf, GUARD, device="cpu")
    for o, d in zip(doffs, data):
        want[o:o + d.numel()] = d
    before = [c.launch_count for c in g.comms]
    g.run(lambda c, r: c.get_multi(views, owner, offs) if r == me else None)
    launches = [c.launch_count - b for c, b in zip(g.comms, before)]
    assert launches[me] == -(-sum(1 for s in sizes if s) // TABLE) and launches[owner] == 0, launches
    assert torch.equal(buf.cpu(), want)


# ---- integration --------------------------------------------------------------------------------

def test_rdt_two_sided_one_launch_per_side(native_lib):
    from ray_b200.rdt import B200CommunicatorMetadata, B200TensorTransport
    from tests.test_gpu_api import Workers

    w = Workers(2)
    w.init("rdt-multi")
    tr = B200TensorTransport()
    B200TensorTransport.group_resolver = staticmethod(lambda src, dst: ("rdt-multi", int(src[-1]), int(dst[-1])))
    try:
        meta_c = tr.get_communicator_metadata("actor0", "actor1", "B200")
        assert isinstance(meta_c, B200CommunicatorMetadata)
        payload = [torch.randn(17, 3), torch.arange(1000, dtype=torch.float32), torch.randn(5).to(torch.float16)]
        sent = [t.to(w.dev(0)) for t in payload]
        meta_t = tr.extract_tensor_transport_metadata("obj-1", sent)

        def f(r):
            comm = w.col.get_group_handle("rdt-multi").comm
            before = comm.launch_count
            if r == 0:
                tr.send_multiple_tensors(sent, meta_t, meta_c)
                return comm.launch_count - before, None
            got = tr.recv_multiple_tensors("obj-1", meta_t, meta_c)
            torch.cuda.current_stream().synchronize()
            return comm.launch_count - before, [g.cpu() for g in got]

        res = w.run(f)
        assert res[0][0] == 1 and res[1][0] == 1, "one launch per side for a 3-tensor object"
        assert all(torch.equal(g, p) for g, p in zip(res[1][1], payload))
    finally:
        B200TensorTransport.group_resolver = None
        w.run(lambda r: w.col.destroy_collective_group("rdt-multi"))


def test_rdt_one_sided_one_receiver_launch(native_lib, monkeypatch):
    import threading

    from ray_b200.rdt import B200IpcTransport
    from tests.test_gpu_api import Workers

    monkeypatch.setenv("B200_HEAP_BYTES", str(64 << 20))
    w = Workers(2)
    w.init("ipc-multi")
    tr = B200IpcTransport()
    B200IpcTransport.group_resolver = staticmethod(lambda src, dst: ("ipc-multi", int(src[-1]), int(dst[-1])))
    B200IpcTransport.publish_resolver = staticmethod(lambda: ("ipc-multi", 0))
    box, ready, done = {}, threading.Event(), threading.Event()
    payload = [torch.randn(1 << 18), torch.arange(1003, dtype=torch.int32), torch.randn(7, 9).to(torch.float16)]
    try:
        meta_c = tr.get_communicator_metadata("actor0", "actor1", "B200_IPC")

        def f(r):
            comm = w.col.get_group_handle("ipc-multi").comm
            if r == 0:
                sent = [t.to(w.dev(0)) for t in payload]
                before = comm.launch_count
                box["meta"] = tr.extract_tensor_transport_metadata("obj-7", sent)
                ready.set()
                done.wait(60)
                tr.garbage_collect("obj-7", box["meta"], sent)
                return comm.launch_count - before
            ready.wait(60)
            before = comm.launch_count
            got = tr.recv_multiple_tensors("obj-7", box["meta"], meta_c)
            torch.cuda.current_stream().synchronize()
            done.set()
            return comm.launch_count - before, [g.cpu() for g in got]

        res = w.run(f)
        assert res[0] == 0 and res[1][0] == 1, res
        assert all(torch.equal(g, p) for g, p in zip(res[1][1], payload))
    finally:
        done.set()
        B200IpcTransport.group_resolver = None
        B200IpcTransport.publish_resolver = None
        w.run(lambda r: w.col.destroy_collective_group("ipc-multi"))


def test_channel_message_is_one_header_and_one_payload_launch(native_lib):
    from ray_b200.channel import TorchTensorAcceleratorChannel
    from tests.test_gpu_channel import Actors

    a = Actors(2)
    try:
        chans = [TorchTensorAcceleratorChannel(a.comms[r], 0, [1]) for r in range(2)]
        msg = [torch.randn(3, 5), torch.arange(7, dtype=torch.int64), torch.randn(11).to(torch.bfloat16),
               torch.randint(0, 255, (1000,), dtype=torch.uint8), torch.randn(4, 4).to(torch.float16)]

        def f(r, c):
            before = c.comm.launch_count
            if r == 0:
                chans[0].write([t.to(a.dev(0)) for t in msg])
                return c.comm.launch_count - before, None
            got = [t.cpu() for t in chans[1].read()]
            return c.comm.launch_count - before, got

        res = a.run(f)
        assert res[0][0] == 2 and res[1][0] == 2, "header + payload, not one launch per tensor"
        assert len(res[1][1]) == len(msg) and all(torch.equal(g, m) for g, m in zip(res[1][1], msg))
    finally:
        for c in a.comms:
            c.destroy()
