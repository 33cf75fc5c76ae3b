"""The single-tensor data-movement entries byte for byte: b200_broadcast, b200_allgather (staged and
pull kernels), b200_send / b200_recv and b200_get (B200Comm.broadcast, allgather, allgather_into,
send, recv and get).

Every operand is a uint8 (or typed) view at a chosen byte offset inside a buffer of random bytes,
with at least 32 guard bytes on each side.  Every case asserts that
  * every destination byte holds what the source held;
  * every other byte of every buffer on every rank is unchanged: the guard bytes, the root's and
    the sender's buffers, the owner's heap;
  * each rank made the launches the entry's plan says.
Sizes sit on the edges of the plans: 16-byte units and their tails, a full row of the grid, the
staging slot and the pieces beyond it, the pull kernel's chunk and launch limit, the point-to-point
chunk, ring and inbox sizes, and the get kernel's bulk segment.  Comparisons run on the device.
"""
import contextlib

import numpy as np
import pytest
import torch

from oracle import collective_oracle as O
from ray_b200 import _native as N

pytestmark = pytest.mark.gpu

SLOT = 2 << 20   # staging slot: the smallest the library allows, so messages of several pieces stay cheap
INBOX = 8 << 20  # per-source inbox: 16 rings x 8 slots of 64 KiB, large enough for the bulk p2p path
HEAP = 16 << 20
GUARD = 32
KTHREADS = 512          # threads per CTA: one row of the grid moves grid * 512 units of 16 bytes
P2P_RING_SLOT = INBOX // 16 // 8
GET_SEG = 256 << 10     # bulk segment of b200_get
GET_LDST_CTAS = 32
OFFS = (0, 1, 8, 15)


@pytest.fixture(scope="module")
def groups(native_lib):
    from ray_b200.testing import LocalGroup

    cache = {}

    def get(n, staging=SLOT):
        if (n, staging) not in cache:
            cache[n, staging] = LocalGroup(n, timeout_ms=20000, staging_bytes=staging, inbox_bytes=INBOX,
                                           heap_bytes=HEAP)
        return cache[n, staging]

    yield get
    for g in cache.values():
        g.destroy()


def _default_blocks(g):
    """The CTA cap LocalGroup set: (SMs-4)/ranks-per-GPU when ranks share a GPU, else 0 (unforced)."""
    if not g.shared_gpu:
        return 0
    per_dev = max(g.devices.count(d) for d in set(g.devices))
    sms = torch.cuda.get_device_properties(g.devices[0]).multi_processor_count
    return max(1, (sms - 4) // per_dev)


def _grid(g):
    b = _default_blocks(g)
    return b if b > 0 else torch.cuda.get_device_properties(g.devices[0]).multi_processor_count


@contextlib.contextmanager
def _knobs(g, blocks=None, params=(), ranks=None):
    """set_blocks / set_param on `ranks` (default: all) for a with-block, then the defaults again."""
    ranks = range(g.world_size) if ranks is None else ranks
    try:
        for r in ranks:
            if blocks is not None:
                g.comms[r].set_blocks(blocks)
            for p, v in params:
                g.comms[r].set_param(p, v)
        yield
    finally:
        for r in ranks:
            if blocks is not None:
                g.comms[r].set_blocks(_default_blocks(g))
            for p, _ in params:
                g.comms[r].set_param(p, -1)


def _pull_plan():
    """(chunk, max_bytes) of the pull all-gather on SLOT (policy.h pipe_plan, PIPE_GATHER): 1 MiB
    chunks rounded to whole 1 MiB quanta that fit the slot; one launch takes whole chunks up to one
    slot (and 512 chunks)."""
    quantum = 1 << 20
    chunk = min(-(-(1 << 20) // quantum) * quantum, SLOT // quantum * quantum)
    return chunk, min(SLOT, 512 * chunk) // chunk * chunk


def _p2p_chunk(nbytes):
    """policy.h p2p_chunk_bytes: a sixteenth of the message in 4 KiB steps, within [16 KiB, ring slot]."""
    c = -(-nbytes // 16)
    c = (c + 4095) // 4096 * 4096
    return min(max(c, 16 << 10), P2P_RING_SLOT)


def _ceil(a, b):
    return -(-a // b)


def _rand(dev, n, seed):
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    return torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev, generator=gen)


class Region:
    """Operands of `sizes` bytes in one device buffer of random bytes: operand i starts offs[i] bytes
    past a 16-byte boundary, with at least GUARD bytes before and after it."""

    def __init__(self, dev, sizes, offs, seed):
        self.sizes, self.starts, pos = list(sizes), [], GUARD
        for s, o in zip(sizes, offs):
            pos = (pos + 15) // 16 * 16 + o
            self.starts.append(pos)
            pos += s + GUARD
        self.buf = _rand(dev, pos, seed)  # allocations start 512-byte aligned
        self.init = self.buf.clone()

    def view(self, i, dtype=torch.uint8):
        s = self.starts[i]
        return self.buf[s:s + self.sizes[i]].view(dtype)

    def initial(self, i, lo=0, hi=None):
        """Bytes [lo, hi) of operand i as they were before the call."""
        s = self.starts[i]
        return self.init[s + lo:s + (self.sizes[i] if hi is None else hi)]

    def want(self, pieces):
        """The initial buffer with bytes placed at (operand, byte offset in it, bytes)."""
        w = self.init.clone()
        for i, at, data in pieces:
            s = self.starts[i] + at
            w[s:s + data.numel()].copy_(data.to(w.device))
        return w


def _diff(buf, want):
    """None when equal, else where the bytes differ."""
    if torch.equal(buf, want):
        return None
    bad = (buf != want).nonzero().flatten()
    return f"{bad.numel()} bytes differ, first at {bad[0].item()}, last at {bad[-1].item()} of {buf.numel()}"


def _counts(g):
    return [c.launch_count for c in g.comms]


def _delta(g, before):
    return [c.launch_count - b for c, b in zip(g.comms, before)]


def _offsets(rng, k, choices=OFFS):
    return [int(x) for x in rng.choice(choices, k)]


# ---- broadcast ---------------------------------------------------------------------------------

def _sizes(g):
    row = _grid(g) * KTHREADS * 16
    return [1, 15, 16, 17, 4095, row - 16, row + 16, SLOT - 16, SLOT, SLOT + 1, 5 * SLOT // 2 + 7]


MULTI_PIECE = (SLOT + 1, 5 * SLOT // 2 + 7)


def _broadcast(g, root, nbytes, seed, choices=OFFS, dtype=torch.uint8):
    """Broadcast from `root` of `nbytes` at offsets drawn per rank from `choices`: every non-root
    buffer ends up as its initial bytes with the root's operand in place; the root's is unchanged."""
    n = g.world_size
    offs = _offsets(np.random.default_rng(seed), n, choices)
    regs = [Region(g.device(r), [nbytes], [offs[r]], seed * 16 + r) for r in range(n)]
    views = [reg.view(0, dtype) for reg in regs]
    src = regs[root].initial(0)
    wants = [reg.init if r == root else reg.want([(0, 0, src)]) for r, reg in enumerate(regs)]
    before = _counts(g)
    g.run(lambda c, r: c.broadcast(views[r], root))
    ctx = (n, root, nbytes, offs, dtype)
    assert _delta(g, before) == [_ceil(nbytes, SLOT)] * n, ctx
    for r in range(n):
        d = _diff(regs[r].buf, wants[r])
        assert d is None, (ctx, r, d)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_broadcast_byte_for_byte(groups, world):
    """Every root, sizes around the unit, the grid row and the staging slot, per-rank offsets; then
    grids of 1 and 3 CTAs on the sizes of several pieces."""
    g = groups(world)
    for root in range(world):
        for i, nbytes in enumerate(_sizes(g)):
            _broadcast(g, root, nbytes, seed=1000 * world + 20 * root + i)
    for k in (1, 3):
        with _knobs(g, blocks=k):
            for root in range(world):
                for i, nbytes in enumerate(MULTI_PIECE):
                    _broadcast(g, root, nbytes, seed=9000 + 100 * k + 10 * root + i)


def test_broadcast_typed_views(groups):
    """Odd element counts of 8-, 2- and 1-byte types: the count-to-bytes conversion, across pieces."""
    g = groups(3)
    for i, (dtype, count) in enumerate([(torch.float64, (SLOT + 24) // 8 + 1), (torch.float64, 3),
                                        (torch.bfloat16, SLOT // 2 + 1), (torch.bfloat16, 5),
                                        (torch.int8, 3 * SLOT // 2 + 1), (torch.int8, 17)]):
        es = torch.empty((), dtype=dtype).element_size()
        choices = OFFS if es == 1 else (0, 8)
        for root in range(3):
            _broadcast(g, root, count * es, seed=700 + 10 * i + root, choices=choices, dtype=dtype)


@pytest.mark.parametrize("world", [3, 4, 8])
def test_broadcast_nvls_byte_for_byte(groups, world):
    """From 64 KiB at three ranks or more the root stores once through the multicast alias."""
    g = groups(world)
    if not g.has_multicast:
        pytest.skip("no NVLS multicast mapping (ranks share a GPU, or the switch has none)")
    for root in range(world):
        for i, nbytes in enumerate([64 << 10, (64 << 10) + 1, SLOT, SLOT + 1, 5 * SLOT // 2 + 7]):
            _broadcast(g, root, nbytes, seed=8000 + 20 * root + i)


# ---- all-gather --------------------------------------------------------------------------------

def _allgather(g, form, nbytes, seed, choices=OFFS, dtype=torch.uint8, step=SLOT):
    """All-gather of `nbytes` per rank in one of three forms:
      list    -- allgather(outs, x): separate outputs, each at its own offset;
      into    -- allgather_into(out, x): outs[p] = out + p * nbytes;
      inplace -- allgather_into(out, out[r * k:(r + 1) * k]).
    Every output holds every rank's input and nothing else changed; ceil(nbytes / step) launches."""
    n = g.world_size
    es = torch.empty((), dtype=dtype).element_size()
    k = nbytes // es
    rng = np.random.default_rng(seed)
    in_offs = _offsets(rng, n, choices)
    ins = [] if form == "inplace" else [Region(g.device(r), [nbytes], [in_offs[r]], seed * 32 + r) for r in range(n)]
    if form == "list":
        outs = [Region(g.device(r), [nbytes] * n, _offsets(rng, n, choices), seed * 32 + 16 + r) for r in range(n)]
        data = [ins[p].initial(0) for p in range(n)]
        wants = [outs[r].want([(p, 0, data[p]) for p in range(n)]) for r in range(n)]
        args = [([outs[r].view(p, dtype) for p in range(n)], ins[r].view(0, dtype)) for r in range(n)]
    else:
        outs = [Region(g.device(r), [n * nbytes], _offsets(rng, 1, choices), seed * 32 + 16 + r) for r in range(n)]
        if form == "into":
            data = [ins[p].initial(0) for p in range(n)]
            args = [(outs[r].view(0, dtype), ins[r].view(0, dtype)) for r in range(n)]
        else:
            data = [outs[p].initial(0, p * nbytes, (p + 1) * nbytes) for p in range(n)]
            args = [(outs[r].view(0, dtype), outs[r].view(0, dtype)[r * k:(r + 1) * k]) for r in range(n)]
        wants = [outs[r].want([(0, p * nbytes, data[p]) for p in range(n)]) for r in range(n)]
    call = (lambda c, r: c.allgather(*args[r])) if form == "list" else (lambda c, r: c.allgather_into(*args[r]))
    before = _counts(g)
    g.run(call)
    ctx = (n, form, nbytes, dtype, seed)
    assert _delta(g, before) == [_ceil(nbytes, step)] * n, ctx
    for r in range(n):
        d = _diff(outs[r].buf, wants[r])
        assert d is None, (ctx, "output", r, d)
        if ins:
            d = _diff(ins[r].buf, ins[r].init)
            assert d is None, (ctx, "input", r, d)


FORMS = ("list", "into", "inplace")


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_staged_allgather_byte_for_byte(groups, world, form):
    """The staged kernel (below the pull kernel's 4 MiB threshold, or misaligned): sizes around the
    unit, the grid row and the slot, with the input and each output at their own offsets; odd sizes
    put the later outputs of allgather_into off alignment.  Then grids of 1 and 3 CTAs."""
    g = groups(world)
    for i, nbytes in enumerate(_sizes(g)):
        _allgather(g, form, nbytes, seed=2000 * world + 50 * FORMS.index(form) + i)
    for k in (1, 3):
        with _knobs(g, blocks=k):
            for i, nbytes in enumerate(MULTI_PIECE):
                _allgather(g, form, nbytes, seed=30000 + 1000 * world + 100 * k + 10 * FORMS.index(form) + i)


def test_allgather_typed_views(groups):
    g = groups(3)
    cases = [(torch.float64, (SLOT + 24) // 8 + 1), (torch.float64, 3), (torch.bfloat16, SLOT // 2 + 1),
             (torch.bfloat16, 5), (torch.int8, 3 * SLOT // 2 + 1), (torch.int8, 17)]
    for i, (dtype, count) in enumerate(cases):
        es = torch.empty((), dtype=dtype).element_size()
        for form in FORMS:
            _allgather(g, form, count * es, seed=600 + 10 * i + FORMS.index(form),
                       choices=OFFS if es == 1 else (0, 8), dtype=dtype)


def _pull_sizes():
    chunk, max_bytes = _pull_plan()
    return [64 << 10, chunk - 16, chunk, chunk + 16, max_bytes, max_bytes + 16, 5 * max_bytes // 2]


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_pull_allgather_byte_for_byte(groups, world):
    """The pull kernel, taken from 64 KiB per rank: aligned whole-unit sizes around its chunk and
    its per-launch limit, ceil(nbytes / max_bytes) launches; then the smallest grids that run it
    (2 and 3 CTAs), and the threshold at 0 (the staged kernel), which must give the same bytes."""
    g = groups(world)
    _, max_bytes = _pull_plan()
    zeros = (0,)
    with _knobs(g, params=[(N.PARAM_AG_PULL_MIN_BYTES, 64 << 10)]):
        for i, nbytes in enumerate(_pull_sizes()):
            for form in FORMS:
                _allgather(g, form, nbytes, seed=40000 + 100 * world + 10 * i + FORMS.index(form),
                           choices=zeros, step=max_bytes)
        for k in (2, 3):
            with _knobs(g, blocks=k):
                for i, nbytes in enumerate((max_bytes + 16, 5 * max_bytes // 2)):
                    for form in FORMS:
                        _allgather(g, form, nbytes, seed=50000 + 100 * world + 10 * k + 3 * i + FORMS.index(form),
                                   choices=zeros, step=max_bytes)
    with _knobs(g, params=[(N.PARAM_AG_PULL_MIN_BYTES, 0)]):
        for i, nbytes in enumerate((max_bytes + 16, 5 * max_bytes // 2)):
            _allgather(g, "inplace", nbytes, seed=60000 + 100 * world + i, choices=zeros)


@pytest.mark.parametrize("world", [2, 3])
def test_pull_allgather_on_one_cta_runs_the_staged_kernel(groups, world):
    """A grid cap of one CTA leaves the pull kernel no worker: an aligned all-gather that would take
    it must run the staged kernel, which works on any grid, and give the same bytes."""
    g = groups(world)
    _, max_bytes = _pull_plan()
    with _knobs(g, blocks=1, params=[(N.PARAM_AG_PULL_MIN_BYTES, 64 << 10)]):
        for i, nbytes in enumerate((64 << 10, max_bytes + 16, 5 * max_bytes // 2)):
            for form in FORMS:
                _allgather(g, form, nbytes, seed=70000 + 100 * world + 10 * i + FORMS.index(form), choices=(0,))
    with _knobs(g, blocks=1):  # the default threshold: 4 MiB per rank
        _allgather(g, "into", 5 * max_bytes // 2, seed=71000 + world, choices=(0,))


def test_auto_allreduce_on_one_cta_runs_a_kernel_that_fits(groups):
    """ALGO_AUTO at two ranks from 16 MiB picks the pull all-reduce, which needs two CTAs: on a grid
    of one it must take the two-shot kernel instead, bit-exact against the rank-ascending oracle.
    An explicit ALGO_PIPE still refuses, before any launch.  The slot holds the whole message: on a
    smaller one each piece falls below 16 MiB and takes the phase kernels anyway."""
    nbytes = 16 << 20
    g = groups(2, staging=nbytes)
    host = [np.random.default_rng(80 + r).standard_normal(nbytes // 4).astype(np.float32) for r in range(2)]
    want = torch.from_numpy(O.reduce_rank_ascending(host, O.SUM).view(np.uint8))
    regs = [Region(g.device(r), [nbytes], [0], 81 + r) for r in range(2)]
    for reg, h in zip(regs, host):
        reg.view(0).copy_(torch.from_numpy(h.view(np.uint8)))
        reg.init = reg.buf.clone()
    wants = [reg.want([(0, 0, want)]) for reg in regs]
    xs = [reg.view(0, torch.float32) for reg in regs]
    with _knobs(g, blocks=1):
        before = _counts(g)
        with torch.cuda.device(g.devices[0]):
            with pytest.raises(N.B200Error, match="needs at least"):
                g.comms[0].allreduce(xs[0], N.SUM, algo=N.ALGO_PIPE)
        assert _delta(g, before) == [0, 0]
        g.run(lambda c, r: c.allreduce(xs[r], N.SUM))
        assert _delta(g, before) == [1, 1]
    for r in range(2):
        d = _diff(regs[r].buf, wants[r])
        assert d is None, (r, d)


# ---- send / recv -------------------------------------------------------------------------------

P2P_PAIRS = {2: [(0, 1), (1, 0)], 3: [(0, 2), (2, 0)], 4: [(0, 3), (3, 0), (1, 2)]}
P2P_OFFS = (0, 3, 8, 15)
RING_ALL = 16 * P2P_RING_SLOT  # 16 chunks of one ring slot: every ring carries one
P2P_SIZES = [1, 15, (16 << 10) - 1, 16 << 10, (16 << 10) + 1, RING_ALL - 16, RING_ALL + 16,
             INBOX - 16, INBOX + 16, 5 * INBOX // 2]


def _p2p(g, src, dst, sizes, seed, s_offs, r_offs, ldst=()):
    """`src` sends each of `sizes` in order, `dst` receives each into a view of one region: every
    received byte, the guard bytes, the sender's buffer unchanged, one launch per message per side.
    Ranks in `ldst` move their bytes with ld/st (B200_PARAM_P2P_BULK_MIN_CHUNK = 0)."""
    n = g.world_size
    sreg = Region(g.device(src), sizes, s_offs, seed)
    rreg = Region(g.device(dst), sizes, r_offs, seed + 1)
    want = rreg.want([(i, 0, sreg.initial(i)) for i in range(len(sizes))])
    sv = [sreg.view(i) for i in range(len(sizes))]
    rv = [rreg.view(i) for i in range(len(sizes))]

    def f(c, r):
        for i in range(len(sizes)):
            if r == src:
                c.send(sv[i], dst)
            elif r == dst:
                c.recv(rv[i], src)

    before = _counts(g)
    with _knobs(g, params=[(N.PARAM_P2P_BULK_MIN_CHUNK, 0)], ranks=ldst):
        g.run(f)
    ctx = (n, src, dst, sizes, s_offs, r_offs, ldst)
    assert _delta(g, before) == [len(sizes) if r in (src, dst) else 0 for r in range(n)], ctx
    d = _diff(rreg.buf, want)
    assert d is None, (ctx, "received", d)
    d = _diff(sreg.buf, sreg.init)
    assert d is None, (ctx, "sender", d)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_send_recv_byte_for_byte(groups, world):
    """Sizes around the minimum chunk, all 16 rings busy, the inbox of one source and beyond; the
    two sides at offsets chosen independently."""
    g = groups(world)
    for k, (src, dst) in enumerate(P2P_PAIRS[world]):
        rng = np.random.default_rng(100 * world + k)
        for i, nbytes in enumerate(P2P_SIZES):
            assert _p2p_chunk(nbytes) <= P2P_RING_SLOT
            _p2p(g, src, dst, [nbytes], 3000 + 100 * world + 20 * k + i,
                 _offsets(rng, 1, P2P_OFFS), _offsets(rng, 1, P2P_OFFS))


@pytest.mark.parametrize("sender,receiver", [("bulk", "bulk"), ("bulk", "ldst"), ("ldst", "bulk"),
                                             ("ldst", "ldst")])
def test_send_recv_every_mechanism_pairing(groups, sender, receiver):
    """Aligned whole-unit messages with chunks of at least 32 KiB take the bulk-copy unit unless that
    side sets B200_PARAM_P2P_BULK_MIN_CHUNK = 0; the wire is the same either way."""
    g = groups(2)
    ldst = [r for r, m in enumerate((sender, receiver)) if m == "ldst"]
    sizes = [RING_ALL - 16, RING_ALL + 16, INBOX + 16, 5 * INBOX // 2]
    assert all(s % 16 == 0 and _p2p_chunk(s) >= 32 << 10 for s in sizes)
    for i, nbytes in enumerate(sizes):
        _p2p(g, 0, 1, [nbytes], 4000 + 10 * len(ldst) + i, [0], [0], ldst=ldst)
        _p2p(g, 1, 0, [nbytes], 4100 + 10 * len(ldst) + i, [0], [0], ldst=[1 - r for r in ldst])


@pytest.mark.parametrize("world", [2, 4])
def test_send_recv_back_to_back_messages(groups, world):
    """Messages of 1 to 129 chunks on one stream with no host sync between them: each starts its
    rings at the sequence numbers the previous one left."""
    g = groups(world)
    sizes = [(16 << 10) + 1, 1, RING_ALL + 16, 3 * (16 << 10), 15, INBOX + 16, 300_003, 17 * 4096 + 5]
    assert len({_ceil(s, _p2p_chunk(s)) for s in sizes}) >= 6
    for k, (src, dst) in enumerate(P2P_PAIRS[world][:2]):
        rng = np.random.default_rng(5000 + world + k)
        _p2p(g, src, dst, sizes, 5100 + 10 * world + k, _offsets(rng, len(sizes), P2P_OFFS),
             _offsets(rng, len(sizes), P2P_OFFS))


# ---- get ---------------------------------------------------------------------------------------

GET_SIZES = [1, 15, 16, 17, GET_SEG - 16, GET_SEG, GET_SEG + 16, 16 * GET_SEG + 16, (1 << 20) + 5]
GET_DST_OFFS = (0, 1, 8)


def _fill_heap(g, owner, seed):
    """Random bytes over the owner's whole heap; -> (heap view, its initial bytes)."""
    heap = g.comms[owner].heap_view(0, HEAP)
    heap.copy_(_rand(g.device(owner), HEAP, seed))
    return heap, heap.clone()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_get_byte_for_byte(groups, world):
    """Every rank, the owner included, gets each size from heap offsets 0, 1, 15, 16 and the heap's
    end into destinations at offsets 0, 1 and 8: one launch per get on the getter, none on the owner.
    1 MiB + 5 misaligned is more than 32 CTAs x 512 units, so the ld/st kernel loops."""
    g = groups(world)
    owner = world - 1
    heap, snap = _fill_heap(g, owner, seed=90 + world)
    assert (1 << 20) + 5 > GET_LDST_CTAS * KTHREADS * 16
    for getter in range(world):
        for i, nbytes in enumerate(GET_SIZES):
            cases = [(off, doff) for off in (0, 1, 15, 16, HEAP - nbytes) for doff in GET_DST_OFFS]
            reg = Region(g.device(getter), [nbytes] * len(cases), [d for _, d in cases],
                         seed=9000 + 100 * getter + i)
            views = [reg.view(j) for j in range(len(cases))]
            want = reg.want([(j, 0, snap[off:off + nbytes]) for j, (off, _) in enumerate(cases)])

            def f(c, r):
                if r == getter:
                    for v, (off, _) in zip(views, cases):
                        c.get(v, owner, off)

            before = _counts(g)
            g.run(f)
            ctx = (world, owner, getter, nbytes)
            assert _delta(g, before) == [len(cases) if r == getter else 0 for r in range(world)], ctx
            d = _diff(reg.buf, want)
            assert d is None, (ctx, d)
    d = _diff(heap, snap)
    assert d is None, ("owner's heap", d)


def test_get_refuses_a_wrapped_heap_range(groups):
    """An offset near 2**64 wraps offset + nbytes back into the heap; the call must still refuse,
    before any launch.  (At -16 the wrapped read would land in the staging slot that precedes the heap.)"""
    g = groups(2)
    c, dev = g.comms[0], g.device(0)
    dst = _rand(dev, 32, 1)
    init = dst.clone()
    before = c.launch_count
    with torch.cuda.device(dev):
        rc = N.load().b200_get(c._h, dst.data_ptr(), 1, 2**64 - 16, 32, None)
        torch.cuda.synchronize(dev)
    assert rc == N.ERR_INVALID, rc
    assert "outside the" in N.last_error()
    assert c.launch_count == before
    assert torch.equal(dst, init)


def test_comm_get_refuses_a_negative_offset(groups):
    g = groups(2)
    c, dev = g.comms[0], g.device(0)
    dst = _rand(dev, 32, 2)
    init = dst.clone()
    before = c.launch_count
    with torch.cuda.device(dev):
        with pytest.raises(ValueError, match="outside the symmetric heap"):
            c.get(dst, 1, -16)
        torch.cuda.synchronize(dev)
    assert c.launch_count == before
    assert torch.equal(dst, init)


# ---- launch order ------------------------------------------------------------------------------

# device launches (staging-slot parity steps) of each operation in the mixed sequence
SEQ_OPS = ("broadcast", "allgather", "pull", "p2p", "get", "barrier")
SEQ_DEVICE_LAUNCHES = {"broadcast": 3, "allgather": 1, "pull": 2, "p2p": 0, "get": 0, "barrier": 1}


@pytest.mark.parametrize("world", [2, 4])
def test_launch_order_mixed_sequence(groups, world):
    """On each rank's stream with no host sync: a broadcast of 3 pieces, a staged all-gather of one,
    a pull all-gather of two, a send/recv, a get and a barrier; the sequence repeats shifted by one
    each round, so every staging kernel starts on both slot parities.  Everything is checked after."""
    g = groups(world)
    n = world
    _, max_bytes = _pull_plan()
    src, dst, owner = 0, n - 1, n - 1
    b_bytes, a_bytes, p_bytes, s_bytes, get_bytes, get_off = 2 * SLOT + 5, 100_001, max_bytes + 4096, 300_003, 70_001, 5
    assert _ceil(b_bytes, SLOT) == 3 and a_bytes <= SLOT and _ceil(p_bytes, max_bytes) == 2
    heap, snap = _fill_heap(g, owner, seed=95)
    rounds = [SEQ_OPS[k:] + SEQ_OPS[:k] for k in range(len(SEQ_OPS))]
    parity, at = {op: set() for op in ("broadcast", "allgather", "pull")}, 0
    for seq in rounds:
        for op in seq:
            if op in parity:
                parity[op].add(at % 2)
            at += SEQ_DEVICE_LAUNCHES[op]
    assert all(p == {0, 1} for p in parity.values()), parity

    rng = np.random.default_rng(96)
    state = []
    for k in range(len(rounds)):
        root = k % n
        s = {"root": root}
        s["b"] = [Region(g.device(r), [b_bytes], _offsets(rng, 1), 10_000 + 100 * k + r) for r in range(n)]
        s["a_in"] = [Region(g.device(r), [a_bytes], _offsets(rng, 1), 20_000 + 100 * k + r) for r in range(n)]
        s["a_out"] = [Region(g.device(r), [a_bytes] * n, _offsets(rng, n), 30_000 + 100 * k + r) for r in range(n)]
        s["p_in"] = [Region(g.device(r), [p_bytes], [0], 40_000 + 100 * k + r) for r in range(n)]
        s["p_out"] = [Region(g.device(r), [n * p_bytes], [0], 50_000 + 100 * k + r) for r in range(n)]
        s["s"] = Region(g.device(src), [s_bytes], _offsets(rng, 1, P2P_OFFS), 60_000 + k)
        s["d"] = Region(g.device(dst), [s_bytes], _offsets(rng, 1, P2P_OFFS), 61_000 + k)
        s["g"] = [Region(g.device(r), [get_bytes], _offsets(rng, 1), 70_000 + 100 * k + r) for r in range(n)]
        s["views"] = {
            "b": [s["b"][r].view(0) for r in range(n)],
            "a": [([s["a_out"][r].view(p) for p in range(n)], s["a_in"][r].view(0)) for r in range(n)],
            "p": [(s["p_out"][r].view(0), s["p_in"][r].view(0)) for r in range(n)],
            "s": s["s"].view(0), "d": s["d"].view(0), "g": [s["g"][r].view(0) for r in range(n)],
        }
        state.append(s)

    def f(c, r):
        for s, seq in zip(state, rounds):
            v = s["views"]
            for op in seq:
                if op == "broadcast":
                    c.broadcast(v["b"][r], s["root"])
                elif op == "allgather":
                    c.allgather(*v["a"][r])
                elif op == "pull":
                    c.allgather_into(*v["p"][r])
                elif op == "p2p":
                    if r == src:
                        c.send(v["s"], dst)
                    elif r == dst:
                        c.recv(v["d"], src)
                elif op == "get":
                    c.get(v["g"][r], owner, get_off)
                else:
                    c.barrier()

    before = _counts(g)
    with _knobs(g, params=[(N.PARAM_AG_PULL_MIN_BYTES, 64 << 10)]):
        g.run(f)
    per_round = [3 + 1 + 2 + (1 if r in (src, dst) else 0) + 1 + 1 for r in range(n)]
    assert _delta(g, before) == [len(rounds) * x for x in per_round]

    for k, s in enumerate(state):
        root = s["root"]
        for r in range(n):
            checks = [
                ("broadcast", s["b"][r], s["b"][r].init if r == root else s["b"][r].want([(0, 0, s["b"][root].initial(0))])),
                ("allgather in", s["a_in"][r], s["a_in"][r].init),
                ("allgather out", s["a_out"][r], s["a_out"][r].want([(p, 0, s["a_in"][p].initial(0)) for p in range(n)])),
                ("pull in", s["p_in"][r], s["p_in"][r].init),
                ("pull out", s["p_out"][r], s["p_out"][r].want([(0, p * p_bytes, s["p_in"][p].initial(0)) for p in range(n)])),
                ("get", s["g"][r], s["g"][r].want([(0, 0, snap[get_off:get_off + get_bytes])])),
            ]
            for what, reg, want in checks:
                d = _diff(reg.buf, want)
                assert d is None, (k, r, what, d)
        d = _diff(s["s"].buf, s["s"].init)
        assert d is None, (k, "sender", d)
        d = _diff(s["d"].buf, s["d"].want([(0, 0, s["s"].initial(0))]))
        assert d is None, (k, "receiver", d)
    d = _diff(heap, snap)
    assert d is None, ("owner's heap", d)
