"""The fused sharded gradient reduce-scatter (b200_grad_reducescatter) against the DDP oracle.

Every case asserts that rank r's shard is bit-identical to elements [r*count, (r+1)*count) of
``O.ddp_grad_sync`` and within the float64 bound of the fused-gradient matrix, that guard bytes
around the output and the gradient are unchanged, that an out-of-place gradient is untouched and
that the call took one launch per staging piece.  Runs with all ranks on one GPU and with one GPU
per rank; the kernel has no switch variant, so it is bit exact in both.
"""
import numpy as np
import pytest
import torch

from oracle import collective_oracle as O
from tests.test_gpu_reduction_matrix import WIRES, Operand, _grad_check, _grad_specials, same_bits

pytestmark = pytest.mark.gpu

SLOT = 2 << 20  # the smallest staging slot (the VMM allocation granularity), so pieces stay cheap
UNIT_ROW = 512  # 16-byte wire units one CTA covers per step (kThreads)


def _piece_elems(world, wire):
    """Shard elements per launch (grad_rs_piece_elems in policy.h)."""
    wes = WIRES[wire][1].itemsize
    return ((SLOT // (world * 16)) * (16 // wes)) & ~7


def _launches(world, wire, count):
    if world == 1:
        return 1
    p = _piece_elems(world, wire)
    return (count + p - 1) // p


@pytest.fixture(scope="module")
def groups(native_lib):
    from ray_b200.testing import LocalGroup

    cache = {}

    def get(n, multicast=True):
        if (n, multicast) not in cache:
            cache[n, multicast] = LocalGroup(n, timeout_ms=20000, staging_bytes=SLOT, inbox_bytes=1 << 20,
                                             enable_multicast=multicast)
        return cache[n, multicast]

    yield get
    for g in cache.values():
        g.destroy()


def _inputs(wire, world, count, scale, seed):
    """Per-rank flat gradients of world * count elements.  At scale 1.0 every stripe starts with the
    special values of the fused-gradient matrix (±0, subnormals, ±inf, NaN, f16 overflow, ties)."""
    rng = np.random.default_rng(seed)
    if scale != 1.0:
        return [rng.standard_normal(world * count).astype(np.float32) for _ in range(world)]
    stripes = [_grad_specials(wire, world, count, rng) for _ in range(world)]  # stripes[q][r]
    return [np.concatenate([stripes[q][r] for q in range(world)]).astype(np.float32) for r in range(world)]


def _run_rs(g, wire, grads, count, scale, offset, in_place=False):
    """One grad_reducescatter over guarded operands; returns the per-rank shards after checking
    guards, untouched inputs and the launch count."""
    world = g.world_size
    tdt = WIRES[wire][0]
    bufs = [Operand(grads[r], "float32", g.device(r), offset, seed=r) for r in range(world)]
    outs = None if in_place else [Operand(np.zeros(count, np.float32), "float32", g.device(r), offset, seed=40 + r)
                                  for r in range(world)]
    before = [c.launch_count for c in g.comms]
    if in_place:
        g.run(lambda c, r: c.grad_reducescatter(bufs[r].view[r * count:(r + 1) * count], bufs[r].view, scale, tdt))
    else:
        g.run(lambda c, r: c.grad_reducescatter(outs[r].view, bufs[r].view, scale, tdt))
    what = (world, wire, count, offset, scale, in_place)
    assert [c.launch_count - b for c, b in zip(g.comms, before)] == [_launches(world, wire, count)] * world, what
    shards = []
    for r in range(world):
        if in_place:
            full, guards = bufs[r].read()
            assert guards, what + (r,)
            # the other stripes are inputs: only the own stripe may change
            rest = np.concatenate([full[:r * count], full[(r + 1) * count:]])
            mine = np.concatenate([grads[r][:r * count], grads[r][(r + 1) * count:]])
            assert np.array_equal(rest.view(np.uint32), mine.view(np.uint32)), what + (r,)
            shards.append(full[r * count:(r + 1) * count].copy())
        else:
            got, guards = outs[r].read()
            assert guards, what + (r,)
            assert bufs[r].unchanged(), ("out-of-place gradient changed",) + what + (r,)
            shards.append(got)
    return shards


def _counts(world, wire):
    E = 4 if wire == "f32" else 8
    row = UNIT_ROW * E
    return (1, 7, 8, 9, E - 1, E + 1, row - 1, row + 1, 2 * _piece_elems(world, wire) + 5)


@pytest.mark.parametrize("wire", list(WIRES))
@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_grad_reducescatter_matrix(groups, world, wire):
    """Wires x worlds 1-8 x shard sizes 1, 7, 8, 9, one wire unit ± 1, one CTA step ± 1 and three
    staging pieces x base offsets 0 and 1 element x scales 1/n, 1.0 and 0.1 (special values at 1.0)."""
    g = groups(world)
    for count in _counts(world, wire):
        assert world == 1 or count < 3 * _piece_elems(world, wire)
        for offset in (0, 1):
            for scale in (1.0 / world, 1.0, 0.1):
                grads = _inputs(wire, world, count, scale, seed=count * 10 + offset + world)
                shards = _run_rs(g, wire, grads, count, scale, offset)
                want_all = O.ddp_grad_sync(grads, wire, scale=scale)[0]
                for r in range(world):
                    what = (world, wire, count, offset, scale, r)
                    sl = slice(r * count, (r + 1) * count)
                    assert same_bits(shards[r], want_all[sl]), what
                    _grad_check(shards[r], [x[sl] for x in grads], scale, wire, False, what)
                    if scale == 1.0 and count >= 12:
                        s = shards[r]
                        assert s[3] == np.inf and s[5] == -np.inf and np.isnan(s[6]), what
                        assert np.isinf(s[4]) == (wire == "f16"), what  # 1e5 overflows f16 only


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_grad_reducescatter_in_place_matches_out_of_place(groups, world):
    """``out`` = the rank's own stripe of ``grad`` gives the same bits, and only that stripe changes."""
    g = groups(world)
    for wire in WIRES:
        for count in (9, UNIT_ROW * 8 + 3, 2 * _piece_elems(world, wire) + 5):
            for offset in (0, 1):
                scale = 1.0 / world
                grads = _inputs(wire, world, count, scale, seed=count + offset + 7 * world)
                a = _run_rs(g, wire, grads, count, scale, offset)
                b = _run_rs(g, wire, grads, count, scale, offset, in_place=True)
                for r in range(world):
                    assert same_bits(a[r], b[r]), (world, wire, count, offset, r)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_grad_reducescatter_shards_concatenate_to_the_grad_allreduce_bucket(groups, world):
    """Without the multicast mapping b200_grad_allreduce reduces on the peer path too: the shards of
    all ranks, concatenated, are bit for bit the bucket it leaves behind."""
    g = groups(world, multicast=False)
    for wire in WIRES:
        tdt = WIRES[wire][0]
        for count in (1, 257, UNIT_ROW * 8 + 3, 2 * _piece_elems(world, wire) + 5):
            grads = _inputs(wire, world, count, 1.0, seed=count + world)
            shards = _run_rs(g, wire, grads, count, 0.1, 0)
            bucket = [torch.from_numpy(grads[r].copy()).to(g.device(r)) for r in range(world)]
            g.run(lambda c, r: c.grad_allreduce(bucket[r], 0.1, tdt))
            want = bucket[0].cpu().numpy()
            assert same_bits(np.concatenate(shards), want), (world, wire, count)


def test_grad_reducescatter_rejects_invalid_arguments_without_launching(groups):
    """The entry point's checks, through the raw binding: status, error text, no launch."""
    from ray_b200 import _native as N

    lib = N.load()
    g1, g2 = groups(1), groups(2, multicast=False)
    h1, h = g1.comms[0]._h, g2.comms[0]._h
    x = torch.zeros(64, device=g2.device(0))
    y = torch.zeros(32, device=g2.device(0))
    x1 = torch.zeros(64, device=g1.device(0))
    X, Y, X1 = x.data_ptr(), y.data_ptr(), x1.data_ptr()
    F32, S, BAD = N.F32, None, 99
    INV, UNS, OK = N.ERR_INVALID, N.ERR_UNSUPPORTED, N.OK
    cases = [
        ("null comm", lambda: lib.b200_grad_reducescatter(None, X, Y, 32, 1.0, F32, S), INV, "null communicator"),
        ("wire dtype", lambda: lib.b200_grad_reducescatter(h, X, Y, 32, 1.0, BAD, S), UNS,
         f"wire dtype must be f32, bf16 or f16 (got {BAD})"),
        ("integer wire dtype", lambda: lib.b200_grad_reducescatter(h, X, Y, 32, 1.0, N.I32, S), UNS,
         f"(got {N.I32})"),
        ("wire dtype before zero count", lambda: lib.b200_grad_reducescatter(h, None, None, 0, 1.0, BAD, S), UNS,
         "wire dtype"),
        ("zero count", lambda: lib.b200_grad_reducescatter(h, None, None, 0, 1.0, F32, S), OK, None),
        ("null grad", lambda: lib.b200_grad_reducescatter(h, None, Y, 32, 1.0, F32, S), INV, "null gradient pointer"),
        ("null out", lambda: lib.b200_grad_reducescatter(h, X, None, 32, 1.0, F32, S), INV, "null output pointer"),
        ("partial overlap", lambda: lib.b200_grad_reducescatter(h, X, X + 16, 32, 1.0, F32, S), INV,
         "output overlaps the gradient"),
        ("overlap from below", lambda: lib.b200_grad_reducescatter(h, X + 64, X + 32, 16, 1.0, F32, S), INV,
         "output overlaps the gradient"),
        ("another rank's stripe", lambda: lib.b200_grad_reducescatter(h, X, X + 32 * 4, 32, 1.0, F32, S), INV,
         "output overlaps the gradient"),
        ("world 1 partial overlap", lambda: lib.b200_grad_reducescatter(h1, X1, X1 + 4, 32, 1.0, F32, S), INV,
         "output overlaps the gradient"),
    ]
    comms = g1.comms + g2.comms
    for what, call, status, text in cases:
        before = [c.launch_count for c in comms]
        got = call()
        assert got == status, (what, got, N.last_error())
        if text is not None:
            assert text in N.last_error(), (what, N.last_error())
        assert [c.launch_count for c in comms] == before, what


def test_grad_reducescatter_python_checks(groups):
    g = groups(2)
    c = g.comms[0]
    dev = g.device(0)
    with pytest.raises(RuntimeError, match="float32"):
        c.grad_reducescatter(torch.zeros(4, device=dev), torch.zeros(8, device=dev, dtype=torch.bfloat16), 1.0)
    with pytest.raises(RuntimeError, match="world_size slices"):
        c.grad_reducescatter(torch.zeros(4, device=dev), torch.zeros(9, device=dev), 1.0)
    with pytest.raises(RuntimeError, match="contiguous"):
        c.grad_reducescatter(torch.zeros(4, device=dev), torch.zeros(16, device=dev)[::2], 1.0)
