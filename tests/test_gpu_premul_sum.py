"""PREMUL_SUM (c10d's ``_make_nccl_premul_sum``) on every reducing entry, through ``PremulSum``.

The property checked everywhere is exact: PREMUL_SUM(f) on x is bit-identical to SUM on
y = round_T(x * f) (computed on the device in a separate pass) through the same entry and algorithm,
with the same launch count; on the peer paths the result is also the rank-ascending oracle of y, and
on NVLS the replicas agree bit for bit.  A float factor is rounded to the operand's dtype first, as
ProcessGroupNCCL does.
"""
import ctypes

import pytest
import torch

from oracle import collective_oracle as O
from ray_b200 import _native as N
from ray_b200.comm import PremulSum
from tests.test_gpu_reduction_matrix import DTYPES, check_result, same_bits

pytestmark = pytest.mark.gpu

STAGING = 2 << 20  # the smallest staging slot: a few MiB span several pieces and windows
WORLDS = [1, 2, 3, 4, 8]
FLOATS = ("float16", "bfloat16", "float32", "float64")
NVLS_OK = ("float16", "bfloat16", "float32")


@pytest.fixture(scope="module")
def groups(native_lib):
    from ray_b200.testing import LocalGroup

    cache = {}

    def get(n, heap=False):
        if (n, heap) not in cache:
            cache[n, heap] = LocalGroup(n, timeout_ms=20000, staging_bytes=STAGING, inbox_bytes=1 << 20,
                                        heap_bytes=(16 << 20) if heap else 0)
        return cache[n, heap]

    yield get
    for g in cache.values():
        g.destroy()


def factors(n):
    """(name, factor spec): a float, or ("device", value) for a one-element CUDA tensor."""
    return [("0.25", 0.25), ("1/3", 1 / 3), ("1/world", 1 / n), ("-2", -2.0), ("device", ("device", 0.75))]


def make_op(spec, dtype, device):
    if isinstance(spec, tuple):
        return PremulSum(torch.tensor([spec[1]], dtype=dtype, device=device))
    return PremulSum(spec)


def prescale(x, spec, dtype):
    """y = round_T(x * f) on the device: fp32 product for f32 / f16 / bf16, double for f64."""
    f = torch.tensor(spec[1] if isinstance(spec, tuple) else spec, dtype=dtype, device=x.device)
    if dtype == torch.float64:
        return x * f
    return (x.float() * f.float()).to(dtype)


def to_np(t, dname):
    return t.detach().contiguous().cpu().view(torch.uint8).numpy().view(DTYPES[dname][1])


def rand(dname, numel, seed, device):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(numel, generator=g, dtype=torch.float64) * 3
    return x.to(DTYPES[dname][0]).to(device)


def oracle(got, ys, dname, what):
    """check_result on the first and last 3000 elements: the exact reference of f64 is computed per
    element in Python, and the reduction is element-wise."""
    k = min(3000, got.numel())
    for sl in (slice(0, k), slice(got.numel() - k, got.numel())):
        check_result(to_np(got[sl], dname), [to_np(y[sl], dname) for y in ys], O.SUM, dname, what)


def launches(g, fn):
    before = [c.launch_count for c in g.comms]
    g.run(fn)
    return [c.launch_count - b for c, b in zip(g.comms, before)]


def same_launches(k_p, k_s, what):
    """SUM's launches; at world 1, where SUM copies or does nothing, one scale kernel per call."""
    assert k_p == (k_s if len(k_s) > 1 else [1]), (what, k_p, k_s)


def algos(g, nbytes):
    out = [N.ALGO_AUTO, N.ALGO_ONESHOT, N.ALGO_TWOSHOT]
    if nbytes <= 32 << 10:
        out.append(N.ALGO_LL)
    return out


# ---- all-reduce ---------------------------------------------------------------------------------

@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dname", FLOATS)
def test_allreduce_bit_identical_to_sum_on_prescaled(groups, world, dname):
    g = groups(world)
    dt = DTYPES[dname][0]
    for numel in (1001, (5 << 20) // DTYPES[dname][1].itemsize + 3):  # one LL-size message, one of 3 pieces
        xs = [rand(dname, numel, 10 * r + numel, g.device(r)) for r in range(world)]
        names = algos(g, numel * xs[0].element_size())
        nvls = g.has_multicast and dname in NVLS_OK
        if nvls:
            names.append(N.ALGO_NVLS)
        for fname, spec in factors(world):
            ys = [prescale(x, spec, dt) for x in xs]
            ops = [make_op(spec, dt, g.device(r)) for r in range(world)]
            for algo in names:
                what = (world, dname, numel, fname, algo)
                got = [torch.empty_like(x) for x in xs]
                want = [y.clone() for y in ys]
                k_p = launches(g, lambda c, r: c.allreduce(xs[r], ops[r], out=got[r], algo=algo))
                k_s = launches(g, lambda c, r: c.allreduce(want[r], N.SUM, algo=algo))
                same_launches(k_p, k_s, what)
                for r in range(world):
                    assert torch.equal(got[r].view(torch.uint8), want[r].view(torch.uint8)), (what, r)
                if world == 1:
                    continue
                if algo == N.ALGO_NVLS:
                    for r in range(1, world):
                        assert torch.equal(got[r].view(torch.uint8), got[0].view(torch.uint8)), (what, r)
                elif algo != N.ALGO_AUTO or not nvls:
                    oracle(got[0], ys, dname, what)
            # in place: same bits again
            inp = [x.clone() for x in xs]
            g.run(lambda c, r: c.allreduce(inp[r], ops[r]))
            want = [y.clone() for y in ys]
            g.run(lambda c, r: c.allreduce(want[r], N.SUM))
            for r in range(world):
                assert torch.equal(inp[r].view(torch.uint8), want[r].view(torch.uint8)), (world, dname, fname, r)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_allreduce_multi_bit_identical(groups, world):
    g = groups(world)
    for dname in FLOATS:
        dt = DTYPES[dname][0]
        sizes = [1, 7, 4097, 100003, 0, 3]
        for fname, spec in factors(world):
            xs = [[rand(dname, s, 100 * r + i, g.device(r)) for i, s in enumerate(sizes)] for r in range(world)]
            ys = [[prescale(t, spec, dt) for t in lst] for lst in xs]
            ops = [make_op(spec, dt, g.device(r)) for r in range(world)]
            k_p = launches(g, lambda c, r: c.allreduce_multi(xs[r], ops[r]))
            k_s = launches(g, lambda c, r: c.allreduce_multi(ys[r], N.SUM))
            assert k_p == k_s, (world, dname, fname)
            for r in range(world):
                for a, b in zip(xs[r], ys[r]):
                    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), (world, dname, fname, r)


def test_auto_above_the_pipe_threshold_runs_twoshot(groups):
    """With the pipelined kernels enabled from 1 MiB, SUM's AUTO choice for an aligned 3 MiB message
    is PIPE; PREMUL_SUM runs the two-shot kernel instead, with its launches and its bits."""
    g = groups(2)
    for c in g.comms:
        c.set_param(N.PARAM_PIPE_MIN_BYTES, 1 << 20)
    try:
        for dname in FLOATS:
            dt = DTYPES[dname][0]
            numel = (3 << 20) // DTYPES[dname][1].itemsize
            xs = [rand(dname, numel, r, g.device(r)) for r in range(2)]
            ys = [prescale(x, 1 / 3, dt) for x in xs]
            got = [x.clone() for x in xs]
            k_p = launches(g, lambda c, r: c.allreduce(got[r], PremulSum(1 / 3)))
            k_s = launches(g, lambda c, r: c.allreduce(ys[r], N.SUM, algo=N.ALGO_TWOSHOT))
            assert k_p == k_s, dname
            for r in range(2):
                assert torch.equal(got[r].view(torch.uint8), ys[r].view(torch.uint8)), (dname, r)
            oracle(got[0], [prescale(x, 1 / 3, dt) for x in xs], dname, dname)
    finally:
        for c in g.comms:
            c.set_param(N.PARAM_PIPE_MIN_BYTES, -1)


@pytest.mark.parametrize("world", [2, 3])
def test_symmetric_heap_operand_is_staged(groups, world):
    """SUM reduces a symmetric-heap operand in place with no staging (one launch for 6 MiB);
    PREMUL_SUM stages it like an ordinary tensor: explicit two-shot SUM's launches and bits."""
    g = groups(world, heap=True)
    numel = (6 << 20) // 4
    for c in g.comms:
        c.symm_reset()
    heap = [c.symm_empty(numel, torch.float32) for c in g.comms]
    xs = [rand("float32", numel, r, g.device(r)) for r in range(world)]
    for h, x in zip(heap, xs):
        h.copy_(x)
    ys = [prescale(x, -2.0, torch.float32) for x in xs]
    ref = [y.clone() for y in ys]
    twoshot = launches(g, lambda c, r: c.allreduce(ref[r], N.SUM, algo=N.ALGO_TWOSHOT))
    got = launches(g, lambda c, r: c.allreduce(heap[r], PremulSum(-2.0)))
    assert got == twoshot
    for r in range(world):
        assert torch.equal(heap[r], ref[r]), r
    for h, y in zip(heap, ys):
        h.copy_(y)
    assert launches(g, lambda c, r: c.allreduce(heap[r], N.SUM)) == [1] * world  # SUM: zero-copy
    for r in range(world):
        assert torch.equal(heap[r], ref[r]), r


# ---- reduce and reduce-scatter ------------------------------------------------------------------

@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dname", FLOATS)
def test_reduce_at_every_root(groups, world, dname):
    g = groups(world)
    dt = DTYPES[dname][0]
    numel = (3 << 20) // DTYPES[dname][1].itemsize + 5
    for fname, spec in (("1/3", 1 / 3), ("-2", -2.0), ("device", ("device", 0.75))):
        xs = [rand(dname, numel, 7 * r + 1, g.device(r)) for r in range(world)]
        ys = [prescale(x, spec, dt) for x in xs]
        ops = [make_op(spec, dt, g.device(r)) for r in range(world)]
        for root in range(world):
            got, want = [x.clone() for x in xs], [y.clone() for y in ys]
            k_p = launches(g, lambda c, r: c.reduce(got[r], root, ops[r]))
            k_s = launches(g, lambda c, r: c.reduce(want[r], root, N.SUM))
            same_launches(k_p, k_s, (dname, fname, root))
            for r in range(world):
                # root: the bits of SUM on y; every other rank: its buffer untouched
                expect = want[r] if r == root else xs[r]
                assert torch.equal(got[r].view(torch.uint8), expect.view(torch.uint8)), (dname, fname, root, r)
            if world > 1:
                oracle(got[root], ys, dname, (fname, root))


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dname", FLOATS)
def test_reducescatter_forms(groups, world, dname):
    """Tensor, flat, uneven and list reduce-scatter: bits of SUM on y, launches of SUM, the oracle."""
    g = groups(world)
    dt = DTYPES[dname][0]
    es = DTYPES[dname][1].itemsize
    m = (1 << 20) // es + 3  # per-rank part: a window of the 2 MiB slot is smaller from 3 ranks on
    for fname, spec in factors(world):
        ops = [make_op(spec, dt, g.device(r)) for r in range(world)]
        flat = [rand(dname, m * world, 3 * r + 2, g.device(r)) for r in range(world)]
        yflat = [prescale(x, spec, dt) for x in flat]
        counts = [m + 17 * q if q % 2 else max(0, m // 3 - q) for q in range(world)]
        parts = [[rand(dname, counts[q], 50 * r + q, g.device(r)) for q in range(world)] for r in range(world)]
        yparts = [[prescale(t, spec, dt) for t in lst] for lst in parts]
        cases = {
            "tensor": (lambda c, r, o, op: c.reducescatter(o[r], list(flat[r].split(m)), op),
                       lambda c, r, o: c.reducescatter(o[r], list(yflat[r].split(m)), N.SUM), [m] * world),
            "flat": (lambda c, r, o, op: c.reducescatter_from(o[r], flat[r], op),
                     lambda c, r, o: c.reducescatter_from(o[r], yflat[r], N.SUM), [m] * world),
            "uneven": (lambda c, r, o, op: c.reducescatterv(o[r], parts[r], op),
                       lambda c, r, o: c.reducescatterv(o[r], yparts[r], N.SUM), counts),
            "list": (lambda c, r, o, op: c.reducescatter_from_multi([o[r]], [flat[r]], op),
                     lambda c, r, o: c.reducescatter_from_multi([o[r]], [yflat[r]], N.SUM), [m] * world),
        }
        for form, (run_p, run_s, outc) in cases.items():
            what = (world, dname, fname, form)
            got = [torch.empty(outc[r], dtype=dt, device=g.device(r)) for r in range(world)]
            want = [torch.empty(outc[r], dtype=dt, device=g.device(r)) for r in range(world)]
            k_p = launches(g, lambda c, r: run_p(c, r, got, ops[r]))
            k_s = launches(g, lambda c, r: run_s(c, r, want))
            same_launches(k_p, k_s, what)
            for r in range(world):
                assert torch.equal(got[r].view(torch.uint8), want[r].view(torch.uint8)), (what, r)
            if world > 1:
                r = world - 1
                if form == "uneven":
                    ins = [yparts[q][r] for q in range(world)]
                else:
                    ins = [yflat[q][r * m:(r + 1) * m] for q in range(world)]
                oracle(got[r], ins, dname, what)


# ---- world 1 ------------------------------------------------------------------------------------

@pytest.mark.parametrize("dname", FLOATS)
def test_world1_writes_the_prescaled_input(groups, dname):
    """World 1 is not the identity: every entry writes y, in place or not, at any alignment."""
    g = groups(1)
    dt = DTYPES[dname][0]
    dev = g.device(0)
    for numel in (1, 13, 70001):
        for off_in, off_out in ((0, 0), (1, 0), (0, 3), (5, 2)):
            src = rand(dname, numel + 8, numel + off_in, dev)
            x = src[off_in:off_in + numel]
            y = prescale(x, 1 / 3, dt)
            out = torch.full((numel + 8,), 7, dtype=dt, device=dev)[off_out:off_out + numel]
            k = launches(g, lambda c, r: c.allreduce(x, PremulSum(1 / 3), out=out))
            assert k == [1] and torch.equal(out, y) and torch.equal(x, src[off_in:off_in + numel])
            for call in (lambda c, t: c.allreduce(t, PremulSum(1 / 3)),
                         lambda c, t: c.reduce(t, 0, PremulSum(1 / 3)),
                         lambda c, t: c.allreduce_multi([t], PremulSum(1 / 3)),
                         lambda c, t: c.reducescatter(t, [t], PremulSum(1 / 3)),
                         lambda c, t: c.reducescatterv(t, [t], PremulSum(1 / 3)),
                         lambda c, t: c.reducescatter_multi([t], [[t]], PremulSum(1 / 3))):
                t = x.clone()
                g.run(lambda c, r: call(c, t))
                assert torch.equal(t.view(torch.uint8), y.view(torch.uint8)), (dname, numel, off_in)
            o = torch.empty_like(x)
            g.run(lambda c, r: c.reducescatter(o, [x], PremulSum(1 / 3)))
            assert torch.equal(o, y)


# ---- CUDA graph ---------------------------------------------------------------------------------

def test_cuda_graph_reads_the_device_factor_at_replay(groups):
    n = 3
    g = groups(n)
    numel = 300001
    fs = [torch.tensor([0.5], dtype=torch.float32, device=g.device(r)) for r in range(n)]
    xs = [rand("float32", numel * n, r, g.device(r)) for r in range(n)]
    ar = [torch.empty(numel * n, dtype=torch.float32, device=g.device(r)) for r in range(n)]
    rs = [torch.empty(numel, dtype=torch.float32, device=g.device(r)) for r in range(n)]

    def f(c, r):
        c.allreduce(xs[r], PremulSum(fs[r]), out=ar[r])
        c.reducescatter_from(rs[r], xs[r], PremulSum(fs[r]))

    g.run(f)
    graphs = []
    for r, c in enumerate(g.comms):
        torch.cuda.set_device(g.devices[r])
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=g.streams[r]):
            f(c, r)
        graphs.append(gr)
    for value in (0.25, -3.0):
        for t in fs:
            t.fill_(value)
        for d in set(g.devices):
            torch.cuda.synchronize(d)
        for r in range(n):
            torch.cuda.set_device(g.devices[r])
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        g.synchronize()
        ys = [to_np(prescale(x, value, torch.float32), "float32") for x in xs]
        want = O.reduce_rank_ascending(ys, O.SUM)
        for r in range(n):
            assert same_bits(to_np(ar[r], "float32"), want), (value, r)
            assert same_bits(to_np(rs[r], "float32"), want[r * numel:(r + 1) * numel]), (value, r)


# ---- refusals and the other ops -----------------------------------------------------------------

def test_refusals_launch_nothing(groups, native_lib):
    g = groups(2)
    c0 = g.comms[0]
    dev = g.device(0)
    x = torch.ones(1000, device=dev)
    before = c0.launch_count
    for t in (torch.ones(10, dtype=torch.int32, device=dev), torch.ones(10, dtype=torch.bool, device=dev)):
        with pytest.raises(RuntimeError, match="PREMUL_SUM"):
            c0.allreduce(t, PremulSum(0.5))
        with pytest.raises(RuntimeError, match="PREMUL_SUM"):
            c0.reduce(t, 0, PremulSum(0.5))
    with pytest.raises(N.B200Error) as e:
        c0.allreduce(x, PremulSum(0.5), algo=N.ALGO_PIPE)
    assert e.value.status == N.ERR_UNSUPPORTED
    with pytest.raises(RuntimeError, match="factor"):  # a device factor of another dtype
        c0.allreduce(x, PremulSum(torch.ones(1, dtype=torch.float64, device=dev)))
    with pytest.raises(RuntimeError, match="factor"):  # ... or size
        PremulSum(torch.ones(2, device=dev))
    h, lib = c0._h, native_lib
    op = ctypes.c_int()
    one = ctypes.c_float(0.5)
    assert lib.b200_op_create_premul(h, ctypes.byref(one), N.I32, N.PREMUL_HOST, ctypes.byref(op)) == N.ERR_UNSUPPORTED
    assert lib.b200_op_create_premul(h, ctypes.byref(one), N.F32, N.PREMUL_HOST, ctypes.byref(op)) == N.OK
    assert not 0 <= op.value < 5
    y = torch.ones(1000, dtype=torch.float16, device=dev)
    assert lib.b200_allreduce(h, y.data_ptr(), y.data_ptr(), 1000, N.F16, op.value, 0, None) == N.ERR_INVALID
    assert lib.b200_op_destroy(h, op.value) == N.OK
    assert lib.b200_allreduce(h, x.data_ptr(), x.data_ptr(), 1000, N.F32, op.value, 0, None) == N.ERR_UNSUPPORTED
    assert "unsupported reduce op" in N.last_error()
    for never in (5, 0x100 + 63, -1, 0x7fff):
        assert lib.b200_reduce(h, x.data_ptr(), 1000, N.F32, never, 0, None) == N.ERR_UNSUPPORTED
    assert lib.b200_op_destroy(h, op.value) == N.ERR_INVALID
    torch.cuda.synchronize(dev)
    assert c0.launch_count == before


def test_premul_interleaved_with_every_op(groups):
    """Premul and plain calls alternate on one communicator; the plain ops still match the oracle."""
    n = 4
    g = groups(n)
    numel = 200003
    xs = [rand("float32", numel, r, g.device(r)) for r in range(n)]
    for op, oname in ((N.SUM, O.SUM), (N.PROD, O.PRODUCT), (N.MIN, O.MIN), (N.MAX, O.MAX), (N.AVG, O.AVG)):
        got_p = [torch.empty_like(x) for x in xs]
        got = [torch.empty_like(x) for x in xs]

        def f(c, r):
            c.allreduce(xs[r], PremulSum(0.25), out=got_p[r])
            c.allreduce(xs[r], op, out=got[r])

        g.run(f)
        want = O.reduce_rank_ascending([to_np(x, "float32") for x in xs], oname)
        want_p = O.reduce_rank_ascending([to_np(prescale(x, 0.25, torch.float32), "float32") for x in xs], O.SUM)
        for r in range(n):
            assert same_bits(to_np(got[r], "float32"), want), (op, r)
            assert same_bits(to_np(got_p[r], "float32"), want_p), (op, r)
