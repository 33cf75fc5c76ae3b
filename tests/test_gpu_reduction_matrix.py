"""Every reducing kernel against the rank-ascending oracle and the exact reference (oracle/exact.py),
across dtype x op x world x size x alignment x grid.

What every case asserts:
  * bit-exact against ``O.reduce_rank_ascending`` wherever DESIGN.md §2 promises it (integers,
    MIN/MAX, fp32/fp64 on the peer-load kernels, fp16/bf16 with fp32 accumulation); NaN compares as
    NaN whatever its bit pattern;
  * floating-point results within the explicit error bound of the exact reference
    (``E.error_bound``: (n-1)·u·Σ|x| for SUM/AVG plus the output rounding, a relative bound for PROD);
  * replicas agree bit for bit;
  * guard bytes on both sides of every operand keep their values, and out-of-place inputs are
    left untouched.

Runs with all ranks on one GPU (the grid is then capped at (SMs-4)/n CTAs per rank) and with one
GPU per rank, where the NVLS cases run as well.
"""
import ml_dtypes
import numpy as np
import pytest
import torch

from oracle import collective_oracle as O
from oracle import exact as E

pytestmark = pytest.mark.gpu

BF16 = O.bfloat16
DTYPES = {  # name -> (torch dtype, numpy dtype)
    "uint8": (torch.uint8, np.dtype(np.uint8)), "int8": (torch.int8, np.dtype(np.int8)),
    "int32": (torch.int32, np.dtype(np.int32)), "uint32": (torch.uint32, np.dtype(np.uint32)),
    "int64": (torch.int64, np.dtype(np.int64)), "uint64": (torch.uint64, np.dtype(np.uint64)),
    "float16": (torch.float16, np.dtype(np.float16)), "bfloat16": (torch.bfloat16, BF16),
    "float32": (torch.float32, np.dtype(np.float32)), "float64": (torch.float64, np.dtype(np.float64)),
}
OPS = {"SUM": O.SUM, "PROD": O.PRODUCT, "MIN": O.MIN, "MAX": O.MAX, "AVG": O.AVG}
WORLDS = [2, 3, 4, 8]
HALF = ("float16", "bfloat16")
NVLS_DTYPES = ("float32", "float16", "bfloat16")
# staging slot of the small-slot groups, so that messages split into pieces cheaply: the library
# rounds the slot up to 2 MiB (the VMM allocation granularity), so this is the smallest there is
SMALL_SLOT = 2 << 20
STAGING = 8 << 20  # staging slot of the other groups
UNITS_PER_ROW = 512   # 16-byte units one rank owns in a two-shot row (kThreads)
BIG_DTYPES = ("uint8", "bfloat16", "float32")  # the messages of several staging pieces: 1-, 2-, 4-byte


@pytest.fixture(scope="module")
def groups(native_lib):
    from ray_b200.testing import LocalGroup

    cache = {}

    def get(n, small=False):
        if (n, small) not in cache:
            cache[n, small] = LocalGroup(n, timeout_ms=20000, staging_bytes=SMALL_SLOT if small else STAGING,
                                         inbox_bytes=1 << 20)
        return cache[n, small]

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


class _Forced:
    """set_blocks(k) on every rank for the duration of a with-block, then LocalGroup's value again."""

    def __init__(self, g, k):
        self.g, self.k = g, k

    def __enter__(self):
        for c in self.g.comms:
            c.set_blocks(self.k)

    def __exit__(self, *exc):
        for c in self.g.comms:
            c.set_blocks(_default_blocks(self.g))


def _row_elems(dname, n):
    return n * UNITS_PER_ROW * 16 // DTYPES[dname][1].itemsize


# ---------------------------------------------------------------------------------------------
# operands with guard bytes
# ---------------------------------------------------------------------------------------------
class Operand:
    """``view`` = ``numel`` elements at element offset ``offset`` from a 16-byte aligned start inside
    a larger device buffer whose other bytes are random guards."""

    def __init__(self, data, dname, device, offset=0, seed=0):
        tdt, ndt = DTYPES[dname]
        es = ndt.itemsize
        self.es, self.ndt, self.numel = es, ndt, data.size
        self.front = 32 // es + offset
        total = self.front + data.size + 32 // es + 1
        host = np.random.default_rng(seed + 7919).integers(0, 256, total * es, dtype=np.uint8)
        host[self.front * es:(self.front + data.size) * es] = np.ascontiguousarray(data, dtype=ndt).view(np.uint8)
        self.host = host
        self.buf = torch.from_numpy(host.copy()).to(device)
        self.view = self.buf.view(tdt)[self.front:self.front + data.size]

    def read(self):
        """-> (value of the view, the buffer's bytes outside the view are unchanged)"""
        b = self.buf.cpu().numpy()
        lo, hi = self.front * self.es, (self.front + self.numel) * self.es
        guards = np.array_equal(b[:lo], self.host[:lo]) and np.array_equal(b[hi:], self.host[hi:])
        return b[lo:hi].view(self.ndt), guards

    def unchanged(self):
        return np.array_equal(self.buf.cpu().numpy(), self.host)


# ---------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------
SUBNORMAL = {"float16": 2.0 ** -20, "bfloat16": 2.0 ** -130, "float32": 2.0 ** -140, "float64": 2.0 ** -1060}


def make_inputs(dname, op, n, numel, seed, specials=True):
    """Per-rank inputs.  Floats: randn of mixed magnitudes (PROD: factors in ±[0.5, 2]), NaN/±inf on
    rank 0 alone, on rank n-1 alone and on both, signed zeros and subnormals.  Integers: the whole
    range, so 8/32/64-bit SUM and PROD wrap."""
    ndt = DTYPES[dname][1]
    rng = np.random.default_rng(seed)
    if not E.is_float(ndt):
        info = np.iinfo(ndt)
        ins = [rng.integers(info.min, info.max, numel, dtype=ndt, endpoint=True) for _ in range(n)]
        if numel >= 4:
            for t in ins:
                t[-4:] = [info.min, info.max, info.min + 1, 1]
        return ins
    span = {"float16": 2, "bfloat16": 3, "float32": 4, "float64": 8}[dname]
    out = []
    for _ in range(n):
        if op == O.PRODUCT:
            x = np.exp2(rng.uniform(-1, 1, numel)) * rng.choice([-1.0, 1.0], numel)
        else:
            x = rng.standard_normal(numel) * 10.0 ** rng.integers(-span, span + 1, numel)
        out.append(x)
    if specials and numel >= 12:
        nan, inf, sub = np.nan, np.inf, SUBNORMAL[dname]
        last = n - 1
        for base in (0, numel - 12):  # at the start and in the ragged tail
            out[0][base + 0] = nan                       # NaN on rank 0 alone
            out[last][base + 1] = nan                    # NaN on rank n-1 alone
            out[0][base + 2] = out[last][base + 2] = nan  # on both
            out[0][base + 3] = inf
            out[last][base + 4] = -inf
            out[0][base + 5], out[last][base + 5] = inf, -inf
            for r in range(n):
                out[r][base + 6] = 0.0                    # +0 everywhere but -0 on rank 0
                out[r][base + 7] = -0.0                   # -0 everywhere
                out[r][base + 8] = 0.0
                out[r][base + 9] = sub * (r + 1)          # subnormals
                out[r][base + 10] = -sub
            out[0][base + 6] = -0.0
            out[last][base + 8] = -0.0                    # +0 on rank 0, -0 on rank n-1
            if op == O.PRODUCT:
                out[last][base + 11] = 0.0
    return [x.astype(ndt) for x in out]


# ---------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------
def same_bits(got, want):
    """Bit equality, except that any NaN matches any NaN."""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape:
        return False
    if E.is_float(got.dtype):
        gn, wn = np.isnan(got), np.isnan(want)
        if not np.array_equal(gn, wn):
            return False
        got, want = got[~gn], want[~wn]
    return np.array_equal(got.view(np.uint8), want.view(np.uint8))


def check_result(got, ins, op, dname, what, nvls=False):
    ndt = DTYPES[dname][1]
    half = dname in HALF
    if not nvls:
        want = O.reduce_rank_ascending(ins, op, accumulate="fp32" if half else "native")
        assert same_bits(got, want), (what, "vs rank-ascending oracle", _first_diff(got, want))
    if E.is_float(ndt):
        acc = np.float32 if half and not nvls else ndt
        ok = E.within_bound(got, ins, op, acc_dtype=acc)
        assert ok.all(), (what, "vs exact reference", int(np.argmin(ok)))


def _first_diff(got, want):
    """(index, got, want) of the first element that differs, for the assertion message."""
    for i in range(got.size):
        if not same_bits(got[i:i + 1], want[i:i + 1]):
            return i, got[i], want[i]
    return None


def run_allreduce(g, dname, op, ins, algo, offset=0, out_of_place=False):
    """One all-reduce over padded operands; checks guards, inputs and replicas; returns rank 0's result."""
    n = g.world_size
    bufs = [Operand(ins[r], dname, g.device(r), offset, seed=r) for r in range(n)]
    outs = [Operand(np.zeros_like(ins[r]), dname, g.device(r), offset, seed=100 + r) for r in range(n)] \
        if out_of_place else bufs
    g.run(lambda c, r: c.allreduce(bufs[r].view, op, out=outs[r].view if out_of_place else None, algo=algo))
    results = []
    for r in range(n):
        got, guards = outs[r].read()
        assert guards, ("guard bytes changed", r)
        if out_of_place:
            assert bufs[r].unchanged(), ("out-of-place input changed", r)
        results.append(got)
    for r in range(1, n):
        assert np.array_equal(results[r].view(np.uint8), results[0].view(np.uint8)), ("replicas differ", r)
    return results[0]


def _algos(g, nbytes):
    from ray_b200 import _native as N

    out = [("auto", N.ALGO_AUTO), ("oneshot", N.ALGO_ONESHOT), ("twoshot", N.ALGO_TWOSHOT)]
    if nbytes <= 64 << 10:
        out.append(("ll", N.ALGO_LL))
    if nbytes % 16 == 0:  # the pipelined kernels move whole 16-byte units (the views are aligned)
        out.append(("pipe", N.ALGO_PIPE))
    return out


def _on_switch(g, dname, op, aname):
    """Whether the all-reduce reduces on the NVSwitch, where the order of the sum is the switch's:
    ALGO_NVLS, and ALGO_PIPE from 3 ranks on with the multicast mapping for SUM / AVG on f32, f16 and
    bf16 (b200_allreduce then takes the NVLS pipelined kernel)."""
    if aname == "nvls":
        return True
    return (aname == "pipe" and g.has_multicast and g.world_size > 2 and dname in NVLS_DTYPES
            and op in (O.SUM, O.AVG))


# ---------------------------------------------------------------------------------------------
# A. all-reduce
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dname", list(DTYPES))
@pytest.mark.parametrize("world", WORLDS)
def test_allreduce_dtype_op_matrix(groups, world, dname):
    """10 dtypes x 5 ops x {LL, one-shot, two-shot, AUTO, PIPE} at 1 element, a ragged 257 and two
    two-shot rows plus a tail (PIPE: two rows plus one 16-byte unit)."""
    g = groups(world)
    es = DTYPES[dname][1].itemsize
    row = _row_elems(dname, world)
    for oname, op in OPS.items():
        for numel in (1, 257, 2 * row + 3, 2 * row + 16 // es):
            algos = [a for a in _algos(g, numel * es) if (a[0] == "pipe") == (numel == 2 * row + 16 // es)]
            switch = any(_on_switch(g, dname, op, aname) for aname, _ in algos)
            # on the switch: finite, normal inputs (its handling of subnormals is not specified)
            ins = make_inputs(dname, op, world, numel, seed=world * 1000 + numel + op, specials=not switch)
            for i, (aname, algo) in enumerate(algos):
                got = run_allreduce(g, dname, op, ins, algo, out_of_place=(i % 2 == 1))
                check_result(got, ins, op, dname, (world, dname, oname, numel, aname),
                             nvls=_on_switch(g, dname, op, aname))


@pytest.mark.parametrize("world", WORLDS)
def test_allreduce_nvls_matrix(groups, world):
    """The switch reduction (SUM / AVG on f32, f16, bf16) at the sizes of the dtype x op matrix,
    within the bound of a sum rounded in the element type; needs one GPU per rank."""
    from ray_b200 import _native as N

    g = groups(world)
    if not g.has_multicast:
        pytest.skip("NVLS needs the multicast mapping, which needs one GPU per rank")
    for dname in ("float32", "float16", "bfloat16"):
        row = _row_elems(dname, world)
        for oname in ("SUM", "AVG"):
            op = OPS[oname]
            for numel in (1, 257, 2 * row + 3):
                # finite, normal inputs: the switch's handling of subnormals is not specified
                ins = make_inputs(dname, op, world, numel, seed=world * 1000 + numel + op, specials=False)
                for i in range(2):
                    got = run_allreduce(g, dname, op, ins, N.ALGO_NVLS, out_of_place=i == 1)
                    check_result(got, ins, op, dname, (world, dname, oname, numel, "nvls"), nvls=True)


@pytest.mark.parametrize("world", WORLDS)
def test_min_max_propagate_nan_from_any_rank(groups, world):
    """A NaN on rank 0, on rank n-1 or on both survives MIN and MAX on every peer-load kernel."""
    from ray_b200 import _native as N

    g = groups(world)
    for dname in ("float32", "float64", "float16", "bfloat16"):
        ndt = DTYPES[dname][1]
        for op in (O.MIN, O.MAX):
            base = np.arange(1.0, 17.0)
            ins = [(base * (r + 1)).astype(ndt) for r in range(world)]
            ins[0][0] = ins[world - 1][1] = ins[0][2] = ins[world - 1][2] = np.nan
            if world > 2:
                ins[1][3] = np.nan  # a middle rank
            for aname, algo in (("ll", N.ALGO_LL), ("oneshot", N.ALGO_ONESHOT), ("twoshot", N.ALGO_TWOSHOT),
                                ("pipe", N.ALGO_PIPE)):
                got = run_allreduce(g, dname, op, ins, algo)
                nanpos = [0, 1, 2] + ([3] if world > 2 else [])
                assert np.all(np.isnan(got[nanpos].astype(np.float64))), (world, dname, op, aname, got[:4])
                check_result(got, ins, op, dname, (world, dname, op, aname))


@pytest.mark.parametrize("world", WORLDS)
def test_allreduce_geometry_sweep(groups, world):
    """{u8, i64, bf16, f32} x {SUM, AVG, MAX}: one row ± 1 element, more rows than grid x UNR, 2.5
    staging slots on the small-slot group, views offset by 1 and 3 elements, grids forced to 1 and
    3 CTAs (PIPE: 4)."""
    from ray_b200 import _native as N

    g, gs = groups(world), groups(world, small=True)
    for dname in ("uint8", "int64", "bfloat16", "float32"):
        es = DTYPES[dname][1].itemsize
        row = _row_elems(dname, world)
        for oname in ("SUM", "AVG", "MAX"):
            op = OPS[oname]
            seed = world * 7 + op

            def case(grp, numel, algos, offset=0, tag=""):
                switch = any(_on_switch(grp, dname, op, aname) for aname, _ in algos)
                ins = make_inputs(dname, op, world, numel, seed=seed + numel, specials=not switch)
                for aname, algo in algos:
                    got = run_allreduce(grp, dname, op, ins, algo, offset=offset)
                    check_result(got, ins, op, dname, (world, dname, oname, numel, aname, offset, tag),
                                 nvls=_on_switch(grp, dname, op, aname))

            two = [("twoshot", N.ALGO_TWOSHOT), ("oneshot", N.ALGO_ONESHOT)]
            for numel in (row - 1, row + 1):
                case(g, numel, two + ([("ll", N.ALGO_LL)] if numel * es <= 64 << 10 else []))
            # more rows than grid x UNR (UNR = 2 in the peer-load reduce loop), in ONE staging piece:
            # the grid is capped so that 2 * grid + 1 rows fit the slot (with one GPU per rank the
            # whole-GPU grid would need more rows than the slot holds, and the message would split)
            k = min(_grid(g), (STAGING // (row * es) - 2) // 2)
            numel = (2 * k + 1) * row + 5
            assert numel * es <= STAGING
            with _Forced(g, k):
                case(g, numel, [("twoshot", N.ALGO_TWOSHOT)], tag=f"rows>grid*UNR, blocks={k}")
            # 2.5 staging slots: the slot loop and the pipeline's chunk pieces
            big = (5 * SMALL_SLOT // 2) // es
            case(gs, big + 3, [("twoshot", N.ALGO_TWOSHOT)], tag="2.5 slots")
            case(gs, big, [("pipe", N.ALGO_PIPE)], tag="2.5 slots")
            for offset in (1, 3):
                case(g, row + 1, two + ([("ll", N.ALGO_LL)] if (row + 1) * es <= 64 << 10 else []), offset=offset)
            for k in (1, 3):
                with _Forced(g, k):
                    case(g, (2 * k + 1) * row + 3, two, tag=f"blocks={k}")
            with _Forced(gs, 4):
                case(gs, big, [("pipe", N.ALGO_PIPE)], tag="blocks=4")


# ---------------------------------------------------------------------------------------------
# B. reduce-scatter and reduce
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", WORLDS)
def test_reducescatter_dtype_op_matrix(groups, world):
    """List form and reducescatter_from, every dtype x op: 1 and 257 elements per rank (slices not
    a multiple of 16 bytes), unaligned outputs, and for three dtypes a case larger than
    staging/world on the small-slot group so the piece loop runs."""
    g, gs = groups(world), groups(world, small=True)
    for dname in DTYPES:
        es = DTYPES[dname][1].itemsize
        for oname, op in OPS.items():
            cases = [(g, 1, 0), (g, 257, 1)]
            if dname in BIG_DTYPES:
                cases.append((gs, (3 * SMALL_SLOT // 2) // world // es + 3, 0))
            for grp, count, offset in cases:
                what = (world, dname, oname, count, offset)
                flat = make_inputs(dname, op, world, world * count, seed=world * 31 + op + count)
                # list form: rank q's tensor i is flat[q][i*count:(i+1)*count]
                ins = [[Operand(flat[q][i * count:(i + 1) * count], dname, grp.device(q), offset, seed=q * 10 + i)
                        for i in range(world)] for q in range(world)]
                outs = [Operand(np.zeros(count, DTYPES[dname][1]), dname, grp.device(r), offset, seed=50 + r)
                        for r in range(world)]
                grp.run(lambda c, r: c.reducescatter(outs[r].view, [o.view for o in ins[r]], op))
                srcs = [Operand(flat[q], dname, grp.device(q), 0, seed=70 + q) for q in range(world)]
                outs2 = [Operand(np.zeros(count, DTYPES[dname][1]), dname, grp.device(r), offset, seed=90 + r)
                         for r in range(world)]
                grp.run(lambda c, r: c.reducescatter_from(outs2[r].view, srcs[r].view, op))
                for r in range(world):
                    col = [flat[q][r * count:(r + 1) * count] for q in range(world)]
                    for o in (outs[r], outs2[r]):
                        got, guards = o.read()
                        assert guards, what
                        check_result(got, col, op, dname, what + (r,))
                    assert all(t.unchanged() for t in ins[r]) and srcs[r].unchanged(), what


@pytest.mark.parametrize("world", WORLDS)
def test_reduce_dtype_op_matrix(groups, world):
    """Reduce to root 0 and to root n-1, every dtype x op, aligned and unaligned buffers, and for
    three dtypes a message larger than a staging slot; only the root's tensor changes."""
    g, gs = groups(world), groups(world, small=True)
    for dname in DTYPES:
        es = DTYPES[dname][1].itemsize
        for oname, op in OPS.items():
            cases = [(g, 1, 0, 0), (g, 257, 1, world - 1)]
            if dname in BIG_DTYPES:
                cases.append((gs, (5 * SMALL_SLOT // 4) // es + 3, 3, world - 1))
            for grp, numel, offset, root in cases:
                what = (world, dname, oname, numel, offset, root)
                ins = make_inputs(dname, op, world, numel, seed=world * 17 + op + numel)
                bufs = [Operand(ins[r], dname, grp.device(r), offset, seed=r) for r in range(world)]
                grp.run(lambda c, r: c.reduce(bufs[r].view, root, op))
                for r in range(world):
                    if r == root:
                        got, guards = bufs[r].read()
                        assert guards, what
                        check_result(got, ins, op, dname, what)
                    else:
                        assert bufs[r].unchanged(), what


# ---------------------------------------------------------------------------------------------
# C. multi-tensor all-reduce
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3, 8])
def test_multi_tensor_allreduce_matrix(groups, world):
    """f16/bf16/f32/f64 x 5 ops on a 70-entry list: zero-size entries in the middle, one tensor
    larger than staging/2 in the middle (single-tensor path), unaligned views, more than 48
    tensors (the table splits); the number of launches is asserted."""
    gs = groups(world, small=True)
    rng = np.random.default_rng(world)
    counts = [int(c) for c in rng.integers(1, 300, 70)]
    counts[20] = counts[45] = 0
    for dname in ("float16", "bfloat16", "float32", "float64"):
        es = DTYPES[dname][1].itemsize
        cnt = list(counts)
        cnt[60] = (SMALL_SLOT // 2) // es + 5  # larger than staging/2
        for oname, op in OPS.items():
            # with the multicast mapping the table kernel reduces f32/f16/bf16 SUM/AVG on the switch:
            # finite, normal inputs there (its handling of subnormals is not specified)
            nvls = gs.has_multicast and op in (O.SUM, O.AVG) and dname != "float64"
            ins = [make_inputs(dname, op, world, c, seed=world * 1000 + i + op, specials=not nvls)
                   for i, c in enumerate(cnt)]
            bufs = [[Operand(ins[i][r], dname, gs.device(r), offset=i % 3, seed=r * 100 + i)
                     for i in range(len(cnt))] for r in range(world)]
            before = gs.comms[0].launch_count
            gs.run(lambda c, r: c.allreduce_multi([b.view for b in bufs[r]], op))
            # tables of 48 and 10 entries (zero-size entries take no slot; the large tensor ends the
            # second), one launch for the large tensor, a table of the 9 after it
            assert gs.comms[0].launch_count - before == 4, (world, dname, oname)
            for i in range(len(cnt)):
                res = []
                for r in range(world):
                    got, guards = bufs[r][i].read()
                    assert guards, (world, dname, oname, i, r)
                    res.append(got)
                    assert np.array_equal(got.view(np.uint8), res[0].view(np.uint8)), (world, dname, oname, i)
                check_result(res[0], [ins[i][r] for r in range(world)], op, dname, (world, dname, oname, i),
                             nvls=nvls)


# ---------------------------------------------------------------------------------------------
# D. fused gradient all-reduce
# ---------------------------------------------------------------------------------------------
WIRES = {"f32": (torch.float32, np.dtype(np.float32)), "bf16": (torch.bfloat16, BF16),
         "f16": (torch.float16, np.dtype(np.float16))}


def _grad_check(got, grads, scale, wire, nvls, what):
    n = len(grads)
    wdt = WIRES[wire][1]
    if not nvls:
        want = O.ddp_grad_sync(grads, wire, scale=scale)[0]
        assert same_bits(got, want), (what, "vs ddp_grad_sync", _first_diff(got, want))
    # float64 mean: every g*scale rounds in fp32 and to the wire, the sum in fp32 (or in the wire
    # type on the switch), the result once more to the wire
    s32 = np.float64(np.float32(scale))
    x = np.stack([g.astype(np.float64) * s32 for g in grads])
    with np.errstate(invalid="ignore"):
        exact = x.sum(axis=0)
        uw, u32 = E.UNIT_ROUNDOFF[wdt], 2.0 ** -24
        acc = uw if nvls else u32
        bound = (u32 + uw + (n - 1) * acc) * np.abs(x).sum(axis=0) * (1 + uw) + uw * np.abs(exact) \
            + (n + 2) * (E.TINY[wdt] + E.TINY[np.dtype(np.float32)])
        g64 = got.astype(np.float64)
        ok = np.abs(g64 - exact) <= bound
        nan = np.isnan(exact)
        ok = np.where(nan, np.isnan(g64), ok)
        fmax = float(ml_dtypes.finfo(wdt).max)
        over = ~nan & (np.isinf(exact) | (np.abs(x).max(axis=0) * (1 - uw) > fmax))
        ok = np.where(over, np.isinf(g64) | np.isnan(g64) | ok, ok)
    assert ok.all(), (what, "vs float64 mean", int(np.argmin(ok)))


def _grad_specials(wire, n, numel, rng):
    grads = [rng.standard_normal(numel).astype(np.float32) * np.float32(10.0) ** rng.integers(-3, 4, numel)
             for _ in range(n)]
    if numel >= 12:
        for r in range(n):
            grads[r][0] = 0.0
            grads[r][1] = -0.0
            grads[r][2] = np.float32(2.0 ** -140) * (r + 1)    # fp32 subnormals
            grads[r][4] = 1e5 if r == 0 else 1.0                # g*scale overflows f16 -> inf
        grads[0][3] = np.inf
        grads[n - 1][5] = -np.inf
        grads[n - 1][6] = np.nan                                 # NaN on one rank
        tie = {"bf16": 1 + 2.0 ** -8, "f16": 1 + 2.0 ** -11, "f32": 1.0}[wire]
        grads[0][7] = tie                                        # halfway: rounds to even (down)
        grads[0][8] = tie + 2 * (tie - 1)                        # halfway: rounds to even (up)
        grads[0][9] = -tie
    return grads


@pytest.mark.parametrize("wire", list(WIRES))
@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_fused_gradient_matrix(groups, native_lib, world, wire):
    """Wires f32/bf16/f16 x worlds 1-8 x sizes 1, 7, 8, 9, one row ± 1, more than 2 staging slots
    x base offsets 0 and 1 element x scales 1/n, 1.0 and 0.1, with ±0, fp32 subnormals, ±inf, NaN
    on one rank, f16 overflow and rounding ties among the gradients (not where the reduction runs
    on the switch, whose handling of subnormals is not specified)."""
    from ray_b200.testing import LocalGroup

    own = world == 1
    g = LocalGroup(1, timeout_ms=20000, staging_bytes=SMALL_SLOT) if own else groups(world, small=True)
    try:
        tdt, wdt = WIRES[wire]
        E_ = 4 if wire == "f32" else 8
        row = world * UNITS_PER_ROW * E_
        slots = (2 * SMALL_SLOT) // wdt.itemsize + 2 * row + 5  # more than 2 staging slots of wire data
        nvls = g.has_multicast and world >= 3
        for numel in (1, 7, 8, 9, row - 1, row + 1, slots):
            for offset in (0, 1):
                for scale in (1.0 / world, 1.0, 0.1):
                    # ties must stay ties after the scale: only exact with scale 1.0
                    rng = np.random.default_rng(numel * 10 + offset + world)
                    specials = scale == 1.0 and not nvls
                    grads = _grad_specials(wire, world, numel, rng) if specials else \
                        [rng.standard_normal(numel).astype(np.float32) for _ in range(world)]
                    bufs = [Operand(grads[r], "float32", g.device(r), offset, seed=r) for r in range(world)]
                    g.run(lambda c, r: c.grad_allreduce(bufs[r].view, scale, tdt))
                    res = []
                    for r in range(world):
                        got, guards = bufs[r].read()
                        assert guards, (world, wire, numel, offset, scale, r)
                        res.append(got)
                        assert np.array_equal(got.view(np.uint8), res[0].view(np.uint8)), "replicas differ"
                    what = (world, wire, numel, offset, scale)
                    _grad_check(res[0], grads, scale, wire, nvls, what)
                    if specials and numel >= 12:
                        s = res[0]
                        assert s[3] == np.inf and s[5] == -np.inf and np.isnan(s[6]), what
                        assert np.isinf(s[4]) == (wire == "f16"), what  # 1e5 overflows f16 only
    finally:
        if own:
            g.destroy()
