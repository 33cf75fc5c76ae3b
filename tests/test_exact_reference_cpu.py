"""CPU checks of the exact reference (oracle/exact.py) and of the rank-ascending oracle against it.

The two are written independently: integers must agree bit for bit (wrapping included), MIN/MAX
must agree bit for bit (NaN from any rank, sign of zero), and floating-point SUM/PROD of the oracle
must lie within the stated error bound of the exact value.
"""
import numpy as np
import pytest

from oracle import collective_oracle as O
from oracle import exact as E

BF16 = O.bfloat16
OPS = {"SUM": O.SUM, "PRODUCT": O.PRODUCT, "MIN": O.MIN, "MAX": O.MAX}
ALL_OPS = {**OPS, "AVG": O.AVG}
INT_DTYPES = [np.uint8, np.int8, np.int32, np.uint32, np.int64, np.uint64]


def _same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _golden_dtype(dname):
    return BF16 if dname == "bfloat16" else np.dtype(dname)


def test_exact_reference_matches_the_oracle_on_every_golden_allreduce_fixture(golden):
    checked = 0
    for key in golden.files:
        parts = key.split("/")
        if parts[0] != "allreduce" or parts[-1] != "in":
            continue
        dname, oname = parts[2], parts[3]
        dt = _golden_dtype(dname)
        ins = [x.view(dt) for x in golden[key]]
        op = OPS[oname]
        want = O.reduce_rank_ascending(ins, op)
        assert _same_bits(want, golden[key[:-len("in")] + "apply_op"].view(dt)), key
        if E.is_float(dt) and op in (O.SUM, O.PRODUCT):
            # the oracle rounds every partial result in the element type
            assert np.all(E.within_bound(want, ins, op, acc_dtype=dt)), key
            wide = O.reduce_rank_ascending(ins, op, accumulate="fp32")
            acc = np.float32 if dt != np.float64 else np.float64
            assert np.all(E.within_bound(wide, ins, op, acc_dtype=acc)), key
        else:
            got = E.exact_reduce(ins, op)
            assert _same_bits(got.astype(dt) if E.is_float(dt) else got, want), key
        checked += 1
    assert checked == 4 * 8 * 4  # worlds x dtypes x ops


def test_exact_reference_matches_the_oracle_on_golden_reduce_and_reducescatter(golden):
    for world in (2, 3, 4, 8):
        for dname in ("float32", "int32"):
            dt = np.dtype(dname)
            ins = list(golden[f"reduce/w{world}/{dname}/in"])
            want = O.reduce_rank_ascending(ins, O.SUM)
            if dname == "int32":
                assert _same_bits(E.exact_reduce(ins, O.SUM), want)
            else:
                assert np.all(E.within_bound(want, ins, O.SUM, acc_dtype=dt))
            lists = golden[f"reducescatter/w{world}/{dname}/in"]
            for r in range(world):
                col = [lists[q][r] for q in range(world)]
                want = O.reduce_rank_ascending(col, O.SUM)
                if dname == "int32":
                    assert _same_bits(E.exact_reduce(col, O.SUM), want)
                else:
                    assert np.all(E.within_bound(want, col, O.SUM, acc_dtype=dt))


@pytest.mark.parametrize("dtype", INT_DTYPES)
@pytest.mark.parametrize("oname", list(ALL_OPS))
@pytest.mark.parametrize("world", [2, 3, 8])
def test_integer_reductions_wrap_like_twos_complement(dtype, oname, world):
    info = np.iinfo(dtype)
    rng = np.random.default_rng(world * 100 + INT_DTYPES.index(dtype) * 10 + ALL_OPS[oname])
    ins = [rng.integers(info.min, info.max, size=300, dtype=dtype, endpoint=True) for _ in range(world)]
    for t in ins:  # the extremes, where wrapping and truncating division are easiest to get wrong
        t[:4] = [info.min, info.max, info.min + 1, info.max - 1]
    want = E.exact_reduce(ins, ALL_OPS[oname])
    assert _same_bits(O.reduce_rank_ascending(ins, ALL_OPS[oname]), want)


def test_integer_avg_is_exact_above_2_to_the_53():
    # the sum wraps modulo 2**64 before the truncating division: (2**63 + 4 - 2**64) / 2
    a, b = np.array([2 ** 62 + 1], np.int64), np.array([2 ** 62 + 3], np.int64)
    for got in (O.reduce_rank_ascending([a, b], O.AVG), E.exact_reduce([a, b], O.AVG)):
        assert got.dtype == np.int64 and int(got[0]) == -(2 ** 62) + 2
    a, b = np.array([2 ** 63 + 1], np.uint64), np.array([2 ** 63 + 3], np.uint64)
    for got in (O.reduce_rank_ascending([a, b], O.AVG), E.exact_reduce([a, b], O.AVG)):
        assert got.dtype == np.uint64 and int(got[0]) == 2
    # no wrap, odd values above 2**53: a float64 detour would round them
    a, b, c = (np.array([2 ** 60 + k], np.int64) for k in (1, 2, 6))
    for got in (O.reduce_rank_ascending([a, b, c], O.AVG), E.exact_reduce([a, b, c], O.AVG)):
        assert int(got[0]) == 2 ** 60 + 3
    # truncation toward zero for negative sums
    a, b = np.array([-7, -128, 5], np.int8), np.array([0, 0, -6], np.int8)
    for got in (O.reduce_rank_ascending([a, b], O.AVG), E.exact_reduce([a, b], O.AVG)):
        assert got.tolist() == [-3, -64, 0]


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.float16, "bfloat16"])
def test_min_max_propagate_nan_from_any_rank_and_keep_the_lower_rank_on_ties(dtype):
    dt = BF16 if dtype == "bfloat16" else np.dtype(dtype)
    nan, inf = float("nan"), float("inf")
    r0 = np.array([1, nan, nan, 0.0, -0.0, -inf, inf, 2], np.float64).astype(dt)
    r1 = np.array([nan, 1, nan, -0.0, 0.0, 1, 1, 2], np.float64).astype(dt)
    for op in (O.MIN, O.MAX):
        for ins in ([r0, r1], [r1, r0], [r0, r1, r1]):
            want = O.reduce_rank_ascending(ins, op)
            got = E.exact_reduce(ins, op)
            assert np.array_equal(np.isnan(want), np.isnan(got))
            assert np.all(np.isnan(want[:3].astype(np.float64)))  # NaN from rank 0, rank >= 1, both
            keep = ~np.isnan(got)
            assert _same_bits(want[keep], got[keep].astype(dt))
            # +0.0 vs -0.0 compare equal: the lower rank's operand is kept
            assert np.signbit(got[3]) == np.signbit(ins[0][3].astype(np.float64))
            assert np.signbit(got[4]) == np.signbit(ins[0][4].astype(np.float64))
    assert E.exact_reduce([r0, r1], O.MIN)[5] == -inf and E.exact_reduce([r0, r1], O.MAX)[6] == inf


def test_non_finite_sums_and_products_follow_ieee():
    nan, inf = float("nan"), float("inf")
    a = np.array([inf, inf, nan, 1, 0.0, inf, 3e38], np.float32)
    b = np.array([1, -inf, 1, nan, inf, inf, 3e38], np.float32)
    s = E.exact_reduce([a, b], O.SUM)
    assert s[0] == inf and np.isnan(s[1]) and np.isnan(s[2]) and np.isnan(s[3]) and s[5] == inf
    assert s[6] == 2 * float(np.float32(3e38))  # exact, and beyond the fp32 range
    ok = E.within_bound(O.reduce_rank_ascending([a, b], O.SUM), [a, b], O.SUM)
    assert ok.all()  # the oracle's overflow to +inf is accepted where the exact sum exceeds fp32
    p = E.exact_reduce([a, b], O.PRODUCT)
    assert p[0] == inf and p[1] == -inf and np.isnan(p[4]) and p[5] == inf
    assert E.within_bound(O.reduce_rank_ascending([a, b], O.PRODUCT), [a, b], O.PRODUCT).all()


def test_subnormals_and_signed_zeros_are_summed_exactly():
    tiny = np.float32(2.0 ** -149)
    a = np.array([tiny, 3 * tiny, -0.0, 2.0 ** -126, -tiny], np.float32)
    b = np.array([tiny, -tiny, -0.0, -(2.0 ** -127), tiny], np.float32)
    s = E.exact_reduce([a, b], O.SUM)
    assert s.tolist() == [2.0 ** -148, 2.0 ** -148, 0.0, 2.0 ** -127, 0.0]
    want = O.reduce_rank_ascending([a, b], O.SUM)
    assert np.array_equal(want.astype(np.float64), s)  # a sum of two fp32 subnormals is exact in fp32
    assert np.signbit(want[2])  # -0.0 + -0.0 == -0.0 in IEEE
    assert E.error_bound([a, b], O.MIN).max() == 0


def test_the_bound_rejects_a_result_off_by_more_than_the_rounding_error():
    rng = np.random.default_rng(3)
    ins = [(rng.standard_normal(1000) * 10.0 ** rng.integers(-3, 4, 1000)).astype(np.float32) for _ in range(4)]
    want = O.reduce_rank_ascending(ins, O.SUM)
    assert E.within_bound(want, ins, O.SUM).all()
    off = want.copy()
    # 4 ulps at the element with the largest sum: beyond (n-1) u sum|x| + u |s| when cancellation is mild
    i = int(np.argmax(np.abs(want) / np.sum(np.abs(np.stack(ins)), axis=0)))
    off[i] = np.nextafter(np.nextafter(np.nextafter(np.nextafter(off[i], np.inf), np.inf), np.inf), np.inf)
    assert not E.within_bound(off, ins, O.SUM)[i]
    avg = O.reduce_rank_ascending(ins, O.AVG)
    assert E.within_bound(avg, ins, O.AVG).all()
    assert not E.within_bound(want, ins, O.AVG).all()  # the sum is not the mean
