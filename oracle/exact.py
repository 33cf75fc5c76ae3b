"""Exact reference of the element-wise reductions over ranks.  TEST INFRASTRUCTURE ONLY.

Written independently of ``collective_oracle.reduce_rank_ascending`` so that the oracle and a
kernel that share an arithmetic mistake cannot pass together:

* integers: Python integers, wrapped modulo 2**bits as two's complement does after every SUM /
  PROD step; AVG is the wrapped sum divided with truncation toward zero (NCCL's sum-then-divide);
* float64 SUM / AVG: the exactly rounded float64 value of the exact sum (``math.fsum``), AVG
  divided by n once; PROD: the exact product (``fractions``) rounded once to float64;
* fp32 / fp16 / bf16 SUM / AVG / PROD: vectorised float64 arithmetic (compensated summation), a
  few float64 roundings away from exact, which is 2**29 times finer than any bound it meets;
* MIN / MAX: a NaN on any rank propagates; among equal values (``+0.0`` / ``-0.0``) the lower
  rank's operand wins, which is the rank-ascending rule of the oracle.

``exact_reduce`` returns integers in their own dtype and floating-point results as float64
(16-bit inputs are widened exactly).  ``error_bound`` is the largest difference from that value a
correct kernel may show; ``within_bound`` applies it.
"""
from __future__ import annotations

import math
from fractions import Fraction
from typing import Sequence

import ml_dtypes
import numpy as np

from .collective_oracle import AVG, MAX, MIN, PRODUCT, SUM, bfloat16

# unit roundoff of each floating-point type
UNIT_ROUNDOFF = {np.dtype(np.float64): 2.0 ** -53, np.dtype(np.float32): 2.0 ** -24,
                 np.dtype(np.float16): 2.0 ** -11}
# smallest positive subnormal: the absolute rounding error of a result that lands below the normal range
TINY = {np.dtype(np.float64): 2.0 ** -1074, np.dtype(np.float32): 2.0 ** -149, np.dtype(np.float16): 2.0 ** -24}
if bfloat16 is not None:
    UNIT_ROUNDOFF[bfloat16] = 2.0 ** -8
    TINY[bfloat16] = 2.0 ** -133


def is_float(dtype) -> bool:
    return np.dtype(dtype) in UNIT_ROUNDOFF


def _wrap(v: int, bits: int, signed: bool) -> int:
    v %= 1 << bits
    return v - (1 << bits) if signed and v >= 1 << (bits - 1) else v


def _int_column(vals: Sequence[int], op: int, bits: int, signed: bool) -> int:
    acc = vals[0]
    for v in vals[1:]:
        if op in (SUM, AVG):
            acc = _wrap(acc + v, bits, signed)
        elif op == PRODUCT:
            acc = _wrap(acc * v, bits, signed)
        elif op == MIN:
            acc = v if v < acc else acc
        elif op == MAX:
            acc = v if v > acc else acc
        else:
            raise ValueError(f"Operation {op} not supported")
    if op == AVG:
        q = abs(acc) // len(vals)
        acc = q if acc >= 0 else -q
    return acc


def _float_column(vals: Sequence[float], op: int) -> float:
    """SUM / AVG / PROD of one float64 column."""
    if not all(math.isfinite(v) for v in vals):
        # IEEE rules for inf / NaN do not depend on the order: inf - inf and 0 * inf are NaN
        acc = vals[0]
        for v in vals[1:]:
            acc = acc * v if op == PRODUCT else acc + v
        return acc / len(vals) if op == AVG else acc
    if op == PRODUCT:
        p = Fraction(1)
        for v in vals:
            p *= Fraction(v)
        return float(p)
    s = math.fsum(vals)
    if op == AVG:
        return float(Fraction(s) / len(vals)) if s else s
    if op != SUM:
        raise ValueError(f"Operation {op} not supported")
    return s


def _narrow_float_reduce(x: np.ndarray, op: int) -> np.ndarray:
    """Vectorised SUM / AVG / PROD over axis 0 of float64 values widened from a type of at most 24
    significand bits.  SUM: compensated (Neumaier) float64 summation, within a few float64 roundings
    of the exact sum, 2**29 times finer than the fp32 rounding it is compared with.  PROD: the
    float64 product, n - 1 float64 roundings."""
    n = x.shape[0]
    with np.errstate(invalid="ignore", over="ignore"):
        plain = x[0].copy()
        for v in x[1:]:
            plain = plain * v if op == PRODUCT else plain + v
        if op == PRODUCT:
            return plain
        s, c = x[0].copy(), np.zeros_like(x[0])
        for v in x[1:]:
            t = s + v
            big = np.abs(s) >= np.abs(v)
            c += np.where(big, (s - t) + v, (v - t) + s)
            s = t
        out = np.where(np.isfinite(plain), s + c, plain)  # inf / NaN follow IEEE, in any order
    return out / n if op == AVG else out


def exact_reduce(tensors: Sequence[np.ndarray], op: int) -> np.ndarray:
    """Element-wise reduction of ``tensors`` (one per rank, same dtype and shape), computed exactly."""
    if len(tensors) == 0:
        raise ValueError("need at least one tensor")
    dtype = np.dtype(tensors[0].dtype)
    shape = tensors[0].shape
    if is_float(dtype):
        x = np.stack([np.asarray(t, dtype=dtype).astype(np.float64).ravel() for t in tensors])
        if op in (MIN, MAX):
            # the extreme value, NaN if any rank holds one; then the lowest rank holding a value
            # equal to it, which settles +0.0 against -0.0
            with np.errstate(invalid="ignore"):
                m = np.min(x, axis=0) if op == MIN else np.max(x, axis=0)
                first = np.argmax(x == m, axis=0)
            out = np.where(np.isnan(m), np.nan, x[first, np.arange(x.shape[1])])
        elif dtype == np.float64:
            cols = x.T
            out = np.fromiter((_float_column(c.tolist(), op) for c in cols), dtype=np.float64, count=cols.shape[0])
        elif op in (SUM, AVG, PRODUCT):
            out = _narrow_float_reduce(x, op)
        else:
            raise ValueError(f"Operation {op} not supported")
        return out.reshape(shape)
    if not np.issubdtype(dtype, np.integer):
        raise ValueError(f"unsupported dtype {dtype}")
    bits, signed = dtype.itemsize * 8, np.issubdtype(dtype, np.signedinteger)
    cols = zip(*[np.asarray(t).ravel().tolist() for t in tensors])  # Python ints
    out = [_int_column(c, op, bits, signed) for c in cols]
    return np.array(out, dtype=dtype).reshape(shape)


def error_bound(tensors: Sequence[np.ndarray], op: int, acc_dtype=None, out_dtype=None) -> np.ndarray:
    """Largest |result - exact_reduce(tensors, op)| of a correct floating-point reduction.

    SUM / AVG: any summation order loses at most (n-1) * u_acc * sum_r |x_r|; AVG's division and the
    final rounding to the output type add one rounding each.  PROD: a relative bound of n - 1
    roundings in the accumulator plus the output rounding.  MIN / MAX select, so they are exact.
    ``acc_dtype`` is the accumulator (fp32 for 16-bit inputs on the peer-load kernels, the element
    type itself for a reduction that rounds every partial sum); ``out_dtype`` is the result type.
    """
    dtype = np.dtype(tensors[0].dtype)
    out_dtype = np.dtype(out_dtype) if out_dtype is not None else dtype
    acc_dtype = np.dtype(acc_dtype) if acc_dtype is not None else out_dtype
    n = len(tensors)
    if op in (MIN, MAX):
        return np.zeros(tensors[0].shape)
    x = np.stack([np.asarray(t).astype(np.float64) for t in tensors])
    ref = np.abs(exact_reduce(tensors, op))
    ua, uo = UNIT_ROUNDOFF[acc_dtype], UNIT_ROUNDOFF[out_dtype]
    with np.errstate(invalid="ignore", over="ignore"):
        if op == PRODUCT:
            acc_err = ((n - 1) * ua * (1 + ua) ** n) * ref
        else:
            acc_err = (n - 1) * ua * np.sum(np.abs(x), axis=0)
            if op == AVG:
                acc_err = acc_err / n + ua * ref
        return acc_err * (1 + uo) + uo * ref + TINY[out_dtype] + TINY[acc_dtype]


def within_bound(got: np.ndarray, tensors: Sequence[np.ndarray], op: int, acc_dtype=None,
                 bound_scale: float = 1.0) -> np.ndarray:
    """Per-element check of ``got`` against the exact reference: NaN where it is NaN, the same
    infinity where it is infinite (or where a finite exact value lies beyond the type's range),
    and within ``bound_scale * error_bound`` everywhere else."""
    dtype = np.dtype(got.dtype)
    g = got.astype(np.float64)
    ref = exact_reduce(tensors, op)
    bound = bound_scale * error_bound(tensors, op, acc_dtype=acc_dtype, out_dtype=dtype)
    fmax = float(ml_dtypes.finfo(dtype).max)
    with np.errstate(invalid="ignore", over="ignore"):
        ok = np.abs(g - ref) <= bound
        nan = np.isnan(ref)
        ok = np.where(nan, np.isnan(g), ok)
        inf = ~nan & (np.isinf(ref) | (np.abs(ref) - bound > fmax))
        ok = np.where(inf, np.isinf(g) & (np.sign(g) == np.sign(ref)), ok)
    return ok
