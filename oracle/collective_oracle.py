"""CPU oracle for Ray's collective / tensor-transport hot path.  TEST INFRASTRUCTURE ONLY.

This module restates, in numpy, the arithmetic and data movement the reference performs
on this path.  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline
leg may import it; the product (``ray_b200``) never does and has no CPU fallback.

Where the arithmetic lives in the reference
-------------------------------------------
Ray itself contains no reduction code on this path: ``NCCLGroup`` / ``_NcclGroup`` hand the
buffers to libnccl through cupy (``python/ray/util/collective/collective_group/
nccl_collective_group.py:200,245,272,297,338,374,400``; ``python/ray/experimental/channel/
nccl_group.py:178,217,289,310,331``; cupy-cuda12x==13.4.0 -> nvidia-nccl-cu12==2.26.2,
``python/requirements_compiled.txt:419,1334``) and ``TorchGLOOGroup`` to torch c10d gloo
(``collective_group/torch_gloo_collective_group.py:217,234,252,258,279,286,290``;
torch==2.7.0, ``requirements_compiled.txt:2324``).  Neither third-party source is in the
reference tree.  The *published* semantics of those collectives are element-wise
reductions over ranks; the reference's own two explicit implementations reduce in
rank-ascending order:

  * ``CPUCommBarrier._apply_op``       python/ray/experimental/channel/cpu_communicator.py:69-89
  * ``MockInternalKVGroup.allreduce``  python/ray/util/collective/examples/mock_internal_kv_example.py:182-229

and that order is what this oracle (and the CUDA kernels on their peer-load paths) use.

How the oracle is pinned
------------------------
``tests/golden/make_golden.py`` (run in the build container, where /root/reference exists)
(1) extracts ``_apply_op`` from the reference source and executes it, and (2) runs the real
``torch.distributed`` gloo collectives through the exact call sequence of
``TorchGLOOGroup`` (including its reduce-scatter emulation and reduce-clone quirk), on
seeded inputs for world sizes 2, 3, 4 and 8.  The inputs and both sets of outputs are
committed as ``tests/golden/collective_golden.npz``; ``tests/test_oracle.py`` checks this
module against them: bit-exact for every integer dtype and for floats at world size 2,
bit-exact against ``_apply_op`` at every world size, and within 1e-6 * sum_r |x_r| of
gloo for fp32 at world sizes > 2 (gloo's ring order is not rank-ascending).

Half-precision note: the reference backends reduce fp16/bf16 in the tensor's dtype
(rounding after every add); ``reduce_rank_ascending(..., accumulate="native")`` restates
that.  The CUDA kernels accumulate 16-bit floats in fp32 and round once
(``accumulate="fp32"``), which is identical at world size 2 and never less accurate.
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np

try:  # bfloat16 for numpy
    import ml_dtypes

    bfloat16 = np.dtype(ml_dtypes.bfloat16)
except Exception:  # pragma: no cover - ml_dtypes ships with the image
    bfloat16 = None

# ray.util.collective.types.ReduceOp numbering (python/ray/util/collective/types.py:55-59)
SUM, PRODUCT, MIN, MAX = 0, 1, 2, 3
# extra value carried by ray.experimental.util.types.ReduceOp (experimental/util/types.py:11-17)
AVG = 4

# The Compiled-Graph enum orders MAX before MIN (SURVEY Q2); translate it to the numbering above.
CGRAPH_TO_COLLECTIVE_OP = {0: SUM, 1: PRODUCT, 2: MAX, 3: MIN, 4: AVG}


def _is_half(dtype: np.dtype) -> bool:
    return dtype == np.float16 or (bfloat16 is not None and dtype == bfloat16)


def reduce_rank_ascending(tensors: Sequence[np.ndarray], op: int, accumulate: str = "native") -> np.ndarray:
    """result = tensors[0]; for t in tensors[1:]: result = result (op) t.

    Follows CPUCommBarrier._apply_op (cpu_communicator.py:69-89) and
    MockInternalKVGroup.allreduce (mock_internal_kv_example.py:182-229).
    ``accumulate="fp32"`` widens 16-bit floats to fp32 for the whole chain and rounds once.
    """
    if len(tensors) == 0:
        raise ValueError("need at least one tensor")
    dtype = tensors[0].dtype
    widen = accumulate == "fp32" and _is_half(dtype)
    work = np.float32 if widen else dtype
    with np.errstate(over="ignore", invalid="ignore"):
        result = tensors[0].astype(work, copy=True)
        for t in tensors[1:]:
            t = t.astype(work, copy=False)
            if op in (SUM, AVG):
                result = (result + t).astype(work, copy=False)
            elif op == PRODUCT:
                result = (result * t).astype(work, copy=False)
            elif op in (MIN, MAX):
                # Spelled out rather than np.minimum / np.maximum, whose pick between equal operands
                # (+0.0 / -0.0) differs by dtype (numpy 2.3: the second for fp32/fp64/bf16, the
                # first for fp16).  Rule: a NaN from any rank propagates; on a tie the lower ranks'
                # value is kept.
                better = (t < result) if op == MIN else (t > result)
                if not np.issubdtype(np.dtype(work), np.integer):
                    better |= np.isnan(t) & ~np.isnan(result)
                result = np.where(better, t, result)
            else:
                raise ValueError(f"Operation {op} not supported")
        if op == AVG:
            n = len(tensors)
            if np.issubdtype(np.dtype(work), np.integer):
                # the wrapped sum divided with truncation toward zero, as an integer ncclAvg does;
                # in integer arithmetic, since a float64 detour loses int64/uint64 sums above 2**53
                div = np.asarray(n, dtype=work)
                q = result // div  # floor division; one more toward zero for a negative inexact quotient
                result = (q + ((result % div != 0) & (result < 0)).astype(work)).astype(work, copy=False)
            else:
                result = (result / np.asarray(n, dtype=work)).astype(work, copy=False)
        return result.astype(dtype, copy=False)


# ---------------------------------------------------------------------------
# ray.util.collective semantics (in-place on each rank's operands)
# ---------------------------------------------------------------------------
def allreduce(per_rank: List[np.ndarray], op: int = SUM, accumulate: str = "native") -> None:
    """collective.allreduce (collective.py:316-331): every rank's tensor becomes the reduction."""
    red = reduce_rank_ascending(per_rank, op, accumulate)
    for t in per_rank:
        t[...] = red


def reduce(per_rank: List[np.ndarray], root: int, op: int = SUM, accumulate: str = "native") -> None:
    """collective.reduce (collective.py:369-392): only the root's tensor changes
    (torch_gloo_collective_group.py:229-240 clones on non-root ranks)."""
    red = reduce_rank_ascending(per_rank, op, accumulate)
    per_rank[root][...] = red


def broadcast(per_rank: List[np.ndarray], root: int) -> None:
    """collective.broadcast (collective.py:431-450)."""
    for r, t in enumerate(per_rank):
        if r != root:
            t[...] = per_rank[root]


def allgather(out_lists: List[List[np.ndarray]], per_rank: List[np.ndarray]) -> None:
    """collective.allgather (collective.py:481-503): out_lists[r][p] = rank p's tensor."""
    for r in range(len(per_rank)):
        for p in range(len(per_rank)):
            out_lists[r][p][...] = per_rank[p]


def reducescatter(outs: List[np.ndarray], in_lists: List[List[np.ndarray]], op: int = SUM,
                  accumulate: str = "native", gloo_quirk: bool = False) -> None:
    """collective.reducescatter (collective.py:530-557): outs[r] = reduce_q in_lists[q][r].

    ``gloo_quirk=True`` additionally reproduces TorchGLOOGroup.reducescatter
    (torch_gloo_collective_group.py:260-282), which all-reduces *every* list member in
    place, so the callers' input lists are overwritten (SURVEY Q13).
    """
    n = len(outs)
    reduced = [reduce_rank_ascending([in_lists[q][i] for q in range(n)], op, accumulate) for i in range(n)]
    for r in range(n):
        outs[r][...] = reduced[r]
    if gloo_quirk:
        for q in range(n):
            for i in range(n):
                in_lists[q][i][...] = reduced[i]


def sendrecv(src: np.ndarray, dst: np.ndarray) -> None:
    """collective.send / recv (collective.py:589-670): a byte-exact copy."""
    dst[...] = src


# ---------------------------------------------------------------------------
# Compiled-Graph (Communicator ABC) semantics: out-of-place, dim-0 layouts
# ---------------------------------------------------------------------------
def cgraph_allreduce(per_rank: List[np.ndarray], cgraph_op: int, accumulate: str = "native") -> List[np.ndarray]:
    """_CollectiveOperation.execute, AllReduceOp branch (dag/collective_node.py:207-232)."""
    red = reduce_rank_ascending(per_rank, CGRAPH_TO_COLLECTIVE_OP[cgraph_op], accumulate)
    return [red.copy() for _ in per_rank]


def cgraph_allgather(per_rank: List[np.ndarray]) -> List[np.ndarray]:
    """AllGatherOp branch (dag/collective_node.py:198-206): [d0*n, ...] rank-major."""
    cat = np.concatenate(per_rank, axis=0)
    return [cat.copy() for _ in per_rank]


def cgraph_reducescatter(per_rank: List[np.ndarray], cgraph_op: int, accumulate: str = "native") -> List[np.ndarray]:
    """ReduceScatterOp branch (dag/collective_node.py:233-247): [d0/n, ...]; d0 % n == 0 required."""
    n = len(per_rank)
    if per_rank[0].shape[0] % n != 0:
        raise ValueError(
            f"Expected the first dimension of the input tensor to be divisible by the world size {n}")
    red = reduce_rank_ascending(per_rank, CGRAPH_TO_COLLECTIVE_OP[cgraph_op], accumulate)
    step = per_rank[0].shape[0] // n
    return [red[r * step:(r + 1) * step].copy() for r in range(n)]


# ---------------------------------------------------------------------------
# Data-parallel gradient synchronisation (the path TorchTrainer / LearnerGroup ride)
# ---------------------------------------------------------------------------
def _round_to(x: np.ndarray, dtype: np.dtype) -> np.ndarray:
    with np.errstate(over="ignore"):  # beyond the type's range rounds to inf, as the kernels do
        return x.astype(dtype).astype(np.float32)


def ddp_grad_sync(per_rank_grads: List[np.ndarray], wire: str = "f32", scale=None) -> List[np.ndarray]:
    """Mean of fp32 gradient buckets as torch DDP computes it under ray.train
    (train/torch/train_loop_utils.py:456-480 wraps the model in DDP; the c10d reducer
    divides each bucket by world_size and all-reduces it with SUM).

    wire="f32": bucket / n, then rank-ascending fp32 sum (exact DDP arithmetic up to order).
    wire="bf16"/"f16": torch's bf16/fp16_compress_hook arithmetic -- cast to the wire type,
    divide by n in the wire type, sum, cast back to fp32.  The kernel multiplies by 1/n in
    fp32 *before* the cast; for power-of-two n both orders are bit-identical (barring
    subnormals) and the kernel accumulates the sum in fp32.

    ``scale`` replaces 1/n by another fp32 factor (the kernel's ``scale`` argument): every
    gradient is multiplied by it in fp32, then cast to the wire type, as above.
    """
    n = len(per_rank_grads)
    inv = np.float32(1.0) / np.float32(n) if scale is None else np.float32(scale)
    if wire == "f32":
        scaled = [(g.astype(np.float32) * inv).astype(np.float32) for g in per_rank_grads]
        red = reduce_rank_ascending(scaled, SUM)
    else:
        wdt = bfloat16 if wire == "bf16" else np.dtype(np.float16)
        scaled = [_round_to(g.astype(np.float32) * inv, wdt) for g in per_rank_grads]
        acc = scaled[0].copy()
        for s in scaled[1:]:
            acc = (acc + s).astype(np.float32)
        red = _round_to(acc, wdt)
    return [red.copy() for _ in range(n)]
