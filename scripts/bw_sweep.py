"""Device-timed bandwidth / latency sweep of the collective kernels (one process, one rank per
GPU, launches replayed from CUDA graphs so host launch overhead does not pollute the numbers).

    python scripts/bw_sweep.py --world 2 [--algos oneshot,twoshot,nvls] [--blocks 0,32,64] \
        [--min 1024 --max 1073741824] [--op allreduce|allgather|reducescatter|broadcast|sendrecv|grad|
                                            grad_rs|grad_rs_unfused|alltoall|alltoall_p2p|
                                            sendrecv_multi|sendrecv_loop|bcast_multi|bcast_loop|
                                            bcast_coalesced|ag_multi|ag_loop|ag_flat|rs_multi|rs_loop|rs_flat|
                                            exchange_batch|exchange_ordered|ring_batch|ring_ordered|
                                            agv|agv_pad|agv_a2a|rsv|rsv_pad|rsv_reduce]
        [--tensors 16,256,resnet50,resnet50_buffers]
        [--split uniform|skew|local|ragged|one_empty] [--wire bfloat16]

Prints one line per (size, algo, blocks): us per launch, algbw, busbw (nccl-tests convention).
--op takes a comma list; the ops then alternate at every size.  For the gradient reduce-scatter
ops the size is one rank's fp32 gradient (all stripes): ``grad_rs`` is the one-launch
b200_grad_reducescatter, ``grad_rs_unfused`` the composition it replaces ((g * scale).to(wire),
a reduce-scatter in the wire type, the cast back to fp32).  For the all-to-all ops the size
is bytes per peer: ``alltoall`` is the one-launch b200_alltoall, ``alltoall_p2p`` the composition
it replaces (n-1 sends on the rank's stream, n-1 receives on a second stream, a local copy).
--split skew gives them MoE-like splits instead: rank r sends size >> k bytes to rank r+k (4:2:1:...,
the own segment the largest); --split local keeps `size` bytes on the rank and sends 16 KiB to each peer.
``sendrecv_multi`` moves a tensor list from rank 0 to rank 1 in one launch per side
(b200_send_multi / b200_recv_multi), ``sendrecv_loop`` with one send and one recv per tensor.
``bcast_multi`` broadcasts a tensor list from rank 0 with b200_broadcast_multi, ``bcast_loop`` with
one b200_broadcast per tensor, and ``bcast_coalesced`` the way DDP's buffer sync does through c10d
today: flatten per dtype, one broadcast per dtype, a copy back into every tensor on the other ranks.
``ag_multi`` all-gathers a tensor list into rank-major outputs (the all_gather_into_tensor layout)
with one b200_allgather_multi call, ``ag_loop`` with one allgather_into per tensor (c10d's coalesced
all-gather before the list call), and ``ag_flat`` the bucket way: copy into one flat buffer, one
b200_allgather, one multi-tensor copy back into the outputs.  ``rs_multi``, ``rs_loop`` and
``rs_flat`` are the same three for reduce-scatter (uint8 SUM).  For these six ops the list is one
rank's part, so every rank holds world_size times it.
The list comes from --tensors: N equal tensors of size / N bytes, ResNet-50's parameter list or
ResNet-50's buffers (fp32 and int64).
``agv`` all-gathers parts of a different size per rank with b200_allgatherv, ``agv_pad`` pads every
part to the largest and runs b200_allgather (the outputs are views of the padded result), ``agv_a2a``
sends the part to every peer with one b200_alltoall.  ``rsv`` reduce-scatters uneven parts with
b200_reducescatterv, ``rsv_pad`` copies the inputs into padded parts and runs b200_reducescatter, and
``rsv_reduce`` makes one b200_reduce per root, as ProcessGroupNCCL does.  Their parts come from
--split: uniform (`size` bytes each), ragged (a few elements off `size`, the last rank a third
shorter), skew (size >> r on rank r) or one_empty (the last rank's part is empty).  Their algbw
counts the sum of all parts.
``exchange_batch`` is a two-rank bidirectional exchange of `size` bytes per direction, both directions
as one b200_p2p_batch per rank; ``exchange_ordered`` is the same exchange as plain send / recv in an
order that cannot wait on itself (even ranks send first, odd ranks receive first).  ``ring_batch`` and
``ring_ordered`` are the same with every rank sending to r+1 and receiving from r-1 (world >= 3).
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from ray_b200 import _native as N
from ray_b200.testing import LocalGroup

ALGOS = {"auto": N.ALGO_AUTO, "oneshot": N.ALGO_ONESHOT, "twoshot": N.ALGO_TWOSHOT, "nvls": N.ALGO_NVLS,
         "ll": N.ALGO_LL}


def time_graphs(g, make_call, iters, reps=3):
    """Capture `iters` launches per rank into one graph per rank; replay; return us per launch
    (max over ranks, best of reps)."""
    graphs = []
    g.run(lambda c, r: make_call(c, r))  # one eager warm-up outside capture (module load, lazy init)
    for r, c in enumerate(g.comms):
        torch.cuda.set_device(g.devices[r])
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=g.streams[r]):
            for _ in range(iters):
                make_call(c, r)
        graphs.append(gr)
    best = None
    for _ in range(reps + 1):
        starts, ends = [], []
        for r in range(g.world_size):
            torch.cuda.set_device(g.devices[r])
            with torch.cuda.stream(g.streams[r]):
                st = torch.cuda.Event(enable_timing=True)
                en = torch.cuda.Event(enable_timing=True)
                st.record()
                graphs[r].replay()
                en.record()
                starts.append(st)
                ends.append(en)
        g.synchronize()
        us = max(s.elapsed_time(e) for s, e in zip(starts, ends)) * 1e3 / iters
        best = us if best is None else min(best, us)
    return best


def alltoall_operands(g, n, numel, dtype, split):
    """ins[r][p] / outs[r][p] for every rank; returns them with the bytes one rank sends."""
    es = torch.empty((), dtype=dtype).element_size()

    def count(p, q):
        if split == "skew":
            return numel >> ((q - p) % n)
        if split == "local":
            return numel if p == q else min(numel, (16 << 10) // es)
        return numel

    counts = [[count(p, q) for q in range(n)] for p in range(n)]
    ins = [[torch.ones(counts[r][p], dtype=dtype, device=g.device(r)) for p in range(n)] for r in range(n)]
    outs = [[torch.empty(counts[p][r], dtype=dtype, device=g.device(r)) for p in range(n)] for r in range(n)]
    return ins, outs, max(sum(row) for row in counts) * es


def alltoall_p2p(c, r, n, outs, ins, side):
    """The host composition the one-launch all-to-all replaces."""
    cur = torch.cuda.current_stream()
    side.wait_stream(cur)
    for step in range(1, n):
        to, frm = (r + step) % n, (r - step) % n
        if ins[to].numel():
            c.send(ins[to], to, stream=cur)
        if outs[frm].numel():
            c.recv(outs[frm], frm, stream=side)
    outs[r].copy_(ins[r])
    cur.wait_stream(side)


def exchange(c, r, k, src, dst, batch):
    """Ranks [0, k) send `src` to r+1 and receive `dst` from r-1 (mod k): one batch, or plain calls with
    even ranks sending first and odd ranks receiving first."""
    if r >= k:
        return
    nxt, prv = (r + 1) % k, (r - 1) % k
    if batch:
        c.p2p_batch([(True, src, nxt), (False, dst, prv)])
    elif r % 2 == 0:
        c.send(src, nxt)
        c.recv(dst, prv)
    else:
        c.recv(dst, prv)
        c.send(src, nxt)


LIST_OPS = ("sendrecv_multi", "sendrecv_loop", "bcast_multi", "bcast_loop", "bcast_coalesced",
            "ag_multi", "ag_loop", "ag_flat", "rs_multi", "rs_loop", "rs_flat")


def tensor_list_specs(recipe, size):
    """(numel, dtype) of each tensor of a --tensors recipe: N equal uint8 tensors of size / N bytes,
    the fp32 parameters of torchvision's ResNet-50 (161 tensors, 102 MB) or its buffers (159 tensors:
    106 fp32, 53 int64, 208 KiB); `size` is ignored by the ResNet-50 recipes."""
    if recipe in ("resnet50", "resnet50_buffers"):
        import torchvision

        m = torchvision.models.resnet50(weights=None)
        return [(t.numel(), t.dtype) for t in (m.parameters() if recipe == "resnet50" else m.buffers())]
    k = int(recipe)
    return [(max(size // k, 1), torch.uint8)] * k


def sendrecv_loop(c, r, sends, recvs):
    """The per-tensor composition the one-launch list send / receive replaces."""
    if r == 0:
        for t in sends:
            c.send(t, 1)
    elif r == 1:
        for t in recvs:
            c.recv(t, 0)


def bcast_loop(c, tensors):
    """One b200_broadcast per tensor: what a weight sync over ray.util.collective.broadcast does."""
    for t in tensors:
        c.broadcast(t, 0)


def bcast_coalesced(c, r, tensors):
    """DDP's buffer sync through c10d's _broadcast_coalesced: one flat bucket per dtype, one
    broadcast per bucket, a copy back into every tensor on the ranks other than the root.  With
    c = None only the torch kernels run (to load them outside any collective)."""
    by_dtype = {}
    for t in tensors:
        by_dtype.setdefault(t.dtype, []).append(t)
    for ts in by_dtype.values():
        flat = torch.cat([t.view(-1) for t in ts])
        if c is not None:
            c.broadcast(flat, 0)
        if r != 0:
            for t, f in zip(ts, flat.split([t.numel() for t in ts])):
                t.view(-1).copy_(f)


def ag_flat(c, n, outs, parts, flat_in, flat_out):
    """The bucket all-gather: copy the list into one flat buffer, one all-gather, one multi-tensor
    copy of every rank's slice back into the rank-major outputs.  With c = None only the torch
    kernels run (to load them outside any collective)."""
    torch.cat(parts, out=flat_in)
    if c is not None:
        c.allgather_into(flat_out, flat_in)
    rows = flat_out.view(n, -1).split([t.numel() for t in parts], dim=1)
    torch._foreach_copy_([o.view(n, -1) for o in outs], list(rows))


def rs_flat(c, n, outs, ins, flat_in, flat_out):
    """The bucket reduce-scatter: one multi-tensor copy of the rank-major inputs into one rank-major
    flat buffer, one reduce-scatter, one multi-tensor copy of the result back into the outputs."""
    rows = flat_in.view(n, -1).split([o.numel() for o in outs], dim=1)
    torch._foreach_copy_(list(rows), [t.view(n, -1) for t in ins])
    if c is not None:
        c.reducescatter_from(flat_out, flat_in, N.SUM)
    torch._foreach_copy_(outs, list(flat_out.split([o.numel() for o in outs])))


V_OPS = ("agv", "agv_pad", "agv_a2a", "rsv", "rsv_pad", "rsv_reduce")


def v_counts(n, numel, split):
    """Element count of every rank's part for the uneven all-gather / reduce-scatter ops."""
    if split == "ragged":  # a few elements off `size`, the last rank shorter (a sharded buffer's remainder)
        return [numel + (p % 3) - 1 for p in range(n - 1)] + [numel - numel // 3]
    if split == "skew":  # 4:2:1...
        return [max(numel >> p, 1) for p in range(n)]
    if split == "one_empty":
        return [numel] * (n - 1) + [0]
    if split == "uniform":
        return [numel] * n
    raise SystemExit(f"--split {split} does not apply to the uneven all-gather / reduce-scatter ops")


def v_call(g, n, op, counts, dtype):
    """The launch sequence of one uneven op on rank r, as call(c, r), and the bytes one rank gathers
    (all-gather) or reduces (reduce-scatter) in total.
      agv        b200_allgatherv
      agv_pad    copy the part into a buffer padded to the largest part, b200_allgather, use views
      agv_a2a    b200_alltoall with the part sent to every peer (the one-launch route without agv)
      rsv        b200_reducescatterv
      rsv_pad    copy the n inputs into padded parts, b200_reducescatter, use a view of the output
      rsv_reduce one b200_reduce per root (ProcessGroupNCCL's uneven reduce-scatter)"""
    m = max(counts)
    dev = g.device
    mine = [torch.ones(counts[r], dtype=dtype, device=dev(r)) for r in range(n)]
    if op == "agv":
        outs = [[torch.empty(k, dtype=dtype, device=dev(r)) for k in counts] for r in range(n)]
        call = lambda c, r: c.allgatherv(outs[r], mine[r])  # noqa: E731
    elif op == "agv_pad":
        pad_in = [torch.zeros(m, dtype=dtype, device=dev(r)) for r in range(n)]
        pad_out = [torch.empty(n * m, dtype=dtype, device=dev(r)) for r in range(n)]

        def call(c, r):
            pad_in[r][:counts[r]].copy_(mine[r])
            c.allgather_into(pad_out[r], pad_in[r])
    elif op == "agv_a2a":
        outs = [[torch.empty(k, dtype=dtype, device=dev(r)) for k in counts] for r in range(n)]
        call = lambda c, r: c.alltoall(outs[r], [mine[r]] * n)  # noqa: E731
    else:
        ins = [[torch.ones(k, dtype=dtype, device=dev(r)) for k in counts] for r in range(n)]
        if op == "rsv":
            call = lambda c, r: c.reducescatterv(mine[r], ins[r], N.SUM)  # noqa: E731
        elif op == "rsv_pad":
            pad_in = [torch.zeros(n, m, dtype=dtype, device=dev(r)) for r in range(n)]
            pad_out = [torch.empty(m, dtype=dtype, device=dev(r)) for r in range(n)]

            def call(c, r):
                torch._foreach_copy_([pad_in[r][q, :counts[q]] for q in range(n)], ins[r])
                c.reducescatter_from(pad_out[r], pad_in[r].view(-1), N.SUM)
        elif op == "rsv_reduce":
            call = lambda c, r: [c.reduce(ins[r][q], q, N.SUM) for q in range(n)]  # noqa: E731
        else:
            raise SystemExit(f"unknown op {op}")
    # load the torch copy kernels outside any collective (see the grad_rs_unfused branch of main)
    for r in range(n):
        with torch.cuda.device(g.devices[r]):
            if op == "agv_pad":
                pad_in[r][:counts[r]].copy_(mine[r])
            elif op == "rsv_pad":
                torch._foreach_copy_([pad_in[r][q, :counts[q]] for q in range(n)], ins[r])
    es = torch.empty((), dtype=dtype).element_size()
    return call, sum(counts) * es


def grad_rs_unfused(c, out, grad, wout, scale, wire):
    """The composition the fused gradient reduce-scatter replaces: scale, cast to the wire type,
    reduce-scatter in the wire type, cast the shard back into the fp32 output."""
    c.reducescatter_from(wout, (grad * scale).to(wire), N.SUM)
    out.copy_(wout)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--algos", default="auto")
    ap.add_argument("--blocks", default="0")
    ap.add_argument("--min", type=int, default=1 << 10)
    ap.add_argument("--max", type=int, default=1 << 30)
    ap.add_argument("--step", type=int, default=4, help="size multiplier between points")
    ap.add_argument("--op", default="allreduce")
    ap.add_argument("--dtype", default="float32")
    ap.add_argument("--symm", action="store_true", help="operands in the symmetric heap (zero copy)")
    ap.add_argument("--nvls-min-world", type=int, default=-1)
    ap.add_argument("--nvls-ctas", default="-1", help="comma list of CTA counts for the NVLS reduce phase")
    ap.add_argument("--split", default="uniform", choices=["uniform", "skew", "local", "ragged", "one_empty"],
                    help="all-to-all ops: bytes per peer; agv / rsv ops: part per rank (see above)")
    ap.add_argument("--wire", default="bfloat16", help="wire dtype of the grad_rs ops")
    ap.add_argument("--tensors", default="1",
                    help="list ops: comma list of recipes, N (N equal tensors of size / N bytes), "
                         "resnet50 (its fp32 parameter list) or resnet50_buffers (its fp32 and int64 "
                         "buffers); the resnet50 recipes are timed once")
    args = ap.parse_args()
    n = args.world
    dtype = getattr(torch, args.dtype)
    heap = (args.max + (4 << 20)) if args.symm else 0
    g = LocalGroup(n, timeout_ms=20000, staging_bytes=512 << 20, heap_bytes=heap, inbox_bytes=64 << 20)
    print(f"# world={n} devices={g.devices} shared={g.shared_gpu} multicast={g.has_multicast} op={args.op} "
          f"dtype={args.dtype} symm={args.symm}")
    for c in g.comms:
        c.set_param(N.PARAM_NVLS_MIN_WORLD, args.nvls_min_world)
    side = [torch.cuda.Stream(device=d) for d in g.devices]  # receive stream of alltoall_p2p
    size = args.min
    es = torch.empty((), dtype=dtype).element_size()
    while size <= args.max:
        numel = size // es
        iters = 50 if size <= (1 << 20) else (20 if size <= (64 << 20) else 6)
        for blocks in [int(b) for b in args.blocks.split(",")]:
            if not g.shared_gpu:
                for c in g.comms:
                    c.set_blocks(blocks)
            for aname, nctas in [(a, int(x)) for a in args.algos.split(",") for x in args.nvls_ctas.split(",")]:
                algo = ALGOS[aname]
                for c in g.comms:
                    c.set_param(N.PARAM_NVLS_CTAS, nctas)
                if algo == N.ALGO_NVLS and not g.has_multicast:
                    continue
                if algo == N.ALGO_ONESHOT and size > (8 << 20):
                    continue
                if algo == N.ALGO_LL and size > (64 << 10):
                    continue
                for op in args.op.split(","):
                    if op in LIST_OPS:
                        continue  # timed per recipe below
                    if args.symm:
                        for c in g.comms:
                            c.symm_reset()
                        xs = [g.comms[r].symm_empty((numel,), dtype) for r in range(n)]
                        for x in xs:
                            x.fill_(1)
                    else:
                        xs = [torch.ones(numel, dtype=dtype, device=g.device(r)) for r in range(n)]
                    if op == "allreduce":
                        call = lambda c, r: c.allreduce(xs[r], N.SUM, algo=algo)  # noqa: E731
                        factor = 2 * (n - 1) / n
                    elif op == "grad":
                        call = lambda c, r: c.grad_allreduce(xs[r], 1.0 / n, torch.bfloat16)  # noqa: E731
                        factor = 2 * (n - 1) / n
                    elif op == "allgather":
                        outs = [torch.empty(n * numel, dtype=dtype, device=g.device(r)) for r in range(n)]
                        call = lambda c, r: c.allgather_into(outs[r], xs[r])  # noqa: E731
                        factor = (n - 1)  # S_total = n*size; busbw = n*size/t*(n-1)/n
                    elif op == "reducescatter":
                        ins = [torch.ones(n * numel, dtype=dtype, device=g.device(r)) for r in range(n)]
                        call = lambda c, r: c.reducescatter_from(xs[r], ins[r], N.SUM)  # noqa: E731
                        factor = (n - 1)
                    elif op in ("grad_rs", "grad_rs_unfused"):
                        # size = one rank's fp32 gradient (all n stripes); out = its shard
                        grads = [torch.ones(size // 4, device=g.device(r)) for r in range(n)]
                        outs = [torch.empty(size // 4 // n, device=g.device(r)) for r in range(n)]
                        wire = getattr(torch, args.wire)
                        if op == "grad_rs":
                            call = lambda c, r: c.grad_reducescatter(outs[r], grads[r], 1.0 / n, wire)  # noqa: E731
                        else:
                            wouts = [torch.empty(size // 4 // n, dtype=wire, device=g.device(r)) for r in range(n)]
                            call = lambda c, r: grad_rs_unfused(c, outs[r], grads[r], wouts[r], 1.0 / n, wire)  # noqa: E731
                            # run the torch kernels once outside any collective: a kernel's first launch
                            # may load its module, which waits for the running grids -- and rank 0's
                            # reduce-scatter grid waits for rank 1, which the host has not issued yet
                            for r in range(n):
                                with torch.cuda.device(g.devices[r]):
                                    (grads[r] * (1.0 / n)).to(wire)
                                    outs[r].copy_(wouts[r])
                        factor = (n - 1) / n
                    elif op == "broadcast":
                        call = lambda c, r: c.broadcast(xs[r], 0)  # noqa: E731
                        factor = 1.0
                    elif op == "sendrecv":
                        call = lambda c, r: (c.send(xs[0], 1) if r == 0 else (c.recv(xs[1], 0) if r == 1 else None))  # noqa: E731
                        factor = 1.0
                    elif op in ("alltoall", "alltoall_p2p"):
                        ins, outs, nbytes = alltoall_operands(g, n, numel, dtype, args.split)
                        if op == "alltoall":
                            call = lambda c, r: c.alltoall(outs[r], ins[r])  # noqa: E731
                        else:
                            call = lambda c, r: alltoall_p2p(c, r, n, outs[r], ins[r], side[r])  # noqa: E731
                        factor = (n - 1) / n  # nccl-tests all-to-all: busbw = algbw * (n-1)/n
                    elif op in V_OPS:
                        call, nbytes = v_call(g, n, op, v_counts(n, numel, args.split), dtype)
                        factor = (n - 1) / n  # of the bytes gathered / reduced per rank
                    elif op in ("exchange_batch", "exchange_ordered", "ring_batch", "ring_ordered"):
                        k = n if op.startswith("ring") else 2
                        if k < 3 and op.startswith("ring"):
                            raise SystemExit(f"{op} needs --world 3 or more")
                        dsts = [torch.empty(numel, dtype=dtype, device=g.device(r)) for r in range(n)]
                        batch = op.endswith("batch")
                        call = lambda c, r: exchange(c, r, k, xs[r], dsts[r], batch)  # noqa: E731
                        factor = 1.0  # algbw: bytes one rank sends (and receives) per launch sequence
                    else:
                        raise SystemExit(f"unknown op {op}")
                    torch.cuda.synchronize()
                    us = time_graphs(g, call, iters)
                    algbw = (nbytes if op.startswith("alltoall") or op in V_OPS else size) / us / 1e3
                    print(f"{op} {size:>11d} B  algo={aname:8s} blocks={blocks:3d} nvls_ctas={nctas:3d} {us:10.2f} us  "
                          f"algbw={algbw:8.1f} GB/s  busbw={algbw * factor:8.1f} GB/s", flush=True)
                    del xs
        # tensor lists: send / receive rank 0 -> rank 1, broadcast from rank 0; the ops alternate per
        # (size, recipe)
        list_ops = [op for op in args.op.split(",") if op in LIST_OPS]
        for recipe in args.tensors.split(",") if list_ops else []:
            if recipe.startswith("resnet50") and size != args.min:
                continue
            specs = tensor_list_specs(recipe, size)
            sizes = [k * torch.empty((), dtype=dt).element_size() for k, dt in specs]
            sends = [torch.ones(s, dtype=torch.uint8, device=g.device(0)) for s in sizes]
            recvs = [torch.empty(s, dtype=torch.uint8, device=g.device(1)) for s in sizes]
            lists = [[torch.ones(k, dtype=dt, device=g.device(r)) for k, dt in specs] for r in range(n)]
            total = sum(sizes)
            gather = [op for op in list_ops if op[:3] in ("ag_", "rs_")]
            if gather:
                # one rank's part: `parts` (inputs of all-gather, outputs of reduce-scatter) and the
                # rank-major `wholes` (outputs of all-gather, inputs of reduce-scatter)
                parts = [[torch.ones(s, dtype=torch.uint8, device=g.device(r)) for s in sizes] for r in range(n)]
                wholes = [[torch.ones(n * s, dtype=torch.uint8, device=g.device(r)) for s in sizes] for r in range(n)]
                flat_part = [torch.empty(total, dtype=torch.uint8, device=g.device(r)) for r in range(n)]
                flat_whole = [torch.empty(n * total, dtype=torch.uint8, device=g.device(r)) for r in range(n)]
            for r in range(n):
                with torch.cuda.device(g.devices[r]):
                    bcast_coalesced(None, r, lists[r])
                    if gather:
                        ag_flat(None, n, wholes[r], parts[r], flat_part[r], flat_whole[r])
                        rs_flat(None, n, parts[r], wholes[r], flat_whole[r], flat_part[r])
            for op in list_ops:
                if op == "sendrecv_multi":
                    call = lambda c, r: (c.send_multi(sends, 1) if r == 0 else  # noqa: E731
                                         (c.recv_multi(recvs, 0) if r == 1 else None))
                elif op == "sendrecv_loop":
                    call = lambda c, r: sendrecv_loop(c, r, sends, recvs)  # noqa: E731
                elif op == "bcast_multi":
                    call = lambda c, r: c.broadcast_multi(lists[r], 0)  # noqa: E731
                elif op == "bcast_loop":
                    call = lambda c, r: bcast_loop(c, lists[r])  # noqa: E731
                elif op == "ag_multi":
                    call = lambda c, r: c.allgather_into_multi(wholes[r], parts[r])  # noqa: E731
                elif op == "ag_loop":
                    call = lambda c, r: [c.allgather_into(o, t) for o, t in zip(wholes[r], parts[r])]  # noqa: E731
                elif op == "ag_flat":
                    call = lambda c, r: ag_flat(c, n, wholes[r], parts[r], flat_part[r], flat_whole[r])  # noqa: E731
                elif op == "rs_multi":
                    call = lambda c, r: c.reducescatter_from_multi(parts[r], wholes[r], N.SUM)  # noqa: E731
                elif op == "rs_loop":
                    call = lambda c, r: [c.reducescatter_from(o, t, N.SUM) for o, t in zip(parts[r], wholes[r])]  # noqa: E731
                elif op == "rs_flat":
                    call = lambda c, r: rs_flat(c, n, parts[r], wholes[r], flat_whole[r], flat_part[r])  # noqa: E731
                else:
                    call = lambda c, r: bcast_coalesced(c, r, lists[r])  # noqa: E731
                torch.cuda.synchronize()
                us = time_graphs(g, call, iters)
                print(f"{op} {total:>11d} B  tensors={recipe}({len(sizes)}) {us:10.2f} us  "
                      f"algbw={total / us / 1e3:8.1f} GB/s", flush=True)
        size *= args.step
    g.destroy()


if __name__ == "__main__":
    main()
