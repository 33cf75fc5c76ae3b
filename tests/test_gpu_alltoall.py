"""All-to-all(v) in one launch (b200_alltoall / B200Comm.alltoall) and the c10d ops built on it:
all_to_all_single, all_to_all, gather and scatter.

Every result is compared bit for bit: out[r][p] must be exactly the bytes rank p passed as its
in[r].  Runs with one GPU (ranks share it) and with one GPU per rank.
"""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORLDS = [2, 3, 4, 8]


@pytest.fixture(scope="module")
def groups(native_lib):
    from ray_b200.testing import LocalGroup

    cache = {}

    def get(n):
        if n not in cache:
            # 8 MiB inbox: the 40 MiB messages wrap every ring several times
            cache[n] = LocalGroup(n, timeout_ms=15000, staging_bytes=8 << 20, inbox_bytes=8 << 20)
        return cache[n]

    yield get
    for g in cache.values():
        g.destroy()


def _bytes(t):
    return t.contiguous().view(torch.uint8) if t.numel() else torch.empty(0, dtype=torch.uint8, device=t.device)


def _check(ins, outs, n):
    """outs[r][p] == ins[p][r], byte for byte (on the host)."""
    for r in range(n):
        for p in range(n):
            got, want = outs[r][p], ins[p][r]
            if got is None or want is None:
                assert (got is None or got.numel() == 0) and (want is None or want.numel() == 0), (r, p)
                continue
            assert np.array_equal(_bytes(got).cpu().numpy(), _bytes(want).cpu().numpy()), (r, p)


def _host_bytes(rng, nbytes):
    return torch.from_numpy(rng.integers(0, 256, nbytes, dtype=np.uint8))


def _uniform(g, n, size, seed=0):
    """ins[r][p]: views of one buffer per rank, size bytes per peer; outs likewise."""
    rng = np.random.default_rng(seed)
    ins, outs = [], []
    for r in range(n):
        buf = _host_bytes(rng, n * size).to(g.device(r))
        ins.append([buf[p * size:(p + 1) * size] for p in range(n)])
        ob = torch.zeros(n * size, dtype=torch.uint8, device=g.device(r))
        outs.append([ob[p * size:(p + 1) * size] for p in range(n)])
    return ins, outs


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("size", [1, 13, 4096, 1 << 20, 40 << 20])
def test_uniform_sizes(groups, world, size):
    g = groups(world)
    ins, outs = _uniform(g, world, size, seed=size)
    g.run(lambda c, r: c.alltoall(outs[r], ins[r]))
    if size >= (40 << 20):
        # compare on the device: 2 x n^2 x 40 MiB would be a lot of host traffic
        for r in range(world):
            for p in range(world):
                assert torch.equal(outs[r][p], ins[p][r].to(outs[r][p].device)), (r, p)
    else:
        _check(ins, outs, world)


@pytest.mark.parametrize("world", WORLDS)
def test_uneven_splits_with_empty_pairs(groups, world):
    g = groups(world)
    rng = np.random.default_rng(100 + world)
    counts = rng.integers(0, 300_000, (world, world))  # counts[p][q]: elements rank p sends to rank q
    counts[rng.random((world, world)) < 0.3] = 0
    counts[world - 1, :] = 0  # one rank sends nothing at all
    counts[0, 1 % world] = 1
    ins, outs = [], []
    for r in range(world):
        vals = rng.standard_normal(int(counts[r].sum())).astype(np.float32)
        buf = torch.from_numpy(vals).to(g.device(r))
        offs = np.concatenate([[0], np.cumsum(counts[r])])
        ins.append([buf[offs[p]:offs[p + 1]] if counts[r, p] else None for p in range(world)])
        outs.append([torch.full((int(counts[p, r]),), -1.0, device=g.device(r)) for p in range(world)])
    g.run(lambda c, r: c.alltoall(outs[r], ins[r]))
    _check(ins, outs, world)


def _dtype_params():
    from ray_b200.comm import TORCH_DTYPE_MAP

    return [str(d).replace("torch.", "") for d in TORCH_DTYPE_MAP]


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dname", _dtype_params())
def test_every_dtype(groups, world, dname):
    g = groups(world)
    dt = getattr(torch, dname)
    es = torch.empty((), dtype=dt).element_size()
    rng = np.random.default_rng(7 * world)
    numel = [int(x) for x in rng.integers(1, 20_000, world)]  # elements rank p sends to each peer
    ins, outs = [], []
    for r in range(world):
        raw = _host_bytes(rng, world * numel[r] * es)
        if dt == torch.bool:
            raw = raw & 1
        buf = raw.view(dt).to(g.device(r))
        ins.append([buf[p * numel[r]:(p + 1) * numel[r]] for p in range(world)])
        outs.append([torch.zeros(numel[p], dtype=dt, device=g.device(r)) for p in range(world)])
    g.run(lambda c, r: c.alltoall(outs[r], ins[r]))
    _check(ins, outs, world)


@pytest.mark.parametrize("world", WORLDS)
def test_unaligned_and_aligned_operands_in_one_launch(groups, world):
    """Odd peers get views at an odd byte offset (ld/st roles), even peers 16-byte aligned ones with
    bulk-sized chunks (bulk roles): both mechanisms meet in one grid."""
    g = groups(world)
    rng = np.random.default_rng(55)
    size = (1 << 20) + 48  # multiple of 16, chunks >= 32 KiB
    stride = size + 64

    def views(buf):
        return [buf[p * stride + (3 if p % 2 else 0):p * stride + (3 if p % 2 else 0) + size] for p in range(world)]

    ins, outs = [], []
    for r in range(world):
        ins.append(views(_host_bytes(rng, world * stride).view(torch.int8).to(g.device(r))))
        outs.append(views(torch.zeros(world * stride, dtype=torch.int8, device=g.device(r))))
    g.run(lambda c, r: c.alltoall(outs[r], ins[r]))
    _check(ins, outs, world)


@pytest.mark.parametrize("world", WORLDS)
def test_one_launch_per_call(groups, world):
    g = groups(world)
    ins, outs = _uniform(g, world, 70_000, seed=3)
    before = [c.launch_count for c in g.comms]
    g.run(lambda c, r: c.alltoall(outs[r], ins[r]))
    assert [c.launch_count - b for c, b in zip(g.comms, before)] == [1] * world
    _check(ins, outs, world)
    empty = [[torch.empty(0, device=g.device(r)) for _ in range(world)] for r in range(world)]
    before = [c.launch_count for c in g.comms]
    g.run(lambda c, r: c.alltoall(empty[r], [torch.empty(0, device=g.device(r))] * world))
    g.run(lambda c, r: c.alltoall([None] * world, [None] * world))
    assert [c.launch_count for c in g.comms] == before


@pytest.mark.parametrize("world", WORLDS)
def test_interleaves_with_send_recv(groups, world):
    """The sequence numbers of every (peer, ring) carry over between all-to-all and send/recv."""
    g = groups(world)
    ins1, outs1 = _uniform(g, world, 300_000, seed=11)
    g.run(lambda c, r: c.alltoall(outs1[r], ins1[r]))
    rng = np.random.default_rng(12)
    msgs = [_host_bytes(rng, 1 << 20).to(g.device(r)) for r in range(world)]  # fits the inbox: eager
    got = [torch.zeros(1 << 20, dtype=torch.uint8, device=g.device(r)) for r in range(world)]

    def ring(c, r):
        c.send(msgs[r], (r + 1) % world)
        c.recv(got[r], (r - 1) % world)

    g.run(ring)
    ins2, outs2 = _uniform(g, world, 5000, seed=13)
    g.run(lambda c, r: c.alltoall(outs2[r], ins2[r]))
    _check(ins1, outs1, world)
    for r in range(world):
        assert torch.equal(got[r].cpu(), msgs[(r - 1) % world].cpu()), r
    _check(ins2, outs2, world)


@pytest.mark.parametrize("world", [2, 4])
def test_cuda_graph_replay(groups, world):
    g = groups(world)
    size = 200_000
    ins, outs = _uniform(g, world, size, seed=21)
    g.run(lambda c, r: c.alltoall(outs[r], ins[r]))  # eager first: kernel attributes are set outside capture
    graphs = []
    for r, c in enumerate(g.comms):
        torch.cuda.set_device(g.devices[r])
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=g.streams[r]):
            c.alltoall(outs[r], ins[r])
        graphs.append(gr)
    for rep in range(2):
        rng = np.random.default_rng(1000 + rep)
        for r in range(world):
            fresh = _host_bytes(rng, world * size).to(g.device(r))
            for p in range(world):
                ins[r][p].copy_(fresh[p * size:(p + 1) * size])
            for p in range(world):
                outs[r][p].zero_()
        for d in set(g.devices):
            torch.cuda.synchronize(d)
        for r in range(world):
            torch.cuda.set_device(g.devices[r])
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        g.synchronize()
        _check(ins, outs, world)


def test_argument_errors_launch_nothing(groups):
    world = 2
    g = groups(world)
    c, dev = g.comms[0], g.device(0)
    x = torch.arange(64, dtype=torch.float32, device=dev)
    ok_in = [x[:32], x[32:]]
    ok_out = [torch.zeros(32, device=dev), torch.zeros(32, device=dev)]
    before = c.launch_count
    with torch.cuda.device(dev):
        with pytest.raises(RuntimeError, match="world_size"):
            c.alltoall(ok_out[:1], ok_in)
        with pytest.raises(RuntimeError, match="world_size"):
            c.alltoall(ok_out, ok_in + [x])
        with pytest.raises(RuntimeError, match="dtype"):
            c.alltoall([ok_out[0], torch.zeros(32, dtype=torch.float64, device=dev)], ok_in)
        with pytest.raises(RuntimeError, match="contiguous"):
            c.alltoall(ok_out, [x.view(32, 2)[:, 0], x[32:]])
        with pytest.raises(RuntimeError, match="overlaps"):
            c.alltoall([ok_out[0], x[16:48]], ok_in)
        with pytest.raises(RuntimeError, match="own segment"):
            c.alltoall([torch.zeros(31, device=dev), ok_out[1]], ok_in)
        with pytest.raises(ValueError, match="not supported"):
            z = torch.zeros(4, dtype=torch.complex64, device=dev)
            c.alltoall([z, z.clone()], [z.clone(), z.clone()])
        # an own segment whose output is its input is not an overlap: nothing to copy, nothing launched
        c.alltoall([x[:32], None], [x[:32], None])
    torch.cuda.synchronize(dev)
    assert c.launch_count == before
    c.check_status()


def test_grid_cap_below_one_cta_per_role_refuses_on_every_rank(groups):
    """Every rank refuses, whatever its counts: no rank is left spinning for a peer that refused."""
    world = 3
    g = groups(world)
    sms = torch.cuda.get_device_properties(g.devices[0]).multi_processor_count
    restore = max(1, (sms - 4) // max(g.devices.count(d) for d in set(g.devices))) if g.shared_gpu else 0
    ins, outs = _uniform(g, world, 4096, seed=5)
    outs[2] = [None, None, None]  # rank 2 receives nothing and sends only to itself
    ins[2] = [None, None, ins[2][2]]
    outs[2][2] = torch.zeros(4096, dtype=torch.uint8, device=g.device(2))
    for r in range(2):
        ins[r][2] = outs[r][2] = None
    before = [c.launch_count for c in g.comms]
    try:
        for c in g.comms:
            c.set_blocks(2)  # < 2 (n - 1) = 4
        for r, c in enumerate(g.comms):
            with torch.cuda.device(g.devices[r]):
                with pytest.raises(RuntimeError, match="capped"):
                    c.alltoall(outs[r], ins[r])
    finally:
        for c in g.comms:
            c.set_blocks(restore)
    assert [c.launch_count for c in g.comms] == before


# ---------------------------------------------------------------------------------------------
# c10d: spawned worker processes, CUDA result against gloo on identical CPU tensors
# ---------------------------------------------------------------------------------------------
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
    dist.all_reduce(torch.zeros(1, device=device))  # the first CUDA op creates the communicator
    if ndev < world:
        sms = torch.cuda.get_device_properties(device).multi_processor_count
        pg.comm.set_blocks((sms - 8) // world)  # co-resident grids when the workers share one GPU

    def same(cuda_t, cpu_t):
        assert cuda_t.dtype == cpu_t.dtype and cuda_t.shape == cpu_t.shape
        assert torch.equal(cuda_t.cpu().view(torch.uint8), cpu_t.view(torch.uint8))

    rng = np.random.default_rng(2024)  # same stream on every rank: the split matrix agrees
    counts = rng.integers(0, 5000, (world, world))  # counts[p][q]: rows rank p sends to rank q
    counts[0, world - 1] = 0
    gen = torch.Generator().manual_seed(rank)
    launches0 = pg.comm.launch_count

    def one_launch(collective, *args, **kwargs):
        before = pg.comm.launch_count
        collective(*args, **kwargs)
        assert pg.comm.launch_count == before + 1, (collective.__name__, pg.comm.launch_count - before)

    # all_to_all_single, uneven splits, 2-D rows
    src = torch.randn(int(counts[rank].sum()), 3, generator=gen)
    in_splits, out_splits = counts[rank].tolist(), counts[:, rank].tolist()
    ref = torch.empty(sum(out_splits), 3)
    dist.all_to_all_single(ref, src, out_splits, in_splits)
    dst = torch.full((sum(out_splits), 3), -1.0, device=device)
    one_launch(dist.all_to_all_single, dst, src.to(device), out_splits, in_splits)
    same(dst, ref)

    # list form (gloo has no list all_to_all: its reference is the equivalent all_to_all_single)
    ins = [torch.randint(-100, 100, (int(counts[rank, p]),), generator=gen, dtype=torch.int64) for p in range(world)]
    ref = torch.empty(sum(out_splits), dtype=torch.int64)
    dist.all_to_all_single(ref, torch.cat(ins), out_splits, in_splits)
    outs = [torch.zeros(int(counts[p, rank]), dtype=torch.int64, device=device) for p in range(world)]
    one_launch(dist.all_to_all, outs, [t.to(device) for t in ins])
    same(torch.cat(outs), ref)

    # gather / scatter at a non-zero root
    root = world - 1
    mine = torch.randn(1000, generator=gen).to(torch.bfloat16)
    ref = [torch.empty_like(mine) for _ in range(world)] if rank == root else None
    dist.gather(mine, ref, dst=root)
    got = [torch.zeros(1000, dtype=torch.bfloat16, device=device) for _ in range(world)] if rank == root else None
    one_launch(dist.gather, mine.to(device), got, dst=root)
    if rank == root:
        for a, b in zip(got, ref):
            same(a, b)
    # ... with the root's own slot of gather_list being its input tensor (NCCL accepts this too)
    mine_d = mine.to(device)
    got = [torch.zeros(1000, dtype=torch.bfloat16, device=device) for _ in range(world)] if rank == root else None
    if rank == root:
        got[root] = mine_d
    one_launch(dist.gather, mine_d, got, dst=root)
    if rank == root:
        for a, b in zip(got, ref):
            same(a, b)
    root = 1
    parts = [torch.randn(777, generator=gen) for _ in range(world)] if rank == root else None
    ref = torch.empty(777)
    dist.scatter(ref, parts, src=root)
    out = torch.zeros(777, device=device)
    one_launch(dist.scatter, out, [p.to(device) for p in parts] if rank == root else None, src=root)
    same(out, ref)
    # ... with the root's own slot of scatter_list being its output tensor
    out = parts[root].to(device) if rank == root else torch.zeros(777, device=device)
    lst = [out if p == root else parts[p].to(device) for p in range(world)] if rank == root else None
    one_launch(dist.scatter, out, lst, src=root)
    same(out, ref)

    # MoE-style dispatch to the expert's rank and the inverse combine
    tokens = torch.randn(4096, 64, generator=gen).to(device)
    dest = torch.randint(0, world, (4096,), generator=gen).to(device)
    order = torch.argsort(dest, stable=True)
    send_counts = torch.bincount(dest, minlength=world)
    recv_counts = torch.empty_like(send_counts)
    one_launch(dist.all_to_all_single, recv_counts, send_counts)
    sc, rc = send_counts.tolist(), recv_counts.tolist()
    dispatched = torch.empty(sum(rc), 64, device=device)
    one_launch(dist.all_to_all_single, dispatched, tokens[order], rc, sc)
    combined = torch.empty(4096, 64, device=device)
    one_launch(dist.all_to_all_single, combined, dispatched, sc, rc)
    back = torch.empty_like(combined)
    back[order] = combined
    assert torch.equal(back, tokens)

    # split sizes that do not add up raise on every rank before anything is launched
    n_before = pg.comm.launch_count
    bad = [1] * world
    bad[0] += 1
    try:
        dist.all_to_all_single(torch.zeros(world, device=device), torch.zeros(world, device=device), [1] * world, bad)
        raise AssertionError("split sizes that do not sum to dim 0 were accepted")
    except RuntimeError:
        pass
    assert pg.comm.launch_count == n_before

    torch.cuda.synchronize()
    pg.comm.check_status()
    launches = pg.comm.launch_count - launches0
    dist.barrier()
    dist.destroy_process_group()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as f:
        f.write(str(launches))


@pytest.mark.parametrize("world", [2, 4])
def test_c10d_alltoall_gather_scatter_match_gloo(native_lib, world):
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_c10d_worker, args=(world, os.path.join(d, "rdzv"), d), nprocs=world, join=True)
        launches = [int(open(os.path.join(d, f"ok{r}")).read()) for r in range(world)]
        assert launches == [9] * world, launches  # one launch per CUDA collective of the worker
