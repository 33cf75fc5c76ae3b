"""DDP's per-forward buffer sync as one b200_broadcast_multi launch (B200DistributedDataParallel,
built by prepare_model(parallel_strategy="ddp")), with real worker processes as in test_gpu_train.py.

The model built by prepare_model and a plain DistributedDataParallel model on the same b200 group
must keep bit-identical parameters and buffers on every rank, step after step, with per-rank inputs
that make every rank's BatchNorm statistics differ before each sync.
"""
import os
import sys
import tempfile

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, init_file, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    import torch.nn as nn
    from torch.distributed.algorithms.join import Join
    from torch.nn.parallel import DistributedDataParallel

    from ray_b200 import train as T

    ndev = torch.cuda.device_count()
    os.environ["LOCAL_RANK"] = str(rank if ndev >= world else 0)
    device = T.get_device()
    torch.cuda.set_device(device)
    T.setup_torch_process_group(T.DEFAULT_GPU_BACKEND, rank, world, f"file://{init_file}", timeout_s=120)
    pg = dist.distributed_c10d._get_default_group()
    assert isinstance(pg, T.B200ProcessGroup)
    if ndev < world:
        x = torch.zeros(1, device=device)
        dist.all_reduce(x)
        pg.comm.set_blocks(32)

    class Net(nn.Module):
        """BatchNorm (fp32 running stats + an int64 counter) and, optionally, a non-contiguous buffer."""

        def __init__(self, strided=False):
            super().__init__()
            self.body = nn.Sequential(nn.Linear(16, 32), nn.BatchNorm1d(32), nn.ReLU(), nn.Linear(32, 4),
                                      nn.BatchNorm1d(4))
            if strided:
                self.register_buffer("extra", torch.arange(12, dtype=torch.float32).view(3, 4).t())

        def forward(self, x):
            y = self.body(x)
            return y + self.extra.sum() if hasattr(self, "extra") else y

    def pair(strided=False, **kwargs):
        torch.manual_seed(0)
        a, b = Net(strided), Net(strided)
        b.load_state_dict(a.state_dict())
        native = T.prepare_model(a, parallel_strategy_kwargs=kwargs or None)
        plain = DistributedDataParallel(b.to(device), device_ids=[device], output_device=device, **kwargs)
        assert isinstance(native, DistributedDataParallel) and type(native) is T.B200DistributedDataParallel
        assert list(native.state_dict()) == list(plain.state_dict())
        return native, plain

    def inputs(step, r):
        gen = torch.Generator().manual_seed(1000 * step + r)
        return torch.randn(8, 16, generator=gen).to(device) * (r + 1), torch.randn(8, 4, generator=gen).to(device)

    def state(m):
        return [t.detach().clone() for t in list(m.module.parameters()) + list(m.module.buffers())]

    def check_same(ma, mb, what):
        for x, y in zip(state(ma), state(mb)):
            assert x.dtype == y.dtype and torch.equal(x, y), what
        # parameters agree across ranks (buffers do not: each forward updates them from local data)
        flat = torch.cat([p.detach().double().flatten() for p in ma.module.parameters()])
        gathered = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(gathered, flat)
        assert all(torch.equal(g, gathered[0]) for g in gathered), what

    def step(m, opt, x, y):
        before = pg.comm.launch_count
        out = m(x)
        launches = pg.comm.launch_count - before
        nn.functional.mse_loss(out, y).backward()
        opt.step()
        opt.zero_grad()
        return launches

    def train(m, steps, extra_shift=False):
        """Launches of each forward's buffer sync.  DDP's second forward also broadcasts the bucket
        layout it rebuilt after the first backward (two launches); that forward is left out."""
        opt = torch.optim.SGD(m.parameters(), lr=0.05)
        launches = []
        for s in range(steps):
            if extra_shift:
                with torch.no_grad():
                    m.module.extra.add_(rank + 1)  # diverges per rank until the next forward's sync
            launches.append(step(m, opt, *inputs(s, rank)))
        return launches[:1] + launches[2:]

    # --- buffer sync: one launch per forward, bit-identical to plain DDP ---------------------
    native, plain = pair()
    ln = train(native, 5)
    lp = train(plain, 5)
    assert ln == [1] * 4, ln
    assert all(l >= 2 for l in lp), lp  # c10d: one broadcast per dtype bucket (fp32, int64)
    check_same(native, plain, "buffer sync")

    # --- broadcast_buffers=False and a model without buffers launch nothing in the forward --------
    native, plain = pair(broadcast_buffers=False)
    assert train(native, 3) == [0, 0]
    train(plain, 3)
    check_same(native, plain, "broadcast_buffers=False")
    torch.manual_seed(0)
    bare = T.prepare_model(nn.Sequential(nn.Linear(16, 4)))
    assert train(bare, 3) == [0, 0]

    # --- a non-contiguous buffer falls back to torch's path, with identical results --------------
    native, plain = pair(strided=True)
    assert not native.module.extra.is_contiguous()
    ln = train(native, 3, extra_shift=True)
    lp = train(plain, 3, extra_shift=True)
    assert ln == lp, (ln, lp)
    check_same(native, plain, "non-contiguous buffer")
    assert torch.equal(native.module.extra.cpu(), plain.module.extra.cpu())

    # --- Join with uneven inputs: the authoritative rank is no longer rank 0 ----------------------
    def train_join(m):
        opt = torch.optim.SGD(m.parameters(), lr=0.05)
        with Join([m]):
            for s in range(2 + rank):
                x, y = inputs(s, rank)
                nn.functional.mse_loss(m(x), y).backward()
                opt.step()
                opt.zero_grad()

    native, plain = pair()
    train_join(native)
    train_join(plain)
    check_same(native, plain, "join")

    torch.cuda.synchronize()
    pg.comm.check_status()
    dist.barrier()
    dist.destroy_process_group()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as f:
        f.write("ok")


@pytest.mark.parametrize("world", [2, 3])
def test_ddp_buffer_sync_is_one_launch_and_matches_plain_ddp(native_lib, world):
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, os.path.join(d, "rdzv"), d), nprocs=world, join=True)
        assert all(open(os.path.join(d, f"ok{r}")).read() == "ok" for r in range(world))
