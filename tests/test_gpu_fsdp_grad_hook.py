"""FSDP's gradient path with ``prepare_model(parallel_strategy="fsdp", gradient_wire_dtype=...)``, with
real worker processes (as Ray Train workers are).  With fewer GPUs than workers the processes share
cuda:0.

For FULL_SHARD, SHARD_GRAD_OP and NO_SHARD with f32 and bf16 wires: three SGD steps against the local
mean-gradient reference, one fused launch per FSDP unit and backward (never FSDP's default
reduce-scatter), and bit-identical full parameters on every rank afterwards.
"""
import os
import sys
import tempfile

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model():
    import torch.nn as nn

    # flat parameter counts 2015 and 455: odd, so FSDP pads every unit at worlds 2 and 4
    return nn.Sequential(nn.Linear(30, 65), nn.ReLU(), nn.Linear(65, 7, bias=False))


def _worker(rank, world, init_file, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    import torch.nn as nn
    from torch.distributed.fsdp import FullyShardedDataParallel as FSDP
    from torch.distributed.fsdp import ShardingStrategy
    from torch.distributed.fsdp.wrap import ModuleWrapPolicy

    from ray_b200 import train as T

    ndev = torch.cuda.device_count()
    os.environ["LOCAL_RANK"] = str(rank if ndev >= world else 0)
    device = T.get_device()
    torch.cuda.set_device(device)
    T.setup_torch_process_group(T.DEFAULT_GPU_BACKEND, rank, world, f"file://{init_file}", timeout_s=120)
    pg = dist.distributed_c10d._get_default_group()
    if ndev < world:
        x = torch.zeros(1, device=device)
        dist.all_reduce(x)
        pg.comm.set_blocks(32)

    # every fused call and its launches; any call of FSDP's default reduce-scatter
    fused, unfused = [], []
    orig_rs, orig_base = pg.grad_reducescatter, pg._reduce_scatter_base

    def counted_rs(out, grad, scale, wire):
        before = pg.comm.launch_count
        work = orig_rs(out, grad, scale, wire)
        fused.append(pg.comm.launch_count - before)
        return work

    def counted_base(*args, **kwargs):
        unfused.append(1)
        return orig_base(*args, **kwargs)

    pg.grad_reducescatter, pg._reduce_scatter_base = counted_rs, counted_base

    # no wire dtype: FSDP's own path, no hook
    plain = T.prepare_model(_model(), parallel_strategy="fsdp")
    assert isinstance(plain, FSDP) and plain._comm_hook is None
    del plain

    loss_fn = nn.MSELoss()
    for strategy in (ShardingStrategy.FULL_SHARD, ShardingStrategy.SHARD_GRAD_OP, ShardingStrategy.NO_SHARD):
        for wire_name, wire in (("f32", torch.float32), ("bf16", torch.bfloat16)):
            what = (world, rank, strategy, wire_name)
            torch.manual_seed(0)
            model = _model()
            assert all(sum(p.numel() for p in m.parameters()) % world for m in model if isinstance(m, nn.Linear))
            ref = _model().to(device)
            ref.load_state_dict(model.state_dict())
            fsdp = T.prepare_model(model, parallel_strategy="fsdp", gradient_wire_dtype=wire,
                                   parallel_strategy_kwargs={"sharding_strategy": strategy,
                                                             "auto_wrap_policy": ModuleWrapPolicy({nn.Linear})})
            assert isinstance(fsdp, FSDP) and fsdp._comm_hook is not None, what
            units = [m for m in FSDP.fsdp_modules(fsdp) if m._handle is not None]
            assert len(units) == 2, what
            sharded = strategy != ShardingStrategy.NO_SHARD
            opt = torch.optim.SGD(fsdp.parameters(), lr=0.1)
            ref_opt = torch.optim.SGD(ref.parameters(), lr=0.1)
            for step in range(3):
                xs = [torch.randn(8, 30, generator=torch.Generator().manual_seed(10 * step + r)).to(device)
                      for r in range(world)]
                ys = [torch.randn(8, 7, generator=torch.Generator().manual_seed(50 * step + r)).to(device)
                      for r in range(world)]
                loss = loss_fn(fsdp(xs[rank]), ys[rank])
                fused.clear()
                unfused.clear()
                before = pg.comm.launch_count
                loss.backward()
                during = pg.comm.launch_count - before
                if sharded:
                    # one fused call of one launch per unit, and FSDP's default path never ran
                    assert fused == [1] * len(units) and not unfused, (what, step, fused, unfused)
                    if strategy == ShardingStrategy.SHARD_GRAD_OP:
                        # parameters stay unsharded through backward: the gradients are all it moves
                        assert during == len(units), (what, step, during)
                opt.step()
                opt.zero_grad()
                ref.zero_grad()
                sum(loss_fn(ref(xs[r]), ys[r]) for r in range(world)).div(world).backward()
                ref_opt.step()
                tol = 1e-5 if wire_name == "f32" else 2e-2
                with FSDP.summon_full_params(fsdp):
                    for (n1, p1), (_, p2) in zip(fsdp.module.named_parameters(), ref.named_parameters()):
                        assert torch.allclose(p1, p2, atol=tol, rtol=tol), (what, step, n1,
                                                                            (p1 - p2).abs().max().item())
            # replicas: the full parameters agree bit for bit on every rank
            with FSDP.summon_full_params(fsdp):
                flat = torch.cat([p.detach().flatten() for p in fsdp.module.parameters()])
            gathered = [torch.empty_like(flat) for _ in range(world)]
            dist.all_gather(gathered, flat)
            for gth in gathered[1:]:
                assert torch.equal(gth, gathered[0]), what
            del fsdp, opt
    torch.cuda.synchronize()
    pg.comm.check_status()
    dist.barrier()
    dist.destroy_process_group()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as f:
        f.write("ok")


@pytest.mark.parametrize("world", [2, 4])
def test_fsdp_fused_gradient_reduce_scatter(native_lib, world):
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, os.path.join(d, "rdzv"), d), nprocs=world, join=True)
        assert all(os.path.exists(os.path.join(d, f"ok{r}")) for r in range(world))
