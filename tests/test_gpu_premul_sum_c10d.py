"""c10d's PREMUL_SUM on a b200 group, with real worker processes: ``dist._make_nccl_premul_sum(f)``
for a float and a CUDA-tensor factor, f32 and bf16, through all_reduce, reduce, reduce_scatter_tensor,
an uneven reduce_scatter, a _coalescing_manager block of reduce_scatter_tensor and
all_reduce_coalesced.  Each result is bit-identical to SUM on the pre-scaled input on the same group,
which also shows that the factor survives c10d's trampoline into the Python process group.
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

    def same(a, b, what):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), what

    for dtype in (torch.float32, torch.bfloat16):
        for kind in ("float", "tensor"):
            value = 1 / 3 if kind == "float" else -0.75
            f = value if kind == "float" else torch.tensor([value], dtype=dtype, device=device)
            fT = torch.tensor(value, dtype=dtype, device=device).float()

            def op():
                return dist._make_nccl_premul_sum(f)

            def pre(x):
                return (x.float() * fT).to(dtype)

            gen = torch.Generator().manual_seed(1000 + rank)
            x = (torch.randn(4099 * world, generator=gen) * 3).to(dtype).to(device)
            what = (dtype, kind)

            a, b = x.clone(), pre(x)
            dist.all_reduce(a, op=op())
            dist.all_reduce(b)
            same(a, b, what + ("all_reduce",))

            for root in range(world):
                a, b = x.clone(), pre(x)
                dist.reduce(a, root, op=op())
                dist.reduce(b, root)
                same(a, b if rank == root else x, what + ("reduce", root))

            m = x.numel() // world
            a, b = torch.empty(m, dtype=dtype, device=device), torch.empty(m, dtype=dtype, device=device)
            dist.reduce_scatter_tensor(a, x, op=op())
            dist.reduce_scatter_tensor(b, pre(x))
            same(a, b, what + ("reduce_scatter_tensor",))

            sizes = [1000 + 37 * q for q in range(world)]
            ins = [x[:s].clone() for s in sizes]
            a, b = torch.empty(sizes[rank], dtype=dtype, device=device), torch.empty(sizes[rank], dtype=dtype,
                                                                                      device=device)
            dist.reduce_scatter(a, ins, op=op())
            dist.reduce_scatter(b, [pre(t) for t in ins])
            same(a, b, what + ("reduce_scatter uneven",))

            outs_a = [torch.empty(m // 2, dtype=dtype, device=device) for _ in range(2)]
            outs_b = [torch.empty(m // 2, dtype=dtype, device=device) for _ in range(2)]
            srcs = [x[:m // 2 * world], x[m // 2 * world:m // 2 * world * 2]]
            with dist._coalescing_manager(async_ops=False):
                for o, s in zip(outs_a, srcs):
                    dist.reduce_scatter_tensor(o, s, op=op())
            with dist._coalescing_manager(async_ops=False):
                for o, s in zip(outs_b, srcs):
                    dist.reduce_scatter_tensor(o, pre(s))
            for i in range(2):
                same(outs_a[i], outs_b[i], what + ("coalesced reduce_scatter_tensor", i))

            ta = [x[:777].clone(), x[777:5000].clone()]
            tb = [pre(t) for t in ta]
            dist.all_reduce_coalesced(ta, op=op())
            dist.all_reduce_coalesced(tb)
            for i in range(2):
                same(ta[i], tb[i], what + ("all_reduce_coalesced", i))

    torch.cuda.synchronize()
    pg.comm.check_status()
    dist.barrier()
    dist.destroy_process_group()
    with open(os.path.join(out_dir, f"ok{rank}"), "w") as fh:
        fh.write("ok")


@pytest.mark.parametrize("world", [2, 3])
def test_c10d_premul_sum(native_lib, world):
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, os.path.join(d, "rdzv"), d), nprocs=world, join=True)
        assert all(os.path.exists(os.path.join(d, f"ok{r}")) for r in range(world))
