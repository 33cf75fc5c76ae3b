"""Worker-side helpers: ``prepare_model`` and the fused gradient communication hook.

``prepare_model`` follows ``ray.train.torch.prepare_model`` (python/ray/train/torch/
train_loop_utils.py:153-190,374-482; v2: python/ray/train/v2/torch/train_loop_utils.py:166-250):
move the module to this worker's device, then wrap it in ``DistributedDataParallel`` with
``device_ids=[device]`` when world_size > 1.  The one addition is ``gradient_wire_dtype``:
when set, the DDP buckets are synchronised by ONE fused kernel per bucket (scale by
1/world, cast to the wire dtype, all-reduce, cast back) instead of the reducer's
div + all-reduce (+ compress-hook casts).  Under ``parallel_strategy="fsdp"`` the same
option reduce-scatters each FSDP unit's gradient with one fused kernel (scale, cast,
reduce-scatter, cast back) instead of FSDP's div + fp32 reduce-scatter + div.

Under ``"ddp"`` the wrapper is ``B200DistributedDataParallel``: on a b200 process group the buffer
sync DDP runs before every forward (``broadcast_buffers=True``, the default) is one
``b200_broadcast_multi`` call for all buffers of all dtypes.
"""
from __future__ import annotations

import logging
from typing import Any, Dict, Optional

import torch
import torch.distributed as dist
from torch.nn.parallel import DistributedDataParallel

from .process_group import B200ProcessGroup

logger = logging.getLogger(__name__)


def get_device() -> torch.device:
    """This worker's device (ray.train.torch.get_device): cuda:LOCAL_RANK if GPUs are visible."""
    import os

    if torch.cuda.is_available():
        idx = int(os.environ.get("LOCAL_RANK", "0")) % torch.cuda.device_count()
        return torch.device("cuda", idx)
    return torch.device("cpu")


def _default_b200_group() -> B200ProcessGroup:
    pg = dist.distributed_c10d._get_default_group()
    if isinstance(pg, B200ProcessGroup):
        return pg
    raise RuntimeError("the default process group is not a b200 group; initialise it with "
                       "B200TorchConfig / setup_torch_process_group(backend='b200')")


def b200_grad_hook(wire_dtype: torch.dtype = torch.bfloat16, process_group: Optional[B200ProcessGroup] = None):
    """DDP communication hook: ``model.register_comm_hook(None, b200_grad_hook(torch.bfloat16))``.

    Semantics of torch's ``allreduce_hook`` (wire fp32) / ``bf16_compress_hook`` /
    ``fp16_compress_hook``: the bucket ends up holding the mean gradient.  The whole
    scale-cast-reduce-cast chain is one launch of ``b200_grad_allreduce``."""

    def hook(state, bucket: "dist.GradBucket") -> torch.futures.Future:
        pg = process_group or state or _default_b200_group()
        buf = bucket.buffer()
        if buf.dtype != torch.float32:
            # non-fp32 parameters: plain all-reduce with pre-division, like the default hook
            buf.div_(pg.size())
            return pg.allreduce([buf]).get_future().then(lambda f: f.value()[0])
        return pg.grad_allreduce(buf, 1.0 / pg.size(), wire_dtype)

    # DDP validates the hook's annotations as objects, not strings (distributed.py:_check_comm_hook)
    hook.__annotations__ = {"bucket": dist.GradBucket, "return": torch.futures.Future[torch.Tensor]}
    return hook


def b200_fsdp_grad_hook(wire_dtype: torch.dtype = torch.bfloat16,
                        process_group: Optional[B200ProcessGroup] = None):
    """FSDP communication hook:
    ``fsdp_model.register_comm_hook(fsdp_model.process_group, b200_fsdp_grad_hook(torch.bfloat16))``.

    FSDP calls it as ``hook(state, grad, output)`` for the sharded strategies (``grad`` is the padded
    flat gradient of one FSDP unit, ``output`` its pre-sized shard) and as ``hook(state, grad)`` for
    ``NO_SHARD``.  Either way the result is the mean gradient, as on FSDP's default path.  For fp32
    gradients the whole scale-cast-reduce-cast chain is one launch: ``b200_grad_reducescatter`` into
    ``output``, or ``b200_grad_allreduce`` in place.  ``wait()`` orders FSDP's post-backward stream
    after it without blocking the host."""

    def hook(state, grad: torch.Tensor, output: Optional[torch.Tensor] = None) -> None:
        pg = process_group or state or _default_b200_group()
        n = pg.size()
        if grad.dtype != torch.float32:
            # low-precision gradients (mixed-precision parameters): pre-divide and reduce as they are
            grad.div_(n)
            work = pg.allreduce([grad]) if output is None else pg._reduce_scatter_base(output, grad)
            work.wait()
        elif output is None:
            pg.grad_allreduce(grad, 1.0 / n, wire_dtype).wait()
        else:
            pg.grad_reducescatter(output, grad, 1.0 / n, wire_dtype).wait()

    return hook


class B200DistributedDataParallel(DistributedDataParallel):
    """``DistributedDataParallel`` whose per-forward buffer sync is one ``b200_broadcast_multi``
    call on a b200 process group, instead of c10d's per-dtype flatten, broadcast and per-buffer
    copy-out.  Everything else is DDP's, including the choice of the authoritative rank (which
    ``Join`` moves off rank 0) and user-registered buffer hooks, which DDP calls instead of this
    method."""

    def _distributed_broadcast_coalesced(self, tensors, buffer_size, authoritative_rank=0):
        pg = self.process_group
        if isinstance(pg, B200ProcessGroup) and all(
                t.is_cuda and t.is_contiguous() and t.device == self.device for t in tensors):
            if tensors:
                # stream-ordered: the caller's stream waits for the broadcast, the host does not
                pg.broadcast_multi(list(tensors), authoritative_rank).wait()
            return
        super()._distributed_broadcast_coalesced(tensors, buffer_size, authoritative_rank)


def prepare_model(model: torch.nn.Module, move_to_device: bool = True, parallel_strategy: Optional[str] = "ddp",
                  parallel_strategy_kwargs: Optional[Dict[str, Any]] = None,
                  gradient_wire_dtype: Optional[torch.dtype] = None) -> torch.nn.Module:
    kwargs = dict(parallel_strategy_kwargs or {})
    device = move_to_device if isinstance(move_to_device, torch.device) else get_device()
    if device.type == "cuda":
        torch.cuda.set_device(device)
    if move_to_device:
        model = model.to(device)
    world_size = dist.get_world_size() if dist.is_initialized() else 1
    if parallel_strategy and world_size > 1:
        if parallel_strategy == "ddp":
            if device.type != "cpu":
                kwargs = {"device_ids": [device], "output_device": device, **kwargs}
            model = B200DistributedDataParallel(model, **kwargs)
            if gradient_wire_dtype is not None:
                model.register_comm_hook(None, b200_grad_hook(gradient_wire_dtype))
        elif parallel_strategy == "fsdp":
            if not torch.cuda.is_available():
                raise RuntimeError("FSDP is only available with GPU-enabled training.")
            from torch.distributed.fsdp import FullyShardedDataParallel

            model = FullyShardedDataParallel(model, **kwargs)
            if gradient_wire_dtype is not None:
                # on the root: FSDP gives the hook (with this state) to every unit it wraps
                model.register_comm_hook(model.process_group, b200_fsdp_grad_hook(gradient_wire_dtype))
        else:
            raise ValueError(f"unknown parallel_strategy {parallel_strategy!r}")
    return model
