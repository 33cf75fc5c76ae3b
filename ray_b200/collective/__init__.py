"""``ray_b200.collective`` -- drop-in for ``ray.util.collective`` on B200
(python/ray/util/collective/__init__.py:1-59 exports the same names)."""
from . import types
from .b200_group import B200Group
from .base_group import BaseGroup
from .collective import (
    GroupManager,
    allgather,
    allgather_multi,
    allgatherv,
    allreduce,
    barrier,
    broadcast,
    broadcast_multi,
    create_collective_group,
    destroy_collective_group,
    get_collective_group_size,
    get_group_handle,
    get_rank,
    init_collective_group,
    is_group_initialized,
    recv,
    reduce,
    reducescatter,
    reducescatter_multi,
    reducescatterv,
    send,
    set_member_id,
    synchronize,
    use_manager,
)
from .registry import _global_registry, register_collective_backend
from .types import Backend, ReduceOp

if not _global_registry.is_registered("B200"):
    register_collective_backend("B200", B200Group)

__all__ = [
    "B200Group", "BaseGroup", "Backend", "ReduceOp", "GroupManager", "types",
    "register_collective_backend", "init_collective_group", "create_collective_group",
    "destroy_collective_group", "is_group_initialized", "get_rank", "get_collective_group_size",
    "get_group_handle", "allreduce", "barrier", "reduce", "broadcast", "broadcast_multi", "allgather", "allgather_multi",
    "allgatherv", "reducescatter", "reducescatter_multi", "reducescatterv", "send", "recv", "synchronize",
    "set_member_id", "use_manager",
]
