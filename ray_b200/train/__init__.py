"""``ray_b200.train`` -- the c10d backend + DDP gradient path TorchTrainer / LearnerGroup ride."""
from .process_group import BACKEND_NAME, B200ProcessGroup, B200Work, batch_isend_irecv, register_b200_backend
from .torch_config import (DEFAULT_GPU_BACKEND, B200TorchConfig, resolve_backend, setup_torch_process_group,
                           shutdown_torch, uses_b200)
from .train_loop_utils import (B200DistributedDataParallel, b200_fsdp_grad_hook, b200_grad_hook, get_device,
                               prepare_model)

__all__ = ["BACKEND_NAME", "B200ProcessGroup", "B200Work", "batch_isend_irecv", "register_b200_backend", "B200TorchConfig",
           "DEFAULT_GPU_BACKEND", "resolve_backend", "setup_torch_process_group", "shutdown_torch", "uses_b200",
           "B200DistributedDataParallel", "b200_grad_hook", "b200_fsdp_grad_hook", "get_device", "prepare_model"]
