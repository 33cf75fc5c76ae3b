"""ray_b200 -- Hopper-native (H100) collectives and tensor transport behind Ray's plugin APIs.

The device work lives in ``libb200_collective.so`` (hand-written sm_90a CUDA, C ABI in
``include/b200_collective.h``); this package is the host-side mirror of the reference
interfaces for that path:

    ray_b200.collective   <->  ray.util.collective             (BaseGroup backend "B200")
    ray_b200.channel      <->  ray.experimental.channel        (Communicator + GPU channel)
    ray_b200.train        <->  ray.train.torch                 (TorchConfig / DDP gradient sync)

There is no CPU fallback: importing the native binding without the built library raises.
"""
__version__ = "0.1.0"
