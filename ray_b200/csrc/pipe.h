// pipe.h — host-side interface of the chunk-pipelined kernels (allreduce_pipe.cu).
#pragma once
#include "kernel_utils.cuh"

namespace b200 {

// Which pipelined kernel runs: for the all-reduce a function of (world, multicast, dtype, op), see
// b200_allreduce.  Geometry of each: pipe_plan() (policy.h).
enum PipeVariant {
  PIPE_NVLS,   // n >= 3: copy-in | multimem.ld_reduce + multimem.st | copy-out
  PIPE_PEER,   // n >= 3: copy-in | peer loads + peer stores         | copy-out
  PIPE_PULL,   // n == 2: copy-in | bulk-load the peer's slot + reduce into the caller's tensor
  PIPE_GATHER  // all-gather: copy-in | bulk-load every peer's slot into the caller's output tensors
};

// `in`/`out` 16-byte aligned, nbytes a multiple of 16 and <= pipe_plan(c, variant).max_bytes
int launch_allreduce_pipe_dyn(b200_comm *c, const char *in, char *out, size_t nbytes, int dtype, int op,
                              int variant, cudaStream_t stream);

// pull all-gather; same operand requirements, nbytes <= pipe_plan(c, PIPE_GATHER).max_bytes
int launch_allgather_pull(b200_comm *c, const char *in, char *const *outs, size_t nbytes, cudaStream_t stream);

}  // namespace b200
