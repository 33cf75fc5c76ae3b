// copy_ops.cu — all-gather (SURVEY K2 with the K6 un-flatten copies fused away) and
// broadcast (K4), each of one tensor or of a tensor list, and the flag-only barrier (K7).
// These kernels move bytes; they do not depend on the element type.  The staged protocols of
// both collectives live in staged.cuh; each kernel here says where a unit comes from and goes.
#include "policy.h"
#include "staged.cuh"
#include "tensor_table.cuh"

namespace b200 {

struct AGArgs {
  const char *in;
  char *outs[kMaxRanks];
  size_t nbytes;  // per rank
  size_t staging_bytes;
};

__global__ void __launch_bounds__(kThreads, 1) allgather_kernel(DevComm c, AGArgs a) {
  const Units un = make_units(a.nbytes);
  const bool in_al = is_aligned16(a.in);
  allgather_body(
      c, a.staging_bytes, un.total(), un.total(), [&](size_t u) { return load_user_unit(a.in, u, un, in_al); },
      [&](size_t u) { return PeerParts<char *>{a.outs, u, un}; });
}

// One window of b200_allgatherv: units [w * W, (w + 1) * W) of every rank's part, W = staging_bytes / 16.
// in and outs[p] point at the window's first byte of their part; nbytes[p] is what of rank p's part
// falls in the window (0 once it is exhausted or empty), units = the largest ceil(nbytes[p] / 16).
struct AGVArgs {
  const char *in;
  char *outs[kMaxRanks];
  size_t nbytes[kMaxRanks];
  size_t units;
  size_t staging_bytes;
};

// Unit u of the uneven parts: rank p's part has it while u < ceil(nbytes[p] / 16).
struct AGVUnit {
  const AGVArgs &a;
  size_t u;
  __device__ __forceinline__ bool has(int p) const { return u < make_units(a.nbytes[p]).total(); }
  __device__ __forceinline__ void store(int p, uint4 v) const {
    const Units un = make_units(a.nbytes[p]);
    if (u < un.total()) store_user_unit(a.outs[p], u, un, is_aligned16(a.outs[p]), v);
  }
};

// The grid (pick_blocks on the window's largest part), the unit -> CTA mapping (grid-stride over
// [0, units)) and the number of launches are functions of the size list, staging_bytes and the
// grid cap alone, never of this rank's own size or alignment.  A rank whose part is exhausted
// still launches and crosses the barrier (DESIGN.md §3: every rank makes every launch).
__global__ void __launch_bounds__(kThreads, 1) allgatherv_kernel(DevComm c, AGVArgs a) {
  const Units mine_un = make_units(a.nbytes[c.rank]);
  const bool in_al = is_aligned16(a.in);
  allgather_body(
      c, a.staging_bytes, mine_un.total(), a.units, [&](size_t u) { return load_user_unit(a.in, u, mine_un, in_al); },
      [&](size_t u) { return AGVUnit{a, u}; });
}

struct BcastArgs {
  char *buf;
  size_t nbytes;
  size_t staging_bytes;
  int root;
};

template <bool NVLS>
__global__ void __launch_bounds__(kThreads, 1) broadcast_kernel(DevComm c, BcastArgs a) {
  const Units un = make_units(a.nbytes);
  const bool al = is_aligned16(a.buf);
  broadcast_body<NVLS>(
      c, a.staging_bytes, a.root, un.total(), [&](size_t u) { return load_user_unit(a.buf, u, un, al); },
      [&](size_t u, uint4 v) { store_user_unit(a.buf, u, un, al, v); });
}

// One window of a table's packed stream (tensor_table.cuh): units [u0, u0 + units), at most one
// staging slot.  The table stays in parameter space (__grid_constant__), indexed in place.
struct BcastTableArgs {
  P2PTable t;
  size_t u0;
  size_t units;
  size_t staging_bytes;
  int root;
};

template <bool NVLS>
__global__ void __launch_bounds__(kThreads, 1)
    broadcast_table_kernel(DevComm c, const __grid_constant__ BcastTableArgs a) {
  broadcast_body<NVLS>(
      c, a.staging_bytes, a.root, a.units, [&](size_t u) { return table_load_unit(a.t, a.u0 + u); },
      [&](size_t u, uint4 v) { table_store_unit(a.t, a.u0 + u, v); });
}

// One window [u0, u0 + units) of a table's packed stream of input units, at most one staging slot.
struct AGTableArgs {
  P2PTable t;                           // the inputs
  char *outs[kP2PTableMax][kMaxRanks];  // outs[k][p]: packed entry k's output for rank p
  size_t u0;
  size_t units;
  size_t staging_bytes;
};
static_assert(fits_param_space<AGTableArgs>(), "all-gather table exceeds the kernel parameter space");

__global__ void __launch_bounds__(kThreads, 1)
    allgather_table_kernel(DevComm c, const __grid_constant__ AGTableArgs a) {
  allgather_body(
      c, a.staging_bytes, a.units, a.units, [&](size_t u) { return table_load_unit(a.t, a.u0 + u); },
      [&](size_t u) {
        const int k = table_entry(a.t.ustart, a.t.count, a.u0 + u);
        return PeerParts<char *>{a.outs[k], a.u0 + u - a.t.ustart[k], make_units(a.t.nbytes[k])};
      });
}

__global__ void barrier_kernel(DevComm c) {
  const uint32_t ep = c.st->launch_ctr * 4u;
  cta_barrier_all(c, ep + 1);
  finish_launch(c);
}

// a kernel of this file's CUDA module, for preload_kernels() (bootstrap.cu)
const void *copy_ops_module_anchor() { return reinterpret_cast<const void *>(&barrier_kernel); }

}  // namespace b200

using namespace b200;

extern "C" int b200_allgather(b200_comm_t c, const void *in, void *const *outs, size_t count,
                              int dtype, void *stream_) {
  int rc;
  size_t es;
  if ((rc = check_usable(c)) || (rc = check_dtype(dtype, &es))) return rc;
  if (count == 0) return B200_OK;
  if (!in || !outs) return null_tensor_error();
  for (int p = 0; p < c->world; ++p)
    if (!outs[p]) {
      set_error("output tensor %d is null", p);
      return B200_ERR_INVALID;
    }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  const size_t total = count * es;
  if (c->world == 1) {
    if (outs[0] != in) B200_CHECK_CUDA(cudaMemcpyAsync(outs[0], in, total, cudaMemcpyDeviceToDevice, stream));
    return B200_OK;
  }
  // Large aligned operands: the pull kernel (TMA copy-in + bulk loads of the peers' slots straight
  // into the caller's output tensors, allreduce_pipe.cu).
  bool aligned = is_aligned16(in) && (total & 15) == 0 && pipe_fits(c);
  for (int p = 0; p < c->world; ++p) aligned = aligned && is_aligned16(outs[p]);
  if (aligned && ag_pull_pays_off(c, total) && pipe_runs(c, PIPE_GATHER)) {
    return for_each_piece(total, pipe_plan(c, PIPE_GATHER).max_bytes, [&](size_t done, size_t nbytes) {
      char *o[kMaxRanks] = {};
      for (int p = 0; p < c->world; ++p) o[p] = static_cast<char *>(outs[p]) + done;
      return launch_allgather_pull(c, static_cast<const char *>(in) + done, o, nbytes, stream);
    });
  }
  return for_each_piece(total, c->staging_bytes, [&](size_t done, size_t nbytes) -> int {
    AGArgs a{};
    a.in = static_cast<const char *>(in) + done;
    for (int p = 0; p < c->world; ++p) a.outs[p] = static_cast<char *>(outs[p]) + done;
    a.nbytes = nbytes;
    a.staging_bytes = c->staging_bytes;
    return launch_staged(c, allgather_kernel, a, make_units(nbytes).total(), stream);
  });
}

extern "C" int b200_allgatherv(b200_comm_t c, const void *in, const size_t *counts, void *const *outs, int dtype,
                               void *stream_) {
  int rc;
  size_t es;
  if ((rc = check_usable(c)) || (rc = check_dtype(dtype, &es)) || (rc = check_list(c->world, counts && outs)))
    return rc;
  const int n = c->world;
  size_t nbytes[kMaxRanks] = {};
  bool even = true;
  for (int p = 0; p < n; ++p) {
    nbytes[p] = counts[p] * es;
    even = even && counts[p] == counts[0];
  }
  if ((rc = check_list_ptrs(outs, nbytes, n))) return rc;
  if (nbytes[c->rank] && !in) return null_tensor_error();
  if (even) return b200_allgather(c, in, outs, counts[0], dtype, stream_);  // also world 1
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  AGVArgs a{};
  a.staging_bytes = c->staging_bytes;
  const VPlan plan = v_plan(nbytes, n, c->staging_bytes / 16);
  return for_each_piece(plan.max_units, plan.window_units, [&](size_t u0, size_t units) -> int {
    for (int p = 0; p < n; ++p) {
      a.nbytes[p] = v_window_bytes(nbytes[p], u0, units);
      a.outs[p] = a.nbytes[p] ? static_cast<char *>(outs[p]) + (u0 << 4) : nullptr;
    }
    a.in = a.nbytes[c->rank] ? static_cast<const char *>(in) + (u0 << 4) : nullptr;
    a.units = units;
    return launch_staged(c, allgatherv_kernel, a, units, stream);
  });
}

extern "C" int b200_broadcast(b200_comm_t c, void *buf, size_t count, int dtype, int root,
                              void *stream_) {
  int rc;
  size_t es;
  if ((rc = check_usable(c)) || (rc = check_dtype(dtype, &es)) || (rc = check_rank(c, root, "root"))) return rc;
  if (count == 0 || c->world == 1) return B200_OK;
  if (!buf) return null_tensor_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  return for_each_piece(count * es, c->staging_bytes, [&](size_t done, size_t nbytes) -> int {
    const BcastArgs a{static_cast<char *>(buf) + done, nbytes, c->staging_bytes, root};
    return launch_staged(c, broadcast_nvls(c, nbytes) ? broadcast_kernel<true> : broadcast_kernel<false>, a,
                         make_units(nbytes).total(), stream);
  });
}

extern "C" int b200_broadcast_multi(b200_comm_t c, void *const *bufs, const size_t *nbytes, int ntensors, int root,
                                    void *stream_) {
  int rc;
  if ((rc = check_usable(c)) || (rc = check_rank(c, root, "root")) ||
      (rc = check_list(ntensors, bufs && nbytes)) || (rc = check_list_ptrs(bufs, nbytes, ntensors)))
    return rc;
  if (ntensors == 0 || c->world == 1) return B200_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  // One launch per window of at most one staging slot of each table's packed stream.
  BcastTableArgs a{};
  a.staging_bytes = c->staging_bytes;
  a.root = root;
  return for_each_window(a.t, bufs, nbytes, ntensors, c->staging_bytes / 16, [](int, int) {},
                         [&](size_t done, size_t units) -> int {
                           a.u0 = done;
                           a.units = units;
                           return launch_staged(c,
                                                broadcast_nvls(c, units * 16) ? broadcast_table_kernel<true>
                                                                              : broadcast_table_kernel<false>,
                                                a, units, stream);
                         });
}

extern "C" int b200_allgather_multi(b200_comm_t c, const void *const *ins, const size_t *nbytes, int ntensors,
                                    void *const *outs, void *stream_) {
  int rc;
  if ((rc = check_usable(c)) || (rc = check_list(ntensors, ins && nbytes && outs)) ||
      (rc = check_list_ptrs(ins, nbytes, ntensors)) ||
      (rc = check_list_rank_ptrs(outs, nbytes, ntensors, c->world, "output")))
    return rc;
  if (ntensors == 0) return B200_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  const int n = c->world;
  if (n == 1) return copy_list_local(outs, ins, nbytes, ntensors, stream);
  // One launch per window of at most one staging slot of each table's stream of input units.
  AGTableArgs a{};
  a.staging_bytes = c->staging_bytes;
  return for_each_window(
      a.t, const_cast<void *const *>(ins), nbytes, ntensors, c->staging_bytes / 16,
      [&](int k, int i) {
        for (int p = 0; p < n; ++p) a.outs[k][p] = static_cast<char *>(outs[size_t(i) * n + p]);
      },
      [&](size_t done, size_t units) -> int {
        a.u0 = done;
        a.units = units;
        return launch_staged(c, allgather_table_kernel, a, units, stream);
      });
}

extern "C" int b200_barrier(b200_comm_t c, void *stream_) {
  int rc = check_usable(c);
  if (rc) return rc;
  if (c->world == 1) return B200_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  barrier_kernel<<<1, 32, 0, stream>>>(c->dev());
  B200_LAUNCH_CHECK(c);
  return B200_OK;
}
