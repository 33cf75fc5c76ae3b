// reduce_ops.cu — reduce-scatter (SURVEY K3, fusing away the K6 flatten copies) and
// reduce-to-root (a6).
//
// reduce-scatter is push based: rank r reads its n input tensors straight from the
// caller's list and writes tensor q into sub-slot r of rank q's staging slot over
// NVLink (the local copy-in and the transfer are the same instruction stream).  After
// one barrier every rank reduces its n sub-slots from local HBM, rank-ascending, into
// the caller's output tensor.  That protocol is reducescatter_push_body (staged.cuh); the
// tensor and list (b200_reducescatter_multi, windows of a packed tensor table, tensor_table.cuh)
// kernels here and the FSDP gradient kernel (grad.cu) say only where a unit comes from and how
// the reduced unit is stored.  The uneven kernel (b200_reducescatterv) writes the protocol out.
#include <vector>

#include "policy.h"
#include "staged.cuh"
#include "tensor_table.cuh"

namespace b200 {

struct RSArgs {
  const char *ins[kMaxRanks];
  char *out;
  size_t nbytes;  // per tensor
  size_t staging_bytes;
};

// PREMUL_SUM (OP = kOpPremulSum, S = Premul<T>) scales the unit source; the body is the plain ops'.
template <typename T, int OP, typename S>
__device__ __forceinline__ void reducescatter_tensor_body(const DevComm &c, const RSArgs &a, const S &scale) {
  const Units un = make_units(a.nbytes);
  reducescatter_push_body(
      c, a.staging_bytes, un.total(), [&](size_t u) { return scaled(PeerParts<const char *>{a.ins, u, un}, scale); },
      [&](size_t u, const uint4(&v)[kMaxRanks], int n) {
        store_user_unit(a.out, u, un, is_aligned16(a.out), reduce_ranks<T, OP>(v, n));
      });
}
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1) reducescatter_kernel(DevComm c, RSArgs a) {
  reducescatter_tensor_body<T, OP>(c, a, NoScale{});
}
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1) reducescatter_kernel(DevComm c, RSArgs a, PremulArg f) {
  reducescatter_tensor_body<T, OP>(c, a, Premul<T>(f));
}

// One window of b200_reducescatterv: units [w * W, (w + 1) * W) of every rank's output part,
// W = floor(staging_bytes / (16 * n)).  ins[q] and out point at the window's first byte of their
// part; nbytes[q] is what of rank q's part falls in the window (0 once it is exhausted or empty).
// units = the largest ceil(nbytes[q] / 16): every sub-slot is units * 16 bytes, so the n sub-slots
// fit one staging slot and both sides derive the layout from the shared sizes.
struct RSVArgs {
  const char *ins[kMaxRanks];
  char *out;
  size_t nbytes[kMaxRanks];
  size_t units;
  size_t staging_bytes;
};

// reducescatter_push_body's protocol with a size per rank, written out: through the shared body
// this kernel keeps its own part's size live across the barrier and needs up to 7 more registers.
// Rank r pushes the window's units of ins[q] into sub-slot r of rank q's slot, crosses the
// barrier, then reduces its own n sub-slots rank-ascending over its own part's units.  The CTA barrier pairs CTA b of every rank, so the grid (pick_blocks
// on the window's largest part), the unit -> CTA mapping (grid-stride over [0, units)) and the
// number of launches depend only on the size list, staging_bytes and the grid cap -- never on this
// rank's own size or alignment.  A rank whose part is exhausted still launches and crosses the
// barrier (DESIGN.md §3).  Every output element has n contributions, so AVG divides by n.
template <typename T, int OP, typename S>
__device__ __forceinline__ void reducescatterv_body(const DevComm &c, const RSVArgs &a, const S &scale) {
  const uint32_t launch = c.st->launch_ctr;
  const uint32_t ep = launch * 4u;
  const int n = c.world, r = c.rank;
  const size_t U = a.units;
  const size_t sub = U << 4;  // bytes per sub-slot
  const size_t off = staging_slot_offset(launch, a.staging_bytes);
  const size_t stride = size_t(gridDim.x) * kThreads;
  const size_t first = size_t(blockIdx.x) * kThreads + threadIdx.x;

  for (size_t u = first; u < U; u += stride) {
    uint4 v[kMaxRanks];
#pragma unroll
    for (int i = 0; i < kMaxRanks; ++i) {
      if (i < n) {
        int q = r + i;
        if (q >= n) q -= n;
        const Units un = make_units(a.nbytes[q]);
        if (u < un.total()) v[i] = scale(load_user_unit(a.ins[q], u, un, is_aligned16(a.ins[q])));
      }
    }
#pragma unroll
    for (int i = 0; i < kMaxRanks; ++i) {
      if (i < n) {
        int q = r + i;
        if (q >= n) q -= n;
        if (u < make_units(a.nbytes[q]).total()) st_vec(c.data[q] + off + size_t(r) * sub + (u << 4), v[i]);
      }
    }
  }

  if (!cta_barrier_all(c, ep + 1)) {
    finish_launch(c);
    return;
  }

  const Units un = make_units(a.nbytes[r]);
  const size_t mine_U = un.total();
  const bool out_al = is_aligned16(a.out);
  const char *mine = c.data[r] + off;
  for (size_t u = first; u < mine_U; u += stride) {
    uint4 v[kMaxRanks];
#pragma unroll
    for (int p = 0; p < kMaxRanks; ++p)
      if (p < n) v[p] = ld_peer(mine + size_t(p) * sub + (u << 4));
    store_user_unit(a.out, u, un, out_al, reduce_ranks<T, OP>(v, n));
  }
  finish_launch(c);
}
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1) reducescatterv_kernel(DevComm c, RSVArgs a) {
  reducescatterv_body<T, OP>(c, a, NoScale{});
}
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1) reducescatterv_kernel(DevComm c, RSVArgs a, PremulArg f) {
  reducescatterv_body<T, OP>(c, a, Premul<T>(f));
}

// One window [u0, u0 + units) of a table's packed stream of output units; n sub-slots of
// units * 16 bytes fit one staging slot.
struct RSTableArgs {
  P2PTable t;                                // the outputs
  const char *ins[kP2PTableMax][kMaxRanks];  // ins[k][q]: packed entry k's contribution to rank q
  size_t u0;
  size_t units;
  size_t staging_bytes;
};
static_assert(fits_param_space<RSTableArgs>(), "reduce-scatter table exceeds the kernel parameter space");

template <typename T, int OP, typename S>
__device__ __forceinline__ void reducescatter_table_body(const DevComm &c, const RSTableArgs &a, const S &scale) {
  reducescatter_push_body(
      c, a.staging_bytes, a.units,
      [&](size_t u) {
        const int k = table_entry(a.t.ustart, a.t.count, a.u0 + u);
        return scaled(PeerParts<const char *>{a.ins[k], a.u0 + u - a.t.ustart[k], make_units(a.t.nbytes[k])}, scale);
      },
      [&](size_t u, const uint4(&v)[kMaxRanks], int n) { table_store_unit(a.t, a.u0 + u, reduce_ranks<T, OP>(v, n)); });
}
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1)
    reducescatter_table_kernel(DevComm c, const __grid_constant__ RSTableArgs a) {
  reducescatter_table_body<T, OP>(c, a, NoScale{});
}
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1)
    reducescatter_table_kernel(DevComm c, const __grid_constant__ RSTableArgs a, PremulArg f) {
  reducescatter_table_body<T, OP>(c, a, Premul<T>(f));
}

struct ReduceArgs {
  char *buf;
  size_t nbytes;
  size_t staging_bytes;
  int root;
};

// Every rank stages its tensor; the root pulls all n copies and reduces in place.
template <typename T, int OP, typename S>
__device__ __forceinline__ void reduce_body(const DevComm &c, const ReduceArgs &a, const S &scale) {
  const uint32_t launch = c.st->launch_ctr;
  const uint32_t ep = launch * 4u;
  const int n = c.world, r = c.rank;
  const Units un = make_units(a.nbytes);
  const size_t U = un.total();
  const bool al = is_aligned16(a.buf);
  const size_t off = staging_slot_offset(launch, a.staging_bytes);
  const size_t stride = size_t(gridDim.x) * kThreads;
  const size_t first = size_t(blockIdx.x) * kThreads + threadIdx.x;

  char *mine = c.data[r] + off;
  for (size_t u = first; u < U; u += stride) st_vec(mine + (u << 4), scale(load_user_unit(a.buf, u, un, al)));

  if (!cta_barrier_all(c, ep + 1)) {
    finish_launch(c);
    return;
  }

  if (r == a.root) {
    for (size_t u = first; u < U; u += stride) {
      uint4 v[kMaxRanks];
#pragma unroll
      for (int p = 0; p < kMaxRanks; ++p)
        if (p < n) v[p] = ld_peer(c.data[p] + off + (u << 4));
      store_user_unit(a.buf, u, un, al, reduce_ranks<T, OP>(v, n));
    }
  }
  finish_launch(c);
}
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1) reduce_kernel(DevComm c, ReduceArgs a) {
  reduce_body<T, OP>(c, a, NoScale{});
}
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1) reduce_kernel(DevComm c, ReduceArgs a, PremulArg f) {
  reduce_body<T, OP>(c, a, Premul<T>(f));
}

// a kernel of this file's CUDA module, for preload_kernels() (bootstrap.cu)
const void *reduce_ops_module_anchor() { return reinterpret_cast<const void *>(static_cast<void (*)(DevComm, RSArgs)>(&reducescatter_kernel<float, B200_SUM>)); }

}  // namespace b200

using namespace b200;

extern "C" int b200_reducescatter(b200_comm_t c, const void *const *ins, void *out, size_t count,
                                  int dtype, int op, void *stream_) {
  int rc;
  size_t es;
  OpArg oa;
  if ((rc = check_usable(c)) || (rc = check_dtype(dtype, &es)) || (rc = check_op(c, op, dtype, &oa))) return rc;
  if (count == 0) return B200_OK;
  if (!ins || !out) return null_tensor_error();
  for (int p = 0; p < c->world; ++p)
    if (!ins[p]) {
      set_error("input tensor %d is null", p);
      return B200_ERR_INVALID;
    }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  const size_t total = count * es;
  if (c->world == 1) {
    if (oa.op == kOpPremulSum) return launch_premul_scale(c, ins[0], out, total, dtype, oa.premul, stream);
    if (ins[0] != out) B200_CHECK_CUDA(cudaMemcpyAsync(out, ins[0], total, cudaMemcpyDeviceToDevice, stream));
    return B200_OK;
  }
  // n sub-slots of the piece must fit one staging slot; keep pieces 16-byte multiples
  const size_t step = (c->staging_bytes / size_t(c->world)) & ~size_t(15);
  return for_each_piece(total, step, [&](size_t done, size_t nbytes) -> int {
    RSArgs a{};
    for (int p = 0; p < c->world; ++p) a.ins[p] = static_cast<const char *>(ins[p]) + done;
    a.out = static_cast<char *>(out) + done;
    a.nbytes = nbytes;
    a.staging_bytes = c->staging_bytes;
    if (oa.op == kOpPremulSum)
      B200_DISPATCH_PREMUL(dtype, T, {
        return launch_staged(c, reducescatter_kernel<T, kOpPremulSum>, a, make_units(nbytes).total(), stream,
                             oa.premul);
      });
    B200_DISPATCH_DTYPE(dtype, T,
                        B200_DISPATCH_OP(op, OP, { return launch_staged(c, reducescatter_kernel<T, OP>, a,
                                                                        make_units(nbytes).total(), stream); }));
  });
}

extern "C" int b200_reducescatterv(b200_comm_t c, const void *const *ins, const size_t *counts, void *out,
                                   int dtype, int op, void *stream_) {
  int rc;
  size_t es;
  OpArg oa;
  if ((rc = check_usable(c)) || (rc = check_dtype(dtype, &es)) || (rc = check_op(c, op, dtype, &oa)) ||
      (rc = check_list(c->world, ins && counts)))
    return rc;
  const int n = c->world;
  size_t nbytes[kMaxRanks] = {};
  bool even = true;
  for (int q = 0; q < n; ++q) {
    nbytes[q] = counts[q] * es;
    even = even && counts[q] == counts[0];
  }
  if ((rc = check_list_ptrs(const_cast<void *const *>(ins), nbytes, n))) return rc;
  if (nbytes[c->rank] && !out) return null_tensor_error();
  if (even) return b200_reducescatter(c, ins, out, counts[0], dtype, op, stream_);  // also world 1
  void (*kernel)(DevComm, RSVArgs) = nullptr;
  void (*premul_kernel)(DevComm, RSVArgs, PremulArg) = nullptr;
  if (oa.op == kOpPremulSum) B200_DISPATCH_PREMUL(dtype, T, { premul_kernel = reducescatterv_kernel<T, kOpPremulSum>; })
  else B200_DISPATCH_DTYPE(dtype, T, B200_DISPATCH_OP(op, OP, { kernel = reducescatterv_kernel<T, OP>; }));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  RSVArgs a{};
  a.staging_bytes = c->staging_bytes;
  // the n sub-slots of a window fill at most one staging slot
  const VPlan plan = v_plan(nbytes, n, c->staging_bytes / (16 * size_t(n)));
  return for_each_piece(plan.max_units, plan.window_units, [&](size_t u0, size_t units) -> int {
    for (int q = 0; q < n; ++q) {
      a.nbytes[q] = v_window_bytes(nbytes[q], u0, units);
      a.ins[q] = a.nbytes[q] ? static_cast<const char *>(ins[q]) + (u0 << 4) : nullptr;
    }
    a.out = a.nbytes[c->rank] ? static_cast<char *>(out) + (u0 << 4) : nullptr;
    a.units = units;
    return premul_kernel ? launch_staged(c, premul_kernel, a, units, stream, oa.premul)
                         : launch_staged(c, kernel, a, units, stream);
  });
}

extern "C" int b200_reducescatter_multi(b200_comm_t c, const void *const *ins, void *const *outs,
                                        const size_t *counts, int ntensors, int dtype, int op, void *stream_) {
  int rc;
  size_t es;
  OpArg oa;
  if ((rc = check_usable(c)) || (rc = check_dtype(dtype, &es)) || (rc = check_op(c, op, dtype, &oa)) ||
      (rc = check_list(ntensors, ins && outs && counts)))
    return rc;
  std::vector<size_t> nbytes(static_cast<size_t>(ntensors));
  for (int i = 0; i < ntensors; ++i) nbytes[i] = counts[i] * es;
  if ((rc = check_list_ptrs(outs, nbytes.data(), ntensors)) ||
      (rc = check_list_rank_ptrs(ins, nbytes.data(), ntensors, c->world, "input")))
    return rc;
  if (ntensors == 0) return B200_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  const int n = c->world;
  if (n == 1 && oa.op == kOpPremulSum) {
    for (int i = 0; i < ntensors; ++i)
      if ((rc = launch_premul_scale(c, ins[i], outs[i], nbytes[i], dtype, oa.premul, stream))) return rc;
    return B200_OK;
  }
  if (n == 1) return copy_list_local(outs, ins, nbytes.data(), ntensors, stream);
  void (*kernel)(DevComm, const RSTableArgs) = nullptr;
  void (*premul_kernel)(DevComm, const RSTableArgs, PremulArg) = nullptr;
  if (oa.op == kOpPremulSum)
    B200_DISPATCH_PREMUL(dtype, T, { premul_kernel = reducescatter_table_kernel<T, kOpPremulSum>; })
  else B200_DISPATCH_DTYPE(dtype, T, B200_DISPATCH_OP(op, OP, { kernel = reducescatter_table_kernel<T, OP>; }));
  // One launch per window of each table's stream of output units; the n sub-slots of a window
  // fill at most one staging slot.
  RSTableArgs a{};
  a.staging_bytes = c->staging_bytes;
  return for_each_window(
      a.t, outs, nbytes.data(), ntensors, c->staging_bytes / (16 * size_t(n)),
      [&](int k, int i) {
        for (int q = 0; q < n; ++q) a.ins[k][q] = static_cast<const char *>(ins[size_t(i) * n + q]);
      },
      [&](size_t done, size_t units) -> int {
        a.u0 = done;
        a.units = units;
        return premul_kernel ? launch_staged(c, premul_kernel, a, units, stream, oa.premul)
                             : launch_staged(c, kernel, a, units, stream);
      });
}

extern "C" int b200_reduce(b200_comm_t c, void *buf, size_t count, int dtype, int op, int root,
                           void *stream_) {
  int rc;
  size_t es;
  OpArg oa;
  if ((rc = check_usable(c)) || (rc = check_dtype(dtype, &es)) || (rc = check_op(c, op, dtype, &oa)) ||
      (rc = check_rank(c, root, "root")))
    return rc;
  if (count == 0) return B200_OK;
  if (!buf) return null_tensor_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (c->world == 1)
    return oa.op == kOpPremulSum ? launch_premul_scale(c, buf, buf, count * es, dtype, oa.premul, stream) : B200_OK;
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  return for_each_piece(count * es, c->staging_bytes, [&](size_t done, size_t nbytes) -> int {
    const ReduceArgs a{static_cast<char *>(buf) + done, nbytes, c->staging_bytes, root};
    if (oa.op == kOpPremulSum)
      B200_DISPATCH_PREMUL(dtype, T, {
        return launch_staged(c, reduce_kernel<T, kOpPremulSum>, a, make_units(nbytes).total(), stream, oa.premul);
      });
    B200_DISPATCH_DTYPE(dtype, T, B200_DISPATCH_OP(op, OP, {
                          return launch_staged(c, reduce_kernel<T, OP>, a, make_units(nbytes).total(), stream);
                        }));
  });
}
