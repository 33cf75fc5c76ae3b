// allreduce.cu — all-reduce kernels (SURVEY K1) and their dispatcher.
//
// Three algorithms, all in ONE launch each (stage-in, cross-GPU barrier, reduce,
// barrier, stage-out are phases of the same persistent grid):
//
//   one-shot : every rank stages its input in its own symmetric slot, then reads
//              all n staged inputs over NVLink and reduces rank-ascending.  One
//              barrier; latency path for small messages.
//   two-shot : the message is cut into rows of n*512 16-byte units; rank r owns
//              units [r*512,(r+1)*512) of every row.  The owner loads its units
//              from all n peers' HBM (rank-ascending reduction), and pushes the
//              result back into all n peers' slots.  Every element is read and
//              written by exactly one thread system-wide, so the reduce-scatter
//              and all-gather halves fuse without a barrier between them.
//   NVLS     : same ownership, but the n loads are one multimem.ld_reduce and the
//              n stores one multimem.st on the NVSwitch multicast alias.
//
// CTA b of every rank works on the same rows in every phase, so a barrier between
// CTA b's of all ranks (flags in the signal pad) is the only synchronisation needed:
// no grid-wide sync, no host involvement.
#include "allreduce_core.cuh"
#include "policy.h"
#include "tensor_table.cuh"

namespace b200 {

struct ARArgs {
  const char *in;
  char *out;
  size_t nbytes;
  size_t staging_bytes;
  long long sym_off;  // >= 0: operand lives in the symmetric data region at this offset
                      //       (zero-copy, in place); < 0: stage through the rotating slot
  int red_ctas;       // CTAs that run the reduce phase (0 or >= grid: all of them)
};

// ---------------------------------------------------------------------------
// one-shot
// ---------------------------------------------------------------------------
template <typename T, int OP, typename S>
__device__ __forceinline__ void allreduce_oneshot_body(const DevComm &c, const ARArgs &a, const S &scale) {
  const uint32_t launch = c.st->launch_ctr;
  const uint32_t ep = launch * 4u;
  const int n = c.world, r = c.rank;
  const Units un = make_units(a.nbytes);
  const size_t U = un.total();
  const bool in_al = is_aligned16(a.in), out_al = is_aligned16(a.out);
  const size_t off = staging_slot_offset(launch, a.staging_bytes);
  const size_t stride = size_t(gridDim.x) * kThreads;
  const size_t first = size_t(blockIdx.x) * kThreads + threadIdx.x;

  char *mine = c.data[r] + off;
  for (size_t u = first; u < U; u += stride) st_vec(mine + (u << 4), scale(load_user_unit(a.in, u, un, in_al)));

  if (!cta_barrier_all(c, ep + 1)) {
    finish_launch(c);
    return;
  }

  for (size_t u = first; u < U; u += stride) {
    uint4 v[kMaxRanks];
#pragma unroll
    for (int p = 0; p < kMaxRanks; ++p)
      if (p < n) v[p] = ld_peer(c.data[p] + off + (u << 4));
    store_user_unit(a.out, u, un, out_al, reduce_ranks<T, OP>(v, n));
  }
  finish_launch(c);
}
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1) allreduce_oneshot_kernel(DevComm c, ARArgs a) {
  allreduce_oneshot_body<T, OP>(c, a, NoScale{});
}
// PREMUL_SUM (OP = kOpPremulSum): the same kernel with the input scaled at stage-in
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1) allreduce_oneshot_kernel(DevComm c, ARArgs a, PremulArg f) {
  allreduce_oneshot_body<T, OP>(c, a, Premul<T>(f));
}

// ---------------------------------------------------------------------------
// low-latency (LL) one-shot: every rank pushes its message straight into each peer's LL slot as
// (word, flag) pairs -- 16-byte stores carrying two pairs, each 8-byte pair lands atomically --
// and then polls its own slots until the flags of this launch appear.  No barrier, no staging
// pass: one NVLink traversal end to end.  At most one 16-byte unit per thread.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void ll_store(void *p, uint32_t a, uint32_t b, uint32_t flag) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a), "r"(flag), "r"(b), "r"(flag)
               : "memory");
}
__device__ __forceinline__ uint4 ll_load(const void *p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

// `a` and `scale` by value: taken by reference, the plain 4-byte kernels schedule four moves differently
template <typename T, int OP, typename S>
__device__ __forceinline__ void allreduce_ll_body(const DevComm &c, ARArgs a, S scale) {
  using Tr = Traits<T>;
  const uint32_t launch = c.st->launch_ctr;
  const uint32_t flag = launch + 1u;  // never 0, never equal to what the slot held two launches ago
  const int n = c.world, r = c.rank;
  const Units un = make_units(a.nbytes);
  const size_t U = un.total();
  const size_t u = size_t(blockIdx.x) * kThreads + threadIdx.x;
  const size_t par_off = (launch & 1u) ? size_t(kMaxRanks) * kLLSlotBytes : 0;
  if (u < U) {
    const uint4 mine = scale(load_user_unit(a.in, u, un, is_aligned16(a.in)));
    // push (start with the next rank so the eight peers are not hit in lock step)
#pragma unroll
    for (int i = 1; i < kMaxRanks; ++i) {
      if (i < n) {
        int p = r + i;
        if (p >= n) p -= n;
        char *dst = c.ll[p] + par_off + size_t(r) * kLLSlotBytes + (u << 5);
        ll_store(dst, mine.x, mine.y, flag);
        ll_store(dst + 16, mine.z, mine.w, flag);
      }
    }
    // collect, rank-ascending
    const char *base = c.ll[r] + par_off + (u << 5);
    typename Tr::Acc acc;
    bool alive = true;
#pragma unroll
    for (int p = 0; p < kMaxRanks; ++p) {
      if (p < n) {
        uint4 v = mine;
        if (p != r) {
          const char *src = base + size_t(p) * kLLSlotBytes;
          uint4 lo, hi;
          unsigned spins = 0;
          unsigned long long t0 = 0;
          while (alive) {
            lo = ll_load(src);
            hi = ll_load(src + 16);
            if (lo.y == flag && lo.w == flag && hi.y == flag && hi.w == flag) break;
            if ((++spins & 0x3ff) == 0) {
              if (*c.abort != 0) {
                give_up(c, B200_ERR_ABORTED);
                alive = false;
              }
              const unsigned long long now = globaltimer_ns();
              if (t0 == 0) t0 = now;
              else if (now - t0 > c.timeout_ns) {
                give_up(c, B200_ERR_TIMEOUT);
                alive = false;
              }
            }
          }
          v = make_uint4(lo.x, lo.z, hi.x, hi.z);
        }
        if (p == 0) acc = Tr::unpack(v);
        else Tr::template reduce<OP>(acc, Tr::unpack(v));
      }
    }
    if (alive) {
      if (OP == B200_AVG) Tr::average(acc, n);
      store_user_unit(a.out, u, un, is_aligned16(a.out), Tr::pack(acc));
    }
  }
  finish_launch(c);
}
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1) allreduce_ll_kernel(DevComm c, ARArgs a) {
  allreduce_ll_body<T, OP>(c, a, NoScale{});
}
// PREMUL_SUM: the scaled unit is what is pushed to the peers and reduced locally
template <typename T, int OP>
__global__ void __launch_bounds__(kThreads, 1) allreduce_ll_kernel(DevComm c, ARArgs a, PremulArg f) {
  allreduce_ll_body<T, OP>(c, a, Premul<T>(f));
}

// ---------------------------------------------------------------------------
// two-shot / NVLS
// ---------------------------------------------------------------------------
template <typename T, int OP, bool NVLS, typename S>
__device__ __forceinline__ void allreduce_twoshot_body(const DevComm &c, const ARArgs &a, const S &scale) {
  const uint32_t launch = c.st->launch_ctr;
  const uint32_t ep = launch * 4u;
  const Units un = make_units(a.nbytes);
  const RowGeom g = make_rows(un.total(), c.world);
  const bool staged = a.sym_off < 0;
  const size_t off = staged ? staging_slot_offset(launch, a.staging_bytes) : size_t(a.sym_off);

  // phase 0: stage this CTA's rows into the local symmetric slot
  if (staged) {
    const bool in_al = is_aligned16(a.in);
    stage_in_rows(c, off, g, [&](size_t u) { return scale(load_user_unit(a.in, u, un, in_al)); });
  }
  // phase 1: reduce the units this rank owns, publish to every peer
  if (!reduce_phase<T, OP, NVLS>(c, ep, off, g, a.red_ctas)) {
    finish_launch(c);
    return;
  }
  // phase 2: copy this CTA's rows out of the local slot
  if (staged) {
    const bool out_al = is_aligned16(a.out);
    stage_out_rows(c, off, g, [&](size_t u, uint4 v) { store_user_unit(a.out, u, un, out_al, v); });
  }
  finish_launch(c);
}
template <typename T, int OP, bool NVLS>
__global__ void __launch_bounds__(kThreads, 1) allreduce_twoshot_kernel(DevComm c, ARArgs a) {
  allreduce_twoshot_body<T, OP, NVLS>(c, a, NoScale{});
}
// PREMUL_SUM: always staged (the zero-copy form has no stage-in to scale at); NVLS reduces as SUM
template <typename T, int OP, bool NVLS>
__global__ void __launch_bounds__(kThreads, 1) allreduce_twoshot_kernel(DevComm c, ARArgs a, PremulArg f) {
  allreduce_twoshot_body<T, OP, NVLS>(c, a, Premul<T>(f));
}

// ---------------------------------------------------------------------------
// multi-tensor (SURVEY K9): the same three phases, but stage-in gathers from / stage-out
// scatters to a table of tensors, so a list of tensors is reduced as ONE message in ONE
// launch with no host-side flatten (dag/collective_node.py:220-232 uses parameters_to_vector).
// ---------------------------------------------------------------------------
template <typename T, int OP, bool NVLS, typename S>
__device__ __forceinline__ void allreduce_multi_body(const DevComm &c, const TensorTable &tb, size_t staging_bytes,
                                                     int red_ctas, const S &scale) {
  const uint32_t launch = c.st->launch_ctr;
  const uint32_t ep = launch * 4u;
  const RowGeom g = make_rows(tb.ustart[tb.count], c.world);
  const size_t off = staging_slot_offset(launch, staging_bytes);

  stage_in_rows(c, off, g, [&](size_t u) {
    const int i = table_entry(tb.ustart, tb.count, u);
    return scale(load_user_unit(tb.ptr[i], u - tb.ustart[i], make_units(tb.nbytes[i]), is_aligned16(tb.ptr[i])));
  });
  if (!reduce_phase<T, OP, NVLS>(c, ep, off, g, red_ctas)) {
    finish_launch(c);
    return;
  }
  stage_out_rows(c, off, g, [&](size_t u, uint4 v) {
    const int i = table_entry(tb.ustart, tb.count, u);
    store_user_unit(tb.ptr[i], u - tb.ustart[i], make_units(tb.nbytes[i]), is_aligned16(tb.ptr[i]), v);
  });
  finish_launch(c);
}
template <typename T, int OP, bool NVLS>
__global__ void __launch_bounds__(kThreads, 1)
allreduce_multi_kernel(DevComm c, const __grid_constant__ TensorTable tb, size_t staging_bytes, int red_ctas) {
  allreduce_multi_body<T, OP, NVLS>(c, tb, staging_bytes, red_ctas, NoScale{});
}
// PREMUL_SUM: the table gather scales each unit
template <typename T, int OP, bool NVLS>
__global__ void __launch_bounds__(kThreads, 1) allreduce_multi_kernel(DevComm c, const __grid_constant__ TensorTable tb,
                                                                      size_t staging_bytes, int red_ctas, PremulArg f) {
  allreduce_multi_body<T, OP, NVLS>(c, tb, staging_bytes, red_ctas, Premul<T>(f));
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
// `f...` is empty for the plain ops and the PremulArg for OP = kOpPremulSum, which picks that kernel.
template <typename T, int OP, typename... F>
static int launch_allreduce(b200_comm *c, const char *in, char *out, size_t nbytes, int algo,
                            long long sym_off, cudaStream_t stream, const F &...f) {
  DevComm dc = c->dev();
  ARArgs a{in, out, nbytes, c->staging_bytes, sym_off, 0};
  const size_t U = make_units(nbytes).total();
  if (algo == B200_ALGO_LL) {
    a.sym_off = -1;
    allreduce_ll_kernel<T, OP><<<int((U + kThreads - 1) / kThreads), kThreads, 0, stream>>>(dc, a, f...);
  } else if (algo == B200_ALGO_ONESHOT) {
    a.sym_off = -1;
    int g = pick_blocks(c, (U + kThreads - 1) / kThreads, 32);
    allreduce_oneshot_kernel<T, OP><<<g, kThreads, 0, stream>>>(dc, a, f...);
  } else {
    const size_t rows = (U + size_t(c->world) * kThreads - 1) / (size_t(c->world) * kThreads);
    int g = pick_blocks(c, rows, c->sm_count);
    if (algo == B200_ALGO_NVLS) {
      a.red_ctas = nvls_ctas(c);
      if (sym_off >= 0) {  // nothing to stage: the whole launch is the reduce phase, which
        const int cap = a.red_ctas > 0 ? a.red_ctas : 64;  // saturates the switch with ~64 CTAs
        if (g > cap && c->forced_blocks == 0) g = cap;
        a.red_ctas = 0;
      }
      if constexpr (Multimem<T>::kSum && (OP == B200_SUM || OP == B200_AVG || OP == kOpPremulSum)) {
        allreduce_twoshot_kernel<T, OP, true><<<g, kThreads, 0, stream>>>(dc, a, f...);
      } else {
        set_error("NVLS all-reduce supports SUM/AVG on f32/f16/bf16 only");
        return B200_ERR_UNSUPPORTED;
      }
    } else {
      allreduce_twoshot_kernel<T, OP, false><<<g, kThreads, 0, stream>>>(dc, a, f...);
    }
  }
  B200_LAUNCH_CHECK(c);
  return B200_OK;
}

// World size 1 of the PREMUL_SUM entries: out = round_T(in * factor), unit by unit, so in place works
// and either pointer may have any alignment.
template <typename T>
__global__ void __launch_bounds__(kThreads) premul_scale_kernel(const char *in, char *out, size_t nbytes,
                                                                PremulArg f) {
  const Premul<T> scale(f);
  const Units un = make_units(nbytes);
  const bool in_al = is_aligned16(in), out_al = is_aligned16(out);
  const size_t stride = size_t(gridDim.x) * kThreads;
  for (size_t u = size_t(blockIdx.x) * kThreads + threadIdx.x; u < un.total(); u += stride)
    store_user_unit(out, u, un, out_al, scale(load_user_unit(in, u, un, in_al)));
}

int launch_premul_scale(b200_comm *c, const void *in, void *out, size_t nbytes, int dtype, const PremulArg &f,
                        cudaStream_t stream) {
  if (nbytes == 0) return B200_OK;
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  const int g = pick_blocks(c, (make_units(nbytes).total() + kThreads - 1) / kThreads, 4 * c->sm_count);
  B200_DISPATCH_PREMUL(dtype, T, {
    premul_scale_kernel<T><<<g, kThreads, 0, stream>>>(static_cast<const char *>(in), static_cast<char *>(out),
                                                       nbytes, f);
  });
  B200_LAUNCH_CHECK(c);
  return B200_OK;
}

// a kernel of this file's CUDA module, for preload_kernels() (bootstrap.cu)
const void *allreduce_module_anchor() { return reinterpret_cast<const void *>(static_cast<void (*)(DevComm, ARArgs)>(&allreduce_ll_kernel<float, B200_SUM>)); }

}  // namespace b200

using namespace b200;

extern "C" int b200_allreduce(b200_comm_t c, const void *in, void *out, size_t count, int dtype,
                              int op, int algo, void *stream_) {
  int rc;
  size_t es;
  OpArg oa;
  if ((rc = check_usable(c)) || (rc = check_dtype(dtype, &es)) || (rc = check_op(c, op, dtype, &oa))) return rc;
  const bool premul = oa.op == kOpPremulSum;
  if (premul && algo == B200_ALGO_PIPE) {
    set_error("PREMUL_SUM does not run on the pipelined all-reduce, whose copies bypass the registers it scales in");
    return B200_ERR_UNSUPPORTED;
  }
  const int red_op = premul ? int(B200_SUM) : op;  // what the algorithm choice sees
  if (count == 0) return B200_OK;
  if (!in || !out) return null_tensor_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  const size_t total = count * es;
  if (c->world == 1) {
    if (premul) return launch_premul_scale(c, in, out, total, dtype, oa.premul, stream);
    if (in != out) B200_CHECK_CUDA(cudaMemcpyAsync(out, in, total, cudaMemcpyDeviceToDevice, stream));
    return B200_OK;
  }
  if (algo == B200_ALGO_NVLS && !c->mc_active) {
    set_error("NVLS requested but the multicast mapping is not active");
    return B200_ERR_UNSUPPORTED;
  }

  // zero-copy when the operand sits in the symmetric heap (and is updated in place)
  // The reduce phase works on whole 16-byte units straight in the heap, so a tensor whose size is
  // not a multiple of 16 bytes would have the bytes that follow it reduced as well: such operands
  // take the staged path (which zero-pads the tail unit in the slot instead).  Every rank must pass
  // the tensor at the same heap offset (b200_symm_alloc / the pool hand out identical offsets when
  // ranks allocate in the same order, which both interfaces require).
  long long sym_off = -1;
  if (in == out && (total & 15) == 0 && b200_symm_contains(c, in, total) && is_aligned16(in))
    sym_off = static_cast<const char *>(in) - reinterpret_cast<const char *>(c->data.va[c->rank]);

  const char *src = static_cast<const char *>(in);
  char *dst = static_cast<char *>(out);

  // Ordinary (staged) operands from pipe_min_bytes() on: the chunk-pipelined kernels, which overlap
  // the two staging passes with the NVLink phase (allreduce_pipe.cu).  They move whole 16-byte
  // units with the bulk-copy engine, so they need aligned operands.
  int pipe_variant = -1;
  if (sym_off < 0 && is_aligned16(in) && is_aligned16(out) && (total & 15) == 0 && pipe_fits(c) &&
      (algo == B200_ALGO_PIPE || (algo == B200_ALGO_AUTO && total >= pipe_min_bytes(c)))) {
    if (c->world == 2) pipe_variant = PIPE_PULL;
    else if (c->mc_active && nvls_capable(dtype, red_op)) pipe_variant = PIPE_NVLS;
    else if (algo == B200_ALGO_PIPE) pipe_variant = PIPE_PEER;  // AUTO without NVLS keeps the two-shot kernel
    if (algo == B200_ALGO_AUTO && pipe_variant >= 0 && !pipe_runs(c, PipeVariant(pipe_variant))) pipe_variant = -1;
  } else if (algo == B200_ALGO_PIPE) {
    set_error("the pipelined all-reduce needs 16-byte aligned operands outside the symmetric heap "
              "and a size that is a multiple of 16 bytes");
    return B200_ERR_UNSUPPORTED;
  }

  // PREMUL_SUM scales each rank's input as stage-in reads it.  The pipelined kernels copy it with
  // the bulk-copy unit and the zero-copy form has no stage-in, so where SUM would take either,
  // PREMUL_SUM takes the staged two-shot kernel: on the switch when SUM's NVLS rule holds for the
  // message, over the peers otherwise.  Every other choice is SUM's.
  if (premul) {
    if (algo == B200_ALGO_AUTO && (pipe_variant >= 0 || (sym_off >= 0 && total > ll_limit(c))))
      algo = c->mc_active && nvls_capable(dtype, red_op) && nvls_pays_off(c, total) ? B200_ALGO_NVLS
                                                                                     : B200_ALGO_TWOSHOT;
    pipe_variant = -1;
    sym_off = -1;
  }

  // Messages larger than one staging slot are processed slot by slot.
  const size_t step = sym_off >= 0         ? total
                      : pipe_variant >= 0 ? pipe_plan(c, PipeVariant(pipe_variant)).max_bytes
                                          : c->staging_bytes;
  return for_each_piece(total, step, [&](size_t done, size_t nbytes) -> int {
    if (pipe_variant >= 0 && (algo == B200_ALGO_PIPE || nbytes >= pipe_min_bytes(c) || nbytes > c->staging_bytes))
      return launch_allreduce_pipe_dyn(c, src + done, dst + done, nbytes, dtype, op, pipe_variant, stream);
    int a = algo;
    if (a == B200_ALGO_AUTO || a == B200_ALGO_PIPE) {
      if (nbytes <= ll_limit(c)) a = B200_ALGO_LL;
      else if (sym_off < 0 && nbytes <= oneshot_limit(c)) a = B200_ALGO_ONESHOT;
      else if (c->mc_active && nvls_capable(dtype, red_op) && nvls_pays_off(c, nbytes)) a = B200_ALGO_NVLS;
      else a = B200_ALGO_TWOSHOT;
    }
    if (a == B200_ALGO_LL && nbytes > kLLMaxPayload) a = B200_ALGO_ONESHOT;
    if (a == B200_ALGO_ONESHOT && nbytes > c->staging_bytes) a = B200_ALGO_TWOSHOT;
    const long long so = sym_off >= 0 ? sym_off + (long long)done : -1;
    int rc2 = B200_OK;
    if (premul) {
      B200_DISPATCH_PREMUL(dtype, T, {
        rc2 = launch_allreduce<T, kOpPremulSum>(c, src + done, dst + done, nbytes, a, so, stream, oa.premul);
      });
      return rc2;
    }
    B200_DISPATCH_DTYPE(dtype, T, B200_DISPATCH_OP(op, OP, {
                          rc2 = launch_allreduce<T, OP>(c, src + done, dst + done, nbytes, a, so, stream);
                        }));
    return rc2;
  });
}

// ---- multi-tensor entry ------------------------------------------------------------
namespace b200 {
template <typename T, int OP, typename... F>
static int launch_multi(b200_comm *c, const TensorTable &tb, cudaStream_t stream, const F &...f) {
  const size_t U = tb.ustart[tb.count];
  const size_t rows = (U + size_t(c->world) * kThreads - 1) / (size_t(c->world) * kThreads);
  int g = pick_blocks(c, rows, c->sm_count);
  if constexpr (Multimem<T>::kSum && (OP == B200_SUM || OP == B200_AVG || OP == kOpPremulSum)) {
    if (c->mc_active) {
      allreduce_multi_kernel<T, OP, true><<<g, kThreads, 0, stream>>>(c->dev(), tb, c->staging_bytes, nvls_ctas(c),
                                                                      f...);
      B200_LAUNCH_CHECK(c);
      return B200_OK;
    }
  }
  allreduce_multi_kernel<T, OP, false><<<g, kThreads, 0, stream>>>(c->dev(), tb, c->staging_bytes, 0, f...);
  B200_LAUNCH_CHECK(c);
  return B200_OK;
}
}  // namespace b200

// Reduces `ntensors` same-dtype tensors as one message: tensors are packed (each starting on
// a 16-byte unit) into launches of up to kMaxTableTensors tensors / one staging slot.  The
// single-launch kernel exists for the floating-point types (gradients, activations); other
// dtypes take one fused launch per tensor.
extern "C" int b200_allreduce_multi(b200_comm_t c, void *const *ptrs, const size_t *counts,
                                    int ntensors, int dtype, int op, void *stream_) {
  int rc;
  size_t es;
  OpArg oa;
  if ((rc = check_usable(c)) || (rc = check_dtype(dtype, &es)) || (rc = check_op(c, op, dtype, &oa))) return rc;
  if (ntensors < 0 || (ntensors > 0 && (!ptrs || !counts))) {
    set_error("invalid tensor list");
    return B200_ERR_INVALID;
  }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool table_ok = (dtype == B200_F32 || dtype == B200_F16 || dtype == B200_BF16 || dtype == B200_F64) &&
                        c->world > 1;
  int i = 0;
  while (i < ntensors) {
    if (counts[i] == 0) {
      ++i;
      continue;
    }
    if (!ptrs[i]) {
      set_error("tensor %d is null", i);
      return B200_ERR_INVALID;
    }
    const size_t bytes_i = counts[i] * es;
    if (!table_ok || bytes_i > c->staging_bytes / 2) {
      // large tensors (or dtypes without a table kernel) go through the single-tensor path
      rc = b200_allreduce(c, ptrs[i], ptrs[i], counts[i], dtype, op, B200_ALGO_AUTO, stream_);
      if (rc) return rc;
      ++i;
      continue;
    }
    B200_CHECK_CUDA(cudaSetDevice(c->device));
    TensorTable tb{};
    size_t units = 0;
    while (i < ntensors && tb.count < kMaxTableTensors) {
      if (counts[i] == 0) {
        ++i;
        continue;
      }
      const size_t b = counts[i] * es;
      const size_t u = (b + 15) >> 4;
      if (!ptrs[i] || b > c->staging_bytes / 2 || ((units + u) << 4) > c->staging_bytes) break;
      tb.ptr[tb.count] = static_cast<char *>(ptrs[i]);
      tb.nbytes[tb.count] = b;
      tb.ustart[tb.count] = static_cast<unsigned int>(units);
      units += u;
      ++tb.count;
      ++i;
    }
    tb.ustart[tb.count] = static_cast<unsigned int>(units);
    if (tb.count == 0) continue;
    if (oa.op == kOpPremulSum) {
      B200_DISPATCH_PREMUL(dtype, T, { rc = launch_multi<T, kOpPremulSum>(c, tb, stream, oa.premul); });
      if (rc) return rc;
      continue;
    }
    switch (dtype) {
      case B200_F32: B200_DISPATCH_OP(op, OP, { rc = launch_multi<float, OP>(c, tb, stream); }); break;
      case B200_F64: B200_DISPATCH_OP(op, OP, { rc = launch_multi<double, OP>(c, tb, stream); }); break;
      case B200_F16: B200_DISPATCH_OP(op, OP, { rc = launch_multi<__half, OP>(c, tb, stream); }); break;
      default: B200_DISPATCH_OP(op, OP, { rc = launch_multi<__nv_bfloat16, OP>(c, tb, stream); }); break;
    }
    if (rc) return rc;
  }
  return B200_OK;
}

// ---- PREMUL_SUM ops (ncclRedOpCreatePreMulSum / ncclRedOpDestroy) ------------------------------
extern "C" int b200_op_create_premul(b200_comm_t c, const void *scalar, int dtype, int residence, int *op) {
  int rc;
  if ((rc = check_usable(c))) return rc;
  if (!scalar || !op || (residence != 0 && residence != 1)) {
    set_error("b200_op_create_premul: null scalar or op, or residence %d is neither 0 (host) nor 1 (device)",
              residence);
    return B200_ERR_INVALID;
  }
  double host = 0.0;
  switch (dtype) {
    case B200_F16: host = residence ? 0.0 : double(__half2float(*static_cast<const __half *>(scalar))); break;
    case B200_BF16: host = residence ? 0.0 : double(__bfloat162float(*static_cast<const __nv_bfloat16 *>(scalar))); break;
    case B200_F32: host = residence ? 0.0 : double(*static_cast<const float *>(scalar)); break;
    case B200_F64: host = residence ? 0.0 : *static_cast<const double *>(scalar); break;
    default: set_error("PREMUL_SUM supports f16, bf16, f32 and f64 only, not dtype %d", dtype); return B200_ERR_UNSUPPORTED;
  }
  for (int i = 0; i < int(sizeof(c->premul_ops) / sizeof(c->premul_ops[0])); ++i) {
    if (c->premul_ops[i].dtype >= 0) continue;
    c->premul_ops[i].dtype = dtype;
    c->premul_ops[i].arg = PremulArg{host, residence ? scalar : nullptr};
    *op = kPremulOpBase + i;
    return B200_OK;
  }
  set_error("b200_op_create_premul: all %d op slots are in use", int(sizeof(c->premul_ops) / sizeof(c->premul_ops[0])));
  return B200_ERR_INVALID;
}

extern "C" int b200_op_destroy(b200_comm_t c, int op) {
  if (!c) {
    set_error("null communicator");
    return B200_ERR_INVALID;
  }
  const int slot = op - kPremulOpBase;
  if (slot < 0 || slot >= int(sizeof(c->premul_ops) / sizeof(c->premul_ops[0])) || c->premul_ops[slot].dtype < 0) {
    set_error("b200_op_destroy: %d is not a live PREMUL_SUM op", op);
    return B200_ERR_INVALID;
  }
  c->premul_ops[slot].dtype = -1;
  return B200_OK;
}
