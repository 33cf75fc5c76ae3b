// staged.cuh — the staged protocols of all-gather, broadcast and push reduce-scatter, written once
// for the forms of each collective: one tensor (copy_ops.cu, reduce_ops.cu), a size per rank
// (allgatherv), a window of a tensor table (tensor_table.cuh) and the fused FSDP gradient
// reduce-scatter (grad.cu).  A body owns the launch counter, the staging slot, the
// grid-stride unit loop, the CTA barrier with its give-up path, the rank rotation and the
// sub-slot layout; its kernel supplies where a unit comes from and where it goes.
//
// Unit u of a launch is staged at byte u * 16 of the slot (all-gather, broadcast) or of sub-slot r
// (reduce-scatter, sub-slots of `units` * 16 bytes).  The CTA barrier pairs CTA b of every rank, so
// CTA b handles the same unit indices on every rank in both phases: `units` and the grid must be
// functions of values every rank shares (DESIGN.md §3), never of this rank's own part alone.
#pragma once
#include "policy.h"

namespace b200 {

// Unit lu of a part that has it for every rank: ptrs[p] is rank p's part of un bytes.  The per-unit
// view of the even and list all-gathers (has, store) and reduce-scatters (load).
template <typename P>
struct PeerParts {
  P const *ptrs;
  size_t lu;
  Units un;
  __device__ __forceinline__ bool has(int) const { return true; }
  __device__ __forceinline__ uint4 load(int q) const { return load_user_unit(ptrs[q], lu, un, is_aligned16(ptrs[q])); }
  __device__ __forceinline__ void store(int p, uint4 v) const {
    store_user_unit(ptrs[p], lu, un, is_aligned16(ptrs[p]), v);
  }
};

// A unit source whose loads are scaled (PREMUL_SUM's reduce-scatter sources); scaled() leaves a
// source as it is under NoScale, so the plain kernels pass the body exactly what they did before.
template <typename Src, typename S>
struct ScaledParts {
  Src src;
  S scale;
  __device__ __forceinline__ uint4 load(int q) const { return scale(src.load(q)); }
};
template <typename Src>
__device__ __forceinline__ Src scaled(const Src &src, const NoScale &) {
  return src;
}
template <typename Src, typename T>
__device__ __forceinline__ ScaledParts<Src, Premul<T>> scaled(const Src &src, const Premul<T> &s) {
  return {src, s};
}

// All-gather: stage units [0, mine_units) of this rank's part, load(u) each, in the own slot; after
// the barrier every unit u of [0, units) with at(u).has(p) is pulled from rank p's slot, and
// at(u).store(p, v) stores it (and stores nothing where rank p's part lacks unit u).  The peer
// loads of a unit are issued as one batch before its stores.
template <typename Load, typename At>
__device__ __forceinline__ void allgather_body(const DevComm &c, size_t staging_bytes, size_t mine_units, size_t units,
                                               Load load, At at) {
  const uint32_t launch = c.st->launch_ctr;
  const uint32_t ep = launch * 4u;
  const int n = c.world, r = c.rank;
  const size_t off = staging_slot_offset(launch, staging_bytes);
  const size_t stride = size_t(gridDim.x) * kThreads;
  const size_t first = size_t(blockIdx.x) * kThreads + threadIdx.x;

  char *mine = c.data[r] + off;
  for (size_t u = first; u < mine_units; u += stride) st_vec(mine + (u << 4), load(u));

  if (!cta_barrier_all(c, ep + 1)) {
    finish_launch(c);
    return;
  }

  for (size_t u = first; u < units; u += stride) {
    const auto dst = at(u);
    uint4 v[kMaxRanks];
#pragma unroll
    for (int i = 0; i < kMaxRanks; ++i) {
      if (i < n) {
        int p = r + i;
        if (p >= n) p -= n;
        if (dst.has(p)) v[i] = ld_peer(c.data[p] + off + (u << 4));
      }
    }
#pragma unroll
    for (int i = 0; i < kMaxRanks; ++i) {
      if (i < n) {
        int p = r + i;
        if (p >= n) p -= n;
        dst.store(p, v[i]);
      }
    }
  }
  finish_launch(c);
}

// Broadcast of `units` units.  NVLS = false: root stages in its slot, every other rank pulls root's
// slot.  NVLS = true: root writes once to the multicast alias (the switch replicates it into every
// rank's slot), the others copy out locally.
// `root` is read where it is used: a list kernel's argument lives in parameter space
// (__grid_constant__), so a copy made up front would sit in a register across the barrier.
template <bool NVLS, typename Load, typename Store>
__device__ __forceinline__ void broadcast_body(const DevComm &c, size_t staging_bytes, const int &root, size_t units,
                                               Load load, Store store) {
  const uint32_t launch = c.st->launch_ctr;
  const uint32_t ep = launch * 4u;
  const int r = c.rank;
  const size_t off = staging_slot_offset(launch, staging_bytes);
  const size_t stride = size_t(gridDim.x) * kThreads;
  const size_t first = size_t(blockIdx.x) * kThreads + threadIdx.x;

  if (r == root) {
    char *dst = (NVLS ? c.mc_data : c.data[r]) + off;
    for (size_t u = first; u < units; u += stride) {
      const uint4 v = load(u);
      if (NVLS) multimem_st(dst + (u << 4), v);
      else st_vec(dst + (u << 4), v);
    }
  }

  if (!cta_barrier_all(c, ep + 1)) {
    finish_launch(c);
    return;
  }

  if (r != root) {
    const char *src = (NVLS ? c.data[r] : c.data[root]) + off;
    for (size_t u = first; u < units; u += stride) store(u, ld_peer(src + (u << 4)));
  }
  finish_launch(c);
}

// Push reduce-scatter: unit u of rank q's input, at(u).load(q), goes to sub-slot r of rank q's
// slot, in rank rotation starting at this rank; after the barrier this rank reads its n sub-slots
// for each unit and hands them, rank-ascending, to reduce_store(u, v, n).  Every thread reduces exactly the units it pushed from its own part, so
// the output may be that part.
template <typename At, typename ReduceStore>
__device__ __forceinline__ void reducescatter_push_body(const DevComm &c, size_t staging_bytes, size_t units, At at,
                                                        ReduceStore reduce_store) {
  const uint32_t launch = c.st->launch_ctr;
  const uint32_t ep = launch * 4u;
  const int n = c.world, r = c.rank;
  const size_t sub = units << 4;  // bytes per sub-slot
  const size_t off = staging_slot_offset(launch, staging_bytes);
  const size_t stride = size_t(gridDim.x) * kThreads;
  const size_t first = size_t(blockIdx.x) * kThreads + threadIdx.x;

  for (size_t u = first; u < units; u += stride) {
    const auto src = at(u);
    uint4 v[kMaxRanks];
#pragma unroll
    for (int i = 0; i < kMaxRanks; ++i) {
      if (i < n) {
        int q = r + i;
        if (q >= n) q -= n;
        v[i] = src.load(q);
      }
    }
#pragma unroll
    for (int i = 0; i < kMaxRanks; ++i) {
      if (i < n) {
        int q = r + i;
        if (q >= n) q -= n;
        st_vec(c.data[q] + off + size_t(r) * sub + (u << 4), v[i]);
      }
    }
  }

  if (!cta_barrier_all(c, ep + 1)) {
    finish_launch(c);
    return;
  }

  const char *mine = c.data[r] + off;
  for (size_t u = first; u < units; u += stride) {
    uint4 v[kMaxRanks];
#pragma unroll
    for (int p = 0; p < kMaxRanks; ++p)
      if (p < n) v[p] = ld_peer(mine + size_t(p) * sub + (u << 4));
    reduce_store(u, v, n);
  }
  finish_launch(c);
}

// ---- host side --------------------------------------------------------------------------------

// Launches a staged kernel on one CTA per kThreads of its `units` units, within the grid cap.
template <typename Args>
inline int launch_staged(b200_comm *c, void (*kernel)(DevComm, Args), const Args &a, size_t units,
                         cudaStream_t stream) {
  const int g = pick_blocks(c, (units + kThreads - 1) / kThreads, c->sm_count);
  kernel<<<g, kThreads, 0, stream>>>(c->dev(), a);
  B200_LAUNCH_CHECK(c);
  return B200_OK;
}
// ... and a PREMUL_SUM kernel, which takes the factor as one more argument
template <typename Args>
inline int launch_staged(b200_comm *c, void (*kernel)(DevComm, Args, PremulArg), const Args &a, size_t units,
                         cudaStream_t stream, const PremulArg &f) {
  const int g = pick_blocks(c, (units + kThreads - 1) / kThreads, c->sm_count);
  kernel<<<g, kThreads, 0, stream>>>(c->dev(), a, f);
  B200_LAUNCH_CHECK(c);
  return B200_OK;
}

}  // namespace b200
