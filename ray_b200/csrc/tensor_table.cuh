// tensor_table.cuh — tensor lists as one packed stream of 16-byte units, shared by the list
// point-to-point calls (p2p.cu: b200_send_multi / b200_recv_multi / b200_get_multi), the list
// broadcast and all-gather (copy_ops.cu: b200_broadcast_multi, b200_allgather_multi) and the list
// reduce-scatter (reduce_ops.cu: b200_reducescatter_multi).  The list collectives run the staged
// protocols of staged.cuh over a window of the stream; this file holds only the table.
//
// A table's tensors form ONE packed stream: tensor i occupies 16-byte units [ustart[i], ustart[i+1])
// with ustart[i+1] = ustart[i] + ceil(nbytes[i] / 16), so no unit mixes two tensors.  The padding of
// a tensor's last unit travels through the wire / staging slot (zeros) and is never stored.  Entries
// are non-empty: the host drops zero-size ones.  A table holds at most kP2PTableMax entries and is
// passed to its kernel as a __grid_constant__ parameter, so the calls can be captured in a CUDA graph.
#pragma once
#include "policy.h"

namespace b200 {

struct P2PTable {
  int count;
  char *ptr[kP2PTableMax];
  unsigned long long nbytes[kP2PTableMax];
  unsigned long long ustart[kP2PTableMax + 1];
};

// the entry that owns unit u of a table's packed message (start strictly increasing); also the
// all-reduce's TensorTable (allreduce_core.cuh), whose starts are unsigned int
template <typename S>
__device__ __forceinline__ int table_entry(const S *start, int count, size_t u) {
  int lo = 0, hi = count - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (start[mid] <= u) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// unit u (of the whole message) of a table, loaded / stored like a unit of a user tensor
__device__ __forceinline__ uint4 table_load_unit(const P2PTable &t, size_t u) {
  const int i = table_entry(t.ustart, t.count, u);
  return load_user_unit(t.ptr[i], u - t.ustart[i], make_units(t.nbytes[i]), is_aligned16(t.ptr[i]));
}
__device__ __forceinline__ void table_store_unit(const P2PTable &t, size_t u, uint4 v) {
  const int i = table_entry(t.ustart, t.count, u);
  store_user_unit(t.ptr[i], u - t.ustart[i], make_units(t.nbytes[i]), is_aligned16(t.ptr[i]), v);
}

// ---- host side --------------------------------------------------------------------------------

// ntensors and the host arrays of a list entry point
inline int check_list(int ntensors, bool arrays) {
  if (ntensors < 0) {
    set_error("ntensors %d is negative", ntensors);
    return B200_ERR_INVALID;
  }
  if (ntensors > 0 && !arrays) {
    set_error("null argument array");
    return B200_ERR_INVALID;
  }
  return B200_OK;
}

inline int check_list_ptrs(const void *const *ptrs, const size_t *nbytes, int ntensors) {
  for (int i = 0; i < ntensors; ++i) {
    if (nbytes[i] && !ptrs[i]) {
      set_error("tensor %d is null but has %zu bytes", i, nbytes[i]);
      return B200_ERR_INVALID;
    }
  }
  return B200_OK;
}

// The per-rank pointers of a gathered or scattered list: ptrs[i * world + p] belongs to entry i
// (nbytes[i] bytes) and rank p.
inline int check_list_rank_ptrs(const void *const *ptrs, const size_t *nbytes, int ntensors, int world,
                                const char *what) {
  for (int i = 0; i < ntensors; ++i)
    for (int p = 0; p < world; ++p)
      if (nbytes[i] && !ptrs[size_t(i) * world + p]) {
        set_error("%s %d of tensor %d is null but has %zu bytes", what, p, i, nbytes[i]);
        return B200_ERR_INVALID;
      }
  return B200_OK;
}

// World 1 of the list all-gather and reduce-scatter: entry i of srcs is copied to dsts[i].
inline int copy_list_local(void *const *dsts, const void *const *srcs, const size_t *nbytes, int ntensors,
                           cudaStream_t stream) {
  for (int i = 0; i < ntensors; ++i)
    if (nbytes[i] && dsts[i] != srcs[i])
      B200_CHECK_CUDA(cudaMemcpyAsync(dsts[i], srcs[i], nbytes[i], cudaMemcpyDeviceToDevice, stream));
  return B200_OK;
}

// Kernel parameters are limited to 32764 bytes on sm_90 (CUDA >= 12.1); a list kernel takes the
// communicator and its table arguments.
template <typename Args>
constexpr bool fits_param_space() {
  return sizeof(DevComm) + sizeof(Args) <= 32764;
}

// Runs launch(lo, hi) over [0, ntensors) cut into runs of at most kP2PTableMax non-empty entries, in
// list order.  The cut depends on the size list alone, so every rank cuts alike.
template <typename Fn>
inline int for_each_table(const size_t *nbytes, int ntensors, Fn launch) {
  int lo = 0, count = 0;
  for (int i = 0; i < ntensors; ++i) {
    if (!nbytes[i]) continue;
    if (count == kP2PTableMax) {
      if (int rc = launch(lo, i)) return rc;
      lo = i;
      count = 0;
    }
    ++count;
  }
  return count ? launch(lo, ntensors) : B200_OK;
}

// Packs the non-empty entries of [lo, hi) into t (which starts zeroed).  Returns whether every
// packed tensor is 16-byte aligned and a whole number of units.
inline bool fill_table(P2PTable &t, void *const *bufs, const size_t *nbytes, int lo, int hi) {
  bool whole_aligned = true;
  for (int i = lo; i < hi; ++i) {
    if (!nbytes[i]) continue;
    const int k = t.count++;
    t.ptr[k] = static_cast<char *>(bufs[i]);
    t.nbytes[k] = nbytes[i];
    t.ustart[k + 1] = t.ustart[k] + (nbytes[i] + 15) / 16;
    whole_aligned = whole_aligned && is_aligned16(bufs[i]) && (nbytes[i] & 15) == 0;
  }
  return whole_aligned;
}

// The launch loop of the list collectives (b200_broadcast_multi, b200_allgather_multi,
// b200_reducescatter_multi): each table of for_each_table is packed into t, pack(k, i) adds what the
// kernel needs beyond the P2PTable for packed entry k (list entry i), and launch(u0, units) then runs
// once per window of at most window_units units of the table's stream, in order.  The windows depend
// on the size list and window_units alone, so every rank makes the same launches.  Entries of t past
// t.count keep stale values of an earlier table; the kernels never read them.
template <typename Pack, typename Launch>
inline int for_each_window(P2PTable &t, void *const *bufs, const size_t *nbytes, int ntensors, size_t window_units,
                           Pack pack, Launch launch) {
  return for_each_table(nbytes, ntensors, [&](int lo, int hi) -> int {
    t.count = 0;
    fill_table(t, bufs, nbytes, lo, hi);
    for (int i = lo, k = 0; i < hi; ++i)
      if (nbytes[i]) pack(k++, i);
    return for_each_piece(t.ustart[t.count], window_units, launch);
  });
}

}  // namespace b200
