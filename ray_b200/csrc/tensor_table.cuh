// tensor_table.cuh — tensor lists as one packed stream of 16-byte units, shared by the list
// point-to-point calls (p2p.cu: b200_send_multi / b200_recv_multi / b200_get_multi) and the list
// broadcast (copy_ops.cu: b200_broadcast_multi).
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

// the entry that owns unit u of a table's packed message (ustart strictly increasing)
__device__ __forceinline__ int table_entry(const unsigned long long *start, int count, size_t u) {
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

}  // namespace b200
