// allreduce_core.cuh — the reduce-and-publish phase shared by the two-shot / NVLS all-reduce,
// the fused gradient kernel and the multi-tensor kernel.  Its per-unit steps, nvls_finish and
// publish_unit, also serve the reduce workers of the pipelined all-reduce (allreduce_pipe.cu); the
// rank-ascending reduce itself is reduce_ranks (common.cuh).
//
// Work decomposition (see DESIGN.md §4): the staged message is U 16-byte units, cut into rows
// of n*kThreads units.  CTA b handles rows b, b+G, ...; inside a row rank r owns the kThreads
// units starting at r*kThreads, thread t owns one of them.
#pragma once
#include "kernel_utils.cuh"

namespace b200 {

struct RowGeom {
  size_t U;          // total units
  size_t row_units;  // n * kThreads
  size_t R;          // rows
};
__device__ __forceinline__ RowGeom make_rows(size_t U, int n) {
  RowGeom g;
  g.U = U;
  g.row_units = size_t(n) * kThreads;
  g.R = (U + g.row_units - 1) / g.row_units;
  return g;
}

// multimem.ld_reduce returns the sum over the n ranks; AVG divides it here, before multimem.st.
template <typename T, int OP>
__device__ __forceinline__ uint4 nvls_finish(uint4 v, int n) {
  if (OP != B200_AVG) return v;
  using Tr = Traits<T>;
  typename Tr::Acc acc = Tr::unpack(v);
  Tr::average(acc, n);
  return Tr::pack(acc);
}

// Store `v` as unit u at byte offset `off` of every rank's data region: the local copy first, then
// the peers in ring order.  n and r are the caller's copies of c.world and c.rank, read before its
// loads: reading them here, after the loads' memory clobbers, compiles the AVG kernels differently.
__device__ __forceinline__ void publish_unit(const DevComm &c, int n, int r, size_t off, size_t u, uint4 v) {
#pragma unroll
  for (int i = 0; i < kMaxRanks; ++i) {
    if (i < n) {
      int p = r + i;
      if (p >= n) p -= n;
      st_vec(c.data[p] + off + (u << 4), v);
    }
  }
}

// Reduce the units this rank owns across all n ranks' buffers at offset `off` of the data
// region and publish the result into every rank's buffer at the same offset.
template <typename T, int OP, bool NVLS>
__device__ __forceinline__ void reduce_publish_rows(const DevComm &c, size_t off, const RowGeom &g,
                                                    size_t G = 0) {
  const int n = c.world, r = c.rank, t = threadIdx.x;
  if (G == 0) G = gridDim.x;  // CTAs [0, G) share the rows of this phase
  if (NVLS) {
    constexpr int UNR = 4;  // 8 in flight measured slower with 8 GPUs on one NVSwitch
    char *mc = c.mc_data + off;
    for (size_t row0 = blockIdx.x; row0 < g.R; row0 += G * UNR) {
      uint4 v[UNR];
#pragma unroll
      for (int j = 0; j < UNR; ++j) {
        const size_t row = row0 + size_t(j) * G;
        const size_t u = row * g.row_units + size_t(r) * kThreads + t;
        if (row < g.R && u < g.U) v[j] = Multimem<T>::ld_reduce_sum(mc + (u << 4));
      }
#pragma unroll
      for (int j = 0; j < UNR; ++j) {
        const size_t row = row0 + size_t(j) * G;
        const size_t u = row * g.row_units + size_t(r) * kThreads + t;
        if (row < g.R && u < g.U) {
          v[j] = nvls_finish<T, OP>(v[j], n);
          multimem_st(mc + (u << 4), v[j]);
        }
      }
    }
  } else {
    constexpr int UNR = 2;
    for (size_t row0 = blockIdx.x; row0 < g.R; row0 += G * UNR) {
      uint4 v[UNR][kMaxRanks];
#pragma unroll
      for (int j = 0; j < UNR; ++j) {
        const size_t row = row0 + size_t(j) * G;
        const size_t u = row * g.row_units + size_t(r) * kThreads + t;
        if (row < g.R && u < g.U) {
#pragma unroll
          for (int p = 0; p < kMaxRanks; ++p)
            if (p < n) v[j][p] = ld_peer(c.data[p] + off + (u << 4));
        }
      }
#pragma unroll
      for (int j = 0; j < UNR; ++j) {
        const size_t row = row0 + size_t(j) * G;
        const size_t u = row * g.row_units + size_t(r) * kThreads + t;
        if (row < g.R && u < g.U) publish_unit(c, n, r, off, u, reduce_ranks<T, OP>(v[j], n));
      }
    }
  }
}

// The synchronised middle of every staged all-reduce: [all ranks staged] -> reduce+publish ->
// [all ranks published].  With red_ctas in (0, grid) the reduce phase runs on the first
// red_ctas CTAs only and the two synchronisations become grid-wide flag waits (the row -> CTA
// mapping differs between the phases); otherwise CTA b only meets CTA b of its peers.
// Returns false if a wait was abandoned (abort / watchdog).
template <typename T, int OP, bool NVLS>
__device__ __forceinline__ bool reduce_phase(const DevComm &c, uint32_t ep, size_t off, const RowGeom &g,
                                             int red_ctas) {
  if (red_ctas > 0 && red_ctas < int(gridDim.x)) {
    cta_signal_all(c, ep + 1);
    if (int(blockIdx.x) < red_ctas) {
      if (!cta_wait_grid(c, gridDim.x, ep + 1)) return false;
      reduce_publish_rows<T, OP, NVLS>(c, off, g, red_ctas);
      cta_signal_all(c, ep + 2);
    }
    return cta_wait_grid(c, red_ctas, ep + 2);
  }
  if (!cta_barrier_all(c, ep + 1)) return false;
  reduce_publish_rows<T, OP, NVLS>(c, off, g);
  return cta_barrier_all(c, ep + 2);
}

// Row-wise staging loops: `load(u)` produces the 16-byte unit u of the (virtual) message,
// `store(u, v)` consumes one.  CTA b touches exactly the rows it reduces/publishes.
template <typename LoadFn>
__device__ __forceinline__ void stage_in_rows(const DevComm &c, size_t off, const RowGeom &g, LoadFn load) {
  const int n = c.world, t = threadIdx.x;
  char *mine = c.data[c.rank] + off;
  for (size_t row = blockIdx.x; row < g.R; row += gridDim.x) {
    uint4 v[kMaxRanks];
    const size_t base = row * g.row_units + t;
#pragma unroll
    for (int k = 0; k < kMaxRanks; ++k) {
      const size_t u = base + size_t(k) * kThreads;
      if (k < n && u < g.U) v[k] = load(u);
    }
#pragma unroll
    for (int k = 0; k < kMaxRanks; ++k) {
      const size_t u = base + size_t(k) * kThreads;
      if (k < n && u < g.U) st_vec(mine + (u << 4), v[k]);
    }
  }
}

template <typename StoreFn>
__device__ __forceinline__ void stage_out_rows(const DevComm &c, size_t off, const RowGeom &g, StoreFn store) {
  const int n = c.world, t = threadIdx.x;
  const char *mine = c.data[c.rank] + off;
  for (size_t row = blockIdx.x; row < g.R; row += gridDim.x) {
    uint4 v[kMaxRanks];
    const size_t base = row * g.row_units + t;
#pragma unroll
    for (int k = 0; k < kMaxRanks; ++k) {
      const size_t u = base + size_t(k) * kThreads;
      if (k < n && u < g.U) v[k] = ld_peer(mine + (u << 4));
    }
#pragma unroll
    for (int k = 0; k < kMaxRanks; ++k) {
      const size_t u = base + size_t(k) * kThreads;
      if (k < n && u < g.U) store(u, v[k]);
    }
  }
}

// ---------------------------------------------------------------------------
// Tensor table for the multi-tensor all-reduce (SURVEY K9): tensor i occupies staged units
// [ustart[i], ustart[i+1]) -- every tensor starts on a 16-byte unit of the staged image, so
// the reduction never sees a unit that mixes two tensors.
// ---------------------------------------------------------------------------
constexpr int kMaxTableTensors = 48;
struct TensorTable {
  int count;
  char *ptr[kMaxTableTensors];
  unsigned long long nbytes[kMaxTableTensors];
  unsigned int ustart[kMaxTableTensors + 1];
};

}  // namespace b200
