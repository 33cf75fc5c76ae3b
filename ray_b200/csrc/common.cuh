// common.cuh — device-side building blocks shared by every kernel of libb200_collective.
//
// Layout of one rank's symmetric memory (all ranks allocate identical sizes, so
// an offset is valid on every peer):
//
//   region "data"  : [ staging slot 0 | staging slot 1 | user heap ]   (one VMM allocation,
//                    mapped on every peer; also bound to the NVLS multicast object)
//   region "sig"   : signal pad, u32 flags written by peers
//                    coll flags  [MAX_BLOCKS][MAX_RANKS]
//                    p2p ready   [MAX_RANKS src][P2P_RINGS][P2P_SLOTS]
//                    p2p ack     [MAX_RANKS dst][P2P_RINGS]
//                    pipe flags  [2 kinds][MAX_PIPE_CHUNKS][MAX_RANKS]
//   region "inbox" : [MAX_RANKS src] x inbox_bytes point-to-point landing area
//   region "ll"    : [2][MAX_RANKS src][128 KiB] flag-in-data slots of the low-latency all-reduce
//
// Rank-local (cudaMalloc) state: launch counter, completion ticket, sticky status,
// p2p sequence numbers.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200_collective.h"

namespace b200 {

constexpr int kMaxRanks = B200_MAX_RANKS;
constexpr int kMaxBlocks = 512;   // upper bound on collective grid size (flag rows)
constexpr int kThreads = 512;     // CTA size of every collective kernel
constexpr int kP2PRings = 16;     // independent sub-rings per ordered pair (one per CTA)
constexpr int kP2PSlots = 8;      // chunks in flight per sub-ring

// signal pad offsets, in u32 words
constexpr size_t kSigCollFlags = 0;
constexpr size_t kSigP2PReady = kSigCollFlags + size_t(kMaxBlocks) * kMaxRanks;
constexpr size_t kSigP2PAck = kSigP2PReady + size_t(kMaxRanks) * kP2PRings * kP2PSlots;
// pipelined all-reduce: per-chunk flags, two kinds (0: "rank p's copy of chunk k is in place",
// 1: "rank p published its stripe of chunk k"), each [kMaxPipeChunks][kMaxRanks]
constexpr int kMaxPipeChunks = 512;
constexpr size_t kSigPipe0 = kSigP2PAck + size_t(kMaxRanks) * kP2PRings;
constexpr size_t kSigPipe1 = kSigPipe0 + size_t(kMaxPipeChunks) * kMaxRanks;
constexpr size_t kSigWords = kSigPipe1 + size_t(kMaxPipeChunks) * kMaxRanks;

// Low-latency (LL) region: [2 parities][kMaxRanks sources][kLLSlotBytes]; payload and flag share
// each 8-byte word pair, so a message needs no separate barrier.
constexpr size_t kLLMaxPayload = size_t(64) << 10;      // bytes of payload per rank per launch
constexpr size_t kLLSlotBytes = 2 * kLLMaxPayload;      // every 4-byte word travels with a 4-byte flag
constexpr size_t kLLRegionBytes = 2 * size_t(kMaxRanks) * kLLSlotBytes;

// rank-local state words
struct LocalState {
  uint32_t launch_ctr;  // number of completed collective launches
  uint32_t done_ctr;    // ticket used to find the last CTA of a launch
  int32_t status;       // sticky b200_status_t set by a kernel that gave up
  uint32_t pad;
  uint32_t send_seq[kMaxRanks][kP2PRings];  // next chunk sequence to peer, per ring
  uint32_t recv_seq[kMaxRanks][kP2PRings];  // next chunk sequence from peer, per ring
  uint32_t pipe_cnt[2][kMaxPipeChunks];     // per-chunk arrival counters of the pipelined kernels
  uint32_t pipe_out_progress[32];           // chunk ring: (launch << 10 | chunks copied out) per copy-out CTA
};

// Passed by value to every kernel.
struct DevComm {
  int rank;
  int world;
  char *data[kMaxRanks];      // peers' data region (index == rank: own)
  uint32_t *sig[kMaxRanks];   // peers' signal pad
  char *inbox[kMaxRanks];     // peers' inbox region
  char *ll[kMaxRanks];        // peers' low-latency region
  char *mc_data;              // multicast alias of the data region (nullptr without NVLS)
  LocalState *st;             // rank-local state
  const volatile int *abort;  // host-mapped abort word
  volatile int *host_status;  // host-mapped mirror of LocalState::status (read without a CUDA call)
  unsigned long long timeout_ns;
  size_t inbox_bytes;         // per-source inbox size
  unsigned long long *trace;  // optional event trace (b200_comm_trace_enable), nullptr normally
  unsigned int trace_cap;     // capacity in events
};

// ---------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys(uint32_t *p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// 128-bit accesses.  Peer and staging data is read exactly once per kernel, so
// bypass L1 allocation; input tensors use the read-only path.
__device__ __forceinline__ uint4 ld_stream(const void *p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
// volatile-free relaxed load used for data written by peers during this kernel
__device__ __forceinline__ uint4 ld_peer(const void *p) {
  uint4 v;
  asm volatile("ld.relaxed.sys.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_vec(void *p, uint4 v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

// NVLS: multimem.st broadcasts 16 bytes to the same offset of every rank's buffer.
__device__ __forceinline__ void multimem_st(void *mc, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

// Optional in-kernel event trace (debugging / profiling aid; see b200_comm_trace_enable):
// word 0 of the buffer is the event counter, events are 2 x u64: globaltimer ns, and
// (blockIdx << 40 | event << 32 | argument).
__device__ __forceinline__ void trace_event(const DevComm &c, unsigned ev, unsigned arg) {
  if (c.trace == nullptr) return;
  const unsigned long long i = atomicAdd(c.trace, 1ull);
  if (i < c.trace_cap) {
    c.trace[2 + 2 * i] = globaltimer_ns();
    c.trace[3 + 2 * i] = (static_cast<unsigned long long>(blockIdx.x) << 40) |
                         (static_cast<unsigned long long>(ev & 0xffu) << 32) | arg;
  }
}

// A kernel that abandons a wait records why: sticky device word (first error wins) plus a
// host-mapped mirror so b200_comm_status() is a plain host load.
__device__ __forceinline__ void give_up(const DevComm &c, int code) {
  if (atomicCAS(&c.st->status, 0, code) == 0) {
    *c.host_status = code;
    __threadfence_system();
  }
}

// ---------------------------------------------------------------------------
// Cross-GPU CTA barrier.
//
// CTA b of every rank meets CTA b of all peers.  `epoch` strictly increases over
// the life of the communicator (launch counter * 4 + phase), flags are written by
// exactly one writer each, so a ">= epoch" test (wrap-safe signed difference) is
// sufficient and flags never need resetting.
//
// Returns false when the wait was abandoned (abort or watchdog); the caller must
// then leave the kernel without touching peer memory again.
// ---------------------------------------------------------------------------
__device__ __forceinline__ bool wait_flag_ge(const DevComm &c, const uint32_t *flag, uint32_t epoch) {
  unsigned spins = 0;
  unsigned long long t0 = 0;
  while (true) {
    uint32_t v = ld_acquire_sys(flag);
    if (int32_t(v - epoch) >= 0) return true;
    if ((++spins & 0x3ff) == 0) {
      if (*c.abort != 0) {
        give_up(c, B200_ERR_ABORTED);
        return false;
      }
      unsigned long long now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > c.timeout_ns) {
        give_up(c, B200_ERR_TIMEOUT);
        return false;
      }
    }
  }
}

__device__ __forceinline__ bool cta_barrier_all(const DevComm &c, uint32_t epoch) {
  __shared__ int ok_flag;
  if (threadIdx.x == 0) ok_flag = 1;
  __syncthreads();  // all prior writes of this CTA are ordered before the release below
  if (threadIdx.x < c.world) {
    const int peer = threadIdx.x;
    st_release_sys(c.sig[peer] + kSigCollFlags + size_t(blockIdx.x) * kMaxRanks + c.rank, epoch);
    bool ok = wait_flag_ge(c, c.sig[c.rank] + kSigCollFlags + size_t(blockIdx.x) * kMaxRanks + peer,
                           epoch);
    if (!ok) ok_flag = 0;
  }
  __syncthreads();
  return ok_flag != 0;
}

// Grid-wide variant, used when a phase runs on fewer CTAs than the previous one (the NVSwitch
// reduction saturates at ~64 CTAs while the HBM staging phases want the whole GPU): every CTA
// announces `epoch`; a CTA that needs ALL of them polls the flags of CTAs [0, nb) of every rank.
__device__ __forceinline__ void cta_signal_all(const DevComm &c, uint32_t epoch) {
  __syncthreads();
  if (threadIdx.x < c.world)
    st_release_sys(c.sig[threadIdx.x] + kSigCollFlags + size_t(blockIdx.x) * kMaxRanks + c.rank, epoch);
}
__device__ __forceinline__ bool cta_wait_grid(const DevComm &c, int nb, uint32_t epoch) {
  // One warp polls, politely: CTAs parked here wait for a whole phase of other CTAs, and
  // hundreds of threads spinning on system-scope loads would steal L2 bandwidth from the very
  // NVLink traffic they are waiting for.  Relaxed polls with back-off, one acquire fence at the end.
  int ok = 1;
  if (threadIdx.x < 32) {
    const uint32_t *flags = c.sig[c.rank] + kSigCollFlags;
    unsigned long long t0 = 0;
    unsigned sleep_ns = 32;
    for (int i = threadIdx.x; i < nb * c.world && ok; i += 32) {
      const int b = i / c.world, p = i - b * c.world;
      const uint32_t *f = flags + size_t(b) * kMaxRanks + p;
      unsigned spins = 0;
      while (int32_t(ld_relaxed_sys(f) - epoch) < 0) {
        __nanosleep(sleep_ns);
        if (sleep_ns < 1024) sleep_ns <<= 1;
        if ((++spins & 0xff) == 0) {
          if (*c.abort != 0) {
            give_up(c, B200_ERR_ABORTED);
            ok = 0;
            break;
          }
          const unsigned long long now = globaltimer_ns();
          if (t0 == 0) t0 = now;
          else if (now - t0 > c.timeout_ns) {
            give_up(c, B200_ERR_TIMEOUT);
            ok = 0;
            break;
          }
        }
      }
    }
    __threadfence_system();  // acquire: order the polls before the data reads that follow
  }
  return __syncthreads_and(ok) != 0;
}

// Called by every CTA at the very end of a collective kernel: the last CTA to get
// here advances the launch counter (device-resident so the launch sequence can be
// captured in a CUDA graph).
__device__ __forceinline__ void finish_launch(const DevComm &c) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    uint32_t t = atomicAdd(&c.st->done_ctr, 1u);
    if (t == gridDim.x - 1) {
      c.st->done_ctr = 0;
      __threadfence();
      atomicAdd(&c.st->launch_ctr, 1u);
    }
  }
}

// ---------------------------------------------------------------------------
// Element traits: how a 16-byte vector of T is unpacked into an accumulator,
// combined, and packed again.  16/8-bit floats accumulate in fp32 and round once.
// ---------------------------------------------------------------------------
// Internal op of the PREMUL_SUM instantiations: every rank's input is scaled as it is read
// (Premul below), and from then on the op is SUM.  Not a b200_op_t value: callers name a PREMUL_SUM
// op by the handle b200_op_create_premul returns.
constexpr int kOpPremulSum = B200_OP_COUNT;

template <int OP, typename A>
__device__ __forceinline__ A combine(A a, A b) {
  if (OP == B200_SUM || OP == B200_AVG || OP == kOpPremulSum) return a + b;
  if (OP == B200_PROD) return a * b;
  // MIN / MAX propagate a NaN from any rank, as np.minimum / np.maximum do: a NaN accumulator
  // survives because every comparison with it is false, and `b != b` picks up a NaN operand (it
  // is always false for the integer types, so their instructions do not change).
  if (OP == B200_MIN) return (b < a || b != b) ? b : a;
  return (b > a || b != b) ? b : a;  // MAX
}

template <typename T>
struct Traits;

template <typename S, int LANES>
struct PlainTraits {
  static constexpr int kLanes = LANES;
  struct Acc {
    S v[LANES];
  };
  static __device__ __forceinline__ Acc unpack(uint4 u) {
    Acc a;
    const S *p = reinterpret_cast<const S *>(&u);
#pragma unroll
    for (int i = 0; i < LANES; ++i) a.v[i] = p[i];
    return a;
  }
  static __device__ __forceinline__ uint4 pack(const Acc &a) {
    uint4 u;
    S *p = reinterpret_cast<S *>(&u);
#pragma unroll
    for (int i = 0; i < LANES; ++i) p[i] = a.v[i];
    return u;
  }
  template <int OP>
  static __device__ __forceinline__ void reduce(Acc &a, const Acc &b) {
#pragma unroll
    for (int i = 0; i < LANES; ++i) a.v[i] = combine<OP, S>(a.v[i], b.v[i]);
  }
  static __device__ __forceinline__ void average(Acc &a, int n) {
#pragma unroll
    for (int i = 0; i < LANES; ++i) a.v[i] = a.v[i] / S(n);
  }
};

template <> struct Traits<float> : PlainTraits<float, 4> {};
template <> struct Traits<double> : PlainTraits<double, 2> {};
template <> struct Traits<int32_t> : PlainTraits<int32_t, 4> {};
template <> struct Traits<uint32_t> : PlainTraits<uint32_t, 4> {};
template <> struct Traits<int64_t> : PlainTraits<int64_t, 2> {};
template <> struct Traits<uint64_t> : PlainTraits<uint64_t, 2> {};
// 8-bit integers: arithmetic in the element type so SUM / PROD wrap modulo 256
// exactly like the CPU reference (gloo reduces in the tensor's dtype).
template <> struct Traits<uint8_t> : PlainTraits<uint8_t, 16> {};
template <> struct Traits<int8_t> : PlainTraits<int8_t, 16> {};

template <typename H>
struct HalfTraits {
  static constexpr int kLanes = 8;
  struct Acc {
    float v[8];
  };
  static __device__ __forceinline__ float to_f(H h);
  static __device__ __forceinline__ H from_f(float f);
  static __device__ __forceinline__ Acc unpack(uint4 u) {
    Acc a;
    const H *p = reinterpret_cast<const H *>(&u);
#pragma unroll
    for (int i = 0; i < 8; ++i) a.v[i] = to_f(p[i]);
    return a;
  }
  static __device__ __forceinline__ uint4 pack(const Acc &a) {
    uint4 u;
    H *p = reinterpret_cast<H *>(&u);
#pragma unroll
    for (int i = 0; i < 8; ++i) p[i] = from_f(a.v[i]);
    return u;
  }
  template <int OP>
  static __device__ __forceinline__ void reduce(Acc &a, const Acc &b) {
#pragma unroll
    for (int i = 0; i < 8; ++i) a.v[i] = combine<OP, float>(a.v[i], b.v[i]);
  }
  static __device__ __forceinline__ void average(Acc &a, int n) {
#pragma unroll
    for (int i = 0; i < 8; ++i) a.v[i] = a.v[i] / float(n);
  }
};
template <> __device__ __forceinline__ float HalfTraits<__half>::to_f(__half h) { return __half2float(h); }
template <> __device__ __forceinline__ __half HalfTraits<__half>::from_f(float f) { return __float2half_rn(f); }
template <> __device__ __forceinline__ float HalfTraits<__nv_bfloat16>::to_f(__nv_bfloat16 h) { return __bfloat162float(h); }
template <> __device__ __forceinline__ __nv_bfloat16 HalfTraits<__nv_bfloat16>::from_f(float f) { return __float2bfloat16_rn(f); }
template <> struct Traits<__half> : HalfTraits<__half> {};
template <> struct Traits<__nv_bfloat16> : HalfTraits<__nv_bfloat16> {};

// v[0] (op) v[1] (op) ... (op) v[n-1], then AVG's division, packed.  The fixed rank-ascending order
// is what makes floating-point SUM / PROD bit-exact against the reference (DESIGN.md §2).
template <typename T, int OP>
__device__ __forceinline__ uint4 reduce_ranks(const uint4 (&v)[kMaxRanks], int n) {
  using Tr = Traits<T>;
  typename Tr::Acc acc = Tr::unpack(v[0]);
#pragma unroll
  for (int p = 1; p < kMaxRanks; ++p)
    if (p < n) Tr::template reduce<OP>(acc, Tr::unpack(v[p]));
  if (OP == B200_AVG) Tr::average(acc, n);
  return Tr::pack(acc);
}

// ---------------------------------------------------------------------------
// PREMUL_SUM's factor.  It reaches a kernel as an argument, never as communicator state, so calls
// with different factors may be in flight at once and a captured graph reads a device factor at
// replay time.  The factor is a value of the operand's dtype: `host` holds it exactly, or `dev`
// points at it and every kernel that uses the op loads it when it starts.
// ---------------------------------------------------------------------------
struct PremulArg {
  double host;
  const void *dev;  // nullptr: use `host`
};

// The scale policy of the reducing kernels: applied to each 16-byte unit of the caller's input as it
// is read into registers, before it reaches a staging slot or a peer.  NoScale is the plain ops'.
struct NoScale {
  __device__ __forceinline__ uint4 operator()(uint4 v) const { return v; }
};

__device__ __forceinline__ float premul_scalar(__half h) { return __half2float(h); }
__device__ __forceinline__ float premul_scalar(__nv_bfloat16 h) { return __bfloat162float(h); }
__device__ __forceinline__ float premul_scalar(float f) { return f; }
__device__ __forceinline__ double premul_scalar(double f) { return f; }
__device__ __forceinline__ float premul_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double premul_mul(double a, double b) { return __dmul_rn(a, b); }

// y = round_T(x * f): the product in double for f64, in fp32 for f32 / f16 / bf16, rounded once to
// T.  The _rn multiplies are never contracted into an FMA with the SUM that follows, so the rank's
// contribution is exactly y.
template <typename T>
struct Premul {
  using S = decltype(premul_scalar(T()));
  S f;
  __device__ __forceinline__ explicit Premul(const PremulArg &a)
      : f(a.dev ? premul_scalar(*static_cast<const T *>(a.dev)) : S(a.host)) {}
  __device__ __forceinline__ uint4 operator()(uint4 v) const {
    using Tr = Traits<T>;
    typename Tr::Acc acc = Tr::unpack(v);
#pragma unroll
    for (int i = 0; i < Tr::kLanes; ++i) acc.v[i] = premul_mul(acc.v[i], f);
    return Tr::pack(acc);
  }
};

// ---------------------------------------------------------------------------
// NVLS reduction: one instruction pulls the same 16 bytes from every rank's
// buffer, reduced inside the switch.  Available for SUM on f32 / f16 / bf16
// (fp32 accumulation for the 16-bit types).  Other (T, OP) pairs have no
// specialisation and are routed to the peer-load kernels by the dispatcher.
// ---------------------------------------------------------------------------
template <typename T>
struct Multimem {
  static constexpr bool kSum = false;
  static __device__ __forceinline__ uint4 ld_reduce_sum(const void *) { return uint4{0, 0, 0, 0}; }
};
template <>
struct Multimem<float> {
  static constexpr bool kSum = true;
  static __device__ __forceinline__ uint4 ld_reduce_sum(const void *mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(mc)
                 : "memory");
    return v;
  }
};
template <>
struct Multimem<__nv_bfloat16> {
  static constexpr bool kSum = true;
  static __device__ __forceinline__ uint4 ld_reduce_sum(const void *mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(mc)
                 : "memory");
    return v;
  }
};
template <>
struct Multimem<__half> {
  static constexpr bool kSum = true;
  static __device__ __forceinline__ uint4 ld_reduce_sum(const void *mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(mc)
                 : "memory");
    return v;
  }
};

}  // namespace b200
