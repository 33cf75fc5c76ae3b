// p2p.cu — point-to-point send / recv (SURVEY K5; the transport under the Compiled-Graph
// GPU channel and RDT's two-sided path).
//
// Sender-push over NVLink into the receiver's inbox, chunked through per-CTA rings:
//
//   receiver's inbox[src] = kP2PRings sub-rings x kP2PSlots chunks
//   CTA b of the send kernel and CTA b of the recv kernel own sub-ring b.
//
//   send: wait until the slot was consumed (ack flag in the SENDER's signal pad),
//         store the chunk into the peer inbox, release-store "ready = seq+1" into
//         the RECEIVER's signal pad.
//   recv: acquire-wait ready == seq+1, copy the chunk from local HBM into the
//         caller's tensor, release-store "ack = seq+1" into the sender's pad.
//
// Sequence numbers persist in rank-local device memory, so messages of any size
// interleave correctly and a send completes without the receiver having been
// launched as long as the message fits the ring (eager protocol).
//
// Two copy mechanisms share this ONE protocol (each side picks its own, per launch):
//   p2p_kernel      : 512 threads x 16-byte ld/st -- small, unaligned or ragged messages
//   p2p_bulk_kernel : one thread per CTA drives the TMA bulk-copy unit (cp.async.bulk, SASS
//                     UBLKCP): user tensor -> shared ring -> peer inbox on the sender, inbox ->
//                     shared ring -> user tensor on the receiver.  A CTA keeps 192 KiB in flight,
//                     so <= 16 CTAs fill the link where the ld/st kernel needed 64; a second
//                     thread publishes the ready / ack flags so the copy thread never waits for a
//                     system-scope fence.
// Both are thin wrappers around p2p_ldst_ring / p2p_bulk_ring (one CTA's share of a message), which
// alltoall_kernel also runs: all 2(n-1) transfers of an all-to-all as roles of one grid, each role
// picking its own copy mechanism.
#include <type_traits>

#include "bulk_copy.cuh"
#include "policy.h"

namespace b200 {

struct P2PArgs {
  char *buf;
  size_t nbytes;
  size_t chunk;  // bytes per chunk of THIS message (<= slot size), same on both sides
  int peer;
};

__device__ __forceinline__ bool cta_wait_flag(const DevComm &c, const uint32_t *flag, uint32_t target) {
  __shared__ int ok;
  if (threadIdx.x == 0) ok = wait_flag_ge(c, flag, target) ? 1 : 0;
  __syncthreads();
  return ok != 0;
}

// One CTA's share of a message: chunks b, b + G, b + 2G, ... over sub-ring b, moved with 16-byte
// ld/st by all kThreads threads.  Both sides of a pair call it with the same (G, chunk).
template <bool SEND>
__device__ __forceinline__ void p2p_ldst_ring(const DevComm &c, int peer, int b, int G, char *buf, size_t nbytes,
                                              size_t chunk) {
  const int me = c.rank;
  const size_t ring_bytes = c.inbox_bytes / kP2PRings;
  const size_t slot_bytes = ring_bytes / kP2PSlots;
  const size_t nchunks = (nbytes + chunk - 1) / chunk;
  const bool al = is_aligned16(buf);

  uint32_t *seq_word = SEND ? &c.st->send_seq[peer][b] : &c.st->recv_seq[peer][b];
  uint32_t seq = *seq_word;

  // sender: data lands in the peer's inbox[me]; receiver: reads its own inbox[peer]
  char *ring = (SEND ? c.inbox[peer] + size_t(me) * c.inbox_bytes : c.inbox[me] + size_t(peer) * c.inbox_bytes) +
               size_t(b) * ring_bytes;
  // ready flags live in the receiver's pad, ack flags in the sender's pad
  uint32_t *ready = (SEND ? c.sig[peer] + kSigP2PReady + (size_t(me) * kP2PRings + b) * kP2PSlots
                          : c.sig[me] + kSigP2PReady + (size_t(peer) * kP2PRings + b) * kP2PSlots);
  uint32_t *ack = (SEND ? c.sig[me] + kSigP2PAck + size_t(peer) * kP2PRings + b
                        : c.sig[peer] + kSigP2PAck + size_t(me) * kP2PRings + b);

  for (size_t j = b; j < nchunks; j += G) {
    const size_t lo = j * chunk;
    const size_t len = (nbytes - lo) < chunk ? (nbytes - lo) : chunk;
    const Units un = make_units(len);
    const size_t U = un.total();
    const uint32_t slot = seq % kP2PSlots;
    char *slot_ptr = ring + size_t(slot) * slot_bytes;
    char *user = buf + lo;
    if (SEND) {
      // slot free once the receiver consumed chunk (seq - kP2PSlots)
      if (!cta_wait_flag(c, ack, seq + 1u - kP2PSlots)) break;
      // 8 x 16 B per thread in flight (one CTA sustains ~20 GB/s this way; large aligned messages
      // take p2p_bulk_kernel instead)
      for (size_t u0 = threadIdx.x; u0 < U; u0 += size_t(kThreads) * 8) {
        uint4 v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const size_t u = u0 + size_t(k) * kThreads;
          if (u < U) v[k] = load_user_unit(user, u, un, al);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const size_t u = u0 + size_t(k) * kThreads;
          if (u < U) st_vec(slot_ptr + (u << 4), v[k]);
        }
      }
      __syncthreads();
      if (threadIdx.x == 0) st_release_sys(ready + slot, seq + 1u);
    } else {
      if (!cta_wait_flag(c, ready + slot, seq + 1u)) break;
      for (size_t u0 = threadIdx.x; u0 < U; u0 += size_t(kThreads) * 8) {
        uint4 v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const size_t u = u0 + size_t(k) * kThreads;
          if (u < U) v[k] = ld_peer(slot_ptr + (u << 4));
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const size_t u = u0 + size_t(k) * kThreads;
          if (u < U) store_user_unit(user, u, un, al, v[k]);
        }
      }
      __syncthreads();
      if (threadIdx.x == 0) st_release_sys(ack, seq + 1u);
    }
    ++seq;
  }
  __syncthreads();
  if (threadIdx.x == 0) *seq_word = seq;
}

template <bool SEND>
__global__ void __launch_bounds__(kThreads, 1) p2p_kernel(DevComm c, P2PArgs a) {
  p2p_ldst_ring<SEND>(c, a.peer, blockIdx.x, gridDim.x, a.buf, a.nbytes, a.chunk);
}

// ---------------------------------------------------------------------------
// bulk-copy variant: same rings, same flags, same sequence numbers
// ---------------------------------------------------------------------------
// The same share of a message moved by the bulk-copy unit; `dyn_smem` holds kBulkSmemBytes.  `buf`
// must be 16-byte aligned and `nbytes` a multiple of 16.  Only threads 0 and 32 drive the transfer;
// warps 2.. run side(thread, nthreads) meanwhile (the all-to-all gives them its own-segment copy).
template <bool SEND, typename SideFn>
__device__ __forceinline__ void p2p_bulk_ring(const DevComm &c, int peer, int b, int G, char *buf, size_t nbytes,
                                              size_t chunk, char *dyn_smem, SideFn side) {
  __shared__ volatile uint32_t mailbox;  // chunks of this CTA whose bytes have all been moved
  __shared__ volatile int stop;
  const int me = c.rank;
  const size_t ring_bytes = c.inbox_bytes / kP2PRings;
  const size_t slot_bytes = ring_bytes / kP2PSlots;
  const size_t nchunks = (nbytes + chunk - 1) / chunk;
  const size_t nq = nchunks > size_t(b) ? (nchunks - 1 - size_t(b)) / size_t(G) + 1 : 0;  // chunks of this CTA

  uint32_t *seq_word = SEND ? &c.st->send_seq[peer][b] : &c.st->recv_seq[peer][b];
  const uint32_t seq0 = *seq_word;
  char *ring = (SEND ? c.inbox[peer] + size_t(me) * c.inbox_bytes : c.inbox[me] + size_t(peer) * c.inbox_bytes) +
               size_t(b) * ring_bytes;
  uint32_t *ready = (SEND ? c.sig[peer] + kSigP2PReady + (size_t(me) * kP2PRings + b) * kP2PSlots
                          : c.sig[me] + kSigP2PReady + (size_t(peer) * kP2PRings + b) * kP2PSlots);
  uint32_t *ack = (SEND ? c.sig[me] + kSigP2PAck + size_t(peer) * kP2PRings + b
                        : c.sig[peer] + kSigP2PAck + size_t(me) * kP2PRings + b);
  if (threadIdx.x == 0) {
    mailbox = 0;
    stop = 0;
  }
  const BulkRing br = bulk_ring_init(dyn_smem);  // contains the __syncthreads

  const uint32_t nq32 = uint32_t(nq);
  if (threadIdx.x == 0 && nq > 0) {
    // ---- copy thread: one segment per chunk ---------------------------------------------------
    auto seg = [&](uint32_t q) {
      const size_t lo = (size_t(b) + size_t(q) * size_t(G)) * chunk;
      const uint32_t len = uint32_t((nbytes - lo) < chunk ? (nbytes - lo) : chunk);
      char *slot = ring + size_t((seq0 + q) % kP2PSlots) * slot_bytes;
      return SEND ? BulkSeg{buf + lo, slot, len} : BulkSeg{slot, buf + lo, len};
    };
    auto gate = [&](uint32_t q, bool block) {
      const uint32_t seq = seq0 + q;
      // sender: the slot was consumed (ack in MY pad); receiver: the chunk landed (ready in MY pad)
      const uint32_t *flag = SEND ? ack : ready + seq % kP2PSlots;
      const uint32_t target = SEND ? seq + 1u - kP2PSlots : seq + 1u;
      if (block) {
        if (!wait_flag_ge(c, flag, target)) return -1;
      } else if (int32_t(ld_acquire_sys(flag) - target) < 0) {
        return 0;
      }
      if (!SEND) fence_proxy_async();  // the peer's stores before our bulk reads
      return 1;
    };
    auto done = [&](uint32_t q) {
      __threadfence_block();
      mailbox = q + 1;
    };
    // the sender's stores cross NVLink, the receiver's stay in local HBM
    const bool ok = SEND ? bulk_copy_segments<BulkRemote>(br, nq32, seg, gate, done)
                         : bulk_copy_segments<BulkLocal>(br, nq32, seg, gate, done);
    if (!ok) stop = 1;
  } else if (threadIdx.x == 32 && nq > 0) {
    // ---- flag thread: publishes "ready" (sender) / "ack" (receiver) for completed chunks ------
    uint32_t published = 0;
    while (published < nq) {
      const uint32_t avail = mailbox;
      if (avail == published) {
        if (stop) break;
        __nanosleep(64);
        continue;
      }
      __threadfence_block();
      fence_proxy_async();
      __threadfence_system();
      for (; published < avail; ++published) {
        const uint32_t seq = seq0 + published;
        if (SEND) st_relaxed_sys(ready + seq % kP2PSlots, seq + 1u);
        else st_relaxed_sys(ack, seq + 1u);
      }
    }
  } else if (threadIdx.x >= 64) {
    side(int(threadIdx.x) - 64, kThreads - 64);
  }
  __syncthreads();
  if (threadIdx.x == 0) *seq_word = seq0 + uint32_t(stop ? mailbox : nq);
}

template <bool SEND>
__global__ void __launch_bounds__(kThreads, 1) p2p_bulk_kernel(DevComm c, P2PArgs a) {
  extern __shared__ __align__(128) char dyn_smem[];
  p2p_bulk_ring<SEND>(c, a.peer, blockIdx.x, gridDim.x, a.buf, a.nbytes, a.chunk, dyn_smem, [](int, int) {});
}

// ---------------------------------------------------------------------------
// all-to-all(v): every send and every receive of this rank as ONE grid.  Each (peer, direction)
// is a role of G CTAs; CTA b of a role runs exactly what CTA b of the standalone send / recv kernel
// would, on sub-ring b with the same chunking and the same persistent sequence numbers.  An
// all-to-all therefore interleaves in stream order with earlier and later b200_send / b200_recv on
// the same pairs.  It does not pair directly with a concurrent plain send / recv on the peer: the
// two may split the message over different numbers of rings.  The grid is co-resident (host side:
// at most one CTA per SM), which keeps the spinning roles deadlock-free.
//
// The own segment needs no peer.  Every CTA copies an equal slice of it, so that the copy overlaps
// the transfers instead of following them: a bulk role's CTA with its warps 2.. while threads 0 / 32
// move the message; an ld/st receive role's CTA before its role (its first chunk is on the way
// meanwhile); an ld/st send role's CTA after its role; and the CTAs past the roles, added when the
// own segment wants more CTAs than the roles have, right away -- with the bulk-copy unit when the
// segment allows it.
// ---------------------------------------------------------------------------
struct A2ARole {
  char *buf;
  size_t nbytes;
  size_t chunk;
  int peer;
  int first;  // first CTA of the role in the grid (prefix table)
  int G;      // CTAs = sub-rings of the role
  int send;
  int bulk;   // move with the bulk-copy unit (operand 16-byte aligned, chunks large enough)
};

struct A2AArgs {
  A2ARole role[2 * (kMaxRanks - 1)];
  int nroles;
  int role_ctas;        // CTAs [role_ctas, grid) only copy the own segment ...
  int own_bulk;         // ... with the bulk-copy unit (both ends 16-byte aligned, whole units)
  const char *own_src;  // this rank's own segment
  char *own_dst;
  size_t own_bytes;
};

// Slice `cta` of `nctas` of [src, src + nbytes) -> dst in local HBM, by `nthr` threads (this one is
// `t`), 8 x 16 B per thread in flight
__device__ __forceinline__ void a2a_own_copy(const char *src, char *dst, size_t nbytes, int cta, int nctas, int t,
                                             int nthr) {
  const Units un = make_units(nbytes);
  const size_t U = un.total();
  const size_t lo = U * size_t(cta) / size_t(nctas), hi = U * size_t(cta + 1) / size_t(nctas);
  const bool sal = is_aligned16(src), dal = is_aligned16(dst);
  for (size_t u0 = lo + size_t(t); u0 < hi; u0 += size_t(8) * nthr) {
    uint4 v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (u0 + size_t(k) * nthr < hi) v[k] = load_user_unit(src, u0 + size_t(k) * nthr, un, sal);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (u0 + size_t(k) * nthr < hi) store_user_unit(dst, u0 + size_t(k) * nthr, un, dal, v[k]);
  }
}

__global__ void __launch_bounds__(kThreads, 1) alltoall_kernel(DevComm c, A2AArgs a) {
  extern __shared__ __align__(128) char dyn_smem[];
  const int cta = int(blockIdx.x), nctas = int(gridDim.x);
  if (cta >= a.role_ctas) {
    if (!a.own_bulk) {
      a2a_own_copy(a.own_src, a.own_dst, a.own_bytes, cta, nctas, int(threadIdx.x), kThreads);
      return;
    }
    const BulkRing br = bulk_ring_init(dyn_smem);
    if (threadIdx.x != 0) return;
    const size_t U = a.own_bytes >> 4;  // whole 16-byte units (own_bulk)
    const size_t lo = (U * size_t(cta) / size_t(nctas)) << 4, hi = (U * size_t(cta + 1) / size_t(nctas)) << 4;
    constexpr size_t kSeg = size_t(256) << 10;
    bulk_copy_segments<BulkLocal>(
        br, uint32_t((hi - lo + kSeg - 1) / kSeg),
        [&](uint32_t i) {
          const size_t o = lo + size_t(i) * kSeg;
          return BulkSeg{a.own_src + o, a.own_dst + o, uint32_t(hi - o < kSeg ? hi - o : kSeg)};
        },
        [&](uint32_t, bool) { return 1; }, [&](uint32_t) {});
    return;
  }
  int i = 0;
  while (i + 1 < a.nroles && cta >= a.role[i + 1].first) ++i;
  const A2ARole &r = a.role[i];
  const int b = cta - r.first;
  if (r.bulk) {
    auto side = [&](int t, int nthr) { a2a_own_copy(a.own_src, a.own_dst, a.own_bytes, cta, nctas, t, nthr); };
    if (r.send) p2p_bulk_ring<true>(c, r.peer, b, r.G, r.buf, r.nbytes, r.chunk, dyn_smem, side);
    else p2p_bulk_ring<false>(c, r.peer, b, r.G, r.buf, r.nbytes, r.chunk, dyn_smem, side);
  } else if (r.send) {
    p2p_ldst_ring<true>(c, r.peer, b, r.G, r.buf, r.nbytes, r.chunk);
    a2a_own_copy(a.own_src, a.own_dst, a.own_bytes, cta, nctas, int(threadIdx.x), kThreads);
  } else {
    a2a_own_copy(a.own_src, a.own_dst, a.own_bytes, cta, nctas, int(threadIdx.x), kThreads);
    __syncthreads();
    p2p_ldst_ring<false>(c, r.peer, b, r.G, r.buf, r.nbytes, r.chunk);
  }
}

// ---------------------------------------------------------------------------
// one-sided get: the receiver pulls [src_off, src_off + nbytes) of a PEER's symmetric heap into a
// local tensor.  No kernel runs on the owner of the data (RDT's one-sided contract,
// experimental/rdt/cuda_ipc_transport.py:57-186); ordering against the owner's writes is the
// caller's event.  Aligned transfers use bulk loads over NVLink + bulk stores (segment engine).
// ---------------------------------------------------------------------------
struct GetArgs {
  const char *src;  // peer mapping of the owner's heap + offset
  char *dst;
  size_t nbytes;
  size_t seg_bytes;
};

__global__ void __launch_bounds__(kThreads, 1) get_bulk_kernel(GetArgs a) {
  extern __shared__ __align__(128) char dyn_smem[];
  const BulkRing br = bulk_ring_init(dyn_smem);
  if (threadIdx.x != 0) return;
  const size_t nseg = (a.nbytes + a.seg_bytes - 1) / a.seg_bytes;
  const uint32_t b = blockIdx.x, G = gridDim.x;
  const uint32_t mine = nseg > b ? uint32_t((nseg - 1 - b) / G + 1) : 0;
  bulk_copy_segments<BulkPull>(
      br, mine,
      [&](uint32_t i) {
        const size_t lo = (size_t(b) + size_t(i) * G) * a.seg_bytes;
        const uint32_t len = uint32_t((a.nbytes - lo) < a.seg_bytes ? (a.nbytes - lo) : a.seg_bytes);
        return BulkSeg{a.src + lo, a.dst + lo, len};
      },
      [&](uint32_t, bool) { return 1; }, [&](uint32_t) {});
}

__global__ void __launch_bounds__(kThreads) get_ldst_kernel(GetArgs a) {
  const Units un = make_units(a.nbytes);
  const size_t U = un.total();
  const bool sal = is_aligned16(a.src), dal = is_aligned16(a.dst);
  for (size_t u = size_t(blockIdx.x) * kThreads + threadIdx.x; u < U; u += size_t(gridDim.x) * kThreads) {
    uint4 v;
    if (sal && u < un.full) v = ld_peer(a.src + (u << 4));
    else v = load_user_unit(a.src, u, un, false);
    store_user_unit(a.dst, u, un, dal, v);
  }
}

static int p2p_common(b200_comm *c, void *buf, size_t nbytes, int peer, cudaStream_t stream, bool send) {
  int rc;
  if ((rc = check_usable(c)) || (rc = check_rank(c, peer, "peer"))) return rc;
  if (peer == c->rank) {
    set_error("peer rank %d is this rank", peer);
    return B200_ERR_INVALID;
  }
  if (nbytes == 0) return B200_OK;
  if (!buf) return null_tensor_error();
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  // Grid is a pure function of the message size so both sides pair CTA b with CTA b.
  const P2PPlan p = p2p_plan(c, buf, nbytes);
  P2PArgs a{static_cast<char *>(buf), nbytes, p.chunk, peer};
  if (p.bulk) {
    auto k = send ? p2p_bulk_kernel<true> : p2p_bulk_kernel<false>;
    if ((rc = set_dyn_smem(c->device, reinterpret_cast<const void *>(k)))) return rc;
    k<<<p.rings, kThreads, kBulkSmemBytes, stream>>>(c->dev(), a);
  } else if (send) {
    p2p_kernel<true><<<p.rings, kThreads, 0, stream>>>(c->dev(), a);
  } else {
    p2p_kernel<false><<<p.rings, kThreads, 0, stream>>>(c->dev(), a);
  }
  B200_LAUNCH_CHECK(c);
  return B200_OK;
}

// a kernel of this file's CUDA module, for preload_kernels() (bootstrap.cu)
const void *p2p_module_anchor() { return reinterpret_cast<const void *>(&get_bulk_kernel); }

}  // namespace b200

using namespace b200;

extern "C" int b200_send(b200_comm_t c, const void *buf, size_t nbytes, int peer, void *stream) {
  return p2p_common(c, const_cast<void *>(buf), nbytes, peer, static_cast<cudaStream_t>(stream), true);
}

extern "C" int b200_recv(b200_comm_t c, void *buf, size_t nbytes, int peer, void *stream) {
  return p2p_common(c, buf, nbytes, peer, static_cast<cudaStream_t>(stream), false);
}

extern "C" int b200_alltoall(b200_comm_t c, const void *const *ins, const size_t *send_counts, void *const *outs,
                             const size_t *recv_counts, int dtype, void *stream_) {
  int rc;
  size_t es;
  if ((rc = check_usable(c)) || (rc = check_dtype(dtype, &es))) return rc;
  if (!ins || !outs || !send_counts || !recv_counts) {
    set_error("null argument array");
    return B200_ERR_INVALID;
  }
  const int n = c->world, me = c->rank;
  size_t total = 0;
  for (int p = 0; p < n; ++p) {
    if (send_counts[p] && !ins[p]) {
      set_error("input %d is null but has %zu elements", p, send_counts[p]);
      return B200_ERR_INVALID;
    }
    if (recv_counts[p] && !outs[p]) {
      set_error("output %d is null but has %zu elements", p, recv_counts[p]);
      return B200_ERR_INVALID;
    }
    total += send_counts[p] + recv_counts[p];
  }
  if (send_counts[me] != recv_counts[me]) {
    set_error("own segment: %zu elements sent but %zu received", send_counts[me], recv_counts[me]);
    return B200_ERR_INVALID;
  }
  // In place is not supported: a receive may land before a send to another peer has read its input.
  // The one exception is an own segment whose output IS its input (c10d gather / scatter at the root
  // with gather_list[root] / scatter_list[root] the rank's own tensor): there is nothing to copy.
  const bool own_alias = send_counts[me] && outs[me] == ins[me];
  if (own_alias) total -= 2 * send_counts[me];
  for (int q = 0; q < n; ++q) {
    if (!recv_counts[q]) continue;
    const uintptr_t olo = reinterpret_cast<uintptr_t>(outs[q]), ohi = olo + recv_counts[q] * es;
    for (int p = 0; p < n; ++p) {
      if (!send_counts[p] || (own_alias && p == me && q == me)) continue;
      const uintptr_t ilo = reinterpret_cast<uintptr_t>(ins[p]), ihi = ilo + send_counts[p] * es;
      if (olo < ihi && ilo < ohi) {
        set_error("output %d overlaps input %d (in-place all-to-all is not supported)", q, p);
        return B200_ERR_INVALID;
      }
    }
  }
  if (total == 0) return B200_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  const size_t own_bytes = own_alias ? 0 : send_counts[me] * es;
  if (n == 1) {
    B200_CHECK_CUDA(cudaMemcpyAsync(outs[0], ins[0], own_bytes, cudaMemcpyDeviceToDevice, stream));
    return B200_OK;
  }
  // Every role needs a CTA.  Checked against the world size rather than this call's counts, so all
  // ranks refuse together instead of one refusing while its peers wait for it.
  const int cap = a2a_grid_cap(c);
  if (cap < 2 * (n - 1)) {
    set_error("all-to-all needs %d co-resident CTAs at world size %d but the grid is capped at %d "
              "(b200_comm_set_blocks)", 2 * (n - 1), n, cap);
    return B200_ERR_INVALID;
  }
  const int kcap = a2a_ring_cap(c, cap);
  A2AArgs a{};
  int grid = 0;
  bool any_bulk = false;
  for (int send = 1; send >= 0; --send) {
    for (int s = 1; s < n; ++s) {
      const int peer = send ? (me + s) % n : (me - s + n) % n;
      const size_t nbytes = (send ? send_counts[peer] : recv_counts[peer]) * es;
      if (nbytes == 0) continue;
      char *buf = send ? const_cast<char *>(static_cast<const char *>(ins[peer])) : static_cast<char *>(outs[peer]);
      // what b200_send / b200_recv would do with this transfer alone, on at most kcap rings
      const P2PPlan p = p2p_plan(c, buf, nbytes);
      const int G = p.rings < kcap ? p.rings : kcap;
      a.role[a.nroles++] = A2ARole{buf, nbytes, p.chunk, peer, grid, G, send, p.bulk};
      any_bulk = any_bulk || p.bulk;
      grid += G;
    }
  }
  // grid <= 2(n-1) * kcap <= cap here
  a.role_ctas = grid;
  a.own_src = static_cast<const char *>(ins[me]);
  a.own_dst = static_cast<char *>(outs[me]);
  a.own_bytes = own_bytes;
  // Every CTA copies a slice of the own segment; a large one gets extra copy-only CTAs, within the
  // cap.  Copy-only CTAs never wait.
  const size_t own_ctas = a2a_own_ctas(own_bytes);
  if (own_ctas > size_t(grid)) grid = int(own_ctas < size_t(cap) ? own_ctas : size_t(cap));
  a.own_bulk = grid > a.role_ctas && is_aligned16(a.own_src) && is_aligned16(a.own_dst) && (own_bytes & 15) == 0;
  any_bulk = any_bulk || a.own_bulk;
  if (any_bulk) {
    if ((rc = set_dyn_smem(c->device, reinterpret_cast<const void *>(alltoall_kernel)))) return rc;
    alltoall_kernel<<<grid, kThreads, kBulkSmemBytes, stream>>>(c->dev(), a);
  } else {
    alltoall_kernel<<<grid, kThreads, 0, stream>>>(c->dev(), a);
  }
  B200_LAUNCH_CHECK(c);
  return B200_OK;
}

extern "C" int b200_symm_base(b200_comm_t c, void **base, size_t *bytes) {
  int rc = check_usable(c);
  if (rc) return rc;
  if (base) *base = reinterpret_cast<char *>(c->data.va[c->rank]) + 2 * c->staging_bytes;
  if (bytes) *bytes = c->heap_bytes;
  return B200_OK;
}

extern "C" int b200_get(b200_comm_t c, void *dst, int src_rank, size_t src_heap_offset, size_t nbytes, void *stream_) {
  int rc;
  if ((rc = check_usable(c)) || (rc = check_rank(c, src_rank, "source"))) return rc;
  if (src_heap_offset + nbytes > c->heap_bytes) {
    set_error("[%zu, %zu) is outside the %zu-byte symmetric heap", src_heap_offset, src_heap_offset + nbytes,
              c->heap_bytes);
    return B200_ERR_INVALID;
  }
  if (nbytes == 0) return B200_OK;
  if (!dst) return null_tensor_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  GetArgs a{reinterpret_cast<const char *>(c->data.va[src_rank]) + 2 * c->staging_bytes + src_heap_offset,
            static_cast<char *>(dst), nbytes, kGetSegBytes};
  if (get_bulk(a.src, a.dst, nbytes)) {
    const size_t nseg = (nbytes + a.seg_bytes - 1) / a.seg_bytes;
    const int g = int(nseg < 16 ? nseg : 16);
    if ((rc = set_dyn_smem(c->device, reinterpret_cast<const void *>(get_bulk_kernel)))) return rc;
    get_bulk_kernel<<<g, kThreads, kBulkSmemBytes, stream>>>(a);
  } else {
    const size_t U = make_units(nbytes).total();
    const int g = int((U + kThreads - 1) / kThreads < 32 ? (U + kThreads - 1) / kThreads : 32);
    get_ldst_kernel<<<g, kThreads, 0, stream>>>(a);
  }
  B200_LAUNCH_CHECK(c);
  return B200_OK;
}
