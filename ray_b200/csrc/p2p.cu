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
// picking its own copy mechanism.  The same two functions move a table of tensors as one message
// (p2p_table_kernel / p2p_bulk_table_kernel: b200_send_multi / b200_recv_multi), and run a batch of
// sends and receives, each on the plain send / recv wire, as one grid (p2p_batch_kernel:
// b200_p2p_batch).
#include <type_traits>

#include "bulk_copy.cuh"
#include "policy.h"
#include "tensor_table.cuh"

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

// ---------------------------------------------------------------------------
// Where the bytes of a message live: one contiguous buffer (char *), or a table of tensors
// (b200_send_multi / b200_recv_multi) whose packed stream of 16-byte units (tensor_table.cuh) is
// the message.
// ---------------------------------------------------------------------------
struct P2PTableArgs {
  P2PTable t;
  size_t nbytes;  // bytes on the wire: 16 * ustart[count]
  size_t chunk;
  int peer;
};

// unit u of the chunk that starts at byte lo of the message
__device__ __forceinline__ uint4 msg_load_unit(char *buf, size_t lo, size_t u, const Units &un, bool al) {
  return load_user_unit(buf + lo, u, un, al);
}
__device__ __forceinline__ uint4 msg_load_unit(const P2PTable *t, size_t lo, size_t u, const Units &, bool) {
  return table_load_unit(*t, (lo >> 4) + u);
}
__device__ __forceinline__ void msg_store_unit(char *buf, size_t lo, size_t u, const Units &un, bool al, uint4 v) {
  store_user_unit(buf + lo, u, un, al, v);
}
__device__ __forceinline__ void msg_store_unit(const P2PTable *t, size_t lo, size_t u, const Units &, bool, uint4 v) {
  table_store_unit(*t, (lo >> 4) + u, v);
}

// One CTA's share of a message: chunks b, b + G, b + 2G, ... over sub-ring b, moved with 16-byte
// ld/st by all kThreads threads.  Both sides of a pair call it with the same (G, chunk).  `msg` is
// a buffer (char *) or a table (const P2PTable *); a table's chunks are whole 16-byte units.
template <bool SEND, typename Msg>
__device__ __forceinline__ void p2p_ldst_ring(const DevComm &c, int peer, int b, int G, Msg msg, size_t nbytes,
                                              size_t chunk) {
  const int me = c.rank;
  const size_t ring_bytes = c.inbox_bytes / kP2PRings;
  const size_t slot_bytes = ring_bytes / kP2PSlots;
  const size_t nchunks = (nbytes + chunk - 1) / chunk;
  const bool al = is_aligned16(msg);

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
          if (u < U) v[k] = msg_load_unit(msg, lo, u, un, al);
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
          if (u < U) msg_store_unit(msg, lo, u, un, al, v[k]);
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
// Bulk segments of one CTA's chunks of a table: a chunk that spans several tensors is one segment
// per (chunk, tensor) pair.  The segment engine asks for segments through three cursors (load, store,
// completion), each in increasing order; `at` keeps one position per cursor and walks forward from
// the nearest one at or below the request, so a lookup costs O(1) amortised -- per segment, never
// per tile.
struct TableSegs {
  struct Pos {
    uint32_t seg;  // segment index within this CTA
    uint32_t q;    // chunk of this CTA
    int t;         // table entry
  };
  const P2PTable &tb;
  size_t b, G, cu, tu;  // CTA, CTAs, units per chunk, units of the message
  Pos p0, p1, p2;       // named, not an array: the copy thread keeps them in registers

  __device__ TableSegs(const P2PTable &t, int b_, int G_, size_t chunk)
      : tb(t), b(size_t(b_)), G(size_t(G_)), cu(chunk >> 4), tu(t.ustart[t.count]) {
    p0 = p1 = p2 = start();
  }
  __device__ Pos start() const { return Pos{0, 0, table_entry(tb.ustart, tb.count, lo(0))}; }
  __device__ size_t lo(uint32_t q) const { return (b + size_t(q) * G) * cu; }
  __device__ size_t hi(uint32_t q) const { return lo(q) + cu < tu ? lo(q) + cu : tu; }
  // segments of the first nq chunks of this CTA
  __device__ uint32_t count(uint32_t nq) const {
    uint32_t n = 0;
    for (uint32_t q = 0; q < nq; ++q)
      n += uint32_t(table_entry(tb.ustart, tb.count, hi(q) - 1) - table_entry(tb.ustart, tb.count, lo(q)) + 1);
    return n;
  }
  __device__ Pos at(uint32_t i) {
    int k = -1;
    uint32_t best = 0;
    if (p0.seg <= i) k = 0, best = p0.seg;
    if (p1.seg <= i && (k < 0 || p1.seg > best)) k = 1, best = p1.seg;
    if (p2.seg <= i && (k < 0 || p2.seg > best)) k = 2;
    Pos p = k == 0 ? p0 : k == 1 ? p1 : k == 2 ? p2 : start();
    while (p.seg < i) {
      ++p.seg;
      if (tb.ustart[p.t + 1] < hi(p.q)) {
        ++p.t;
      } else {
        ++p.q;
        p.t = table_entry(tb.ustart, tb.count, lo(p.q));
      }
    }
    if (k == 1) p1 = p;
    else if (k == 2) p2 = p;
    else p0 = p;
    return p;
  }
  __device__ bool opens_chunk(const Pos &p) const { return tb.ustart[p.t] <= lo(p.q); }
  __device__ bool closes_chunk(const Pos &p) const { return tb.ustart[p.t + 1] >= hi(p.q); }
  // (user bytes, offset in the chunk, bytes) of segment p: every tensor of a bulk table is whole units
  __device__ BulkSeg seg(const Pos &p, char *chunk_slot, bool send) const {
    const size_t s = tb.ustart[p.t], e = tb.ustart[p.t + 1];
    const size_t ulo = s > lo(p.q) ? s : lo(p.q), uhi = e < hi(p.q) ? e : hi(p.q);
    char *user = tb.ptr[p.t] + ((ulo - s) << 4);
    char *slot = chunk_slot + ((ulo - lo(p.q)) << 4);
    const uint32_t len = uint32_t((uhi - ulo) << 4);
    return send ? BulkSeg{user, slot, len} : BulkSeg{slot, user, len};
  }
};

// The same share of a message moved by the bulk-copy unit; `dyn_smem` holds kBulkSmemBytes.  A
// buffer `msg` must be 16-byte aligned and `nbytes` a multiple of 16; so must every tensor of a
// table.  Only threads 0 and 32 drive the transfer; warps 2.. run side(thread, nthreads) meanwhile
// (the all-to-all gives them its own-segment copy).
template <bool SEND, typename Msg, typename SideFn>
__device__ __forceinline__ void p2p_bulk_ring(const DevComm &c, int peer, int b, int G, Msg msg, size_t nbytes,
                                              size_t chunk, char *dyn_smem, SideFn side) {
  constexpr bool kTable = std::is_same<Msg, const P2PTable *>::value;
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
    // ---- copy thread: one segment per chunk (per chunk and tensor for a table) ------------------
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
    auto copy = [&](uint32_t nsegs, auto seg, auto seg_gate, auto seg_done) {
      return SEND ? bulk_copy_segments<BulkRemote>(br, nsegs, seg, seg_gate, seg_done)
                  : bulk_copy_segments<BulkLocal>(br, nsegs, seg, seg_gate, seg_done);
    };
    bool ok;
    if constexpr (kTable) {
      // a chunk's gate runs before its first segment, its done after its last
      TableSegs ts(*msg, b, G, chunk);
      ok = copy(
          ts.count(nq32),
          [&](uint32_t i) {
            const TableSegs::Pos p = ts.at(i);
            return ts.seg(p, ring + size_t((seq0 + p.q) % kP2PSlots) * slot_bytes, SEND);
          },
          [&](uint32_t i, bool block) {
            const TableSegs::Pos p = ts.at(i);
            return ts.opens_chunk(p) ? gate(p.q, block) : 1;
          },
          [&](uint32_t i) {
            const TableSegs::Pos p = ts.at(i);
            if (ts.closes_chunk(p)) done(p.q);
          });
    } else {
      auto seg = [&](uint32_t q) {
        const size_t lo = (size_t(b) + size_t(q) * size_t(G)) * chunk;
        const uint32_t len = uint32_t((nbytes - lo) < chunk ? (nbytes - lo) : chunk);
        char *slot = ring + size_t((seq0 + q) % kP2PSlots) * slot_bytes;
        return SEND ? BulkSeg{msg + lo, slot, len} : BulkSeg{slot, msg + lo, len};
      };
      ok = copy(nq32, seg, gate, done);
    }
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

// A table of tensors as one message (b200_send_multi / b200_recv_multi): the same rings, flags and
// sequence numbers, so it interleaves with b200_send / b200_recv in stream order.  The table stays
// in parameter space (__grid_constant__), indexed in place.
template <bool SEND>
__global__ void __launch_bounds__(kThreads, 1) p2p_table_kernel(DevComm c, const __grid_constant__ P2PTableArgs a) {
  p2p_ldst_ring<SEND>(c, a.peer, blockIdx.x, gridDim.x, &a.t, a.nbytes, a.chunk);
}

template <bool SEND>
__global__ void __launch_bounds__(kThreads, 1)
    p2p_bulk_table_kernel(DevComm c, const __grid_constant__ P2PTableArgs a) {
  extern __shared__ __align__(128) char dyn_smem[];
  p2p_bulk_ring<SEND>(c, a.peer, blockIdx.x, gridDim.x, &a.t, a.nbytes, a.chunk, dyn_smem, [](int, int) {});
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
// grouped point-to-point (b200_p2p_batch): a list of sends and receives as ONE co-resident grid.
// Op i is the very message b200_send / b200_recv would make for its buffer -- p2p_plan's chunk and
// R rings, on the same sub-rings and persistent sequence numbers -- so it pairs with a plain send /
// recv on the peer or with an op of the peer's batch, in any mix.
//
// Each (peer, direction) present is a role of G CTAs (p2p_batch_ctas), holding its ops in list
// order.  Sub-ring r of every op of the role belongs to CTA r mod G, which runs exactly what CTA r of
// the standalone p2p_kernel / p2p_bulk_kernel would, for each of its (op, sub-ring) pairs in
// lexicographic order.  One sub-ring's messages therefore stay serialised on one CTA, in order.
//
// Why folding cannot deadlock against any peer: number the messages of a directed pair m = 0, 1, ...
// in stream order (the same numbering on both sides), and consider the smallest (m, r) that some
// side has not finished.  Every CTA of either side serving it has finished all its smaller items, so
// it is serving (m, r) right now -- the grid is co-resident, and a plain kernel runs only once the
// stream reached message m.  A sender of (m, r) waits only for acks of earlier chunks of sub-ring r,
// which the receiver of (m, r) or of an earlier message on r gives; a receiver waits only for chunks
// of (m, r).  So both ends of (m, r) run and it completes: a waiting CTA only ever waits on a
// lexicographically earlier-or-equal (m, r) of the other side, whatever G each side chose.
// ---------------------------------------------------------------------------
struct P2PBatchOp {
  char *buf;
  size_t nbytes;
  size_t chunk;  // p2p_plan's, the same on both sides
  int rings;     // R: p2p_plan's sub-rings for nbytes
  int bulk;      // this side moves the op with the bulk-copy unit
};

struct P2PBatchRole {
  int peer;
  int send;
  int first;   // first CTA of the role in the grid
  int G;       // CTAs of the role
  int lo, hi;  // its ops: op[lo, hi), in list order
};

struct P2PBatchArgs {
  P2PBatchRole role[2 * (kMaxRanks - 1)];
  int nroles;
  P2PBatchOp op[kP2PTableMax];  // grouped by role
};
static_assert(fits_param_space<P2PBatchArgs>(), "p2p batch table exceeds the kernel parameter space");

// Called by every thread between two ring calls of one CTA.  The barrier orders the previous call's
// write-back of the sequence word (thread 0) before the next call reads it (every thread), and its
// shared words before their reset.  Returns whether a wait was abandoned: the ring functions record
// an abort or a watchdog expiry in the sticky status word, from thread 0, before they return.
__device__ __forceinline__ bool p2p_batch_gave_up(const DevComm &c) {
  return __syncthreads_or(threadIdx.x == 0 && *reinterpret_cast<volatile int32_t *>(&c.st->status) != 0) != 0;
}

__global__ void __launch_bounds__(kThreads, 1) p2p_batch_kernel(DevComm c, const __grid_constant__ P2PBatchArgs a) {
  extern __shared__ __align__(128) char dyn_smem[];
  const int cta = int(blockIdx.x);
  int i = 0;
  while (i + 1 < a.nroles && cta >= a.role[i + 1].first) ++i;
  const P2PBatchRole &r = a.role[i];
  const int b = cta - r.first;
  for (int k = r.lo; k < r.hi; ++k) {
    const P2PBatchOp &o = a.op[k];
    for (int ring = b; ring < o.rings; ring += r.G) {
      if (o.bulk) {
        if (r.send) p2p_bulk_ring<true>(c, r.peer, ring, o.rings, o.buf, o.nbytes, o.chunk, dyn_smem, [](int, int) {});
        else p2p_bulk_ring<false>(c, r.peer, ring, o.rings, o.buf, o.nbytes, o.chunk, dyn_smem, [](int, int) {});
        bulk_ring_inval(dyn_smem);
      } else if (r.send) {
        p2p_ldst_ring<true>(c, r.peer, ring, o.rings, o.buf, o.nbytes, o.chunk);
      } else {
        p2p_ldst_ring<false>(c, r.peer, ring, o.rings, o.buf, o.nbytes, o.chunk);
      }
      if (p2p_batch_gave_up(c)) return;
    }
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

// A list of gets in one launch (b200_get_multi).  start[] is a prefix over the entries: their first
// 16-byte unit for the ld/st kernel, their first bulk segment for the bulk kernel.
struct GetTable {
  int count;
  const char *src[kP2PTableMax];  // peer mapping of the owner's heap + offset
  char *dst[kP2PTableMax];
  unsigned long long nbytes[kP2PTableMax];
  unsigned long long start[kP2PTableMax + 1];
  size_t seg_bytes;
};

// Segments b, b + G, b + 2G, ... of nseg() segments of a get (seg_of(k): global segment k), pulled
// by thread 0
template <typename NsegFn, typename SegOf>
__device__ __forceinline__ void get_bulk_segments(char *dyn_smem, NsegFn nsegs, SegOf seg_of) {
  const BulkRing br = bulk_ring_init(dyn_smem);
  if (threadIdx.x != 0) return;
  const size_t nseg = nsegs();
  const uint32_t b = blockIdx.x, G = gridDim.x;
  const uint32_t mine = nseg > b ? uint32_t((nseg - 1 - b) / G + 1) : 0;
  bulk_copy_segments<BulkPull>(
      br, mine, [&](uint32_t i) { return seg_of(size_t(b) + size_t(i) * G); }, [&](uint32_t, bool) { return 1; },
      [&](uint32_t) {});
}

__global__ void __launch_bounds__(kThreads, 1) get_bulk_kernel(GetArgs a) {
  extern __shared__ __align__(128) char dyn_smem[];
  get_bulk_segments(dyn_smem, [&] { return (a.nbytes + a.seg_bytes - 1) / a.seg_bytes; }, [&](size_t k) {
    const size_t lo = k * a.seg_bytes;
    const uint32_t len = uint32_t((a.nbytes - lo) < a.seg_bytes ? (a.nbytes - lo) : a.seg_bytes);
    return BulkSeg{a.src + lo, a.dst + lo, len};
  });
}

// entry i is aligned and whole units on both ends (host check); its segments are [start[i], start[i+1])
__global__ void __launch_bounds__(kThreads, 1) get_bulk_table_kernel(const __grid_constant__ GetTable a) {
  extern __shared__ __align__(128) char dyn_smem[];
  get_bulk_segments(dyn_smem, [&] { return size_t(a.start[a.count]); }, [&](size_t k) {
    const int i = table_entry(a.start, a.count, k);
    const size_t lo = (k - a.start[i]) * a.seg_bytes;
    const uint32_t len = uint32_t((a.nbytes[i] - lo) < a.seg_bytes ? (a.nbytes[i] - lo) : a.seg_bytes);
    return BulkSeg{a.src[i] + lo, a.dst[i] + lo, len};
  });
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

// unit u of the packed list is unit u - start[i] of entry i; alignment is taken per entry
__global__ void __launch_bounds__(kThreads) get_ldst_table_kernel(const __grid_constant__ GetTable a) {
  const size_t U = a.start[a.count];
  for (size_t u = size_t(blockIdx.x) * kThreads + threadIdx.x; u < U; u += size_t(gridDim.x) * kThreads) {
    const int i = table_entry(a.start, a.count, u);
    const Units un = make_units(a.nbytes[i]);
    const size_t w = u - a.start[i];
    uint4 v;
    if (is_aligned16(a.src[i]) && w < un.full) v = ld_peer(a.src[i] + (w << 4));
    else v = load_user_unit(a.src[i], w, un, false);
    store_user_unit(a.dst[i], w, un, is_aligned16(a.dst[i]), v);
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

// ---- tensor lists -----------------------------------------------------------------------------

static int p2p_multi_common(b200_comm *c, void *const *bufs, const size_t *nbytes, int ntensors, int peer,
                            cudaStream_t stream, bool send) {
  int rc;
  if ((rc = check_usable(c)) || (rc = check_rank(c, peer, "peer"))) return rc;
  if (peer == c->rank) {
    set_error("peer rank %d is this rank", peer);
    return B200_ERR_INVALID;
  }
  if ((rc = check_list(ntensors, bufs && nbytes)) || (rc = check_list_ptrs(bufs, nbytes, ntensors))) return rc;
  if (ntensors == 0) return B200_OK;
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  return for_each_table(nbytes, ntensors, [&](int lo, int hi) -> int {
    P2PTableArgs a{};
    const bool whole_aligned = fill_table(a.t, bufs, nbytes, lo, hi);
    a.nbytes = size_t(a.t.ustart[a.t.count]) * 16;
    const P2PPlan p = p2p_table_plan(c, a.nbytes, a.t.count, whole_aligned);
    a.chunk = p.chunk;
    a.peer = peer;
    if (p.bulk) {
      auto k = send ? p2p_bulk_table_kernel<true> : p2p_bulk_table_kernel<false>;
      if (int rc2 = set_dyn_smem(c->device, reinterpret_cast<const void *>(k))) return rc2;
      k<<<p.rings, kThreads, kBulkSmemBytes, stream>>>(c->dev(), a);
    } else if (send) {
      p2p_table_kernel<true><<<p.rings, kThreads, 0, stream>>>(c->dev(), a);
    } else {
      p2p_table_kernel<false><<<p.rings, kThreads, 0, stream>>>(c->dev(), a);
    }
    B200_LAUNCH_CHECK(c);
    return B200_OK;
  });
}

static int p2p_batch(b200_comm *c, void *const *bufs, const size_t *nbytes, const int *peers, const int *is_send,
                     int nops, cudaStream_t stream) {
  int rc;
  if ((rc = check_usable(c)) || (rc = check_list(nops, bufs && nbytes && peers && is_send))) return rc;
  if (nops > kP2PTableMax) {
    set_error("%d operations in one batch; at most %d fit one launch", nops, kP2PTableMax);
    return B200_ERR_INVALID;
  }
  for (int i = 0; i < nops; ++i) {
    if ((rc = check_rank(c, peers[i], "peer"))) return rc;
    if (peers[i] == c->rank) {
      set_error("operation %d: peer rank %d is this rank", i, peers[i]);
      return B200_ERR_INVALID;
    }
  }
  if ((rc = check_list_ptrs(bufs, nbytes, nops))) return rc;
  // Every role needs a CTA.  Checked against the world size rather than this batch's ops, so all
  // ranks refuse together instead of one refusing while its peers wait for it.
  const int n = c->world, cap = a2a_grid_cap(c);
  if (cap < 2 * (n - 1)) {
    set_error("a p2p batch needs %d co-resident CTAs at world size %d but the grid is capped at %d "
              "(b200_comm_set_blocks)", 2 * (n - 1), n, cap);
    return B200_ERR_INVALID;
  }
  P2PBatchArgs a{};
  int nops_live = 0, roles = 0, max_rings[2 * (kMaxRanks - 1)] = {};
  bool any_bulk = false;
  for (int send = 1; send >= 0; --send) {
    for (int peer = 0; peer < n; ++peer) {
      const int lo = nops_live;
      for (int i = 0; i < nops; ++i) {
        if (!nbytes[i] || peers[i] != peer || (is_send[i] != 0) != (send != 0)) continue;
        // exactly what b200_send / b200_recv would launch for this buffer
        const P2PPlan p = p2p_plan(c, bufs[i], nbytes[i]);
        a.op[nops_live++] = P2PBatchOp{static_cast<char *>(bufs[i]), nbytes[i], p.chunk, p.rings, p.bulk};
        any_bulk = any_bulk || p.bulk;
        if (p.rings > max_rings[roles]) max_rings[roles] = p.rings;
      }
      if (nops_live > lo) a.role[roles++] = P2PBatchRole{peer, send, 0, 0, lo, nops_live};
    }
  }
  if (roles == 0) return B200_OK;
  int grid = 0;
  for (int i = 0; i < roles; ++i) {
    a.role[i].first = grid;
    a.role[i].G = p2p_batch_ctas(cap, roles, max_rings[i]);
    grid += a.role[i].G;  // <= cap: roles <= 2(n-1) <= cap, and G <= max(1, cap / roles)
  }
  a.nroles = roles;
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  if (any_bulk) {
    if ((rc = set_dyn_smem(c->device, reinterpret_cast<const void *>(p2p_batch_kernel)))) return rc;
    p2p_batch_kernel<<<grid, kThreads, kBulkSmemBytes, stream>>>(c->dev(), a);
  } else {
    p2p_batch_kernel<<<grid, kThreads, 0, stream>>>(c->dev(), a);
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

extern "C" int b200_send_multi(b200_comm_t c, const void *const *bufs, const size_t *nbytes, int ntensors, int peer,
                               void *stream) {
  return p2p_multi_common(c, const_cast<void *const *>(bufs), nbytes, ntensors, peer,
                          static_cast<cudaStream_t>(stream), true);
}

extern "C" int b200_recv_multi(b200_comm_t c, void *const *bufs, const size_t *nbytes, int ntensors, int peer,
                               void *stream) {
  return p2p_multi_common(c, bufs, nbytes, ntensors, peer, static_cast<cudaStream_t>(stream), false);
}

extern "C" int b200_p2p_batch(b200_comm_t c, void *const *bufs, const size_t *nbytes, const int *peers,
                              const int *is_send, int nops, void *stream) {
  return p2p_batch(c, bufs, nbytes, peers, is_send, nops, static_cast<cudaStream_t>(stream));
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
  if (src_heap_offset > c->heap_bytes || nbytes > c->heap_bytes - src_heap_offset) {
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

extern "C" int b200_get_multi(b200_comm_t c, void *const *dsts, int src_rank, const size_t *src_heap_offsets,
                              const size_t *nbytes, int ntensors, void *stream_) {
  int rc;
  if ((rc = check_usable(c)) || (rc = check_rank(c, src_rank, "source")) ||
      (rc = check_list(ntensors, dsts && src_heap_offsets && nbytes)))
    return rc;
  for (int i = 0; i < ntensors; ++i) {
    if (src_heap_offsets[i] > c->heap_bytes || nbytes[i] > c->heap_bytes - src_heap_offsets[i]) {
      set_error("tensor %d: [%zu, %zu) is outside the %zu-byte symmetric heap", i, src_heap_offsets[i],
                src_heap_offsets[i] + nbytes[i], c->heap_bytes);
      return B200_ERR_INVALID;
    }
  }
  if ((rc = check_list_ptrs(dsts, nbytes, ntensors))) return rc;
  if (ntensors == 0) return B200_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200_CHECK_CUDA(cudaSetDevice(c->device));
  const char *heap = reinterpret_cast<const char *>(c->data.va[src_rank]) + 2 * c->staging_bytes;
  return for_each_table(nbytes, ntensors, [&](int lo, int hi) -> int {
    GetTable a{};
    a.seg_bytes = kGetSegBytes;
    bool whole_aligned = true;
    size_t total = 0;
    for (int i = lo; i < hi; ++i) {
      if (!nbytes[i]) continue;
      const int k = a.count++;
      a.src[k] = heap + src_heap_offsets[i];
      a.dst[k] = static_cast<char *>(dsts[i]);
      a.nbytes[k] = nbytes[i];
      total += nbytes[i];
      whole_aligned = whole_aligned && is_aligned16(a.src[k]) && is_aligned16(a.dst[k]) && (nbytes[i] & 15) == 0;
    }
    const bool bulk = get_table_bulk(total, a.count, whole_aligned);
    const size_t step = bulk ? a.seg_bytes : 16;  // start[] counts segments or 16-byte units
    for (int k = 0; k < a.count; ++k) a.start[k + 1] = a.start[k] + (a.nbytes[k] + step - 1) / step;
    const size_t n = a.start[a.count];
    if (bulk) {
      const int g = int(n < 16 ? n : 16);
      if (int rc2 = set_dyn_smem(c->device, reinterpret_cast<const void *>(get_bulk_table_kernel))) return rc2;
      get_bulk_table_kernel<<<g, kThreads, kBulkSmemBytes, stream>>>(a);
    } else {
      const int g = int((n + kThreads - 1) / kThreads < 32 ? (n + kThreads - 1) / kThreads : 32);
      get_ldst_table_kernel<<<g, kThreads, 0, stream>>>(a);
    }
    B200_LAUNCH_CHECK(c);
    return B200_OK;
  });
}
