// policy.h — every launch decision of the library: algorithm thresholds, CTA counts, chunk sizes.
// The defaults are break-evens measured with one GPU per rank on an NVSwitch system, none re-measured
// on H100.  A b200_param_t left at -1 takes the default; whether 0 is a value or also means the
// default is stated per parameter.
#pragma once
#include "bulk_copy.cuh"
#include "kernel_utils.cuh"
#include "pipe.h"

namespace b200 {

// CTAs a launch may use: b200_comm_set_blocks when set, else one per SM
inline int grid_cap(const b200_comm *c) { return c->forced_blocks > 0 ? c->forced_blocks : c->sm_count; }

// One CTA per work item, at most `cap` (b200_comm_set_blocks overrides it) and kMaxBlocks.
inline int pick_blocks(const b200_comm *c, size_t work_items, int cap) {
  if (c->forced_blocks > 0) cap = grid_cap(c);
  size_t want = work_items < 1 ? 1 : work_items;
  int g = int(want < size_t(cap) ? want : size_t(cap));
  if (g > kMaxBlocks) g = kMaxBlocks;
  return g < 1 ? 1 : g;
}

// ---- all-reduce ------------------------------------------------------------------------------

inline bool nvls_capable(int dtype, int op) {
  return (dtype == B200_F32 || dtype == B200_F16 || dtype == B200_BF16) &&
         (op == B200_SUM || op == B200_AVG);
}

// With two ranks the switch reduction saves no traffic and the peer-load kernel is faster; from
// five ranks on NVLS wins at every size (tuned with one GPU per rank on an NVSwitch system).
// B200_PARAM_NVLS_MIN_WORLD >= 0 replaces the rule by "world >= value".
inline bool nvls_pays_off(const b200_comm *c, size_t nbytes) {
  const long long min_world = c->params[B200_PARAM_NVLS_MIN_WORLD];
  if (min_world >= 0) return c->world >= min_world;
  if (c->world <= 2) return false;
  if (c->world <= 4) return nbytes >= (size_t(128) << 20);
  return true;
}

// Zero-copy operands: the NVSwitch reduction saturates with far fewer CTAs than the GPU has SMs
// (64 CTAs beat a whole-GPU grid), so those launches are capped at 64 CTAs.  Staged operands
// keep CTA-to-CTA barriers over the whole grid by default: running their reduce phase on fewer
// CTAs (B200_PARAM_NVLS_CTAS > 0) needs grid-wide waits, which serialise the phases and are slower.
inline int nvls_ctas(const b200_comm *c) {
  const long long v = c->params[B200_PARAM_NVLS_CTAS];
  return v > 0 ? int(v) : 0;
}

// LL pays n-1 flag-doubled pushes per rank: its break-even against the one-shot kernel is
// ~32 KiB with 2 ranks and ~4 KiB with 8 (one GPU per rank, NVSwitch).
inline size_t ll_limit(const b200_comm *c) {
  const long long v = c->params[B200_PARAM_LL_MAX_BYTES];
  const size_t lim = v >= 0 ? size_t(v) : (size_t(64) << 10) / size_t(c->world) / (c->world > 4 ? 2 : 1);
  return lim < kLLMaxPayload ? lim : kLLMaxPayload;
}

// Each rank reads world * nbytes in the one-shot scheme.  Break-even against the two-shot kernel
// is ~1 MiB with 2 ranks and ~256 KiB with 8; the 0.5 MB PPO gradient vector of BASELINE
// configs[3] falls on the one-shot side at 2 and 4 ranks.
inline size_t oneshot_limit(const b200_comm *c) {
  const long long v = c->params[B200_PARAM_ONESHOT_MAX_BYTES];
  if (v >= 0) return size_t(v);
  return (size_t(5) << 19) / size_t(c->world);  // 2.5 MiB / n
}

// Break-even of the pipelined kernels against the phase-by-phase ones (one GPU per rank, NVSwitch).
inline size_t pipe_min_bytes(const b200_comm *c) {
  const long long v = c->params[B200_PARAM_PIPE_MIN_BYTES];
  if (v >= 0) return size_t(v);
  // 2 ranks: the pull kernel wins from 16 MiB; NVLS roles from 128 MiB
  return c->world == 2 ? (size_t(16) << 20) : (size_t(128) << 20);
}

// ---- pipelined kernels (allreduce_pipe.cu) ---------------------------------------------------

// Chunks are whole multiples of this, so C / G is a whole number of tiles for any power-of-two G <= 32.
constexpr size_t kPipeQuantum = size_t(32) * kBulkTile;

// the staging slot holds at least one chunk
inline bool pipe_fits(const b200_comm *c) { return c->staging_bytes >= kPipeQuantum; }

struct PipePlan {
  size_t chunk;      // C: a multiple of kPipeQuantum that fits the slot (0: the slot is too small)
  int copy_ctas;     // CTAs per copy role (power of two)
  int work_ctas;     // reduce / pull CTAs; < 1 when the grid cap leaves none
  int grid;
  uint32_t ring;     // chunks of the slot used as a ring by messages larger than it (0: no ring)
  size_t max_bytes;  // largest message one launch takes, in whole chunks
};

// Defaults (tuned on an NVSwitch system with one GPU per rank; not re-tuned on H100, where the
// B200_PARAM_PIPE_* parameters override them; 0 means the default for all three):
//   all-reduce, 2 ranks (pull)   : 1 MiB chunks, 32 copy-in + 32 pull CTAs
//   all-reduce, 3-4 ranks        : 4 MiB chunks, 16 + 16 copy CTAs, 64 reduce CTAs
//   all-reduce, 5-8 ranks        : 8 MiB chunks, 16 + 16 copy CTAs, 32 reduce CTAs (the switch
//                                  reduction saturates with few CTAs)
//   all-gather (pull)            : 1 MiB chunks, 16 copy-in CTAs + 64 / 48 / 32 pull CTAs at
//                                  2 / 3-4 / 5-8 ranks (pull CTAs also move the rank's own tensor
//                                  in -> out: half of all bytes at 2 ranks, 1/8 at 8)
inline PipePlan pipe_plan(const b200_comm *c, PipeVariant variant) {
  PipePlan p{};
  const int n = c->world;
  const long long vc = c->params[B200_PARAM_PIPE_CHUNK_BYTES];
  size_t C = vc > 0                          ? size_t(vc)
             : variant == PIPE_GATHER || n == 2 ? (size_t(1) << 20)
                                                : (n <= 4 ? (size_t(4) << 20) : (size_t(8) << 20));
  C = round_up(C, kPipeQuantum);
  const size_t fit = c->staging_bytes / kPipeQuantum * kPipeQuantum;
  p.chunk = C < fit ? C : fit;
  if (p.chunk == 0) return p;

  // chunk ring of the n >= 3 all-reduce: on whenever the slot holds at least 4 chunks.  The pull
  // kernels have none: there the READER of a slot is a peer.
  const bool ring_kernel = variant == PIPE_NVLS || variant == PIPE_PEER;
  if (ring_kernel && c->staging_bytes / p.chunk >= 4) p.ring = uint32_t(c->staging_bytes / p.chunk);
  size_t cap = p.ring ? ~size_t(0) : c->staging_bytes;
  const size_t by_chunks = size_t(kMaxPipeChunks) * p.chunk;  // per-chunk flags and counters
  cap = cap < by_chunks ? cap : by_chunks;
  p.max_bytes = cap / p.chunk * p.chunk;  // whole chunks, so a split message continues on a chunk boundary

  const long long pc = c->params[B200_PARAM_PIPE_COPY_CTAS];
  const long long pr = c->params[B200_PARAM_PIPE_RED_CTAS];
  int G = pc > 0 ? int(pc) : (variant == PIPE_PULL ? 32 : 16);
  int W = pr > 0 ? int(pr)
      : variant == PIPE_PULL   ? 32
      : variant == PIPE_GATHER ? (n == 2 ? 64 : (n <= 4 ? 48 : 32))
                               : (n <= 4 ? 64 : 32);
  const int roles = ring_kernel ? 2 : 1;  // copy roles: copy-in (+ copy-out for the n >= 3 all-reduce)
  const int cap_ctas = grid_cap(c);
  if (roles * G + W > cap_ctas) {  // shared-GPU harness / small parts: shrink, keep at least one worker
    while (G > 1 && roles * G + 1 > cap_ctas / 2) G /= 2;
    W = cap_ctas - roles * G;
  }
  p.copy_ctas = 1;  // the largest power of two <= min(G, 32)
  while (p.copy_ctas * 2 <= (G > 32 ? 32 : G)) p.copy_ctas *= 2;
  p.work_ctas = W;
  p.grid = roles * p.copy_ctas + W;
  return p;
}

// An automatic choice takes a pipelined kernel only when the grid cap leaves it a worker CTA; below
// that the phase-by-phase kernels, which run on any grid, take the message.  An explicit
// B200_ALGO_PIPE is refused instead.  The cap is the same on every rank, so all ranks choose alike.
inline bool pipe_runs(const b200_comm *c, PipeVariant variant) { return pipe_plan(c, variant).work_ctas >= 1; }

// ---- all-gather, broadcast, gradient all-reduce ----------------------------------------------

// Per-rank size from which an aligned all-gather takes the pull kernel (B200_PARAM_AG_PULL_MIN_BYTES;
// 0 = never).  4 ranks: 1 MiB/rank takes 49 us pulled vs 28 us staged.
inline bool ag_pull_pays_off(const b200_comm *c, size_t nbytes) {
  const long long v = c->params[B200_PARAM_AG_PULL_MIN_BYTES];
  if (v == 0) return false;
  return nbytes >= (v > 0 ? size_t(v) : (size_t(4) << 20));
}

// Windows of the uneven all-gather and reduce-scatter (b200_allgatherv, b200_reducescatterv): window
// w covers units [w * W, (w + 1) * W) of every rank's part, so launches = ceil(max_units / W).  The
// plan is a function of the size list and W (from staging_bytes and the world size) alone, so every
// rank makes the same launches whatever its own part.
struct VPlan {
  size_t max_units;     // the largest part, in 16-byte units
  size_t window_units;  // W
};
inline VPlan v_plan(const size_t *nbytes, int n, size_t window_units) {
  VPlan v{0, window_units};
  for (int p = 0; p < n; ++p) {
    const size_t u = (nbytes[p] + 15) / 16;
    if (u > v.max_units) v.max_units = u;
  }
  return v;
}
// Bytes of a part of `nbytes` inside the window of `units` units that starts at unit u0 (0 once the
// part is exhausted).
inline size_t v_window_bytes(size_t nbytes, size_t u0, size_t units) {
  const size_t done = u0 << 4;
  if (nbytes <= done) return 0;
  const size_t left = nbytes - done;
  return left < (units << 4) ? left : (units << 4);
}

// The multicast store pays off once more than one peer would pull from the root.
inline bool broadcast_nvls(const b200_comm *c, size_t nbytes) {
  return c->mc_active && c->world > 2 && nbytes >= (size_t(64) << 10);
}

// The gradient kernel's reduce phase runs on the switch from 3 ranks on (B200_PARAM_NVLS_MIN_WORLD >= 0
// replaces the 3).
inline bool grad_nvls(const b200_comm *c) {
  const long long v = c->params[B200_PARAM_NVLS_MIN_WORLD];
  return c->mc_active && c->world >= (v >= 0 ? v : 3);
}

// Shard elements per launch of the fused gradient reduce-scatter: the n sub-slots of a piece,
// ceil(m / E) 16-byte wire units each (E = 16 / wire element size), fill at most one staging slot.
// A multiple of 8 elements, so every piece starts on a whole wire unit and keeps its stripe's
// 16-byte alignment.
inline size_t grad_rs_piece_elems(const b200_comm *c, size_t wire_es) {
  const size_t units = c->staging_bytes / (size_t(c->world) * 16);
  return (units * (16 / wire_es)) & ~size_t(7);
}

// ---- point-to-point, all-to-all, get (p2p.cu) ------------------------------------------------

// Chunk size is a pure function of the message size, so sender and receiver agree: big messages
// use whole ring slots; mid-size ones are cut into kP2PRings pieces so that every CTA (one per
// ring) carries one chunk and the message moves in parallel instead of through one CTA.
inline size_t p2p_chunk_bytes(size_t nbytes, size_t slot_bytes) {
  size_t c = (nbytes + kP2PRings - 1) / kP2PRings;
  c = (c + 4095) & ~size_t(4095);
  if (c < (size_t(16) << 10)) c = size_t(16) << 10;
  return c < slot_bytes ? c : slot_bytes;
}

struct P2PPlan {
  size_t chunk;  // bytes per chunk, the same on both sides
  int rings;     // sub-rings = CTAs, one chunk each at least
  bool bulk;     // this side moves its bytes with the bulk-copy unit
};

// The protocol (rings, slots, chunking) is a function of the message size alone; HOW this side
// moves its bytes is a local choice: the bulk-copy unit when the tensor is 16-byte aligned, a
// whole number of 16-byte units and the chunks are big enough to be worth a TMA pipeline
// (B200_PARAM_P2P_BULK_MIN_CHUNK, default 32 KiB; 0 = never).
inline P2PPlan p2p_plan(const b200_comm *c, const void *buf, size_t nbytes) {
  P2PPlan p;
  p.chunk = p2p_chunk_bytes(nbytes, c->inbox_bytes / kP2PRings / kP2PSlots);
  const size_t nchunks = (nbytes + p.chunk - 1) / p.chunk;
  p.rings = int(nchunks < size_t(kP2PRings) ? nchunks : size_t(kP2PRings));
  const long long pb = c->params[B200_PARAM_P2P_BULK_MIN_CHUNK];
  const size_t bulk_min_chunk = pb >= 0 ? size_t(pb) : (size_t(32) << 10);
  p.bulk = is_aligned16(buf) && (nbytes & 15) == 0 && p.chunk >= bulk_min_chunk && pb != 0;
  return p;
}

// Tensor lists (b200_send_multi / b200_recv_multi / b200_get_multi) travel as tables of at most
// kP2PTableMax non-empty entries, one launch per table.  The table is a __grid_constant__ kernel
// parameter: CUDA >= 12.1 allows 32764 bytes of parameters on sm_90, and 256 entries take about
// 6 KiB (send / recv / broadcast), 8 KiB (get) or 22 KiB (all-gather / reduce-scatter, which add
// kMaxRanks per-rank pointers to each entry).  What a parameter block that large costs per launch
// has not been measured in isolation.
constexpr int kP2PTableMax = B200_P2P_TABLE_MAX;

// A table is ONE message of 16 * (sum of ceil(nbytes[i] / 16)) bytes: the protocol (chunk, rings)
// is p2p_plan's for that packed size, a pure function of the size list.  This side moves its bytes
// with the bulk-copy unit when p2p_plan would for the packed size, every tensor of its table is
// 16-byte aligned and whole units, and the tensors average at least kP2PTableBulkMinAvg bytes: every
// (chunk, tensor) piece is a bulk segment with its own set-up, which small tensors do not repay.
// The 32 KiB threshold mirrors B200_PARAM_P2P_BULK_MIN_CHUNK's default; it was not tuned.
constexpr size_t kP2PTableBulkMinAvg = size_t(32) << 10;
inline P2PPlan p2p_table_plan(const b200_comm *c, size_t wire_bytes, int count, bool whole_aligned) {
  P2PPlan p = p2p_plan(c, nullptr, wire_bytes);
  p.bulk = p.bulk && whole_aligned && wire_bytes / size_t(count) >= kP2PTableBulkMinAvg;
  return p;
}

// All-to-all grid: at most one CTA per SM keeps it co-resident even with the bulk roles'
// shared-memory ring.  Both sides of a pair derive their rings from this cap, so
// b200_comm_set_blocks must be identical on every rank.
inline int a2a_grid_cap(const b200_comm *c) {
  const int cap = grid_cap(c);
  return cap > c->sm_count ? c->sm_count : cap;
}

// rings per (peer, direction) role: the 2(n-1) roles share the grid
inline int a2a_ring_cap(const b200_comm *c, int cap) {
  const int k = cap / (2 * (c->world - 1));
  return k < 1 ? 1 : (k > kP2PRings ? kP2PRings : k);
}

// CTAs of one (peer, direction) role of b200_p2p_batch: the roles present share the co-resident grid,
// and a role never takes more CTAs than its largest op has sub-rings.  A local choice: each op keeps
// p2p_plan's rings on the wire, and a role with fewer CTAs than rings folds several sub-rings onto
// one CTA, so the peer may choose differently.
inline int p2p_batch_ctas(int cap, int roles, int max_rings) {
  int g = cap / roles;
  if (g < 1) g = 1;
  if (g > max_rings) g = max_rings;
  return g > kP2PRings ? kP2PRings : g;
}

// A large own segment gets copy-only CTAs, one per 64 KiB: a local copy of MiBs next to small
// remote messages would otherwise crawl through the few role CTAs.
inline size_t a2a_own_ctas(size_t own_bytes) { return (own_bytes + (size_t(64) << 10) - 1) / (size_t(64) << 10); }

// b200_get moves aligned whole-unit ranges of at least one bulk segment with the bulk-copy unit.
constexpr size_t kGetSegBytes = size_t(256) << 10;
inline bool get_bulk(const void *src, const void *dst, size_t nbytes) {
  return is_aligned16(src) && is_aligned16(dst) && (nbytes & 15) == 0 && nbytes >= kGetSegBytes;
}
// b200_get_multi: one table takes the bulk kernel when every entry is aligned whole units on both
// ends and the entries average at least one bulk segment, the single get's threshold.
inline bool get_table_bulk(size_t total_bytes, int count, bool whole_aligned) {
  return whole_aligned && total_bytes / size_t(count) >= kGetSegBytes;
}

}  // namespace b200
