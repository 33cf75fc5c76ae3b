/*
 * b200_collective.h — C ABI of libb200_collective.so
 *
 * Hopper-native (H100, sm_90a) replacement for the device-side work that Ray's
 * GPU collective / tensor-transport hot path delegates to libnccl.  Every entry
 * point takes plain pointers, sizes and a raw cudaStream_t: no torch, cupy or
 * Ray types cross this boundary.  All functions return 0 on success or a
 * negative b200_status_t; b200_last_error() returns a per-thread message.
 *
 * Each function cites the reference call site it replaces
 * (paths relative to the reference tree, python/ray/...).
 *
 * Threading: a communicator may be used from any host thread, one call at a
 * time (the reference guards only its group map, util/collective/collective.py:136-138).
 * b200_comm_abort() and b200_comm_status() are safe from any thread at any time.
 *
 * Stream semantics: every collective is enqueued on the caller's stream and
 * returns without host synchronisation (util/collective/collective_group/
 * nccl_collective_group.py:591-639 enqueues and returns as well).  Collectives of
 * one communicator must be stream-ordered with respect to each other.
 */
#ifndef B200_COLLECTIVE_H_
#define B200_COLLECTIVE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_MAX_RANKS 8      /* one NVSwitch domain of a single HGX H100 host */
#define B200_HANDLE_BYTES 256 /* size of the opaque bootstrap blob */

typedef struct b200_comm *b200_comm_t;

typedef enum {
  B200_OK = 0,
  B200_ERR_INVALID = -1,      /* bad argument (maps to ValueError / RuntimeError in Python) */
  B200_ERR_CUDA = -2,         /* a CUDA runtime / driver call failed */
  B200_ERR_SYSTEM = -3,       /* socket / fd passing failure during bootstrap */
  B200_ERR_UNSUPPORTED = -4,  /* dtype/op combination or feature not available */
  B200_ERR_ABORTED = -5,      /* b200_comm_abort() was called (maps to RayChannelError) */
  B200_ERR_TIMEOUT = -6,      /* a device-side wait exceeded the watchdog */
  B200_ERR_TOO_LARGE = -7     /* message does not fit the staging / inbox configuration */
} b200_status_t;

/* Element types.  Mirrors the dtypes the reference maps onto ncclDataType_t
 * (util/collective/collective_group/nccl_util.py:30-71; torch.bool travels as int8). */
typedef enum {
  B200_U8 = 0,
  B200_I8 = 1,
  B200_I32 = 2,
  B200_U32 = 3,
  B200_I64 = 4,
  B200_U64 = 5,
  B200_F16 = 6,
  B200_BF16 = 7,
  B200_F32 = 8,
  B200_F64 = 9,
  B200_DTYPE_COUNT = 10
} b200_dtype_t;

/* Reduction operators.  Numbering follows ray.util.collective.types.ReduceOp
 * (util/collective/types.py:55-59: SUM0 PRODUCT1 MIN2 MAX3); AVG is the extra
 * value the Compiled-Graph enum carries (experimental/util/types.py:11-17).  The
 * Python layer translates the cgraph numbering (MAX2 MIN3 AVG4) to this one. */
typedef enum {
  B200_SUM = 0,
  B200_PROD = 1,
  B200_MIN = 2,
  B200_MAX = 3,
  B200_AVG = 4,
  B200_OP_COUNT = 5
} b200_op_t;

/* PREMUL_SUM (ncclRedOpCreatePreMulSum / ncclRedOpDestroy): an op handle, passed as the `op` of
 * b200_allreduce, b200_allreduce_multi, b200_reduce, b200_reducescatter, b200_reducescatterv and
 * b200_reducescatter_multi, that reduces as SUM over y_r = round_T(x_r * factor): each rank scales
 * its input as it reads it, before anything reaches a peer, computing the product in double for
 * f64 and in fp32 for f32 / f16 / bf16, rounded once to T.  The result is therefore bit-identical
 * to SUM on y through the same entry and algorithm.  dtype: the one operand dtype the op may be
 * used with (f16, bf16, f32, f64; integer dtypes return B200_ERR_UNSUPPORTED).  scalar points at
 * one value of that dtype.  residence 0: *scalar is read now.  residence 1: scalar is a device
 * pointer that every kernel using the op reads when it runs, so a captured graph replays with the
 * value it holds then; keeping it alive until those kernels ran is the caller's job.  Handles lie
 * outside [0, B200_OP_COUNT); a handle used with another dtype returns B200_ERR_INVALID, and a
 * destroyed or never-created one B200_ERR_UNSUPPORTED, as any unknown op does.  Destroying an op
 * after calls were enqueued with it is allowed: they copied the factor into their arguments.  At
 * world size 1 the entries write y (one scale kernel per tensor) instead of copying. */
int b200_op_create_premul(b200_comm_t comm, const void *scalar, int dtype, int residence, int *op);
int b200_op_destroy(b200_comm_t comm, int op);

/* Algorithm selector for b200_allreduce (B200_ALGO_AUTO picks by size / dtype / op). */
typedef enum {
  B200_ALGO_AUTO = 0,
  B200_ALGO_ONESHOT = 1,  /* every rank reads all peers' staged inputs (latency path) */
  B200_ALGO_TWOSHOT = 2,  /* owner reduces its stripe from peer HBM, pushes result to all peers */
  B200_ALGO_NVLS = 3,     /* multimem.ld_reduce + multimem.st through the NVSwitch */
  B200_ALGO_LL = 4,       /* flag-in-data push, no barrier (<= 64 KiB) */
  B200_ALGO_PIPE = 5      /* chunk-pipelined roles in one launch, 16-byte aligned ordinary tensors.
                             n == 2: TMA copy-in | bulk pull of the peer's slot, reduced into the output;
                             n >= 3: TMA copy-in | NVLS or peer ld/st reduce | TMA copy-out, the slot
                             a ring of chunks */
} b200_algo_t;

typedef struct {
  size_t staging_bytes; /* per-slot staging size; two slots are allocated (0 -> default 256 MiB) */
  size_t heap_bytes;    /* symmetric user heap for zero-copy operands (0 -> none) */
  size_t inbox_bytes;   /* per-peer point-to-point inbox (0 -> default 32 MiB) */
  int enable_multicast; /* 1: try to create the NVLS multicast mapping, 0: never */
  int timeout_ms;       /* device-side watchdog for peer waits (0 -> default 600000 = 10 min) */
} b200_config_t;

/* ---- lifecycle / bootstrap ------------------------------------------------
 * Replaces NCCLGroup._get_nccl_collective_communicator + Rendezvous
 * (util/collective/collective_group/nccl_collective_group.py:36-125,414-468) and
 * _NcclGroup.__init__ (experimental/channel/nccl_group.py:29-114): instead of an
 * ncclUniqueId, every rank publishes one opaque B200_HANDLE_BYTES blob through
 * Ray's store (named actor / GCS KV / __ray_call__), then maps its peers.  */

/* Allocate this rank's symmetric memory on `device`, start the fd-passing
 * endpoint.  `cfg` may be NULL for defaults. */
int b200_comm_create(int world_size, int rank, int device, const b200_config_t *cfg,
                     b200_comm_t *out);

/* Fill `blob` (B200_HANDLE_BYTES) with this rank's bootstrap handle. */
int b200_comm_export_handle(b200_comm_t comm, void *blob);

/* `blobs` = world_size consecutive handles in rank order.  Maps every peer's
 * buffers, sets up the multicast mapping when available.  Collective: blocks
 * until all ranks called it. */
int b200_comm_connect(b200_comm_t comm, const void *blobs);

/* Replaces _NcclGroup.destroy (nccl_group.py:347-365) / NCCLGroup.destroy_group
 * (nccl_collective_group.py:161-185).  Implies abort. */
int b200_comm_destroy(b200_comm_t comm);

/* Unblocks every device-side wait of this communicator (ncclCommAbort stand-in,
 * nccl_group.py:360-364).  Sticky: later calls fail with B200_ERR_ABORTED. */
int b200_comm_abort(b200_comm_t comm);

/* 0 while healthy; B200_ERR_ABORTED / B200_ERR_TIMEOUT once a kernel gave up.
 * Reading it is only meaningful after the stream was synchronised. */
int b200_comm_status(b200_comm_t comm);

int b200_comm_rank(b200_comm_t comm);
int b200_comm_world_size(b200_comm_t comm);
/* 1 when the NVLS multicast mapping is active. */
int b200_comm_has_multicast(b200_comm_t comm);

/* Symmetric user heap: collective bump allocation (all ranks must issue the
 * same sequence).  Tensors placed here are reduced in place with no staging
 * copies.  `*out` is a device pointer valid on this rank. */
int b200_symm_alloc(b200_comm_t comm, size_t nbytes, void **out);
/* Resets the bump pointer (collective). */
int b200_symm_reset(b200_comm_t comm);
/* 1 if [ptr, ptr+nbytes) lies inside this rank's symmetric heap. */
int b200_symm_contains(b200_comm_t comm, const void *ptr, size_t nbytes);

/* torch.cuda.memory.CUDAPluggableAllocator entry points: after b200_pool_bind(comm) every
 * allocation torch routes through them comes from comm's symmetric heap, so ordinary
 * torch tensors created under `torch.cuda.use_mem_pool(...)` are zero-copy operands
 * (the counterpart of ncclMemAlloc + buffer registration).  All ranks must allocate the
 * same sequence of sizes.  Blocks are recycled through size-keyed free lists. */
int b200_pool_bind(b200_comm_t comm);
void *b200_pool_alloc(size_t size, int device, void *stream);
void b200_pool_free(void *ptr, size_t size, int device, void *stream);

/* ---- collectives ------------------------------------------------------------ */

/* out[i] = op over ranks of in[i]; in == out allowed (in place).
 * Replaces ncclAllReduce at nccl_collective_group.py:200-207 and nccl_group.py:293-312.
 * A PREMUL_SUM op runs on LL, ONESHOT, TWOSHOT and NVLS wherever SUM does, with SUM's launches;
 * B200_ALGO_PIPE returns B200_ERR_UNSUPPORTED before anything is launched.  AUTO makes SUM's choice,
 * except where SUM would take the pipelined kernels or the zero-copy symmetric-heap form, neither
 * of which reads the input into registers: there it takes the staged two-shot kernel, NVLS when
 * SUM's NVLS rule holds for the message. */
int b200_allreduce(b200_comm_t comm, const void *in, void *out, size_t count,
                   int dtype, int op, int algo, void *stream);

/* outs[p] (p < world_size) receives rank p's `in` (count elements each).
 * Writes straight into the caller's n output tensors: replaces ncclAllGather plus
 * the flat scratch buffer and n device copies at nccl_collective_group.py:283-319,
 * 685-726; with outs[p] = base + p*count*elsize it is nccl_group.py:274-291. */
int b200_allgather(b200_comm_t comm, const void *in, void *const *outs, size_t count,
                   int dtype, void *stream);

/* out = op over ranks q of (rank q's ins[this rank]).  Reads the caller's n input
 * tensors directly: replaces the n device copies + ncclReduceScatter at
 * nccl_collective_group.py:321-360 and nccl_group.py:314-333.  Takes a PREMUL_SUM op: each input
 * unit is scaled as it is pushed. */
int b200_reducescatter(b200_comm_t comm, const void *const *ins, void *out, size_t count,
                       int dtype, int op, void *stream);

/* All-gather with a size per rank.  counts: host array of world_size element counts, the same on
 * every rank.  outs[p] (counts[p] elements) receives rank p's `in` (counts[this rank] elements).
 * A zero count moves nothing, and its pointer may be NULL; if all counts are zero nothing is
 * launched.  When all counts are equal the call is exactly b200_allgather: it delegates, so it
 * makes the same launches (the pull kernel for large aligned parts included).  The only overlap
 * allowed is the in-place form, outs[this rank] == in.  World size 1: cudaMemcpyAsync when not in
 * place, no kernel.  Launches: every part is cut into windows of W = staging_bytes / 16 units of 16
 * bytes; window w covers units [w * W, (w + 1) * W) of every part, so launches = ceil(max_p U_p / W)
 * with U_p = ceil(bytes_p / 16).  Each runs b200_allgather's staged protocol on the staging slots
 * and launch counter shared by every collective, so it interleaves with them in stream order; a
 * rank whose part is exhausted or empty still makes every launch.  A count list that differs
 * between ranks breaks the contract, as mismatched send / recv sizes do; it cannot be detected
 * locally.  Refused calls (NULL arrays, a NULL pointer with a non-zero count) launch nothing and
 * return B200_ERR_INVALID; a bad dtype returns B200_ERR_UNSUPPORTED.  Replaces ProcessGroupNCCL's
 * all-gather of unequal sizes, a coalesced group of one ncclBroadcast per rank. */
int b200_allgatherv(b200_comm_t comm, const void *in, const size_t *counts, void *const *outs,
                    int dtype, void *stream);

/* Reduce-scatter with a size per rank.  counts: host array of world_size element counts, the same
 * on every rank.  ins[q] (counts[q] elements) is this rank's contribution to rank q; out
 * (counts[this rank] elements) = op over ranks of that rank's ins[this rank], rank-ascending, so
 * it is bit-identical to b200_reducescatter on equal sizes.  A zero count moves nothing, and its
 * pointer may be NULL; if all counts are zero nothing is launched.  When all counts are equal the
 * call is exactly b200_reducescatter: it delegates, so it makes the same launches.  The only
 * overlap allowed is the in-place form, out == ins[this rank].  World size 1: cudaMemcpyAsync when
 * not in place, no kernel (AVG over one rank is the identity).  Launches: the output parts are cut
 * into windows of W = floor(staging_bytes / (16 * world_size)) units, window w covering units
 * [w * W, (w + 1) * W) of every part, so launches = ceil(max_q U_q / W) with U_q = ceil(bytes_q /
 * 16); the world_size sub-slots of a window fill at most one staging slot.  Each runs on the
 * staging slots and launch counter shared by every collective, so it interleaves with them in
 * stream order.  A count list that differs between ranks breaks the contract, as mismatched send /
 * recv sizes do; it cannot be detected locally.  Refused calls (NULL arrays, a NULL pointer with a
 * non-zero count) launch nothing and return B200_ERR_INVALID; a bad dtype or op returns
 * B200_ERR_UNSUPPORTED.  Takes a PREMUL_SUM op, with the same launches.  Replaces ProcessGroupNCCL's
 * reduce-scatter of unequal sizes, a coalesced group of one ncclReduce per rank. */
int b200_reducescatterv(b200_comm_t comm, const void *const *ins, const size_t *counts, void *out,
                        int dtype, int op, void *stream);

/* In-place copy of root's buffer to every rank.  Replaces ncclBroadcast at
 * nccl_collective_group.py:257-281. */
int b200_broadcast(b200_comm_t comm, void *buf, size_t count, int dtype, int root,
                   void *stream);

/* Only root's buffer is modified.  Replaces ncclReduce at nccl_collective_group.py:231-255.
 * Takes a PREMUL_SUM op (every rank's buffer is scaled as it is staged, none is written but root's). */
int b200_reduce(b200_comm_t comm, void *buf, size_t count, int dtype, int op, int root,
                void *stream);

/* Flag-only device barrier (the reference all-reduces a 1-element array,
 * nccl_collective_group.py:211-229). */
int b200_barrier(b200_comm_t comm, void *stream);

/* Point-to-point.  Replaces ncclSend / ncclRecv at nccl_collective_group.py:362-412,
 * 641-682 and nccl_group.py:149-241.  Eager up to the inbox size. */
int b200_send(b200_comm_t comm, const void *buf, size_t nbytes, int peer, void *stream);
int b200_recv(b200_comm_t comm, void *buf, size_t nbytes, int peer, void *stream);

/* All-to-all(v).  ins[p] (send_counts[p] elements) goes to rank p; outs[p] (recv_counts[p]
 * elements) receives what rank p passed as its ins[this rank].  ins, outs, send_counts and
 * recv_counts are host arrays of world_size entries.  A zero count skips that direction of the
 * pair, and its pointer may be NULL.  Pairwise contract, as for send/recv: send_counts[q] on rank
 * p == recv_counts[p] on rank q.  No output may overlap an input (no in-place all-to-all), except
 * that outs[this rank] may be ins[this rank] itself (then there is nothing to copy).
 * One launch: every send and receive of this rank runs as a role of one grid on the
 * point-to-point rings, so it interleaves in stream order with earlier and later b200_send /
 * b200_recv on the same pairs (it does not stand in for a peer's concurrent b200_send /
 * b200_recv); the own segment is copied in the same launch.  b200_comm_set_blocks must be the same
 * on every rank; below 2 * (world_size - 1) CTAs every rank returns B200_ERR_INVALID.
 * Counterpart of ProcessGroupNCCL's alltoall_base / alltoall (ncclSend / ncclRecv in a group). */
int b200_alltoall(b200_comm_t comm, const void *const *ins, const size_t *send_counts,
                  void *const *outs, const size_t *recv_counts, int dtype, void *stream);

/* One-sided get (RDT's one-sided transport, experimental/rdt/cuda_ipc_transport.py:57-186, without
 * its same-GPU restriction): copies [src_heap_offset, +nbytes) of rank `src_rank`'s symmetric heap
 * into `dst` with a kernel that runs on THIS rank only.  The caller orders it after the owner's
 * writes (an interprocess event in the RDT transport).  b200_symm_base returns this rank's heap
 * base and size, so that an address inside it can be turned into the offset a peer passes here.  A
 * range outside the heap, or a NULL destination with a non-zero size, refuses the call before
 * anything is launched. */
int b200_symm_base(b200_comm_t comm, void **base, size_t *bytes);
int b200_get(b200_comm_t comm, void *dst, int src_rank, size_t src_heap_offset, size_t nbytes, void *stream);

/* Point-to-point transfer of a tensor LIST as one message (RDT objects, Compiled-Graph channel
 * messages).  bufs / nbytes are host arrays of ntensors entries; sizes are in BYTES, so one list
 * may mix dtypes.  Pairwise contract: the receiver passes the same sequence of sizes as the
 * sender.  A zero-size entry moves nothing, and its pointer may be NULL.  Launches: one per table
 * of at most B200_P2P_TABLE_MAX non-empty entries, in list order.  Each launch is one message on
 * the same rings and persistent sequence numbers as b200_send / b200_recv, so it interleaves with
 * them in stream order.  Wire layout: tensor i starts on a 16-byte unit of the message (units
 * ustart[i+1] = ustart[i] + ceil(nbytes[i] / 16)); padding travels but is never stored.  Each
 * side picks its own copy mechanism (ld/st or the bulk-copy unit).  Refused calls (peer out of
 * range or this rank, ntensors < 0, NULL arrays with ntensors > 0, a NULL pointer with a non-zero
 * size) launch nothing and return B200_ERR_INVALID.  Counterpart of looping ncclSend / ncclRecv
 * per tensor (collective_tensor_transport.py). */
#define B200_P2P_TABLE_MAX 256
int b200_send_multi(b200_comm_t comm, const void *const *bufs, const size_t *nbytes, int ntensors,
                    int peer, void *stream);
int b200_recv_multi(b200_comm_t comm, void *const *bufs, const size_t *nbytes, int ntensors,
                    int peer, void *stream);
/* One-sided list get: dsts[i] <- [src_heap_offsets[i], +nbytes[i]) of src_rank's heap, one launch
 * per table of at most B200_P2P_TABLE_MAX non-empty entries; nothing runs on the owner.  Any range
 * outside the heap, or a NULL destination with a non-zero size, refuses the whole call before
 * anything is launched. */
int b200_get_multi(b200_comm_t comm, void *const *dsts, int src_rank, const size_t *src_heap_offsets,
                   const size_t *nbytes, int ntensors, void *stream);

/* A batch of point-to-point operations in ONE launch (ncclGroupStart/End of sends and receives).
 * Op i sends (is_send[i] != 0) or receives nbytes[i] bytes at bufs[i] to / from rank peers[i]; the
 * arrays are host arrays of nops entries.  Wire identity: each op is exactly the message b200_send /
 * b200_recv would make for its buffer (same chunking and sub-rings, same persistent sequence
 * numbers), so it pairs with a plain b200_send / b200_recv on the peer or with an op of the peer's
 * batch, in any mix, and interleaves in stream order with every other send / recv on the pair.  It
 * does NOT pair with a b200_alltoall segment or a b200_send_multi / b200_recv_multi message, whose
 * wire differs.  Order: ops to the same (peer, direction) are consecutive messages in list order;
 * different (peer, direction) pairs progress concurrently, with no order implied between them.  So
 * a bidirectional or ring exchange of messages larger than the inbox completes in one batch, where
 * a send queued ahead of its matching receive would wait for it.  Each side picks ld/st or the
 * bulk-copy unit per op exactly as b200_send / b200_recv do.  A zero-size op moves nothing and its
 * pointer may be NULL; a batch whose ops are all empty launches nothing.  Refused calls launch
 * nothing and return B200_ERR_INVALID: nops < 0 or > B200_P2P_TABLE_MAX (a larger batch is not
 * split, since separate launches could deadlock again), NULL arrays with nops > 0, a peer out of
 * range or this rank, a NULL pointer with a non-zero size, and a grid cap (b200_comm_set_blocks)
 * below 2 * (world_size - 1) -- checked against the world size, so every rank refuses together.
 * The op table is a kernel parameter, so the call can be captured in a CUDA graph.  Counterpart of
 * ncclSend / ncclRecv between ncclGroupStart and ncclGroupEnd (c10d's batch_isend_irecv). */
int b200_p2p_batch(b200_comm_t comm, void *const *bufs, const size_t *nbytes, const int *peers,
                   const int *is_send, int nops, void *stream);

/* In-place broadcast of a tensor LIST from root: bufs[i] (nbytes[i] bytes) on every rank receives
 * root's bufs[i].  Sizes are in BYTES, so one list may mix dtypes; every rank passes the same size
 * sequence.  A zero-size entry moves nothing and its pointer may be NULL.  Layout: the packed
 * stream of b200_send_multi, tables of at most B200_P2P_TABLE_MAX non-empty entries in list order.
 * Launches: one per window of at most staging_bytes of each table's stream, i.e. the sum over
 * tables of ceil(16 * units / staging_bytes); a tensor may span windows.  Each launch runs
 * b200_broadcast's protocol on the same staging slots and launch counter, so it interleaves with
 * every other collective in stream order.  Refused calls (root out of range, ntensors < 0, NULL
 * arrays with ntensors > 0, a NULL pointer with a non-zero size) launch nothing and return
 * B200_ERR_INVALID; at world size 1, or when every entry is empty, nothing is launched.  Replaces
 * c10d's flatten + ncclBroadcast + per-tensor copy-out of DDP's buffer sync
 * (_broadcast_coalesced) and a loop of ncclBroadcast per tensor (weight sync). */
int b200_broadcast_multi(b200_comm_t comm, void *const *bufs, const size_t *nbytes, int ntensors,
                         int root, void *stream);

/* All-gather of a tensor LIST: outs has ntensors * world_size entries, and outs[i * world_size + p]
 * (nbytes[i] bytes) receives rank p's ins[i].  Sizes are in BYTES, so one list may mix dtypes; every
 * rank passes the same size sequence.  A zero-size entry moves nothing and its pointers may be NULL.
 * The only overlap allowed is c10d's in-place form, outs[i * world_size + this rank] == ins[i]; no
 * other output may overlap an input.  Layout: the packed stream of b200_send_multi over the inputs,
 * tables of at most B200_P2P_TABLE_MAX non-empty entries in list order.  Launches: one per window of
 * at most staging_bytes of each table's stream, i.e. the sum over tables of
 * ceil(16 * units / staging_bytes), a function of the size list and staging_bytes alone.  Each launch
 * runs b200_allgather's staged protocol on the same staging slots and launch counter, so it
 * interleaves with every other collective in stream order.  Refused calls (ntensors < 0, NULL arrays
 * with ntensors > 0, a NULL pointer with a non-zero size) launch nothing and return
 * B200_ERR_INVALID.  At world size 1 every entry that is not in place is copied with
 * cudaMemcpyAsync; a list that is empty, or whose entries are all empty, launches nothing.  Replaces
 * one ncclAllGather per tensor of c10d's coalesced all-gather (allgather_into_tensor_coalesced,
 * allgather_coalesced). */
int b200_allgather_multi(b200_comm_t comm, const void *const *ins, const size_t *nbytes, int ntensors,
                         void *const *outs, void *stream);

/* Reduce-scatter of a tensor LIST: ins has ntensors * world_size entries, and ins[i * world_size + q]
 * (counts[i] elements) is this rank's contribution to rank q's outs[i]; outs[i] = op over ranks of
 * (that rank's ins[i * world_size + this rank]), reduced rank-ascending.  One dtype and one op per
 * call; every rank passes the same count sequence.  The result is bit-identical to b200_reducescatter
 * run on each tensor alone.  A zero-count entry moves nothing and its pointers may be NULL.  The only
 * overlap allowed is c10d's in-place form, outs[i] == ins[i * world_size + this rank].  Launches:
 * outputs are packed as in b200_allgather_multi, and each table's stream of output units is cut into
 * windows of at most floor(staging_bytes / (16 * world_size)) units (the world_size sub-slots of a
 * window fill one staging slot), one launch each, on the same staging slots and launch counter as
 * every other collective.  Refused calls (ntensors < 0, NULL arrays with ntensors > 0, a NULL pointer
 * with a non-zero count) launch nothing and return B200_ERR_INVALID; a bad dtype or op returns
 * B200_ERR_UNSUPPORTED as in b200_reducescatter.  At world size 1 every entry that is not in place is
 * copied with cudaMemcpyAsync (AVG over one rank is the identity).  Takes a PREMUL_SUM op, with the
 * same launches.  Replaces one ncclReduceScatter per tensor of c10d's coalesced reduce-scatter
 * (reduce_scatter_tensor_coalesced). */
int b200_reducescatter_multi(b200_comm_t comm, const void *const *ins, void *const *outs,
                             const size_t *counts, int ntensors, int dtype, int op, void *stream);

/* Fused data-parallel gradient synchronisation (SURVEY K8): for a flat fp32
 * bucket computes grad[i] = sum_r wire(grad_r[i] * scale) in one launch, where
 * wire() is a cast to `wire_dtype` (B200_BF16 / B200_F16 compress the NVLink
 * traffic; B200_F32 keeps DDP's exact arithmetic).  Replaces the c10d reducer's
 * div + ncclAllReduce (+ bf16_compress_hook casts) reached from
 * train/torch/config.py:144 and train/torch/train_loop_utils.py:456-480. */
int b200_grad_allreduce(b200_comm_t comm, float *grad, size_t count, float scale,
                        int wire_dtype, void *stream);

/* Fused sharded gradient synchronisation (FSDP / ZeRO counterpart of b200_grad_allreduce):
 * grad holds world_size * count fp32 elements (rank q's stripe at grad + q * count); out (count
 * elements) receives sum_r wire(grad_r[this rank's stripe] * scale), cast back to fp32 -- bit for
 * bit this rank's stripe of what b200_grad_allreduce leaves in the bucket on the peer path.  One
 * launch per piece of at most staging_bytes / world_size bytes of wire data per rank.  out may be
 * this rank's own stripe (grad + rank * count) but must not overlap grad otherwise.  Replaces
 * FSDP's div + fp32 ncclReduceScatter + div (and its compress-hook casts). */
int b200_grad_reducescatter(b200_comm_t comm, const float *grad, float *out, size_t count,
                            float scale, int wire_dtype, void *stream);

/* Multi-tensor all-reduce (SURVEY K9): reduces `ntensors` same-dtype tensors as one
 * message without a host-side flatten (replaces parameters_to_vector + views at
 * dag/collective_node.py:220-232).  ptrs/counts are host arrays.  Takes a PREMUL_SUM op: the
 * table kernel scales as it gathers, and tensors it does not take go through b200_allreduce. */
int b200_allreduce_multi(b200_comm_t comm, void *const *ptrs, const size_t *counts,
                         int ntensors, int dtype, int op, void *stream);

/* ---- introspection ---------------------------------------------------------- */
const char *b200_last_error(void);
const char *b200_version(void);
size_t b200_dtype_size(int dtype);
/* Number of device kernels this library launched on behalf of `comm` so far. */
uint64_t b200_comm_launch_count(b200_comm_t comm);
/* Tuning knob: force the CTA count used by collectives (0 = automatic). */
int b200_comm_set_blocks(b200_comm_t comm, int nblocks);

/* In-kernel event trace (profiling aid, off by default): allocates room for `capacity` events
 * (0 frees it); instrumented kernels then record (globaltimer ns, CTA, event id, argument).
 * b200_comm_trace_read synchronises the device, copies up to max_events events (2 x u64 each:
 * ns, blockIdx << 40 | event << 32 | argument) and returns how many; `reset` != 0 clears it. */
int b200_comm_trace_enable(b200_comm_t comm, unsigned int capacity);
int b200_comm_trace_read(b200_comm_t comm, unsigned long long *out, unsigned int max_events, int reset);

/* Host-side self-test (no GPU needed) of the work decomposition of the pipelined kernels: runs the
 * very inline functions the kernels use and checks that copy shares tile the message, that the
 * expected arrival counts match, that reduce work items tile every chunk exactly once and that
 * ring positions are respected.  0 = consistent; otherwise b200_last_error() says what broke. */
int b200_selftest_pipe_geometry(size_t nbytes, size_t chunk_bytes, int copy_ctas, int world, int red_ctas,
                                unsigned ring_chunks);

/* Tuning parameters (must be set identically on every rank; -1 restores the default). */
typedef enum {
  B200_PARAM_ONESHOT_MAX_BYTES = 0, /* all-reduce messages up to this size use the one-shot kernel */
  B200_PARAM_NVLS_MIN_WORLD = 1,    /* AUTO uses the NVLS kernels from this world size on (default 3) */
  B200_PARAM_NVLS_CTAS = 2,         /* CTAs of the NVSwitch reduce phase: zero-copy default 64, staged default all */
  B200_PARAM_LL_MAX_BYTES = 3,      /* all-reduce messages up to this size use the LL kernel (default 32 KiB / 2 ranks ... 4 KiB / 8 ranks) */
  B200_PARAM_PIPE_MIN_BYTES = 4,    /* AUTO uses the pipelined kernels from this size on (ordinary, 16-byte aligned tensors) */
  B200_PARAM_PIPE_CHUNK_BYTES = 5,  /* pipeline chunk size (all-reduce default 1 MiB at 2 ranks, 4 MiB at 3-4, 8 MiB at 5-8; rounded up to 1 MiB multiples) */
  B200_PARAM_PIPE_COPY_CTAS = 6,    /* CTAs per TMA copy role (power of two; all-reduce default 32 at 2 ranks, 16 otherwise; pull all-gather 16) */
  B200_PARAM_PIPE_RED_CTAS = 7,     /* CTAs of the reduce / pull role (all-reduce default 32 at 2 ranks, 64 at 3-4, 32 at 5-8; pull all-gather 64, 48, 32) */
  B200_PARAM_P2P_BULK_MIN_CHUNK = 8, /* send/recv: chunks from this size on move with the TMA bulk-copy kernel (0 = never; default 32 KiB) */
  B200_PARAM_AG_PULL_MIN_BYTES = 9, /* all-gather: per-rank size from which the pull kernel is used (0 = never; default 4 MiB) */
  B200_PARAM_COUNT = 10
} b200_param_t;
int b200_comm_set_param(b200_comm_t comm, int param, long long value);

#ifdef __cplusplus
}
#endif
#endif /* B200_COLLECTIVE_H_ */
