// kernel_utils.cuh — copy/stage helpers, argument checks and launch plumbing shared by the
// collective kernels.  Launch decisions live in policy.h.
#pragma once
#include "comm.h"

namespace b200 {

// A message of `nbytes` is processed in 16-byte units.  `full` units are complete,
// a trailing partial unit (tail bytes) is staged zero-padded.
struct Units {
  size_t full;   // number of complete 16-byte units
  int tail;      // bytes in the trailing partial unit (0..15)
  __host__ __device__ size_t total() const { return full + (tail ? 1 : 0); }
};
__host__ __device__ inline Units make_units(size_t nbytes) {
  Units u;
  u.full = nbytes >> 4;
  u.tail = int(nbytes & 15);
  return u;
}

// Load unit `u` of a user tensor (arbitrary alignment handled by the slow path).
__device__ __forceinline__ uint4 load_user_unit(const char *src, size_t u, const Units &un, bool aligned) {
  if (u < un.full) {
    if (aligned) return ld_stream(src + (u << 4));
    uint4 v;
    unsigned char *b = reinterpret_cast<unsigned char *>(&v);
#pragma unroll
    for (int i = 0; i < 16; ++i) b[i] = reinterpret_cast<const unsigned char *>(src)[(u << 4) + i];
    return v;
  }
  uint4 v = make_uint4(0, 0, 0, 0);
  unsigned char *b = reinterpret_cast<unsigned char *>(&v);
  for (int i = 0; i < un.tail; ++i) b[i] = reinterpret_cast<const unsigned char *>(src)[(u << 4) + i];
  return v;
}

__device__ __forceinline__ void store_user_unit(char *dst, size_t u, const Units &un, bool aligned, uint4 v) {
  if (u < un.full) {
    if (aligned) {
      st_vec(dst + (u << 4), v);
      return;
    }
    const unsigned char *b = reinterpret_cast<const unsigned char *>(&v);
#pragma unroll
    for (int i = 0; i < 16; ++i) reinterpret_cast<unsigned char *>(dst)[(u << 4) + i] = b[i];
    return;
  }
  const unsigned char *b = reinterpret_cast<const unsigned char *>(&v);
  for (int i = 0; i < un.tail; ++i) reinterpret_cast<unsigned char *>(dst)[(u << 4) + i] = b[i];
}

__host__ __device__ inline bool is_aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Offset of the staging slot used by the current launch (two slots alternate so a
// rank may start staging the next message while a slow peer still reads the previous
// one; see DESIGN.md "slot rotation").
__device__ __forceinline__ size_t staging_slot_offset(uint32_t launch, size_t staging_bytes) {
  return (launch & 1u) ? staging_bytes : 0;
}

// Argument checks of the entry points: each sets the error text and returns its status, or
// B200_OK, so they chain as `if ((rc = check_a(..)) || (rc = check_b(..))) return rc;`.
inline int check_dtype(int dtype, size_t *es) {
  *es = b200_dtype_size(dtype);
  if (*es == 0) {
    set_error("unsupported dtype %d", dtype);
    return B200_ERR_UNSUPPORTED;
  }
  return B200_OK;
}

inline int check_op(int op) {
  if (op < 0 || op >= B200_OP_COUNT) {
    set_error("unsupported reduce op %d", op);
    return B200_ERR_UNSUPPORTED;
  }
  return B200_OK;
}

// Handles of b200_op_create_premul lie outside [0, B200_OP_COUNT).
constexpr int kPremulOpBase = 0x100;

// The op argument of a reducing entry: a b200_op_t value, or a live PREMUL_SUM handle, which must be
// used with the dtype it was created for.  A handle resolves to kOpPremulSum and its factor.
struct OpArg {
  int op;
  PremulArg premul;
};
inline int check_op(const b200_comm *c, int op, int dtype, OpArg *out) {
  out->op = op;
  out->premul = PremulArg{0.0, nullptr};
  if (op >= 0 && op < B200_OP_COUNT) return B200_OK;
  const int slot = op - kPremulOpBase;
  const int nslots = int(sizeof(c->premul_ops) / sizeof(c->premul_ops[0]));
  if (slot < 0 || slot >= nslots || c->premul_ops[slot].dtype < 0) return check_op(op);
  if (c->premul_ops[slot].dtype != dtype) {
    set_error("PREMUL_SUM op %d was created for dtype %d, used with dtype %d", op, c->premul_ops[slot].dtype, dtype);
    return B200_ERR_INVALID;
  }
  out->op = kOpPremulSum;
  out->premul = c->premul_ops[slot].arg;
  return B200_OK;
}

// World size 1 of a PREMUL_SUM entry: out = round_T(in * factor), in place or not, any alignment
// (allreduce.cu).  One launch.
int launch_premul_scale(b200_comm *c, const void *in, void *out, size_t nbytes, int dtype, const PremulArg &f,
                        cudaStream_t stream);

// `what`: "root", "peer" or "source"
inline int check_rank(const b200_comm *c, int r, const char *what) {
  if (r < 0 || r >= c->world) {
    set_error("%s rank %d out of range for world size %d", what, r, c->world);
    return B200_ERR_INVALID;
  }
  return B200_OK;
}

inline int null_tensor_error() {
  set_error("null tensor pointer");
  return B200_ERR_INVALID;
}

// Runs fn(done, n) -> status over [0, total) in pieces of at most `step` bytes (or elements),
// in order; stops at the first failing piece.
template <typename Fn>
inline int for_each_piece(size_t total, size_t step, Fn fn) {
  for (size_t done = 0; done < total;) {
    const size_t n = (total - done) < step ? (total - done) : step;
    if (int rc = fn(done, n)) return rc;
    done += n;
  }
  return B200_OK;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize = bulk-copy ring, once per (device, kernel)
int set_dyn_smem(int device, const void *fn);

#define B200_LAUNCH_CHECK(c)                                                     \
  do {                                                                           \
    cudaError_t _e = cudaGetLastError();                                         \
    if (_e != cudaSuccess) {                                                     \
      b200::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), \
                      __FILE__, __LINE__);                                       \
      return B200_ERR_CUDA;                                                      \
    }                                                                            \
    (c)->launches.fetch_add(1);                                                  \
  } while (0)

// Dispatch helpers ---------------------------------------------------------------
#define B200_DISPATCH_DTYPE(dtype, T, ...)                                   \
  switch (dtype) {                                                           \
    case B200_U8: { using T = uint8_t; __VA_ARGS__; break; }                 \
    case B200_I8: { using T = int8_t; __VA_ARGS__; break; }                  \
    case B200_I32: { using T = int32_t; __VA_ARGS__; break; }                \
    case B200_U32: { using T = uint32_t; __VA_ARGS__; break; }               \
    case B200_I64: { using T = int64_t; __VA_ARGS__; break; }                \
    case B200_U64: { using T = uint64_t; __VA_ARGS__; break; }               \
    case B200_F16: { using T = __half; __VA_ARGS__; break; }                 \
    case B200_BF16: { using T = __nv_bfloat16; __VA_ARGS__; break; }         \
    case B200_F32: { using T = float; __VA_ARGS__; break; }                  \
    case B200_F64: { using T = double; __VA_ARGS__; break; }                 \
    default: b200::set_error("unsupported dtype %d", int(dtype)); return B200_ERR_UNSUPPORTED; \
  }

#define B200_DISPATCH_OP(op, OP, ...)                                        \
  switch (op) {                                                              \
    case B200_SUM: { constexpr int OP = B200_SUM; __VA_ARGS__; break; }      \
    case B200_PROD: { constexpr int OP = B200_PROD; __VA_ARGS__; break; }    \
    case B200_MIN: { constexpr int OP = B200_MIN; __VA_ARGS__; break; }      \
    case B200_MAX: { constexpr int OP = B200_MAX; __VA_ARGS__; break; }      \
    case B200_AVG: { constexpr int OP = B200_AVG; __VA_ARGS__; break; }      \
    default: b200::set_error("unsupported reduce op %d", int(op)); return B200_ERR_UNSUPPORTED; \
  }

// The dtypes a PREMUL_SUM op exists for (b200_op_create_premul refuses the others).  Its kernels are
// separate instantiations with OP = kOpPremulSum and a PremulArg argument, so B200_DISPATCH_OP keeps
// instantiating exactly the plain ops' kernels.
#define B200_DISPATCH_PREMUL(dtype, T, ...)                                  \
  switch (dtype) {                                                           \
    case B200_F16: { using T = __half; __VA_ARGS__; break; }                 \
    case B200_BF16: { using T = __nv_bfloat16; __VA_ARGS__; break; }         \
    case B200_F32: { using T = float; __VA_ARGS__; break; }                  \
    case B200_F64: { using T = double; __VA_ARGS__; break; }                 \
    default: b200::set_error("PREMUL_SUM supports f16, bf16, f32 and f64 only"); return B200_ERR_UNSUPPORTED; \
  }

}  // namespace b200
