// bulk_bench.cu — per-SM throughput of cp.async.bulk copies (local HBM and peer over NVLink).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/bulk_bench scripts/bulk_bench.cu
//   scripts/bulk_bench            (runs the whole matrix; needs 1 GPU, uses a 2nd one if present)
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <stdint.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void *dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// mode 0: copy (load+store), 1: loads only, 2: stores only.  LANES issuing threads per CTA (warp w,
// lane 0), each with its own ring of STAGES tiles.
template <int STAGES, int LA, int LANES, int LAG = -1>
__global__ void __launch_bounds__(512, 1) bench_kernel(const char *src, char *dst, size_t bytes_per_lane, uint32_t tile, int mode) {
  extern __shared__ __align__(128) char smem[];
  const int lane_id = threadIdx.x / 32;
  if ((threadIdx.x & 31) != 0 || lane_id >= LANES) return;
  const uint32_t ring = smem_u32(smem) + lane_id * (STAGES * tile);
  const uint32_t bars = smem_u32(smem) + LANES * STAGES * tile + lane_id * STAGES * 8;
  for (int s = 0; s < STAGES; ++s) mbar_init(bars + 8 * s, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  const size_t base = (size_t(blockIdx.x) * LANES + lane_id) * bytes_per_lane;
  const uint32_t nt = uint32_t(bytes_per_lane / tile);
  constexpr int RP = STAGES - LA - 1;
  uint32_t li = 0, sj = 0;
  while (sj < nt) {
    while (li < nt && li - sj < LA) {
      const int s = li % STAGES;
      if (mode != 2) {
        mbar_expect_tx(bars + 8 * s, tile);
        bulk_g2s(ring + s * tile, src + base + size_t(li) * tile, tile, bars + 8 * s);
      }
      ++li;
    }
    const int s = sj % STAGES;
    if (mode != 2) {
      while (!mbar_try_wait(bars + 8 * s, (sj / STAGES) & 1)) {}
    }
    if (mode != 1) {
      bulk_s2g(dst + base + size_t(sj) * tile, ring + s * tile, tile);
      bulk_commit();
      bulk_wait_read<RP>();
      if (LAG >= 0 && sj >= LAG) bulk_wait<(LAG >= 0 ? LAG : 0)>();
    }
    ++sj;
  }
  bulk_wait<0>();
}

__global__ void ldst_kernel(const uint4 *src, uint4 *dst, size_t units) {
  const size_t stride = size_t(gridDim.x) * blockDim.x * 8;
  for (size_t u0 = size_t(blockIdx.x) * blockDim.x * 8 + threadIdx.x; u0 < units; u0 += stride) {
    uint4 v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) if (u0 + k * blockDim.x < units) v[k] = src[u0 + k * blockDim.x];
#pragma unroll
    for (int k = 0; k < 8; ++k) if (u0 + k * blockDim.x < units) dst[u0 + k * blockDim.x] = v[k];
  }
}

template <int STAGES, int LA, int LANES, int LAG = -1>
static void run(const char *name, const char *src, char *dst, int ctas, uint32_t tile, int mode, size_t total) {
  const size_t smem = size_t(LANES) * STAGES * tile + LANES * STAGES * 8 + 128;
  if (smem > 227 * 1024) return;
  auto k = bench_kernel<STAGES, LA, LANES, LAG>;
  CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  size_t per_lane = total / (size_t(ctas) * LANES) / tile * tile;
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  float best = 1e9;
  for (int rep = 0; rep < 4; ++rep) {
    CK(cudaEventRecord(a));
    k<<<ctas, 512, smem>>>(src, dst, per_lane, tile, mode);
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    float ms; CK(cudaEventElapsedTime(&ms, a, b));
    if (rep && ms < best) best = ms;
  }
  const double gb = double(per_lane) * ctas * LANES / 1e9;
  printf("%-8s mode=%d ctas=%3d lanes=%d tile=%3uK stages=%2d la=%d lag=%2d : %8.1f us  %7.1f GB/s  (%.1f GB/s per CTA)\n", name, mode, ctas, LANES,
         tile >> 10, STAGES, LA, LAG, best * 1e3, gb / (best * 1e-3), gb / (best * 1e-3) / ctas);
  fflush(stdout);
}

int main() {
  int ndev = 0;
  CK(cudaGetDeviceCount(&ndev));
  const size_t total = size_t(512) << 20;
  char *src, *dst, *rdst = nullptr;
  CK(cudaSetDevice(0));
  CK(cudaMalloc(&src, total)); CK(cudaMalloc(&dst, total));
  CK(cudaMemset(src, 1, total));
  if (ndev > 1) {
    int can = 0; CK(cudaDeviceCanAccessPeer(&can, 0, 1));
    if (can) {
      CK(cudaSetDevice(1)); CK(cudaMalloc(&rdst, total)); CK(cudaSetDevice(0));
      CK(cudaDeviceEnablePeerAccess(1, 0));
    }
  }
  for (int remote = 0; remote < (rdst ? 2 : 1); ++remote) {
    char *d = remote ? rdst : dst;
    const char *nm = remote ? "remote" : "local";
    for (int ctas : {1, 16}) {
      run<6, 3, 1>(nm, src, d, ctas, 32 << 10, 0, total);
      run<6, 3, 1, 2>(nm, src, d, ctas, 32 << 10, 0, total);
      run<6, 3, 1, 3>(nm, src, d, ctas, 32 << 10, 0, total);
      run<6, 3, 1, 4>(nm, src, d, ctas, 32 << 10, 0, total);
      run<6, 3, 1, 6>(nm, src, d, ctas, 32 << 10, 0, total);
      run<6, 3, 1, 8>(nm, src, d, ctas, 32 << 10, 0, total);
      run<6, 3, 1, 12>(nm, src, d, ctas, 32 << 10, 0, total);
      run<6, 3, 1, 16>(nm, src, d, ctas, 32 << 10, 0, total);
      run<6, 3, 1, 24>(nm, src, d, ctas, 32 << 10, 0, total);
      run<6, 4, 1>(nm, src, d, ctas, 32 << 10, 0, total);
      run<6, 4, 1, 12>(nm, src, d, ctas, 32 << 10, 0, total);
      run<12, 6, 1, 12>(nm, src, d, ctas, 16 << 10, 0, total);
      run<12, 6, 1, 24>(nm, src, d, ctas, 16 << 10, 0, total);
    }
  }
  return 0;
}
