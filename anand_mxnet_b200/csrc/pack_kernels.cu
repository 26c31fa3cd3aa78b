// pack_kernels.cu -- TMA-staged packing: copy MANY arrays (gradient tensors of 12 B .. 94 MB) into /
// out of fusion (staging) buffers in ONE launch, with the bulk-copy engine instead of 157
// cudaMemcpyAsync calls.
//
// Every array is cut (on the host, once per prepared launch) into tiles of <= 16 KB. A CTA walks
// its tiles with a 4-stage shared-memory ring driven by ONE elected thread:
//     cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes   (global -> smem, TMA)
//     mbarrier.try_wait                                                     (tile landed)
//     cp.async.bulk.global.shared::cta.bulk_group                           (smem -> global, TMA)
// so no data ever passes through registers (SASS: UBLKCP). Bulk copies need 16-byte aligned
// addresses and sizes; the sub-16-byte tail of a tile (and tiles whose ends are unaligned) are
// moved by the other threads with plain byte loads. Copy-only, HBM-bound: 2 bytes of traffic per
// byte packed.
#include <cstdio>

#include "common.h"
#include "kernels.h"

namespace b200kv {
namespace {

constexpr int kStages = 4;
constexpr int kPackThreads = 128;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_store(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_wait_read_all() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void tma_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// bytes of `it` that the bulk engine can move: both ends 16-byte aligned, size multiple of 16
__device__ __forceinline__ uint32_t bulk_bytes(const PackItem& it) {
  const bool ok = ((reinterpret_cast<uintptr_t>(it.src) | reinterpret_cast<uintptr_t>(it.dst)) & 15) == 0;
  return ok ? static_cast<uint32_t>(it.bytes & ~static_cast<uint64_t>(15)) : 0u;
}

__global__ void __launch_bounds__(kPackThreads) pack_bulk_kernel(const PackItem* items, int n_items) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t bars[kStages];
  unsigned char* ring = smem;
  constexpr uint32_t kTile = kPackTileBytes;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) mbar_init(&bars[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // ---- the bulk path: one thread drives the TMA ring over this CTA's tiles
    constexpr int kAhead = kStages - 1;
    int issued = 0, stored = 0;
    uint32_t phase_bits = 0;  // parity per stage
    auto tile_at = [&](int j) { return blockIdx.x + j * gridDim.x; };
    auto drain_one = [&]() {
      const int t = tile_at(stored);
      const int s = stored % kStages;
      const PackItem it = items[t];
      const uint32_t nb = bulk_bytes(it);
      if (nb) {
        mbar_wait(&bars[s], (phase_bits >> s) & 1u);
        phase_bits ^= (1u << s);
        tma_store(it.dst, ring + s * kTile, nb);
      }
      tma_commit();
      ++stored;
    };
    for (int j = 0; tile_at(j) < n_items; ++j) {
      const int s = j % kStages;
      if (j >= kStages) tma_wait_read_all();  // the store that last used this stage has read it
      const PackItem it = items[tile_at(j)];
      const uint32_t nb = bulk_bytes(it);
      if (nb) {
        mbar_expect_tx(&bars[s], nb);
        tma_load(ring + s * kTile, it.src, nb, &bars[s]);
      }
      ++issued;
      if (issued - stored > kAhead) drain_one();
    }
    while (stored < issued) drain_one();
    tma_wait_all();
  } else {
    // ---- tails and unaligned tiles: plain byte copies by the other threads
    for (int t = blockIdx.x; t < n_items; t += gridDim.x) {
      const PackItem it = items[t];
      const uint32_t nb = bulk_bytes(it);
      const unsigned char* s = static_cast<const unsigned char*>(it.src);
      unsigned char* d = static_cast<unsigned char*>(it.dst);
      for (uint64_t b = nb + (threadIdx.x - 1); b < it.bytes; b += kPackThreads - 1) d[b] = s[b];
    }
  }
}

// Register-path variant for lists with a pinned-HOST side: the SMs issue the PCIe reads / writes
// themselves (16-byte accesses, four per thread in flight), exactly what the fused kernel does when
// it reads gradients from host memory: with both PCIe directions busy, SM-issued loads / stores
// keep more of the link busy than bulk-copy (TMA) transfers do.
constexpr int kLdstThreads = 256;
__global__ void __launch_bounds__(kLdstThreads) pack_ldst_kernel(const PackItem* items, int n_items) {
  for (int t = blockIdx.x; t < n_items; t += gridDim.x) {
    const PackItem it = items[t];
    const uint32_t nb = bulk_bytes(it);           // 16-byte aligned prefix
    const uint4* s = static_cast<const uint4*>(it.src);
    uint4* d = static_cast<uint4*>(it.dst);
    const uint32_t nvec = nb / 16;
    for (uint32_t v0 = threadIdx.x; v0 < nvec; v0 += 4 * kLdstThreads) {
      uint4 x[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t v = v0 + u * kLdstThreads;
        if (v < nvec) x[u] = __ldcs(s + v);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t v = v0 + u * kLdstThreads;
        if (v < nvec) __stcs(d + v, x[u]);
      }
    }
    const unsigned char* sb = static_cast<const unsigned char*>(it.src);
    unsigned char* db = static_cast<unsigned char*>(it.dst);
    for (uint64_t b = nb + threadIdx.x; b < it.bytes; b += kLdstThreads) db[b] = sb[b];
  }
}

}  // namespace

void LaunchPackBulk(const PackItem* d_items, int n_items, cudaStream_t stream, bool host_io) {
  if (n_items <= 0) return;
  if (host_io) {
    constexpr int kHostCtas = 96;
    const int grid = n_items < kHostCtas ? n_items : kHostCtas;
    pack_ldst_kernel<<<grid, kLdstThreads, 0, stream>>>(d_items, n_items);
    KV_CUDA(cudaGetLastError());
    return;
  }
  const int smem = kStages * kPackTileBytes;
  // per-device attribute: set on every launch (cheap) so multi-GPU processes are covered
  KV_CUDA(cudaFuncSetAttribute(pack_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  // 3 CTAs of 64 KB fit an SM; enough CTAs to cover all 132 SMs, each looping over its tiles
  const int cap = kNumSMs * 3;
  const int grid = n_items < cap ? n_items : cap;
  pack_bulk_kernel<<<grid, kPackThreads, smem, stream>>>(d_items, n_items);
  KV_CUDA(cudaGetLastError());
}

}  // namespace b200kv
