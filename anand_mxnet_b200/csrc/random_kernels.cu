// random_kernels.cu -- the reference's GPU normal sampler (kernels.h, LaunchRandSeed / LaunchRandNormal).
//
// The stream is fixed by the reference: curandStatePhilox4_32_10_t states seeded with
// curand_init(seed, id, 0) (common/random_generator.cu), and LaunchRNG's mapping (random/sampler.h):
// nthread = min(ceil(N / 64), 32768), step = ceil(N / nthread), thread t draws elements
// [t*step, min((t+1)*step, N)) in order from state t, which it holds in registers and writes back
// whole, curand's cached Box-Muller value included. Element i is
// OType(normal() * scale + loc) with contraction on: one fmaf (float, half, bfloat16: the float
// normal rounded once) or one fma in double (curand_normal_double). This file is compiled with
// -fmad=true like the reference's GPU build, so curand's own Box-Muller arithmetic contracts as it
// does there (build.py).
//
// The store order is free. A thread owns a contiguous run, so storing as it draws puts the 32 lanes
// of a warp step*sizeof(T) bytes apart. The staged kernel instead has each lane draw 128 B of its
// run into a per-warp shared tile, then the warp writes each lane's 128 B as 8 lanes x 16 B (4 runs
// per store instruction) when out and step allow 16-B vectors, else lane-contiguous scalars.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <curand_kernel.h>

#include <algorithm>

#include "common.h"
#include "kernels.h"

namespace b200kv {

static_assert(sizeof(curandStatePhilox4_32_10_t) == kRandStateBytes, "a state is persisted whole");

namespace {

constexpr int kSeedThreads = 256;   // the reference's kBaseThreadNum
constexpr int kNormalThreads = 64;  // 2 warps: 512 CTAs for 32768 states spread over all 132 SMs

__global__ void __launch_bounds__(kSeedThreads) rand_seed_kernel(curandStatePhilox4_32_10_t* states,
                                                                  uint32_t seed) {
  const int id = blockIdx.x * kSeedThreads + threadIdx.x;
  if (id < kRandStates) curand_init(seed, id, 0, states + id);
}

// RandGenerator<gpu, T>::Impl::normal() * scale + loc, as T
template <typename T>
struct Draw;
template <>
struct Draw<float> {
  static __device__ __forceinline__ float Get(curandStatePhilox4_32_10_t* s, float loc, float scale) {
    return __fmaf_rn(curand_normal(s), scale, loc);
  }
};
template <>
struct Draw<double> {
  static __device__ __forceinline__ double Get(curandStatePhilox4_32_10_t* s, float loc, float scale) {
    return __fma_rn(curand_normal_double(s), static_cast<double>(scale), static_cast<double>(loc));
  }
};
template <>
struct Draw<__half> {
  static __device__ __forceinline__ __half Get(curandStatePhilox4_32_10_t* s, float loc, float scale) {
    return __float2half_rn(__fmaf_rn(curand_normal(s), scale, loc));
  }
};
template <>
struct Draw<__nv_bfloat16> {
  static __device__ __forceinline__ __nv_bfloat16 Get(curandStatePhilox4_32_10_t* s, float loc, float scale) {
    return __float2bfloat16_rn(__fmaf_rn(curand_normal(s), scale, loc));
  }
};

// kStaged = false: each thread stores as it draws (the reference's order; kept for bench_random.py)
template <typename T, bool kStaged>
__global__ void __launch_bounds__(kNormalThreads)
    normal_kernel(curandStatePhilox4_32_10_t* states, T* __restrict__ out, uint64_t n, uint64_t step,
                  uint32_t nthread, float loc, float scale, uint32_t vec) {
  constexpr int kRun = 128 / sizeof(T);         // elements a lane draws per round
  constexpr int kPerVec = 16 / sizeof(T);
  constexpr int kPad = sizeof(T) >= 4 ? 1 : 4 / sizeof(T);  // tile rows 4 B apart in banks
  const uint32_t t = blockIdx.x * kNormalThreads + threadIdx.x;
  const uint64_t start = static_cast<uint64_t>(t) * step;
  const uint64_t len = t < nthread && start < n ? (n - start < step ? n - start : step) : 0;
  curandStatePhilox4_32_10_t st;
  if (len > 0) st = states[t];
  if constexpr (!kStaged) {
    for (uint64_t i = 0; i < len; ++i) out[start + i] = Draw<T>::Get(&st, loc, scale);
  } else {
    __shared__ T smem[kNormalThreads / 32][32][kRun + kPad];
    T(*tile)[kRun + kPad] = smem[threadIdx.x / 32];
    const int lane = threadIdx.x & 31;
    const uint64_t warp_t0 = t - lane;
    for (uint64_t r = 0; __any_sync(~0u, r < len); r += kRun) {
      const int cnt = r < len ? static_cast<int>(len - r < kRun ? len - r : kRun) : 0;
      for (int k = 0; k < cnt; ++k) tile[lane][k] = Draw<T>::Get(&st, loc, scale);
      __syncwarp();
      if (vec) {
        // every run starts 16-B aligned (out aligned, step % kPerVec == 0, r % kRun == 0)
        constexpr int kLanesPerRun = kRun / kPerVec;  // 8
        const int j = lane % kLanesPerRun;
#pragma unroll 1
        for (int sb = 0; sb < 32; sb += 32 / kLanesPerRun) {
          const int s = sb + lane / kLanesPerRun;
          const int cs = __shfl_sync(~0u, cnt, s);
          T* dst = out + (warp_t0 + s) * step + r + j * kPerVec;
          if ((j + 1) * kPerVec <= cs) {
            uint4 v;
            T* e = reinterpret_cast<T*>(&v);
#pragma unroll
            for (int q = 0; q < kPerVec; ++q) e[q] = tile[s][j * kPerVec + q];
            *reinterpret_cast<uint4*>(dst) = v;
          } else {
            for (int q = 0; j * kPerVec + q < cs; ++q) dst[q] = tile[s][j * kPerVec + q];
          }
        }
      } else {
#pragma unroll 1
        for (int s = 0; s < 32; ++s) {
          const int cs = __shfl_sync(~0u, cnt, s);
          T* dst = out + (warp_t0 + s) * step + r;
          for (int k = lane; k < cs; k += 32) dst[k] = tile[s][k];
        }
      }
      __syncwarp();
    }
  }
  if (len > 0) states[t] = st;
}

template <typename T>
void Launch(void* states, void* out, uint64_t n, float loc, float scale, bool staged, cudaStream_t st) {
  const uint64_t nloop = (n + kRandMinPerThread - 1) / kRandMinPerThread;
  const uint64_t nthread = std::min<uint64_t>(nloop, kRandStates);
  const uint64_t step = (n + nthread - 1) / nthread;
  const unsigned blocks = static_cast<unsigned>((nthread + kNormalThreads - 1) / kNormalThreads);
  auto* s = static_cast<curandStatePhilox4_32_10_t*>(states);
  T* o = static_cast<T*>(out);
  const uint32_t vec = (reinterpret_cast<uintptr_t>(out) & 15) == 0 && step % (16 / sizeof(T)) == 0;
  if (staged) {
    normal_kernel<T, true><<<blocks, kNormalThreads, 0, st>>>(s, o, n, step, static_cast<uint32_t>(nthread),
                                                              loc, scale, vec);
  } else {
    normal_kernel<T, false><<<blocks, kNormalThreads, 0, st>>>(s, o, n, step, static_cast<uint32_t>(nthread),
                                                               loc, scale, vec);
  }
}

}  // namespace

void LaunchRandSeed(void* states, uint32_t seed, cudaStream_t st) {
  rand_seed_kernel<<<(kRandStates + kSeedThreads - 1) / kSeedThreads, kSeedThreads, 0, st>>>(
      static_cast<curandStatePhilox4_32_10_t*>(states), seed);
  KV_CUDA(cudaGetLastError());
}

void LaunchRandNormal(int dtype, void* states, void* out, uint64_t n, float loc, float scale, bool staged,
                      cudaStream_t st) {
  if (n == 0) return;
  switch (dtype) {
    case kFloat16: Launch<__half>(states, out, n, loc, scale, staged, st); break;
    case kBfloat16: Launch<__nv_bfloat16>(states, out, n, loc, scale, staged, st); break;
    case kFloat32: Launch<float>(states, out, n, loc, scale, staged, st); break;
    case kFloat64: Launch<double>(states, out, n, loc, scale, staged, st); break;
    default: KV_FATAL << "_random_normal: unsupported dtype " << DTypeName(dtype);
  }
  KV_CUDA(cudaGetLastError());
}

}  // namespace b200kv
