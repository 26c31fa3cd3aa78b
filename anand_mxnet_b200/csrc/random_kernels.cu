// random_kernels.cu -- the reference's GPU samplers (kernels.h, LaunchRandSeed / LaunchRandNormal /
// LaunchRandSample).
//
// The stream is fixed by the reference: curandStatePhilox4_32_10_t states seeded with
// curand_init(seed, id, 0) (common/random_generator.cu), and LaunchRNG's mapping (random/sampler.h):
// nthread = min(ceil(N / 64), 32768), step = ceil(N / nthread), thread t draws elements
// [t*step, min((t+1)*step, N)) in order from state t, which it holds in registers and writes back
// whole, curand's cached Box-Muller value included. Normal element i is
// OType(normal() * scale + loc) with contraction on: one fmaf (float, half, bfloat16: the float
// normal rounded once) or one fma in double (curand_normal_double). This file is compiled with
// -fmad=true like the reference's GPU build, so curand's own Box-Muller arithmetic and the samplers'
// mixed float / double expressions contract as they do there (build.py).
//
// The store order is free. A thread owns a contiguous run, so storing as it draws puts the 32 lanes
// of a warp step*sizeof(T) bytes apart. The staged kernels instead have each lane draw 128 B of its
// run into a per-warp shared tile, then the warp writes each lane's 128 B as 8 lanes x 16 B (4 runs
// per store instruction) when out and step allow 16-B vectors, else lane-contiguous scalars.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <curand_kernel.h>

#include <algorithm>
#include <type_traits>

#include "common.h"
#include "kernels.h"

namespace b200kv {

static_assert(sizeof(curandStatePhilox4_32_10_t) == kRandStateBytes, "a state is persisted whole");

namespace {

constexpr int kSeedThreads = 256;   // the reference's kBaseThreadNum
constexpr int kDrawThreads = 64;  // 2 warps: 512 CTAs for 32768 states spread over all 132 SMs

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

// The staged store of thread t's run: len elements from draw(&st) (len == 0: t draws nothing), through
// the warp's shared tile, to out[t*step, t*step + len). vec: out and step allow 16-B vectors. Every
// lane of the warp calls it.
template <typename T, typename DrawFn>
__device__ __forceinline__ void DrawRunStaged(curandStatePhilox4_32_10_t* st, T* __restrict__ out, uint64_t step,
                                              uint64_t len, uint32_t t, uint32_t vec, const DrawFn& draw) {
  constexpr int kRun = 128 / sizeof(T);         // elements a lane draws per round
  constexpr int kPerVec = 16 / sizeof(T);
  constexpr int kPad = sizeof(T) >= 4 ? 1 : 4 / sizeof(T);  // tile rows 4 B apart in banks
  __shared__ T smem[kDrawThreads / 32][32][kRun + kPad];
  T(*tile)[kRun + kPad] = smem[threadIdx.x / 32];
  const int lane = threadIdx.x & 31;
  const uint64_t warp_t0 = t - lane;
  for (uint64_t r = 0; __any_sync(~0u, r < len); r += kRun) {
    const int cnt = r < len ? static_cast<int>(len - r < kRun ? len - r : kRun) : 0;
    for (int k = 0; k < cnt; ++k) tile[lane][k] = draw(st);
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

// kStaged = false: each thread stores as it draws (the reference's order; kept for bench_random.py)
template <typename T, bool kStaged>
__global__ void __launch_bounds__(kDrawThreads)
    normal_kernel(curandStatePhilox4_32_10_t* states, T* __restrict__ out, uint64_t n, uint64_t step,
                  uint32_t nthread, float loc, float scale, uint32_t vec) {
  const uint32_t t = blockIdx.x * kDrawThreads + threadIdx.x;
  const uint64_t start = static_cast<uint64_t>(t) * step;
  const uint64_t len = t < nthread && start < n ? (n - start < step ? n - start : step) : 0;
  curandStatePhilox4_32_10_t st;
  if (len > 0) st = states[t];
  if constexpr (!kStaged) {
    for (uint64_t i = 0; i < len; ++i) out[start + i] = Draw<T>::Get(&st, loc, scale);
  } else {
    DrawRunStaged(&st, out, step, len, t, vec,
                  [loc, scale](curandStatePhilox4_32_10_t* s) { return Draw<T>::Get(s, loc, scale); });
  }
  if (len > 0) states[t] = st;
}

// ---- the scalar-parameter samplers of random/sampler.h. RandGenerator<gpu, G>::Impl draws in
// double for double outputs and in float for every other output type (half_t included): Gen<T>.
template <typename T>
using Gen = typename std::conditional<std::is_same<T, double>::value, double, float>::type;

// Impl::uniform(): 1 - curand_uniform, in [0, 1); the double form subtracts from a float 1
template <typename G>
__device__ __forceinline__ G Uniform01(curandStatePhilox4_32_10_t* s);
template <>
__device__ __forceinline__ float Uniform01<float>(curandStatePhilox4_32_10_t* s) {
  return static_cast<float>(1.0) - curand_uniform(s);
}
template <>
__device__ __forceinline__ double Uniform01<double>(curandStatePhilox4_32_10_t* s) {
  return static_cast<float>(1.0) - curand_uniform_double(s);
}

// Impl::normal()
template <typename G>
__device__ __forceinline__ G Normal01(curandStatePhilox4_32_10_t* s);
template <>
__device__ __forceinline__ float Normal01<float>(curandStatePhilox4_32_10_t* s) {
  return curand_normal(s);
}
template <>
__device__ __forceinline__ double Normal01<double>(curandStatePhilox4_32_10_t* s) {
  return curand_normal_double(s);
}

// OType(x): half_t(x) rounds float(x) to nearest even (mshadow half.h); bfloat16 likewise (the
// extension's definition: the float32 result rounded once)
template <typename T>
struct Out {
  template <typename X>
  static __device__ __forceinline__ T Of(X x) { return static_cast<T>(x); }
};
template <>
struct Out<__half> {
  template <typename X>
  static __device__ __forceinline__ __half Of(X x) { return __float2half_rn(static_cast<float>(x)); }
};
template <>
struct Out<__nv_bfloat16> {
  template <typename X>
  static __device__ __forceinline__ __nv_bfloat16 Of(X x) { return __float2bfloat16_rn(static_cast<float>(x)); }
};

// SampleUniformKernel: OType(lower + (upper - lower) * uniform()), lower and upper float
template <typename T>
struct UniformDraw {
  float lower, upper;
  __device__ __forceinline__ T operator()(curandStatePhilox4_32_10_t* s) const {
    const Gen<T> u = Uniform01<Gen<T>>(s);
    return Out<T>::Of(lower + (upper - lower) * u);
  }
};

// SampleExponentialKernel: OType(-log(1.0 - uniform()) / lambda), in double
template <typename T>
struct ExponentialDraw {
  float lambda;
  __device__ __forceinline__ T operator()(curandStatePhilox4_32_10_t* s) const {
    const Gen<T> u = Uniform01<Gen<T>>(s);
    return Out<T>::Of(-log(1.0 - u) / lambda);
  }
};

// SampleGamma in FType = Gen<T>: Marsaglia-Tsang, one normal and one uniform per attempt that gets
// past Z > -k, and one more uniform for alpha < 1. The literals are double, as in the reference, so
// d, k and c are rounded from double and the acceptance test is evaluated in double.
template <typename T>
struct GammaDraw {
  float alpha, beta;
  __device__ __forceinline__ T operator()(curandStatePhilox4_32_10_t* s) const {
    using F = Gen<T>;
    const F d = alpha < 1 ? alpha + 2.0 / 3.0 : alpha - 1.0 / 3.0;
    const F k = sqrt(9.0 * d);
    const F c = 1.0 / k;
    F sample;
    while (true) {
      const F z = Normal01<F>(s);
      if (z > -k) {
        const F x = 1.0 + c * z;
        const F v = x * x * x;
        if (log(1.0 - Uniform01<F>(s)) < 0.5 * z * z + d * (1.0 - v + log(v))) {
          sample = d * v * beta;
          break;
        }
      }
    }
    return Out<T>::Of(alpha < 1 ? sample * pow(Uniform01<F>(s), F(1.0 / alpha)) : sample);
  }
};

// SampleRandIntKernel with int64 bounds: OType(lower + rand_int64() % (upper - lower)), where
// rand_int64() = int64(uint32(curand() << 31)) + curand() takes the shifted draw first (nvcc's
// order in the reference's build). range = upper - lower > 0.
//
// x = rand_int64() < 2^33, so x % range is x when range > x; otherwise the quotient is below 2^33
// and the double quotient of the two exact operands is floor(x / range) or one more, which one
// correction step settles. This is the same remainder without the 64-bit division routine, whose
// call costs the int64 kernel a stack frame.
__device__ __forceinline__ int64_t RandInt64Mod(curandStatePhilox4_32_10_t* s, int64_t range) {
  const unsigned hi = curand(s);
  const unsigned lo = curand(s);
  const int64_t x = static_cast<int64_t>(hi << 31) + lo;
  if (range > x) return x;
  const int64_t q = static_cast<int64_t>(static_cast<double>(x) / static_cast<double>(range));
  const int64_t r = x - q * range;
  return r < 0 ? r + range : r;
}

template <typename T>
struct RandIntDraw {
  int64_t lower, range;
  __device__ __forceinline__ T operator()(curandStatePhilox4_32_10_t* s) const {
    return static_cast<T>(lower + RandInt64Mod(s, range));
  }
};

template <typename Dist, typename T>
__global__ void __launch_bounds__(kDrawThreads)
    sample_kernel(curandStatePhilox4_32_10_t* states, T* __restrict__ out, uint64_t n, uint64_t step,
                  uint32_t nthread, Dist dist, uint32_t vec) {
  const uint32_t t = blockIdx.x * kDrawThreads + threadIdx.x;
  const uint64_t start = static_cast<uint64_t>(t) * step;
  const uint64_t len = t < nthread && start < n ? (n - start < step ? n - start : step) : 0;
  curandStatePhilox4_32_10_t st;
  if (len > 0) st = states[t];
  DrawRunStaged(&st, out, step, len, t, vec, dist);
  if (len > 0) states[t] = st;
}

// LaunchRNG's nthread and step for n > 0 elements, the grid, and whether 16-B stores apply
struct DrawShape {
  uint64_t nthread, step;
  unsigned blocks;
  uint32_t vec;
};
template <typename T>
DrawShape ShapeFor(const void* out, uint64_t n) {
  DrawShape d;
  const uint64_t nloop = (n + kRandMinPerThread - 1) / kRandMinPerThread;
  d.nthread = std::min<uint64_t>(nloop, kRandStates);
  d.step = (n + d.nthread - 1) / d.nthread;
  d.blocks = static_cast<unsigned>((d.nthread + kDrawThreads - 1) / kDrawThreads);
  d.vec = (reinterpret_cast<uintptr_t>(out) & 15) == 0 && d.step % (16 / sizeof(T)) == 0;
  return d;
}

template <typename T, typename Dist>
void LaunchSample(void* states, void* out, uint64_t n, const Dist& dist, cudaStream_t st) {
  const DrawShape d = ShapeFor<T>(out, n);
  sample_kernel<Dist, T><<<d.blocks, kDrawThreads, 0, st>>>(static_cast<curandStatePhilox4_32_10_t*>(states),
                                                             static_cast<T*>(out), n, d.step,
                                                             static_cast<uint32_t>(d.nthread), dist, d.vec);
}

template <typename T>
void LaunchFloatSample(int dist, void* states, void* out, uint64_t n, const RandParams& p, cudaStream_t st) {
  switch (dist) {
    case kRandUniform: LaunchSample<T>(states, out, n, UniformDraw<T>{p.a, p.b}, st); break;
    case kRandExponential: LaunchSample<T>(states, out, n, ExponentialDraw<T>{p.a}, st); break;
    case kRandGamma: LaunchSample<T>(states, out, n, GammaDraw<T>{p.a, p.b}, st); break;
    default: KV_FATAL << "random sampler " << dist << " has no floating-point form";
  }
}

template <typename T>
void Launch(void* states, void* out, uint64_t n, float loc, float scale, bool staged, cudaStream_t st) {
  const DrawShape d = ShapeFor<T>(out, n);
  auto* s = static_cast<curandStatePhilox4_32_10_t*>(states);
  T* o = static_cast<T*>(out);
  if (staged) {
    normal_kernel<T, true><<<d.blocks, kDrawThreads, 0, st>>>(s, o, n, d.step, static_cast<uint32_t>(d.nthread),
                                                              loc, scale, d.vec);
  } else {
    normal_kernel<T, false><<<d.blocks, kDrawThreads, 0, st>>>(s, o, n, d.step, static_cast<uint32_t>(d.nthread),
                                                               loc, scale, d.vec);
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

void LaunchRandSample(int dist, int dtype, void* states, void* out, uint64_t n, const RandParams& p,
                      cudaStream_t st) {
  if (n == 0) return;
  if (dist == kRandInt) {
    KV_CHECK(p.hi > p.lo) << "_random_randint: the range must not be empty";
    const RandIntDraw<int32_t> d32{p.lo, p.hi - p.lo};
    const RandIntDraw<int64_t> d64{p.lo, p.hi - p.lo};
    switch (dtype) {
      case kInt32: LaunchSample<int32_t>(states, out, n, d32, st); break;
      case kInt64: LaunchSample<int64_t>(states, out, n, d64, st); break;
      default: KV_FATAL << "_random_randint: unsupported dtype " << DTypeName(dtype);
    }
  } else {
    switch (dtype) {
      case kFloat16: LaunchFloatSample<__half>(dist, states, out, n, p, st); break;
      case kBfloat16: LaunchFloatSample<__nv_bfloat16>(dist, states, out, n, p, st); break;
      case kFloat32: LaunchFloatSample<float>(dist, states, out, n, p, st); break;
      case kFloat64: LaunchFloatSample<double>(dist, states, out, n, p, st); break;
      default: KV_FATAL << "random sampler: unsupported dtype " << DTypeName(dtype);
    }
  }
  KV_CUDA(cudaGetLastError());
}

}  // namespace b200kv
