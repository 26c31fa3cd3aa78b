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
// lane of the warp calls it. draw is called once per element in run order (it may keep a cursor),
// and every element's draw happens before the warp stores that element.
template <typename T, typename DrawFn>
__device__ __forceinline__ void DrawRunStaged(curandStatePhilox4_32_10_t* st, T* __restrict__ out, uint64_t step,
                                              uint64_t len, uint32_t t, uint32_t vec, DrawFn&& draw) {
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

// mshadow's half_t as a parameter type (half.h): every operator with a half_t operand rounds
// float(a) OP float(b) to half, and a comparison compares the two floats. The multi-sample kernels
// do their parameter arithmetic in it, as the reference's do with IType half_t.
struct HalfT {
  __half h;
  HalfT() = default;
  __device__ __forceinline__ HalfT(float f) : h(__float2half_rn(f)) {}
  __device__ __forceinline__ operator float() const { return __half2float(h); }
};
static_assert(sizeof(HalfT) == 2, "a float16 parameter array is read as HalfT");
#define B200KV_HALF_OP(R, OP)                                                                           \
  __device__ __forceinline__ R operator OP(HalfT a, HalfT b) { return R(float(a) OP float(b)); }           \
  template <typename X>                                                                                    \
  __device__ __forceinline__ R operator OP(HalfT a, X b) { return R(float(a) OP float(b)); }               \
  template <typename X>                                                                                    \
  __device__ __forceinline__ R operator OP(X a, HalfT b) { return R(float(a) OP float(b)); }
B200KV_HALF_OP(HalfT, +)
B200KV_HALF_OP(HalfT, -)
B200KV_HALF_OP(HalfT, *)
B200KV_HALF_OP(HalfT, /)
B200KV_HALF_OP(bool, <)
B200KV_HALF_OP(bool, >)
#undef B200KV_HALF_OP

// The draws of sampler.h with parameters of type P (float for the scalar samplers; IType for the
// multi-sample ones), written as the reference writes them so that the mixed float / double / half_t
// arithmetic and its contraction are the same.

// SampleUniformKernel: OType(lower + (upper - lower) * uniform())
template <typename T, typename P>
__device__ __forceinline__ T UniformOf(curandStatePhilox4_32_10_t* s, P lower, P upper) {
  const Gen<T> u = Uniform01<Gen<T>>(s);
  return Out<T>::Of(lower + (upper - lower) * u);
}

// SampleNormalKernel: OType(normal() * std + mean)
template <typename T, typename P>
__device__ __forceinline__ T NormalOf(curandStatePhilox4_32_10_t* s, P mean, P std) {
  return Out<T>::Of(Normal01<Gen<T>>(s) * std + mean);
}

// SampleExponentialKernel: OType(-log(1.0 - uniform()) / lambda)
template <typename T, typename P>
__device__ __forceinline__ T ExponentialOf(curandStatePhilox4_32_10_t* s, P lambda) {
  const Gen<T> u = Uniform01<Gen<T>>(s);
  return Out<T>::Of(-log(1.0 - u) / lambda);
}

// SampleGamma in FType = Gen<T>: Marsaglia-Tsang, one normal and one uniform per attempt that gets
// past Z > -k, and one more uniform for alpha < 1. The literals are double, as in the reference, so
// d, k and c are rounded from double and the acceptance test is evaluated in double.
//
// The reference loops until an attempt is accepted, which never happens when d is NaN, <= 0 or +inf
// (alpha NaN, +-inf or <= -2/3). Here an element gets kGammaAttempts attempts; one that exhausts
// them is NaN, without alpha < 1's last uniform, and the thread goes on to its next element. For
// alpha > 0, d >= 2/3 and an attempt fails with probability below about 0.05, so a valid element
// exhausts the budget with probability near 1e-80 (DESIGN.md §8).
constexpr int kGammaAttempts = 64;
template <typename T, typename P>
__device__ __forceinline__ T GammaOf(curandStatePhilox4_32_10_t* s, P alpha, P beta) {
  using F = Gen<T>;
  const F d = alpha < 1 ? alpha + 2.0 / 3.0 : alpha - 1.0 / 3.0;
  const F k = sqrt(9.0 * d);
  const F c = 1.0 / k;
  F sample;
  int attempt = 0;
  for (; attempt < kGammaAttempts; ++attempt) {
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
  if (attempt == kGammaAttempts) return Out<T>::Of(F(NAN));
  return Out<T>::Of(alpha < 1 ? sample * pow(Uniform01<F>(s), F(1.0 / alpha)) : sample);
}

// the scalar samplers' draws (sample_op.h: float parameters)
template <typename T>
struct UniformDraw {
  float lower, upper;
  __device__ __forceinline__ T operator()(curandStatePhilox4_32_10_t* s) const { return UniformOf<T>(s, lower, upper); }
};

template <typename T>
struct ExponentialDraw {
  float lambda;
  __device__ __forceinline__ T operator()(curandStatePhilox4_32_10_t* s) const { return ExponentialOf<T>(s, lambda); }
};

template <typename T>
struct GammaDraw {
  float alpha, beta;
  __device__ __forceinline__ T operator()(curandStatePhilox4_32_10_t* s) const { return GammaOf<T>(s, alpha, beta); }
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

// ---- the multi-sample kernels of multisample_op.h: sampler.h's kernels with nParm > 1, element i
// drawing with parameters i / nBatch, nBatch = 1 + (N - 1) / nParm. P is the parameter arrays' type
// (HalfT for float16), T the output's.

// A thread's parameter cursor: a and b point at the parameters of the next element it draws, and
// left elements remain in their batch. Set once per thread from the run's first element and advanced
// per draw, so the hot loop divides nothing. Each draw reads its parameters before the element is
// stored (DrawRunStaged), so out may be a parameter array itself (nBatch 1).
template <int kDist, typename P, typename T>
struct ParamDraw {
  const P* a;
  const P* b;
  uint64_t nbatch, left;
  __device__ __forceinline__ T operator()(curandStatePhilox4_32_10_t* s) {
    const P x = *a;
    const P y = kDist == kRandExponential ? x : *b;
    if (--left == 0) {
      left = nbatch;
      ++a;
      ++b;
    }
    if constexpr (kDist == kRandUniform) return UniformOf<T>(s, x, y);
    else if constexpr (kDist == kRandNormal) return NormalOf<T>(s, x, y);
    else if constexpr (kDist == kRandExponential) return ExponentialOf<T>(s, x);
    else return GammaOf<T>(s, x, y);
  }
};

// x / d and x % d for x < 2^52 from the host's inv = 1.0 / d: the double product is within one of
// the quotient, which one correction step settles (no 64-bit division routine, so no stack frame)
__device__ __forceinline__ void DivModBatch(uint64_t x, uint64_t d, double inv, uint64_t* q, uint64_t* r) {
  uint64_t qq = static_cast<uint64_t>(static_cast<double>(x) * inv);
  int64_t rr = static_cast<int64_t>(x - qq * d);
  if (rr < 0) {
    --qq;
    rr += static_cast<int64_t>(d);
  } else if (rr >= static_cast<int64_t>(d)) {
    ++qq;
    rr -= static_cast<int64_t>(d);
  }
  *q = qq;
  *r = static_cast<uint64_t>(rr);
}

// min blocks 1: without it ptxas caps some instantiations near 40-64 registers and spills; a full
// launch is 512 CTAs, about 4 per SM, so the registers cost no occupancy the launch could use
template <int kDist, typename P, typename T>
__global__ void __launch_bounds__(kDrawThreads, 1)
    param_draw_kernel(curandStatePhilox4_32_10_t* states, T* out, uint64_t n, uint64_t step, uint32_t nthread,
                      const P* a, const P* b, uint64_t nbatch, double inv_nbatch, uint32_t vec) {
  const uint32_t t = blockIdx.x * kDrawThreads + threadIdx.x;
  const uint64_t start = static_cast<uint64_t>(t) * step;
  const uint64_t len = t < nthread && start < n ? (n - start < step ? n - start : step) : 0;
  curandStatePhilox4_32_10_t st;
  ParamDraw<kDist, P, T> draw{a, b, nbatch, 0};
  if (len > 0) {
    st = states[t];
    uint64_t p, rem;
    DivModBatch(start, nbatch, inv_nbatch, &p, &rem);
    draw.a += p;
    draw.b += p;
    draw.left = nbatch - rem;
  }
  DrawRunStaged(&st, out, step, len, t, vec, draw);
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

template <int kDist, typename P, typename T>
void LaunchParam(void* states, const void* a, const void* b, uint64_t nparm, void* out, uint64_t n,
                 cudaStream_t st) {
  const DrawShape d = ShapeFor<T>(out, n);
  const uint64_t nbatch = 1 + (n - 1) / nparm;
  param_draw_kernel<kDist, P, T><<<d.blocks, kDrawThreads, 0, st>>>(
      static_cast<curandStatePhilox4_32_10_t*>(states), static_cast<T*>(out), n, d.step,
      static_cast<uint32_t>(d.nthread), static_cast<const P*>(a), static_cast<const P*>(b), nbatch,
      1.0 / static_cast<double>(nbatch), d.vec);
}

template <int kDist, typename P>
void LaunchParamOut(int otype, void* states, const void* a, const void* b, uint64_t nparm, void* out, uint64_t n,
                    cudaStream_t st) {
  switch (otype) {
    case kFloat16: LaunchParam<kDist, P, __half>(states, a, b, nparm, out, n, st); break;
    case kFloat32: LaunchParam<kDist, P, float>(states, a, b, nparm, out, n, st); break;
    case kFloat64: LaunchParam<kDist, P, double>(states, a, b, nparm, out, n, st); break;
    default: KV_FATAL << "multi-sample: unsupported output dtype " << DTypeName(otype);
  }
}

template <int kDist>
void LaunchParamDist(int ptype, int otype, void* states, const void* a, const void* b, uint64_t nparm, void* out,
                     uint64_t n, cudaStream_t st) {
  switch (ptype) {
    case kFloat16: LaunchParamOut<kDist, HalfT>(otype, states, a, b, nparm, out, n, st); break;
    case kFloat32: LaunchParamOut<kDist, float>(otype, states, a, b, nparm, out, n, st); break;
    case kFloat64: LaunchParamOut<kDist, double>(otype, states, a, b, nparm, out, n, st); break;
    default: KV_FATAL << "multi-sample: unsupported parameter dtype " << DTypeName(ptype);
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

void LaunchRandSampleParams(int dist, int ptype, int otype, void* states, const void* a, const void* b,
                            uint64_t nparm, void* out, uint64_t n, cudaStream_t st) {
  if (n == 0) return;
  KV_CHECK(nparm > 0 && n % nparm == 0) << "multi-sample: " << n << " outputs for " << nparm << " parameters";
  KV_CHECK(n < (uint64_t{1} << 52)) << "multi-sample: " << n << " outputs is past the kernel's index range";
  switch (dist) {
    case kRandUniform: LaunchParamDist<kRandUniform>(ptype, otype, states, a, b, nparm, out, n, st); break;
    case kRandNormal: LaunchParamDist<kRandNormal>(ptype, otype, states, a, b, nparm, out, n, st); break;
    case kRandExponential: LaunchParamDist<kRandExponential>(ptype, otype, states, a, a, nparm, out, n, st); break;
    case kRandGamma: LaunchParamDist<kRandGamma>(ptype, otype, states, a, b, nparm, out, n, st); break;
    default: KV_FATAL << "multi-sample: no sampler " << dist;
  }
  KV_CUDA(cudaGetLastError());
}

}  // namespace b200kv
