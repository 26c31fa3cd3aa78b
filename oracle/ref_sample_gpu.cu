// TEST INFRASTRUCTURE ONLY (see DESIGN.md §6) -- the reference's own GPU uniform, exponential,
// gamma and randint samplers behind a C interface for the tests: RandGenerator<gpu>
// (include/mxnet/random_generator.h, src/common/random_generator.cu, compiled beside this file by
// oracle/sample_gpu.mk) and the UniformSampler, ExponentialSampler, GammaSampler and RandIntSampler
// of src/operator/random/sampler.h, called as uniform_op, exponential_op, gamma_op and rand_int_op
// call them (sample_op.h: float parameters, int64 for randint, each one element in device memory,
// nParm 1). The states travel through host memory so that the tests hold every byte of them, in the
// layout of oracle/ref_random_gpu.cu's seeded states; mxref_sample_time keeps them on the device and
// times the launches alone.
#include <mxnet/random_generator.h>

#include <cstdint>
#include <cstring>

#include "operator/mxnet_op.h"
#include "operator/random/sampler.h"

namespace {

using mshadow::gpu;
typedef mxnet::common::random::RandGenerator<gpu, float> GenF;
constexpr size_t kBytes = 32768 * sizeof(curandStatePhilox4_32_10_t);
static_assert(sizeof(GenF) == sizeof(void*), "the generator is its state pointer");

// the generator's state pointer (its one, private, member)
curandStatePhilox4_32_10_t** StatesOf(GenF* g) { return reinterpret_cast<curandStatePhilox4_32_10_t**>(g); }

int Check() { return cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess ? 0 : -1; }

enum { kUniform = 0, kExponential = 1, kGamma = 2, kRandInt = 3 };

// the sampler of `dist` over out[0, n) from gen, its parameters at d_par (float, or int64 for
// randint), as the *_op functions of sample_op.h call it
template <typename OType>
void Sample(int dist, mshadow::Stream<gpu>* s, GenF* gen, void* d_par, OType* d_out, int64_t n) {
  using mshadow::Shape1;
  using mshadow::Tensor;
  auto* g = reinterpret_cast<mxnet::common::random::RandGenerator<gpu, OType>*>(gen);
  Tensor<gpu, 1, OType> out(d_out, Shape1(n), s);
  float* fp = static_cast<float*>(d_par);
  int64_t* ip = static_cast<int64_t*>(d_par);
  Tensor<gpu, 1, float> p0(fp, Shape1(1), s), p1(fp + 1, Shape1(1), s);
  switch (dist) {
    case kUniform: mxnet::op::UniformSampler<gpu>().Sample(p0, p1, out, g, s); break;
    case kExponential: mxnet::op::ExponentialSampler<gpu>().Sample(p0, out, g, s); break;
    case kGamma: mxnet::op::GammaSampler<gpu>().Sample(p0, p1, out, g, s); break;
    case kRandInt:
      mxnet::op::RandIntSampler<gpu>().Sample(Tensor<gpu, 1, int64_t>(ip, Shape1(1), s),
                                              Tensor<gpu, 1, int64_t>(ip + 1, Shape1(1), s), out, g, s);
      break;
  }
}

// par: the two parameters as the operator holds them (2 floats, or 2 int64 for randint)
template <typename OType>
int Sampled(int dist, void* host_states, int64_t n, const void* par, void* host_out) {
  GenF gen;
  GenF::AllocState(&gen);
  cudaMemcpy(*StatesOf(&gen), host_states, kBytes, cudaMemcpyHostToDevice);
  void* d_par = nullptr;
  OType* d_out = nullptr;
  cudaMalloc(&d_par, 2 * sizeof(int64_t));
  cudaMemcpy(d_par, par, 2 * sizeof(int64_t), cudaMemcpyHostToDevice);
  cudaMalloc(&d_out, (n > 0 ? n : 1) * sizeof(OType));
  mshadow::Stream<gpu> s;
  Sample<OType>(dist, &s, &gen, d_par, d_out, n);
  int rc = Check();
  if (n > 0) cudaMemcpy(host_out, d_out, n * sizeof(OType), cudaMemcpyDeviceToHost);
  cudaMemcpy(host_states, *StatesOf(&gen), kBytes, cudaMemcpyDeviceToHost);
  cudaFree(d_out);
  cudaFree(d_par);
  GenF::FreeState(&gen);
  return rc == 0 ? Check() : rc;
}

int SampledAny(int dist, void* host_states, int64_t n, const void* par, int type_flag, void* host_out) {
  if (dist == kRandInt) {
    switch (type_flag) {
      case 4: return Sampled<int32_t>(dist, host_states, n, par, host_out);
      case 6: return Sampled<int64_t>(dist, host_states, n, par, host_out);
      default: return -1;
    }
  }
  switch (type_flag) {
    case 0: return Sampled<float>(dist, host_states, n, par, host_out);
    case 1: return Sampled<double>(dist, host_states, n, par, host_out);
    case 2: return Sampled<mshadow::half::half_t>(dist, host_states, n, par, host_out);
    default: return -1;
  }
}

// ms per launch over `reps` launches after `warmup`, CUDA events around the launches only
template <typename OType>
int Timed(int dist, int64_t n, const void* par, int warmup, int reps, float* ms) {
  GenF gen;
  GenF::AllocState(&gen);
  mshadow::Stream<gpu> s;
  gen.Seed(&s, 17);
  void* d_par = nullptr;
  OType* d_out = nullptr;
  cudaMalloc(&d_par, 2 * sizeof(int64_t));
  cudaMemcpy(d_par, par, 2 * sizeof(int64_t), cudaMemcpyHostToDevice);
  cudaMalloc(&d_out, (n > 0 ? n : 1) * sizeof(OType));
  for (int i = 0; i < warmup; ++i) Sample<OType>(dist, &s, &gen, d_par, d_out, n);
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  cudaEventRecord(a, 0);
  for (int i = 0; i < reps; ++i) Sample<OType>(dist, &s, &gen, d_par, d_out, n);
  cudaEventRecord(b, 0);
  int rc = Check();
  cudaEventElapsedTime(ms, a, b);
  *ms /= reps;
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  cudaFree(d_out);
  cudaFree(d_par);
  GenF::FreeState(&gen);
  return rc == 0 ? Check() : rc;
}

}  // namespace

extern "C" {

// uniform_op / exponential_op / gamma_op's draw of n elements of type_flag (0 float32, 1 float64,
// 2 float16) with float parameters (low, high), (lam) or (alpha, beta); states as for normal
int mxref_sample_uniform(void* host_states, int64_t n, float low, float high, int type_flag, void* host_out) {
  const float par[4] = {low, high, 0, 0};
  return SampledAny(kUniform, host_states, n, par, type_flag, host_out);
}

int mxref_sample_exponential(void* host_states, int64_t n, float lam, int type_flag, void* host_out) {
  const float par[4] = {lam, 0, 0, 0};
  return SampledAny(kExponential, host_states, n, par, type_flag, host_out);
}

int mxref_sample_gamma(void* host_states, int64_t n, float alpha, float beta, int type_flag, void* host_out) {
  const float par[4] = {alpha, beta, 0, 0};
  return SampledAny(kGamma, host_states, n, par, type_flag, host_out);
}

// rand_int_op's draw with int64 bounds into type_flag 4 (int32) or 6 (int64)
int mxref_sample_randint(void* host_states, int64_t n, int64_t low, int64_t high, int type_flag, void* host_out) {
  const int64_t par[2] = {low, high};
  return SampledAny(kRandInt, host_states, n, par, type_flag, host_out);
}

// the reference's launch alone: ms per call of sampler dist (0 uniform, 1 exponential, 2 gamma,
// 3 randint) over n elements of type_flag, the generator on the device, p0 / p1 its parameters
int mxref_sample_time(int dist, int64_t n, double p0, double p1, int type_flag, int warmup, int reps, float* ms) {
  const float fpar[4] = {static_cast<float>(p0), static_cast<float>(p1), 0, 0};
  const int64_t ipar[2] = {static_cast<int64_t>(p0), static_cast<int64_t>(p1)};
  const void* par = dist == kRandInt ? static_cast<const void*>(ipar) : static_cast<const void*>(fpar);
  switch (type_flag) {
    case 0: return Timed<float>(dist, n, par, warmup, reps, ms);
    case 1: return Timed<double>(dist, n, par, warmup, reps, ms);
    case 2: return Timed<mshadow::half::half_t>(dist, n, par, warmup, reps, ms);
    case 4: return Timed<int32_t>(dist, n, par, warmup, reps, ms);
    case 6: return Timed<int64_t>(dist, n, par, warmup, reps, ms);
    default: return -1;
  }
}

}  // extern "C"
