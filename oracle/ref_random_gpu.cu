// TEST INFRASTRUCTURE ONLY (see DESIGN.md §6) -- the reference's own GPU normal sampler behind a
// C interface for the tests: RandGenerator<gpu, float> (include/mxnet/random_generator.h,
// src/common/random_generator.cu, compiled beside this file by oracle/random_gpu.mk) and
// LaunchRNG<SampleNormalKernel<gpu>> (src/operator/random/sampler.h), called as normal_op calls
// them (sample_op.h: loc and scale each one float in device memory, nParm 1). The states travel
// through host memory so that the tests hold every byte of them.
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

template <typename OType>
int Normal(void* host_states, int64_t n, float loc, float scale, void* host_out) {
  GenF gen;
  GenF::AllocState(&gen);
  cudaMemcpy(*StatesOf(&gen), host_states, kBytes, cudaMemcpyHostToDevice);
  float par[2] = {loc, scale};
  float* d_par = nullptr;
  OType* d_out = nullptr;
  cudaMalloc(&d_par, sizeof(par));
  cudaMemcpy(d_par, par, sizeof(par), cudaMemcpyHostToDevice);
  cudaMalloc(&d_out, (n > 0 ? n : 1) * sizeof(OType));
  mshadow::Stream<gpu> s;
  auto* g = reinterpret_cast<mxnet::common::random::RandGenerator<gpu, OType>*>(&gen);
  mxnet::op::LaunchRNG<mxnet::op::SampleNormalKernel<gpu>, gpu>(&s, g, static_cast<mxnet::index_t>(n),
                                                               static_cast<mxnet::index_t>(1),
                                                               static_cast<mxnet::index_t>(n), d_par,
                                                               d_par + 1, d_out);
  int rc = Check();
  if (n > 0) cudaMemcpy(host_out, d_out, n * sizeof(OType), cudaMemcpyDeviceToHost);
  cudaMemcpy(host_states, *StatesOf(&gen), kBytes, cudaMemcpyDeviceToHost);
  cudaFree(d_out);
  cudaFree(d_par);
  GenF::FreeState(&gen);
  return rc == 0 ? Check() : rc;
}

}  // namespace

extern "C" {

int mxref_rand_state_bytes(void) { return static_cast<int>(sizeof(curandStatePhilox4_32_10_t)); }

// RandGenerator<gpu, float>::Seed(seed) on a fresh copy of 32768 states, copied to host_states
int mxref_rand_seed(uint32_t seed, void* host_states) {
  GenF gen;
  GenF::AllocState(&gen);
  mshadow::Stream<gpu> s;
  gen.Seed(&s, seed);
  int rc = Check();
  cudaMemcpy(host_states, *StatesOf(&gen), kBytes, cudaMemcpyDeviceToHost);
  GenF::FreeState(&gen);
  return rc == 0 ? Check() : rc;
}

// normal_op's draw of n elements of type_flag (mshadow: 0 float32, 1 float64, 2 float16) from the
// states in host_states, which are replaced by the states the launch leaves
int mxref_rand_normal(void* host_states, int64_t n, float loc, float scale, int type_flag, void* host_out) {
  switch (type_flag) {
    case 0: return Normal<float>(host_states, n, loc, scale, host_out);
    case 1: return Normal<double>(host_states, n, loc, scale, host_out);
    case 2: return Normal<mshadow::half::half_t>(host_states, n, loc, scale, host_out);
    default: return -1;
  }
}

}  // extern "C"
