// TEST INFRASTRUCTURE ONLY (see DESIGN.md §6) -- the reference's own GPU multi-sample samplers behind
// a C interface for the tests: RandGenerator<gpu> (src/common/random_generator.cu, compiled beside
// this file by oracle/sample_params_gpu.mk) and the UniformSampler, NormalSampler, GammaSampler and
// ExponentialSampler of src/operator/random/sampler.h, called as multisample_op.h's SamplerCaller
// calls them: typed parameter arrays of nParm elements (IType float16 / float32 / float64) and an
// output of n elements (OType likewise). The states travel through host memory in the layout of
// oracle/ref_random_gpu.cu's seeded states; mxref_multisample_time keeps them on the device and times
// the launches alone.
//
// Never call it with a gamma parameter whose draw cannot end (alpha NaN, +-inf or <= -2/3): the
// reference's loop would not return.
#include <mxnet/random_generator.h>

#include <cstdint>
#include <vector>

#include "operator/mxnet_op.h"
#include "operator/random/sampler.h"

namespace {

using mshadow::gpu;
using mshadow::half::half_t;
typedef mxnet::common::random::RandGenerator<gpu, float> GenF;
constexpr size_t kBytes = 32768 * sizeof(curandStatePhilox4_32_10_t);
static_assert(sizeof(GenF) == sizeof(void*), "the generator is its state pointer");

curandStatePhilox4_32_10_t** StatesOf(GenF* g) { return reinterpret_cast<curandStatePhilox4_32_10_t**>(g); }

int Check() { return cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess ? 0 : -1; }

enum { kUniform = 0, kNormal = 1, kGamma = 2, kExponential = 3 };

size_t TypeSize(int flag) { return flag == 1 ? 8 : flag == 0 ? 4 : 2; }

// SamplerCaller<gpu, IType, OType, Sampler, inum>::op over device arrays a, b (nparm) and out (n)
template <typename IType, typename OType>
void Sample(int dist, mshadow::Stream<gpu>* s, GenF* gen, const void* a, const void* b, int64_t nparm,
            void* out, int64_t n) {
  using mshadow::Shape1;
  using mshadow::Tensor;
  auto* g = reinterpret_cast<mxnet::common::random::RandGenerator<gpu, OType>*>(gen);
  Tensor<gpu, 1, IType> ta(static_cast<IType*>(const_cast<void*>(a)), Shape1(nparm), s);
  Tensor<gpu, 1, IType> tb(static_cast<IType*>(const_cast<void*>(b)), Shape1(nparm), s);
  Tensor<gpu, 1, OType> to(static_cast<OType*>(out), Shape1(n), s);
  switch (dist) {
    case kUniform: mxnet::op::UniformSampler<gpu>().Sample(ta, tb, to, g, s); break;
    case kNormal: mxnet::op::NormalSampler<gpu>().Sample(ta, tb, to, g, s); break;
    case kGamma: mxnet::op::GammaSampler<gpu>().Sample(ta, tb, to, g, s); break;
    case kExponential: mxnet::op::ExponentialSampler<gpu>().Sample(ta, to, g, s); break;
  }
}

template <typename IType>
int SampleAnyOut(int dist, int otype, mshadow::Stream<gpu>* s, GenF* gen, const void* a, const void* b,
                 int64_t nparm, void* out, int64_t n) {
  switch (otype) {
    case 0: Sample<IType, float>(dist, s, gen, a, b, nparm, out, n); return 0;
    case 1: Sample<IType, double>(dist, s, gen, a, b, nparm, out, n); return 0;
    case 2: Sample<IType, half_t>(dist, s, gen, a, b, nparm, out, n); return 0;
    default: return -1;
  }
}

int SampleAny(int dist, int ptype, int otype, mshadow::Stream<gpu>* s, GenF* gen, const void* a, const void* b,
              int64_t nparm, void* out, int64_t n) {
  switch (ptype) {
    case 0: return SampleAnyOut<float>(dist, otype, s, gen, a, b, nparm, out, n);
    case 1: return SampleAnyOut<double>(dist, otype, s, gen, a, b, nparm, out, n);
    case 2: return SampleAnyOut<half_t>(dist, otype, s, gen, a, b, nparm, out, n);
    default: return -1;
  }
}

}  // namespace

extern "C" {

// The multi-sample draw of sampler dist (0 uniform, 1 normal, 2 gamma, 3 exponential; b unused) of n
// outputs of type flag otype from nparm parameters of type flag ptype (0 float32, 1 float64,
// 2 float16) at host_a, host_b, from the generator copy at host_states (advanced in place)
int mxref_multisample(int dist, void* host_states, int ptype, int otype, int64_t nparm, const void* host_a,
                      const void* host_b, int64_t n, void* host_out) {
  GenF gen;
  GenF::AllocState(&gen);
  cudaMemcpy(*StatesOf(&gen), host_states, kBytes, cudaMemcpyHostToDevice);
  const size_t pbytes = nparm * TypeSize(ptype), obytes = n * TypeSize(otype);
  void *a = nullptr, *b = nullptr, *out = nullptr;
  cudaMalloc(&a, pbytes);
  cudaMalloc(&b, pbytes);
  cudaMalloc(&out, obytes > 0 ? obytes : 1);
  cudaMemcpy(a, host_a, pbytes, cudaMemcpyHostToDevice);
  cudaMemcpy(b, host_b, pbytes, cudaMemcpyHostToDevice);
  mshadow::Stream<gpu> s;
  int rc = SampleAny(dist, ptype, otype, &s, &gen, a, b, nparm, out, n);
  rc = rc == 0 ? Check() : rc;
  if (n > 0) cudaMemcpy(host_out, out, obytes, cudaMemcpyDeviceToHost);
  cudaMemcpy(host_states, *StatesOf(&gen), kBytes, cudaMemcpyDeviceToHost);
  cudaFree(out);
  cudaFree(b);
  cudaFree(a);
  GenF::FreeState(&gen);
  return rc == 0 ? Check() : rc;
}

// the reference's launch alone: ms per call of sampler dist over n outputs from nparm parameters, all
// of them (a, b) = (host_a[0], host_b[0]) (one element each, of type flag ptype), the generator on
// the device, CUDA events around `reps` launches after `warmup`
int mxref_multisample_time(int dist, int ptype, int otype, int64_t nparm, const void* host_a, const void* host_b,
                           int64_t n, int warmup, int reps, float* ms) {
  GenF gen;
  GenF::AllocState(&gen);
  mshadow::Stream<gpu> s;
  gen.Seed(&s, 17);
  const size_t ts = TypeSize(ptype);
  std::vector<char> ha(nparm * ts), hb(nparm * ts);
  for (int64_t i = 0; i < nparm; ++i) {
    memcpy(&ha[i * ts], host_a, ts);
    memcpy(&hb[i * ts], host_b, ts);
  }
  void *a = nullptr, *b = nullptr, *out = nullptr;
  cudaMalloc(&a, ha.size());
  cudaMalloc(&b, hb.size());
  cudaMalloc(&out, n * TypeSize(otype));
  cudaMemcpy(a, ha.data(), ha.size(), cudaMemcpyHostToDevice);
  cudaMemcpy(b, hb.data(), hb.size(), cudaMemcpyHostToDevice);
  int rc = 0;
  for (int i = 0; i < warmup && rc == 0; ++i) rc = SampleAny(dist, ptype, otype, &s, &gen, a, b, nparm, out, n);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventRecord(e0, 0);
  for (int i = 0; i < reps && rc == 0; ++i) rc = SampleAny(dist, ptype, otype, &s, &gen, a, b, nparm, out, n);
  cudaEventRecord(e1, 0);
  rc = rc == 0 ? Check() : rc;
  cudaEventElapsedTime(ms, e0, e1);
  *ms /= reps;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(out);
  cudaFree(b);
  cudaFree(a);
  GenF::FreeState(&gen);
  return rc == 0 ? Check() : rc;
}

}  // extern "C"
