// sample_param_ops.cc -- sampling with NDArray parameters (random/multisample_op.h, .cc, .cu):
// _sample_uniform(low, high), _sample_normal(mu, sigma), _sample_gamma(alpha, beta) and
// _sample_exponential(lam), with the reference's aliases sample_<name>, and _rdiv_scalar, which the
// reference's exponential(scale=NDArray) calls to pass lam = 1.0 / scale.
//
// The output has the parameters' shape followed by MultiSampleParam's shape, and element i draws with
// parameters i / nBatch. Each call takes the GPU's next generator copy through SampleInto, so these
// samplers and the scalar ones share one stream per GPU. Parameter values are not checked, as in the
// reference: a negative sigma or a low above high draws what the reference draws; a gamma element
// whose draw cannot end is NaN (random_kernels.cu, GammaOf). Every refusal comes before any
// generator is created or advanced.
#include <string>
#include <vector>

#include "kernels.h"
#include "ops.h"
#include "random_ops.h"

namespace b200kv {
namespace {

bool SampleParamDTypeOk(int t) { return t == kFloat16 || t == kFloat32 || t == kFloat64; }

// the bytes of a overlap those of b (both non-empty dense arrays)
bool Overlaps(const NDArray& a, const NDArray& b) {
  const char* a0 = static_cast<const char*>(a.data());
  const char* b0 = static_cast<const char*>(b.data());
  return a0 < b0 + b.ByteSize() && b0 < a0 + a.ByteSize();
}

// MultiSampleParam's dtype enum: None, float16, float32, float64 (-1 is None)
int MultiSampleDType(const Params& p, const char* n) {
  const std::string* s = Find(p, "dtype");
  const int t = s != nullptr ? ParseDType(*s, n) : -1;
  KV_CHECK(t != kBfloat16) << n << ": Invalid Input: 'bfloat16', valid values are: {'None', 'float16', "
                           << "'float32', 'float64'}";
  return t;
}

// _sample_uniform, _sample_normal, _sample_gamma (2 inputs) and _sample_exponential (1 input);
// variant: RandDist
void MultiSample(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                 const Params& p) {
  const char* n = op.name;
  RejectUnknownKeys(p, {"shape", "dtype"});
  const std::string* shape_s = Find(p, "shape");
  const std::vector<int64_t> sshape = shape_s != nullptr ? ParseShape(*shape_s, n) : std::vector<int64_t>();
  for (int64_t d : sshape) KV_CHECK(d > 0) << "shape parameter must be non-zero within each dimension";
  const int dtype = MultiSampleDType(p, n);
  const size_t nin = op.variant == kRandExponential ? 1 : 2;
  KV_CHECK(in.size() == nin) << n << " takes " << nin << (nin == 1 ? " input" : " inputs") << " ("
                             << in.size() << " given)";

  const NDArray& a0 = in[0];
  for (size_t i = 0; i < in.size(); ++i) {
    const NDArray& a = in[i];
    KV_CHECK(a.stype() == kDefaultStorage) << n << ": parameter " << i << " must be a dense array; got "
                                           << StypeName(a.stype());
    KV_CHECK(a.shape() == a0.shape()) << n << ": parameter " << i << " shape differs from parameter 0";
    KV_CHECK(a.dtype() == a0.dtype()) << n << ": parameter " << i << " dtype " << DTypeName(a.dtype())
                                      << " differs from parameter 0 dtype " << DTypeName(a0.dtype());
  }
  KV_CHECK(a0.Size() > 0) << n << ": the parameter arrays must not be empty";
  KV_CHECK(SampleParamDTypeOk(a0.dtype())) << n << ": parameter arrays of float16, float32 and float64 only; got "
                                           << DTypeName(a0.dtype())
                                           << " (integer and bfloat16 parameters are not supported)";

  std::vector<int64_t> oshape = a0.shape();
  oshape.insert(oshape.end(), sshape.begin(), sshape.end());
  int otype = dtype == -1 ? kFloat32 : dtype;
  if (!outputs->empty()) {
    const NDArray& o = (*outputs)[0];
    KV_CHECK(o.stype() == kDefaultStorage) << n << ": out must be a dense array; got " << StypeName(o.stype());
    KV_CHECK(o.shape() == oshape) << n << ": out has the wrong shape";
    KV_CHECK(dtype == -1 || o.dtype() == dtype) << "Inferred output type does not match requested type: "
                                                << DTypeName(o.dtype()) << " vs " << DTypeName(dtype);
    otype = o.dtype();
  }
  KV_CHECK(SampleParamDTypeOk(otype)) << "Output type must be float16, float32, or float64: dtype is "
                                      << DTypeName(otype);
  for (size_t i = 0; i < in.size(); ++i) {
    KV_CHECK(in[i].on_gpu()) << n << " samples on the GPU only (the reference's CPU generator is a different "
                             << "stream); parameter " << i << " is on " << in[i].ctx().str();
    KV_CHECK(in[i].dev() == a0.dev()) << n << ": all operands must be on the same GPU";
  }
  if (!outputs->empty()) {
    const NDArray& o = (*outputs)[0];
    KV_CHECK(o.on_gpu() && o.dev() == a0.dev()) << n << ": out must be on the parameters' GPU, "
                                                << a0.ctx().str() << "; it is on " << o.ctx().str();
    for (size_t i = 0; i < in.size(); ++i) {
      const bool same = o.data() == in[i].data() && o.ByteSize() == in[i].ByteSize() &&
                        o.dtype() == in[i].dtype();
      KV_CHECK(same || !Overlaps(o, in[i])) << n << ": out overlaps parameter " << i
                                            << " without being it";
    }
  }

  const NDArray o = OutOr(outputs, 0, oshape, a0.ctx(), otype);
  const int dist = op.variant;
  const uint64_t nparm = a0.Size();
  const uint64_t size = o.Size();
  const void* pa = a0.data();
  const void* pb = in.back().data();
  SampleInto(o, n, [&](void* states, cudaStream_t stream) {
    LaunchRandSampleParams(dist, a0.dtype(), otype, states, pa, pb, nparm, o.data(), size, stream);
  }, in);
}

// _rdiv_scalar: scalar / x (mshadow_op::rdiv), its scalar parsed as _div_scalar's (std::stod, then
// DType(alpha) in the kernel); floating dtypes only, as for _div_scalar
void RDivScalar(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                const Params& p) {
  KV_CHECK_EQ(in.size(), 1u) << op.name << " expects 1 input";
  const double scalar = StodD(p, "scalar", op.name);
  const int t = in[0].dtype();
  KV_CHECK(t == kFloat16 || t == kBfloat16 || t == kFloat32 || t == kFloat64)
      << op.name << ": integer division is not supported (" << DTypeName(t)
      << "); divide float16, bfloat16, float32 or float64 arrays";
  NDArray o = OutOr(outputs, 0, in[0].shape(), in[0].ctx(), t);
  Elementwise(kEwRDivScalar, in[0], nullptr, scalar, o);
}

}  // namespace

const std::vector<OpInfo> kSampleParamOps = {
    {"_sample_uniform", MultiSample, kRandUniform},
    {"sample_uniform", MultiSample, kRandUniform},
    {"_sample_normal", MultiSample, kRandNormal},
    {"sample_normal", MultiSample, kRandNormal},
    {"_sample_gamma", MultiSample, kRandGamma},
    {"sample_gamma", MultiSample, kRandGamma},
    {"_sample_exponential", MultiSample, kRandExponential},
    {"sample_exponential", MultiSample, kRandExponential},
    {"_rdiv_scalar", RDivScalar, 0},
};

}  // namespace b200kv
