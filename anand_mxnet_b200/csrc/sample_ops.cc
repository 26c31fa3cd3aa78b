// sample_ops.cc -- the scalar-parameter sampling operators of random/sample_op.cc besides
// _random_normal: _random_uniform, _random_exponential, _random_gamma and _random_randint, and the
// _like forms of uniform, normal, exponential and gamma (SampleUniformLikeParam and its siblings),
// which take shape, context and dtype from their input. Each call draws from its GPU's next
// generator copy through SampleInto (random_ops.cc), so all samplers share one stream per GPU as in
// the reference. Parameters are parsed as the reference's Param structs parse them (float fields:
// dmlc::stof; randint's int64 bounds: an integer literal) and checked as sample_op.h checks them,
// before any generator is created or advanced.
#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <string>

#include "kernels.h"
#include "ops.h"
#include "random_ops.h"

namespace b200kv {
namespace {

constexpr int kNormalLike = -1;  // the variant of _random_normal_like (RandNormalInto)

// SampleRandIntParam's int64 low / high
int64_t RequiredInt64(const Params& p, const char* key, const char* op) {
  const std::string v = Required<std::string>(p, key, op);
  char* end = nullptr;
  errno = 0;
  const long long x = std::strtoll(v.c_str(), &end, 10);
  KV_CHECK(end != v.c_str() && *end == '\0' && errno == 0) << op << ": invalid int64 " << key << "='" << v << "'";
  return x;
}

void RejectKeys(int dist, const Params& p, bool like) {
  switch (dist) {
    case kRandUniform:
      like ? RejectUnknownKeys(p, {"low", "high"}) : RejectUnknownKeys(p, {"low", "high", "shape", "ctx", "dtype"});
      break;
    case kRandExponential:
      like ? RejectUnknownKeys(p, {"lam"}) : RejectUnknownKeys(p, {"lam", "shape", "ctx", "dtype"});
      break;
    case kRandGamma:
      like ? RejectUnknownKeys(p, {"alpha", "beta"})
           : RejectUnknownKeys(p, {"alpha", "beta", "shape", "ctx", "dtype"});
      break;
    case kRandInt: RejectUnknownKeys(p, {"low", "high", "shape", "ctx", "dtype"}); break;
    case kNormalLike: RejectUnknownKeys(p, {"loc", "scale"}); break;
  }
}

// The distribution's parameters with their defaults, refused as uniform_op, exponential_op, gamma_op
// and rand_int_op refuse them (a NaN fails every check)
RandParams DistParams(int dist, const char* n, const Params& p) {
  RandParams r;
  switch (dist) {
    case kRandUniform:
      r.a = GetF(p, "low", 0.0f);
      r.b = GetF(p, "high", 1.0f);
      KV_CHECK(r.b >= r.a) << "low must be less or equal to high in uniform distribution";
      break;
    case kRandExponential:
      r.a = GetF(p, "lam", 1.0f);
      KV_CHECK(r.a > 0) << "lambda parameter in exponential distribution has to be positive";
      break;
    case kRandGamma:
      r.a = GetF(p, "alpha", 1.0f);
      r.b = GetF(p, "beta", 1.0f);
      KV_CHECK(r.a > 0) << "alpha parameter in gamma distribution has to be positive";
      KV_CHECK(r.b > 0) << "beta parameter in gamma distribution has to be positive";
      // this library's own check: the reference's draw never ends for alpha = +inf
      KV_CHECK(std::isfinite(r.a)) << n << ": alpha must be finite (the gamma draw does not end for alpha = inf)";
      break;
    case kRandInt: {
      r.lo = RequiredInt64(p, "low", n);
      r.hi = RequiredInt64(p, "high", n);
      KV_CHECK(r.hi >= r.lo) << "low must be less or equal to high in uniform distribution";
      // the reference draws x % (high - low): undefined for an empty range, and for a range past int64
      int64_t range = 0;
      KV_CHECK(r.hi > r.lo) << n << ": high must be greater than low (the range [low, high) is empty)";
      KV_CHECK(!__builtin_sub_overflow(r.hi, r.lo, &range)) << n << ": high - low must fit in int64";
      break;
    }
  }
  return r;
}

void Draw(int dist, const char* n, const NDArray& o, const RandParams& r) {
  const uint64_t size = o.Size();
  SampleInto(o, n, [&](void* states, cudaStream_t stream) {
    LaunchRandSample(dist, o.dtype(), states, size > 0 ? o.data() : nullptr, size, r, stream);
  });
}

// _random_uniform, _random_exponential, _random_gamma, _random_randint (variant: RandDist)
void RandomSample(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                  const Params& p) {
  const char* n = op.name;
  RejectKeys(op.variant, p, false);
  KV_CHECK(in.empty()) << n << " takes no inputs";
  const SampleTarget t = ParseSampleTarget(n, p, *outputs, op.variant == kRandInt);
  const RandParams r = DistParams(op.variant, n, p);
  Draw(op.variant, n, OutOr(outputs, 0, t.shape, t.ctx, t.dtype), r);
}

// _random_{uniform,normal,exponential,gamma}_like (variant: RandDist or kNormalLike): data's shape,
// context and dtype; data's values are not read, so out may be data itself
void RandomSampleLike(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                      const Params& p) {
  const char* n = op.name;
  RejectKeys(op.variant, p, true);
  KV_CHECK(in.size() == 1) << n << " takes one input, data";
  const NDArray& data = in[0];
  KV_CHECK(data.stype() == kDefaultStorage) << n << ": data must be a dense array; got " << StypeName(data.stype());
  if (!outputs->empty()) {
    const NDArray& o = (*outputs)[0];
    KV_CHECK(o.stype() == kDefaultStorage) << n << ": out must be a dense array; got " << StypeName(o.stype());
    KV_CHECK(o.shape() == data.shape()) << n << ": out has the wrong shape";
    KV_CHECK(o.dtype() == data.dtype()) << n << ": out dtype " << DTypeName(o.dtype()) << " differs from data dtype "
                                        << DTypeName(data.dtype());
    KV_CHECK(o.ctx() == data.ctx()) << n << ": out is on " << o.ctx().str() << ", data on " << data.ctx().str();
  }
  CheckSampleDType(n, data.dtype(), false);
  KV_CHECK(data.ctx().is_gpu()) << n << " samples on the GPU only (the reference's CPU generator is a "
                                << "different stream)";
  if (op.variant == kNormalLike) {
    const float loc = GetF(p, "loc", 0.0f);
    const float scale = GetF(p, "scale", 1.0f);
    KV_CHECK(scale > 0) << "scale parameter in gaussian has to be positive";
    RandNormalInto(OutOr(outputs, 0, data.shape(), data.ctx(), data.dtype()), loc, scale, true);
    return;
  }
  const RandParams r = DistParams(op.variant, n, p);
  Draw(op.variant, n, OutOr(outputs, 0, data.shape(), data.ctx(), data.dtype()), r);
}

}  // namespace

const std::vector<OpInfo> kSampleOps = {
    {"_random_uniform", RandomSample, kRandUniform},
    {"_random_exponential", RandomSample, kRandExponential},
    {"_random_gamma", RandomSample, kRandGamma},
    {"_random_randint", RandomSample, kRandInt},
    {"_random_uniform_like", RandomSampleLike, kRandUniform},
    {"_random_normal_like", RandomSampleLike, kNormalLike},
    {"_random_exponential_like", RandomSampleLike, kRandExponential},
    {"_random_gamma_like", RandomSampleLike, kRandGamma},
};

}  // namespace b200kv
