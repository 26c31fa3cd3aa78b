// random_ops.cc -- the GPU parallel random generators (ResourceParallelRandom<gpu>, resource.cc:
// 205-360), their seeding (MXRandomSeed / MXRandomSeedContext), the draw path every sampler takes
// (SampleInto), and the sampling operator _random_normal (random/sample_op.cc, SampleNormalParam and
// normal_op in sample_op.h). The other samplers' operators are in sample_ops.cc.
//
// Each GPU holds kRandCopies copies of kRandStates Philox states, allocated and seeded on its first
// sampling call or per-device seed. Copy i is seeded with dev + i*16 + global_seed*127 (global seed
// 0 until MXRandomSeed); MXRandomSeedContext seeds i*16 + seed*127, without the device term. Each
// sampling call takes copy ++curr_ptr % kRandCopies (GetNext pre-increments, so the first call after
// a seed takes copy 1). Every copy is an engine variable: a seed or a draw is a write to it on the
// GPU's compute lane, so calls, seeds and state reads stay in issue order.
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>

#include "engine.h"
#include "kernels.h"
#include "ops.h"
#include "random_ops.h"

namespace b200kv {
namespace {

constexpr int kRandCopies = 4;     // MXNET_GPU_PARALLEL_RAND_COPY's default
constexpr uint32_t kMaxNumGPUs = 16;
constexpr uint32_t kRandMagic = 127;
constexpr size_t kCopyBytes = static_cast<size_t>(kRandStates) * kRandStateBytes;

struct DevRandom {
  void* states[kRandCopies] = {};
  Var var[kRandCopies];
  size_t curr_ptr = 0;
};

uint32_t g_global_seed = 0;
DevRandom g_rand[kMaxDevices];

void SeedCopy(int dev, int i, uint32_t seed) {
  DevRandom& R = g_rand[dev];
  LaneOp lop(dev);
  lop.Write(&R.var[i]);
  LaunchRandSeed(R.states[i], seed, lop.stream());
  Engine::Get()->CountLaunch("rand_seed", kCopyBytes);
  lop.Issue();
}

// the device's copies, allocated and seeded with the global seed on first use
DevRandom& Generators(int dev) {
  KV_CHECK(dev >= 0 && dev < kMaxDevices) << "invalid GPU id " << dev;
  DevRandom& R = g_rand[dev];
  if (R.states[0] == nullptr) {
    DeviceGuard g(dev);
    for (int i = 0; i < kRandCopies; ++i) KV_CUDA(cudaMalloc(&R.states[i], kCopyBytes));
    for (int i = 0; i < kRandCopies; ++i) {
      SeedCopy(dev, i, static_cast<uint32_t>(dev) + i * kMaxNumGPUs + g_global_seed * kRandMagic);
    }
  }
  return R;
}

void RandomNormal(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                  const Params& p) {
  const char* n = op.name;
  RejectUnknownKeys(p, {"loc", "scale", "shape", "ctx", "dtype"});
  KV_CHECK(in.empty()) << n << " takes no inputs";
  const float loc = GetF(p, "loc", 0.0f);
  const float scale = GetF(p, "scale", 1.0f);
  const SampleTarget t = ParseSampleTarget(n, p, *outputs, false);
  KV_CHECK(scale > 0) << "scale parameter in gaussian has to be positive";
  NDArray o = OutOr(outputs, 0, t.shape, t.ctx, t.dtype);
  RandNormalInto(o, loc, scale, true);
}

}  // namespace

// "gpu(1)", "cpu(0)", "cpu_pinned(0)" (Context::FromString); an empty string is the CPU
Context ParseCtx(const std::string& s, const char* op) {
  if (s.empty()) return Context::CPU();
  const size_t open = s.find('(');
  KV_CHECK(open != std::string::npos && s.back() == ')') << op << ": invalid context '" << s << "'";
  const std::string type = s.substr(0, open);
  const int id = std::atoi(s.c_str() + open + 1);
  if (type == "gpu") return Context{kGPU, id};
  KV_CHECK(type == "cpu" || type == "cpu_pinned" || type == "cpu_shared") << op << ": invalid context '" << s << "'";
  return Context::CPU();
}

// TShape "(2, 3)", "[2, 3]", "(5,)", "5" or "()"
std::vector<int64_t> ParseShape(const std::string& s, const char* op) {
  std::vector<int64_t> out;
  const char* p = s.c_str();
  while (*p) {
    if (*p == '(' || *p == ')' || *p == '[' || *p == ']' || *p == ',' || *p == ' ' || *p == 'L') {
      ++p;
      continue;
    }
    char* end = nullptr;
    const long long v = std::strtoll(p, &end, 10);
    KV_CHECK(end != p && v >= 0) << op << ": invalid shape '" << s << "'";
    out.push_back(v);
    p = end;
  }
  return out;
}

int ParseDType(const std::string& s, const char* op, bool integer) {
  if (s == "None") return -1;
  if (integer) {
    if (s == "int32") return kInt32;
    if (s == "int64") return kInt64;
    KV_FATAL << op << ": Invalid Input: '" << s << "', valid values are: {'None', 'int32', 'int64'}";
  }
  if (s == "float32") return kFloat32;
  if (s == "float64") return kFloat64;
  if (s == "float16") return kFloat16;
  if (s == "bfloat16") return kBfloat16;
  KV_FATAL << op << ": Invalid Input: '" << s << "', valid values are: {'None', 'bfloat16', 'float16', "
           << "'float32', 'float64'}";
  return -1;
}

SampleTarget ParseSampleTarget(const char* n, const Params& p, const std::vector<NDArray>& outputs,
                               bool integer) {
  const std::string* shape_s = Find(p, "shape");
  const std::string* dtype_s = Find(p, "dtype");
  const std::string* ctx_s = Find(p, "ctx");
  const bool has_shape = shape_s != nullptr && !ParseShape(*shape_s, n).empty();
  SampleTarget t;
  if (has_shape) t.shape = ParseShape(*shape_s, n);
  t.dtype = dtype_s != nullptr ? ParseDType(*dtype_s, n, integer) : -1;
  t.ctx = ParseCtx(ctx_s != nullptr ? *ctx_s : "", n);
  if (!outputs.empty()) {
    // the output's context, shape and dtype decide; a given shape or dtype must agree with them
    const NDArray& o = outputs[0];
    KV_CHECK(o.stype() == kDefaultStorage) << n << ": out must be a dense array; got " << StypeName(o.stype());
    KV_CHECK(!has_shape || o.shape() == t.shape) << n << ": out has the wrong shape";
    KV_CHECK(t.dtype == -1 || o.dtype() == t.dtype) << n << ": out dtype " << DTypeName(o.dtype())
                                                    << " differs from dtype " << DTypeName(t.dtype);
    t.shape = o.shape();
    t.dtype = o.dtype();
    t.ctx = o.ctx();
  } else {
    KV_CHECK(has_shape) << n << ": shape is required when no out is given";
  }
  if (t.dtype == -1) t.dtype = integer ? kInt32 : kFloat32;
  CheckSampleDType(n, t.dtype, integer);
  KV_CHECK(t.ctx.dev_type == kGPU) << n << " samples on the GPU only (the reference's CPU generator is a "
                                   << "different stream)";
  return t;
}

void CheckSampleDType(const char* n, int dtype, bool integer) {
  if (integer) {
    KV_CHECK(dtype == kInt32 || dtype == kInt64) << n << ": int32 and int64 outputs only; got "
                                                 << DTypeName(dtype);
  } else {
    KV_CHECK(dtype == kFloat32 || dtype == kFloat64 || dtype == kFloat16 || dtype == kBfloat16)
        << n << ": float16, bfloat16, float32 and float64 outputs only; got " << DTypeName(dtype);
  }
}

void SampleInto(const NDArray& out, const char* launch_name,
                const std::function<void(void* states, cudaStream_t stream)>& launch,
                const std::vector<NDArray>& reads) {
  KV_CHECK(out.on_gpu() && out.stype() == kDefaultStorage) << launch_name << ": out must be a dense GPU array";
  const int dev = out.dev();
  DevRandom& R = Generators(dev);
  const size_t i = ++R.curr_ptr % kRandCopies;
  LaneOp lop(dev);
  for (const NDArray& a : reads) lop.Read(a);
  lop.Write(&R.var[i]).Write(out);
  launch(R.states[i], lop.stream());
  if (out.Size() > 0) Engine::Get()->CountLaunch(launch_name, out.Size() * DTypeSize(out.dtype()));
  lop.Issue();
}

void RandNormalInto(const NDArray& out, float loc, float scale, bool staged) {
  const uint64_t size = out.Size();
  SampleInto(out, "_random_normal", [&](void* states, cudaStream_t stream) {
    LaunchRandNormal(out.dtype(), states, size > 0 ? out.data() : nullptr, size, loc, scale, staged, stream);
  });
}

void RandomSeed(uint32_t seed) {
  g_global_seed = seed;
  for (int dev = 0; dev < kMaxDevices; ++dev) {
    DevRandom& R = g_rand[dev];
    if (R.states[0] == nullptr) continue;
    for (int i = 0; i < kRandCopies; ++i) {
      SeedCopy(dev, i, static_cast<uint32_t>(dev) + i * kMaxNumGPUs + seed * kRandMagic);
    }
    R.curr_ptr = 0;
  }
}

void RandomSeedContext(uint32_t seed, Context ctx) {
  if (ctx.dev_type != kGPU) return;  // no CPU generator here: CPU sampling is refused
  DevRandom& R = Generators(ctx.dev_id);
  for (int i = 0; i < kRandCopies; ++i) SeedCopy(ctx.dev_id, i, i * kMaxNumGPUs + seed * kRandMagic);
  R.curr_ptr = 0;
}

void RandomStates(int dev, int copy, void* host, size_t bytes) {
  KV_CHECK(copy >= 0 && copy < kRandCopies) << "generator copy " << copy << " out of range";
  KV_CHECK_EQ(bytes, kCopyBytes) << "a generator copy holds " << kCopyBytes << " bytes";
  DevRandom& R = Generators(dev);
  Engine::Get()->WaitToRead(R.var[copy]);
  DeviceGuard g(dev);
  KV_CUDA(cudaMemcpy(host, R.states[copy], bytes, cudaMemcpyDeviceToHost));
}

const std::vector<OpInfo> kRandomOps = {
    {"_random_normal", RandomNormal, 0},
};

}  // namespace b200kv
