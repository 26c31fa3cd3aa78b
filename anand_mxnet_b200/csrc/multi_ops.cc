// multi_ops.cc -- host side of the multi-tensor optimizer operators (SURVEY 8f-f1), the
// `update_on_kvstore=False` half of the path: after the in-place all-reduce every GPU runs the
// optimizer on its replica with these operators (python/mxnet/optimizer/optimizer.py LARS :798-1055,
// LAMB :1251-1370; contrib AdamW). Kernels: multi_tensor_kernels.cu.
//
// Reference operator definitions (argument order, attributes, error texts):
//   multi_sum_sq                          src/operator/contrib/multi_sum_sq.cc:34-60
//   multi_lars                            src/operator/contrib/multi_lars.cc:35-53
//   _adamw_update, _mp_adamw_update       src/operator/contrib/adamw.cc:34-141
//   _multi_adamw_update, _multi_mp_...    src/operator/contrib/adamw.cc:143-255
//   lamb_update_phase1/2, mp_lamb_...     src/operator/optimizer_op.cc:926-1095
//   _multi_lamb_update, _multi_mp_...     src/operator/contrib/multi_lamb.cc:174-251
#include <cmath>
#include <cstring>
#include <memory>
#include <unordered_map>

#include "kernels.h"
#include "op_params.h"
#include "ops.h"

namespace b200kv {
namespace {

struct MTPlan {
  int dev = -1;
  void *d_tensors = nullptr, *d_chunks = nullptr, *d_part = nullptr;
  size_t bt = 0, bc = 0, bp = 0;
  int n_chunks = 0, n_tensors = 0;
  ~MTPlan() {
    Engine* e = Engine::Get();
    e->Free(dev, d_tensors, bt);
    e->Free(dev, d_chunks, bc);
    e->Free(dev, d_part, bp);
  }
};

std::unordered_map<uint64_t, std::shared_ptr<MTPlan>>& Plans() {
  static auto* m = new std::unordered_map<uint64_t, std::shared_ptr<MTPlan>>();
  return *m;
}

uint64_t Mix(uint64_t h, uint64_t v) { return h ^ (v + 0x9e3779b97f4a7c15ULL + (h << 6) + (h >> 2)); }

bool Aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

// One group (<= kMTMaxTensors tensors) of one operator call: device tables cached by the
// operands' addresses, like the dense kernel's plans.
std::shared_ptr<MTPlan> GetPlan(int dev, int op, std::vector<MTTensor>* tensors, int n_partials,
                                cudaStream_t st) {
  uint64_t sig = Mix(0x4d54, static_cast<uint64_t>(op) * 131 + n_partials);
  for (auto& t : *tensors) {
    for (void* p : t.p) sig = Mix(sig, reinterpret_cast<uint64_t>(p));
    sig = Mix(sig, (static_cast<uint64_t>(t.size) << 32) | t.aux);
  }
  auto& cache = Plans();
  auto it = cache.find(sig);
  if (it != cache.end()) return it->second;
  if (cache.size() > 512) cache.clear();
  Engine* eng = Engine::Get();
  auto plan = std::make_shared<MTPlan>();
  plan->dev = dev;
  std::vector<MTChunk> chunks;
  for (size_t i = 0; i < tensors->size(); ++i) {
    MTTensor& t = (*tensors)[i];
    t.first_chunk = static_cast<uint32_t>(chunks.size());
    for (uint32_t off = 0; off < t.size; off += kMTChunk) {
      chunks.push_back(MTChunk{static_cast<uint32_t>(i), off, std::min<uint32_t>(kMTChunk, t.size - off), 0});
    }
  }
  plan->n_tensors = static_cast<int>(tensors->size());
  plan->n_chunks = static_cast<int>(chunks.size());
  plan->bt = tensors->size() * sizeof(MTTensor);
  plan->bc = std::max<size_t>(chunks.size(), 1) * sizeof(MTChunk);
  plan->bp = std::max<size_t>(chunks.size(), 1) * sizeof(float) * std::max(n_partials, 1);
  plan->d_tensors = eng->Alloc(dev, plan->bt);
  plan->d_chunks = eng->Alloc(dev, plan->bc);
  plan->d_part = eng->Alloc(dev, plan->bp);
  KV_CUDA(cudaMemcpyAsync(plan->d_tensors, tensors->data(), plan->bt, cudaMemcpyHostToDevice, st));
  if (!chunks.empty()) {
    KV_CUDA(cudaMemcpyAsync(plan->d_chunks, chunks.data(), chunks.size() * sizeof(MTChunk),
                            cudaMemcpyHostToDevice, st));
  }
  cache[sig] = plan;
  return plan;
}

struct Call {
  int op = 0, dtype = kFloat32, dev = -1;
  bool mp = false;
  std::vector<MTTensor> tensors;
  std::vector<float4> per_tensor;   // scalars of tensor i (may be empty)
  float f[12] = {0};
  const float *d0 = nullptr, *d1 = nullptr;
  int n_partials = 0;               // 0: elementwise, 1 or 2: sums of squares
  float *out0 = nullptr, *out1 = nullptr;
  std::vector<NDArray> reads, writes;
};

void Run(Call& c) {
  KV_CHECK(!c.tensors.empty());
  Engine* eng = Engine::Get();
  LaneOp op(c.dev);
  cudaStream_t st = op.stream();
  for (auto& a : c.reads) {
    KV_CHECK(a.on_gpu() && a.dev() == c.dev) << "all operands must be on the same GPU (no CPU fallback)";
    op.Read(a);
  }
  for (auto& a : c.writes) {
    KV_CHECK(a.on_gpu() && a.dev() == c.dev) << "all operands must be on the same GPU (no CPU fallback)";
    op.Write(a);
  }
  for (size_t g0 = 0; g0 < c.tensors.size(); g0 += kMTMaxTensors) {
    const size_t g1 = std::min(c.tensors.size(), g0 + kMTMaxTensors);
    std::vector<MTTensor> group(c.tensors.begin() + g0, c.tensors.begin() + g1);
    auto plan = GetPlan(c.dev, c.op, &group, c.n_partials, st);
    MTLaunch L;
    L.op = c.op;
    L.dtype = c.dtype;
    L.mp = c.mp;
    L.tensors = static_cast<const MTTensor*>(plan->d_tensors);
    L.chunks = static_cast<const MTChunk*>(plan->d_chunks);
    L.n_chunks = plan->n_chunks;
    std::memset(&L.s, 0, sizeof(L.s));
    for (size_t i = g0; i < g1 && i < c.per_tensor.size(); ++i) L.s.t[i - g0] = c.per_tensor[i];
    std::memcpy(L.s.f, c.f, sizeof(c.f));
    L.s.d0 = c.d0;
    L.s.d1 = c.d1;
    if (c.n_partials >= 1) L.part0 = static_cast<float*>(plan->d_part);
    if (c.n_partials >= 2) L.part1 = static_cast<float*>(plan->d_part) + std::max(plan->n_chunks, 1);
    LaunchMultiTensor(L, st);
    eng->CountLaunch("multi_tensor", 0);
    if (c.n_partials >= 1) {
      LaunchMultiTensorFinalize(L.tensors, plan->n_tensors, L.part0, L.part1, c.out0, c.out1, st);
      eng->CountLaunch("multi_tensor_finalize", 0);
    }
  }
  op.Issue();
}

MTTensor Tensor(std::initializer_list<const NDArray*> arrs, size_t size, uint32_t aux, int dtype) {
  MTTensor t;
  std::memset(&t, 0, sizeof(t));
  KV_CHECK(size < (1ULL << 32)) << "tensors of 2^32 or more elements are not supported";
  t.size = static_cast<uint32_t>(size);
  t.aux = aux;
  bool ok = true;
  int i = 0;
  for (const NDArray* a : arrs) {
    if (a != nullptr && !a->is_none()) {
      t.p[i] = a->data();
      const size_t need = a->dtype() == kFloat32 ? 16 : (DTypeSize(a->dtype()) == 2 ? 8 : 16);
      ok = ok && Aligned(t.p[i], need);
    }
    ++i;
  }
  (void)dtype;
  t.vec_ok = ok ? 1u : 0u;
  return t;
}

void CheckF32(const NDArray& a, size_t size, const char* what, const std::string& op) {
  KV_CHECK_EQ(a.dtype(), kFloat32) << op << ": " << what << " must be float32";
  KV_CHECK_EQ(a.Size(), size) << op << ": " << what << " shape mismatch";
}

NDArray OutOr(std::vector<NDArray>* outputs, size_t i, const std::vector<int64_t>& shape, Context ctx,
              int dtype) {
  if (outputs->size() > i) return (*outputs)[i];
  NDArray o(shape, ctx, dtype);
  outputs->push_back(o);
  return o;
}

// the front-end passes out=weight; a distinct out receives the weight first (then updated in place)
NDArray InPlace(const std::vector<NDArray>& in, size_t widx, std::vector<NDArray>* outputs, size_t oidx) {
  NDArray o = OutOr(outputs, oidx, in[widx].shape(), in[widx].ctx(), in[widx].dtype());
  if (!o.SameStorage(in[widx])) CopyFromTo(in[widx], o);
  return o;
}

float Required(const Params& p, const char* key, const std::string& op) {
  KV_CHECK(Find(p, key) != nullptr) << "Required parameter " << key << " of " << op << " is missing";
  return GetF(p, key, 0.f);
}

void CheckMP(const NDArray& w, bool mp, const std::string& op) {
  if (mp) {
    KV_CHECK(DTypeSize(w.dtype()) == 2 && w.dtype() != kInt8)
        << op << ": the multi-precision form expects 16-bit weights";
  } else {
    KV_CHECK_EQ(w.dtype(), kFloat32)
        << op << ": 16-bit weights without an fp32 master copy are not supported on this path "
        << "(use the mp_ / multi_precision form)";
  }
}

}  // namespace

bool MultiTensorOp(const std::string& n, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                   const Params& p) {
  // ------------------------------------------------------------------------------- multi_sum_sq
  if (n == "multi_sum_sq") {
    const int num = GetI(p, "num_arrays", -1);
    KV_CHECK(num >= 1) << "Required parameter num_arrays of multi_sum_sq is missing";
    KV_CHECK_EQ(static_cast<int>(in.size()), num) << "multi_sum_sq: expected num_arrays inputs";
    Call c;
    c.op = kMTSumSq;
    c.dtype = in[0].dtype();
    c.dev = in[0].dev();
    KV_CHECK(in[0].on_gpu()) << "multi_sum_sq runs on GPU arrays only (no CPU fallback)";
    NDArray out = OutOr(outputs, 0, {num}, in[0].ctx(), kFloat32);
    CheckF32(out, num, "out", n);
    for (int i = 0; i < num; ++i) {
      KV_CHECK_EQ(in[i].dtype(), c.dtype) << "multi_sum_sq: array_" << i << " dtype differs from array_0";
      c.tensors.push_back(Tensor({&in[i]}, in[i].Size(), i, c.dtype));
      c.reads.push_back(in[i]);
    }
    c.n_partials = 1;
    c.out0 = static_cast<float*>(out.data());
    c.writes.push_back(out);
    Run(c);
    return true;
  }
  // --------------------------------------------------------------------------------- multi_lars
  if (n == "multi_lars") {
    KV_CHECK_EQ(in.size(), 4u) << "multi_lars expects lrs, weights_sum_sq, grads_sum_sq, wds";
    if (in[0].dtype() != kFloat32) KV_FATAL << "MultiLARS only support float";
    const size_t cnt = in[1].Size();
    for (int i = 0; i < 4; ++i) CheckF32(in[i], cnt, "input", n);
    NDArray out = OutOr(outputs, 0, in[0].shape(), in[0].ctx(), kFloat32);
    CheckF32(out, cnt, "out", n);
    const float eta = Required(p, "eta", n), eps = Required(p, "eps", n);
    const float rescale = GetF(p, "rescale_grad", 1.0f);
    KV_CHECK(in[0].on_gpu()) << "multi_lars runs on GPU arrays only (no CPU fallback)";
    LaneOp op(in[0].dev());
    op.Read(in[0]).Read(in[1]).Read(in[2]).Read(in[3]).Write(out);
    LaunchMultiLars(static_cast<int>(cnt), static_cast<float*>(out.data()),
                    static_cast<const float*>(in[0].data()), static_cast<const float*>(in[1].data()),
                    static_cast<const float*>(in[2].data()), static_cast<const float*>(in[3].data()),
                    eta, eps, rescale, op.stream());
    Engine::Get()->CountLaunch("multi_lars", 0);
    op.Issue();
    return true;
  }
  // --------------------------------------------------------------------- adamw (single + multi)
  if (n == "_adamw_update" || n == "_mp_adamw_update" || n == "_multi_adamw_update" ||
      n == "_multi_mp_adamw_update") {
    const bool multi = n.find("_multi_") == 0;
    const bool mp = n.find("_mp_") != std::string::npos;
    const int stride = mp ? 5 : 4;
    const int num = multi ? GetI(p, "num_weights", 1) : 1;
    KV_CHECK_EQ(static_cast<int>(in.size()), num * stride + 1)
        << n << ": expected " << (multi ? "num_weights*" : "") << stride << " + 1 inputs";
    const NDArray& rescale = in[num * stride];
    CheckF32(rescale, 1, "rescale_grad", n);
    std::vector<float> lrs, wds, etas;
    if (multi) {
      lrs = GetTuple(p, "lrs");
      wds = GetTuple(p, "wds");
      etas = GetTuple(p, "etas");
      KV_CHECK_EQ(static_cast<int>(lrs.size()), num)
          << "Number of learning rates is inconsistent with num_weights parameter passed. Expected "
          << "number of learning rates: " << num << ", and got " << lrs.size();
      KV_CHECK_EQ(static_cast<int>(wds.size()), num)
          << "Number of weight decays is inconsistent with num_weights parameter passed. Expected "
          << "number of weight decays: " << num << ", and got " << wds.size();
      KV_CHECK_EQ(static_cast<int>(etas.size()), num)
          << "Number of learning rates schedule multiplier is inconsistent with num_weights "
          << "parameter passed. Expected number of learning rates schedule multiplier: " << num
          << ", and got " << etas.size();
    } else {
      lrs = {Required(p, "lr", n)};
      etas = {Required(p, "eta", n)};
      wds = {GetF(p, "wd", 0.f)};
    }
    Call c;
    c.op = multi ? kMTMultiAdamW : kMTAdamW;
    c.mp = mp;
    c.dtype = in[0].dtype();
    KV_CHECK(in[0].on_gpu()) << n << " runs on GPU arrays only (no CPU fallback)";
    c.dev = in[0].dev();
    CheckMP(in[0], mp, n);
    c.f[0] = GetF(p, "clip_gradient", -1.0f);
    c.f[1] = GetF(p, "beta1", 0.9f);
    c.f[2] = GetF(p, "beta2", 0.999f);
    c.f[3] = GetF(p, "epsilon", 1e-8f);
    c.d0 = static_cast<const float*>(rescale.data());
    c.reads.push_back(rescale);
    for (int i = 0; i < num; ++i) {
      const NDArray& w = in[i * stride];
      const NDArray& g = in[i * stride + 1];
      const NDArray& mean = in[i * stride + 2];
      const NDArray& var = in[i * stride + 3];
      KV_CHECK_EQ(w.dtype(), c.dtype) << n << ": all weights must share a dtype";
      KV_CHECK_EQ(g.dtype(), c.dtype) << n << ": weight / grad dtype mismatch";
      KV_CHECK_EQ(g.Size(), w.Size()) << n << ": weight / grad shape mismatch";
      CheckF32(mean, w.Size(), "mean", n);
      CheckF32(var, w.Size(), "var", n);
      NDArray out = InPlace(in, i * stride, outputs, i);
      NDArray w32;
      if (mp) {
        w32 = in[i * stride + 4];
        CheckF32(w32, w.Size(), "weight32", n);
      }
      c.tensors.push_back(Tensor({&w, &g, &mean, &var, mp ? &w32 : nullptr, &out}, w.Size(), i, c.dtype));
      c.per_tensor.push_back(make_float4(lrs[i], wds[i], etas[i], 0.f));
      if (!out.SameStorage(w)) c.reads.push_back(w);
      // _adamw_update rewrites grad with the rescaled gradient (reference side effect)
      if (!mp && !multi) c.writes.push_back(g); else c.reads.push_back(g);
      c.writes.push_back(mean);
      c.writes.push_back(var);
      c.writes.push_back(out);
      if (mp) c.writes.push_back(w32);
    }
    Run(c);
    return true;
  }
  // ------------------------------------------------------------------------- lamb phase 1 / 2
  if (n == "lamb_update_phase1" || n == "mp_lamb_update_phase1") {
    const bool mp = n[0] == 'm';
    KV_CHECK_EQ(in.size(), mp ? 5u : 4u) << n << ": wrong number of inputs";
    const NDArray &w = in[0], &g = in[1], &mean = in[2], &var = in[3];
    KV_CHECK(w.on_gpu()) << n << " runs on GPU arrays only (no CPU fallback)";
    CheckMP(w, mp, n);
    KV_CHECK_EQ(g.dtype(), w.dtype()) << n << ": weight / grad dtype mismatch";
    KV_CHECK_EQ(g.Size(), w.Size()) << n << ": weight / grad shape mismatch";
    CheckF32(mean, w.Size(), "mean", n);
    CheckF32(var, w.Size(), "var", n);
    NDArray out = OutOr(outputs, 0, w.shape(), w.ctx(), kFloat32);
    CheckF32(out, w.Size(), "out", n);
    KV_CHECK(Find(p, "t") != nullptr) << "Required parameter t of " << n << " is missing";
    const int t = GetI(p, "t", 0);
    const float beta1 = GetF(p, "beta1", 0.9f), beta2 = GetF(p, "beta2", 0.999f);
    Call c;
    c.op = kMTLambPhase1;
    c.mp = mp;
    c.dtype = w.dtype();
    c.dev = w.dev();
    c.f[0] = GetF(p, "clip_gradient", -1.0f);
    c.f[1] = GetF(p, "rescale_grad", 1.0f);
    c.f[2] = beta1;
    // DType(std::pow(param.beta1, param.t)): float base, int exponent -> pow in double
    c.f[3] = static_cast<float>(std::pow(static_cast<double>(beta1), static_cast<double>(t)));
    c.f[4] = beta2;
    c.f[5] = static_cast<float>(std::pow(static_cast<double>(beta2), static_cast<double>(t)));
    c.f[6] = Required(p, "wd", n);
    c.f[7] = GetF(p, "epsilon", 1e-6f);
    c.f[8] = GetB(p, "bias_correction", true) ? 1.f : 0.f;
    NDArray w32;
    if (mp) {
      w32 = in[4];
      CheckF32(w32, w.Size(), "weight32", n);
      c.reads.push_back(w32);
    }
    c.tensors.push_back(Tensor({&w, &g, &mean, &var, mp ? &w32 : nullptr, &out}, w.Size(), 0, c.dtype));
    c.reads.push_back(w);
    c.reads.push_back(g);
    c.writes.push_back(mean);
    c.writes.push_back(var);
    c.writes.push_back(out);
    Run(c);
    return true;
  }
  if (n == "lamb_update_phase2" || n == "mp_lamb_update_phase2") {
    const bool mp = n[0] == 'm';
    KV_CHECK_EQ(in.size(), mp ? 5u : 4u) << n << ": wrong number of inputs";
    const NDArray &w = in[0], &g = in[1], &r1 = in[2], &r2 = in[3];
    KV_CHECK(w.on_gpu()) << n << " runs on GPU arrays only (no CPU fallback)";
    CheckMP(w, mp, n);
    CheckF32(g, w.Size(), "g", n);
    CheckF32(r1, 1, "r1", n);
    CheckF32(r2, 1, "r2", n);
    NDArray out = OutOr(outputs, 0, w.shape(), w.ctx(), w.dtype());
    KV_CHECK_EQ(out.dtype(), w.dtype()) << n << ": out dtype mismatch";
    KV_CHECK_EQ(out.Size(), w.Size()) << n << ": out shape mismatch";
    Call c;
    c.op = kMTLambPhase2;
    c.mp = mp;
    c.dtype = w.dtype();
    c.dev = w.dev();
    c.f[0] = Required(p, "lr", n);
    c.f[1] = GetF(p, "lower_bound", -1.0f);
    c.f[2] = GetF(p, "upper_bound", -1.0f);
    c.d0 = static_cast<const float*>(r1.data());
    c.d1 = static_cast<const float*>(r2.data());
    NDArray w32;
    if (mp) {
      w32 = in[4];
      CheckF32(w32, w.Size(), "weight32", n);
      c.reads.push_back(w32);
    }
    c.tensors.push_back(Tensor({&w, &g, nullptr, nullptr, mp ? &w32 : nullptr, &out}, w.Size(), 0, c.dtype));
    if (!out.SameStorage(w)) c.reads.push_back(w);
    c.reads.push_back(g);
    c.reads.push_back(r1);
    c.reads.push_back(r2);
    c.writes.push_back(out);
    Run(c);
    return true;
  }
  // ------------------------------------------------------------------------------- multi lamb
  if (n == "_multi_lamb_update" || n == "_multi_mp_lamb_update") {
    const bool mp = n.find("_mp_") != std::string::npos;
    const int stride = mp ? 5 : 4;
    const int num = GetI(p, "num_tensors", 1);
    KV_CHECK(num <= 45) << "Invalid number of tensors, the maximum value is 45, and got " << num;
    KV_CHECK_EQ(static_cast<int>(in.size()), num * stride) << n << ": expected num_tensors*" << stride << " inputs";
    std::vector<float> lrs = GetTuple(p, "learning_rates"), wds = GetTuple(p, "wds");
    std::vector<int> steps = GetIntTuple(p, "step_count");
    KV_CHECK_EQ(static_cast<int>(lrs.size()), num)
        << "Number of learning rates is inconsistent with num_tensors parameter passed. Expected "
        << "number of learning rates: " << num << ", and got " << lrs.size();
    KV_CHECK_EQ(static_cast<int>(wds.size()), num)
        << "Number of weight decays is inconsistent with num_tensors parameter passed. Expected "
        << "number of weight decays: " << num << ", and got " << wds.size();
    KV_CHECK_EQ(static_cast<int>(steps.size()), num)
        << "Number of step counts is inconsistent with num_tensors.Expected number of step counts: "
        << num << ", and got " << steps.size();
    KV_CHECK(in[0].on_gpu()) << n << " runs on GPU arrays only (no CPU fallback)";
    const int dev = in[0].dev();
    const int dtype = in[0].dtype();
    CheckMP(in[0], mp, n);
    const float beta1 = GetF(p, "beta1", 0.9f), beta2 = GetF(p, "beta2", 0.999f);
    size_t total = 0;
    for (int i = 0; i < num; ++i) total += (in[i * stride].Size() + 3) & ~static_cast<size_t>(3);
    NDArray temp_g({static_cast<int64_t>(std::max<size_t>(total, 1))}, Context::GPU(dev), kFloat32);
    NDArray sums({static_cast<int64_t>(2 * num)}, Context::GPU(dev), kFloat32);  // [w^2 | temp_g^2]
    Call s1, s2;
    s1.op = kMTMultiLambStep1;
    s2.op = kMTMultiLambStep2;
    s1.mp = s2.mp = mp;
    s1.dtype = s2.dtype = dtype;
    s1.dev = s2.dev = dev;
    s1.f[0] = GetF(p, "clip_gradient", -1.0f);
    s1.f[1] = GetF(p, "rescale_grad", 1.0f);
    s1.f[2] = beta1;
    s1.f[3] = beta2;
    s1.f[4] = GetF(p, "epsilon", 1e-6f);
    s1.f[5] = GetB(p, "bias_correction", true) ? 1.f : 0.f;
    s1.n_partials = 2;
    s1.out0 = static_cast<float*>(sums.data());
    s1.out1 = static_cast<float*>(sums.data()) + num;
    s2.f[0] = GetF(p, "lower_bound", -1.0f);
    s2.f[1] = GetF(p, "upper_bound", -1.0f);
    s2.d0 = s1.out0;
    s2.d1 = s1.out1;
    size_t off = 0;
    for (int i = 0; i < num; ++i) {
      const NDArray& w = in[i * stride];
      const NDArray& g = in[i * stride + 1];
      const NDArray& mean = in[i * stride + 2];
      const NDArray& var = in[i * stride + 3];
      KV_CHECK_EQ(w.dtype(), dtype) << n << ": all weights must share a dtype";
      KV_CHECK_EQ(g.dtype(), dtype) << n << ": weight / grad dtype mismatch";
      KV_CHECK_EQ(g.Size(), w.Size()) << n << ": weight / grad shape mismatch";
      CheckF32(mean, w.Size(), "mean", n);
      CheckF32(var, w.Size(), "var", n);
      NDArray out = InPlace(in, i * stride, outputs, i);
      NDArray w32;
      if (mp) {
        w32 = in[i * stride + 4];
        CheckF32(w32, w.Size(), "weight32", n);
      }
      MTTensor t = Tensor({&out, &g, &mean, &var, mp ? &w32 : nullptr, nullptr}, w.Size(), i, dtype);
      t.p[5] = static_cast<float*>(temp_g.data()) + off;
      off += (w.Size() + 3) & ~static_cast<size_t>(3);
      s1.tensors.push_back(t);
      s2.tensors.push_back(t);
      // 1 - powf(beta, step): evaluated with the host C library, as the reference's CPU kernel does
      const float c1 = 1.0f - std::pow(beta1, static_cast<float>(steps[i]));
      const float c2 = 1.0f - std::pow(beta2, static_cast<float>(steps[i]));
      s1.per_tensor.push_back(make_float4(lrs[i], wds[i], c1, c2));
      s2.per_tensor.push_back(make_float4(lrs[i], wds[i], c1, c2));
      s1.reads.push_back(out);
      s1.reads.push_back(g);
      s1.writes.push_back(mean);
      s1.writes.push_back(var);
      s2.writes.push_back(out);
      if (mp) {
        s1.reads.push_back(w32);
        s2.writes.push_back(w32);
      }
    }
    s1.writes.push_back(temp_g);
    s1.writes.push_back(sums);
    s2.reads.push_back(temp_g);
    s2.reads.push_back(sums);
    Run(s1);
    Run(s2);
    return true;
  }
  return false;
}

}  // namespace b200kv
