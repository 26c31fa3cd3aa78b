// ops.cc -- see ops.h.
#include "ops.h"

#include <algorithm>
#include <cstring>
#include <map>
#include <memory>
#include <unordered_map>

#include "kernels.h"
#include "op_params.h"
#include "rowsparse.h"
#include "scalar_parse.h"

namespace b200kv {

void PlanChunks(uint64_t goff, size_t size, uint32_t key_slot, int ndev, int owner_fixed,
                std::vector<std::vector<ChunkDesc>>* per_slot);  // kvstore.cc
// NAG / Signum / RMSProp / FTML / Ftrl / sparse AdaGrad / GroupAdaGrad operators; false when `name` is not one of them
bool UpdateOp(const std::string& name, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
              const Params& p);  // update_ops.cc

namespace {

const std::map<std::string, OpInfo>& Registry() {
  static std::map<std::string, OpInfo> r;
  if (r.empty()) {
    for (const char* n :
         {"sgd_update", "sgd_mom_update", "mp_sgd_update", "mp_sgd_mom_update", "multi_sgd_update",
          "multi_sgd_mom_update", "multi_mp_sgd_update", "multi_mp_sgd_mom_update", "adam_update",
          "_copyto", "_plus", "elemwise_add", "_minus", "elemwise_sub", "_mul", "elemwise_mul",
          "_plus_scalar", "_mul_scalar", "_set_value", "cast", "Cast", "zeros_like", "sqrt",
          // multi-tensor optimizer operators (multi_ops.cc)
          "multi_sum_sq", "multi_lars", "preloaded_multi_sgd_update", "preloaded_multi_sgd_mom_update",
          "preloaded_multi_mp_sgd_update", "preloaded_multi_mp_sgd_mom_update", "_adamw_update",
          "_mp_adamw_update", "_multi_adamw_update", "_multi_mp_adamw_update", "lamb_update_phase1",
          "lamb_update_phase2", "mp_lamb_update_phase1", "mp_lamb_update_phase2",
          "_multi_lamb_update", "_multi_mp_lamb_update",
          // single-tensor operators of the callback route (update_ops.cc)
          "nag_mom_update", "mp_nag_mom_update", "signsgd_update", "signum_update", "rmsprop_update",
          "rmspropalex_update", "ftml_update", "ftrl_update", "_sparse_ftrl_update",
          "_sparse_adagrad_update", "_contrib_group_adagrad_update"}) {
      r[n] = OpInfo{n};
    }
  }
  return r;
}

struct AdhocKey {
  NDArray w, g, s1, s2, w32;
  float lr = 0.f, wd = 0.f;
};

struct AdhocPlan {
  int dev = -1;
  void *d_keys = nullptr, *d_chunks = nullptr, *d_hyper = nullptr;
  size_t bk = 0, bc = 0, bh = 0;
  int n_chunks = 0;
  ~AdhocPlan() {
    Engine* e = Engine::Get();
    e->Free(dev, d_keys, bk);
    e->Free(dev, d_chunks, bc);
    e->Free(dev, d_hyper, bh);
  }
};

std::unordered_map<uint64_t, std::shared_ptr<AdhocPlan>>& PlanCache() {
  static auto* m = new std::unordered_map<uint64_t, std::shared_ptr<AdhocPlan>>();
  return *m;
}

uint64_t Mix(uint64_t h, const void* p) {
  uint64_t v = reinterpret_cast<uint64_t>(p);
  return h ^ (v + 0x9e3779b97f4a7c15ULL + (h << 6) + (h >> 2));
}

// One fused launch over a list of (weight, grad, state...) tuples that live on one GPU.
void RunAdhoc(int opt, std::vector<AdhocKey>& keys, const DenseLaunch& scalars,
              const NDArray* lrs = nullptr, const NDArray* wds = nullptr) {
  KV_CHECK(!keys.empty());
  const int dtype = keys[0].w.dtype();
  KV_CHECK(keys[0].w.on_gpu()) << "optimizer operators run on GPU arrays only (no CPU fallback)";
  const int dev = keys[0].w.dev();
  Engine* eng = Engine::Get();
  uint64_t sig = static_cast<uint64_t>(opt) * 1315423911u;
  for (auto& k : keys) {
    KV_CHECK(k.w.on_gpu() && k.w.dev() == dev) << "all operands must be on the same GPU";
    KV_CHECK_EQ(k.w.dtype(), dtype) << "all weights of one call must share a dtype";
    KV_CHECK_EQ(k.w.stype(), kDefaultStorage);
    if (!k.g.is_none()) {
      KV_CHECK(k.g.on_gpu() && k.g.dev() == dev) << "all operands must be on the same GPU";
      KV_CHECK_EQ(k.g.Size(), k.w.Size()) << "weight / grad shape mismatch";
      KV_CHECK_EQ(k.g.dtype(), dtype) << "weight / grad dtype mismatch";
    }
    for (const NDArray* a : {&k.s1, &k.s2, &k.w32}) {
      if (a->is_none()) continue;
      KV_CHECK(a->on_gpu() && a->dev() == dev) << "all operands must be on the same GPU";
      KV_CHECK_EQ(a->dtype(), kFloat32) << "optimizer states must be float32";
      KV_CHECK_EQ(a->Size(), k.w.Size()) << "state shape mismatch";
    }
    sig = Mix(sig, k.w.data());
    sig = Mix(sig, k.g.is_none() ? nullptr : k.g.data());
    sig = Mix(sig, k.s1.is_none() ? nullptr : k.s1.data());
    sig = Mix(sig, k.s2.is_none() ? nullptr : k.s2.data());
    sig = Mix(sig, k.w32.is_none() ? nullptr : k.w32.data());
    sig = Mix(sig, reinterpret_cast<const void*>(k.w.Size()));
  }
  auto& cache = PlanCache();
  std::shared_ptr<AdhocPlan> plan;
  auto it = cache.find(sig);
  LaneOp op(dev);
  cudaStream_t st = op.stream();
  if (it != cache.end()) {
    plan = it->second;
  } else {
    if (cache.size() > 512) cache.clear();
    plan = std::make_shared<AdhocPlan>();
    plan->dev = dev;
    std::vector<KeyDesc> kd(keys.size());
    std::vector<std::vector<ChunkDesc>> chunks(1);
    auto aligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    for (size_t i = 0; i < keys.size(); ++i) {
      KeyDesc& K = kd[i];
      std::memset(&K, 0, sizeof(K));
      AdhocKey& k = keys[i];
      K.w = k.w.data();
      K.w_in = K.w;
      bool ok = aligned(K.w);
      if (!k.g.is_none()) {
        K.src[0] = k.g.data();
        K.n_src = 1;
        ok = ok && aligned(K.src[0]);
      }
      K.s1 = k.s1.is_none() ? nullptr : static_cast<float*>(k.s1.data());
      K.s2 = k.s2.is_none() ? nullptr : static_cast<float*>(k.s2.data());
      K.w32 = k.w32.is_none() ? nullptr : static_cast<float*>(k.w32.data());
      ok = ok && aligned(K.s1) && aligned(K.s2) && aligned(K.w32);
      K.vec_ok = ok ? 1u : 0u;
      PlanChunks(0, k.w.Size(), static_cast<uint32_t>(i), 1, 0, &chunks);
    }
    plan->n_chunks = static_cast<int>(chunks[0].size());
    plan->bk = kd.size() * sizeof(KeyDesc);
    plan->bc = std::max<size_t>(chunks[0].size(), 1) * sizeof(ChunkDesc);
    plan->bh = keys.size() * 2 * sizeof(float);
    plan->d_keys = eng->Alloc(dev, plan->bk);
    plan->d_chunks = eng->Alloc(dev, plan->bc);
    plan->d_hyper = eng->Alloc(dev, plan->bh);
    KV_CUDA(cudaMemcpyAsync(plan->d_keys, kd.data(), plan->bk, cudaMemcpyHostToDevice, st));
    if (!chunks[0].empty()) {
      KV_CUDA(cudaMemcpyAsync(plan->d_chunks, chunks[0].data(),
                              chunks[0].size() * sizeof(ChunkDesc), cudaMemcpyHostToDevice, st));
    }
    cache[sig] = plan;
  }
  std::vector<float> hyper(keys.size() * 2);
  for (size_t i = 0; i < keys.size(); ++i) {
    hyper[2 * i] = keys[i].lr;
    hyper[2 * i + 1] = keys[i].wd;
  }
  KV_CUDA(cudaMemcpyAsync(plan->d_hyper, hyper.data(), plan->bh, cudaMemcpyHostToDevice, st));
  for (auto& k : keys) op.Read(k.g).Write(k.w).Write(k.s1).Write(k.s2).Write(k.w32);
  DenseLaunch L = scalars;
  if (lrs != nullptr) {
    // preloaded_multi_*: per-tensor lr / wd are read from device arrays by the kernel
    for (const NDArray* a : {lrs, wds}) {
      KV_CHECK(a->on_gpu() && a->dev() == dev) << "lrs / wds must live on the weights' GPU";
      KV_CHECK_EQ(a->dtype(), kFloat32) << "lrs / wds must be float32";
      KV_CHECK_EQ(a->Size(), keys.size()) << "Number of learning rates / weight decays is "
                                          << "inconsistent with num_weights parameter passed";
      op.Read(*a);
    }
    L.lrs = static_cast<const float*>(lrs->data());
    L.wds = static_cast<const float*>(wds->data());
  }
  L.keys = static_cast<const KeyDesc*>(plan->d_keys);
  L.chunks = static_cast<const ChunkDesc*>(plan->d_chunks);
  L.hyper = static_cast<const float*>(plan->d_hyper);
  L.n_chunks = plan->n_chunks;
  L.max_src = 1;
  L.dtype = dtype;
  L.opt = opt;
  LaunchDenseFused(L, st);
  eng->CountLaunch("dense_fused(op)", 0);
  op.Issue();
}

// lazy row_sparse gradient: update only the rows listed (optimizer_op-inl.h:452-565,803-876,1410-1470)
void RunRspUpdate(int opt, const NDArray& w, const NDArray& g, const NDArray& s1, const NDArray& s2,
                  RspUpdateLaunch L) {
  KV_CHECK(w.on_gpu() && g.on_gpu() && w.dev() == g.dev()) << "all operands must be on the same GPU";
  KV_CHECK_EQ(w.dtype(), kFloat32) << "row_sparse optimizer updates are float32";
  KV_CHECK_EQ(w.stype(), kDefaultStorage) << "row_sparse weights with row_sparse gradients: the "
                                          << "store keeps sparse-updated weights dense";
  if (!g.storage_initialized()) return;  // all-zero gradient: lazy update touches nothing
  LaneOp op(w.dev());
  op.Read(g).Write(w).Write(s1).Write(s2);
  L.opt = opt;
  L.w = static_cast<float*>(w.data());
  L.s1 = s1.is_none() ? nullptr : static_cast<float*>(s1.data());
  L.s2 = s2.is_none() ? nullptr : static_cast<float*>(s2.data());
  L.gidx = g.row_ids();
  L.gval = static_cast<const float*>(g.data());
  L.nrows = g.nnr();
  L.row_len = static_cast<int64_t>(w.RowLength());
  LaunchRspUpdate(L, op.stream());
  Engine::Get()->CountLaunch("rsp_update", 0);
  op.Issue();
}

NDArray OutOrInput(std::vector<NDArray>* outputs, size_t i, const NDArray& like) {
  if (outputs->size() > i) return (*outputs)[i];
  NDArray o(like.shape(), like.ctx(), like.dtype());
  outputs->push_back(o);
  return o;
}

void Elementwise(int op, const NDArray& a, const NDArray* b, float scalar, const NDArray& out) {
  KV_CHECK(out.on_gpu()) << "elementwise operators run on GPU arrays only";
  const int dev = out.dev();
  LaneOp lop(dev);
  if (op != kEwFill) {
    KV_CHECK(a.on_gpu() && a.dev() == dev) << "all operands must be on the same GPU";
    KV_CHECK_EQ(a.Size(), out.Size()) << "elementwise shape mismatch";
    KV_CHECK_EQ(a.dtype(), out.dtype()) << "elementwise dtype mismatch";
    lop.Read(a);
  }
  if (b) {
    KV_CHECK(b->on_gpu() && b->dev() == dev) << "all operands must be on the same GPU";
    KV_CHECK_EQ(b->Size(), out.Size()) << "elementwise shape mismatch";
    KV_CHECK_EQ(b->dtype(), out.dtype()) << "elementwise dtype mismatch";
    lop.Read(*b);
  }
  lop.Write(out);
  LaunchElementwise(op, out.dtype(), out.data(), op == kEwFill ? nullptr : a.data(),
                    b ? b->data() : nullptr, scalar, out.Size(), lop.stream());
  Engine::Get()->CountLaunch("elementwise", 0);
  lop.Issue();
}

}  // namespace

const OpInfo* FindOp(const std::string& name) {
  auto& r = Registry();
  auto it = r.find(name);
  return it == r.end() ? nullptr : &it->second;
}

void InvokeOp(const OpInfo* op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
              const Params& p) {
  const std::string& n = op->name;
  DenseLaunch S;
  S.rescale = GetF(p, "rescale_grad", 1.0f);
  S.clip = GetF(p, "clip_gradient", -1.0f);
  auto in_place = [&](size_t widx, size_t oidx) {
    // the front-end always passes out=weight; a distinct out gets the weight copied first
    NDArray o = OutOrInput(outputs, oidx, in[widx]);
    if (!o.SameStorage(in[widx])) CopyFromTo(in[widx], o);
    return o;
  };
  if (n == "sgd_update" || n == "sgd_mom_update" || n == "adam_update") {
    const bool mom = n == "sgd_mom_update";
    const bool adam = n == "adam_update";
    const size_t nin = adam ? 4 : (mom ? 3 : 2);
    KV_CHECK_EQ(in.size(), nin) << n << " expects " << nin << " inputs";
    NDArray w = in_place(0, 0);
    if (in[1].stype() == kRowSparseStorage) {
      RspUpdateLaunch L;
      L.lr = GetF(p, "lr", 0.f);
      L.wd = GetF(p, "wd", 0.f);
      L.momentum = GetF(p, "momentum", 0.f);
      L.rescale = S.rescale;
      L.clip = S.clip;
      L.beta1 = GetF(p, "beta1", 0.9f);
      L.beta2 = GetF(p, "beta2", 0.999f);
      L.eps = GetF(p, "epsilon", 1e-8f);
      const int kind = adam ? kOptAdam : (mom ? kOptSGD : kOptSGDSingle);
      if (GetB(p, "lazy_update", true)) {
        RunRspUpdate(kind, w, in[1], (mom || adam) ? in[2] : NDArray(), adam ? in[3] : NDArray(), L);
      } else {
        // standard update: every row moves (SGDUpdateEx / SGDMomUpdateEx / AdamUpdateEx with
        // lazy_update=False, optimizer_op-inl.h:540-565, 955-1004, 1520-1564)
        L.opt = kind;
        RunRspStdUpdate(w, in[1], (mom || adam) ? in[2] : NDArray(), adam ? in[3] : NDArray(), L);
      }
      return;
    }
    AdhocKey k;
    k.w = w;
    k.g = in[1];
    k.lr = GetF(p, "lr", 0.f);
    k.wd = GetF(p, "wd", 0.f);
    KV_CHECK(Find(p, "lr") != nullptr) << "Required parameter lr of " << n << " is missing";
    if (mom) k.s1 = in[2];
    if (adam) {
      k.s1 = in[2];
      k.s2 = in[3];
      S.beta1 = GetF(p, "beta1", 0.9f);
      S.beta2 = GetF(p, "beta2", 0.999f);
      S.eps = GetF(p, "epsilon", 1e-8f);
    }
    S.momentum = GetF(p, "momentum", 0.f);
    std::vector<AdhocKey> keys{k};
    RunAdhoc(adam ? kOptAdam : (mom ? kOptSGD : kOptSGDSingle), keys, S);
    return;
  }
  if (n == "mp_sgd_update" || n == "mp_sgd_mom_update") {
    const bool mom = n == "mp_sgd_mom_update";
    KV_CHECK_EQ(in.size(), mom ? 4u : 3u) << n << ": wrong number of inputs";
    AdhocKey k;
    k.w = in_place(0, 0);
    k.g = in[1];
    if (mom) k.s1 = in[2];
    k.w32 = in[mom ? 3 : 2];
    k.lr = GetF(p, "lr", 0.f);
    k.wd = GetF(p, "wd", 0.f);
    S.momentum = GetF(p, "momentum", 0.f);
    std::vector<AdhocKey> keys{k};
    RunAdhoc(mom ? kOptSGD : kOptSGDSingle, keys, S);
    return;
  }
  if (MultiTensorOp(n, in, outputs, p)) return;  // multi_ops.cc: sum_sq, lars, adamw, lamb
  if (UpdateOp(n, in, outputs, p)) return;       // update_ops.cc: nag, signum, rmsprop, ftml, ftrl
  if (n.rfind("multi_", 0) == 0 || n.rfind("preloaded_multi_", 0) == 0) {
    // multi_[mp_]sgd[_mom]_update (optimizer_op-inl.h:207-380) and the preloaded_ forms
    // (contrib/preloaded_multi_sgd-inl.h:154-330: same kernel, lrs / wds are two trailing INPUT
    // arrays on the device instead of tuple attributes)
    const bool preloaded = n.rfind("preloaded_", 0) == 0;
    const bool mp = n.find("_mp_") != std::string::npos;
    const bool mom = n.find("_mom_") != std::string::npos;
    const int stride = 2 + (mom ? 1 : 0) + (mp ? 1 : 0);
    const int num = GetI(p, "num_weights", 1);
    KV_CHECK_EQ(static_cast<int>(in.size()), num * stride + (preloaded ? 2 : 0))
        << n << ": expected num_weights*" << stride << (preloaded ? " + 2" : "") << " inputs";
    std::vector<float> lrs, wds;
    if (!preloaded) {
      lrs = GetTuple(p, "lrs");
      wds = GetTuple(p, "wds");
      KV_CHECK_EQ(static_cast<int>(lrs.size()), num) << n << ": len(lrs) != num_weights";
      KV_CHECK_EQ(static_cast<int>(wds.size()), num) << n << ": len(wds) != num_weights";
    }
    S.momentum = GetF(p, "momentum", 0.f);
    std::vector<AdhocKey> keys(num);
    for (int i = 0; i < num; ++i) {
      AdhocKey& k = keys[i];
      k.w = in_place(i * stride, i);
      k.g = in[i * stride + 1];
      int j = 2;
      if (mom) k.s1 = in[i * stride + j++];
      if (mp) k.w32 = in[i * stride + j++];
      k.lr = preloaded ? 0.f : lrs[i];
      k.wd = preloaded ? 0.f : wds[i];
    }
    if (preloaded) {
      for (auto& k : keys) {
        KV_CHECK_EQ(k.w.dtype(), keys[0].w.dtype()) << n << ": all weights must share a dtype";
      }
      RunAdhoc(kOptSGD, keys, S, &in[num * stride], &in[num * stride + 1]);
      return;
    }
    // group by dtype: one launch each (Updater aggregates by dtype anyway, optimizer.py:2104-2113)
    std::map<int, std::vector<AdhocKey>> by_dtype;
    for (auto& k : keys) by_dtype[k.w.dtype()].push_back(k);
    for (auto& kv : by_dtype) RunAdhoc(kOptSGD, kv.second, S);
    return;
  }
  if (n == "_copyto") {
    KV_CHECK_EQ(in.size(), 1u);
    NDArray o = OutOrInput(outputs, 0, in[0]);
    CopyFromTo(in[0], o);
    return;
  }
  if (n == "_plus" || n == "elemwise_add" || n == "_minus" || n == "elemwise_sub" || n == "_mul" ||
      n == "elemwise_mul") {
    KV_CHECK_EQ(in.size(), 2u);
    NDArray o = OutOrInput(outputs, 0, in[0]);
    const int e = (n == "_plus" || n == "elemwise_add") ? kEwAdd
                  : (n == "_minus" || n == "elemwise_sub") ? kEwSub : kEwMul;
    Elementwise(e, in[0], &in[1], 0.f, o);
    return;
  }
  if (n == "_plus_scalar" || n == "_mul_scalar") {
    KV_CHECK_EQ(in.size(), 1u);
    NDArray o = OutOrInput(outputs, 0, in[0]);
    Elementwise(n == "_plus_scalar" ? kEwAddScalar : kEwMulScalar, in[0], nullptr,
                GetF(p, "scalar", 0.f), o);
    return;
  }
  if (n == "sqrt") {
    KV_CHECK_EQ(in.size(), 1u);
    NDArray o = OutOrInput(outputs, 0, in[0]);
    Elementwise(kEwSqrt, in[0], nullptr, 0.f, o);
    return;
  }
  if (n == "_set_value") {
    KV_CHECK(outputs->size() == 1) << "_set_value needs an out array";
    Elementwise(kEwFill, NDArray(), nullptr, GetF(p, "src", 0.f), (*outputs)[0]);
    return;
  }
  if (n == "zeros_like") {
    KV_CHECK_EQ(in.size(), 1u);
    NDArray o = OutOrInput(outputs, 0, in[0]);
    Elementwise(kEwFill, NDArray(), nullptr, 0.f, o);
    return;
  }
  if (n == "cast" || n == "Cast") {
    KV_CHECK_EQ(in.size(), 1u);
    const std::string* dt = Find(p, "dtype");
    KV_CHECK(dt != nullptr) << "cast: dtype is required";
    int dtype = -1;
    if (*dt == "float32") dtype = kFloat32;
    else if (*dt == "float16") dtype = kFloat16;
    else if (*dt == "bfloat16") dtype = kBfloat16;
    else if (*dt == "float64") dtype = kFloat64;
    else if (*dt == "int32") dtype = kInt32;
    else if (*dt == "int64") dtype = kInt64;
    KV_CHECK(dtype >= 0) << "cast: unsupported dtype " << *dt;
    NDArray o;
    if (outputs->empty()) {
      o = NDArray(in[0].shape(), in[0].ctx(), dtype);
      outputs->push_back(o);
    } else {
      o = (*outputs)[0];
    }
    KV_CHECK(in[0].on_gpu() && o.on_gpu() && in[0].dev() == o.dev()) << "cast runs on one GPU";
    LaneOp op(o.dev());
    op.Read(in[0]).Write(o);
    LaunchCast(o.data(), o.dtype(), in[0].data(), in[0].dtype(), o.Size(), op.stream());
    Engine::Get()->CountLaunch("cast", 0);
    op.Issue();
    return;
  }
  KV_FATAL << "operator " << n << " is registered but not implemented";
}

}  // namespace b200kv
