// ops.cc -- see ops.h.
#include "ops.h"

#include <algorithm>
#include <cstring>
#include <unordered_map>

#include "kernels.h"
#include "rowsparse.h"
#include "scalar_parse.h"

namespace b200kv {

void PlanChunks(uint64_t goff, size_t size, uint32_t key_slot, int ndev, int owner_fixed,
                std::vector<std::vector<ChunkDesc>>* per_slot);  // kvstore.cc

void TableCache::Tables::Upload(int i, size_t size, const void* host, size_t host_bytes, cudaStream_t st) {
  bytes[i] = size;
  d[i] = Engine::Get()->Alloc(dev, size);
  if (host_bytes > 0) KV_CUDA(cudaMemcpyAsync(d[i], host, host_bytes, cudaMemcpyHostToDevice, st));
}

TableCache::Tables::~Tables() {
  for (int i = 0; i < 3; ++i) Engine::Get()->Free(dev, d[i], bytes[i]);
}

const TableCache::Tables* TableCache::Find(const std::vector<uint64_t>& key) const {
  auto it = map_.find(key);
  return it == map_.end() ? nullptr : it->second.get();
}

const TableCache::Tables* TableCache::Insert(std::vector<uint64_t> key, std::unique_ptr<Tables> tables) {
  if (map_.size() > 512) map_.clear();
  return (map_[std::move(key)] = std::move(tables)).get();
}

NDArray OutOr(std::vector<NDArray>* outputs, size_t i, const std::vector<int64_t>& shape, Context ctx,
              int dtype) {
  if (outputs->size() > i) return (*outputs)[i];
  NDArray o(shape, ctx, dtype);
  outputs->push_back(o);
  return o;
}

NDArray InPlace(const std::vector<NDArray>& in, size_t widx, std::vector<NDArray>* outputs, size_t oidx) {
  NDArray o = OutOr(outputs, oidx, in[widx].shape(), in[widx].ctx(), in[widx].dtype());
  if (!o.SameStorage(in[widx])) CopyFromTo(in[widx], o);
  return o;
}

const char* StypeName(int stype) { return stype == kRowSparseStorage ? "row_sparse" : "default"; }

void ZeroFillEmptyRspStates(const std::vector<NDArray>& states, int64_t rows, const char* launch_name) {
  std::vector<const NDArray*> fill;
  for (const NDArray& a : states) {
    if (!a.is_none() && a.stype() == kRowSparseStorage && a.nnr() == 0) fill.push_back(&a);
  }
  if (fill.empty()) return;
  for (const NDArray* a : fill) a->CheckAndAllocRows(rows);
  LaneOp lop(fill[0]->dev());
  for (const NDArray* a : fill) lop.Write(*a);
  for (const NDArray* a : fill) {
    const size_t row_bytes = a->RowLength() * DTypeSize(a->dtype());
    KV_CUDA(cudaMemsetAsync(a->data(), 0, static_cast<size_t>(rows) * row_bytes, lop.stream()));
    LaunchFillRowIds(a->row_ids(), rows, lop.stream());
    Engine::Get()->CountLaunch(launch_name, static_cast<uint64_t>(rows) * (row_bytes + 8));
  }
  lop.Issue();
}

void CheckRspTable(const char* op, const char* func, const std::vector<NDArray>& in,
                   const std::vector<NDArray>& outputs) {
  const NDArray& w = in[0];
  const int64_t rows = w.shape()[0];
  KV_CHECK(w.stype() != kRowSparseStorage || w.nnr() == rows)
      << func << " for RowSparse weights is only implemented for RowSparse weights with all rows "
      << "containing non-zeros. Expects weights.data.shape[0] (" << w.nnr() << ") == weights.shape[0] ("
      << rows << ").";
  for (size_t i = 2; i < in.size(); ++i) {
    KV_CHECK(in[i].stype() != kRowSparseStorage || in[i].nnr() == 0 || in[i].nnr() == rows)
        << op << ": a row_sparse optimizer state must hold every row or none (it holds "
        << in[i].nnr() << " of " << rows << ")";
  }
  KV_CHECK(outputs.size() == 1 && outputs[0].SameStorage(w) && outputs[0].stype() == w.stype() &&
           outputs[0].data() == w.data())
      << op << ": out must be the weight itself (kWriteInplace is expected for sparse " << op << ")";
}

const OpInfo* FindOp(const std::string& name) {
  static const auto* table = [] {
    auto* m = new std::unordered_map<std::string, const OpInfo*>();
    for (const std::vector<OpInfo>* family :
         {&kCoreOps, &kMultiTensorOps, &kUpdateOps, &kArithOps, &kReduceOps, &kSumOps, &kRandomOps,
          &kSampleOps, &kSampleParamOps}) {
      for (const OpInfo& op : *family) {
        KV_CHECK(m->emplace(op.name, &op).second) << "operator " << op.name << " is declared twice";
      }
    }
    return m;
  }();
  auto it = table->find(name);
  return it == table->end() ? nullptr : it->second;
}

namespace {

// Dense operands only: the kernel walks Size() elements from data(), and a row_sparse array's
// data() holds only its stored rows. Every check runs before anything is enqueued. per_row: b holds
// one value per row of a's trailing axis.
void CheckedElementwise(int op, const NDArray& a, const NDArray* b, bool per_row, double scalar,
                        const NDArray& out, double scalar2) {
  KV_CHECK(out.on_gpu()) << "elementwise operators run on GPU arrays only";
  KV_CHECK(out.stype() == kDefaultStorage)
      << "elementwise operators take dense arrays only; out is not dense (default storage)";
  KV_CHECK(ElementwiseDTypeOk(out.dtype()))
      << "elementwise operators take float16, bfloat16, float32, float64, int32 and int64 arrays; got "
      << DTypeName(out.dtype());
  const int dev = out.dev();
  size_t b_row = 1;
  if (per_row) {
    KV_CHECK(!a.shape().empty()) << "a row broadcast needs an operand of rank 1 or more";
    b_row = static_cast<size_t>(a.shape().back());
  }
  if (op != kEwFill) {
    KV_CHECK(a.on_gpu() && a.dev() == dev) << "all operands must be on the same GPU";
    KV_CHECK(a.stype() == kDefaultStorage)
        << "elementwise operators take dense arrays only; an input is not dense (default storage)";
    KV_CHECK_EQ(a.Size(), out.Size()) << "elementwise shape mismatch";
    KV_CHECK_EQ(a.dtype(), out.dtype()) << "elementwise dtype mismatch";
  }
  if (b) {
    KV_CHECK(b->on_gpu() && b->dev() == dev) << "all operands must be on the same GPU";
    KV_CHECK(b->stype() == kDefaultStorage)
        << "elementwise operators take dense arrays only; an input is not dense (default storage)";
    KV_CHECK_EQ(b->Size() * b_row, out.Size()) << "elementwise shape mismatch";
    KV_CHECK_EQ(b->dtype(), out.dtype()) << "elementwise dtype mismatch";
  }
  LaneOp lop(dev);
  if (op != kEwFill) lop.Read(a);
  if (b) lop.Read(*b);
  lop.Write(out);
  LaunchElementwise(op, out.dtype(), out.data(), op == kEwFill ? nullptr : a.data(),
                    b ? b->data() : nullptr, scalar, out.Size(), lop.stream(), scalar2,
                    per_row ? b_row : 0);
  Engine::Get()->CountLaunch("elementwise", 0);
  lop.Issue();
}

}  // namespace

void Elementwise(int op, const NDArray& a, const NDArray* b, double scalar, const NDArray& out,
                 double scalar2) {
  CheckedElementwise(op, a, b, false, scalar, out, scalar2);
}

void ElementwiseRows(int op, const NDArray& a, const NDArray& b, const NDArray& out) {
  CheckedElementwise(op, a, &b, true, 0.0, out, 0.0);
}

namespace {

struct AdhocKey {
  NDArray w, g, s1, s2, w32;
  float lr = 0.f, wd = 0.f;
};

// One fused launch over a list of (weight, grad, state...) tuples that live on one GPU.
void RunAdhoc(int opt, std::vector<AdhocKey>& keys, const DenseLaunch& scalars,
              const NDArray* lrs = nullptr, const NDArray* wds = nullptr) {
  static auto* cache = new TableCache();
  KV_CHECK(!keys.empty());
  const int dtype = keys[0].w.dtype();
  KV_CHECK(keys[0].w.on_gpu()) << "optimizer operators run on GPU arrays only (no CPU fallback)";
  const int dev = keys[0].w.dev();
  auto addr = [](const NDArray& a) { return reinterpret_cast<uint64_t>(a.is_none() ? nullptr : a.data()); };
  std::vector<uint64_t> sig{static_cast<uint64_t>(opt)};
  sig.reserve(1 + 6 * keys.size());
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
    sig.insert(sig.end(), {addr(k.w), addr(k.g), addr(k.s1), addr(k.s2), addr(k.w32), k.w.Size()});
  }
  LaneOp op(dev);
  cudaStream_t st = op.stream();
  const TableCache::Tables* plan = cache->Find(sig);
  if (plan == nullptr) {
    auto t = std::make_unique<TableCache::Tables>(dev);
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
    const std::vector<ChunkDesc>& c = chunks[0];
    const size_t bk = kd.size() * sizeof(KeyDesc), bc = c.size() * sizeof(ChunkDesc);
    t->n_chunks = static_cast<int>(c.size());
    t->Upload(0, bk, kd.data(), bk, st);
    t->Upload(1, std::max(bc, sizeof(ChunkDesc)), c.data(), bc, st);
    t->Upload(2, keys.size() * 2 * sizeof(float), nullptr, 0, st);  // lr / wd: written on every call
    plan = cache->Insert(std::move(sig), std::move(t));
  }
  std::vector<float> hyper(keys.size() * 2);
  for (size_t i = 0; i < keys.size(); ++i) {
    hyper[2 * i] = keys[i].lr;
    hyper[2 * i + 1] = keys[i].wd;
  }
  KV_CUDA(cudaMemcpyAsync(plan->d[2], hyper.data(), plan->bytes[2], cudaMemcpyHostToDevice, st));
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
  L.keys = static_cast<const KeyDesc*>(plan->d[0]);
  L.chunks = static_cast<const ChunkDesc*>(plan->d[1]);
  L.hyper = static_cast<const float*>(plan->d[2]);
  L.n_chunks = plan->n_chunks;
  L.max_src = 1;
  L.dtype = dtype;
  L.opt = opt;
  LaunchDenseFused(L, st);
  Engine::Get()->CountLaunch("dense_fused(op)", 0);
  op.Issue();
}

// Weight dtypes, checked before InPlace copies a weight into a distinct out. The fused step computes
// in float32 and rounds once on store. The reference's non-mp forms compute in the weight's own
// type and round after every operation (optimizer_op-inl.h:225-250, 410-418), so they take float32
// weights only; 16-bit weights go through the mp forms, which keep a float32 master copy.
void CheckWeightDTypes(const OpInfo& op, const std::vector<NDArray>& in, int num, int stride, bool mp) {
  for (int i = 0; i < num; ++i) {
    const int dt = in[static_cast<size_t>(i) * stride].dtype();
    if (mp) {
      KV_CHECK(dt == kFloat32 || dt == kFloat16 || dt == kBfloat16)
          << op.name << " takes float32, float16 or bfloat16 weights; weight " << i << " is "
          << DTypeName(dt);
    } else if (dt != kFloat32) {
      std::string mp_form = op.name;
      const size_t at = mp_form.find("sgd");
      mp_form = at == std::string::npos ? "a float32 master copy (multi_precision=True)"
                                        : mp_form.insert(at, "mp_");
      KV_FATAL << op.name << " takes float32 weights; weight " << i << " is " << DTypeName(dt)
               << " (float16 / bfloat16 weights need " << mp_form << ")";
    }
  }
}

// rescale_grad and clip_gradient, which every operator call parses first (InvokeOp)
DenseLaunch GradScalars(const Params& p) {
  DenseLaunch S;
  S.rescale = GetF(p, "rescale_grad", 1.0f);
  S.clip = GetF(p, "clip_gradient", -1.0f);
  return S;
}

// sgd_update, sgd_mom_update and adam_update on a row_sparse weight (SGDUpdateEx, SGDMomUpdateEx,
// AdamUpdateEx: optimizer_op-inl.h:548-565, 972-1004, 1531-1564), float32 only:
//   (row_sparse weight, row_sparse grad[, row_sparse states])  lazy_update: lazy, else standard
//   (row_sparse weight, row_sparse grad, dense states)         standard, whatever lazy_update says
// The weight holds every row, so its values are the row-major table and the dense weight's kernels
// serve it. A row_sparse state holds every row, or none yet: then it is zero-filled first, in both
// forms and even when the gradient is empty. Every check runs before anything is enqueued.
void SgdAdamRspWeight(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                      const UpdateLaunch& L, bool lazy) {
  const NDArray& w = in[0];
  const int kind = op.variant;
  if (in.size() > 2 && in[2].stype() == kDefaultStorage) lazy = false;  // StdOptStorageType (:912-917)
  KV_CHECK(!w.shape().empty()) << op.name << ": the weight needs at least one dimension";
  for (const NDArray& a : in) {
    KV_CHECK(a.on_gpu() && a.dev() == w.dev()) << op.name << ": all operands must be on the same GPU";
    KV_CHECK_EQ(a.dtype(), kFloat32) << "row_sparse optimizer updates are float32";
    KV_CHECK(a.shape() == w.shape()) << op.name << ": weight / grad / state shape mismatch";
  }
  // the reference's function names (optimizer_op-inl.h:541, 859, 958, 1472, 1523); kWriteInplace is
  // expected (optimizer_op-inl.h:497, 818, 1426)
  const char* func = kind == kOptSGDSingle ? "SGDUpdate"
                     : kind == kOptSGD     ? "SGDMomUpdate"
                     : lazy                ? "AdamUpdate"
                                           : "AdamStdUpdate";
  CheckRspTable(op.name, func, in, *outputs);
  const std::vector<NDArray> states(in.begin() + 2, in.end());
  ZeroFillEmptyRspStates(states, w.shape()[0], "rsp_state_fill");
  SgdAdamRspUpdate(kind, lazy, L, w, in[1], states);
}

// sgd_update, sgd_mom_update, adam_update (variant: the kOpt* kernel code): dense weight with a dense
// or row_sparse grad and dense states, or a row_sparse weight (SgdAdamRspWeight)
void SgdAdam(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
             const Params& p) {
  DenseLaunch S = GradScalars(p);
  const int kind = op.variant;
  const bool mom = kind == kOptSGD;
  const bool adam = kind == kOptAdam;
  const size_t nin = adam ? 4 : (mom ? 3 : 2);
  KV_CHECK_EQ(in.size(), nin) << op.name << " expects " << nin << " inputs";
  CheckWeightDTypes(op, in, 1, 0, false);
  // storage types (SGDUpdateEx, SGDMomUpdateEx, AdamUpdateEx, StdOptStorageType), checked before a
  // distinct out is written: states share one stype; a dense weight takes dense states, a
  // row_sparse weight a row_sparse gradient
  const int wst = in[0].stype();
  KV_CHECK(outputs->empty() || (*outputs)[0].stype() == wst) << "Inconsistent weight stype and output stype";
  KV_CHECK(!adam || in[2].stype() == in[3].stype()) << "Inconsistent mean stype and var stype";
  const int sst = nin > 2 ? in[2].stype() : kDefaultStorage;
  const bool rsp_g = in[1].stype() == kRowSparseStorage;
  if (wst != kDefaultStorage || sst != kDefaultStorage) {
    std::string got;
    for (const NDArray& a : in) got += std::string(got.empty() ? "" : ", ") + StypeName(a.stype());
    KV_CHECK(wst == kRowSparseStorage && rsp_g)
        << op.name << ": storage types (" << got << ") are not supported: row_sparse states need a "
        << "row_sparse weight, and a row_sparse weight a row_sparse gradient";
  }
  auto rsp_launch = [&] {
    UpdateLaunch L;
    L.lr = GetF(p, "lr", 0.f);
    L.wd = GetF(p, "wd", 0.f);
    L.momentum = GetF(p, "momentum", 0.f);
    L.rescale = S.rescale;
    L.clip = S.clip;
    L.beta1 = GetF(p, "beta1", 0.9f);
    L.beta2 = GetF(p, "beta2", 0.999f);
    L.eps = GetF(p, "epsilon", 1e-8f);
    return L;
  };
  if (wst == kRowSparseStorage) {
    Required(p, "lr", op.name);
    SgdAdamRspWeight(op, in, outputs, rsp_launch(), GetB(p, "lazy_update", true));
    return;
  }
  NDArray w = InPlace(in, 0, outputs, 0);
  if (rsp_g) {
    // SGDUpdateEx / SGDMomUpdateEx / AdamUpdateEx (optimizer_op-inl.h:540-565, 955-1004, 1520-1564)
    const UpdateLaunch L = rsp_launch();
    SgdAdamRspUpdate(kind, GetB(p, "lazy_update", true), L, w, in[1],
                     std::vector<NDArray>(in.begin() + 2, in.end()));
    return;
  }
  AdhocKey k;
  k.w = w;
  k.g = in[1];
  k.lr = GetF(p, "lr", 0.f);
  k.wd = GetF(p, "wd", 0.f);
  Required(p, "lr", op.name);
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
  RunAdhoc(kind, keys, S);
}

// mp_sgd_update, mp_sgd_mom_update (variant: kOptSGDSingle / kOptSGD)
void MpSgd(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
           const Params& p) {
  DenseLaunch S = GradScalars(p);
  const bool mom = op.variant == kOptSGD;
  KV_CHECK_EQ(in.size(), mom ? 4u : 3u) << op.name << ": wrong number of inputs";
  CheckWeightDTypes(op, in, 1, 0, true);
  AdhocKey k;
  k.w = InPlace(in, 0, outputs, 0);
  k.g = in[1];
  if (mom) k.s1 = in[2];
  k.w32 = in[mom ? 3 : 2];
  k.lr = GetF(p, "lr", 0.f);
  k.wd = GetF(p, "wd", 0.f);
  S.momentum = GetF(p, "momentum", 0.f);
  std::vector<AdhocKey> keys{k};
  RunAdhoc(op.variant, keys, S);
}

// multi_[mp_]sgd[_mom]_update (optimizer_op-inl.h:207-380) and the preloaded_ forms
// (contrib/preloaded_multi_sgd-inl.h:154-330: same kernel, lrs / wds are two trailing INPUT
// arrays on the device instead of tuple attributes); variant: kOpMom | kOpMp | kOpPreloaded
void MultiSgd(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
              const Params& p) {
  DenseLaunch S = GradScalars(p);
  const char* n = op.name;
  const bool preloaded = op.variant & kOpPreloaded;
  const bool mp = op.variant & kOpMp;
  const bool mom = op.variant & kOpMom;
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
  CheckWeightDTypes(op, in, num, stride, mp);
  S.momentum = GetF(p, "momentum", 0.f);
  std::vector<AdhocKey> keys(num);
  for (int i = 0; i < num; ++i) {
    AdhocKey& k = keys[i];
    k.w = InPlace(in, i * stride, outputs, i);
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
}

void Copy(const OpInfo&, const std::vector<NDArray>& in, std::vector<NDArray>* outputs, const Params&) {
  KV_CHECK_EQ(in.size(), 1u);
  CopyFromTo(in[0], OutOr(outputs, 0, in[0].shape(), in[0].ctx(), in[0].dtype()));
}

// _plus, _minus, _mul and their elemwise_ aliases (variant: the kEw* code)
void Binary(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs, const Params&) {
  KV_CHECK_EQ(in.size(), 2u);
  NDArray o = OutOr(outputs, 0, in[0].shape(), in[0].ctx(), in[0].dtype());
  Elementwise(op.variant, in[0], &in[1], 0.f, o);
}

// _plus_scalar, _mul_scalar and sqrt (variant: the kEw* code)
void Unary(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs, const Params& p) {
  KV_CHECK_EQ(in.size(), 1u);
  NDArray o = OutOr(outputs, 0, in[0].shape(), in[0].ctx(), in[0].dtype());
  Elementwise(op.variant, in[0], nullptr, op.variant == kEwSqrt ? 0.0 : StodD(p, "scalar", op.name), o);
}

void SetValue(const OpInfo&, const std::vector<NDArray>&, std::vector<NDArray>* outputs, const Params& p) {
  KV_CHECK(outputs->size() == 1) << "_set_value needs an out array";
  Elementwise(kEwFill, NDArray(), nullptr, GetF(p, "src", 0.f), (*outputs)[0]);
}

// `a[:] = v` (ndarray.py:504): InitOpWithScalarParam's double `value`, parsed by dmlc::stod, then
// Fill's static_cast<DType> (init_op.h:241-257, 416-421). Only into an existing out here.
void Full(const OpInfo& op, const std::vector<NDArray>&, std::vector<NDArray>* outputs, const Params& p) {
  KV_CHECK(outputs->size() == 1) << "_full needs an out array";
  double val = Required<double>(p, "value", op.name);
  if (val == 0) val = 0.0;  // Fill's val == 0 branch writes zero bytes: -0.0 stores +0.0
  Elementwise(kEwFill, NDArray(), nullptr, val, (*outputs)[0]);
}

// zeros_like, _sparse_zeros_like: the result takes out's storage type, else the input's
void ZerosLike(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
               const Params&) {
  const char* n = op.name;
  KV_CHECK_EQ(in.size(), 1u);
  const bool rsp_out = outputs->empty() ? in[0].stype() == kRowSparseStorage
                                        : (*outputs)[0].stype() == kRowSparseStorage;
  if (!rsp_out) {
    NDArray o = OutOr(outputs, 0, in[0].shape(), in[0].ctx(), in[0].dtype());
    Elementwise(kEwFill, NDArray(), nullptr, 0.0, o);
    return;
  }
  // a row_sparse result stores no rows (FillZerosRspImpl, init_op.h:496-502): its storage is kept,
  // nothing is launched. The write is declared first, so work issued before still sees the rows.
  KV_CHECK(in[0].on_gpu()) << n << " runs on GPU arrays only (no CPU fallback)";
  if (!outputs->empty()) {
    const NDArray& o = (*outputs)[0];
    KV_CHECK(o.on_gpu() && o.dev() == in[0].dev()) << "all operands must be on the same GPU";
    KV_CHECK(o.shape() == in[0].shape()) << n << ": out shape mismatch";
    KV_CHECK_EQ(o.dtype(), in[0].dtype()) << n << ": out dtype mismatch";
  }
  if (outputs->empty()) outputs->push_back(NDArray::RowSparse(in[0].shape(), in[0].ctx(), in[0].dtype()));
  const NDArray& o = (*outputs)[0];
  LaneOp lop(o.dev());
  lop.Write(o);
  lop.Issue();
  o.SetNnr(0);
}

// cast, Cast
void Cast(const OpInfo&, const std::vector<NDArray>& in, std::vector<NDArray>* outputs, const Params& p) {
  KV_CHECK_EQ(in.size(), 1u);
  const std::string* dt = Find(p, "dtype");
  KV_CHECK(dt != nullptr) << "cast: dtype is required";
  int dtype = -1;
  for (int t : {kFloat32, kFloat16, kBfloat16, kFloat64, kInt32, kInt64}) {
    if (*dt == DTypeName(t)) dtype = t;
  }
  KV_CHECK(dtype >= 0) << "cast: unsupported dtype " << *dt;
  NDArray o = OutOr(outputs, 0, in[0].shape(), in[0].ctx(), dtype);
  KV_CHECK(in[0].on_gpu() && o.on_gpu() && in[0].dev() == o.dev()) << "cast runs on one GPU";
  KV_CHECK_EQ(o.dtype(), dtype) << "cast: out dtype differs from dtype=" << *dt;
  KV_CHECK_EQ(o.Size(), in[0].Size()) << "cast: out shape mismatch";
  LaneOp lop(o.dev());
  lop.Read(in[0]).Write(o);
  LaunchCast(o.data(), o.dtype(), in[0].data(), in[0].dtype(), o.Size(), lop.stream());
  Engine::Get()->CountLaunch("cast", 0);
  lop.Issue();
}

}  // namespace

void InvokeOp(const OpInfo* op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
              const Params& p) {
  GradScalars(p);  // parsed, so that a malformed value is refused before the operator's own checks
  op->run(*op, in, outputs, p);
}

const std::vector<OpInfo> kCoreOps = {
    {"sgd_update", SgdAdam, kOptSGDSingle},
    {"sgd_mom_update", SgdAdam, kOptSGD},
    {"adam_update", SgdAdam, kOptAdam},
    {"mp_sgd_update", MpSgd, kOptSGDSingle},
    {"mp_sgd_mom_update", MpSgd, kOptSGD},
    {"multi_sgd_update", MultiSgd, 0},
    {"multi_sgd_mom_update", MultiSgd, kOpMom},
    {"multi_mp_sgd_update", MultiSgd, kOpMp},
    {"multi_mp_sgd_mom_update", MultiSgd, kOpMp | kOpMom},
    {"preloaded_multi_sgd_update", MultiSgd, kOpPreloaded},
    {"preloaded_multi_sgd_mom_update", MultiSgd, kOpPreloaded | kOpMom},
    {"preloaded_multi_mp_sgd_update", MultiSgd, kOpPreloaded | kOpMp},
    {"preloaded_multi_mp_sgd_mom_update", MultiSgd, kOpPreloaded | kOpMp | kOpMom},
    {"_copyto", Copy, 0},
    {"_plus", Binary, kEwAdd},
    {"elemwise_add", Binary, kEwAdd},
    {"_minus", Binary, kEwSub},
    {"elemwise_sub", Binary, kEwSub},
    {"_mul", Binary, kEwMul},
    {"elemwise_mul", Binary, kEwMul},
    {"_plus_scalar", Unary, kEwAddScalar},
    {"_mul_scalar", Unary, kEwMulScalar},
    {"sqrt", Unary, kEwSqrt},
    {"_set_value", SetValue, 0},
    {"_full", Full, 0},
    {"zeros_like", ZerosLike, 0},
    {"_sparse_zeros_like", ZerosLike, 0},
    {"cast", Cast, 0},
    {"Cast", Cast, 0},
};

}  // namespace b200kv
