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
//   all_finite, multi_all_finite          src/operator/contrib/all_finite.cc:42-166
//   reset_arrays                          src/operator/contrib/reset_arrays.cc:32-66
// Extensions without a reference operator (the reference composes them from NDArray arithmetic):
//   _b200kv_clip_global_norm              python/mxnet/gluon/utils.py:118-157
//   _b200kv_multi_scale                   python/mxnet/contrib/amp/amp.py:340-346 (unscale)
#include <algorithm>
#include <cmath>
#include <cstring>
#include <unordered_map>

#include "kernels.h"
#include "op_params.h"
#include "ops.h"

namespace b200kv {
namespace {

bool Aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

// One group (<= kMTMaxTensors tensors) of one operator call: device tables cached by the
// operands' addresses, like the dense kernel's plans. d[0]: the tensors, d[1]: their chunks,
// d[2]: n_partials floats per chunk.
const TableCache::Tables* GetPlan(int dev, int op, std::vector<MTTensor>* tensors, int n_partials,
                                  cudaStream_t st) {
  static auto* cache = new TableCache();
  std::vector<uint64_t> key{static_cast<uint64_t>(op), static_cast<uint64_t>(n_partials)};
  key.reserve(2 + 8 * tensors->size());
  for (auto& t : *tensors) {
    for (void* p : t.p) key.push_back(reinterpret_cast<uint64_t>(p));
    key.push_back((static_cast<uint64_t>(t.size) << 32) | t.aux);
    // vec_ok depends on the operands' dtypes as well as their addresses (a float16 array at an
    // 8-byte aligned address is vectorised, a float32 one there is not): a table cached for one
    // dtype must not serve another at the same addresses
    key.push_back(t.vec_ok);
  }
  if (const TableCache::Tables* hit = cache->Find(key)) return hit;
  auto plan = std::make_unique<TableCache::Tables>(dev);
  std::vector<MTChunk> chunks;
  for (size_t i = 0; i < tensors->size(); ++i) {
    MTTensor& t = (*tensors)[i];
    t.first_chunk = static_cast<uint32_t>(chunks.size());
    // 64-bit offset: for a size in (2^32 - kMTChunk, 2^32) a uint32 offset would wrap past the
    // last chunk and the loop would never end. Every chunk's own offset still fits in uint32.
    for (uint64_t off = 0; off < t.size; off += kMTChunk) {
      chunks.push_back(MTChunk{static_cast<uint32_t>(i), static_cast<uint32_t>(off),
                               static_cast<uint32_t>(std::min<uint64_t>(kMTChunk, t.size - off)), 0});
    }
  }
  plan->n_chunks = static_cast<int>(chunks.size());
  const size_t bt = tensors->size() * sizeof(MTTensor), nc = std::max<size_t>(chunks.size(), 1);
  plan->Upload(0, bt, tensors->data(), bt, st);
  plan->Upload(1, nc * sizeof(MTChunk), chunks.data(), chunks.size() * sizeof(MTChunk), st);
  plan->Upload(2, nc * sizeof(float) * std::max(n_partials, 1), nullptr, 0, st);
  return cache->Insert(std::move(key), std::move(plan));
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
    const TableCache::Tables* plan = GetPlan(c.dev, c.op, &group, c.n_partials, st);
    MTLaunch L;
    L.op = c.op;
    L.dtype = c.dtype;
    L.mp = c.mp;
    L.tensors = static_cast<const MTTensor*>(plan->d[0]);
    L.chunks = static_cast<const MTChunk*>(plan->d[1]);
    L.n_chunks = plan->n_chunks;
    std::memset(&L.s, 0, sizeof(L.s));
    for (size_t i = g0; i < g1 && i < c.per_tensor.size(); ++i) L.s.t[i - g0] = c.per_tensor[i];
    std::memcpy(L.s.f, c.f, sizeof(c.f));
    L.s.d0 = c.d0;
    L.s.d1 = c.d1;
    if (c.n_partials >= 1) L.part0 = static_cast<float*>(plan->d[2]);
    if (c.n_partials >= 2) L.part1 = static_cast<float*>(plan->d[2]) + std::max(plan->n_chunks, 1);
    LaunchMultiTensor(L, st);
    eng->CountLaunch("multi_tensor", 0);
    if (c.n_partials >= 1) {
      LaunchMultiTensorFinalize(L.tensors, static_cast<int>(group.size()), L.part0, L.part1, c.out0,
                                c.out1, st);
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

void CheckF32(const NDArray& a, size_t size, const char* what, const char* op) {
  KV_CHECK_EQ(a.dtype(), kFloat32) << op << ": " << what << " must be float32";
  KV_CHECK_EQ(a.Size(), size) << op << ": " << what << " shape mismatch";
}

// the weight32 input in[i] of an mp_ form, checked against the weight; none in the other forms
NDArray Weight32(const std::vector<NDArray>& in, size_t i, bool mp, const NDArray& w, const char* op) {
  if (mp) CheckF32(in[i], w.Size(), "weight32", op);
  return mp ? in[i] : NDArray();
}

void CheckMP(const NDArray& w, bool mp, const char* op) {
  if (mp) {
    KV_CHECK(DTypeSize(w.dtype()) == 2 && w.dtype() != kInt8)
        << op << ": the multi-precision form expects 16-bit weights";
  } else {
    KV_CHECK_EQ(w.dtype(), kFloat32)
        << op << ": 16-bit weights without an fp32 master copy are not supported on this path "
        << "(use the mp_ / multi_precision form)";
  }
}

// per-GPU scratch of _b200kv_clip_global_norm: [0] the factor, [1 ...] the tile partials. Every
// use is on the GPU's compute lane, so consecutive calls share it in stream order; it only grows.
struct ClipScratch {
  float* p = nullptr;
  size_t bytes = 0;
};
float* ClipScratchFor(int dev, size_t floats) {
  static auto* m = new std::unordered_map<int, ClipScratch>();
  ClipScratch& s = (*m)[dev];
  const size_t need = floats * sizeof(float);
  if (s.bytes < need) {
    Engine* eng = Engine::Get();
    if (s.p != nullptr) eng->Free(dev, s.p, s.bytes);
    s.bytes = std::max(need, 2 * s.bytes);
    s.p = static_cast<float*>(eng->Alloc(dev, s.bytes));
  }
  return s.p;
}

// The operand list both operators share, checked in full before anything is enqueued: float32,
// dense or row_sparse (its stored rows), one GPU, under 2^32 elements each, no memory listed twice.
// Returns the groups of <= kCNMaxArrays arrays with their tile counts.
struct ClipGroup {
  ClipNormArrays arrays{};
  uint32_t tiles = 0;
};
std::vector<ClipGroup> ClipOperands(const char* op, const std::vector<NDArray>& in, const Params& p,
                                    const char* scalar_key) {
  RejectUnknownKeys(p, {"num_arrays", scalar_key});
  const int num = Required<int>(p, "num_arrays", op);
  KV_CHECK(num >= 1) << op << ": num_arrays must be at least 1, got " << num;
  KV_CHECK_EQ(static_cast<int>(in.size()), num) << op << ": expected num_arrays inputs";
  KV_CHECK(in[0].on_gpu()) << op << " runs on GPU arrays only (no CPU fallback)";
  const int dev = in[0].dev();
  std::vector<ClipGroup> groups((num + kCNMaxArrays - 1) / kCNMaxArrays);
  std::vector<std::pair<uintptr_t, uintptr_t>> spans;  // [begin, end) of every non-empty operand
  for (int i = 0; i < num; ++i) {
    const NDArray& a = in[i];
    KV_CHECK(a.on_gpu() && a.dev() == dev)
        << op << ": array_" << i << " is not on array_0's GPU; all operands must be on the same GPU "
        << "(no CPU fallback)";
    KV_CHECK(a.dtype() == kFloat32)
        << op << ": array_" << i << " is " << DTypeName(a.dtype())
        << "; only float32 is served (16-bit gradients are not served yet)";
    KV_CHECK(a.stype() == kDefaultStorage || a.stype() == kRowSparseStorage)
        << op << ": array_" << i << " has csr storage; dense and row_sparse arrays are served";
    const bool rsp = a.stype() == kRowSparseStorage;
    const uint64_t n = rsp ? static_cast<uint64_t>(a.nnr()) * a.RowLength() : a.Size();
    KV_CHECK(n < (1ULL << 32)) << op << ": array_" << i << " has 2^32 or more elements";
    ClipNormArrays& A = groups[i / kCNMaxArrays].arrays;
    A.n[i % kCNMaxArrays] = static_cast<uint32_t>(n);
    A.p[i % kCNMaxArrays] = n > 0 ? static_cast<float*>(a.data()) : nullptr;
    A.count = i % kCNMaxArrays + 1;
    if (n > 0) {
      const uintptr_t b = reinterpret_cast<uintptr_t>(a.data());
      spans.emplace_back(b, b + n * sizeof(float));
    }
  }
  std::sort(spans.begin(), spans.end());
  for (size_t i = 1; i < spans.size(); ++i) {
    KV_CHECK(spans[i].first >= spans[i - 1].second)
        << op << ": two operands share memory (the same storage listed twice); each would be scaled twice";
  }
  uint64_t total = 0;
  for (ClipGroup& g : groups) total += g.tiles = ClipNormTiles(g.arrays);
  KV_CHECK(total < (1ULL << 31)) << op << ": more than 2^31 tiles of " << kCNTileBytes << " bytes";
  return groups;
}

void MultiSumSq(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                const Params& p) {
  const int num = GetI(p, "num_arrays", -1);
  KV_CHECK(num >= 1) << "Required parameter num_arrays of multi_sum_sq is missing";
  KV_CHECK_EQ(static_cast<int>(in.size()), num) << "multi_sum_sq: expected num_arrays inputs";
  Call c;
  c.op = kMTSumSq;
  c.dtype = in[0].dtype();
  c.dev = in[0].dev();
  KV_CHECK(in[0].on_gpu()) << "multi_sum_sq runs on GPU arrays only (no CPU fallback)";
  NDArray out = OutOr(outputs, 0, {num}, in[0].ctx(), kFloat32);
  CheckF32(out, num, "out", op.name);
  for (int i = 0; i < num; ++i) {
    KV_CHECK_EQ(in[i].dtype(), c.dtype) << "multi_sum_sq: array_" << i << " dtype differs from array_0";
    c.tensors.push_back(Tensor({&in[i]}, in[i].Size(), i, c.dtype));
    c.reads.push_back(in[i]);
  }
  c.n_partials = 1;
  c.out0 = static_cast<float*>(out.data());
  c.writes.push_back(out);
  Run(c);
}

// all_finite, multi_all_finite (variant: kOpMulti)
void AllFinite(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
               const Params& p) {
  const char* n = op.name;
  const bool multi = op.variant & kOpMulti;
  if (multi) RejectUnknownKeys(p, {"num_arrays", "init_output"});  // MultiAllFiniteParam
  else RejectUnknownKeys(p, {"init_output"});                        // AllFiniteParam
  const int num = multi ? GetI(p, "num_arrays", 1) : 1;
  KV_CHECK(num >= 1 && num <= kAFMaxArrays)
      << n << ": num_arrays must be in 1.." << kAFMaxArrays << ", got " << num;
  KV_CHECK_EQ(static_cast<int>(in.size()), num) << n << ": expected num_arrays inputs";
  const bool init = GetB(p, "init_output", true);
  const int dtype = in[0].dtype();
  KV_CHECK(dtype == kFloat16 || dtype == kBfloat16 || dtype == kFloat32 || dtype == kFloat64)
      << "This operation only support floating point types, not " << DTypeName(dtype);
  KV_CHECK(in[0].on_gpu()) << n << " runs on GPU arrays only (no CPU fallback)";
  const int dev = in[0].dev();
  AllFiniteArrays arrays;
  arrays.count = num;
  for (int i = 0; i < num; ++i) {
    const NDArray& a = in[i];
    KV_CHECK(a.on_gpu() && a.dev() == dev) << "all operands must be on the same GPU (no CPU fallback)";
    KV_CHECK_EQ(a.dtype(), dtype) << n << ": array_" << i << " dtype differs from array_0";
    // a row_sparse array's absent rows are zeros, which are finite: its stored rows decide
    const bool rsp = a.stype() == kRowSparseStorage;
    arrays.n[i] = rsp ? static_cast<uint64_t>(a.nnr()) * a.RowLength() : a.Size();
    arrays.p[i] = arrays.n[i] > 0 ? a.data() : nullptr;
  }
  NDArray out = OutOr(outputs, 0, {1}, in[0].ctx(), kFloat32);
  KV_CHECK(out.stype() == kDefaultStorage && out.dtype() == kFloat32 && out.Size() == 1)
      << n << ": out must be a float32 array of one element";
  KV_CHECK(out.on_gpu() && out.dev() == dev) << "all operands must be on the same GPU (no CPU fallback)";
  LaneOp lop(dev);
  for (const NDArray& a : in) lop.Read(a);
  lop.Write(out);
  Engine* eng = Engine::Get();
  if (init) {
    LaunchElementwise(kEwFill, kFloat32, out.data(), nullptr, nullptr, 1.0f, 1, lop.stream());
    eng->CountLaunch("elementwise", 0);
  }
  LaunchAllFinite(dtype, arrays, static_cast<float*>(out.data()), lop.stream());
  eng->CountLaunch("all_finite", 0);
  lop.Issue();
}

void ClipGlobalNorm(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                    const Params& p) {
  const char* n = op.name;
  std::vector<ClipGroup> groups = ClipOperands(n, in, p, "max_norm");
  const float max_norm = StodF(p, "max_norm", n);
  KV_CHECK(max_norm > 0.f) << n << ": max_norm must be positive and not nan, got "
                           << *Find(p, "max_norm");
  const int dev = in[0].dev();
  if (!outputs->empty()) {
    const NDArray& o = (*outputs)[0];
    KV_CHECK(o.stype() == kDefaultStorage && o.dtype() == kFloat32 && o.shape().size() == 1 &&
             o.shape()[0] == 1 && o.on_gpu() && o.dev() == dev)
        << n << ": total_norm must be a dense (1,) float32 array on the inputs' GPU";
  }
  NDArray norm = OutOr(outputs, 0, {1}, in[0].ctx(), kFloat32);
  uint32_t total = 0;
  for (const ClipGroup& g : groups) total += g.tiles;
  LaneOp lop(dev);
  for (const NDArray& a : in) lop.Write(a);
  lop.Write(norm);
  Engine* eng = Engine::Get();
  float* scratch = ClipScratchFor(dev, 1 + static_cast<size_t>(total));
  uint32_t off = 0;
  for (const ClipGroup& g : groups) {
    if (g.tiles == 0) continue;  // only empty arrays: nothing to read
    LaunchClipNormPartial(g.arrays, g.tiles, scratch + 1 + off, lop.stream());
    eng->CountLaunch("clip_norm_partial", 0);
    off += g.tiles;
  }
  LaunchClipNormFold(scratch + 1, total, max_norm, static_cast<float*>(norm.data()), scratch, lop.stream());
  eng->CountLaunch("clip_norm_fold", 0);
  for (const ClipGroup& g : groups) {
    if (g.tiles == 0) continue;
    LaunchClipNormScale(g.arrays, g.tiles, scratch, 1.f, lop.stream());
    eng->CountLaunch("clip_norm_scale", 0);
  }
  lop.Issue();
}

void MultiScale(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                const Params& p) {
  const char* n = op.name;
  std::vector<ClipGroup> groups = ClipOperands(n, in, p, "scalar");
  const float scalar = StodF(p, "scalar", n);
  KV_CHECK(outputs->empty()) << n << " scales its inputs in place and has no output";
  LaneOp lop(in[0].dev());
  for (const NDArray& a : in) lop.Write(a);
  for (const ClipGroup& g : groups) {
    if (g.tiles == 0) continue;
    LaunchClipNormScale(g.arrays, g.tiles, nullptr, scalar, lop.stream());
    Engine::Get()->CountLaunch("clip_norm_scale", 0);
  }
  lop.Issue();
}

void ResetArrays(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                 const Params& p) {
  const char* n = op.name;
  RejectUnknownKeys(p, {"num_arrays"});  // ResetArraysParam
  const int num = Required<int>(p, "num_arrays", n);
  KV_CHECK(num >= 1) << n << ": num_arrays must be at least 1, got " << num;
  KV_CHECK_EQ(static_cast<int>(in.size()), num) << n << ": expected num_arrays inputs";
  KV_CHECK(outputs->empty()) << n << " zeroes its inputs in place and has no output";
  KV_CHECK(in[0].on_gpu()) << n << " runs on GPU arrays only (no CPU fallback)";
  const int dev = in[0].dev();
  std::vector<ResetArraysList> groups;  // the dense arrays with bytes to write
  for (int i = 0; i < num; ++i) {
    const NDArray& a = in[i];
    KV_CHECK(a.on_gpu() && a.dev() == dev)
        << n << ": array_" << i << " is not on array_0's GPU; all operands must be on the same GPU "
        << "(no CPU fallback)";
    // MSHADOW_REAL_TYPE_SWITCH (mshadow/base.h:1130-1143), plus bfloat16 as all_finite serves it
    switch (a.dtype()) {
      case kFloat16: case kBfloat16: case kFloat32: case kFloat64: break;
      case kUint8: KV_FATAL << "This operation only support floating point types not uint8";
      case kInt8: KV_FATAL << "This operation only support floating point types not int8";
      case kInt32: KV_FATAL << "This operation only support floating point types, not int32";
      case kInt64: KV_FATAL << "This operation only support floating point types, not int64";
      default: KV_FATAL << n << ": array_" << i << " has unsupported dtype " << DTypeName(a.dtype());
    }
    KV_CHECK(a.stype() == kDefaultStorage || a.stype() == kRowSparseStorage)
        << n << ": array_" << i << " has csr storage; dense and row_sparse arrays are served";
    if (a.stype() != kDefaultStorage || a.ByteSize() == 0) continue;
    if (groups.empty() || groups.back().count == kRAMaxArrays) {
      groups.emplace_back();
      groups.back().count = 0;
    }
    ResetArraysList& g = groups.back();
    g.p[g.count] = a.data();
    g.bytes[g.count] = a.ByteSize();
    ++g.count;
  }
  // every input is written (FMutateInputs): the zeroing follows pending readers and writers of
  // each, and a pull anchor hands its value back to the store first
  LaneOp lop(dev);
  for (const NDArray& a : in) lop.Write(a);
  Engine* eng = Engine::Get();
  for (ResetArraysList& g : groups) {
    if (LaunchResetArrays(g, lop.stream()) > 0) eng->CountLaunch("reset_arrays", 0);
  }
  lop.Issue();
  // a row_sparse input keeps its storage and stores no rows, where the reference's storage
  // fallback leaves it (dense temp, zeroed, cast back: imperative_utils.h:419-444). Work issued
  // before this call read its rows already; the write declared above orders whatever follows.
  for (const NDArray& a : in) {
    if (a.stype() == kRowSparseStorage) a.SetNnr(0);
  }
}

void MultiLars(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
               const Params& p) {
  const char* n = op.name;
  KV_CHECK_EQ(in.size(), 4u) << "multi_lars expects lrs, weights_sum_sq, grads_sum_sq, wds";
  if (in[0].dtype() != kFloat32) KV_FATAL << "MultiLARS only support float";
  const size_t cnt = in[1].Size();
  for (int i = 0; i < 4; ++i) CheckF32(in[i], cnt, "input", n);
  NDArray out = OutOr(outputs, 0, in[0].shape(), in[0].ctx(), kFloat32);
  CheckF32(out, cnt, "out", n);
  const float eta = Required(p, "eta", n), eps = Required(p, "eps", n);
  const float rescale = GetF(p, "rescale_grad", 1.0f);
  KV_CHECK(in[0].on_gpu()) << "multi_lars runs on GPU arrays only (no CPU fallback)";
  LaneOp lop(in[0].dev());
  lop.Read(in[0]).Read(in[1]).Read(in[2]).Read(in[3]).Write(out);
  LaunchMultiLars(static_cast<int>(cnt), static_cast<float*>(out.data()),
                  static_cast<const float*>(in[0].data()), static_cast<const float*>(in[1].data()),
                  static_cast<const float*>(in[2].data()), static_cast<const float*>(in[3].data()),
                  eta, eps, rescale, lop.stream());
  Engine::Get()->CountLaunch("multi_lars", 0);
  lop.Issue();
}

// _adamw_update and its mp / multi forms (variant: kOpMulti | kOpMp)
void AdamW(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
           const Params& p) {
  const char* n = op.name;
  const bool multi = op.variant & kOpMulti;
  const bool mp = op.variant & kOpMp;
  const int stride = mp ? 5 : 4;
  const int num = multi ? GetI(p, "num_weights", 1) : 1;
  KV_CHECK(num >= 1) << n << ": num_weights must be at least 1, got " << num;
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
    NDArray w32 = Weight32(in, i * stride + 4, mp, w, n);
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
}

// lamb_update_phase1 / 2 and their mp_ forms (variant: kOpMp)
void LambPhase1(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                const Params& p) {
  const char* n = op.name;
  const bool mp = op.variant & kOpMp;
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
  const int t = Required<int>(p, "t", n);
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
  NDArray w32 = Weight32(in, 4, mp, w, n);
  if (mp) c.reads.push_back(w32);
  c.tensors.push_back(Tensor({&w, &g, &mean, &var, mp ? &w32 : nullptr, &out}, w.Size(), 0, c.dtype));
  c.reads.push_back(w);
  c.reads.push_back(g);
  c.writes.push_back(mean);
  c.writes.push_back(var);
  c.writes.push_back(out);
  Run(c);
}

void LambPhase2(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                const Params& p) {
  const char* n = op.name;
  const bool mp = op.variant & kOpMp;
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
  NDArray w32 = Weight32(in, 4, mp, w, n);
  if (mp) c.reads.push_back(w32);
  c.tensors.push_back(Tensor({&w, &g, nullptr, nullptr, mp ? &w32 : nullptr, &out}, w.Size(), 0, c.dtype));
  if (!out.SameStorage(w)) c.reads.push_back(w);
  c.reads.push_back(g);
  c.reads.push_back(r1);
  c.reads.push_back(r2);
  c.writes.push_back(out);
  Run(c);
}

// _multi_lamb_update, _multi_mp_lamb_update (variant: kOpMp)
void MultiLamb(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
               const Params& p) {
  const char* n = op.name;
  const bool mp = op.variant & kOpMp;
  const int stride = mp ? 5 : 4;
  const int num = GetI(p, "num_tensors", 1);
  KV_CHECK(num >= 1) << n << ": num_tensors must be at least 1, got " << num;
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
    NDArray w32 = Weight32(in, i * stride + 4, mp, w, n);
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
}

}  // namespace

const std::vector<OpInfo> kMultiTensorOps = {
    {"multi_sum_sq", MultiSumSq, 0},
    {"all_finite", AllFinite, 0},
    {"multi_all_finite", AllFinite, kOpMulti},
    {"_b200kv_clip_global_norm", ClipGlobalNorm, 0},
    {"_b200kv_multi_scale", MultiScale, 0},
    {"reset_arrays", ResetArrays, 0},
    {"multi_lars", MultiLars, 0},
    {"_adamw_update", AdamW, 0},
    {"_mp_adamw_update", AdamW, kOpMp},
    {"_multi_adamw_update", AdamW, kOpMulti},
    {"_multi_mp_adamw_update", AdamW, kOpMulti | kOpMp},
    {"lamb_update_phase1", LambPhase1, 0},
    {"mp_lamb_update_phase1", LambPhase1, kOpMp},
    {"lamb_update_phase2", LambPhase2, 0},
    {"mp_lamb_update_phase2", LambPhase2, kOpMp},
    {"_multi_lamb_update", MultiLamb, 0},
    {"_multi_mp_lamb_update", MultiLamb, kOpMp},
};

}  // namespace b200kv
