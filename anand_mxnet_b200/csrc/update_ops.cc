// update_ops.cc -- host side of the single-tensor optimizer operators that the reference's NAG,
// Signum, RMSProp, FTML and Ftrl optimizers call from their `update` (the per-key updater callback
// of the store, and the local updaters of update_on_kvstore=False), plus the row_sparse forms of
// ftrl_update, AdaGrad's _sparse_adagrad_update and GroupAdaGrad's _contrib_group_adagrad_update.
// Kernels: update_kernels.cu (dense), rowsparse_kernels.cu (row_sparse).
//
// Reference operator definitions (inputs, parameter structs, kernels):
//   nag_mom_update, mp_nag_mom_update    src/operator/optimizer_op.cc:712-762, optimizer_op-inl.h:1032-1160
//   ftml_update                          optimizer_op.cc:626-660, optimizer_op-inl.h:1163-1249
//   rmsprop_update, rmspropalex_update   optimizer_op.cc:763-853, optimizer_op-inl.h:1915-2099
//   ftrl_update, _sparse_ftrl_update     optimizer_op.cc:854-893, optimizer_op-inl.h:2101-2314
//   signsgd_update, signum_update        optimizer_op.cc:49-104, optimizer_op-inl.h:2319-2452
//   _sparse_adagrad_update               optimizer_op.cc:895-924, optimizer_op-inl.h:2454-2649
//   _contrib_group_adagrad_update        contrib/optimizer_op.cc:53-86, contrib/optimizer_op-inl.h:46-243
//
// Dense float32 arrays (mp_nag_mom_update: float16 / bfloat16 weights with float32 mom and
// weight32), or the row_sparse forms in float32 (RspUpdateOp). The reference would densify a
// row_sparse gradient of a dense-weight ftrl_update and run 16-bit weights of the other operators
// in half precision; both are refused here before anything is launched.
#include <cctype>
#include <cerrno>
#include <cmath>
#include <limits>

#include "kernels.h"
#include "op_params.h"
#include "ops.h"

namespace b200kv {
namespace {

struct Spec {
  const char* name;
  int op;
  int nin;                 // weight, grad, states...
  const char* launch_name; // CountLaunch keeps the pointer
  int bytes_per_elem;      // algorithmic traffic of one element (float32 / mp float16)
};

const Spec kSpecs[] = {
    {"nag_mom_update", kUpdNAG, 3, "update_op(nag_mom_update)", 20},
    {"mp_nag_mom_update", kUpdMPNAG, 4, "update_op(mp_nag_mom_update)", 20},
    {"signsgd_update", kUpdSignSGD, 2, "update_op(signsgd_update)", 12},
    {"signum_update", kUpdSignum, 3, "update_op(signum_update)", 20},
    {"rmsprop_update", kUpdRMSProp, 3, "update_op(rmsprop_update)", 20},
    {"rmspropalex_update", kUpdRMSPropAlex, 5, "update_op(rmspropalex_update)", 36},
    {"ftml_update", kUpdFTML, 5, "update_op(ftml_update)", 36},
    {"ftrl_update", kUpdFtrl, 4, "update_op(ftrl_update)", 28},
    // row_sparse only: the alias of ftrl_update (MXNET_ADD_SPARSE_OP_ALIAS, optimizer_op.cc:855)
    // and AdaGrad's operator (optimizer_op.cc:895-924, optimizer_op-inl.h:2454-2649)
    {"_sparse_ftrl_update", kUpdFtrl, 4, "update_op(ftrl_update)", 28},
    {"_sparse_adagrad_update", kUpdAdaGrad, 3, "update_op(_sparse_adagrad_update)", 20},
    // GroupAdaGrad's operator: g 4 + w 4+4 per element; the history is one float per row
    {"_contrib_group_adagrad_update", kUpdGroupAdaGrad, 3, "update_op(_contrib_group_adagrad_update)", 12},
};

// Restatement of dmlc::stod == ParseFloat<double, true> (3rdparty/dmlc-core/include/dmlc/
// strtonum.h:99-254, 497-510), the parser of double fields (FieldEntry<double>, parameter.h:1106-1125)
// such as FTML's epsilon. Like stof it is not correctly rounded: float(int part) + double(frac
// digits) / double(10^k), then scaled by powers of ten.
double DmlcStod(const std::string& s) {
  constexpr unsigned kMaxExponent = 308U;
  constexpr double kMaxSigForMaxExp = 1.79769313486231570;
  constexpr double kMaxSigForNegMaxExp = 2.22507385850720139;
  constexpr int kStrtofMaxDigits = 19;
  const char* p = s.c_str();
  while (std::isspace(static_cast<unsigned char>(*p))) ++p;
  bool positive = true;
  if (*p == '-') {
    positive = false;
    ++p;
  } else if (*p == '+') {
    ++p;
  }
  auto finish = [&](double value, const char* end) -> double {
    KV_CHECK(end != s.c_str() && *end == '\0')
        << "Invalid Parameter format: expect double but value='" << s << "'";
    return value;
  };
  {
    int i = 0;
    while (i < 8 && static_cast<char>((*p) | 32) == "infinity"[i]) { ++i; ++p; }
    if (i == 3 || i == 8) {
      return finish(positive ? std::numeric_limits<double>::infinity()
                             : -std::numeric_limits<double>::infinity(), p);
    }
    p -= i;
    i = 0;
    while (i < 3 && static_cast<char>((*p) | 32) == "nan"[i]) { ++i; ++p; }
    if (i == 3) return finish(std::numeric_limits<double>::quiet_NaN(), p);
    p -= i;
  }
  const char* num_start = p;
  uint64_t predec = 0;
  for (; std::isdigit(static_cast<unsigned char>(*p)); ++p) {
    predec = predec * 10ULL + static_cast<uint64_t>(*p - '0');
  }
  double value = static_cast<double>(predec);
  if (*p == '.') {
    uint64_t pow10 = 1, val2 = 0;
    int digit_cnt = 0;
    ++p;
    while (std::isdigit(static_cast<unsigned char>(*p))) {
      if (digit_cnt < kStrtofMaxDigits) {
        val2 = val2 * 10ULL + static_cast<uint64_t>(*p - '0');
        pow10 *= 10ULL;
      }
      ++p;
      ++digit_cnt;
    }
    value += static_cast<double>(val2) / static_cast<double>(pow10);
  }
  KV_CHECK(p != num_start) << "Invalid Parameter format: expect double but value='" << s << "'";
  if (*p == 'e' || *p == 'E') {
    ++p;
    bool frac = false;
    double scale = 1.0;
    unsigned expon = 0;
    if (*p == '-') {
      frac = true;
      ++p;
    } else if (*p == '+') {
      ++p;
    }
    for (; std::isdigit(static_cast<unsigned char>(*p)); ++p) {
      expon = expon * 10U + static_cast<unsigned>(*p - '0');
    }
    KV_CHECK(expon <= kMaxExponent) << "Out of range value '" << s << "'";
    KV_CHECK(!(expon == kMaxExponent && ((!frac && value > kMaxSigForMaxExp) ||
                                         (frac && value < kMaxSigForNegMaxExp))))
        << "Out of range value '" << s << "'";
    while (expon >= 8U) { scale *= static_cast<double>(1E8f); expon -= 8U; }
    while (expon > 0U) { scale *= static_cast<double>(10.0f); expon -= 1U; }
    value = frac ? (value / scale) : (value * scale);
  }
  if (*p == 'f' || *p == 'F') ++p;
  return finish(positive ? value : -value, p);
}

float Required(const Params& p, const char* key, const std::string& op) {
  KV_CHECK(Find(p, key) != nullptr) << "Required parameter " << key << " of " << op << " is missing";
  return GetF(p, key, 0.f);
}

// dmlc::Parameter set_range(lo, hi) (parameter.h:752-762)
float InRange(float v, const char* key, float lo, float hi) {
  KV_CHECK(!(v < lo || v > hi)) << "value " << v << " for Parameter " << key << " exceed bound [" << lo
                                << ',' << hi << ']';
  return v;
}

const char* StypeName(int stype) { return stype == kRowSparseStorage ? "row_sparse" : "default"; }

// ftrl_update (FtrlUpdateEx, optimizer_op-inl.h:2291-2314), _sparse_adagrad_update
// (AdagradStorageType / AdagradUpdateEx, 2480-2501, 2620-2649) and _contrib_group_adagrad_update
// (GroupAdagradStorageType / GroupAdagradUpdateEx, contrib/optimizer_op-inl.h:67-93, 216-242) with
// row_sparse operands: only the rows listed in the gradient move. Every check runs before anything
// is enqueued, so a refused call leaves all operands as they were. Accepted forms:
//   ftrl_update / _sparse_ftrl_update   (row_sparse weight, grad, z, n)
//   _sparse_adagrad_update              (row_sparse weight, grad, history), wd == 0
//                                       (dense weight, row_sparse grad, dense history), wd == 0
//   _contrib_group_adagrad_update       the same two forms; history has one value per row
void RspUpdateOp(const Spec& spec, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
                 const Params& p) {
  const std::string n = spec.name;
  const int op = spec.op;
  const NDArray& w = in[0];
  const NDArray& g = in[1];
  const int wst = w.stype();
  UpdateLaunch L;
  L.op = op;
  L.dtype = kFloat32;
  L.lr = Required(p, "lr", n);
  L.wd = GetF(p, "wd", 0.f);
  L.rescale = GetF(p, "rescale_grad", 1.0f);
  L.clip = GetF(p, "clip_gradient", -1.0f);
  if (op == kUpdFtrl) {  // FtrlParam
    L.lamda1 = GetF(p, "lamda1", 0.01f);
    L.beta = GetF(p, "beta", 1.0f);
    KV_CHECK(wst == kRowSparseStorage && g.stype() == kRowSparseStorage)
        << n << ": the row_sparse form needs row_sparse weight, grad, z and n (a dense weight with a "
        << "row_sparse gradient is not supported)";
  } else if (op == kUpdGroupAdaGrad) {  // GroupAdagradParam (contrib/optimizer_op-inl.h:46-65)
    for (const auto& kv : p) {  // dmlc::Parameter::Init rejects unknown keys (wd among them)
      KV_CHECK(kv.first == "lr" || kv.first == "rescale_grad" || kv.first == "clip_gradient" ||
               kv.first == "epsilon")
          << "Cannot find argument '" << kv.first << "', Possible Arguments: lr, rescale_grad, "
          << "clip_gradient, epsilon";
    }
    L.eps = GetF(p, "epsilon", 1.0e-5f);
    const int hst = in[2].stype();
    // all-dense operands dispatch to an FCompute the reference does not register
    KV_CHECK(g.stype() == kRowSparseStorage || wst != kDefaultStorage || hst != kDefaultStorage)
        << "Operator " << n << " is not implemented for GPU (dense weight, grad and history)";
    KV_CHECK(g.stype() == kRowSparseStorage && hst == wst)  // GroupAdagradStorageType (:67-93)
        << "Operator not implemented: operator = " << n << "\ninput storage types = ["
        << StypeName(wst) << ", " << StypeName(g.stype()) << ", " << StypeName(hst) << ", ]";
  } else {  // AdagradParam; AdagradUpdateDnsRspDnsImpl (2569-2570) checks wd first
    L.eps = GetF(p, "epsilon", 1.0e-7f);
    KV_CHECK(L.wd == 0.f) << "sparse adagrad_update does not support wd.";
    KV_CHECK(g.stype() == kRowSparseStorage && in[2].stype() == wst)
        << n << ": supported storage types are (row_sparse, row_sparse, row_sparse) and (default, "
        << "row_sparse, default), got (" << StypeName(wst) << ", " << StypeName(g.stype()) << ", "
        << StypeName(in[2].stype()) << ")";
  }
  KV_CHECK(!w.shape().empty()) << n << ": the weight needs at least one dimension";
  const int64_t rows = w.shape()[0];
  for (size_t i = 0; i < in.size(); ++i) {
    const NDArray& a = in[i];
    KV_CHECK(a.on_gpu() && a.dev() == w.dev()) << n << ": all operands must be on the same GPU";
    KV_CHECK_EQ(a.dtype(), kFloat32) << n << ": row_sparse updates run on float32 arrays only, got "
                                     << DTypeName(a.dtype());
    if (op == kUpdGroupAdaGrad && i == 2) {
      // GroupAdagradShape (contrib/optimizer_op.cc:37-51) checks only history.shape[0]; the kernel
      // addresses one value per row, so a wider history is refused here
      KV_CHECK(!a.shape().empty() && a.shape()[0] == rows && a.Size() == static_cast<size_t>(rows))
          << n << ": history must hold one value per weight row, e.g. shape (" << rows << ", 1)";
    } else {
      KV_CHECK(a.shape() == w.shape()) << n << ": weight / grad / state shape mismatch";
    }
  }
  // CheckAllRowsPresent (operator_common.h:500-511)
  const char* func = op == kUpdFtrl ? "FtrlUpdate" : op == kUpdAdaGrad ? "AdagradUpdate" : "GroupAdagradUpdate";
  KV_CHECK(wst != kRowSparseStorage || w.nnr() == rows)
      << func << " for RowSparse weights is only implemented for RowSparse weights with all rows "
      << "containing non-zeros. Expects weights.data.shape[0] (" << w.nnr() << ") == weights.shape[0] ("
      << rows << ").";
  // the states' rows are addressed by the table row id, like the weight's: a row_sparse state holds
  // every row, or none yet (then it is zero-filled first, FillDnsZerosRspImpl)
  for (size_t i = 2; i < in.size(); ++i) {
    KV_CHECK(in[i].stype() != kRowSparseStorage || in[i].nnr() == 0 || in[i].nnr() == rows)
        << n << ": a row_sparse optimizer state must hold every row or none (it holds "
        << in[i].nnr() << " of " << rows << ")";
  }
  // kWriteInplace is expected (optimizer_op-inl.h:2235, 2572)
  KV_CHECK(outputs->size() == 1 && (*outputs)[0].SameStorage(w) && (*outputs)[0].stype() == wst &&
           (*outputs)[0].data() == w.data())
      << n << ": out must be the weight itself (kWriteInplace is expected for sparse " << spec.name
      << ")";

  Engine* eng = Engine::Get();
  LaneOp lop(w.dev());
  std::vector<const NDArray*> fill;
  for (size_t i = 2; i < in.size(); ++i) {
    if (in[i].stype() == kRowSparseStorage && in[i].nnr() == 0) {
      in[i].CheckAndAllocRows(rows);
      fill.push_back(&in[i]);
    }
  }
  const bool update = g.storage_initialized();
  if (!update && fill.empty()) return;  // an all-zero gradient changes nothing
  if (update) lop.Read(g);
  lop.Write(w);
  for (size_t i = 2; i < in.size(); ++i) lop.Write(in[i]);
  cudaStream_t st = lop.stream();
  for (const NDArray* a : fill) {
    KV_CUDA(cudaMemsetAsync(a->data(), 0, static_cast<size_t>(rows) * a->RowLength() * sizeof(float), st));
    LaunchFillRowIds(a->row_ids(), rows, st);
    eng->CountLaunch(spec.launch_name, static_cast<uint64_t>(rows) * (a->RowLength() * 4 + 8));
  }
  if (update) {
    L.w = w.data();
    L.out = w.data();
    L.g = g.data();
    L.gidx = g.row_ids();
    L.nnr = g.nnr();
    L.row_len = static_cast<int64_t>(w.RowLength());
    for (size_t i = 2; i < in.size(); ++i) L.s[i - 2] = static_cast<float*>(in[i].data());
    LaunchRspRowUpdateOp(L, st);
    // + 8 B of id per row, and GroupAdaGrad's history value read and written
    const int64_t per_row = op == kUpdGroupAdaGrad ? 16 : 8;
    eng->CountLaunch(spec.launch_name,
                     static_cast<uint64_t>(L.nnr) * (spec.bytes_per_elem * L.row_len + per_row));
  }
  lop.Issue();
}

}  // namespace

bool UpdateOp(const std::string& n, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
              const Params& p) {
  const Spec* spec = nullptr;
  for (const Spec& s : kSpecs) {
    if (n == s.name) spec = &s;
  }
  if (spec == nullptr) return false;
  const int op = spec->op;
  KV_CHECK_EQ(static_cast<int>(in.size()), spec->nin) << n << " expects " << spec->nin << " inputs";
  const NDArray& w = in[0];
  const NDArray& g = in[1];
  if (op == kUpdFtrl) {  // FtrlUpdateEx (optimizer_op-inl.h:2303-2306)
    for (int i : {2, 3}) {
      KV_CHECK(in[i].stype() == w.stype())
          << "Inconsistent storage type detected between  " << (i == 2 ? "z" : "n") << ".stype = "
          << in[i].stype() << " and weight.stype = " << w.stype();
    }
  }
  if (op == kUpdAdaGrad || op == kUpdGroupAdaGrad || w.stype() == kRowSparseStorage) {
    RspUpdateOp(*spec, in, outputs, p);
    return true;
  }
  for (const NDArray& a : in) {
    KV_CHECK(a.stype() == kDefaultStorage)
        << n << ": row_sparse weights, gradients or states are not supported (dense arrays only)";
  }
  KV_CHECK(w.on_gpu()) << n << " runs on GPU arrays only (no CPU fallback)";
  const int dev = w.dev();
  const int dtype = w.dtype();
  if (op == kUpdMPNAG) {
    KV_CHECK(dtype == kFloat16 || dtype == kBfloat16)
        << n << ": the multi-precision form expects float16 / bfloat16 weights, got " << DTypeName(dtype);
  } else {
    KV_CHECK_EQ(dtype, kFloat32)
        << n << ": " << DTypeName(dtype) << " weights without an fp32 master copy are not supported "
        << "(float32 only; use multi_precision=True for 16-bit weights)";
  }
  for (const NDArray& a : in) {
    KV_CHECK(a.on_gpu() && a.dev() == dev) << n << ": all operands must be on the same GPU";
  }
  KV_CHECK_EQ(g.dtype(), dtype) << n << ": weight / grad dtype mismatch";
  KV_CHECK_EQ(g.Size(), w.Size()) << n << ": weight / grad shape mismatch";
  for (int i = 2; i < spec->nin; ++i) {
    KV_CHECK_EQ(in[i].dtype(), kFloat32) << n << ": optimizer states must be float32";
    KV_CHECK_EQ(in[i].Size(), w.Size()) << n << ": state shape mismatch";
  }
  NDArray out;
  if (outputs->empty()) {
    out = NDArray(w.shape(), w.ctx(), dtype);
    outputs->push_back(out);
  } else {
    out = (*outputs)[0];
  }
  KV_CHECK(out.on_gpu() && out.dev() == dev) << n << ": out must be on the weight's GPU";
  KV_CHECK(out.stype() == kDefaultStorage) << n << ": out must be a dense array";
  KV_CHECK_EQ(out.dtype(), dtype) << n << ": out dtype mismatch";
  KV_CHECK_EQ(out.Size(), w.Size()) << n << ": out shape mismatch";
  const bool out_is_w = out.SameStorage(w);
  KV_CHECK(!out_is_w || out.data() == w.data()) << n << ": out overlaps the weight without being it";

  UpdateLaunch L;
  L.op = op;
  L.dtype = dtype;
  L.lr = Required(p, "lr", n);
  L.wd = GetF(p, "wd", 0.f);
  L.rescale = GetF(p, "rescale_grad", 1.0f);
  L.clip = GetF(p, "clip_gradient", -1.0f);
  switch (op) {
    case kUpdNAG: case kUpdMPNAG:  // NAGMomParam
      L.momentum = GetF(p, "momentum", 0.f);
      break;
    case kUpdSignSGD:  // SignSGDParam
      break;
    case kUpdSignum:  // SignumParam
      L.momentum = GetF(p, "momentum", 0.f);
      L.wd_lh = GetF(p, "wd_lh", 0.f);
      break;
    case kUpdRMSProp: case kUpdRMSPropAlex:  // RMSPropParam, RMSPropAlexParam
      L.gamma1 = GetF(p, "gamma1", 0.95f);
      L.gamma2 = GetF(p, "gamma2", 0.9f);
      L.eps = GetF(p, "epsilon", 1e-8f);
      L.clip_weights = GetF(p, "clip_weights", -1.0f);
      break;
    case kUpdFTML: {  // FTMLParam: epsilon is a double field, the clip field is clip_grad
      L.beta1 = InRange(GetF(p, "beta1", 0.6f), "beta1", 0.f, 1.f);
      L.beta2 = InRange(GetF(p, "beta2", 0.999f), "beta2", 0.f, 1.f);
      const std::string* e = Find(p, "epsilon");
      L.eps = static_cast<float>(e ? DmlcStod(*e) : static_cast<double>(1e-8f));
      KV_CHECK(Find(p, "t") != nullptr) << "Required parameter t of " << n << " is missing";
      const int t = GetI(p, "t", 0);
      L.clip = GetF(p, "clip_grad", -1.0f);
      // power::Map(beta, DType(t)) is ::powf of the host C library (math_functions-inl.h:58-61,126):
      // evaluated here once per call rather than with the device's powf
      L.p1 = ::powf(L.beta1, static_cast<float>(t));
      L.p2 = ::powf(L.beta2, static_cast<float>(t));
      break;
    }
    case kUpdFtrl:  // FtrlParam
      L.lamda1 = GetF(p, "lamda1", 0.01f);
      L.beta = GetF(p, "beta", 1.0f);
      break;
  }
  L.w = w.data();
  L.g = g.data();
  L.out = out.data();
  for (int i = 2; i < spec->nin; ++i) L.s[i - 2] = static_cast<float*>(in[i].data());
  L.n = w.Size();
  L.out_is_w = out_is_w;

  LaneOp lop(dev);
  lop.Read(g);
  if (!out_is_w) lop.Read(w);
  lop.Write(out);
  for (int i = 2; i < spec->nin; ++i) lop.Write(in[i]);
  LaunchUpdateOp(L, lop.stream());
  Engine::Get()->CountLaunch(spec->launch_name, static_cast<uint64_t>(spec->bytes_per_elem) * L.n);
  lop.Issue();
  return true;
}

}  // namespace b200kv
