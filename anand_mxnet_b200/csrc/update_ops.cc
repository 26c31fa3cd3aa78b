// update_ops.cc -- host side of the single-tensor optimizer operators that the reference's NAG,
// Signum, RMSProp, FTML and Ftrl optimizers call from their `update` (the per-key updater callback
// of the store, and the local updaters of update_on_kvstore=False), plus the row_sparse forms of
// ftrl_update, AdaGrad's _sparse_adagrad_update and GroupAdaGrad's _contrib_group_adagrad_update.
// Kernels: update_kernels.cu and update_rsp_grad_kernels.cu (dense weights, with a dense or a
// row_sparse gradient), rowsparse_kernels.cu (row_sparse weights, and the lazy dense-weight forms of
// AdaGrad / GroupAdaGrad).
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
// Storage forms (UpdateOp), all float32 but mp_nag_mom_update's 16-bit weight and gradient:
//   all dense                          every operator (mp_nag_mom_update: float16 / bfloat16 weight
//                                      and gradient with float32 mom and weight32)
//   dense weight and states, a row_sparse gradient
//                                      every operator but mp_nag_mom_update. The reference has no
//                                      FComputeEx for this pair and falls back to the dense
//                                      FCompute on the densified gradient (imperative_utils.h:
//                                      185-198, CastStorageRspDnsImpl): every row moves, absent rows
//                                      with g = +0.0f. Here the kernel reads the stored rows through
//                                      a row map instead of a dense copy (BuildRowMap).
//   row_sparse weight, grad and states ftrl_update (RspUpdateOp): only the gradient's rows move
//   AdaGrad / GroupAdaGrad             their own row_sparse forms (RspUpdateOp)
// Everything else is refused before anything is enqueued: a row_sparse weight or state with the
// other operators (the reference would densify the weight, update it and cast it back), and 16-bit
// weights without a master copy (the reference would update them in half precision).
#include <cctype>
#include <cerrno>
#include <cmath>
#include <limits>

#include "kernels.h"
#include "op_params.h"
#include "ops.h"
#include "rowsparse.h"

namespace b200kv {
namespace {

struct Spec {
  const char* name;
  int op;
  int nin;                 // weight, grad, states...
  const char* launch_name; // CountLaunch keeps the pointer
  int bytes_per_elem;      // algorithmic traffic of one element (float32 / mp float16)
  const char* rsp_grad_launch_name;  // the dense-weight pass over a row_sparse gradient
};

const Spec kSpecs[] = {
    {"nag_mom_update", kUpdNAG, 3, "update_op(nag_mom_update)", 20, "update_op(nag_mom_update, row_sparse grad)"},
    {"mp_nag_mom_update", kUpdMPNAG, 4, "update_op(mp_nag_mom_update)", 20, nullptr},
    {"signsgd_update", kUpdSignSGD, 2, "update_op(signsgd_update)", 12, "update_op(signsgd_update, row_sparse grad)"},
    {"signum_update", kUpdSignum, 3, "update_op(signum_update)", 20, "update_op(signum_update, row_sparse grad)"},
    {"rmsprop_update", kUpdRMSProp, 3, "update_op(rmsprop_update)", 20, "update_op(rmsprop_update, row_sparse grad)"},
    {"rmspropalex_update", kUpdRMSPropAlex, 5, "update_op(rmspropalex_update)", 36,
     "update_op(rmspropalex_update, row_sparse grad)"},
    {"ftml_update", kUpdFTML, 5, "update_op(ftml_update)", 36, "update_op(ftml_update, row_sparse grad)"},
    {"ftrl_update", kUpdFtrl, 4, "update_op(ftrl_update)", 28, "update_op(ftrl_update, row_sparse grad)"},
    // the alias of ftrl_update (MXNET_ADD_SPARSE_OP_ALIAS, optimizer_op.cc:855) and AdaGrad's
    // operator (optimizer_op.cc:895-924, optimizer_op-inl.h:2454-2649)
    {"_sparse_ftrl_update", kUpdFtrl, 4, "update_op(ftrl_update)", 28, "update_op(ftrl_update, row_sparse grad)"},
    {"_sparse_adagrad_update", kUpdAdaGrad, 3, "update_op(_sparse_adagrad_update)", 20, nullptr},
    // GroupAdaGrad's operator: g 4 + w 4+4 per element; the history is one float per row
    {"_contrib_group_adagrad_update", kUpdGroupAdaGrad, 3, "update_op(_contrib_group_adagrad_update)", 12, nullptr},
};

// dmlc::Parameter set_range(lo, hi) (parameter.h:752-762)
float InRange(float v, const char* key, float lo, float hi) {
  KV_CHECK(!(v < lo || v > hi)) << "value " << v << " for Parameter " << key << " exceed bound [" << lo
                                << ',' << hi << ']';
  return v;
}

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
  const char* n = spec.name;
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
        << n << ": the row_sparse form needs row_sparse weight, grad, z and n";
  } else if (op == kUpdGroupAdaGrad) {  // GroupAdagradParam (contrib/optimizer_op-inl.h:46-65)
    RejectUnknownKeys(p, {"lr", "rescale_grad", "clip_gradient", "epsilon"});  // wd among the unknown
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
  // the states' rows are addressed by the table row id, like the weight's: a row_sparse state holds
  // every row, or none yet (then it is zero-filled first, FillDnsZerosRspImpl); kWriteInplace is
  // expected (optimizer_op-inl.h:2235, 2572)
  const char* func = op == kUpdFtrl ? "FtrlUpdate" : op == kUpdAdaGrad ? "AdagradUpdate" : "GroupAdagradUpdate";
  CheckRspTable(n, func, in, *outputs);

  // a state with no rows is zero-filled even when the gradient is empty
  const std::vector<NDArray> states(in.begin() + 2, in.end());
  ZeroFillEmptyRspStates(states, rows, spec.launch_name);
  RunRspRowUpdate(L, w, g, states, spec.launch_name, spec.bytes_per_elem);
}

std::string Stypes(const std::vector<NDArray>& in) {
  std::string t;
  for (const NDArray& a : in) t += std::string(t.empty() ? "" : ", ") + StypeName(a.stype());
  return t;
}

// every operator of kSpecs (variant: its index there): the row_sparse-weight forms and AdaGrad /
// GroupAdaGrad in RspUpdateOp, dense weights and states here, with a dense or a row_sparse gradient
void UpdateOp(const OpInfo& info, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
              const Params& p) {
  const Spec& spec = kSpecs[info.variant];
  const char* n = spec.name;
  const int op = spec.op;
  KV_CHECK_EQ(static_cast<int>(in.size()), spec.nin) << n << " expects " << spec.nin << " inputs";
  const NDArray& w = in[0];
  const NDArray& g = in[1];
  if (op == kUpdFtrl) {  // FtrlUpdateEx (optimizer_op-inl.h:2303-2306)
    for (int i : {2, 3}) {
      KV_CHECK(in[i].stype() == w.stype())
          << "Inconsistent storage type detected between  " << (i == 2 ? "z" : "n") << ".stype = "
          << in[i].stype() << " and weight.stype = " << w.stype();
    }
  }
  if (op == kUpdAdaGrad || op == kUpdGroupAdaGrad || (op == kUpdFtrl && w.stype() == kRowSparseStorage)) {
    RspUpdateOp(spec, in, outputs, p);
    return;
  }
  bool dense_tables = w.stype() == kDefaultStorage;
  for (int i = 2; i < spec.nin; ++i) dense_tables = dense_tables && in[i].stype() == kDefaultStorage;
  const bool rsp_grad = g.stype() == kRowSparseStorage;
  KV_CHECK(dense_tables && (rsp_grad || g.stype() == kDefaultStorage))
      << "Operator " << n << " is not implemented for storage types (" << Stypes(in) << "): it takes a "
      << "dense weight and dense states with a dense or row_sparse gradient"
      << (op == kUpdFtrl ? ", or row_sparse weight, grad, z and n" : "");
  KV_CHECK(!rsp_grad || op != kUpdMPNAG)
      << n << ": a row_sparse gradient is not supported (16-bit weights would need 16-bit row_sparse "
      << "values; use nag_mom_update on float32 weights)";
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
  if (rsp_grad) {
    // ElemwiseShape: every operand has the weight's shape, not only its size
    KV_CHECK_EQ(g.dtype(), kFloat32) << n << ": row_sparse gradients are float32, got " << DTypeName(g.dtype());
    KV_CHECK(!w.shape().empty()) << n << ": the weight needs at least one dimension";
    KV_CHECK(g.shape() == w.shape()) << n << ": weight / grad shape mismatch";
  }
  KV_CHECK_EQ(g.dtype(), dtype) << n << ": weight / grad dtype mismatch";
  KV_CHECK_EQ(g.Size(), w.Size()) << n << ": weight / grad shape mismatch";
  for (int i = 2; i < spec.nin; ++i) {
    KV_CHECK_EQ(in[i].dtype(), kFloat32) << n << ": optimizer states must be float32";
    KV_CHECK_EQ(in[i].Size(), w.Size()) << n << ": state shape mismatch";
    KV_CHECK(!rsp_grad || in[i].shape() == w.shape()) << n << ": state shape mismatch";
  }
  NDArray out = OutOr(outputs, 0, w.shape(), w.ctx(), dtype);
  KV_CHECK(out.on_gpu() && out.dev() == dev) << n << ": out must be on the weight's GPU";
  KV_CHECK(out.stype() == kDefaultStorage) << n << ": out must be a dense array";
  KV_CHECK_EQ(out.dtype(), dtype) << n << ": out dtype mismatch";
  KV_CHECK_EQ(out.Size(), w.Size()) << n << ": out shape mismatch";
  KV_CHECK(!rsp_grad || out.shape() == w.shape()) << n << ": out shape mismatch";
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
      const int t = Required<int>(p, "t", n);
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
  if (rsp_grad) {
    RunRspGradUpdate(L, w, g, std::vector<NDArray>(in.begin() + 2, in.end()), out, spec.rsp_grad_launch_name,
                     spec.bytes_per_elem);
    return;
  }
  L.w = w.data();
  L.g = g.data();
  L.out = out.data();
  for (int i = 2; i < spec.nin; ++i) L.s[i - 2] = static_cast<float*>(in[i].data());
  L.n = w.Size();
  L.out_is_w = out_is_w;

  LaneOp lop(dev);
  lop.Read(g);
  if (!out_is_w) lop.Read(w);
  lop.Write(out);
  for (int i = 2; i < spec.nin; ++i) lop.Write(in[i]);
  LaunchUpdateOp(L, lop.stream());
  Engine::Get()->CountLaunch(spec.launch_name, static_cast<uint64_t>(spec.bytes_per_elem) * L.n);
  lop.Issue();
}

}  // namespace

const std::vector<OpInfo> kUpdateOps = [] {
  std::vector<OpInfo> rows;
  for (const Spec& s : kSpecs) rows.push_back({s.name, UpdateOp, static_cast<int>(&s - kSpecs)});
  return rows;
}();

}  // namespace b200kv
