// TEST INFRASTRUCTURE ONLY -- never linked into or loaded by the product library.
//
// oracle/_ref/libmxref_group_adagrad.so: the reference's own parameter parser and CPU kernel of
// _contrib_group_adagrad_update, compiled from src/operator/contrib/optimizer_op-inl.h where it
// lies (nothing is copied):
//   GroupAdagradParam::Init, Kernel<GroupAdagradDnsRspKernel<cpu>, cpu>::Launch   (:46-65, :96-139)
// The NDArray-level dispatch around the kernel needs the reference's NDArray (libmxnet), which does
// not build here; it is restated below on flat buffers, each step citing the code it follows.
// The entry point has the calling convention of oracle/ref_sparse_update_ops.cc, so the same
// Python front-end (golden_sparse_update_ops.RefSparseUpdate) drives both libraries.
#include <cstdint>
#include <cstring>
#include <sstream>
#include <string>
#include <vector>
#include <dmlc/logging.h>
#include <mshadow/tensor.h>
#include <nnvm/op.h>
#include "operator/contrib/optimizer_op-inl.h"

using namespace mxnet;

namespace mxnet {
namespace op {
// the parameter manager contrib/optimizer_op.cc:32 registers
DMLC_REGISTER_PARAMETER(GroupAdagradParam);
}  // namespace op
// the OMP thread-count policy consulted by Kernel<OP,cpu>::Launch (src/engine/openmp.cc): one thread
namespace engine {
OpenMP::OpenMP() : omp_num_threads_set_in_environment_(false) {}
OpenMP* OpenMP::Get() {
  static OpenMP inst;
  return &inst;
}
int OpenMP::GetRecommendedOMPThreadCount(bool) const { return 1; }
}  // namespace engine
}  // namespace mxnet

namespace {

using mxnet::op::mxnet_op::Kernel;
using mshadow::cpu;

const char* StypeString(int stype) { return stype == kRowSparseStorage ? "row_sparse" : "default"; }

// CheckAllRowsPresent (operator_common.h:500-511) on (stype, storage rows, rows)
void CheckAllRowsPresent(int stype, int64_t nnr, int64_t rows, const std::string& param) {
  if (stype == kRowSparseStorage) {
    CHECK(nnr == rows) << "GroupAdagradUpdate for RowSparse " << param << " is only implemented for "
                       << "RowSparse " << param << " with all rows containing non-zeros. Expects "
                       << param << ".data.shape[0] (" << nnr << ") == " << param << ".shape[0] ("
                       << rows << ").";
  } else {
    CHECK(stype == kDefaultStorage);
  }
}

void GroupAdagrad(const nnvm::NodeAttrs& attrs, const int* stype, int64_t* nnr, float** data,
                  const int64_t* gidx, int64_t rows, int64_t row_len, bool inplace) {
  using mxnet::op::GroupAdagradParam;
  const GroupAdagradParam& param = nnvm::get<GroupAdagradParam>(attrs.parsed);
  // GroupAdagradStorageType (:67-93): all-default dispatches to FCompute, which is not registered
  // (Imperative::Invoke, imperative.cc:82-85); other forms than the two below do not dispatch
  // (SetShapeType, imperative_utils.h:194-195)
  const bool all_dns = stype[0] == kDefaultStorage && stype[1] == kDefaultStorage &&
                       stype[2] == kDefaultStorage;
  CHECK(!all_dns) << "Operator _contrib_group_adagrad_update is not implemented for CPU.";
  CHECK(stype[1] == kRowSparseStorage &&
        (stype[0] == kRowSparseStorage || stype[0] == kDefaultStorage) && stype[2] == stype[0])
      << "Operator not implemented: operator = _contrib_group_adagrad_update\ninput storage types = ["
      << StypeString(stype[0]) << ", " << StypeString(stype[1]) << ", " << StypeString(stype[2]) << ", ]";
  // GroupAdagradUpdateEx (:216-242) -> GroupAdagradUpdateRspRspRspImpl (:191-213)
  if (stype[0] == kRowSparseStorage) {
    CheckAllRowsPresent(stype[0], nnr[0], rows, "weights");
    if (nnr[2] == 0) {  // FillDnsZerosRspImpl (tensor/init_op.h:474-487): every row, zeros
      std::memset(data[2], 0, static_cast<size_t>(rows) * sizeof(float));
      nnr[2] = rows;
    } else {
      CheckAllRowsPresent(stype[2], nnr[2], rows, "states");
    }
  }
  // GroupAdagradUpdateDnsRspDnsImpl (:144-185)
  CHECK(inplace) << "kWriteInplace is expected for sparse group_adagrad_update";
  if (nnr[1] == 0) return;  // !grad.storage_initialized()
  Kernel<mxnet::op::GroupAdagradDnsRspKernel<cpu>, cpu>::Launch(
      nullptr, static_cast<size_t>(nnr[1]), static_cast<index_t>(row_len), data[0], data[2],
      data[0], gidx, static_cast<const float*>(data[1]), static_cast<float>(param.clip_gradient),
      static_cast<float>(param.rescale_grad), static_cast<float>(param.lr),
      static_cast<float>(param.epsilon));
}

}  // namespace

extern "C" {

// One call of _contrib_group_adagrad_update (nin 3: weight, grad, history) on float32 operands.
// stype[i]: 0 default, 1 row_sparse. nnr[i]: stored rows of a row_sparse operand (in / out: a
// filled history comes back with nnr == rows). data[1] holds nnr[1] gradient rows of row_len with
// ids gidx; data[0] is a rows x row_len buffer, data[2] a rows x 1 buffer (a row_sparse weight or
// history holds its rows in id order 0..rows-1). inplace: out is the weight.
// Returns 0, or -1 with the dmlc::Error text in `err`.
int mxref_sparse_update(const char* op, int nin, const int* stype, int64_t* nnr, float** data,
                        const int64_t* gidx, int64_t rows, int64_t row_len, int inplace, int nparam,
                        const char** keys, const char** vals, char* err, int errlen) {
  try {
    nnvm::NodeAttrs attrs;
    attrs.name = op;
    for (int i = 0; i < nparam; ++i) attrs.dict[keys[i]] = vals[i];
    if (std::string(op) != "_contrib_group_adagrad_update") {
      throw dmlc::Error(std::string("unknown operator ") + op);
    }
    CHECK_EQ(nin, 3);
    // ParamParser<GroupAdagradParam> (operator_common.h:480-498) restated around the reference's own
    // GroupAdagradParam::Init: its error path reads attrs->op->name, and this library has no
    // nnvm::Op registry to point attrs.op at
    mxnet::op::GroupAdagradParam param;
    try {
      param.Init(attrs.dict);
    } catch (const dmlc::ParamError& e) {
      std::ostringstream os;
      os << e.what() << ", in operator " << op << "(name=\"" << attrs.name << "\"";
      for (const auto& k : attrs.dict) os << ", " << k.first << "=\"" << k.second << "\"";
      os << ")";
      throw dmlc::ParamError(os.str());
    }
    attrs.parsed = std::move(param);
    GroupAdagrad(attrs, stype, nnr, data, gidx, rows, row_len, inplace != 0);
    return 0;
  } catch (const std::exception& e) {
    if (err && errlen > 0) {
      std::strncpy(err, e.what(), errlen - 1);
      err[errlen - 1] = '\0';
    }
    return -1;
  }
}

}  // extern "C"
