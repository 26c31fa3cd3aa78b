// TEST INFRASTRUCTURE ONLY -- never linked into or loaded by the product library.
//
// oracle/_ref/libmxref_sparse_update.so: the reference's own parameter parsers and row_sparse CPU
// kernels of ftrl_update and _sparse_adagrad_update, compiled from src/operator/optimizer_op-inl.h
// where it lies (nothing is copied):
//   ParamParser<FtrlParam>, Kernel<FtrlDnsRspDnsKernel<kWriteInplace>, cpu>::Launch   (:2186-2219)
//   ParamParser<AdagradParam>, Kernel<AdagradDnsRspDnsKernel<cpu>, cpu>::Launch        (:2507-2531)
// The NDArray-level dispatch around those kernels needs the reference's NDArray (libmxnet), which
// does not build here; it is restated below on flat buffers, each step citing the code it follows.
// A library of its own (built by oracle/sparse_update_ops.mk), so the other oracle libraries stay
// as they are.
#include <cstdint>
#include <cstring>
#include <sstream>
#include <string>
#include <vector>
#include <dmlc/logging.h>
#include <mshadow/tensor.h>
#include <nnvm/op.h>
#include "operator/optimizer_op-inl.h"

using namespace mxnet;

namespace mxnet {
namespace op {
// the parameter managers optimizer_op.cc:36-44 registers
DMLC_REGISTER_PARAMETER(FtrlParam);
DMLC_REGISTER_PARAMETER(AdagradParam);
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

// CheckAllRowsPresent (operator_common.h:500-511) on (stype, storage rows, rows)
void CheckAllRowsPresent(int stype, int64_t nnr, int64_t rows, const std::string& func) {
  if (stype == kRowSparseStorage) {
    CHECK(nnr == rows) << func << " for RowSparse weights is only implemented for RowSparse weights "
                       << "with all rows containing non-zeros. Expects weights.data.shape[0] (" << nnr
                       << ") == weights.shape[0] (" << rows << ").";
  } else {
    CHECK(stype == kDefaultStorage);
  }
}

// FillDnsZerosRspImpl (tensor/init_op.h:474-487) of a state with no stored rows: every row, zeros.
// The ids 0..rows-1 (PopulateFullIdxRspKernel) are implied by nnr == rows.
void FillDnsZerosRsp(float* data, int64_t* nnr, int64_t rows, int64_t row_len) {
  std::memset(data, 0, static_cast<size_t>(rows * row_len) * sizeof(float));
  *nnr = rows;
}

bool AllRsp(int nin, const int* stype) {  // common::ContainsOnlyStorage(inputs, kRowSparseStorage)
  for (int i = 0; i < nin; ++i) {
    if (stype[i] != kRowSparseStorage) return false;
  }
  return true;
}

void Ftrl(const nnvm::NodeAttrs& attrs, const int* stype, int64_t* nnr, float** data,
          const int64_t* gidx, int64_t rows, int64_t row_len, bool inplace) {
  using mxnet::op::FtrlParam;
  const FtrlParam& param = nnvm::get<FtrlParam>(attrs.parsed);
  // FtrlUpdateEx (optimizer_op-inl.h:2297-2313); out is the weight, so out_stype == weight_stype
  CHECK_EQ(stype[2], stype[0]) << "Inconsistent storage type detected between "
                               << " z.stype = " << stype[2] << " and weight.stype = " << stype[0];
  CHECK_EQ(stype[3], stype[0]) << "Inconsistent storage type detected between "
                               << " n.stype = " << stype[3] << " and weight.stype = " << stype[0];
  CHECK(AllRsp(4, stype)) << "ftrl_update: this oracle serves the all-row_sparse form only";
  // FtrlUpdateRspRspRspImpl (2261-2289)
  CheckAllRowsPresent(stype[0], nnr[0], rows, "FtrlUpdate");
  for (int i : {2, 3}) {
    if (nnr[i] == 0) FillDnsZerosRsp(data[i], &nnr[i], rows, row_len);
  }
  // FtrlUpdateDnsRspDnsImpl (2222-2259)
  if (nnr[1] == 0) return;
  CHECK(inplace) << "kWriteInplace is expected for sparse ftrl_update";
  Kernel<mxnet::op::FtrlDnsRspDnsKernel<kWriteInplace>, cpu>::Launch(
      nullptr, static_cast<size_t>(nnr[1]), static_cast<nnvm::dim_t>(row_len), data[0], data[2],
      data[3], static_cast<const float*>(data[0]), gidx, static_cast<const float*>(data[1]),
      static_cast<float>(param.clip_gradient), static_cast<float>(param.lamda1),
      static_cast<float>(param.beta), static_cast<float>(param.lr), static_cast<float>(param.wd),
      static_cast<float>(param.rescale_grad));
}

void Adagrad(const nnvm::NodeAttrs& attrs, const int* stype, int64_t* nnr, float** data,
             const int64_t* gidx, int64_t rows, int64_t row_len, bool inplace) {
  using mxnet::op::AdagradParam;
  const AdagradParam& param = nnvm::get<AdagradParam>(attrs.parsed);
  // AdagradStorageType (2480-2501) dispatches only with wd == 0; AdagradUpdateDnsRspDnsImpl
  // (2569-2570) states the reason
  CHECK_EQ(param.wd, 0.0f) << "sparse adagrad_update does not support wd.";
  CHECK(stype[1] == kRowSparseStorage &&
        (stype[0] == kRowSparseStorage || stype[0] == kDefaultStorage) && stype[2] == stype[0])
      << "_sparse_adagrad_update: unsupported storage types (" << stype[0] << ", " << stype[1] << ", "
      << stype[2] << ")";
  // AdagradUpdateEx (2620-2649) -> AdagradUpdateRspRspRspImpl (2596-2618)
  if (AllRsp(3, stype)) {
    CheckAllRowsPresent(stype[0], nnr[0], rows, "AdagradUpdate");
    if (nnr[2] == 0) FillDnsZerosRsp(data[2], &nnr[2], rows, row_len);
  }
  // AdagradUpdateDnsRspDnsImpl (2557-2594), CPU: one kernel index per gradient row
  if (nnr[1] == 0) return;
  CHECK(inplace) << "kWriteInplace is expected for sparse adagrad_update";
  Kernel<mxnet::op::AdagradDnsRspDnsKernel<cpu>, cpu>::Launch(
      nullptr, static_cast<size_t>(nnr[1]), static_cast<index_t>(row_len), data[0], data[2],
      static_cast<const float*>(data[0]), gidx, static_cast<const float*>(data[1]),
      static_cast<float>(param.clip_gradient), static_cast<float>(param.epsilon),
      static_cast<float>(param.lr), static_cast<float>(param.rescale_grad));
}

}  // namespace

extern "C" {

// One call of ftrl_update (nin 4: weight, grad, z, n) or _sparse_adagrad_update (nin 3: weight,
// grad, history) on float32 operands. stype[i]: 0 default, 1 row_sparse. nnr[i]: stored rows of a
// row_sparse operand (in / out: a filled state comes back with nnr == rows). data[1] holds nnr[1]
// gradient rows with ids gidx; every other data[i] is a rows x row_len buffer (a row_sparse
// weight or state holds its rows in id order 0..rows-1). inplace: out is the weight.
// Returns 0, or -1 with the dmlc::Error text in `err`.
int mxref_sparse_update(const char* op, int nin, const int* stype, int64_t* nnr, float** data,
                        const int64_t* gidx, int64_t rows, int64_t row_len, int inplace, int nparam,
                        const char** keys, const char** vals, char* err, int errlen) {
  try {
    nnvm::NodeAttrs attrs;
    attrs.name = op;
    for (int i = 0; i < nparam; ++i) attrs.dict[keys[i]] = vals[i];
    const std::string name(op);
    if (name == "ftrl_update" || name == "_sparse_ftrl_update") {
      CHECK_EQ(nin, 4);
      mxnet::op::ParamParser<mxnet::op::FtrlParam>(&attrs);
      Ftrl(attrs, stype, nnr, data, gidx, rows, row_len, inplace != 0);
    } else if (name == "_sparse_adagrad_update") {
      CHECK_EQ(nin, 3);
      mxnet::op::ParamParser<mxnet::op::AdagradParam>(&attrs);
      Adagrad(attrs, stype, nnr, data, gidx, rows, row_len, inplace != 0);
    } else {
      throw dmlc::Error(std::string("unknown operator ") + op);
    }
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
