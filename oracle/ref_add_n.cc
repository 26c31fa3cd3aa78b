// TEST INFRASTRUCTURE ONLY -- never linked into or loaded by the product library.
//
// oracle/_ref/libmxref_add_n.so: the reference's own add_n arithmetic on the CPU, compiled where it
// lies (nothing is copied; oracle/add_n.mk):
//   ElementWiseSumCompute_          tensor/elemwise_sum.h:48-98 (all dense: 2-4 inputs right-nested,
//                                   else the left chain), for every MSHADOW_TYPE_SWITCH dtype
//   ElementwiseSumContainsDnsImpl   ndarray_function.cc:207-276 (> 4 inputs, some dense), cut out at
//                                   build time
//   CastStorageRspDnsImpl           cast_storage-inl.h:138-163 (the storage fallback's densify of a
//                                   row_sparse input, then ElementWiseSumCompute_), cut out at build time
// The two excerpts take mxnet::NDArray, which cannot exist without libmxnet (Storage / Engine): they
// compile unchanged against a stand-in `NDArray` offering exactly the accessors they use, backed by
// the reference's real TBlob / TShape / mshadow types, as oracle/ref_sparse.cc does for the
// row_sparse reduce. The all-row_sparse form is ElementwiseSumRsp, served by libmxref.so
// (mxref_rsp_reduce).
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
#include <dmlc/logging.h>
#include <mshadow/tensor.h>
#include <mxnet/base.h>
#include <mxnet/resource.h>
#include <mxnet/tensor_blob.h>
#include "operator/mxnet_op.h"
#include "operator/tensor/cast_storage-inl.h"
#include "operator/tensor/elemwise_binary_op-inl.h"
#include "operator/tensor/elemwise_sum.h"

namespace mxnet {
// the OMP thread-count policy consulted by Kernel<OP,cpu>::Launch (src/engine/openmp.cc): one thread
namespace engine {
OpenMP::OpenMP() : omp_num_threads_set_in_environment_(false) {}
OpenMP* OpenMP::Get() {
  static OpenMP inst;
  return &inst;
}
int OpenMP::GetRecommendedOMPThreadCount(bool) const { return 1; }
}  // namespace engine
// the tuning policy of Kernel<OP,cpu>::Launch for tuned functors (src/operator/operator_tune.cc,
// not linked here): no OpenMP, which does not change any element's result
namespace op {
namespace mxnet_op {
template <typename OP, typename DType>
bool tuned_op<OP, DType>::UseOMP(size_t, size_t) { return false; }
}  // namespace mxnet_op
}  // namespace op
}  // namespace mxnet

namespace mxref_sum {

using mshadow::cpu;
using mxnet::OpContext;
using mxnet::Resource;
using mxnet::TBlob;
using mxnet::kWriteTo;
using mxnet::op::CastStorageRspDnsKernel;
namespace mxnet_op = mxnet::op::mxnet_op;
enum { kDefaultStorage = 0, kRowSparseStorage = 1, kCSRStorage = 2 };
namespace rowsparse { enum { kIdx = 0 }; }
namespace csr { enum { kIndPtr = 0, kIdx = 1 }; }

// stand-in for mxnet::NDArray: a dense (rows x row_len) array, or a row_sparse one with nnr rows and
// int64 ids, of mshadow dtype flag `dtype`
struct NDArray {
  void* val = nullptr;
  int64_t* idx = nullptr;
  int stype = kDefaultStorage;
  int type = mshadow::kFloat32;
  int64_t rows = 0, row_len = 0, nnr = 0;
  int storage_type() const { return stype; }
  int dtype() const { return type; }
  bool storage_initialized() const { return stype == kDefaultStorage || nnr > 0; }
  mxnet::TShape shape() const { return mxnet::TShape(mshadow::Shape2(rows, row_len)); }
  TBlob data() const {
    const int64_t r = stype == kDefaultStorage ? rows : nnr;
    return TBlob(val, mxnet::TShape(mshadow::Shape2(r, row_len)), cpu::kDevMask, type);
  }
  int aux_type(int) const { return mshadow::kInt64; }
  mxnet::TShape aux_shape(int) const { return mxnet::TShape(mshadow::Shape1(nnr)); }
  TBlob aux_data(int) const {
    return TBlob(idx, mxnet::TShape(mshadow::Shape1(nnr)), cpu::kDevMask, mshadow::kInt64);
  }
};

// ---- the reference's two function templates, extracted at build time (see oracle/add_n.mk)
#include "_ref/excerpt_cast_rsp_dns.inc"
#include "_ref/excerpt_sum_contains_dns.inc"

}  // namespace mxref_sum

extern "C" {

// One add_n call as ElementWiseSumComputeExCPU and the storage fallback dispatch it
// (elemwise_sum.cc:101-125), on operands of `rows` x `row_len` elements of mshadow dtype flag
// `dtype`: stypes[i] 0 is dense (vals[i] holds every element), 1 row_sparse (nnr[i] rows of vals[i]
// with ascending int64 ids[i]). The out is dense. At least one input must be dense: all row_sparse
// inputs are ElementwiseSumRsp (libmxref.so). Returns 0, or -1 with the error text in `err`.
int mxref_add_n(int n, const int* stypes, void* const* vals, int64_t* const* ids, const int64_t* nnr, int dtype,
                int64_t rows, int64_t row_len, void* out, char* err, int errlen) {
  try {
    using namespace mxref_sum;
    CHECK_GE(n, 1);
    std::vector<NDArray> nds(n);
    bool any_dense = false;
    for (int i = 0; i < n; ++i) {
      nds[i].val = vals[i];
      nds[i].idx = ids[i];
      nds[i].stype = stypes[i];
      nds[i].type = dtype;
      nds[i].rows = rows;
      nds[i].row_len = row_len;
      nds[i].nnr = stypes[i] == kRowSparseStorage ? nnr[i] : rows;
      any_dense = any_dense || stypes[i] == kDefaultStorage;
    }
    CHECK(any_dense) << "all-row_sparse inputs: use mxref_rsp_reduce";
    NDArray o;
    o.val = out;
    o.type = dtype;
    o.rows = rows;
    o.row_len = row_len;
    OpContext ctx;
    ctx.is_train = false;
    ctx.need_grad = false;
    ctx.run_ctx.stream = nullptr;
    if (n > 4 && any_dense) {
      ElementwiseSumContainsDnsImpl(nullptr, Resource(), nds, &o);
      return 0;
    }
    // dense inputs as they are, row_sparse ones densified by the fallback's cast
    const size_t bytes = static_cast<size_t>(rows * row_len) * mshadow::mshadow_sizeof(dtype);
    std::vector<std::vector<char>> tmp;
    std::vector<TBlob> in;
    for (int i = 0; i < n; ++i) {
      if (stypes[i] == kDefaultStorage) {
        in.push_back(nds[i].data());
        continue;
      }
      tmp.emplace_back(bytes);
      TBlob d(static_cast<void*>(tmp.back().data()), nds[i].shape(), cpu::kDevMask, dtype);
      CastStorageRspDnsImpl<cpu>(ctx, nds[i], &d);
      in.push_back(d);
    }
    std::vector<TBlob> outs{o.data()};
    std::vector<mxnet::OpReqType> req(1, mxnet::kWriteTo);
    nnvm::NodeAttrs attrs;
    MSHADOW_TYPE_SWITCH(dtype, DType, {
      mxnet::op::ElementWiseSumCompute_<cpu, DType>(attrs, ctx, in, req, outs);
    });
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
