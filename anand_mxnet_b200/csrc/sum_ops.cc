// sum_ops.cc -- add_n and its aliases ElementWiseSum, _sparse_add_n, _sparse_ElementWiseSum
// (tensor/elemwise_sum.cc:101-164): the sum of num_args arrays of one shape and dtype on one GPU.
//
// Storage dispatch (ElemwiseStorageAttr<false, true, false>, elemwise_op_common.h:51-93, then
// ElementWiseSumComputeExCPU and ElementwiseSum<cpu>, ndarray_function.cc:178-300):
//   all dense                    dense       ElementWiseSumCompute_: 2-4 inputs a0 + (a1 + (a2 + a3)),
//                                            else out = a0, out = out + a_i (LaunchAddN, one launch
//                                            per 200 inputs)
//   all row_sparse               row_sparse  ElementwiseSumRsp: the union of ids, each row +0 plus
//                                            the inputs that hold it, in order (SumRowSparse)
//   > 4 inputs, some dense       dense       ElementwiseSumContainsDnsImpl: out = a0 (+0 when a0 is
//                                            row_sparse), then each dense input adds every element
//                                            and each row_sparse input its stored rows only
//   any other mix                dense       storage fallback: row_sparse inputs densified (absent
//                                            rows +0), then the all-dense rule
// The row_sparse inputs of the two mixed forms are densified into temporaries: zeros then their rows
// (LaunchRspScatterRows). In the > 4 form absent rows are -0.0 instead, the identity of IEEE +, so
// that they leave out exactly as it was, a -0.0 included. Row_sparse inputs are float32.
//
// Every check runs before anything is enqueued. out may be input 0 itself (FInplaceOption {0, 0});
// an out that overlaps any other input is refused, since the left chain would read an input it has
// already overwritten.
#include <cstring>

#include "kernels.h"
#include "op_params.h"
#include "ops.h"
#include "rowsparse.h"

namespace b200kv {
namespace {

bool AddNDTypeOk(int t) {  // MSHADOW_TYPE_SWITCH's dtypes, and bfloat16
  return t == kFloat16 || t == kBfloat16 || t == kFloat32 || t == kFloat64 || t == kUint8 ||
         t == kInt8 || t == kInt32 || t == kInt64;
}

// the bytes of a dense array overlap those of b (both non-empty)
bool Overlaps(const NDArray& a, const NDArray& b) {
  if (a.Size() == 0 || b.Size() == 0) return false;
  const char* a0 = static_cast<const char*>(a.data());
  const char* b0 = static_cast<const char*>(b.data());
  return a0 < b0 + b.ByteSize() && b0 < a0 + a.ByteSize();
}

void AddN(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
          const Params& p) {
  const char* n = op.name;
  RejectUnknownKeys(p, {"num_args"});  // ElementWiseSumParam
  const int num = Required<int>(p, "num_args", n);
  KV_CHECK(num >= 1) << n << ": num_args must be at least 1, got " << num;
  KV_CHECK_EQ(static_cast<int>(in.size()), num) << n << ": expected num_args inputs";
  const NDArray& a0 = in[0];
  KV_CHECK(a0.on_gpu()) << n << " runs on GPU arrays only (no CPU fallback)";
  const int dev = a0.dev();
  const int dtype = a0.dtype();
  KV_CHECK(AddNDTypeOk(dtype)) << n << ": float16, bfloat16, float32, float64, uint8, int8, int32 and "
                               << "int64 arrays only; got " << DTypeName(dtype);
  bool any_dense = false, any_rsp = false;
  for (size_t i = 0; i < in.size(); ++i) {
    const NDArray& a = in[i];
    KV_CHECK(a.on_gpu() && a.dev() == dev) << "all operands must be on the same GPU (no CPU fallback)";
    KV_CHECK(a.stype() == kDefaultStorage || a.stype() == kRowSparseStorage)
        << n << " takes dense and row_sparse arrays only; input " << i << " is neither";
    KV_CHECK(a.shape() == a0.shape()) << n << ": input " << i << " shape differs from input 0";
    KV_CHECK_EQ(a.dtype(), dtype) << n << ": input " << i << " dtype differs from input 0";
    any_dense = any_dense || a.stype() == kDefaultStorage;
    any_rsp = any_rsp || a.stype() == kRowSparseStorage;
  }
  KV_CHECK(!any_rsp || dtype == kFloat32) << n << ": row_sparse inputs are float32; got " << DTypeName(dtype);
  KV_CHECK(!any_rsp || !a0.shape().empty()) << n << ": row_sparse inputs need at least one dimension";
  const int out_stype = any_dense ? kDefaultStorage : kRowSparseStorage;
  if (!outputs->empty()) {
    const NDArray& o = (*outputs)[0];
    KV_CHECK(o.on_gpu() && o.dev() == dev) << "all operands must be on the same GPU (no CPU fallback)";
    KV_CHECK(o.stype() == out_stype) << n << ": out must be " << StypeName(out_stype) << " for these inputs";
    KV_CHECK(o.shape() == a0.shape()) << n << ": out has the wrong shape";
    KV_CHECK_EQ(o.dtype(), dtype) << n << ": out dtype differs from the inputs'";
    for (size_t i = 0; i < in.size(); ++i) {
      const NDArray& a = in[i];
      const bool shares = out_stype == kRowSparseStorage
                              ? a.SameStorage(o)
                              : a.stype() == kDefaultStorage && Overlaps(a, o);
      const bool is_in0 = i == 0 && a.SameStorage(o) && (out_stype == kRowSparseStorage ||
                                                         (a.data() == o.data() && a.Size() == o.Size()));
      KV_CHECK(!shares || is_in0) << n << ": out overlaps input " << i << "; only input 0 itself may be out";
    }
  }
  if (out_stype == kRowSparseStorage) {
    if (outputs->empty()) outputs->push_back(NDArray::RowSparse(a0.shape(), a0.ctx(), dtype));
    SumRowSparse(in, (*outputs)[0]);
    return;
  }
  NDArray o = OutOr(outputs, 0, a0.shape(), a0.ctx(), dtype);
  const uint64_t size = o.Size();
  Engine* eng = Engine::Get();
  // ElementwiseSumContainsDnsImpl (> 4 inputs, some dense) or the fallback's densified inputs: the
  // temporaries start as -0.0 (an ew_kernel fill) or +0.0 (ZerosOn), then take the stored rows
  const bool contains_dns = in.size() > 4 && any_rsp;
  std::vector<NDArray> dense_tmp(in.size());
  for (size_t i = 0; i < in.size(); ++i) {
    if (in[i].stype() == kDefaultStorage) continue;
    if (contains_dns) {
      dense_tmp[i] = NDArray(a0.shape(), a0.ctx(), kFloat32);
      if (size > 0) Elementwise(kEwFill, NDArray(), nullptr, -0.0, dense_tmp[i]);
    } else {
      dense_tmp[i] = ZerosOn(a0.shape(), dev, kFloat32);
    }
  }
  LaneOp lop(dev);
  for (const NDArray& a : in) lop.Read(a);
  for (const NDArray& t : dense_tmp) lop.Write(t);
  lop.Write(o);
  std::vector<const void*> ptrs;
  for (size_t i = 0; i < in.size(); ++i) {
    const NDArray& a = in[i];
    if (a.stype() == kRowSparseStorage && size > 0 && a.storage_initialized()) {
      LaunchRspScatterRows(a.row_ids(), static_cast<const float*>(a.data()), a.nnr(),
                           static_cast<int64_t>(a.RowLength()), static_cast<float*>(dense_tmp[i].data()),
                           lop.stream());
      eng->CountLaunch("add_n(densify rows)", static_cast<uint64_t>(a.nnr()) * (a.RowLength() * 8 + 8));
    }
    const NDArray& src = a.stype() == kDefaultStorage ? a : dense_tmp[i];
    ptrs.push_back(size > 0 ? src.data() : nullptr);
  }
  const bool zero_first = contains_dns && a0.stype() == kRowSparseStorage;
  const int launches = LaunchAddN(dtype, ptrs.data(), static_cast<int>(ptrs.size()), zero_first, o.data(),
                                  size, lop.stream());
  for (int i = 0; i < launches; ++i) eng->CountLaunch("add_n", 0);
  lop.Issue();
}

}  // namespace

const std::vector<OpInfo> kSumOps = {
    {"add_n", AddN, 0},
    {"ElementWiseSum", AddN, 0},
    {"_sparse_add_n", AddN, 0},
    {"_sparse_ElementWiseSum", AddN, 0},
};

}  // namespace b200kv
