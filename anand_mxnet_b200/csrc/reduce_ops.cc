// reduce_ops.cc -- the two operators the dense-gradient branches of the reference's AdaGrad and
// GroupAdaGrad call beyond the arithmetic of arith_ops.cc (python/mxnet/optimizer/optimizer.py:
// 1682-1688, contrib.py:94-100): `square(grad)` and `mean(x, axis=1, keepdims=True)`.
//
// Reference operator definitions:
//   square   tensor/elemwise_unary_op_basic.cc; mshadow_op.h:536, math_functions-inl.h:139-147
//   mean     tensor/broadcast_reduce_sum_value.cc:82-85 (ReduceAxesParam, broadcast_reduce_op.h;
//            ReduceAxesCompute<cpu, red::sum, normalize=true>, broadcast_reduce_op.h:606-688)
//
// mean serves the trailing axis of a dense GPU array of rank 2 or more, in float16, bfloat16,
// float32 or float64, one launch of the row-mean kernel (reduce_kernels.cu). Every other axis,
// exclude=True, integer dtypes and an `out` of another shape or dtype are refused before anything
// is enqueued.
#include "kernels.h"
#include "op_params.h"
#include "ops.h"

namespace b200kv {
namespace {

// square: mshadow_op::square on every Elementwise dtype
void Square(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
            const Params&) {
  KV_CHECK_EQ(in.size(), 1u) << op.name << " expects 1 input";
  NDArray o = OutOr(outputs, 0, in[0].shape(), in[0].ctx(), in[0].dtype());
  Elementwise(kEwSquare, in[0], nullptr, 0.0, o);
}

// ReduceAxesParam's axis, a bare int or a tuple such as "(1,)", naming the last of `ndim` axes
bool NamesLastAxis(const Params& p, size_t ndim) {
  const std::string* v = Find(p, "axis");
  if (v == nullptr || *v == "None") return false;
  const std::vector<int> axes = GetIntTuple(p, "axis");
  if (axes.size() != 1) return false;
  const int a = axes[0];
  return a == -1 || a == static_cast<int>(ndim) - 1;
}

// mean(data, axis, keepdims, exclude) over the trailing axis
void Mean(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
          const Params& p) {
  KV_CHECK_EQ(in.size(), 1u) << op.name << " expects 1 input";
  RejectUnknownKeys(p, {"axis", "keepdims", "exclude"});
  const NDArray& x = in[0];
  KV_CHECK(x.on_gpu()) << op.name << " runs on GPU arrays only";
  KV_CHECK(x.stype() == kDefaultStorage) << op.name << " takes dense arrays only";
  const int t = x.dtype();
  KV_CHECK(t == kFloat16 || t == kBfloat16 || t == kFloat32 || t == kFloat64)
      << op.name << ": float16, bfloat16, float32 and float64 arrays only; got " << DTypeName(t);
  const std::vector<int64_t>& shape = x.shape();
  KV_CHECK(shape.size() >= 2) << op.name << ": only the last axis of an array of rank 2 or more is "
                              << "supported; got rank " << shape.size();
  const std::string* axis = Find(p, "axis");
  KV_CHECK(NamesLastAxis(p, shape.size()))
      << op.name << ": only the last axis (" << shape.size() - 1 << " or -1) is supported; got axis="
      << (axis ? *axis : std::string("None"));
  KV_CHECK(!GetB(p, "exclude", false)) << op.name << ": exclude=True is not supported";
  std::vector<int64_t> small(shape.begin(), shape.end() - 1);
  if (GetB(p, "keepdims", false)) small.push_back(1);
  if (!outputs->empty()) {
    const NDArray& o = (*outputs)[0];
    KV_CHECK(o.on_gpu() && o.dev() == x.dev()) << "all operands must be on the same GPU";
    KV_CHECK(o.stype() == kDefaultStorage) << op.name << " takes dense arrays only; out is not dense";
    KV_CHECK(o.shape() == small) << op.name << ": out has the wrong shape";
    KV_CHECK_EQ(o.dtype(), t) << op.name << ": out dtype differs from the input's";
  }
  NDArray o = OutOr(outputs, 0, small, x.ctx(), t);
  const int64_t cols = shape.back();
  const int64_t rows = static_cast<int64_t>(o.Size());
  LaneOp lop(x.dev());
  lop.Read(x).Write(o);
  LaunchRowMean(t, o.data(), x.data(), rows, cols, lop.stream());
  Engine::Get()->CountLaunch("row_mean", 0);
  lop.Issue();
}

}  // namespace

const std::vector<OpInfo> kReduceOps = {
    {"square", Square, 0},
    {"mean", Mean, 0},
};

}  // namespace b200kv
