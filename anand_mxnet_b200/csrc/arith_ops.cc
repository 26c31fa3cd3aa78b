// arith_ops.cc -- the NDArray arithmetic that the reference's Adamax, Nadam and AdaDelta optimizers
// compose in their `update` (python/mxnet/optimizer/optimizer.py:1768-1825, 1904-2029): `nd + nd`,
// `nd - nd`, `nd * nd`, `nd / nd`, `nd / scalar`, maximum, abs and clip. Each call is one launch of
// the elementwise kernel (misc_kernels.cu) through Elementwise.
//
// Reference operator definitions:
//   broadcast_add / _sub / _mul / _div / _maximum   tensor/elemwise_binary_broadcast_op_basic.cc,
//                                                    _extended.cc; mshadow_op.h:350-356, 1083-1092
//   _div_scalar                                     tensor/elemwise_binary_scalar_op_basic.cc:162-176
//   abs                                             tensor/elemwise_unary_op_basic.cc:707; mshadow_op.h:545
//   clip                                            tensor/matrix_op.cc:657-700, matrix_op-inl.h:1593-1617
//
// Operands of one shape, or an rhs of one value per row: shape lhs.shape[:-1] + (1,) against an lhs
// of rank 2 or more, the `grad / sqrt(history + eps)` of the reference's GroupAdaGrad (contrib.py:
// 94-100). Every other broadcast is refused. Integer division is refused, since the reference's
// integer arithmetic traps on a zero divisor.
#include <algorithm>
#include <sstream>

#include "kernels.h"
#include "op_params.h"
#include "ops.h"

namespace b200kv {
namespace {

std::string ShapeText(const std::vector<int64_t>& s) {
  std::ostringstream os;
  os << "(";
  for (size_t i = 0; i < s.size(); ++i) os << (i ? ", " : "") << s[i];
  os << (s.size() == 1 ? ",)" : ")");
  return os.str();
}

void RefuseIntegerDivision(const OpInfo& op, const NDArray& a) {
  const int t = a.dtype();
  KV_CHECK(t == kFloat16 || t == kBfloat16 || t == kFloat32 || t == kFloat64)
      << op.name << ": integer division is not supported (" << DTypeName(t)
      << "); divide float16, bfloat16, float32 or float64 arrays";
}

// rhs's shape is lhs's with its last axis 1, lhs of rank 2 or more
bool RowOperand(const std::vector<int64_t>& lhs, const std::vector<int64_t>& rhs) {
  return lhs.size() >= 2 && rhs.size() == lhs.size() && rhs.back() == 1 &&
         std::equal(lhs.begin(), lhs.end() - 1, rhs.begin());
}

// broadcast_add, broadcast_sub, broadcast_mul, broadcast_div, broadcast_maximum (variant: the kEw*
// code)
void Broadcast(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
               const Params&) {
  KV_CHECK_EQ(in.size(), 2u) << op.name << " expects 2 inputs";
  const bool same = in[0].shape() == in[1].shape();
  KV_CHECK(same || RowOperand(in[0].shape(), in[1].shape()))
      << op.name << ": operands of shapes " << ShapeText(in[0].shape()) << " and "
      << ShapeText(in[1].shape()) << " would broadcast; only operands of equal shapes are supported, "
      << "or an rhs of shape lhs.shape[:-1] + (1,)";
  if (op.variant == kEwDiv) RefuseIntegerDivision(op, in[0]);
  NDArray o = OutOr(outputs, 0, in[0].shape(), in[0].ctx(), in[0].dtype());
  if (same) Elementwise(op.variant, in[0], &in[1], 0.0, o);
  else ElementwiseRows(op.variant, in[0], in[1], o);
}

// _div_scalar (its scalar: std::stod, then DType(alpha) in the kernel) and abs (variant: the kEw* code)
void Unary(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
           const Params& p) {
  KV_CHECK_EQ(in.size(), 1u) << op.name << " expects 1 input";
  const bool div = op.variant == kEwDivScalar;
  const double scalar = div ? StodD(p, "scalar", op.name) : 0.0;
  if (div) RefuseIntegerDivision(op, in[0]);
  NDArray o = OutOr(outputs, 0, in[0].shape(), in[0].ctx(), in[0].dtype());
  Elementwise(op.variant, in[0], nullptr, scalar, o);
}

// clip: ClipParam's two required real_t fields, parsed by dmlc::stof
void Clip(const OpInfo& op, const std::vector<NDArray>& in, std::vector<NDArray>* outputs,
          const Params& p) {
  KV_CHECK_EQ(in.size(), 1u) << op.name << " expects 1 input";
  RejectUnknownKeys(p, {"a_min", "a_max"});
  const float a_min = Required(p, "a_min", op.name);
  const float a_max = Required(p, "a_max", op.name);
  NDArray o = OutOr(outputs, 0, in[0].shape(), in[0].ctx(), in[0].dtype());
  Elementwise(kEwClip, in[0], nullptr, a_min, o, a_max);
}

}  // namespace

const std::vector<OpInfo> kArithOps = {
    {"broadcast_add", Broadcast, kEwAdd},
    {"broadcast_sub", Broadcast, kEwSub},
    {"broadcast_mul", Broadcast, kEwMul},
    {"broadcast_div", Broadcast, kEwDiv},
    {"broadcast_maximum", Broadcast, kEwMax},
    {"_div_scalar", Unary, kEwDivScalar},
    {"abs", Unary, kEwAbs},
    {"clip", Clip, 0},
};

}  // namespace b200kv
