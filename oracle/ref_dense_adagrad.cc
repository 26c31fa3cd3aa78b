// TEST INFRASTRUCTURE ONLY -- never linked into or loaded by the product library.
//
// oracle/_ref/libmxref_dense_adagrad.so: the operators the dense-gradient branches of the
// reference's AdaGrad and GroupAdaGrad add to the Adamax / Nadam / AdaDelta arithmetic, for half_t,
// float32, float64, int32 and int64, evaluated with the reference's own code, compiled where it
// lies (nothing is copied). It builds on oracle/ref_ndarray_ops.cc, included whole:
//   square              mshadow_op::square over math::sqr           mshadow_op.h:536,
//                                                                   math_functions-inl.h:139-147
//   mean                ReduceAxesParam's dmlc::Parameter parse, ReduceAxesShapeImpl, then
//                       ReduceAxesComputeImpl's body: broadcast::Reduce<red::sum, ..., safe_acc =
//                       false> (seq_reduce_compute) and `out /= scalar<DType>(M)`
//                                                                   broadcast_reduce_op.h:606-688
//                       (the body is called directly, not ReduceAxesComputeImpl itself: that asks
//                       an OpContext for a temp-space resource, which needs libmxnet's resource
//                       manager; the CPU Reduce never reads the workspace)
//   broadcast_add / _sub / _mul / _div / _maximum with a row operand
//                       BinaryBroadcastCompute<cpu, OP>'s broadcasting branch: the shapes
//                       compacted, then binary_broadcast_kernel   elemwise_binary_broadcast_op.h:
//                                                                   191-215, 366-395
// Dtype codes are mshadow's type flags (0 float32, 1 float64, 2 float16, 4 int32, 6 int64).
#include "ref_ndarray_ops.cc"
#include "operator/tensor/broadcast_reduce_op.h"

namespace mxnet {
namespace op {
DMLC_REGISTER_PARAMETER(ReduceAxesParam);

// ReduceAxesComputeImpl<cpu, red::sum, safe_acc = false, normalize = true>'s body, from the
// compacted shapes on
template <typename DType>
void MxrefMean(const void* in, void* out, const TShape& src_shape, const TShape& dst_shape, int dtype) {
  using namespace mshadow;
  using namespace mshadow::expr;
  Stream<cpu> stream;
  Stream<cpu>* s = &stream;
  char ws_byte = 0;
  Tensor<cpu, 1, char> workspace(&ws_byte, Shape1(0));
  const TBlob in_data(const_cast<void*>(in), src_shape, cpu::kDevMask, dtype);
  const TBlob out_data(out, dst_shape, cpu::kDevMask, dtype);
  BROADCAST_NDIM_SWITCH(dst_shape.ndim(), NDim, {
    broadcast::Reduce<red::sum, NDim, DType, op::mshadow_op::identity, false>(s, out_data, kWriteTo,
                                                                             workspace, in_data);
    auto o = out_data.FlatTo2D<cpu, DType>(s);
    o /= scalar<DType>(src_shape.Size() / dst_shape.Size());
  });
}

// BinaryBroadcastCompute<cpu, OP>'s broadcasting branch (elemwise_binary_broadcast_op.h:373-393);
// the equal-shape branch it takes otherwise is the elementwise functor of ref_ndarray_ops.cc
template <typename OP, typename DType>
void MxrefBroadcast(const void* a, const void* b, void* out, const TShape& ls, const TShape& rs) {
  mshadow::Stream<cpu> stream;
  mxnet::TShape new_lshape, new_rshape, new_oshape;
  const int ndim = BinaryBroadcastShapeCompact(ls, rs, ls, &new_lshape, &new_rshape, &new_oshape);
  if (!ndim) throw std::invalid_argument("operands of equal shapes: not a broadcast");
  BROADCAST_NDIM_SWITCH(ndim, NDim, {
    mshadow::Shape<NDim> oshape = new_oshape.get<NDim>();
    mshadow::Shape<NDim> lstride = mxnet_op::calc_stride(new_lshape.get<NDim>());
    mshadow::Shape<NDim> rstride = mxnet_op::calc_stride(new_rshape.get<NDim>());
    mxnet_op::Kernel<mxnet_op::binary_broadcast_kernel<NDim, OP>, cpu>::template LaunchEx(
        &stream, new_oshape.Size(), kWriteTo, lstride, rstride, oshape,
        static_cast<DType*>(const_cast<void*>(a)), static_cast<DType*>(const_cast<void*>(b)),
        static_cast<DType*>(out));
  });
}
}  // namespace op
}  // namespace mxnet

namespace {

mxnet::TShape ShapeOf(int ndim, const int64_t* shape) {
  mxnet::TShape s(ndim, 1);
  for (int i = 0; i < ndim; ++i) s[i] = shape[i];
  return s;
}

template <typename OP>
void RowBroadcast(int dtype, const void* a, const void* b, void* out, int ndim, const int64_t* lshape,
                  const int64_t* rshape) {
  REF_TYPE_SWITCH(dtype, DType, {
    mxnet::op::MxrefBroadcast<OP, DType>(a, b, out, ShapeOf(ndim, lshape), ShapeOf(ndim, rshape));
  });
}

}  // namespace

extern "C" {

int mxref_da_square(int dtype, const void* a, void* out, int64_t n, char* err, int errlen) {
  try {
    REF_TYPE_SWITCH(dtype, DType, {
      const DType* x = static_cast<const DType*>(a);
      DType* o = static_cast<DType*>(out);
      for (int64_t i = 0; i < n; ++i) o[i] = mop::square::Map(x[i]);
    });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

// mean(data, axis=..., keepdims=..., exclude=...) on a float dtype: the output's shape
// (out_ndim, out_shape: room for 8) and values. `out` holds room for the keepdims-shaped result.
int mxref_da_mean(int dtype, const void* in, int ndim, const int64_t* shape, const char* axis,
                  const char* keepdims, const char* exclude, void* out, int* out_ndim,
                  int64_t* out_shape, char* err, int errlen) {
  try {
    mxnet::op::ReduceAxesParam param;
    std::vector<std::pair<std::string, std::string>> kw;
    if (axis) kw.emplace_back("axis", axis);
    if (keepdims) kw.emplace_back("keepdims", keepdims);
    if (exclude) kw.emplace_back("exclude", exclude);
    param.Init(kw);
    const mxnet::TShape ishape = ShapeOf(ndim, shape);
    const mxnet::TShape oshape =
        mxnet::op::ReduceAxesShapeImpl(ishape, param.axis, param.keepdims, param.exclude);
    *out_ndim = oshape.ndim();
    for (int i = 0; i < oshape.ndim(); ++i) out_shape[i] = oshape[i];
    // ReduceAxesCompute: `small` is the keepdims shape
    const mxnet::TShape small = mxnet::op::ReduceAxesShapeImpl(ishape, param.axis, true, param.exclude);
    mxnet::TShape src_shape, dst_shape;
    mxnet::op::BroadcastReduceShapeCompact(ishape, small, &src_shape, &dst_shape);
    REF_TYPE_SWITCH(dtype, DType, { mxnet::op::MxrefMean<DType>(in, out, src_shape, dst_shape, dtype); });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

// op: 0 broadcast_add, 1 broadcast_sub, 2 broadcast_mul, 3 broadcast_div, 4 broadcast_maximum;
// lhs and rhs of rank ndim, out of lhs's shape
int mxref_da_broadcast(int op, int dtype, const void* a, const void* b, void* out, int ndim,
                       const int64_t* lshape, const int64_t* rshape, char* err, int errlen) {
  try {
    switch (op) {
      case 0: RowBroadcast<mop::plus>(dtype, a, b, out, ndim, lshape, rshape); break;
      case 1: RowBroadcast<mop::minus>(dtype, a, b, out, ndim, lshape, rshape); break;
      case 2: RowBroadcast<mop::mul>(dtype, a, b, out, ndim, lshape, rshape); break;
      case 3: RowBroadcast<mop::div>(dtype, a, b, out, ndim, lshape, rshape); break;
      default: RowBroadcast<mop::maximum>(dtype, a, b, out, ndim, lshape, rshape); break;
    }
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

}  // extern "C"
