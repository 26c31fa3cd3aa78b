// TEST INFRASTRUCTURE ONLY -- never linked into or loaded by the product library.
//
// oracle/_ref/libmxref_arith.so: the arithmetic the reference's Adamax, Nadam and AdaDelta
// optimizers compose, for half_t, float32, float64, int32 and int64, evaluated with the reference's
// own code, compiled where it lies (nothing is copied). It builds on oracle/ref_ndarray_ops.cc,
// included whole, whose mxref_nd_binary already runs broadcast_add / _sub / _mul's functors:
//   broadcast_div / broadcast_maximum   mshadow_op::div, maximum             mshadow_op.h:352, 1083-1092
//   _div_scalar                         the attribute parser it registers (std::stod), captured from
//                                       elemwise_binary_scalar_op_basic.cc:162, then DType(alpha) and
//                                       mshadow_op::div
//   abs                                 mshadow_op::abs over math::fabs      mshadow_op.h:545
//   clip                                ClipParam's dmlc::Parameter parse of a_min / a_max, then the
//                                       clip kernel's Map                    matrix_op-inl.h:1593-1617
// Dtype codes are mshadow's type flags (0 float32, 1 float64, 2 float16, 4 int32, 6 int64).
#include "ref_ndarray_ops.cc"
#include "operator/tensor/matrix_op-inl.h"

namespace mxnet {
namespace op {
DMLC_REGISTER_PARAMETER(ClipParam);
}  // namespace op
}  // namespace mxnet

extern "C" {

// op: 0 broadcast_div, 1 broadcast_maximum
int mxref_ar_binary(int op, int dtype, const void* a, const void* b, void* out, int64_t n, char* err,
                    int errlen) {
  try {
    REF_TYPE_SWITCH(dtype, DType, {
      if (op == 0) Map2<mop::div, DType>(a, b, out, n);
      else Map2<mop::maximum, DType>(a, b, out, n);
    });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

// _div_scalar(scalar=...): the parsed double, and the array
int mxref_ar_div_scalar(int dtype, const void* a, const char* scalar, double* parsed, void* out,
                        int64_t n, char* err, int errlen) {
  try {
    nnvm::NodeAttrs attrs;
    attrs.dict["scalar"] = scalar;
    mxref_nd::CapturedOp::Get("_div_scalar").parser(&attrs);
    const double alpha = nnvm::get<double>(attrs.parsed);
    *parsed = alpha;
    REF_TYPE_SWITCH(dtype, DType, { MapScalar<mop::div, DType>(a, alpha, out, n); });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

int mxref_ar_abs(int dtype, const void* a, void* out, int64_t n, char* err, int errlen) {
  try {
    REF_TYPE_SWITCH(dtype, DType, {
      const DType* x = static_cast<const DType*>(a);
      DType* o = static_cast<DType*>(out);
      for (int64_t i = 0; i < n; ++i) o[i] = mop::abs::Map(x[i]);
    });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

// clip(a_min=..., a_max=...): the parsed bounds, and the array
int mxref_ar_clip(int dtype, const void* a, const char* a_min, const char* a_max, float* parsed,
                  void* out, int64_t n, char* err, int errlen) {
  try {
    mxnet::op::ClipParam param;
    param.Init(std::vector<std::pair<std::string, std::string>>{{"a_min", a_min}, {"a_max", a_max}});
    parsed[0] = param.a_min;
    parsed[1] = param.a_max;
    REF_TYPE_SWITCH(dtype, DType, {
      const DType* x = static_cast<const DType*>(a);
      DType* o = static_cast<DType*>(out);
      for (int64_t i = 0; i < n; ++i) mxnet::op::clip::Map(i, o, x, param.a_min, param.a_max);
    });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

}  // extern "C"
