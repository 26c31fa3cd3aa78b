// TEST INFRASTRUCTURE ONLY -- never linked into or loaded by the product library.
//
// oracle/_ref/libmxref_rdiv.so: _rdiv_scalar (scalar / x), the operator the reference's
// exponential(scale=NDArray) calls for lam = 1.0 / scale, evaluated with the reference's own code on
// top of the arithmetic oracle (ref_arith_ops.cc, included whole): the attribute parser
// _rdiv_scalar registers (std::stod), captured from elemwise_binary_scalar_op_basic.cc:185, then
// BinaryScalarOp's DType(alpha) and mshadow_op::rdiv (mshadow_op.h:709). Dtype codes are mshadow's
// type flags (0 float32, 1 float64, 2 float16).
#include "ref_arith_ops.cc"

extern "C" {

// _rdiv_scalar(scalar=...): the parsed double, and the array
int mxref_ar_rdiv_scalar(int dtype, const void* a, const char* scalar, double* parsed, void* out, int64_t n,
                         char* err, int errlen) {
  try {
    nnvm::NodeAttrs attrs;
    attrs.dict["scalar"] = scalar;
    mxref_nd::CapturedOp::Get("_rdiv_scalar").parser(&attrs);
    const double alpha = nnvm::get<double>(attrs.parsed);
    *parsed = alpha;
    REF_TYPE_SWITCH(dtype, DType, { MapScalar<mop::rdiv, DType>(a, alpha, out, n); });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

}  // extern "C"
