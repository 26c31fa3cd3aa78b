// TEST INFRASTRUCTURE ONLY -- never linked into or loaded by the product library.
//
// oracle/_ref/libmxref_clip.so: the scalar arithmetic of gluon.utils.clip_global_norm
// (python/mxnet/gluon/utils.py:143-153) and of amp.unscale's `g[:] *= scale`, evaluated with the
// reference's own functors, compiled from src/operator/mshadow_op.h and mshadow/base.h where they
// lie (nothing is copied):
//   sqrt              mshadow_op::square_root                         mshadow_op.h:627
//   _plus_scalar      mshadow_op::plus, scalar std::stod -> DType     mshadow_op.h:354,
//   _rdiv_scalar      mshadow_op::rdiv, likewise                      mshadow_op.h:709,
//   _mul_scalar       mshadow_op::mul, likewise                       elemwise_binary_scalar_op.h:364-365
//   min(concat(s, 1)) mshadow::red::minimum from its initial value    mshadow/base.h:947-991
//   broadcast_mul     mshadow_op::mul                                 mshadow_op.h:350
// The Python front-end formats every scalar with str(); `1e-8` therefore arrives as "1e-08".
#include <cstdint>
#include <cstring>
#include <string>
#include <mshadow/base.h>
#include "operator/mshadow_op.h"

namespace {

// the attr parser of MXNET_OPERATOR_REGISTER_BINARY_SCALAR, then BinaryScalarOp::Compute's DType(alpha)
float Scalar(const char* s) { return static_cast<float>(std::stod(std::string(s))); }

int Fail(const std::exception& e, char* err, int errlen) {
  if (err && errlen > 0) {
    std::strncpy(err, e.what(), errlen - 1);
    err[errlen - 1] = '\0';
  }
  return -1;
}

}  // namespace

extern "C" {

// utils.py:144: total_norm = sqrt(sum of squares)
float mxref_clip_sqrt(float ss) { return mxnet::op::mshadow_op::square_root::Map(ss); }

// utils.py:150-151: scale = min(concat(max_norm / (total_norm + 1e-8), ones(1)))
int mxref_clip_scale(float total_norm, const char* max_norm, float* scale, char* err, int errlen) {
  try {
    using namespace mxnet::op::mshadow_op;
    const float t = plus::Map(total_norm, Scalar("1e-08"));
    const float s = rdiv::Map(t, Scalar(max_norm));
    float m;
    mshadow::red::minimum::SetInitValue(m);
    mshadow::red::minimum::Reduce(m, s);
    mshadow::red::minimum::Reduce(m, 1.0f);
    *scale = m;
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

// utils.py:153: arr *= scale (broadcast_mul by the (1,) array), in place
void mxref_clip_mul(float* x, int64_t n, float scale) {
  for (int64_t i = 0; i < n; ++i) x[i] = mxnet::op::mshadow_op::mul::Map(x[i], scale);
}

// amp.py:345: g[:] *= scalar (_mul_scalar), in place
int mxref_mul_scalar(float* x, int64_t n, const char* scalar, char* err, int errlen) {
  try {
    const float s = Scalar(scalar);
    for (int64_t i = 0; i < n; ++i) x[i] = mxnet::op::mshadow_op::mul::Map(x[i], s);
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

// utils.py:136-143: the sum of the arrays' squared 2-norms as the CPU folds it in float32, element
// by element in list order (square = mul(x, x), then plus). The GPU's association differs, so this
// is a tolerance reference, not a bit reference.
float mxref_clip_sum_sq(const float* const* arrays, const int64_t* sizes, int n) {
  using namespace mxnet::op::mshadow_op;
  float ss = 0.f;
  for (int k = 0; k < n; ++k) {
    for (int64_t i = 0; i < sizes[k]; ++i) ss = plus::Map(ss, square::Map(arrays[k][i]));
  }
  return ss;
}

}  // extern "C"
