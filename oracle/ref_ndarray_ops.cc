// TEST INFRASTRUCTURE ONLY -- never linked into or loaded by the product library.
//
// oracle/_ref/libmxref_ndarith.so: the NDArray arithmetic, fill and cast operators that custom
// updaters run, for half_t, float32, float64, int32 and int64, evaluated with the reference's own
// code, compiled where it lies (nothing is copied):
//   _plus / _minus / _mul      mshadow_op::plus, minus, mul                     mshadow_op.h:350-356
//   _plus_scalar / _minus_scalar / _mul_scalar
//                              the attribute parser each one registers (std::stod), captured from
//                              elemwise_binary_scalar_op_basic.cc compiled in place with
//                              NNVM_REGISTER_OP redefined, then BinaryScalarOp's DType(alpha)
//                              and the functor           elemwise_binary_scalar_op_basic.cc:29-45,
//                                                        123-140; elemwise_binary_scalar_op.h:347-375
//   sqrt                       mshadow_op::square_root over math::sqrt   mshadow_op.h:627,
//                                                                        math_functions-inl.h:43-55
//   _full (a[:] = v)           InitOpWithScalarParam's dmlc::Parameter parse of `value`, then Fill's
//                              static_cast<DType> into mshadow_op::identity      init_op.h:241-260, 381-421
//   cast / astype              CastCompute's tcast<DstDType> over mshadow tensors  elemwise_unary_op.h:476
// Dtype codes are mshadow's type flags (0 float32, 1 float64, 2 float16, 4 int32, 6 int64).
// Fill itself cannot be linked without libmxnet (features::is_enabled); its two branches are
// restated below around the reference's conversion and functor.
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <string>
#include <mshadow/base.h>
#include <mshadow/tensor.h>
#include "operator/mshadow_op.h"
#include "operator/tensor/init_op.h"
#include "operator/tensor/elemwise_binary_scalar_op.h"

namespace mxref_nd {
// An NNVM_REGISTER_OP stand-in that keeps the attribute parser an operator registers and drops
// every other attribute: this library has no nnvm::Op registry.
struct CapturedOp {
  std::function<void(nnvm::NodeAttrs*)> parser;
  template <typename F> CapturedOp& set_attr_parser(F f) {
    parser = f;
    return *this;
  }
  template <typename... A> CapturedOp& set_num_inputs(A&&...) { return *this; }
  template <typename... A> CapturedOp& set_num_outputs(A&&...) { return *this; }
  template <typename T, typename... A> CapturedOp& set_attr(A&&...) { return *this; }
  template <typename... A> CapturedOp& add_argument(A&&...) { return *this; }
  template <typename... A> CapturedOp& add_arguments(A&&...) { return *this; }
  template <typename... A> CapturedOp& add_alias(A&&...) { return *this; }
  template <typename... A> CapturedOp& describe(A&&...) { return *this; }
  static CapturedOp& Get(const std::string& name) {
    static std::map<std::string, CapturedOp> ops;
    return ops[name];
  }
};
}  // namespace mxref_nd

#undef NNVM_REGISTER_OP
#define NNVM_REGISTER_OP(name) \
  static ::mxref_nd::CapturedOp& captured_##name __attribute__((unused)) = \
      ::mxref_nd::CapturedOp::Get(#name)

// the operators' own registrations, compiled where they lie
#include "operator/tensor/elemwise_binary_scalar_op_basic.cc"

namespace mxnet {
namespace op {
DMLC_REGISTER_PARAMETER(InitOpWithScalarParam);
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

using mshadow::half::half_t;
namespace mop = mxnet::op::mshadow_op;

int Fail(const std::exception& e, char* err, int errlen) {
  if (err && errlen > 0) {
    std::strncpy(err, e.what(), errlen - 1);
    err[errlen - 1] = '\0';
  }
  return -1;
}

#define REF_TYPE_SWITCH(flag, DType, ...)                   \
  switch (flag) {                                           \
    case 0: { typedef float DType; __VA_ARGS__ } break;     \
    case 1: { typedef double DType; __VA_ARGS__ } break;    \
    case 2: { typedef half_t DType; __VA_ARGS__ } break;    \
    case 4: { typedef int32_t DType; __VA_ARGS__ } break;   \
    case 6: { typedef int64_t DType; __VA_ARGS__ } break;   \
    default: throw std::invalid_argument("unsupported dtype flag " + std::to_string(flag)); \
  }

template <typename OP, typename DType>
void Map2(const void* a, const void* b, void* out, int64_t n) {
  const DType* x = static_cast<const DType*>(a);
  const DType* y = static_cast<const DType*>(b);
  DType* o = static_cast<DType*>(out);
  for (int64_t i = 0; i < n; ++i) o[i] = OP::Map(x[i], y[i]);
}

template <typename OP, typename DType>
void MapScalar(const void* a, double alpha, void* out, int64_t n) {
  const DType* x = static_cast<const DType*>(a);
  DType* o = static_cast<DType*>(out);
  const DType s = DType(alpha);
  for (int64_t i = 0; i < n; ++i) o[i] = OP::Map(x[i], s);
}

}  // namespace

extern "C" {

// op: 0 plus, 1 minus, 2 mul
int mxref_nd_binary(int op, int dtype, const void* a, const void* b, void* out, int64_t n, char* err,
                    int errlen) {
  try {
    REF_TYPE_SWITCH(dtype, DType, {
      if (op == 0) Map2<mop::plus, DType>(a, b, out, n);
      else if (op == 1) Map2<mop::minus, DType>(a, b, out, n);
      else Map2<mop::mul, DType>(a, b, out, n);
    });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

// op: 0 _plus_scalar, 1 _minus_scalar, 2 _mul_scalar; `scalar` is the attribute string
int mxref_nd_scalar(int op, int dtype, const void* a, const char* scalar, void* out, int64_t n,
                    char* err, int errlen) {
  try {
    static const char* const kNames[] = {"_plus_scalar", "_minus_scalar", "_mul_scalar"};
    nnvm::NodeAttrs attrs;
    attrs.dict["scalar"] = scalar;
    mxref_nd::CapturedOp::Get(kNames[op]).parser(&attrs);
    const double alpha = nnvm::get<double>(attrs.parsed);
    REF_TYPE_SWITCH(dtype, DType, {
      if (op == 0) MapScalar<mop::plus, DType>(a, alpha, out, n);
      else if (op == 1) MapScalar<mop::minus, DType>(a, alpha, out, n);
      else MapScalar<mop::mul, DType>(a, alpha, out, n);
    });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

int mxref_nd_sqrt(int dtype, const void* a, void* out, int64_t n, char* err, int errlen) {
  try {
    REF_TYPE_SWITCH(dtype, DType, {
      const DType* x = static_cast<const DType*>(a);
      DType* o = static_cast<DType*>(out);
      for (int64_t i = 0; i < n; ++i) o[i] = mop::square_root::Map(x[i]);
    });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

// _full(value=...): the parsed double, and the array Fill leaves
int mxref_nd_full(int dtype, const char* value, double* parsed, void* out, int64_t n, char* err,
                  int errlen) {
  try {
    mxnet::op::InitOpWithScalarParam param;
    param.Init(std::vector<std::pair<std::string, std::string>>{{"value", value}});
    const double val = param.value;
    *parsed = val;
    REF_TYPE_SWITCH(dtype, DType, {
      DType* o = static_cast<DType*>(out);
      if (val == 0) {
        std::memset(o, 0, n * sizeof(DType));  // Fill's val == 0 branch: set_to_int<0> / memset
      } else {
        for (int64_t i = 0; i < n; ++i) o[i] = mop::identity::Map(static_cast<DType>(val));
      }
    });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

// cast(dtype=out_dtype)
int mxref_nd_cast(int out_dtype, const void* in, int in_dtype, void* out, int64_t n, char* err,
                  int errlen) {
  try {
    REF_TYPE_SWITCH(out_dtype, DstDType, {
      REF_TYPE_SWITCH(in_dtype, SrcDType, {
        mshadow::Tensor<mshadow::cpu, 1, DstDType> o(static_cast<DstDType*>(out),
                                                     mshadow::Shape1(n));
        mshadow::Tensor<mshadow::cpu, 1, SrcDType> x(
            const_cast<SrcDType*>(static_cast<const SrcDType*>(in)), mshadow::Shape1(n));
        if (n != 0) o = mshadow::expr::tcast<DstDType>(x);
      });
    });
    return 0;
  } catch (const std::exception& e) {
    return Fail(e, err, errlen);
  }
}

}  // extern "C"
