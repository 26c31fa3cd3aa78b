// misc_kernels.cu -- small elementwise kernels behind the imperative-op surface (custom updaters
// written in the host language: `local += recv`, `weight[:] += grad * rescale`, casts, fills).
// Not on the measured hot path; kept simple: one element per thread, grid-stride.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "common.h"
#include "kernels.h"

namespace b200kv {
namespace {

// The 16-bit types compute in float and round once (half.h:45-66, MSHADOW_HALF_OPERATOR; bfloat16
// is treated the same). Every other type computes in its own arithmetic, as mshadow_op's functors
// do for float, double, int32 and int64.
template <typename T> struct Is16 : std::false_type {};
template <> struct Is16<__half> : std::true_type {};
template <> struct Is16<__nv_bfloat16> : std::true_type {};

template <typename T> struct Calc { typedef T type; };
template <> struct Calc<__half> { typedef float type; };
template <> struct Calc<__nv_bfloat16> { typedef float type; };

__device__ __forceinline__ float Widen(__half x) { return __half2float(x); }
__device__ __forceinline__ float Widen(__nv_bfloat16 x) { return __bfloat162float(x); }
template <typename T> __device__ __forceinline__ T Widen(T x) { return x; }

// float -> T, rounding to nearest even: half_t's float constructor (half.h:322-330)
template <typename T> __device__ __forceinline__ T FromFloat(float x) { return static_cast<T>(x); }
template <> __device__ __forceinline__ __half FromFloat<__half>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ __nv_bfloat16 FromFloat<__nv_bfloat16>(float x) {
  return __float2bfloat16_rn(x);
}

template <typename T> __device__ __forceinline__ T Narrow(typename Calc<T>::type x) {
  if constexpr (Is16<T>::value) return FromFloat<T>(x);
  else return x;
}

// DType(alpha) for the double scalar of an operator; half_t(double) goes through float
// (half.h:118, 322-330), and bfloat16 likewise. Integers truncate.
template <typename T> __device__ __forceinline__ T FromDouble(double s) {
  if constexpr (Is16<T>::value) return FromFloat<T>(__double2float_rn(s));
  else return static_cast<T>(s);
}

__device__ __forceinline__ float Add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double Add(double a, double b) { return __dadd_rn(a, b); }
template <typename I> __device__ __forceinline__ I Add(I a, I b) { return a + b; }
__device__ __forceinline__ float Sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double Sub(double a, double b) { return __dsub_rn(a, b); }
template <typename I> __device__ __forceinline__ I Sub(I a, I b) { return a - b; }
__device__ __forceinline__ float Mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double Mul(double a, double b) { return __dmul_rn(a, b); }
template <typename I> __device__ __forceinline__ I Mul(I a, I b) { return a * b; }
// math::sqrt (math_functions-inl.h:43-55, 92): float in float, integers in double, then DType(...)
__device__ __forceinline__ float Sqrt(float a) { return __fsqrt_rn(a); }
__device__ __forceinline__ double Sqrt(double a) { return __dsqrt_rn(a); }
template <typename I> __device__ __forceinline__ I Sqrt(I a) {
  return static_cast<I>(__dsqrt_rn(static_cast<double>(a)));
}
// mshadow_op::div (mshadow_op.h:352): a / b. Integer arrays never reach it: the operators refuse them.
__device__ __forceinline__ float Div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double Div(double a, double b) { return __ddiv_rn(a, b); }
template <typename I> __device__ __forceinline__ I Div(I a, I b) { return a / b; }
// mshadow_op::maximum (mshadow_op.h:1083-1092): a NaN `a` is returned, else a > b ? a : b, so a NaN
// `b` and equal values (-0 against +0) give b. `a != a` is IsNan for floats and false for integers.
template <typename C> __device__ __forceinline__ C Max(C a, C b) { return a != a ? a : (a > b ? a : b); }
// mshadow_op::abs over math::fabs (mshadow_op.h:545, math_functions-inl.h:43-55): fabsf for float,
// fabs for double, integers through double and back
__device__ __forceinline__ float Abs(float a) { return fabsf(a); }
__device__ __forceinline__ double Abs(double a) { return fabs(a); }
template <typename I> __device__ __forceinline__ I Abs(I a) {
  return static_cast<I>(fabs(static_cast<double>(a)));
}
// the clip kernel (matrix_op-inl.h:1604-1617): each element against the float bounds in C++'s
// arithmetic, so an integer converts to float and a double compares with the widened bound; a
// bound taken is converted to the dtype (the 16-bit types round it from float). NaN falls through.
template <typename C> __device__ __forceinline__ C Clip(C x, float lo, float hi) {
  if (x > hi) return static_cast<C>(hi);
  if (x < lo) return static_cast<C>(lo);
  return x;
}
// mshadow_op::square over math::sqr (mshadow_op.h:536, math_functions-inl.h:139-147): float(a) *
// float(a) for every type but double, then DType(...); an integer square above 2^24 loses bits
__device__ __forceinline__ float Square(float a) { return __fmul_rn(a, a); }
__device__ __forceinline__ double Square(double a) { return __dmul_rn(a, a); }
template <typename I> __device__ __forceinline__ I Square(I a) {
  const float f = static_cast<float>(a);
  return static_cast<I>(__fmul_rn(f, f));
}

// b_row > 0: b holds one value per row of b_row elements, read as b[i / b_row] (the row broadcast
// of binary_broadcast_kernel with an rhs of shape lhs.shape[:-1] + (1,))
template <typename T>
__global__ void ew_kernel(int op, T* out, const T* a, const T* b, double scalar, double scalar2,
                          size_t n, size_t b_row) {
  typedef typename Calc<T>::type C;
  const T s = FromDouble<T>(scalar);
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    if (op == kEwFill) {
      out[i] = s;
      continue;
    }
    if (op == kEwCopy) {
      out[i] = a[i];
      continue;
    }
    const C x = Widen(a[i]);
    const size_t j = b_row ? i / b_row : i;
    C r;
    switch (op) {
      case kEwAdd: r = Add(x, Widen(b[j])); break;
      case kEwSub: r = Sub(x, Widen(b[j])); break;
      case kEwMul: r = Mul(x, Widen(b[j])); break;
      case kEwAddScalar: r = Add(x, Widen(s)); break;
      case kEwMulScalar: r = Mul(x, Widen(s)); break;
      case kEwDiv: r = Div(x, Widen(b[j])); break;
      case kEwMax: r = Max(x, Widen(b[j])); break;
      case kEwDivScalar: r = Div(x, Widen(s)); break;
      case kEwAbs: r = Abs(x); break;
      case kEwClip: r = Clip(x, static_cast<float>(scalar), static_cast<float>(scalar2)); break;
      case kEwSquare: r = Square(x); break;
      case kEwRDivScalar: r = Div(Widen(s), x); break;  // mshadow_op::rdiv
      default: r = Sqrt(x); break;  // kEwSqrt
    }
    out[i] = Narrow<T>(r);
  }
}

// tcast<TO>(in) (elemwise_unary_op.h:476): TO(x). A 16-bit side converts through float, as half_t
// does (half.h:118-126, 322-330); every other pair converts directly.
template <typename TO, typename TI>
__global__ void cast_kernel(TO* out, const TI* in, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    if constexpr (std::is_same<TO, TI>::value) {
      out[i] = in[i];
    } else if constexpr (Is16<TO>::value || Is16<TI>::value) {
      out[i] = FromFloat<TO>(static_cast<float>(Widen(in[i])));
    } else {
      out[i] = static_cast<TO>(in[i]);
    }
  }
}

inline int GridFor(size_t n) {
  size_t blocks = (n + 255) / 256;
  return static_cast<int>(blocks < 1 ? 1 : (blocks > kNumSMs * 16 ? kNumSMs * 16 : blocks));
}

template <typename T>
void ew_launch(int op, void* out, const void* a, const void* b, double scalar, double scalar2,
               size_t n, size_t b_row, cudaStream_t s) {
  ew_kernel<T><<<GridFor(n), 256, 0, s>>>(op, static_cast<T*>(out), static_cast<const T*>(a),
                                          static_cast<const T*>(b), scalar, scalar2, n, b_row);
}

template <typename TO>
void cast_from(void* out, const void* in, int in_dtype, size_t n, cudaStream_t s) {
  const int g = GridFor(n);
  switch (in_dtype) {
    case kFloat32: cast_kernel<TO, float><<<g, 256, 0, s>>>(static_cast<TO*>(out), static_cast<const float*>(in), n); break;
    case kFloat16: cast_kernel<TO, __half><<<g, 256, 0, s>>>(static_cast<TO*>(out), static_cast<const __half*>(in), n); break;
    case kBfloat16: cast_kernel<TO, __nv_bfloat16><<<g, 256, 0, s>>>(static_cast<TO*>(out), static_cast<const __nv_bfloat16*>(in), n); break;
    case kFloat64: cast_kernel<TO, double><<<g, 256, 0, s>>>(static_cast<TO*>(out), static_cast<const double*>(in), n); break;
    case kInt32: cast_kernel<TO, int32_t><<<g, 256, 0, s>>>(static_cast<TO*>(out), static_cast<const int32_t*>(in), n); break;
    case kInt64: cast_kernel<TO, int64_t><<<g, 256, 0, s>>>(static_cast<TO*>(out), static_cast<const int64_t*>(in), n); break;
    case kUint8: cast_kernel<TO, uint8_t><<<g, 256, 0, s>>>(static_cast<TO*>(out), static_cast<const uint8_t*>(in), n); break;
    case kInt8: cast_kernel<TO, int8_t><<<g, 256, 0, s>>>(static_cast<TO*>(out), static_cast<const int8_t*>(in), n); break;
    default: KV_FATAL << "cast: unsupported source dtype " << DTypeName(in_dtype);
  }
}

}  // namespace

bool ElementwiseDTypeOk(int dtype) {
  return dtype == kFloat32 || dtype == kFloat16 || dtype == kBfloat16 || dtype == kFloat64 ||
         dtype == kInt32 || dtype == kInt64;
}

void LaunchElementwise(int op, int dtype, void* out, const void* a, const void* b, double scalar,
                       size_t n, cudaStream_t stream, double scalar2, size_t b_row) {
  if (n == 0) return;
  switch (dtype) {
    case kFloat32: ew_launch<float>(op, out, a, b, scalar, scalar2, n, b_row, stream); break;
    case kFloat16: ew_launch<__half>(op, out, a, b, scalar, scalar2, n, b_row, stream); break;
    case kBfloat16: ew_launch<__nv_bfloat16>(op, out, a, b, scalar, scalar2, n, b_row, stream); break;
    case kFloat64: ew_launch<double>(op, out, a, b, scalar, scalar2, n, b_row, stream); break;
    case kInt32: ew_launch<int32_t>(op, out, a, b, scalar, scalar2, n, b_row, stream); break;
    case kInt64: ew_launch<int64_t>(op, out, a, b, scalar, scalar2, n, b_row, stream); break;
    default: KV_FATAL << "elementwise op: unsupported dtype " << DTypeName(dtype);
  }
  KV_CUDA(cudaGetLastError());
}

void LaunchCast(void* out, int out_dtype, const void* in, int in_dtype, size_t n,
                cudaStream_t stream) {
  if (n == 0) return;
  switch (out_dtype) {
    case kFloat32: cast_from<float>(out, in, in_dtype, n, stream); break;
    case kFloat16: cast_from<__half>(out, in, in_dtype, n, stream); break;
    case kBfloat16: cast_from<__nv_bfloat16>(out, in, in_dtype, n, stream); break;
    case kFloat64: cast_from<double>(out, in, in_dtype, n, stream); break;
    case kInt32: cast_from<int32_t>(out, in, in_dtype, n, stream); break;
    case kInt64: cast_from<int64_t>(out, in, in_dtype, n, stream); break;
    default: KV_FATAL << "cast: unsupported target dtype " << DTypeName(out_dtype);
  }
  KV_CUDA(cudaGetLastError());
}

}  // namespace b200kv
