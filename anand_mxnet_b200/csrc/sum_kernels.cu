// sum_kernels.cu -- add_n / ElementWiseSum over dense arrays (kernels.h, LaunchAddN).
//
// The reference runs one kernel for 2-4 inputs (Sum::sum's right-nested a[i] + sum(i, b...),
// tensor/elemwise_sum.h:37-46) and otherwise n kernels that each read and write out
// (elemwise_sum.h:83-92). Here one launch reads every input once and writes out once, in the same
// association, so that HBM traffic is (n + 1) element sizes per element instead of about 3n.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "common.h"
#include "kernels.h"

namespace b200kv {
namespace {

constexpr int kAddNThreads = 256;
// inputs whose 16-B vectors one thread loads before it folds them: every load of a batch is in
// flight at once. 4 keeps every instantiation at 64 registers or fewer with no spills (8 needs 79).
constexpr int kAddNBatch = 4;

// the input list of one launch, by value in the kernel parameters (no device table)
struct AddNList {
  const void* p[kAddNMaxArrays];
  int32_t count;     // 1..kAddNMaxArrays
  uint32_t right;    // 2-4 inputs: a0 + (a1 + (a2 + a3)); else the left chain
  uint32_t zero_first;
  uint32_t vec;      // every input and out 16-byte aligned: 16-B vectors, then a scalar tail
};
static_assert(sizeof(AddNList) <= 4096, "kernel parameters stay small");

// one + in the dtype: float and double round to nearest; half_t and bfloat16 add in float and
// round once (half.h MSHADOW_HALF_OPERATOR); integers wrap (computed unsigned, so no signed overflow)
__device__ __forceinline__ float Add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double Add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ __half Add(__half a, __half b) {
  return __float2half_rn(__fadd_rn(__half2float(a), __half2float(b)));
}
__device__ __forceinline__ __nv_bfloat16 Add(__nv_bfloat16 a, __nv_bfloat16 b) {
  return __float2bfloat16_rn(__fadd_rn(__bfloat162float(a), __bfloat162float(b)));
}
__device__ __forceinline__ uint8_t Add(uint8_t a, uint8_t b) { return static_cast<uint8_t>(a + b); }
__device__ __forceinline__ int8_t Add(int8_t a, int8_t b) {
  return static_cast<int8_t>(static_cast<uint8_t>(static_cast<uint8_t>(a) + static_cast<uint8_t>(b)));
}
__device__ __forceinline__ int32_t Add(int32_t a, int32_t b) {
  return static_cast<int32_t>(static_cast<uint32_t>(a) + static_cast<uint32_t>(b));
}
__device__ __forceinline__ int64_t Add(int64_t a, int64_t b) {
  return static_cast<int64_t>(static_cast<uint64_t>(a) + static_cast<uint64_t>(b));
}

// a unit U is one element (U = T) or one 16-B vector of 16 / sizeof(T) elements (U = uint4)
template <typename T, typename U>
__device__ __forceinline__ U AddU(const U& a, const U& b) {
  if constexpr (sizeof(U) == sizeof(T)) {
    return Add(a, b);
  } else {
    constexpr int kLanes = sizeof(U) / sizeof(T);
    U r;
    const T* x = reinterpret_cast<const T*>(&a);
    const T* y = reinterpret_cast<const T*>(&b);
    T* z = reinterpret_cast<T*>(&r);
#pragma unroll
    for (int l = 0; l < kLanes; ++l) z[l] = Add(x[l], y[l]);
    return r;
  }
}

template <typename U>
__device__ __forceinline__ U Load(const void* p, uint64_t j) {
  return static_cast<const U*>(p)[j];
}

// out unit j = the fold of unit j of every input. Loads of a batch are issued before any add.
template <typename T, typename U>
__device__ __forceinline__ void SumUnit(const AddNList& A, U* out, uint64_t j) {
  U acc;
  if (A.right) {
    U r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k < A.count) r[k] = Load<U>(A.p[k], j);
    }
    if (A.count == 2) acc = AddU<T>(r[0], r[1]);
    else if (A.count == 3) acc = AddU<T>(r[0], AddU<T>(r[1], r[2]));
    else acc = AddU<T>(r[0], AddU<T>(r[1], AddU<T>(r[2], r[3])));
  } else {
    memset(&acc, 0, sizeof(U));  // +0 in every dtype
    for (int b = 0; b < A.count; b += kAddNBatch) {
      U r[kAddNBatch];
#pragma unroll
      for (int k = 0; k < kAddNBatch; ++k) {
        if (b + k < A.count) r[k] = Load<U>(A.p[b + k], j);
      }
#pragma unroll
      for (int k = 0; k < kAddNBatch; ++k) {
        if (b + k < A.count) acc = (b + k == 0 && !A.zero_first) ? r[k] : AddU<T>(acc, r[k]);
      }
    }
  }
  out[j] = acc;
}

// Grid-stride over out's 16-B vectors when every base is aligned, then element by element over the
// rest (all of it for a slice such as a[1:]). Plain loads and stores: out may be in[0] itself, and
// each element is read before it is written by the same thread.
template <typename T>
__global__ void __launch_bounds__(kAddNThreads) add_n_kernel(const AddNList A, T* out, uint64_t n) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kAddNThreads;
  const uint64_t i0 = static_cast<uint64_t>(blockIdx.x) * kAddNThreads + threadIdx.x;
  uint64_t scalar_from = 0;
  if (A.vec) {
    constexpr uint64_t kPerVec = 16 / sizeof(T);
    const uint64_t nvec = n / kPerVec;
    for (uint64_t j = i0; j < nvec; j += stride) SumUnit<T, uint4>(A, reinterpret_cast<uint4*>(out), j);
    scalar_from = nvec * kPerVec;
  }
  for (uint64_t e = scalar_from + i0; e < n; e += stride) SumUnit<T, T>(A, out, e);
}

template <typename T>
void Launch(const AddNList& A, void* out, uint64_t n, cudaStream_t st) {
  const uint64_t units = A.vec ? std::max<uint64_t>(n / (16 / sizeof(T)), 1) : n;
  const uint64_t blocks = std::min<uint64_t>((units + kAddNThreads - 1) / kAddNThreads, kNumSMs * 32);
  add_n_kernel<T><<<static_cast<unsigned>(blocks), kAddNThreads, 0, st>>>(A, static_cast<T*>(out), n);
}

}  // namespace

int LaunchAddN(int dtype, const void* const* in, int n_in, bool zero_first, void* out, uint64_t n,
               cudaStream_t st) {
  KV_CHECK(n_in >= 1);
  if (n == 0) return 0;
  auto aligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  int launches = 0;
  for (int next = 0; next < n_in;) {
    AddNList A;
    A.count = 0;
    if (next > 0) A.p[A.count++] = out;  // the chain so far
    while (A.count < kAddNMaxArrays && next < n_in) A.p[A.count++] = in[next++];
    A.right = launches == 0 && !zero_first && n_in >= 2 && n_in <= 4;
    A.zero_first = launches == 0 && zero_first;
    bool vec = aligned(out);
    for (int i = 0; i < A.count; ++i) vec = vec && aligned(A.p[i]);
    A.vec = vec;
    switch (dtype) {
      case kFloat16: Launch<__half>(A, out, n, st); break;
      case kBfloat16: Launch<__nv_bfloat16>(A, out, n, st); break;
      case kFloat32: Launch<float>(A, out, n, st); break;
      case kFloat64: Launch<double>(A, out, n, st); break;
      case kUint8: Launch<uint8_t>(A, out, n, st); break;
      case kInt8: Launch<int8_t>(A, out, n, st); break;
      case kInt32: Launch<int32_t>(A, out, n, st); break;
      case kInt64: Launch<int64_t>(A, out, n, st); break;
      default: KV_FATAL << "add_n: unsupported dtype " << DTypeName(dtype);
    }
    KV_CUDA(cudaGetLastError());
    ++launches;
  }
  return launches;
}

}  // namespace b200kv
