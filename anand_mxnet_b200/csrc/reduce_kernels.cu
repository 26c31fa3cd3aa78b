// reduce_kernels.cu -- the mean over the trailing axis (the reference's `mean(x, axis=-1)`), one
// result per row.
//
// The reference folds each output serially, k = 0..M-1, with red::sum's Kahan step in the dtype
// (broadcast_reduce-inl.h:161-175, mshadow/base.h:833-842), then divides by DType(M)
// (broadcast_reduce_op.h:630-633). That order is the result, so a row cannot be split: each thread
// owns one row and folds it alone. To keep the global loads coalesced anyway, a CTA of one warp
// owns 32 rows and walks them in tiles of 32 columns. The warp loads a tile with consecutive lanes
// on consecutive addresses of the flattened tile (a tile is contiguous when a row fits in it),
// stores it to shared memory, and each lane then folds its row out of shared memory while the
// warp's loads of the next tile are in flight. Row blocks are taken grid-stride.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "common.h"
#include "kernels.h"

namespace b200kv {
namespace {

constexpr int kRows = 32;  // rows per CTA = threads per CTA (one warp)
constexpr int kTile = 32;  // columns per tile

// the arithmetic type: float for the 16-bit types, which round every step back to the dtype, as
// half_t's operators do (half.h:45-66); bfloat16 is treated the same
template <typename T> struct Calc { typedef T type; };
template <> struct Calc<__half> { typedef float type; };
template <> struct Calc<__nv_bfloat16> { typedef float type; };

__device__ __forceinline__ float Widen(__half x) { return __half2float(x); }
__device__ __forceinline__ float Widen(__nv_bfloat16 x) { return __bfloat162float(x); }
template <typename T> __device__ __forceinline__ T Widen(T x) { return x; }

// the value a step leaves in a DType variable
template <typename T> __device__ __forceinline__ typename Calc<T>::type Round(typename Calc<T>::type x) {
  if constexpr (std::is_same<T, __half>::value) return __half2float(__float2half_rn(x));
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return __bfloat162float(__float2bfloat16_rn(x));
  else return x;
}
template <typename T> __device__ __forceinline__ T Store(typename Calc<T>::type x) {
  if constexpr (std::is_same<T, __half>::value) return __float2half_rn(x);
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return __float2bfloat16_rn(x);
  else return x;
}

__device__ __forceinline__ float Add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double Add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float Sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double Sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float Div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double Div(double a, double b) { return __ddiv_rn(a, b); }

template <typename T>
__global__ void __launch_bounds__(kRows) row_mean_kernel(T* __restrict__ out, const T* __restrict__ in,
                                                          int64_t rows, int64_t cols) {
  typedef typename Calc<T>::type C;
  __shared__ C tile[kRows][kTile + 1];  // +1: lane r reading tile[r][j] hits 32 distinct banks
  const int lane = threadIdx.x;
  // DType(M): the count converted to the dtype (a 16-bit dtype rounds it from float)
  const C count = Round<T>(static_cast<C>(cols));
  for (int64_t r0 = static_cast<int64_t>(blockIdx.x) * kRows; r0 < rows;
       r0 += static_cast<int64_t>(gridDim.x) * kRows) {
    const int nr = static_cast<int>(rows - r0 < kRows ? rows - r0 : kRows);
    const T* base = in + r0 * cols;
    T pre[kTile];
    // the tile at column c0, flattened: element e = lane + 32 k sits at (e / w, e % w)
    auto load = [&](int64_t c0) {
      const int w = static_cast<int>(cols - c0 < kTile ? cols - c0 : kTile);
      const int n = nr * w, q = kRows / w, rm = kRows % w;
      int row = lane / w, col = lane % w;
#pragma unroll
      for (int k = 0; k < kTile; ++k) {
        if (lane + k * kRows < n) pre[k] = base[row * cols + c0 + col];
        row += q;
        col += rm;
        if (col >= w) {
          col -= w;
          ++row;
        }
      }
    };
    auto stage = [&](int64_t c0) {
      const int w = static_cast<int>(cols - c0 < kTile ? cols - c0 : kTile);
      const int n = nr * w, q = kRows / w, rm = kRows % w;
      int row = lane / w, col = lane % w;
#pragma unroll
      for (int k = 0; k < kTile; ++k) {
        if (lane + k * kRows < n) tile[row][col] = Widen(pre[k]);
        row += q;
        col += rm;
        if (col >= w) {
          col -= w;
          ++row;
        }
      }
    };
    C acc = 0, residual = 0;  // red::sum::SetInitValue
    if (cols > 0) load(0);      // no columns: 0 / DType(0)
    for (int64_t c0 = 0; c0 < cols; c0 += kTile) {
      __syncwarp();  // every lane is done reading the previous tile
      stage(c0);
      __syncwarp();
      if (c0 + kTile < cols) load(c0 + kTile);
      const int w = static_cast<int>(cols - c0 < kTile ? cols - c0 : kTile);
      if (lane < nr) {
        for (int j = 0; j < w; ++j) {
          // red::sum::Reduce(dst, src, residual), every operation rounded to the dtype
          const C y = Round<T>(Sub(tile[lane][j], residual));
          const C t = Round<T>(Add(acc, y));
          residual = isinf(t) ? C(0) : Round<T>(Sub(Round<T>(Sub(t, acc)), y));
          acc = t;
        }
      }
    }
    if (lane < nr) out[r0 + lane] = Store<T>(Div(acc, count));
  }
}

template <typename T>
void row_mean_launch(void* out, const void* in, int64_t rows, int64_t cols, cudaStream_t s) {
  const int64_t blocks = (rows + kRows - 1) / kRows;
  // 32 resident CTAs of one warp per SM; beyond that the row blocks are taken grid-stride
  const int grid = static_cast<int>(blocks < kNumSMs * 32 ? blocks : kNumSMs * 32);
  row_mean_kernel<T><<<grid, kRows, 0, s>>>(static_cast<T*>(out), static_cast<const T*>(in), rows, cols);
}

}  // namespace

void LaunchRowMean(int dtype, void* out, const void* in, int64_t rows, int64_t cols, cudaStream_t stream) {
  if (rows == 0) return;
  switch (dtype) {
    case kFloat32: row_mean_launch<float>(out, in, rows, cols, stream); break;
    case kFloat16: row_mean_launch<__half>(out, in, rows, cols, stream); break;
    case kBfloat16: row_mean_launch<__nv_bfloat16>(out, in, rows, cols, stream); break;
    case kFloat64: row_mean_launch<double>(out, in, rows, cols, stream); break;
    default: KV_FATAL << "mean: unsupported dtype " << DTypeName(dtype);
  }
  KV_CUDA(cudaGetLastError());
}

}  // namespace b200kv
