// update_kernel.cuh -- the elementwise kernel of the single-tensor optimizer operators, shared by
// update_kernels.cu (dense gradients: nag_mom_update / mp_nag_mom_update, signsgd_update /
// signum_update, rmsprop_update / rmspropalex_update, ftml_update, ftrl_update) and
// update_rsp_grad_kernels.cu (the same float32 operators with a row_sparse gradient, and the
// standard forms of sgd_update, sgd_mom_update and adam_update).
//
// One elementwise kernel update_kernel<OP, T, RSPG> over one flat tensor: a grid-stride loop whose
// body moves 16 bytes per operand (float4, or 8 x 16 bit) when every operand is 16-byte aligned, and
// a scalar loop for the rest (unaligned slices, the tail). With RSPG the gradient is row_sparse:
// element i of row r = i / row_len reads gval[row_map[r] * row_len + i % row_len], or +0.0f when
// row_map[r] < 0 (the reference densifies such a gradient first, CastStorageRspDnsImpl), so every
// row of the table moves without a dense gradient in memory. Each Step<OP> (opt_math.cuh, shared
// with the row_sparse forms in rowsparse_kernels.cu) follows the expression tree of the reference's
// CPU kernel as written (src/operator/optimizer_op-inl.h), one explicitly rounded IEEE operation per
// node, so the results equal the reference's bit for bit.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "common.h"
#include "kernels.h"
#include "opt_math.cuh"

namespace b200kv {
namespace {

constexpr int kThreads = 256;

template <typename T> __device__ __forceinline__ float ToF(T x);
template <> __device__ __forceinline__ float ToF<float>(float x) { return x; }
template <> __device__ __forceinline__ float ToF<__half>(__half x) { return __half2float(x); }
template <> __device__ __forceinline__ float ToF<__nv_bfloat16>(__nv_bfloat16 x) { return __bfloat162float(x); }

template <typename T> __device__ __forceinline__ T FromF(float x);
template <> __device__ __forceinline__ float FromF<float>(float x) { return x; }
template <> __device__ __forceinline__ __half FromF<__half>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ __nv_bfloat16 FromF<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }

// V consecutive elements of a 16-byte group, as floats
template <typename T, int V>
__device__ __forceinline__ void LoadT(const void* p, size_t v, float (&x)[V]) {
  const uint4 raw = reinterpret_cast<const uint4*>(p)[v];
  const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
  for (int j = 0; j < V; ++j) x[j] = ToF<T>(e[j]);
}
template <typename T, int V>
__device__ __forceinline__ void StoreT(void* p, size_t v, const float (&x)[V]) {
  uint4 raw;
  T* e = reinterpret_cast<T*>(&raw);
#pragma unroll
  for (int j = 0; j < V; ++j) e[j] = FromF<T>(x[j]);
  reinterpret_cast<uint4*>(p)[v] = raw;
}
template <int V>
__device__ __forceinline__ void LoadF(const float* p, size_t v, float (&x)[V]) {
#pragma unroll
  for (int q = 0; q < V / 4; ++q) {
    const float4 f = reinterpret_cast<const float4*>(p)[v * (V / 4) + q];
    x[4 * q] = f.x; x[4 * q + 1] = f.y; x[4 * q + 2] = f.z; x[4 * q + 3] = f.w;
  }
}
template <int V>
__device__ __forceinline__ void StoreF(float* p, size_t v, const float (&x)[V]) {
#pragma unroll
  for (int q = 0; q < V / 4; ++q) {
    reinterpret_cast<float4*>(p)[v * (V / 4) + q] =
        make_float4(x[4 * q], x[4 * q + 1], x[4 * q + 2], x[4 * q + 3]);
  }
}

// the gradient of the V elements of 16-byte group v (RSPG: float32, row_len % V == 0, so one row);
// returns whether that row is stored in the gradient (always, without RSPG)
template <typename T, int V, bool RSPG>
__device__ __forceinline__ bool LoadGrad(const UpdateLaunch& a, size_t v, float (&g)[V]) {
  if (!RSPG) {
    LoadT<T, V>(a.g, v, g);
    return true;
  }
  const size_t i = v * V;
  const size_t r = i / a.row_len;
  const int32_t gi = a.row_map[r];
  if (gi < 0) {
#pragma unroll
    for (int j = 0; j < V; ++j) g[j] = 0.f;
    return false;
  }
  LoadF<V>(static_cast<const float*>(a.g) + static_cast<size_t>(gi) * a.row_len + (i - r * a.row_len), 0, g);
  return true;
}
template <typename T, bool RSPG>
__device__ __forceinline__ float GradAt(const UpdateLaunch& a, size_t i, bool& present) {
  present = true;
  if (!RSPG) return ToF<T>(static_cast<const T*>(a.g)[i]);
  const size_t r = i / a.row_len;
  const int32_t gi = a.row_map[r];
  present = gi >= 0;
  return gi < 0 ? 0.f : static_cast<const float*>(a.g)[static_cast<size_t>(gi) * a.row_len + (i - r * a.row_len)];
}

template <int OP, typename T, bool RSPG>
__global__ void __launch_bounds__(kThreads) update_kernel(const UpdateLaunch a, const bool vec) {
  constexpr int V = 16 / sizeof(T);
  constexpr int NS = NumStates(OP);
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t nv = vec ? a.n / V : 0;
  for (size_t v = tid; v < nv; v += stride) {
    float w[V], g[V], st[3][V], o[V];
    if (ReadsWeight(OP)) LoadT<T, V>(a.w, v, w);
    const bool present = LoadGrad<T, V, RSPG>(a, v, g);
#pragma unroll
    for (int k = 0; k < NS; ++k) LoadF<V>(a.s[k], v, st[k]);
#pragma unroll
    for (int j = 0; j < V; ++j) {
      float s[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < NS; ++k) s[k] = st[k][j];
      o[j] = Step<OP>(a, ReadsWeight(OP) ? w[j] : 0.f, g[j], s, present);
#pragma unroll
      for (int k = 0; k < NS; ++k) st[k][j] = s[k];
    }
    StoreT<T, V>(a.out, v, o);
#pragma unroll
    for (int k = 0; k < NS; ++k) StoreF<V>(a.s[k], v, st[k]);
  }
  const T* w = static_cast<const T*>(a.w);
  T* out = static_cast<T*>(a.out);
  for (size_t i = nv * V + tid; i < a.n; i += stride) {
    float s[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < NS; ++k) s[k] = a.s[k][i];
    bool present;
    const float g = GradAt<T, RSPG>(a, i, present);
    const float r = Step<OP>(a, ReadsWeight(OP) ? ToF<T>(w[i]) : 0.f, g, s, present);
    out[i] = FromF<T>(r);
#pragma unroll
    for (int k = 0; k < NS; ++k) a.s[k][i] = s[k];
  }
}

bool Aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <int OP, typename T, bool RSPG = false>
void Launch(const UpdateLaunch& L, cudaStream_t stream) {
  constexpr int V = 16 / sizeof(T);
  bool vec = Aligned16(L.g) && Aligned16(L.out) && (!ReadsWeight(OP) || Aligned16(L.w));
  for (int k = 0; k < NumStates(OP); ++k) vec = vec && Aligned16(L.s[k]);
  if (RSPG) vec = vec && L.row_len % V == 0;  // a 16-byte group never straddles two rows
  const size_t items = vec ? (L.n / V + L.n % V) : L.n;
  const size_t want = (items + kThreads - 1) / kThreads;
  // RSPG: one thread per item, as the table-wide pass runs 30-56-register CTAs of which a capped
  // grid would leave part of its last wave empty
  const int grid = static_cast<int>(std::max<size_t>(1, RSPG ? want : std::min<size_t>(want, kNumSMs * 8)));
  update_kernel<OP, T, RSPG><<<grid, kThreads, 0, stream>>>(L, vec);
  KV_CUDA(cudaGetLastError());
}

}  // namespace
}  // namespace b200kv
