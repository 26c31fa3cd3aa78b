// multi_tensor_kernels.cu -- the multi-tensor optimizer operators next to the KVStore path
// (SURVEY 8f-f1): multi_sum_sq, multi_lars, _[mp_]adamw_update, _multi_[mp_]adamw_update,
// [mp_]lamb_update_phase1/2, _multi_[mp_]lamb_update, the AMP overflow check
// [multi_]all_finite (its own kernel and launch list, below), and gradient clipping by global
// norm / the bulk unscale (_b200kv_clip_global_norm, _b200kv_multi_scale: three kernels, below),
// and reset_arrays (ParameterDict.zero_grad: one byte-wise kernel for every dtype, below).
//
// One launch covers every tensor of the call: a device table of MTTensor descriptors + a list of
// <= 8192-element chunks (one 256-thread CTA each, 16-byte accesses, streaming loads/stores), the
// per-tensor scalars (lr / wd / eta / bias-correction terms) travelling by value in the kernel
// parameters. All of it is HBM-bound elementwise work; the only reductions are sums of squares,
// done deterministically: per-thread sequential partial -> fixed shuffle tree -> one partial per
// chunk -> a second kernel folds a tensor's partials in a fixed tree (same result every run, which
// the reference's test asserts: tests/python/gpu/test_operator_gpu.py:279).
//
// Arithmetic is IEEE fp32 with explicit round-to-nearest intrinsics (no FMA contraction) in the
// reference's CPU expression trees -- each functor cites the file:line it follows -- so every
// elementwise result is bit-identical to the reference / oracle/kvoracle.c. Sums of squares differ
// from the reference CPU's sequential loop in association only (tolerance 1e-5 relative, the
// reference's own bound).
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "common.h"
#include "kernels.h"

namespace b200kv {
namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float clipf(float x, float b) { return x > b ? b : (x < -b ? -b : x); }
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float dvd(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float sqr(float a) { return __fsqrt_rn(a); }

template <typename T> struct Cv;
template <> struct Cv<float> {
  static __device__ __forceinline__ float to_f(float v) { return v; }
  static __device__ __forceinline__ float from_f(float v) { return v; }
};
template <> struct Cv<__half> {
  static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};
template <> struct Cv<__nv_bfloat16> {
  static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};

// 4 consecutive elements
template <typename T> struct L4 {
  static __device__ __forceinline__ void ld(const T* p, float (&x)[4]) {
    const uint2 raw = __ldcs(reinterpret_cast<const uint2*>(p));
    const T* h = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i) x[i] = Cv<T>::to_f(h[i]);
  }
  static __device__ __forceinline__ void st(T* p, const float (&x)[4]) {
    uint2 raw;
    T* h = reinterpret_cast<T*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = Cv<T>::from_f(x[i]);
    __stcs(reinterpret_cast<uint2*>(p), raw);
  }
};
template <> struct L4<float> {
  static __device__ __forceinline__ void ld(const float* p, float (&x)[4]) {
    const float4 t = __ldcs(reinterpret_cast<const float4*>(p));
    x[0] = t.x; x[1] = t.y; x[2] = t.z; x[3] = t.w;
  }
  static __device__ __forceinline__ void st(float* p, const float (&x)[4]) {
    __stcs(reinterpret_cast<float4*>(p), make_float4(x[0], x[1], x[2], x[3]));
  }
};
template <typename T> struct L1 {
  static __device__ __forceinline__ void ld(const T* p, float (&x)[1]) { x[0] = Cv<T>::to_f(*p); }
  static __device__ __forceinline__ void st(T* p, const float (&x)[1]) { *p = Cv<T>::from_f(x[0]); }
};
template <typename T, int V> struct LS;
template <typename T> struct LS<T, 4> : L4<T> {};
template <typename T> struct LS<T, 1> : L1<T> {};

// deterministic block sum: fixed shuffle tree, then the warp leaders in index order
__device__ __forceinline__ float block_sum(float v) {
  __shared__ float s_part[kThreads / 32];
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = __fadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
  __syncthreads();  // s_part may still be read by the previous call
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < kThreads / 32; ++i) r = __fadd_rn(r, s_part[i]);
  }
  return r;  // valid in thread 0
}

// ---------------------------------------------------------------------------------------------
// functors: V elements of tensor t starting at element `base`; s = launch scalars; k = tensor
// index inside the launch (per-tensor scalars s.t[k])

// multi_sum_sq (src/operator/contrib/multi_sum_sq.cc:64-78; GPU form multi_sum_sq.cu:92-118:
// widen to float, square, accumulate in float)
template <typename T> struct SumSqOp {
  static constexpr bool kReduce = true;
  template <int V>
  static __device__ __forceinline__ void run(const MTTensor& t, const MTScalars&, int, uint32_t base,
                                             float& acc0, float&) {
    float x[V];
    LS<T, V>::ld(static_cast<const T*>(t.p[0]) + base, x);
#pragma unroll
    for (int i = 0; i < V; ++i) acc0 = add(acc0, mul(x[i], x[i]));
  }
};

// _adamw_update (adamw-inl.h:176-208, mshadow expression form; the reference writes the rescaled /
// clipped gradient back into `grad`), _mp_adamw_update (adamw-inl.h:108-131) and the multi-tensor
// forms (adamw-inl.h:340-372: mean = beta1*(mean - g) + g). s.t[k] = (lr, wd, eta, -).
// s.f: 0 clip, 1 beta1, 2 beta2, 3 eps. s.d0 = rescale_grad (device scalar): a zero / inf / nan
// value skips the update (adamw-inl.h:449-461).
template <typename T, bool MP, bool MULTI> struct AdamWOp {
  static constexpr bool kReduce = false;
  template <int V>
  static __device__ __forceinline__ void run(const MTTensor& t, const MTScalars& s, int k,
                                             uint32_t base, float&, float&) {
    const float rescale = *s.d0;
    if (!isfinite(rescale) || rescale == 0.f) return;
    const float lr = s.t[k].x, wd = s.t[k].y, eta = s.t[k].z;
    const float clip = s.f[0], beta1 = s.f[1], beta2 = s.f[2], eps = s.f[3];
    float w[V], g[V], m[V], v[V];
    if (MP) LS<float, V>::ld(static_cast<const float*>(t.p[4]) + base, w);
    else LS<T, V>::ld(static_cast<const T*>(t.p[0]) + base, w);
    LS<T, V>::ld(static_cast<const T*>(t.p[1]) + base, g);
    LS<float, V>::ld(static_cast<const float*>(t.p[2]) + base, m);
    LS<float, V>::ld(static_cast<const float*>(t.p[3]) + base, v);
#pragma unroll
    for (int i = 0; i < V; ++i) {
      float sg = mul(rescale, g[i]);
      if (clip >= 0.f) sg = clipf(sg, clip);
      g[i] = sg;
      if (MULTI) {
        m[i] = add(mul(beta1, sub(m[i], sg)), sg);
        const float adj = mul(sg, sg);
        v[i] = add(mul(beta2, sub(v[i], adj)), adj);
      } else {
        m[i] = add(mul(beta1, m[i]), mul(sub(1.f, beta1), sg));
        v[i] = add(mul(beta2, v[i]), mul(sub(1.f, beta2), mul(sg, sg)));
      }
      w[i] = sub(w[i], mul(eta, add(dvd(mul(lr, m[i]), add(sqr(v[i]), eps)), mul(wd, w[i]))));
    }
    LS<float, V>::st(static_cast<float*>(t.p[2]) + base, m);
    LS<float, V>::st(static_cast<float*>(t.p[3]) + base, v);
    if (MP) LS<float, V>::st(static_cast<float*>(t.p[4]) + base, w);
    LS<T, V>::st(static_cast<T*>(t.p[5]) + base, w);
    if (!MP && !MULTI) LS<T, V>::st(static_cast<T*>(t.p[1]) + base, g);  // the reference's side effect
  }
};

// lamb_update_phase1 / mp_lamb_update_phase1 (optimizer_op-inl.h:1621-1648, 1772-1801).
// s.f: 0 clip, 1 rescale, 2 beta1, 3 beta1_t, 4 beta2, 5 beta2_t, 6 wd, 7 eps, 8 bias_correction.
// With a 16-bit gradient the reference's `grad * rescale` is a half_t product (rounded to half).
template <typename T, bool MP> struct LambPhase1Op {
  static constexpr bool kReduce = false;
  template <int V>
  static __device__ __forceinline__ void run(const MTTensor& t, const MTScalars& s, int,
                                             uint32_t base, float&, float&) {
    const float clip = s.f[0], rescale = s.f[1], beta1 = s.f[2], beta1_t = s.f[3], beta2 = s.f[4],
                beta2_t = s.f[5], wd = s.f[6], eps = s.f[7];
    const bool bias = s.f[8] != 0.f;
    float w[V], g[V], m[V], v[V], out[V];
    if (MP) LS<float, V>::ld(static_cast<const float*>(t.p[4]) + base, w);
    else LS<T, V>::ld(static_cast<const T*>(t.p[0]) + base, w);
    LS<T, V>::ld(static_cast<const T*>(t.p[1]) + base, g);
    LS<float, V>::ld(static_cast<const float*>(t.p[2]) + base, m);
    LS<float, V>::ld(static_cast<const float*>(t.p[3]) + base, v);
#pragma unroll
    for (int i = 0; i < V; ++i) {
      float gr = mul(g[i], rescale);
      if (sizeof(T) == 2) gr = Cv<T>::to_f(Cv<T>::from_f(gr));
      if (clip >= 0.f) gr = clipf(gr, clip);
      m[i] = add(mul(beta1, m[i]), mul(sub(1.f, beta1), gr));
      v[i] = add(mul(beta2, v[i]), mul(mul(sub(1.f, beta2), gr), gr));
      float r = add(dvd(m[i], add(sqr(v[i]), eps)), mul(wd, w[i]));
      if (bias) {
        // mean_hat divides in DOUBLE (`1. - beta1_t`), var_hat in float (`1 - beta2_t`)
        const float mean_hat = static_cast<float>(
            __ddiv_rn(static_cast<double>(m[i]), __dsub_rn(1.0, static_cast<double>(beta1_t))));
        const float var_hat = dvd(v[i], sub(1.f, beta2_t));
        r = add(dvd(mean_hat, add(sqr(var_hat), eps)), mul(wd, w[i]));
      }
      out[i] = r;
    }
    LS<float, V>::st(static_cast<float*>(t.p[2]) + base, m);
    LS<float, V>::st(static_cast<float*>(t.p[3]) + base, v);
    LS<float, V>::st(static_cast<float*>(t.p[5]) + base, out);
  }
};

// lamb_update_phase2 / mp_lamb_update_phase2 (optimizer_op-inl.h:1705-1729, 1862-1886).
// s.f: 0 lr, 1 lower_bound, 2 upper_bound; s.d0 / s.d1 = r1 / r2 (device scalars).
// The mp form writes ONLY the 16-bit output from weight32 - lr*g; weight32 stays as it was.
template <typename T, bool MP> struct LambPhase2Op {
  static constexpr bool kReduce = false;
  template <int V>
  static __device__ __forceinline__ void run(const MTTensor& t, const MTScalars& s, int,
                                             uint32_t base, float&, float&) {
    float lr = s.f[0];
    const float lb = s.f[1], ub = s.f[2];
    float r1 = *s.d0;
    const float r2 = *s.d1;
    if (lb >= 0) r1 = fmaxf(r1, lb);
    if (ub >= 0) r1 = fminf(r1, ub);
    if (!(r1 == 0.0f || r2 == 0.0f)) lr = dvd(mul(lr, r1), r2);
    float w[V], g[V];
    if (MP) LS<float, V>::ld(static_cast<const float*>(t.p[4]) + base, w);
    else LS<T, V>::ld(static_cast<const T*>(t.p[0]) + base, w);
    LS<float, V>::ld(static_cast<const float*>(t.p[1]) + base, g);
#pragma unroll
    for (int i = 0; i < V; ++i) w[i] = sub(w[i], mul(lr, g[i]));
    LS<T, V>::st(static_cast<T*>(t.p[5]) + base, w);
  }
};

// _multi_[mp_]lamb_update step 1 (multi_lamb.cc:33-77) fused with BOTH sums of squares the
// reference computes in separate passes (multi_lamb-inl.h:325-331): sum w^2 of the weight INPUT
// (the 16-bit weights in the mp form) and sum temp_g^2. s.t[k] = (lr, wd, 1-beta1^t, 1-beta2^t)
// (the powf terms are evaluated on the host with the C library, as the reference CPU does).
// s.f: 0 clip, 1 rescale, 2 beta1, 3 beta2, 4 eps, 5 bias_correction.
template <typename T, bool MP> struct MultiLambStep1Op {
  static constexpr bool kReduce = true;
  template <int V>
  static __device__ __forceinline__ void run(const MTTensor& t, const MTScalars& s, int k,
                                             uint32_t base, float& acc_w, float& acc_g) {
    const float wd = s.t[k].y, c1 = s.t[k].z, c2 = s.t[k].w;
    const float clip = s.f[0], rescale = s.f[1], beta1 = s.f[2], beta2 = s.f[3], eps = s.f[4];
    const bool bias = s.f[5] != 0.f;
    float wi[V], w[V], g[V], m[V], v[V], out[V];
    LS<T, V>::ld(static_cast<const T*>(t.p[0]) + base, wi);
    if (MP) {
      LS<float, V>::ld(static_cast<const float*>(t.p[4]) + base, w);
    } else {
#pragma unroll
      for (int i = 0; i < V; ++i) w[i] = wi[i];
    }
    LS<T, V>::ld(static_cast<const T*>(t.p[1]) + base, g);
    LS<float, V>::ld(static_cast<const float*>(t.p[2]) + base, m);
    LS<float, V>::ld(static_cast<const float*>(t.p[3]) + base, v);
#pragma unroll
    for (int i = 0; i < V; ++i) {
      float sg = mul(g[i], rescale);
      if (clip >= 0.f) sg = clipf(sg, clip);
      m[i] = add(mul(beta1, m[i]), mul(sub(1.f, beta1), sg));
      v[i] = add(mul(beta2, v[i]), mul(mul(sub(1.f, beta2), sg), sg));
      float r;
      if (bias) {
        r = add(dvd(dvd(m[i], c1), add(sqr(dvd(v[i], c2)), eps)), mul(wd, w[i]));
      } else {
        r = add(dvd(m[i], add(sqr(v[i]), eps)), mul(wd, w[i]));
      }
      out[i] = r;
      acc_w = add(acc_w, mul(wi[i], wi[i]));
      acc_g = add(acc_g, mul(r, r));
    }
    LS<float, V>::st(static_cast<float*>(t.p[2]) + base, m);
    LS<float, V>::st(static_cast<float*>(t.p[3]) + base, v);
    LS<float, V>::st(static_cast<float*>(t.p[5]) + base, out);
  }
};

// step 2 (multi_lamb.cc:79-118). s.t[k].x = lr; s.f: 0 lower_bound, 1 upper_bound;
// s.d0 / s.d1 = per-tensor sums of squares (weights / temp_g), indexed by t.aux.
template <typename T, bool MP> struct MultiLambStep2Op {
  static constexpr bool kReduce = false;
  template <int V>
  static __device__ __forceinline__ void run(const MTTensor& t, const MTScalars& s, int k,
                                             uint32_t base, float&, float&) {
    const float lb = s.f[0], ub = s.f[1];
    float r1 = sqr(s.d0[t.aux]);
    const float r2 = sqr(s.d1[t.aux]);
    if (lb >= 0) r1 = fmaxf(r1, lb);
    if (ub >= 0) r1 = fminf(r1, ub);
    const float r = (r1 == 0.0f || r2 == 0.0f) ? 1.0f : dvd(r1, r2);
    const float lr_adjusted = mul(s.t[k].x, r);
    float w[V], g[V];
    if (MP) LS<float, V>::ld(static_cast<const float*>(t.p[4]) + base, w);
    else LS<T, V>::ld(static_cast<const T*>(t.p[0]) + base, w);
    LS<float, V>::ld(static_cast<const float*>(t.p[5]) + base, g);
#pragma unroll
    for (int i = 0; i < V; ++i) w[i] = sub(w[i], mul(lr_adjusted, g[i]));
    if (MP) LS<float, V>::st(static_cast<float*>(t.p[4]) + base, w);
    LS<T, V>::st(static_cast<T*>(t.p[0]) + base, w);
  }
};

template <class Op>
__global__ void __launch_bounds__(kThreads) mt_kernel(const MTTensor* tensors, const MTChunk* chunks,
                                                      const MTScalars s, float* part0, float* part1) {
  const MTChunk c = chunks[blockIdx.x];
  const MTTensor t = tensors[c.tensor];
  float a0 = 0.f, a1 = 0.f;
  const uint32_t nvec = t.vec_ok ? c.len / 4 : 0;
  for (uint32_t v = threadIdx.x; v < nvec; v += kThreads) {
    Op::template run<4>(t, s, static_cast<int>(c.tensor), c.off + v * 4, a0, a1);
  }
  for (uint32_t e = nvec * 4 + threadIdx.x; e < c.len; e += kThreads) {
    Op::template run<1>(t, s, static_cast<int>(c.tensor), c.off + e, a0, a1);
  }
  if (Op::kReduce) {
    const float r0 = block_sum(a0);
    if (threadIdx.x == 0) part0[blockIdx.x] = r0;
    if (part1 != nullptr) {
      const float r1 = block_sum(a1);
      if (threadIdx.x == 0) part1[blockIdx.x] = r1;
    }
  }
}

// out[t.aux] = sum of the tensor's chunk partials, fixed order: one CTA per tensor
__global__ void __launch_bounds__(kThreads) mt_finalize_kernel(const MTTensor* tensors,
                                                               const float* part0, const float* part1,
                                                               float* out0, float* out1) {
  const MTTensor t = tensors[blockIdx.x];
  const uint32_t n = static_cast<uint32_t>((static_cast<uint64_t>(t.size) + kMTChunk - 1) / kMTChunk);
  float a0 = 0.f, a1 = 0.f;
  for (uint32_t i = threadIdx.x; i < n; i += kThreads) {
    a0 = __fadd_rn(a0, part0[t.first_chunk + i]);
    if (part1) a1 = __fadd_rn(a1, part1[t.first_chunk + i]);
  }
  const float r0 = block_sum(a0);
  if (threadIdx.x == 0) out0[t.aux] = r0;
  if (part1) {
    const float r1 = block_sum(a1);
    if (threadIdx.x == 0) out1[t.aux] = r1;
  }
}

// multi_lars (multi_lars-inl.h:61-74)
__global__ void lars_kernel(int n, float* out, const float* lrs, const float* wsq, const float* gsq,
                            const float* wds, float eta, float eps, float rescale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float w_norm = sqr(wsq[i]);
  const bool valid = w_norm > 0.f && gsq[i] > 0.f;
  out[i] = valid ? dvd(mul(mul(lrs[i], eta), w_norm),
                       add(add(mul(sqr(gsq[i]), rescale), mul(wds[i], w_norm)), eps))
                 : lrs[i];
}

// ---------------------------------------------------------------------------------------------
// all_finite / multi_all_finite (contrib/all_finite.cc:32-40, 64-77): non-finite means
// !std::isfinite(static_cast<float>(x)). The 16- and 32-bit types test their raw bits (exponent all
// ones), which is exactly that; float64 is cast first, as the reference does, so a finite double
// that rounds to +-inf in float counts as non-finite.
constexpr int kAFThreads = 256;
constexpr int kAFLoads = kAFTileBytes / 16 / kAFThreads;  // independent 16-B loads per thread
static_assert(kAFLoads * 16 * kAFThreads == kAFTileBytes, "a tile is whole loads of every thread");

template <typename T> struct AfBits;
template <uint32_t kMask2> struct AfBits16 {  // two 16-bit values per word, exponent mask kMask2
  typedef uint16_t Raw;
  static __device__ __forceinline__ bool bad(uint4 r) {
    const uint32_t m = kMask2;
    return (__vcmpeq2(r.x & m, m) | __vcmpeq2(r.y & m, m) | __vcmpeq2(r.z & m, m) |
            __vcmpeq2(r.w & m, m)) != 0u;
  }
  static __device__ __forceinline__ bool bad(uint16_t h) {
    return (h & (kMask2 & 0xFFFFu)) == (kMask2 & 0xFFFFu);
  }
};
template <> struct AfBits<__half> : AfBits16<0x7C007C00u> {};
template <> struct AfBits<__nv_bfloat16> : AfBits16<0x7F807F80u> {};
template <> struct AfBits<float> {
  typedef uint32_t Raw;
  static __device__ __forceinline__ bool bad(uint32_t w) { return (w & 0x7F800000u) == 0x7F800000u; }
  static __device__ __forceinline__ bool bad(uint4 r) { return bad(r.x) | bad(r.y) | bad(r.z) | bad(r.w); }
};
template <> struct AfBits<double> {
  typedef unsigned long long Raw;
  static __device__ __forceinline__ bool bad(unsigned long long b) {
    return !isfinite(__double2float_rn(__longlong_as_double(static_cast<long long>(b))));
  }
  static __device__ __forceinline__ bool bad(uint4 r) {
    return bad((static_cast<unsigned long long>(r.y) << 32) | r.x) |
           bad((static_cast<unsigned long long>(r.w) << 32) | r.z);
  }
};

// The tiled launches below (all_finite, clip_norm_*, reset_arrays) give one CTA per tile of a list
// of arrays; CTA b works on the last array whose first tile is <= b. Arrays without tiles share
// their first tile with the next array and are never found.
__device__ __forceinline__ int tile_owner(const uint32_t* first_tile, int count, uint32_t b) {
  int lo = 0, hi = count - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first_tile[mid] <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// One CTA per tile; the CTA finds its array by a binary search over the first-tile prefix. A
// 16-byte aligned array is read with kAFLoads independent 16-B loads per thread before any test
// (plus a scalar tail in its last tile); any other base is read element by element. Default-cached
// loads: in a training step the update reads the same gradients right after the check.
template <typename T>
__global__ void __launch_bounds__(kAFThreads) all_finite_kernel(const AllFiniteArrays A, float* out) {
  typedef typename AfBits<T>::Raw Raw;
  constexpr uint32_t kTileElems = kAFTileBytes / sizeof(T);
  constexpr uint32_t kPerVec = 16 / sizeof(T);
  const uint32_t b = blockIdx.x;
  if (b >= A.first_tile[A.count]) return;  // the whole CTA: the launch of an all-empty list
  const int lo = tile_owner(A.first_tile, A.count, b);
  const uint64_t e0 = static_cast<uint64_t>(b - A.first_tile[lo]) * kTileElems;
  const uint32_t len = static_cast<uint32_t>(min(static_cast<uint64_t>(kTileElems), A.n[lo] - e0));
  const Raw* p = static_cast<const Raw*>(A.p[lo]) + e0;
  bool bad = false;
  uint32_t scalar_from = 0;
  if ((reinterpret_cast<uintptr_t>(A.p[lo]) & 15) == 0) {
    const uint32_t nvec = len / kPerVec;
    const uint4* v = reinterpret_cast<const uint4*>(p);
    uint4 r[kAFLoads];
#pragma unroll
    for (int i = 0; i < kAFLoads; ++i) {
      const uint32_t j = threadIdx.x + i * kAFThreads;
      r[i] = j < nvec ? v[j] : make_uint4(0u, 0u, 0u, 0u);  // zero bits are finite in every dtype
    }
#pragma unroll
    for (int i = 0; i < kAFLoads; ++i) bad |= AfBits<T>::bad(r[i]);
    scalar_from = nvec * kPerVec;
  }
  for (uint32_t e = scalar_from + threadIdx.x; e < len; e += kAFThreads) bad |= AfBits<T>::bad(p[e]);
  if (__syncthreads_or(bad) && threadIdx.x == 0) *out = 0.0f;
}

// ---------------------------------------------------------------------------------------------
// _b200kv_clip_global_norm (python/mxnet/gluon/utils.py:118-157) and _b200kv_multi_scale (the bulk
// form of amp.unscale, contrib/amp/amp.py:331-346), float32. The array list travels by value and
// the work is tiled by bytes exactly as for all_finite_kernel: one CTA per kCNTileBytes tile, found
// by binary search over the first-tile prefix; a 16-byte aligned array moves kCNLoads independent
// 16-B vectors per thread before any arithmetic, any other base (a[1:]) and the tail go element
// by element. All loads and stores are default-cached: the scaling pass and then the optimizer
// read the same gradients next (a streaming hint on the stores has not been measured).
constexpr int kCNThreads = kThreads;  // block_sum's width
constexpr int kCNLoads = kCNTileBytes / 16 / kCNThreads;
constexpr uint32_t kCNTileElems = kCNTileBytes / sizeof(float);
static_assert(kCNLoads * 16 * kCNThreads == kCNTileBytes, "a tile is whole loads of every thread");

// part[blockIdx.x] = the tile's sum of x*x: per-thread sequential partial in element order, then
// block_sum's fixed tree. Padding lanes add +0.0f, which leaves a sum of squares bitwise unchanged.
__global__ void __launch_bounds__(kCNThreads) clip_norm_partial_kernel(const ClipNormArrays A, float* part) {
  const uint32_t b = blockIdx.x;
  const int k = tile_owner(A.first_tile, A.count, b);
  const uint32_t e0 = (b - A.first_tile[k]) * kCNTileElems;
  const uint32_t len = min(kCNTileElems, A.n[k] - e0);
  const float* p = A.p[k] + e0;
  float acc = 0.f;
  uint32_t scalar_from = 0;
  if ((reinterpret_cast<uintptr_t>(A.p[k]) & 15) == 0) {
    const uint32_t nvec = len / 4;
    const float4* v = reinterpret_cast<const float4*>(p);
    float4 r[kCNLoads];
#pragma unroll
    for (int i = 0; i < kCNLoads; ++i) {
      const uint32_t j = threadIdx.x + i * kCNThreads;
      r[i] = j < nvec ? v[j] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < kCNLoads; ++i) {
      acc = add(acc, mul(r[i].x, r[i].x));
      acc = add(acc, mul(r[i].y, r[i].y));
      acc = add(acc, mul(r[i].z, r[i].z));
      acc = add(acc, mul(r[i].w, r[i].w));
    }
    scalar_from = nvec * 4;
  }
  for (uint32_t e = scalar_from + threadIdx.x; e < len; e += kCNThreads) acc = add(acc, mul(p[e], p[e]));
  const float r = block_sum(acc);
  if (threadIdx.x == 0) part[b] = r;
}

// One CTA: thread t folds part[t], part[t + 256], ... in that order, then block_sum. The norm, and
// the factor of utils.py:150-151 in float32 as the reference's scalar operators compute it:
// _plus_scalar(1e-8), _rdiv_scalar(max_norm), min(concat(scale, 1)). A norm that is inf or nan
// gives the factor 1, so the scaling pass leaves the arrays as they are.
__global__ void __launch_bounds__(kCNThreads) clip_norm_fold_kernel(const float* part, uint32_t n_part,
                                                                    float max_norm, float* total_norm,
                                                                    float* scale) {
  float acc = 0.f;
  constexpr int kBatch = 8;  // loads in flight per thread; past the end they are +0.0f
  for (uint32_t i0 = threadIdx.x; i0 < n_part; i0 += kBatch * kCNThreads) {
    float v[kBatch];
#pragma unroll
    for (int j = 0; j < kBatch; ++j) {
      const uint32_t i = i0 + j * kCNThreads;
      v[j] = i < n_part ? part[i] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < kBatch; ++j) acc = add(acc, v[j]);
  }
  const float ss = block_sum(acc);
  if (threadIdx.x == 0) {
    const float norm = sqr(ss);
    float s = dvd(max_norm, add(norm, 1e-8f));
    s = s < 1.f ? s : 1.f;
    *total_norm = norm;
    *scale = isfinite(norm) ? s : 1.f;
  }
}

// x = x * s in place. s == 1 is the identity on every finite value (and the factor the fold gives
// for a non-finite norm), so the CTA returns before it reads anything.
__global__ void __launch_bounds__(kCNThreads) clip_norm_scale_kernel(const ClipNormArrays A,
                                                                     const float* scale_dev, float scale) {
  const float s = scale_dev != nullptr ? *scale_dev : scale;
  if (s == 1.f) return;
  const uint32_t b = blockIdx.x;
  const int k = tile_owner(A.first_tile, A.count, b);
  const uint32_t e0 = (b - A.first_tile[k]) * kCNTileElems;
  const uint32_t len = min(kCNTileElems, A.n[k] - e0);
  float* p = A.p[k] + e0;
  uint32_t scalar_from = 0;
  if ((reinterpret_cast<uintptr_t>(A.p[k]) & 15) == 0) {
    const uint32_t nvec = len / 4;
    float4* v = reinterpret_cast<float4*>(p);
    float4 r[kCNLoads];
#pragma unroll
    for (int i = 0; i < kCNLoads; ++i) {
      const uint32_t j = threadIdx.x + i * kCNThreads;
      if (j < nvec) r[i] = v[j];
    }
#pragma unroll
    for (int i = 0; i < kCNLoads; ++i) {
      const uint32_t j = threadIdx.x + i * kCNThreads;
      if (j < nvec) v[j] = make_float4(mul(r[i].x, s), mul(r[i].y, s), mul(r[i].z, s), mul(r[i].w, s));
    }
    scalar_from = nvec * 4;
  }
  for (uint32_t e = scalar_from + threadIdx.x; e < len; e += kCNThreads) p[e] = mul(p[e], s);
}

// ---------------------------------------------------------------------------------------------
// reset_arrays (contrib/reset_arrays.cc; the reference runs one cudaMemsetAsync per array): zero
// bytes whatever the dtype. One CTA per kRATileBytes tile of an array, counted from its base, found
// as for all_finite_kernel. The 16-byte aligned body of a tile is written with kRAStores 16-B
// stores per thread; the unaligned head and tail around it (< 16 bytes each, only when the base is
// not 16-byte aligned, as for a[1:]) byte by byte. No byte outside [p, p + bytes) is written.
// Default-cached stores: the next writer of a gradient is backward's accumulation (a streaming
// hint has not been measured).
constexpr int kRAThreads = 256;
constexpr int kRAStores = kRATileBytes / 16 / kRAThreads;
static_assert(kRAStores * 16 * kRAThreads == kRATileBytes, "a tile is whole stores of every thread");

__global__ void __launch_bounds__(kRAThreads) reset_arrays_kernel(const ResetArraysList A) {
  const uint32_t b = blockIdx.x;
  const int k = tile_owner(A.first_tile, A.count, b);
  const uint64_t off = static_cast<uint64_t>(b - A.first_tile[k]) * kRATileBytes;
  const uint64_t len = min(static_cast<uint64_t>(kRATileBytes), A.bytes[k] - off);
  unsigned char* lo = static_cast<unsigned char*>(A.p[k]) + off;
  unsigned char* hi = lo + len;
  uint4* v0 = reinterpret_cast<uint4*>((reinterpret_cast<uintptr_t>(lo) + 15) & ~static_cast<uintptr_t>(15));
  uint4* v1 = reinterpret_cast<uint4*>(reinterpret_cast<uintptr_t>(hi) & ~static_cast<uintptr_t>(15));
  if (reinterpret_cast<unsigned char*>(v0) >= reinterpret_cast<unsigned char*>(v1)) {
    // no whole aligned 16 bytes in the tile (< 32 bytes): every byte alone
    for (uint32_t e = threadIdx.x; e < len; e += kRAThreads) lo[e] = 0;
    return;
  }
  const uint32_t nvec = static_cast<uint32_t>(v1 - v0);  // <= kRAStores * kRAThreads
#pragma unroll
  for (int i = 0; i < kRAStores; ++i) {
    const uint32_t j = threadIdx.x + i * kRAThreads;
    if (j < nvec) v0[j] = make_uint4(0u, 0u, 0u, 0u);
  }
  const uint32_t head = static_cast<uint32_t>(reinterpret_cast<unsigned char*>(v0) - lo);  // < 16
  const uint32_t tail = static_cast<uint32_t>(hi - reinterpret_cast<unsigned char*>(v1));  // < 16
  if (threadIdx.x < head) lo[threadIdx.x] = 0;
  if (threadIdx.x >= 32 && threadIdx.x - 32 < tail) reinterpret_cast<unsigned char*>(v1)[threadIdx.x - 32] = 0;
}

template <class Op>
void launch(const MTLaunch& L, cudaStream_t st) {
  mt_kernel<Op><<<L.n_chunks, kThreads, 0, st>>>(L.tensors, L.chunks, L.s, L.part0, L.part1);
}

template <template <typename, bool> class Op>
void launch_tm(const MTLaunch& L, cudaStream_t st) {
  if (L.dtype == kFloat32) { KV_CHECK(!L.mp); return launch<Op<float, false>>(L, st); }
  KV_CHECK(L.mp) << "16-bit weights need the multi-precision (fp32 master copy) form of this operator";
  if (L.dtype == kFloat16) return launch<Op<__half, true>>(L, st);
  if (L.dtype == kBfloat16) return launch<Op<__nv_bfloat16, true>>(L, st);
  KV_FATAL << "unsupported dtype " << DTypeName(L.dtype);
}

template <bool MULTI>
void launch_adamw(const MTLaunch& L, cudaStream_t st) {
  if (L.dtype == kFloat32) { KV_CHECK(!L.mp); return launch<AdamWOp<float, false, MULTI>>(L, st); }
  KV_CHECK(L.mp) << "16-bit weights need the multi-precision (fp32 master copy) form of this operator";
  if (L.dtype == kFloat16) return launch<AdamWOp<__half, true, MULTI>>(L, st);
  if (L.dtype == kBfloat16) return launch<AdamWOp<__nv_bfloat16, true, MULTI>>(L, st);
  KV_FATAL << "unsupported dtype " << DTypeName(L.dtype);
}

}  // namespace

void LaunchMultiTensor(const MTLaunch& L, cudaStream_t st) {
  if (L.n_chunks <= 0) return;
  switch (L.op) {
    case kMTSumSq:
      if (L.dtype == kFloat32) launch<SumSqOp<float>>(L, st);
      else if (L.dtype == kFloat16) launch<SumSqOp<__half>>(L, st);
      else if (L.dtype == kBfloat16) launch<SumSqOp<__nv_bfloat16>>(L, st);
      else KV_FATAL << "multi_sum_sq: unsupported dtype " << DTypeName(L.dtype);
      break;
    case kMTAdamW: launch_adamw<false>(L, st); break;
    case kMTMultiAdamW: launch_adamw<true>(L, st); break;
    case kMTLambPhase1: launch_tm<LambPhase1Op>(L, st); break;
    case kMTLambPhase2: launch_tm<LambPhase2Op>(L, st); break;
    case kMTMultiLambStep1: launch_tm<MultiLambStep1Op>(L, st); break;
    case kMTMultiLambStep2: launch_tm<MultiLambStep2Op>(L, st); break;
    default: KV_FATAL << "unknown multi-tensor op " << L.op;
  }
  KV_CUDA(cudaGetLastError());
}

void LaunchMultiTensorFinalize(const MTTensor* tensors, int n_tensors, const float* part0,
                               const float* part1, float* out0, float* out1, cudaStream_t st) {
  if (n_tensors <= 0) return;
  mt_finalize_kernel<<<n_tensors, kThreads, 0, st>>>(tensors, part0, part1, out0, out1);
  KV_CUDA(cudaGetLastError());
}

void LaunchMultiLars(int n, float* out, const float* lrs, const float* wsq, const float* gsq,
                     const float* wds, float eta, float eps, float rescale, cudaStream_t st) {
  if (n <= 0) return;
  lars_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, out, lrs, wsq, gsq, wds, eta, eps, rescale);
  KV_CUDA(cudaGetLastError());
}

void LaunchAllFinite(int dtype, AllFiniteArrays& A, float* out, cudaStream_t st) {
  KV_CHECK(A.count >= 1 && A.count <= kAFMaxArrays);
  const uint64_t tile_elems = kAFTileBytes / DTypeSize(dtype);
  uint64_t tiles = 0;
  for (int i = 0; i < A.count; ++i) {
    A.first_tile[i] = static_cast<uint32_t>(tiles);
    tiles += (A.n[i] + tile_elems - 1) / tile_elems;
    KV_CHECK(tiles < (1ULL << 31)) << "all_finite: more than 2^31 tiles of " << kAFTileBytes << " bytes";
  }
  A.first_tile[A.count] = static_cast<uint32_t>(tiles);
  const unsigned grid = static_cast<unsigned>(std::max<uint64_t>(tiles, 1));
  switch (dtype) {
    case kFloat16: all_finite_kernel<__half><<<grid, kAFThreads, 0, st>>>(A, out); break;
    case kBfloat16: all_finite_kernel<__nv_bfloat16><<<grid, kAFThreads, 0, st>>>(A, out); break;
    case kFloat32: all_finite_kernel<float><<<grid, kAFThreads, 0, st>>>(A, out); break;
    case kFloat64: all_finite_kernel<double><<<grid, kAFThreads, 0, st>>>(A, out); break;
    default: KV_FATAL << "all_finite: unsupported dtype " << DTypeName(dtype);
  }
  KV_CUDA(cudaGetLastError());
}

uint32_t ClipNormTiles(ClipNormArrays& A) {
  KV_CHECK(A.count >= 1 && A.count <= kCNMaxArrays);
  uint32_t tiles = 0;  // <= 200 arrays x 2^20 tiles each
  for (int i = 0; i < A.count; ++i) {
    A.first_tile[i] = tiles;
    tiles += static_cast<uint32_t>((static_cast<uint64_t>(A.n[i]) + kCNTileElems - 1) / kCNTileElems);
  }
  A.first_tile[A.count] = tiles;
  return tiles;
}

void LaunchClipNormPartial(const ClipNormArrays& A, uint32_t tiles, float* part, cudaStream_t st) {
  KV_CHECK(tiles >= 1 && tiles == A.first_tile[A.count]);
  clip_norm_partial_kernel<<<tiles, kCNThreads, 0, st>>>(A, part);
  KV_CUDA(cudaGetLastError());
}

void LaunchClipNormFold(const float* part, uint32_t n_part, float max_norm, float* total_norm,
                        float* scale, cudaStream_t st) {
  clip_norm_fold_kernel<<<1, kCNThreads, 0, st>>>(part, n_part, max_norm, total_norm, scale);
  KV_CUDA(cudaGetLastError());
}

void LaunchClipNormScale(const ClipNormArrays& A, uint32_t tiles, const float* scale_dev, float scale,
                         cudaStream_t st) {
  KV_CHECK(tiles >= 1 && tiles == A.first_tile[A.count]);
  clip_norm_scale_kernel<<<tiles, kCNThreads, 0, st>>>(A, scale_dev, scale);
  KV_CUDA(cudaGetLastError());
}

int LaunchResetArrays(ResetArraysList& A, cudaStream_t st) {
  KV_CHECK(A.count >= 1 && A.count <= kRAMaxArrays);
  uint64_t tiles = 0;
  for (int i = 0; i < A.count; ++i) {
    A.first_tile[i] = static_cast<uint32_t>(tiles);
    tiles += (A.bytes[i] + kRATileBytes - 1) / kRATileBytes;
    KV_CHECK(tiles < (1ULL << 31)) << "reset_arrays: more than 2^31 tiles of " << kRATileBytes << " bytes";
  }
  A.first_tile[A.count] = static_cast<uint32_t>(tiles);
  if (tiles == 0) return 0;
  reset_arrays_kernel<<<static_cast<unsigned>(tiles), kRAThreads, 0, st>>>(A);
  KV_CUDA(cudaGetLastError());
  return 1;
}

}  // namespace b200kv
