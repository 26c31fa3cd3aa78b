// dense_kernels.cu -- the hot kernel of the KVStore path on H100 (sm_90a).
//
// ONE launch per device does, for every chunk the device owns:
//     merged = sum over sources (local HBM or peer HBM through NVLink-mapped pointers), in the
//              reference's association order
//     (w, state) = optimizer_step(w, rescale/clip(merged), state)          [optional]
//     store w (+ fp32 master) locally, and broadcast w to every pull target (local or peer)
// replacing, per key, the reference's (N-1) cudaMemcpyPeerAsync + ElementwiseSum + Python updater
// callback -> optimizer kernel + N broadcast copies (src/kvstore/comm.h:503-616,
// src/ndarray/ndarray_function-inl.h:387-434, src/operator/optimizer_op-inl.h).
//
// Bandwidth-bound elementwise work: no tensor cores, no shared-memory staging of data (every byte
// is touched once). What matters is 16-byte coalesced accesses, enough independent loads in flight
// per SM to cover HBM/NVLink latency (all source loads of a vector are issued before the first
// add), streaming cache hints, and a grid of one CTA per 4096-element chunk so the 132 SMs stay
// full even though tensor sizes range from 3 to 23M elements.
//
// Arithmetic: IEEE fp32 round-to-nearest with NO fused multiply-add (explicit __f*_rn intrinsics;
// the file is also compiled with -fmad=false) so results are bit-identical to the reference's CPU
// build (`-O3 -msse3`), i.e. to oracle/kvoracle.c. Expression trees per optimizer are cited below.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.h"
#include "kernels.h"
#include "opt_math.cuh"

namespace b200kv {
namespace {

constexpr int kThreads = 256;

// ---- storage types: fp32 / fp16 / bf16 --------------------------------------------------------
template <typename T> struct Cvt;
template <> struct Cvt<float> {
  static __device__ __forceinline__ float to_f(float x) { return x; }
  static __device__ __forceinline__ float from_f(float x) { return x; }
  static __device__ __forceinline__ float round(float x) { return x; }
};
template <> struct Cvt<__half> {
  static __device__ __forceinline__ float to_f(__half x) { return __half2float(x); }
  static __device__ __forceinline__ __half from_f(float x) { return __float2half_rn(x); }
  static __device__ __forceinline__ float round(float x) { return __half2float(__float2half_rn(x)); }
};
template <> struct Cvt<__nv_bfloat16> {
  static __device__ __forceinline__ float to_f(__nv_bfloat16 x) { return __bfloat162float(x); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float x) { return __float2bfloat16_rn(x); }
  static __device__ __forceinline__ float round(float x) {
    return __bfloat162float(__float2bfloat16_rn(x));
  }
};

// V elements per thread per access: 16-byte packs on the vector path, 1 on the scalar tail path.
template <typename T, int V> struct IO;
template <typename T> struct IO<T, 8> {  // T = __half / __nv_bfloat16: 8 x 16 bit = 16 bytes
  static __device__ __forceinline__ void ld(const T* p, float (&x)[8]) {
    uint4 raw = __ldcs(reinterpret_cast<const uint4*>(p));
    const T* h = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = Cvt<T>::to_f(h[i]);
  }
  static __device__ __forceinline__ void st(T* p, const float (&x)[8]) {
    uint4 raw;
    T* h = reinterpret_cast<T*>(&raw);
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = Cvt<T>::from_f(x[i]);
    __stcs(reinterpret_cast<uint4*>(p), raw);
  }
};
template <typename T> struct IO<T, 1> {
  static __device__ __forceinline__ void ld(const T* p, float (&x)[1]) {
    const unsigned short u = __ldcs(reinterpret_cast<const unsigned short*>(p));
    x[0] = Cvt<T>::to_f(*reinterpret_cast<const T*>(&u));
  }
  static __device__ __forceinline__ void st(T* p, const float (&x)[1]) {
    T v = Cvt<T>::from_f(x[0]);
    __stcs(reinterpret_cast<unsigned short*>(p), *reinterpret_cast<unsigned short*>(&v));
  }
};

template <> struct IO<float, 4> {
  static __device__ __forceinline__ void ld(const float* p, float (&x)[4]) {
    float4 t = __ldcs(reinterpret_cast<const float4*>(p));
    x[0] = t.x; x[1] = t.y; x[2] = t.z; x[3] = t.w;
  }
  static __device__ __forceinline__ void st(float* p, const float (&x)[4]) {
    __stcs(reinterpret_cast<float4*>(p), make_float4(x[0], x[1], x[2], x[3]));
  }
};
template <> struct IO<float, 8> {
  static __device__ __forceinline__ void ld(const float* p, float (&x)[8]) {
    float4 a = __ldcs(reinterpret_cast<const float4*>(p));
    float4 b = __ldcs(reinterpret_cast<const float4*>(p) + 1);
    x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
  }
  static __device__ __forceinline__ void st(float* p, const float (&x)[8]) {
    __stcs(reinterpret_cast<float4*>(p), make_float4(x[0], x[1], x[2], x[3]));
    __stcs(reinterpret_cast<float4*>(p) + 1, make_float4(x[4], x[5], x[6], x[7]));
  }
};
template <> struct IO<float, 1> {
  static __device__ __forceinline__ void ld(const float* p, float (&x)[1]) { x[0] = __ldcs(p); }
  static __device__ __forceinline__ void st(float* p, const float (&x)[1]) { __stcs(p, x[0]); }
};

// Process V consecutive elements, starting at element off + v*V. EVERY load is issued before the
// first arithmetic instruction or store: n_src + 1 + states 16-byte loads in flight per thread,
// which is what covers NVLink latency when the sources are peer memory.
template <typename T, int MAXSRC, int OPT, int V>
__device__ __forceinline__ void process(const KeyDesc& k, uint32_t off, uint32_t v, int n_src, int n_out,
                                        int order, const Hyper& h) {
  float acc[V];
  float wv[V], s1[V], s2[V];
  const bool has_mom = k.s1 != nullptr;
  const bool mp = k.w32 != nullptr;
  const uint32_t base = off + v * V;
  if (OPT != kOptPullOnly) {
    float g[MAXSRC][V];
#pragma unroll
    for (int i = 0; i < MAXSRC; ++i) {
      if (i < n_src) IO<T, V>::ld(static_cast<const T*>(k.src[i]) + base, g[i]);
    }
    if (OPT != kOptAssign) {
      if (mp) {
        IO<float, V>::ld(k.w32 + base, wv);
      } else {
        IO<T, V>::ld(static_cast<const T*>(k.w_in) + base, wv);
      }
      if ((OPT == kOptSGD && has_mom) || OPT == kOptAdam) IO<float, V>::ld(k.s1 + base, s1);
      if (OPT == kOptAdam) IO<float, V>::ld(k.s2 + base, s2);
    }
    // ---- merged gradient in the reference's association; 16-bit dtypes round after every add,
    // as mshadow's half arithmetic does (3rdparty/mshadow/mshadow/half.h:45-66)
#pragma unroll
    for (int j = 0; j < V; ++j) acc[j] = g[0][j];
    if (order == kOrderDevice) {
      // ((g0+g1)+g2)+...   (ndarray_function-inl.h:402-431)
#pragma unroll
      for (int i = 1; i < MAXSRC; ++i) {
        if (i < n_src) {
#pragma unroll
          for (int j = 0; j < V; ++j) acc[j] = Cvt<T>::round(__fadd_rn(acc[j], g[i][j]));
        }
      }
    } else {
      // g0 + (((g1+g2)+g3)+g4) + (((g5+..  (comm.h:357-392)
#pragma unroll
      for (int i = 1; i < MAXSRC; i += 4) {
        if (i < n_src) {
          float t[V];
#pragma unroll
          for (int j = 0; j < V; ++j) t[j] = g[i][j];
#pragma unroll
          for (int q = 1; q < 4; ++q) {
            if (i + q < MAXSRC && i + q < n_src) {
#pragma unroll
              for (int j = 0; j < V; ++j) t[j] = Cvt<T>::round(__fadd_rn(t[j], g[i + q][j]));
            }
          }
#pragma unroll
          for (int j = 0; j < V; ++j) acc[j] = Cvt<T>::round(__fadd_rn(acc[j], t[j]));
        }
      }
    }
    // ---- optimizer step
    if (OPT == kOptTest && sizeof(T) == 2) {
      // weight[:] += grad * rescale_grad on a 16-bit key: _mul_scalar then _plus, each rounding
      // to T as mshadow's half arithmetic does, with the scalar cast to T first (a Test key never
      // carries an fp32 master)
      const float r = Cvt<T>::round(h.rescale);
#pragma unroll
      for (int j = 0; j < V; ++j) {
        acc[j] = Cvt<T>::round(__fadd_rn(wv[j], Cvt<T>::round(__fmul_rn(acc[j], r))));
      }
    } else if (OPT != kOptAssign) {
#pragma unroll
      for (int j = 0; j < V; ++j) acc[j] = step<OPT>(wv[j], acc[j], s1[j], s2[j], has_mom, h);
      if ((OPT == kOptSGD && has_mom) || OPT == kOptAdam) IO<float, V>::st(k.s1 + base, s1);
      if (OPT == kOptAdam) IO<float, V>::st(k.s2 + base, s2);
      if (mp) IO<float, V>::st(k.w32 + base, acc);
    }
    IO<T, V>::st(static_cast<T*>(k.w) + base, acc);
  } else {
    IO<T, V>::ld(static_cast<const T*>(k.w_in) + base, acc);
  }
  // ---- broadcast to every pull target (peer stores ride NVLink)
  for (int o = 0; o < n_out; ++o) IO<T, V>::st(static_cast<T*>(k.out[o]) + base, acc);
}

// ---- NVLS variant of one fp32 vector: the cross-rank sum happens INSIDE the NVSwitch
// (multimem.ld_reduce on the multicast mapping of the ranks' arenas) and one multimem.st delivers
// the new weights to every rank, so each GPU receives S/N + (N-1)/N*S bytes per step instead of
// 2*(N-1)/N*S. The switch's summation order is unspecified: results match the reference within
// fp32 rounding (1e-6 relative), not bit for bit -- this path is opt-in (B200KV_NVLS=1).
__device__ __forceinline__ float4 multimem_ld_reduce_f32x4(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_f32x4(float* mc, const float (&x)[4]) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(x[0]),
               "f"(x[1]), "f"(x[2]), "f"(x[3])
               : "memory");
}

template <int V> struct MM;
template <> struct MM<4> {
  static __device__ __forceinline__ void ld_reduce(const float* mc, float (&x)[4]) {
    const float4 g = multimem_ld_reduce_f32x4(mc);
    x[0] = g.x; x[1] = g.y; x[2] = g.z; x[3] = g.w;
  }
  static __device__ __forceinline__ void st(float* mc, const float (&x)[4]) { multimem_st_f32x4(mc, x); }
};
template <> struct MM<1> {
  static __device__ __forceinline__ void ld_reduce(const float* mc, float (&x)[1]) {
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.f32 %0, [%1];" : "=f"(x[0]) : "l"(mc) : "memory");
  }
  static __device__ __forceinline__ void st(float* mc, const float (&x)[1]) {
    asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(mc), "f"(x[0]) : "memory");
  }
};

// every multimem.ld_reduce (and the local weight / state loads) is issued before the first store
template <int OPT, int V>
__device__ __forceinline__ void process_nvls(const KeyDesc& k, uint32_t off, uint32_t v, const Hyper& h) {
  float acc[V], wv[V], s1[V], s2[V];
  const bool has_mom = k.s1 != nullptr;
  float* w = static_cast<float*>(k.w);
  const uint32_t base = off + v * V;
  if (OPT != kOptPullOnly) {
    MM<V>::ld_reduce(static_cast<const float*>(k.src[kMaxSrc - 1]) + base, acc);
    if (OPT != kOptAssign) {
      IO<float, V>::ld(w + base, wv);
      if ((OPT == kOptSGD && has_mom) || OPT == kOptAdam) IO<float, V>::ld(k.s1 + base, s1);
      if (OPT == kOptAdam) IO<float, V>::ld(k.s2 + base, s2);
#pragma unroll
      for (int j = 0; j < V; ++j) acc[j] = step<OPT>(wv[j], acc[j], s1[j], s2[j], has_mom, h);
      if ((OPT == kOptSGD && has_mom) || OPT == kOptAdam) IO<float, V>::st(k.s1 + base, s1);
      if (OPT == kOptAdam) IO<float, V>::st(k.s2 + base, s2);
    }
    IO<float, V>::st(w + base, acc);
  } else {
    IO<float, V>::ld(w + base, acc);
  }
  const int n_mc = static_cast<int>(k.nvls) - 1;
  for (int o = 0; o < n_mc; ++o) MM<V>::st(static_cast<float*>(k.out[kMaxDst - 2 + o]) + base, acc);
}

struct KernelArgs {
  const KeyDesc* keys;
  const ChunkDesc* chunks;
  const float2* hyper;  // per key (lr, wd); re-uploaded only when a value changes
  const float* lrs;     // preloaded_multi_*: per-key lr / wd live in two device arrays instead
  const float* wds;
  int order;
  float momentum, rescale, clip, beta1, beta2, eps;
  // one-rank-per-GPU launches (group.h): IPC-mapped signal pads of every rank, or null
  uint32_t* const* pads;
  uint32_t* counter;  // CTAs of this rank that have finished
  int rank, world;
  uint32_t epoch;
  int n_chunks;
  uint32_t* err_word;
  unsigned long long timeout_ns;
  int barrier_mask;
};

// ---- cross-process barrier on IPC-mapped signal pads ------------------------------------------
// pad layout per rank: start flags [kMaxDevices], end flags [kMaxDevices], one 128-byte line each.
// Rank r writes its epoch into slot r of EVERY peer's pad; it waits on its OWN pad (local memory
// written remotely), so spinning never crosses NVLink.
constexpr int kPadStrideK = 32;
constexpr int kMaxDevK = 16;

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// threads 0..world-1 of the calling CTA each handle one peer; `phase` 0 = start, 1 = end.
__device__ __forceinline__ void peer_signal_and_wait(const KernelArgs& a, int phase, bool signal) {
  const int t = threadIdx.x;
  if (t < a.world && t != a.rank) {
    const int base = phase * kMaxDevK * kPadStrideK;
    if (signal) st_release_sys(a.pads[t] + base + a.rank * kPadStrideK, a.epoch);
    const uint32_t* mine = a.pads[a.rank] + base + t * kPadStrideK;
    const unsigned long long t0 = globaltimer_ns();
    uint32_t spins = 0;
    while (static_cast<int32_t>(ld_acquire_sys(mine) - a.epoch) < 0) {
      __nanosleep(spins < 64 ? 32 : 1000);   // back off: a waiting rank should not hammer its L2
      if ((++spins & 1023u) == 0 && a.timeout_ns != 0 && globaltimer_ns() - t0 > a.timeout_ns) {
        // the peer never launched the matching call (B200KV_PEER_TIMEOUT_S, default 10 minutes: a
        // checkpoint, an evaluation pass or a data-loader stall on one rank are ordinary). Report
        // through host-visible memory and stop waiting; no __trap, the context stays alive.
        volatile uint32_t* ew = a.err_word;   // pinned host memory: plain stores (no PCIe atomics)
        if (ew != nullptr && ew[0] == 0u) {
          ew[1] = (static_cast<uint32_t>(phase) << 31) | (a.epoch & 0x7fffffffu);
          __threadfence_system();
          ew[0] = static_cast<uint32_t>(t) + 1u;
        }
        break;
      }
    }
  }
}

template <typename T, int MAXSRC, int OPT>
constexpr int MinBlocks() {
  if (sizeof(T) != 4 || MAXSRC > 8) return 1;   // 16-bit packs carry 8 values per load
  if (MAXSRC == 1) return 5;
  const int adam = OPT == kOptAdam ? 1 : 0;                            // two more state vectors
  return (MAXSRC <= 2 ? 5 : 4) - adam;
}

// NVLS: the instantiation for launches whose sums happen in the NVSwitch (fp32, MAXSRC = 1).
// One group of V elements per thread: for local and peer-memory sources the kernel is limited by
// the link, not by loads in flight, and the registers of a second group cost resident CTAs.
template <typename T, int MAXSRC, int OPT, bool NVLS>
// resident CTAs per SM matter more than registers here (every CTA starts with two dependent
// descriptor loads): the caps below keep the register budgets of the round-1 kernel (48 / 48 / 64)
__global__ void __launch_bounds__(kThreads, MinBlocks<T, MAXSRC, OPT>())
dense_fused_kernel(const KernelArgs a) {
  constexpr int V = 16 / sizeof(T);
  __shared__ KeyDesc sk;
  __shared__ uint32_t s_last;
  if (a.pads != nullptr && (a.barrier_mask & 1)) {
    // start barrier: a rank's kernel only starts after its stream produced its gradients, so
    // "every peer has started" == "every peer's gradients (and pull targets) are ready". With the
    // gate launch (group.h) this wait runs in a one-CTA kernel ahead of this one, so that a rank
    // waiting for a late peer does not hold every SM with spinning CTAs.
    peer_signal_and_wait(a, 0, blockIdx.x == 0);
    __syncthreads();
  }
  if (static_cast<int>(blockIdx.x) < a.n_chunks) {
  const ChunkDesc c = a.chunks[blockIdx.x];
  {
    constexpr int NW = sizeof(KeyDesc) / 16;
    static_assert(sizeof(KeyDesc) % 16 == 0 && NW <= kThreads, "KeyDesc layout");
    const uint4* gk = reinterpret_cast<const uint4*>(a.keys + c.key);
    if (threadIdx.x < NW) reinterpret_cast<uint4*>(&sk)[threadIdx.x] = gk[threadIdx.x];
  }
  __syncthreads();
  Hyper h;
  const float2 lw = a.lrs != nullptr ? make_float2(a.lrs[c.key], a.wds[c.key]) : a.hyper[c.key];
  h.lr = lw.x; h.wd = lw.y; h.momentum = a.momentum; h.rescale = a.rescale; h.clip = a.clip;
  h.beta1 = a.beta1; h.beta2 = a.beta2; h.eps = a.eps;
  const int n_src = sk.n_src, n_out = sk.n_out;
  const uint32_t nvec = sk.vec_ok ? c.len / V : 0;
  if (NVLS) {
    // (host side: NVLS plans are fp32 and every key of the launch carries multicast addresses)
    for (uint32_t v = threadIdx.x; v < nvec; v += kThreads) process_nvls<OPT, 4>(sk, c.off, v, h);
    const uint32_t ntail = c.len - nvec * 4;
    for (uint32_t e = threadIdx.x; e < ntail; e += kThreads) process_nvls<OPT, 1>(sk, c.off + nvec * 4, e, h);
  } else {
    for (uint32_t v = threadIdx.x; v < nvec; v += kThreads) {
      process<T, MAXSRC, OPT, V>(sk, c.off, v, n_src, n_out, a.order, h);
    }
    const uint32_t ntail = c.len - nvec * V;
    for (uint32_t e = threadIdx.x; e < ntail; e += kThreads) {
      process<T, MAXSRC, OPT, 1>(sk, c.off + nvec * V, e, n_src, n_out, a.order, h);
    }
  }
  }  // blockIdx.x < n_chunks
  if (a.pads != nullptr && (a.barrier_mask & 2)) {
    // end barrier: the LAST CTA of this rank to finish tells every peer "I have read your
    // gradients and written your weights" and waits for the same from them; the kernel -- hence
    // everything the stream runs after it -- completes only when all peers are done with us.
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();  // this CTA's peer stores are visible system-wide ...
      const uint32_t done = atomicAdd(a.counter, 1u);  // ... before it is counted as finished
      s_last = (done == gridDim.x - 1) ? 1u : 0u;
    }
    __syncthreads();
    if (s_last) {
      __threadfence_system();
      peer_signal_and_wait(a, 1, true);
      __syncthreads();
      if (threadIdx.x == 0) *a.counter = 0;  // ready for the next launch (stream-ordered)
    }
  }
}

// ---- the other mshadow dtypes (float64, int32, int64, uint8, int8): reduce / assign / broadcast
// only -- the reference's reducers are instantiated for every dtype (MSHADOW_TYPE_SWITCH,
// src/kvstore/comm.h:273, ndarray_function-inl.h:399) while its optimizer operators are floating
// point. Same chunk list, same association orders, native arithmetic of T, element-wise path.
template <typename T>
__global__ void __launch_bounds__(kThreads) dense_plain_kernel(const KernelArgs a, int opt) {
  __shared__ KeyDesc sk;
  __shared__ uint32_t s_last;
  if (a.pads != nullptr && (a.barrier_mask & 1)) {
    peer_signal_and_wait(a, 0, blockIdx.x == 0);
    __syncthreads();
  }
  if (static_cast<int>(blockIdx.x) < a.n_chunks) {
    const ChunkDesc c = a.chunks[blockIdx.x];
    constexpr int NW = sizeof(KeyDesc) / 16;
    const uint4* gk = reinterpret_cast<const uint4*>(a.keys + c.key);
    if (threadIdx.x < NW) reinterpret_cast<uint4*>(&sk)[threadIdx.x] = gk[threadIdx.x];
    __syncthreads();
    const int n_src = sk.n_src, n_out = sk.n_out;
    for (uint32_t e = threadIdx.x; e < c.len; e += kThreads) {
      const uint32_t i = c.off + e;
      T acc;
      if (opt != kOptPullOnly) {
        acc = static_cast<const T*>(sk.src[0])[i];
        if (a.order == kOrderDevice) {
          for (int k = 1; k < n_src; ++k) acc = static_cast<T>(acc + static_cast<const T*>(sk.src[k])[i]);
        } else {
          for (int k = 1; k < n_src; k += 4) {
            T t = static_cast<const T*>(sk.src[k])[i];
            for (int q = 1; q < 4 && k + q < n_src; ++q) t = static_cast<T>(t + static_cast<const T*>(sk.src[k + q])[i]);
            acc = static_cast<T>(acc + t);
          }
        }
        static_cast<T*>(sk.w)[i] = acc;
      } else {
        acc = static_cast<const T*>(sk.w_in)[i];
      }
      for (int o = 0; o < n_out; ++o) static_cast<T*>(sk.out[o])[i] = acc;
    }
  }
  if (a.pads != nullptr && (a.barrier_mask & 2)) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();
      const uint32_t done = atomicAdd(a.counter, 1u);
      s_last = (done == gridDim.x - 1) ? 1u : 0u;
    }
    __syncthreads();
    if (s_last) {
      __threadfence_system();
      peer_signal_and_wait(a, 1, true);
      __syncthreads();
      if (threadIdx.x == 0) *a.counter = 0;
    }
  }
}

template <typename T>
void launch_plain(const DenseLaunch& p, cudaStream_t s) {
  KV_CHECK(p.opt == kOptAssign || p.opt == kOptPullOnly)
      << "optimizers on the store run on float32 / float16 / bfloat16 keys; " << DTypeName(p.dtype)
      << " keys are reduced, assigned and pulled";
  KV_CHECK(!p.nvls);
  KernelArgs a{p.keys, p.chunks, reinterpret_cast<const float2*>(p.hyper), p.lrs, p.wds, p.order, p.momentum,
               p.rescale, p.clip, p.beta1, p.beta2, p.eps, p.signal_pads, p.counter, p.rank, p.world,
               p.epoch, p.n_chunks, p.err_word, p.timeout_ns, p.barrier_mask};
  const int grid = p.n_chunks > 0 ? p.n_chunks : 1;
  dense_plain_kernel<T><<<grid, kThreads, 0, s>>>(a, p.opt);
}

template <typename T, int MAXSRC, int OPT, bool NVLS = false>
void launch_one(const DenseLaunch& p, cudaStream_t s) {
  KernelArgs a{p.keys, p.chunks, reinterpret_cast<const float2*>(p.hyper), p.lrs, p.wds, p.order, p.momentum,
               p.rescale, p.clip, p.beta1, p.beta2, p.eps, p.signal_pads, p.counter, p.rank, p.world,
               p.epoch, p.n_chunks, p.err_word, p.timeout_ns, p.barrier_mask};
  const int grid = p.n_chunks > 0 ? p.n_chunks : 1;  // a rank with no chunk still joins the barriers
  dense_fused_kernel<T, MAXSRC, OPT, NVLS><<<grid, kThreads, 0, s>>>(a);
}

template <typename T, int OPT>
void launch_src(const DenseLaunch& p, cudaStream_t s) {
  if (p.nvls) {
    if constexpr (sizeof(T) == 4) return launch_one<T, 1, OPT, true>(p, s);
    KV_FATAL << "NVLS launches are float32";
  }
  if (OPT == kOptPullOnly || p.max_src <= 1) return launch_one<T, 1, OPT>(p, s);
  if (p.max_src <= 2) return launch_one<T, 2, OPT>(p, s);
  if (p.max_src <= 4) return launch_one<T, 4, OPT>(p, s);
  if (p.max_src <= 8) return launch_one<T, 8, OPT>(p, s);
  return launch_one<T, 16, OPT>(p, s);
}

template <typename T>
void launch_opt(const DenseLaunch& p, cudaStream_t s) {
  switch (p.opt) {
    case kOptAssign: return launch_src<T, kOptAssign>(p, s);
    case kOptSGD: return launch_src<T, kOptSGD>(p, s);
    case kOptSGDSingle: return launch_src<T, kOptSGDSingle>(p, s);
    case kOptAdam: return launch_src<T, kOptAdam>(p, s);
    case kOptTest: return launch_src<T, kOptTest>(p, s);
    case kOptPullOnly: return launch_src<T, kOptPullOnly>(p, s);
  }
  KV_FATAL << "unknown optimizer kind " << p.opt;
}

}  // namespace

void LaunchDenseFused(const DenseLaunch& p, cudaStream_t stream) {
  if (p.n_chunks <= 0 && p.signal_pads == nullptr) return;
  KV_CHECK(p.max_src <= kMaxSrc) << "at most " << kMaxSrc << " values per key";
  switch (p.dtype) {
    case kFloat32: launch_opt<float>(p, stream); break;
    case kFloat16: launch_opt<__half>(p, stream); break;
    case kBfloat16: launch_opt<__nv_bfloat16>(p, stream); break;
    case kFloat64: launch_plain<double>(p, stream); break;
    case kInt32: launch_plain<int32_t>(p, stream); break;
    case kInt64: launch_plain<int64_t>(p, stream); break;
    case kUint8: launch_plain<uint8_t>(p, stream); break;
    case kInt8: launch_plain<int8_t>(p, stream); break;
    default: KV_FATAL << "dense KVStore kernels: unsupported dtype " << DTypeName(p.dtype);
  }
  KV_CUDA(cudaGetLastError());
}

}  // namespace b200kv
