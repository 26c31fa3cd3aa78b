// rowsparse_kernels.cu -- row_sparse push / row_sparse_pull kernels for sm_90a.
//
// Reference semantics (bit-exact targets, all integer/index results identical):
//   * reduce: out ids = ascending unique union of the sources' ids; out rows start at 0.0f and the
//     sources are accumulated in list order (src/ndarray/ndarray_function.cc:59-175 on CPU,
//     ndarray_function.cu:104-190 on GPU -- the GPU version marks a flag array as long as the whole
//     table (1M rows -> 8 MB scan); here the union is a radix sort over the <= N*nnr ids actually
//     present, independent of table height);
//   * unique: sort + unique of the requested row ids (src/kvstore/kvstore_utils.cu:43-97);
//   * retain: every requested id is emitted, rows copied where present else zero
//     (src/operator/tensor/sparse_retain-inl.h:121-150,262-323);
//   * lazy optimizer updates over the gradient's rows (optimizer_op-inl.h:426-475,749-801,1350-1408).
//
// Row gathers/scatters are HBM- (or NVLink-) bound: one warp per row, 16-byte accesses along the
// row, all of a row's source loads issued before the ordered adds. The id bookkeeping is arranged
// so that no warp ever chases pointers through PEER memory: the union sorts (id, position) pairs,
// which hands every output row its source rows directly (the first version binary-searched every
// source's id list per row -- a chain of dependent peer loads per row made that kernel many times
// slower than its traffic). Row counts stay on the device: grids cover the upper bound and surplus warps
// exit, so a push with a fused optimizer never blocks the host.
#include <cub/cub.cuh>

#include "common.h"
#include "kernels.h"
#include "opt_math.cuh"

namespace b200kv {
namespace {

constexpr int kWarpsPerBlock = 8;

// lower bound by the whole warp: 32 probes per round (log33 n rounds instead of log2 n)
__device__ __forceinline__ int64_t warp_lower_bound(const int64_t* a, int64_t n, int64_t key, int lane) {
  int64_t lo = 0, hi = n;  // the answer lies in [lo, hi]
  while (lo < hi) {
    const int64_t len = hi - lo;
    const int64_t step = (len + 32) / 33;
    const int64_t p = lo + (lane + 1) * step - 1;
    const bool lt = p < hi ? (a[p] < key) : false;
    const int c = __popc(__ballot_sync(0xffffffffu, lt));  // probes are sorted: a prefix is true
    const int64_t nlo = lo + c * step;
    const int64_t nhi = c == 32 ? hi : min(hi, lo + (c + 1) * step - 1);
    lo = nlo;
    hi = nhi;
  }
  return lo;
}

// index of the segment that contains i: largest s with start[s] <= i (start ascending, small)
__device__ __forceinline__ int find_segment(const int64_t* start, int nseg, int64_t i) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (start[mid] <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---------------------------------------------------------------------------------------------
// row_sparse forms of the operators (ftrl_update, _sparse_adagrad_update, lazy sgd_update /
// sgd_mom_update / adam_update): one warp per gradient row in a grid-stride loop, the row id read
// once per row, then the row's elements through the same Step<OP> as the dense update_kernel; out is
// the weight itself
template <int OP>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) rsp_row_update_kernel(const UpdateLaunch a,
                                                                              const bool vec) {
  constexpr int NS = NumStates(OP);
  constexpr int NA = NS > 0 ? NS : 1;  // sgd_update has no state, an array needs one entry
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = static_cast<int64_t>(gridDim.x) * kWarpsPerBlock;
  const int64_t len = a.row_len;
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5); r < a.nnr;
       r += nwarps) {
    const int64_t off = a.gidx[r] * len;
    const float* g = static_cast<const float*>(a.g) + r * len;
    float* w = static_cast<float*>(a.out) + off;
    float* s[NA];
#pragma unroll
    for (int k = 0; k < NS; ++k) s[k] = a.s[k] + off;
    if (vec) {
      for (int64_t v = lane; v < len / 4; v += 32) {
        const float4 g4 = __ldcs(reinterpret_cast<const float4*>(g) + v);
        const float4 w4 = reinterpret_cast<const float4*>(w)[v];
        float4 s4[NA];
#pragma unroll
        for (int k = 0; k < NS; ++k) s4[k] = reinterpret_cast<const float4*>(s[k])[v];
        const float gx[4] = {g4.x, g4.y, g4.z, g4.w}, wx[4] = {w4.x, w4.y, w4.z, w4.w};
        float o[4], sx[NA][4];
#pragma unroll
        for (int k = 0; k < NS; ++k) {
          sx[k][0] = s4[k].x; sx[k][1] = s4[k].y; sx[k][2] = s4[k].z; sx[k][3] = s4[k].w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float st[3] = {0.f, 0.f, 0.f};
#pragma unroll
          for (int k = 0; k < NS; ++k) st[k] = sx[k][j];
          o[j] = Step<OP>(a, wx[j], gx[j], st);
#pragma unroll
          for (int k = 0; k < NS; ++k) sx[k][j] = st[k];
        }
        reinterpret_cast<float4*>(w)[v] = make_float4(o[0], o[1], o[2], o[3]);
#pragma unroll
        for (int k = 0; k < NS; ++k) {
          reinterpret_cast<float4*>(s[k])[v] = make_float4(sx[k][0], sx[k][1], sx[k][2], sx[k][3]);
        }
      }
    } else {
      for (int64_t j = lane; j < len; j += 32) {
        float st[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < NS; ++k) st[k] = s[k][j];
        w[j] = Step<OP>(a, w[j], __ldcs(g + j), st);
#pragma unroll
        for (int k = 0; k < NS; ++k) s[k][j] = st[k];
      }
    }
  }
}

// ---- _contrib_group_adagrad_update: GroupAdagradDnsRspKernel<cpu> (contrib/optimizer_op-inl.h:96-139)
//   gr_j = clip(g_j * rescale);  ssq = ((0 + gr_0^2) + gr_1^2) + ... + gr_{L-1}^2   (left fold)
//   h[r] = h[r] + ssq / (float)L;   w_j = w_j - (lr * gr_j) / sqrt(h[r] + eps)
// One warp per gradient row. The row is cut into tiles of kGaTile elements; lane k holds the
// contiguous run [16k, 16k+16) of a tile in registers, so the fold order is lane 0's run, then lane
// 1's, ...: every lane squares its run in parallel, then the running sum walks the lanes in order,
// each lane adding its 16 squares with one rounding per add and handing the sum on by __shfl_sync.
// Elements past the row's end hold +0.0f: the running sum is never -0.0f (it starts at +0.0f and
// adds squares), so adding +0.0f leaves it bitwise unchanged. The chain is ~32 x (16 adds + 1
// shuffle) deep per tile; other warps' row traffic, and for one-tile rows this warp's own L2
// prefetches issued before the fold, cover it.
constexpr int kGaPer = 16;
constexpr int kGaTile = 32 * kGaPer;

// lane's run of one tile of a row (`row` at the tile's first element, `n` elements left in the
// row), +0.0f past the end; vector form: n % 4 == 0 and `row` 16-B aligned
template <bool VEC, bool STREAM>
__device__ __forceinline__ void GaLoad(const float* row, int64_t n, int lane, float (&x)[kGaPer]) {
  const int64_t o = static_cast<int64_t>(lane) * kGaPer;
  if (VEC) {
#pragma unroll
    for (int v = 0; v < kGaPer / 4; ++v) {
      float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
      if (o + 4 * v < n) {
        const float4* p = reinterpret_cast<const float4*>(row + o) + v;
        f = STREAM ? __ldcs(p) : *p;
      }
      x[4 * v] = f.x; x[4 * v + 1] = f.y; x[4 * v + 2] = f.z; x[4 * v + 3] = f.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < kGaPer; ++j) x[j] = o + j < n ? (STREAM ? __ldcs(row + o + j) : row[o + j]) : 0.f;
  }
}

template <bool VEC>
__device__ __forceinline__ void GaStore(float* row, int64_t n, int lane, const float (&x)[kGaPer]) {
  const int64_t o = static_cast<int64_t>(lane) * kGaPer;
  if (VEC) {
#pragma unroll
    for (int v = 0; v < kGaPer / 4; ++v) {
      if (o + 4 * v < n) {
        reinterpret_cast<float4*>(row + o)[v] = make_float4(x[4 * v], x[4 * v + 1], x[4 * v + 2], x[4 * v + 3]);
      }
    }
  } else {
#pragma unroll
    for (int j = 0; j < kGaPer; ++j) {
      if (o + j < n) row[o + j] = x[j];
    }
  }
}

// L2 prefetch of a run of n (<= kGaTile) floats: one 128-B line per lane
__device__ __forceinline__ void GaPrefetchL2(const float* p, int64_t n, int lane) {
  if (lane * 32 < n + 31) {
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p + (lane * 32 < n ? lane * 32 : n - 1)));
  }
}

// the rescaled and clipped gradient (get_grad_rescaled, :110-118), in place; the padding past the
// row's end stays +0.0f whatever rescale_grad is (0 * inf would be NaN)
__device__ __forceinline__ void GaRescale(const UpdateLaunch& a, int64_t n, int lane, float (&x)[kGaPer]) {
  const int64_t o = static_cast<int64_t>(lane) * kGaPer;
#pragma unroll
  for (int j = 0; j < kGaPer; ++j) {
    if (o + j < n) {
      x[j] = __fmul_rn(x[j], a.rescale);
      if (a.clip >= 0.f) x[j] = clipf(x[j], a.clip);
    }
  }
}

// continues the left fold `s` over one tile of n (> 0) elements; returns it in every lane
__device__ __forceinline__ float GaFold(float s, const float (&gr)[kGaPer], int64_t n) {
  const int lanes = n >= kGaTile ? 32 : static_cast<int>((n + kGaPer - 1) / kGaPer);
  for (int k = 0; k < lanes; ++k) {
    float t = s;  // only lane k's t is kept
#pragma unroll
    for (int j = 0; j < kGaPer; ++j) t = __fadd_rn(t, __fmul_rn(gr[j], gr[j]));
    s = __shfl_sync(0xffffffffu, t, k);
  }
  return s;
}

// w_j - (lr * gr_j) / den
__device__ __forceinline__ void GaStep(const UpdateLaunch& a, float den, const float (&gr)[kGaPer],
                                       float (&w)[kGaPer]) {
#pragma unroll
  for (int j = 0; j < kGaPer; ++j) w[j] = __fsub_rn(w[j], __fdiv_rn(__fmul_rn(a.lr, gr[j]), den));
}

// ONE_TILE (row_len <= kGaTile): the gradient row stays in registers between the fold and the
// update. Before the fold, the warp asks L2 for this row's weight and the next row's gradient
// (prefetches hold no registers), so the loads after the fold find them there. Longer rows read
// the gradient twice, tile by tile: once for the fold, once for the update.
template <bool VEC, bool ONE_TILE>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, ONE_TILE ? 4 : 3) rsp_group_adagrad_kernel(const UpdateLaunch a) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = static_cast<int64_t>(gridDim.x) * kWarpsPerBlock;
  const int64_t len = a.row_len;
  const float flen = static_cast<float>(len);  // ssq / row_length: float / (float)index_t
  const float* g = static_cast<const float*>(a.g);
  float* w = static_cast<float*>(a.out);
  float* h = a.s[0];
  int64_t r = static_cast<int64_t>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5);
  if (ONE_TILE) {
    for (; r < a.nnr; r += nwarps) {
      const int64_t row = a.gidx[r];
      float* wp = w + row * len;
      GaPrefetchL2(wp, len, lane);
      float gr[kGaPer], wv[kGaPer];
      GaLoad<VEC, true>(g + r * len, len, lane, gr);
      if (r + nwarps < a.nnr) GaPrefetchL2(g + (r + nwarps) * len, len, lane);
      const float h0 = h[row];
      GaRescale(a, len, lane, gr);
      const float hn = __fadd_rn(h0, __fdiv_rn(GaFold(0.f, gr, len), flen));
      GaLoad<VEC, false>(wp, len, lane, wv);
      GaStep(a, __fsqrt_rn(__fadd_rn(hn, a.eps)), gr, wv);
      GaStore<VEC>(wp, len, lane, wv);
      if (lane == 0) h[row] = hn;
    }
  } else {
    for (; r < a.nnr; r += nwarps) {
      const int64_t row = a.gidx[r];
      const float* gp = g + r * len;
      float* wp = w + row * len;
      float s = 0.f, x[kGaPer];
      for (int64_t b = 0; b < len; b += kGaTile) {
        GaLoad<VEC, true>(gp + b, len - b, lane, x);
        GaRescale(a, len - b, lane, x);
        s = GaFold(s, x, len - b);
      }
      const float hn = __fadd_rn(h[row], __fdiv_rn(s, flen));
      const float den = __fsqrt_rn(__fadd_rn(hn, a.eps));
      for (int64_t b = 0; b < len; b += kGaTile) {
        float wv[kGaPer];
        GaLoad<VEC, true>(gp + b, len - b, lane, x);
        GaLoad<VEC, false>(wp + b, len - b, lane, wv);
        GaRescale(a, len - b, lane, x);
        GaStep(a, den, x, wv);
        GaStore<VEC>(wp + b, len - b, lane, wv);
      }
      if (lane == 0) h[row] = hn;
    }
  }
}

__global__ void fill_row_ids_kernel(int64_t* ids, int64_t rows) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < rows; i += stride) {
    ids[i] = i;
  }
}

// ---------------------------------------------------------------------------------------------
// push: union + ordered sum

// ids outside [lo, hi) (a row-range shard merges only its own rows) become `sentinel`, which sorts
// behind every real id and forms one trailing segment that the sum kernel skips
__global__ void rsp_tag_kernel(RspSources s, int64_t lo, int64_t hi, int64_t sentinel, int64_t* keys,
                               uint32_t* vals) {
  const int64_t total = s.start[s.nsrc];
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int k = find_segment(s.start, s.nsrc, i);
    const int64_t id = s.idx[k][i - s.start[k]];
    keys[i] = (id >= lo && id < hi) ? id : sentinel;
    vals[i] = static_cast<uint32_t>(i);
  }
}

struct HeadPred {
  const int64_t* keys;
  __device__ __forceinline__ bool operator()(const uint32_t& i) const {
    return i == 0 || keys[i] != keys[i - 1];
  }
};

struct MergeSum {
  RspSources s;
  const int64_t* keys;   // sorted ids
  const uint32_t* vals;  // concatenation positions, source order inside equal ids
  const uint32_t* seg;   // segment starts
  const int64_t* d_nnr;
  int64_t* out_idx; float* out_val;  // the merged gradient (OPT < 0)
  int64_t row_len;
  RspUpdateLaunch u;                 // OPT >= 0: the lazy optimizer step consumes the sum in registers
  int64_t sentinel;                  // ids >= sentinel are out-of-shard fillers (0: none)
};

// OPT < 0: write the merged row_sparse gradient. OPT = kOptSGDSingle / kOptSGD / kOptAdam: the row
// sum never touches memory -- the same warp applies the lazy update to row `id` of w (+ state).
// One warp per union row. Lane j resolves the row pointer of the j-th contributing source (one
// parallel step instead of a per-source pointer chase) and parks it in shared memory; the row is
// then processed in tiles of 4 x 32 float4 so that every lane keeps 4 source loads (+ the weight /
// state loads of the tile) in flight.
// The row work shared by both union front-ends: `rows[0..cnt)` are the source rows of union row r
// (id `id`) in SOURCE ORDER.
template <int OPT>
__device__ __forceinline__ void rsp_sum_row(const MergeSum& p, const float* const* rows, int cnt,
                                            int64_t id, int64_t r, int lane) {
  Hyper h{p.u.lr, p.u.wd, p.u.momentum, p.u.rescale, p.u.clip, p.u.beta1, p.u.beta2, p.u.eps};
  float* out = OPT < 0 ? p.out_val + r * p.row_len : nullptr;
  float* w = OPT < 0 ? nullptr : p.u.w + id * p.row_len;
  float* s1 = (OPT == kOptSGD || OPT == kOptAdam) ? p.u.s1 + id * p.row_len : nullptr;
  float* s2 = OPT == kOptAdam ? p.u.s2 + id * p.row_len : nullptr;
  auto one = [&](float wv, float gv, float& a, float& c) -> float {
    if (OPT == kOptAdam) return step_adam_lazy(wv, gv, a, c, h);
    return step<(OPT < 0 ? kOptSGDSingle : OPT)>(wv, gv, a, c, OPT == kOptSGD, h);
  };
  bool vec = (p.row_len % 4 == 0);
  if (OPT < 0) {
    vec = vec && ((reinterpret_cast<uintptr_t>(p.out_val) & 15) == 0);
  } else {
    vec = vec && ((reinterpret_cast<uintptr_t>(p.u.w) & 15) == 0) &&
          (!p.u.s1 || (reinterpret_cast<uintptr_t>(p.u.s1) & 15) == 0) &&
          (!p.u.s2 || (reinterpret_cast<uintptr_t>(p.u.s2) & 15) == 0);
  }
  for (int k = 0; k < p.s.nsrc; ++k) vec = vec && ((reinterpret_cast<uintptr_t>(p.s.val[k]) & 15) == 0);
  if (vec) {
    constexpr int U = 4;
    const int64_t nv = p.row_len / 4;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int64_t v0 = lane; v0 < nv; v0 += 32 * U) {
      float4 wv[U], a[U], c[U], acc[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t v = v0 + 32 * u;
        acc[u] = zero; wv[u] = zero; a[u] = zero; c[u] = zero;
        if (v < nv) {
          if (OPT >= 0) wv[u] = reinterpret_cast<const float4*>(w)[v];
          if (OPT == kOptSGD || OPT == kOptAdam) a[u] = reinterpret_cast<const float4*>(s1)[v];
          if (OPT == kOptAdam) c[u] = reinterpret_cast<const float4*>(s2)[v];
        }
      }
      for (int j = 0; j < cnt; ++j) {
        const float4* row = reinterpret_cast<const float4*>(rows[j]);
        float4 x[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t v = v0 + 32 * u;
          x[u] = v < nv ? __ldcs(row + v) : zero;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          acc[u].x = __fadd_rn(acc[u].x, x[u].x); acc[u].y = __fadd_rn(acc[u].y, x[u].y);
          acc[u].z = __fadd_rn(acc[u].z, x[u].z); acc[u].w = __fadd_rn(acc[u].w, x[u].w);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t v = v0 + 32 * u;
        if (v >= nv) continue;
        if (OPT < 0) {
          reinterpret_cast<float4*>(out)[v] = acc[u];
        } else {
          wv[u].x = one(wv[u].x, acc[u].x, a[u].x, c[u].x);
          wv[u].y = one(wv[u].y, acc[u].y, a[u].y, c[u].y);
          wv[u].z = one(wv[u].z, acc[u].z, a[u].z, c[u].z);
          wv[u].w = one(wv[u].w, acc[u].w, a[u].w, c[u].w);
          reinterpret_cast<float4*>(w)[v] = wv[u];
          if (OPT == kOptSGD || OPT == kOptAdam) reinterpret_cast<float4*>(s1)[v] = a[u];
          if (OPT == kOptAdam) reinterpret_cast<float4*>(s2)[v] = c[u];
        }
      }
    }
  } else {
    for (int64_t col = lane; col < p.row_len; col += 32) {
      float acc = 0.f;
      for (int j = 0; j < cnt; ++j) acc = __fadd_rn(acc, rows[j][col]);
      if (OPT < 0) {
        out[col] = acc;
      } else {
        float a = 0.f, c = 0.f;
        if (OPT == kOptSGD || OPT == kOptAdam) a = s1[col];
        if (OPT == kOptAdam) c = s2[col];
        w[col] = one(w[col], acc, a, c);
        if (OPT == kOptSGD || OPT == kOptAdam) s1[col] = a;
        if (OPT == kOptAdam) s2[col] = c;
      }
    }
  }
}

template <int OPT>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) rsp_sum_kernel(MergeSum p) {
  __shared__ const float* s_rows[kWarpsPerBlock][kMaxSrc];
  const int warp = threadIdx.x >> 5;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kWarpsPerBlock + warp;
  const int64_t nnr = *p.d_nnr;
  if (r >= nnr) return;
  const int lane = threadIdx.x & 31;
  const int64_t total = p.s.start[p.s.nsrc];
  const uint32_t b = p.seg[r];
  const uint32_t e = r + 1 < nnr ? p.seg[r + 1] : static_cast<uint32_t>(total);
  const int64_t id = p.keys[b];
  if (p.sentinel != 0 && id >= p.sentinel) return;  // the out-of-shard filler segment
  if (OPT < 0 && lane == 0) p.out_idx[r] = id;
  // this row's sources, in source order; a row_sparse array holds an id at most once, so there
  // are at most nsrc <= kMaxSrc of them (anything beyond is a malformed input and is ignored)
  const int cnt = min(static_cast<int>(e - b), kMaxSrc);
  if (lane < cnt) {
    const int64_t pos = p.vals[b + lane];
    const int k = find_segment(p.s.start, p.s.nsrc, pos);
    s_rows[warp][lane] = p.s.val[k] + (pos - p.s.start[k]) * p.row_len;
  }
  __syncwarp();
  rsp_sum_row<OPT>(p, s_rows[warp], cnt, id, r, lane);
}


// ---------------------------------------------------------------------------------------------
// Bitmap union: the ids of a push (or the requested ids of a pull) are marked in a bitmap over the
// table's row range, a popcount prefix over the bitmap ranks them, and every id finds its place in
// the ascending unique union with two loads -- no sort. 1 M rows = 31 250 words: the bitmap and
// its prefix stay in L2 and the whole bookkeeping of a push is three launches of a few
// microseconds (mark, scan, scatter) where the radix sort of (id, position) pairs took nine
// (histogram, 3 x onesweep, select ...), which took longer than half of the row traffic's time. Tables taller than kBitmapMaxWords*32 rows keep the sort path.
constexpr int64_t kBitmapMaxWords = int64_t{1} << 18;   // per group: 8 M rows
constexpr int64_t kBitmapMaxTotalWords = int64_t{1} << 22;
constexpr int kScanThreads = 1024;

// B200KV_RSP_SORT=1 forces the radix-sort union (read per call so tests can cover both paths)
bool BitmapDisabled() {
  const char* z = std::getenv("B200KV_RSP_SORT");
  return z != nullptr && z[0] != '\0' && z[0] != '0';
}

__global__ void bm_mark_push_kernel(RspSources s, int64_t lo, int64_t hi, uint32_t* bitmap,
                                    uint32_t* srcpos, int64_t table_words) {
  const int64_t total = s.start[s.nsrc];
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = tid; i < total; i += nth) {
    const int k = find_segment(s.start, s.nsrc, i);
    const int64_t id = s.idx[k][i - s.start[k]];
    if (id >= lo && id < hi) {
      const int64_t r = id - lo;
      atomicOr(&bitmap[r >> 5], 1u << (r & 31));
    }
  }
  for (int64_t j = tid; j < table_words; j += nth) srcpos[j] = 0u;   // source table of the union rows
}

// Rank of every bitmap word. Grid (blocks of 1024 words, groups): each CTA scans the popcounts of
// its 1024 words (one word per thread) -> prefix[w] = set bits before w INSIDE the block, and
// publishes the block's total; the last CTA of a group to finish turns the totals into exclusive
// block bases and writes the group's count. rank(word w) = block_base[w / 1024] + prefix[w].
constexpr int kScanBlock = kScanThreads;

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t c, uint32_t* wsum, uint32_t* total) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t incl = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const uint32_t v = wsum[lane];
    uint32_t wi = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    wsum[lane] = wi - v;
    if (lane == 31) *total = wi;
  }
  __syncthreads();
  const uint32_t excl = wsum[warp] + incl - c;
  __syncthreads();   // wsum is reused by the caller's next round
  return excl;
}

__global__ void __launch_bounds__(kScanThreads) bm_scan_kernel(const uint32_t* bitmap, int64_t nwords,
                                                               int nblocks, uint32_t* prefix,
                                                               uint32_t* block_base, uint32_t* done,
                                                               int64_t* d_count) {
  __shared__ uint32_t wsum[32];
  __shared__ uint32_t s_total, s_last;
  const int g = blockIdx.y;
  const int64_t w = static_cast<int64_t>(blockIdx.x) * kScanBlock + threadIdx.x;
  const uint32_t c = w < nwords ? __popc(bitmap[g * nwords + w]) : 0u;
  const uint32_t excl = block_exclusive_scan(c, wsum, &s_total);
  if (w < nwords) prefix[g * nwords + w] = excl;
  if (threadIdx.x == 0) {
    block_base[static_cast<int64_t>(g) * nblocks + blockIdx.x] = s_total;
    __threadfence();
    s_last = (atomicAdd(&done[g], 1u) == static_cast<uint32_t>(nblocks) - 1u) ? 1u : 0u;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  uint32_t running = 0;
  uint32_t* bb = block_base + static_cast<int64_t>(g) * nblocks;
  for (int b0 = 0; b0 < nblocks; b0 += kScanBlock) {
    const int i = b0 + threadIdx.x;
    const uint32_t v = i < nblocks ? __ldcg(bb + i) : 0u;
    const uint32_t e = block_exclusive_scan(v, wsum, &s_total);
    if (i < nblocks) bb[i] = running + e;
    running += s_total;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    d_count[g] = running;
    done[g] = 0;   // ready for the next call (the memset of the bitmap covers it as well)
  }
}

// every (source, position) pair finds its union row: uid[u] = id, srcpos[u][k] = position + 1
__global__ void bm_scatter_push_kernel(RspSources s, int64_t lo, int64_t hi, const uint32_t* bitmap,
                                       const uint32_t* prefix, const uint32_t* block_base, int64_t* uid,
                                       uint32_t* srcpos) {
  const int64_t total = s.start[s.nsrc];
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int k = find_segment(s.start, s.nsrc, i);
    const int64_t id = s.idx[k][i - s.start[k]];
    if (id < lo || id >= hi) continue;
    const int64_t r = id - lo;
    const uint32_t word = bitmap[r >> 5];
    const uint32_t u = block_base[r >> 15] + prefix[r >> 5] + __popc(word & ((1u << (r & 31)) - 1u));
    uid[u] = id;
    srcpos[static_cast<int64_t>(u) * s.nsrc + k] = static_cast<uint32_t>(i - s.start[k]) + 1u;
  }
}

struct MergeSumBm {
  MergeSum m;              // sources, outputs, fused update (keys / vals / seg unused)
  const int64_t* uid;      // union ids, ascending
  const uint32_t* srcpos;  // [union row][source] -> position + 1, 0 = the source lacks the row
};

// Persistent warps over the union rows. The bookkeeping of the NEXT row (its id and source
// positions: two independent loads) is fetched before the current row's data is touched, so a
// warp's dependent chain is just row pointer -> row data.
template <int OPT>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) rsp_sum_bm_kernel(MergeSumBm q) {
  __shared__ const float* s_rows[kWarpsPerBlock][kMaxSrc];
  const MergeSum& p = q.m;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t nnr = *p.d_nnr;
  const int64_t nwarps = static_cast<int64_t>(gridDim.x) * kWarpsPerBlock;
  const int nsrc = p.s.nsrc;
  int64_t r = static_cast<int64_t>(blockIdx.x) * kWarpsPerBlock + warp;
  int64_t id = 0;
  uint32_t pos = 0;
  if (r < nnr) {
    id = q.uid[r];
    pos = lane < nsrc ? q.srcpos[r * nsrc + lane] : 0u;
  }
  while (r < nnr) {
    const int64_t rn = r + nwarps;
    int64_t id_n = 0;
    uint32_t pos_n = 0;
    if (rn < nnr) {
      id_n = q.uid[rn];
      pos_n = lane < nsrc ? q.srcpos[rn * nsrc + lane] : 0u;
    }
    const uint32_t mask = __ballot_sync(0xffffffffu, pos != 0u);
    if (pos != 0u) {
      s_rows[warp][__popc(mask & ((1u << lane) - 1u))] =
          p.s.val[lane] + static_cast<int64_t>(pos - 1u) * p.row_len;
    }
    __syncwarp();
    if (OPT < 0 && lane == 0) p.out_idx[r] = id;
    rsp_sum_row<OPT>(p, s_rows[warp], __popc(mask), id, r, lane);
    __syncwarp();
    r = rn;
    id = id_n;
    pos = pos_n;
  }
}

// ---- pull: per item one bitmap; ids of any integer / float dtype
__device__ __forceinline__ int64_t load_id(const void* ids, int dtype, int64_t i);
__device__ __forceinline__ int find_item(const RetainItem* items, int nitems, int64_t i);

__global__ void bm_mark_pull_kernel(const RetainItem* items, int nitems, int64_t total, int64_t nwords,
                                    uint32_t* bitmap) {
  const int64_t cap = nwords * 32;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int k = find_item(items, nitems, i);
    const int64_t id = load_id(items[k].ids, items[k].ids_dtype, i - items[k].start);
    if (id >= 0 && id < cap) atomicOr(&bitmap[k * nwords + (id >> 5)], 1u << (id & 31));
  }
}

constexpr int kBmMaxItems = 1024;
// uniq[off[k] + j] = j-th smallest requested id of item k; off[] = prefix of the items' counts
__global__ void bm_emit_pull_kernel(const uint32_t* bitmap, const uint32_t* prefix,
                                    const uint32_t* block_base, int nblocks, const int64_t* count,
                                    int nitems, int64_t nwords, int64_t* uniq, int64_t* off) {
  __shared__ int64_t s_off[kBmMaxItems + 1];
  if (threadIdx.x == 0) {
    int64_t acc = 0;
    for (int k = 0; k < nitems; ++k) { s_off[k] = acc; acc += count[k]; }
    s_off[nitems] = acc;
  }
  __syncthreads();
  if (blockIdx.x == 0) {
    for (int k = threadIdx.x; k <= nitems; k += blockDim.x) off[k] = s_off[k];
  }
  const int64_t all = nwords * nitems;
  for (int64_t j = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; j < all;
       j += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    uint32_t word = bitmap[j];
    if (word == 0u) continue;
    const int k = static_cast<int>(j / nwords);
    const int64_t w = j - k * nwords;
    int64_t* dst = uniq + s_off[k] + block_base[static_cast<int64_t>(k) * nblocks + (w >> 10)] + prefix[j];
    while (word) {
      const int b = __ffs(word) - 1;
      *dst++ = (w << 5) + b;
      word &= word - 1u;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// the row map of a row_sparse gradient for the updates that move EVERY table row
// (update_rsp_grad_kernels.cu): row_map[r] = position of row r in the gradient, or -1

__global__ void row_map_scatter_kernel(const int64_t* gidx, int64_t nnr, int32_t* row_map) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nnr;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    row_map[gidx[i]] = static_cast<int32_t>(i);
  }
}

// ---------------------------------------------------------------------------------------------
// storage casts (src/operator/tensor/cast_storage-inl.h:74-140): dense -> row_sparse keeps the
// rows with any element != 0; row_sparse -> dense scatters the rows over zeros

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
row_nonzero_flag_kernel(const float* data, int64_t rows, int64_t row_len, uint8_t* flags) {
  const int64_t row = static_cast<int64_t>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* r = data + row * row_len;
  bool any = false;
  for (int64_t j = lane; j < row_len; j += 32) any = any || (r[j] != 0.f);
  any = __any_sync(0xffffffffu, any);
  if (lane == 0) flags[row] = any ? 1 : 0;
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
rsp_scatter_rows_kernel(const int64_t* idx, const float* val, int64_t nnr, int64_t row_len, float* dense) {
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5);
  if (r >= nnr) return;
  const int lane = threadIdx.x & 31;
  const float* src = val + r * row_len;
  float* dst = dense + idx[r] * row_len;
  for (int64_t j = lane; j < row_len; j += 32) dst[j] = src[j];
}

struct MergeLayout {
  size_t keys, keys_sorted, vals, vals_sorted, seg, temp, temp_bytes, total;
};

// workspace of the bitmap union of a push: bitmap + prefix over the row range, union ids, source table
struct BmMergeLayout {
  bool ok = false;
  int64_t nwords = 0;
  int nblocks = 0;
  size_t bitmap = 0, done = 0, prefix = 0, block_base = 0, uid = 0, srcpos = 0, total = 0;
  size_t zero_bytes = 0;   // bitmap + done counter: cleared before every use
};

BmMergeLayout LayoutMergeBm(int64_t n, int id_bits, int nsrc, int64_t lo, int64_t hi) {
  auto up = [](size_t b) { return (b + 255) & ~static_cast<size_t>(255); };
  BmMergeLayout l;
  if (BitmapDisabled() || id_bits < 1 || id_bits > 40) return l;
  const int64_t top = std::min(hi, int64_t{1} << id_bits);
  if (top <= lo) return l;
  l.nwords = (top - lo + 31) / 32;
  if (l.nwords > kBitmapMaxWords) return l;
  l.ok = true;
  l.nblocks = static_cast<int>((l.nwords + kScanBlock - 1) / kScanBlock);
  l.bitmap = 0;
  l.done = up(static_cast<size_t>(l.nwords) * 4);
  l.zero_bytes = l.done + 256;
  l.prefix = l.zero_bytes;
  l.block_base = l.prefix + up(static_cast<size_t>(l.nwords) * 4);
  l.uid = l.block_base + up(static_cast<size_t>(l.nblocks) * 4);
  l.srcpos = l.uid + up(static_cast<size_t>(n) * 8);
  l.total = l.srcpos + up(static_cast<size_t>(n) * std::max(nsrc, 1) * 4) + 256;
  return l;
}

MergeLayout LayoutMerge(int64_t n) {
  auto up = [](size_t b) { return (b + 255) & ~static_cast<size_t>(255); };
  MergeLayout l;
  const size_t k = up(static_cast<size_t>(n) * sizeof(int64_t));
  const size_t v = up(static_cast<size_t>(n) * sizeof(uint32_t));
  size_t t1 = 0, t2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t1, static_cast<const int64_t*>(nullptr),
                                  static_cast<int64_t*>(nullptr), static_cast<const uint32_t*>(nullptr),
                                  static_cast<uint32_t*>(nullptr), static_cast<int>(n));
  cub::DeviceSelect::If(nullptr, t2, cub::CountingInputIterator<uint32_t>(0),
                        static_cast<uint32_t*>(nullptr), static_cast<int64_t*>(nullptr),
                        static_cast<int>(n), HeadPred{nullptr});
  l.keys = 0;
  l.keys_sorted = k;
  l.vals = 2 * k;
  l.vals_sorted = 2 * k + v;
  l.seg = 2 * k + 2 * v;
  l.temp = 2 * k + 3 * v;
  l.temp_bytes = up(std::max(t1, t2));
  l.total = l.temp + l.temp_bytes + 256;
  return l;
}

// ---------------------------------------------------------------------------------------------
// pull: batched unique + retain

__device__ __forceinline__ int64_t load_id(const void* ids, int dtype, int64_t i) {
  switch (dtype) {
    case kInt64: return static_cast<const int64_t*>(ids)[i];
    case kInt32: return static_cast<const int32_t*>(ids)[i];
    case kFloat32: return static_cast<int64_t>(static_cast<const float*>(ids)[i]);
    case kFloat64: return static_cast<int64_t>(static_cast<const double*>(ids)[i]);
    case kUint8: return static_cast<const uint8_t*>(ids)[i];
    case kInt8: return static_cast<const int8_t*>(ids)[i];
    case kFloat16: return static_cast<int64_t>(__half2float(static_cast<const __half*>(ids)[i]));
    default: return 0;
  }
}

__device__ __forceinline__ int find_item(const RetainItem* items, int nitems, int64_t i) {
  int lo = 0, hi = nitems - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (items[mid].start <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void retain_gather_kernel(const RetainItem* items, int nitems, int64_t total, int id_bits,
                                     int64_t* comp) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int k = find_item(items, nitems, i);
    const int64_t id = load_id(items[k].ids, items[k].ids_dtype, i - items[k].start);
    comp[i] = (static_cast<int64_t>(k) << id_bits) | id;
  }
}

__global__ void retain_bounds_kernel(const int64_t* uniq, const int64_t* d_count, int nitems,
                                     int id_bits, int64_t* off) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > nitems) return;
  const int64_t n = *d_count;
  if (k == nitems) { off[k] = n; return; }
  const int64_t key = static_cast<int64_t>(k) << id_bits;
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (uniq[mid] < key) lo = mid + 1; else hi = mid;
  }
  off[k] = lo;
}

// Persistent warps over the (item, unique id) rows of the batch. A row's bookkeeping (which item,
// which id: three dependent loads) is fetched for the NEXT row before the current row is copied, so
// the copy loop never waits for it.
struct RetainRow {
  int k;         // item, -1: past the item's unique count (nothing to do)
  int64_t j;     // position among the item's unique ids
  int64_t id;
};

__device__ __forceinline__ RetainRow retain_fetch(const RetainItem* items, int nitems, int64_t i,
                                                 int64_t total, int id_bits, const int64_t* uniq,
                                                 const int64_t* off) {
  RetainRow r{-1, 0, 0};
  if (i >= total) return r;
  const int k = find_item(items, nitems, i);
  const int64_t j = i - items[k].start;
  const int64_t o = off[k];
  if (j >= off[k + 1] - o) return r;
  r.k = k;
  r.j = j;
  r.id = uniq[o + j] & ((int64_t{1} << id_bits) - 1);
  return r;
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
retain_kernel(const RetainItem* items, int nitems, int64_t total, int id_bits, const int64_t* uniq,
              const int64_t* off) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = static_cast<int64_t>(gridDim.x) * kWarpsPerBlock;
  int64_t i = static_cast<int64_t>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5);
  RetainRow cur = retain_fetch(items, nitems, i, total, id_bits, uniq, off);
  while (i < total) {
    const RetainRow nxt = retain_fetch(items, nitems, i + nwarps, total, id_bits, uniq, off);
    if (cur.k >= 0) {
      const RetainItem it = items[cur.k];
      const int64_t id = cur.id;
      if (lane == 0) it.out_idx[cur.j] = id;
      int64_t srow = -1;
      const float* src_base = it.src_val;
      if (it.shard_vbase != nullptr) {
        // the table is cut into row ranges over several GPUs: vbase[d] + id*row_len is row `id`
        src_base = it.shard_vbase[id / it.rows_per_shard];
        srow = id;
      } else if (it.src_dense_rows) {
        srow = id;
      } else if (it.src_nnr > 0) {
        const int64_t lb = warp_lower_bound(it.src_idx, it.src_nnr, id, lane);
        if (lb < it.src_nnr && it.src_idx[lb] == id) srow = lb;
      }
      float* out = it.out_val + cur.j * it.row_len;
      const float* src = srow >= 0 ? src_base + srow * it.row_len : nullptr;
      const bool vec = (it.row_len % 4 == 0) && ((reinterpret_cast<uintptr_t>(it.out_val) & 15) == 0) &&
                       ((reinterpret_cast<uintptr_t>(src_base) & 15) == 0);
      if (vec) {
        const int64_t nv = it.row_len / 4;
        const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int64_t v0 = lane; v0 < nv; v0 += 128) {   // 4 x 16 bytes in flight per lane
          float4 x[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int64_t v = v0 + 32 * u;
            x[u] = (src && v < nv) ? __ldcs(reinterpret_cast<const float4*>(src) + v) : zero;
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int64_t v = v0 + 32 * u;
            if (v < nv) __stcs(reinterpret_cast<float4*>(out) + v, x[u]);
          }
        }
      } else {
        for (int64_t c = lane; c < it.row_len; c += 32) out[c] = src ? src[c] : 0.f;
      }
    }
    cur = nxt;
    i += nwarps;
  }
}

// ---------------------------------------------------------------------------------------------
// whole-value pull of a row_sparse value: every target in one pass (see LaunchRspBroadcast)

// One row to every target: `src` (null: a row the value does not hold) is read once, in units of
// T, 4 units in flight per lane; dense targets get it (or zeros) at table row `row`, row_sparse
// targets at position `pos` (< 0: none).
template <typename T>
__device__ __forceinline__ void bcast_row(const RspBroadcastLaunch& p, const T* src, int64_t row, int64_t pos,
                                          int lane) {
  const int64_t nu = p.row_bytes / static_cast<int64_t>(sizeof(T));
  for (int64_t v0 = lane; v0 < nu; v0 += 128) {
    T x[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int64_t v = v0 + 32 * u;
      x[u] = (src != nullptr && v < nu) ? src[v] : T{};
    }
    for (int t = 0; t < p.n_dns; ++t) {
      T* out = reinterpret_cast<T*>(static_cast<char*>(p.dns[t]) + row * p.row_bytes);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (v0 + 32 * u < nu) out[v0 + 32 * u] = x[u];
      }
    }
    if (pos >= 0) {
      for (int t = 0; t < p.n_rsp; ++t) {
        T* out = reinterpret_cast<T*>(static_cast<char*>(p.rsp_val[t]) + pos * p.row_bytes);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (v0 + 32 * u < nu) out[v0 + 32 * u] = x[u];
        }
      }
    }
  }
  if (pos >= 0 && lane < p.n_rsp) p.rsp_idx[lane][pos] = row;
}

// Persistent warps, each over a contiguous range of the domain: the table's rows when a dense
// target is present (one lower bound finds the range's first stored row, then the warp walks the
// ids alongside the rows), else the stored rows. The id of the next stored row is loaded before
// the current row is copied, so the copy never waits for it.
template <typename T>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
rsp_broadcast_kernel(const __grid_constant__ RspBroadcastLaunch p) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = static_cast<int64_t>(gridDim.x) * kWarpsPerBlock;
  const int64_t warp = static_cast<int64_t>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5);
  const bool dense = p.n_dns > 0;
  const int64_t domain = dense ? p.rows : p.nnr;
  const int64_t per = (domain + nwarps - 1) / nwarps;
  const int64_t lo = warp * per, hi = min(domain, lo + per);
  if (lo >= hi) return;
  const T* val = static_cast<const T*>(p.src_val);
  const int64_t row_units = p.row_bytes / static_cast<int64_t>(sizeof(T));
  int64_t pos = dense ? warp_lower_bound(p.src_idx, p.nnr, lo, lane) : lo;
  int64_t next = pos < p.nnr ? p.src_idx[pos] : INT64_MAX;
  for (int64_t i = lo; i < hi; ++i) {
    const int64_t row = dense ? i : next;
    if (row == next) {
      const int64_t cur = pos++;
      next = pos < p.nnr ? p.src_idx[pos] : INT64_MAX;
      bcast_row<T>(p, val + cur * row_units, row, cur, lane);
    } else {
      bcast_row<T>(p, static_cast<const T*>(nullptr), row, -1, lane);
    }
  }
}

struct RetainLayout {
  size_t items, comp, sorted, uniq, count, temp, temp_bytes, total;
  // bitmap unique (id_bits > 0 and the table is short enough): bitmap + prefix per item live in the
  // region the sort path uses for its keys and temporaries
  bool bm = false;
  int64_t nwords = 0;
  int nblocks = 0;
  size_t bm_bitmap = 0, bm_done = 0, bm_zero_bytes = 0, bm_prefix = 0, bm_block_base = 0;
};

RetainLayout LayoutRetain(int nitems, int64_t n, int id_bits = 0) {
  auto up = [](size_t b) { return (b + 255) & ~static_cast<size_t>(255); };
  RetainLayout l;
  const size_t k = up(static_cast<size_t>(n) * sizeof(int64_t));
  size_t t1 = 0, t2 = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, t1, static_cast<const int64_t*>(nullptr),
                                 static_cast<int64_t*>(nullptr), static_cast<int>(n));
  cub::DeviceSelect::Unique(nullptr, t2, static_cast<const int64_t*>(nullptr),
                            static_cast<int64_t*>(nullptr), static_cast<int64_t*>(nullptr),
                            static_cast<int>(n));
  l.items = 0;
  l.comp = up(static_cast<size_t>(nitems) * sizeof(RetainItem));
  l.sorted = l.comp + k;
  l.uniq = l.sorted + k;
  l.count = l.uniq + k;
  l.temp = l.count + up(static_cast<size_t>(nitems + 1) * sizeof(int64_t));
  l.temp_bytes = up(std::max(t1, t2));
  l.total = l.temp + l.temp_bytes + 256;
  if (id_bits >= 1 && id_bits <= 40 && !BitmapDisabled() && nitems <= kBmMaxItems) {
    const int64_t nwords = ((int64_t{1} << id_bits) + 31) / 32;
    if (nwords <= kBitmapMaxWords && nwords * nitems <= kBitmapMaxTotalWords) {
      l.bm = true;
      l.nwords = nwords;
      l.nblocks = static_cast<int>((nwords + kScanBlock - 1) / kScanBlock);
      const size_t bytes = up(static_cast<size_t>(nwords) * nitems * 4);
      l.bm_bitmap = l.temp;
      l.bm_done = l.bm_bitmap + bytes;
      l.bm_zero_bytes = bytes + up(static_cast<size_t>(nitems) * 4);
      l.bm_prefix = l.bm_bitmap + l.bm_zero_bytes;
      l.bm_block_base = l.bm_prefix + bytes;
      l.total = std::max(l.total, l.bm_block_base + up(static_cast<size_t>(l.nblocks) * nitems * 4) + 256);
    }
  }
  return l;
}

int GridFor(int64_t n, int threads) {
  return static_cast<int>(std::min<int64_t>((n + threads - 1) / threads, kNumSMs * 8));
}

}  // namespace

void LaunchRspRowUpdateOp(const UpdateLaunch& L, cudaStream_t stream) {
  if (L.nnr <= 0 || L.row_len <= 0) return;
  KV_CHECK_EQ(L.dtype, kFloat32) << "row_sparse optimizer operators run on float32 arrays";
  KV_CHECK(L.out == L.w) << "row_sparse optimizer operators update the weight in place";
  auto aligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  bool vec = L.row_len % 4 == 0 && aligned(L.g) && aligned(L.out);
  const int blocks = static_cast<int>(std::min<int64_t>((L.nnr + kWarpsPerBlock - 1) / kWarpsPerBlock,
                                                        kNumSMs * 16));
  if (L.op == kUpdGroupAdaGrad) {  // one history value per row: only g and w move along the row
    const dim3 grid(blocks), block(kWarpsPerBlock * 32);
    if (L.row_len <= kGaTile) {
      if (vec) rsp_group_adagrad_kernel<true, true><<<grid, block, 0, stream>>>(L);
      else rsp_group_adagrad_kernel<false, true><<<grid, block, 0, stream>>>(L);
    } else {
      if (vec) rsp_group_adagrad_kernel<true, false><<<grid, block, 0, stream>>>(L);
      else rsp_group_adagrad_kernel<false, false><<<grid, block, 0, stream>>>(L);
    }
    KV_CUDA(cudaGetLastError());
    return;
  }
  for (int k = 0; k < NumStates(L.op); ++k) vec = vec && aligned(L.s[k]);
  // one warp per gradient row: CTAs that retire are replaced until the last row, where a capped
  // grid of 40-56-register CTAs (6 or fewer resident per SM) leaves its last wave part empty
  const int row_blocks = static_cast<int>((L.nnr + kWarpsPerBlock - 1) / kWarpsPerBlock);
  switch (L.op) {
    case kUpdFtrl: rsp_row_update_kernel<kUpdFtrl><<<row_blocks, kWarpsPerBlock * 32, 0, stream>>>(L, vec); break;
    case kUpdAdaGrad: rsp_row_update_kernel<kUpdAdaGrad><<<row_blocks, kWarpsPerBlock * 32, 0, stream>>>(L, vec); break;
    case kUpdSGD: rsp_row_update_kernel<kUpdSGD><<<row_blocks, kWarpsPerBlock * 32, 0, stream>>>(L, vec); break;
    case kUpdSGDMom: rsp_row_update_kernel<kUpdSGDMom><<<row_blocks, kWarpsPerBlock * 32, 0, stream>>>(L, vec); break;
    case kUpdAdamLazy: rsp_row_update_kernel<kUpdAdamLazy><<<row_blocks, kWarpsPerBlock * 32, 0, stream>>>(L, vec); break;
    default: KV_FATAL << "row_sparse optimizer operator: unsupported operator " << L.op;
  }
  KV_CUDA(cudaGetLastError());
}

void LaunchFillRowIds(int64_t* ids, int64_t rows, cudaStream_t stream) {
  if (rows <= 0) return;
  fill_row_ids_kernel<<<GridFor(rows, 256), 256, 0, stream>>>(ids, rows);
  KV_CUDA(cudaGetLastError());
}

size_t RspMergeWorkspaceBytes(int64_t total_ids, int id_bits, int nsrc, int64_t lo, int64_t hi) {
  const int64_t n = std::max<int64_t>(total_ids, 1);
  const BmMergeLayout b = LayoutMergeBm(n, id_bits, nsrc, lo, hi);
  return b.ok ? b.total : LayoutMerge(n).total;
}

void LaunchRspMerge(const RspSources& srcs, int id_bits, int64_t row_len, int64_t* out_idx,
                    float* out_val, int64_t* d_nnr, void* workspace, size_t workspace_bytes,
                    cudaStream_t stream, const RspUpdateLaunch* fused_update, int64_t lo, int64_t hi) {
  const int64_t total = srcs.start[srcs.nsrc];
  KV_CHECK(srcs.nsrc >= 1 && srcs.nsrc <= kMaxSrc);
  KV_CHECK(total > 0 && total < (1LL << 31)) << "row_sparse push: " << total << " row ids";
  KV_CHECK(id_bits >= 1 && id_bits <= 63);
  char* ws = static_cast<char*>(workspace);
  const BmMergeLayout bl = LayoutMergeBm(total, id_bits, srcs.nsrc, lo, hi);
  if (bl.ok) {
    // ---- bitmap union: mark, scan, scatter, then persistent warps over the union rows
    KV_CHECK(workspace_bytes >= bl.total) << "rsp merge: workspace too small";
    const int64_t top = std::min(hi, int64_t{1} << id_bits);
    uint32_t* bitmap = reinterpret_cast<uint32_t*>(ws + bl.bitmap);
    uint32_t* prefix = reinterpret_cast<uint32_t*>(ws + bl.prefix);
    int64_t* uid = reinterpret_cast<int64_t*>(ws + bl.uid);
    uint32_t* srcpos = reinterpret_cast<uint32_t*>(ws + bl.srcpos);
    uint32_t* block_base = reinterpret_cast<uint32_t*>(ws + bl.block_base);
    uint32_t* done = reinterpret_cast<uint32_t*>(ws + bl.done);
    KV_CUDA(cudaMemsetAsync(bitmap, 0, bl.zero_bytes, stream));
    const int64_t table_words = total * srcs.nsrc;
    bm_mark_push_kernel<<<GridFor(std::max(total, table_words / 4), 256), 256, 0, stream>>>(
        srcs, lo, top, bitmap, srcpos, table_words);
    bm_scan_kernel<<<dim3(bl.nblocks, 1), kScanThreads, 0, stream>>>(bitmap, bl.nwords, bl.nblocks, prefix,
                                                                       block_base, done, d_nnr);
    bm_scatter_push_kernel<<<GridFor(total, 256), 256, 0, stream>>>(srcs, lo, top, bitmap, prefix, block_base,
                                                                     uid, srcpos);
    KV_CUDA(cudaGetLastError());
    if (row_len <= 0) return;
    MergeSumBm q;
    q.m = MergeSum{srcs, nullptr, nullptr, nullptr, d_nnr, out_idx, out_val, row_len, RspUpdateLaunch(), 0};
    q.uid = uid;
    q.srcpos = srcpos;
    const int threads = kWarpsPerBlock * 32;
    const int blocks = static_cast<int>(std::min<int64_t>((total + kWarpsPerBlock - 1) / kWarpsPerBlock, kNumSMs * 6));
    if (fused_update == nullptr) {
      rsp_sum_bm_kernel<-1><<<blocks, threads, 0, stream>>>(q);
    } else {
      q.m.u = *fused_update;
      switch (q.m.u.opt) {
        case kOptSGDSingle: rsp_sum_bm_kernel<kOptSGDSingle><<<blocks, threads, 0, stream>>>(q); break;
        case kOptSGD: rsp_sum_bm_kernel<kOptSGD><<<blocks, threads, 0, stream>>>(q); break;
        case kOptAdam: rsp_sum_bm_kernel<kOptAdam><<<blocks, threads, 0, stream>>>(q); break;
        default: KV_FATAL << "row_sparse push: unsupported optimizer kind " << q.m.u.opt;
      }
    }
    KV_CUDA(cudaGetLastError());
    return;
  }
  const MergeLayout l = LayoutMerge(total);
  KV_CHECK(workspace_bytes >= l.total) << "rsp merge: workspace too small";
  int64_t* keys = reinterpret_cast<int64_t*>(ws + l.keys);
  int64_t* keys_sorted = reinterpret_cast<int64_t*>(ws + l.keys_sorted);
  uint32_t* vals = reinterpret_cast<uint32_t*>(ws + l.vals);
  uint32_t* vals_sorted = reinterpret_cast<uint32_t*>(ws + l.vals_sorted);
  uint32_t* seg = reinterpret_cast<uint32_t*>(ws + l.seg);
  const bool ranged = lo > 0 || hi < (int64_t{1} << id_bits);
  KV_CHECK(!ranged || fused_update != nullptr) << "row-range merges feed a fused update";
  const int64_t sentinel = ranged ? (int64_t{1} << id_bits) : 0;
  rsp_tag_kernel<<<GridFor(total, 256), 256, 0, stream>>>(srcs, lo, hi, sentinel, keys, vals);
  KV_CUDA(cudaGetLastError());
  size_t tb = l.temp_bytes;
  KV_CUDA(cub::DeviceRadixSort::SortPairs(ws + l.temp, tb, keys, keys_sorted, vals, vals_sorted,
                                          static_cast<int>(total), 0, id_bits + (ranged ? 1 : 0), stream));
  tb = l.temp_bytes;
  KV_CUDA(cub::DeviceSelect::If(ws + l.temp, tb, cub::CountingInputIterator<uint32_t>(0), seg, d_nnr,
                                static_cast<int>(total), HeadPred{keys_sorted}, stream));
  if (row_len <= 0) return;
  MergeSum m{srcs, keys_sorted, vals_sorted, seg, d_nnr, out_idx, out_val, row_len, RspUpdateLaunch(), sentinel};
  const int blocks = static_cast<int>((total + kWarpsPerBlock - 1) / kWarpsPerBlock);
  const int threads = kWarpsPerBlock * 32;
  if (fused_update == nullptr) {
    rsp_sum_kernel<-1><<<blocks, threads, 0, stream>>>(m);
  } else {
    m.u = *fused_update;
    switch (m.u.opt) {
      case kOptSGDSingle: rsp_sum_kernel<kOptSGDSingle><<<blocks, threads, 0, stream>>>(m); break;
      case kOptSGD: rsp_sum_kernel<kOptSGD><<<blocks, threads, 0, stream>>>(m); break;
      case kOptAdam: rsp_sum_kernel<kOptAdam><<<blocks, threads, 0, stream>>>(m); break;
      default: KV_FATAL << "row_sparse push: unsupported optimizer kind " << m.u.opt;
    }
  }
  KV_CUDA(cudaGetLastError());
}

size_t RetainBatchWorkspaceBytes(int nitems, int64_t total_ids, int id_bits) {
  return LayoutRetain(std::max(nitems, 1), std::max<int64_t>(total_ids, 1), id_bits).total;
}

void LaunchUniqueBatch(const RetainItem* h_items, int nitems, int64_t total, int id_bits,
                       int64_t* d_off, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  KV_CHECK(nitems >= 1 && total > 0 && total < (1LL << 31));
  int item_bits = 0;
  while ((1 << item_bits) < nitems) ++item_bits;
  KV_CHECK(id_bits >= 1 && id_bits + item_bits <= 62) << "row_sparse_pull: id space too large";
  const RetainLayout l = LayoutRetain(nitems, total, id_bits);
  KV_CHECK(workspace_bytes >= l.total) << "retain batch: workspace too small";
  char* ws = static_cast<char*>(workspace);
  RetainItem* items = reinterpret_cast<RetainItem*>(ws + l.items);
  int64_t* comp = reinterpret_cast<int64_t*>(ws + l.comp);
  int64_t* sorted = reinterpret_cast<int64_t*>(ws + l.sorted);
  int64_t* uniq = reinterpret_cast<int64_t*>(ws + l.uniq);
  int64_t* count = reinterpret_cast<int64_t*>(ws + l.count);
  KV_CUDA(cudaMemcpyAsync(items, h_items, nitems * sizeof(RetainItem), cudaMemcpyHostToDevice, stream));
  if (l.bm) {
    // bitmap unique: mark every item's ids in its own bitmap, rank them, emit them in order
    uint32_t* bitmap = reinterpret_cast<uint32_t*>(ws + l.bm_bitmap);
    uint32_t* prefix = reinterpret_cast<uint32_t*>(ws + l.bm_prefix);
    uint32_t* block_base = reinterpret_cast<uint32_t*>(ws + l.bm_block_base);
    uint32_t* done = reinterpret_cast<uint32_t*>(ws + l.bm_done);
    KV_CUDA(cudaMemsetAsync(bitmap, 0, l.bm_zero_bytes, stream));
    bm_mark_pull_kernel<<<GridFor(total, 256), 256, 0, stream>>>(items, nitems, total, l.nwords, bitmap);
    bm_scan_kernel<<<dim3(l.nblocks, nitems), kScanThreads, 0, stream>>>(bitmap, l.nwords, l.nblocks, prefix,
                                                                          block_base, done, count);
    bm_emit_pull_kernel<<<GridFor(l.nwords * nitems, 256), 256, 0, stream>>>(
        bitmap, prefix, block_base, l.nblocks, count, nitems, l.nwords, uniq, d_off);
    KV_CUDA(cudaGetLastError());
    return;
  }
  retain_gather_kernel<<<GridFor(total, 256), 256, 0, stream>>>(items, nitems, total, id_bits, comp);
  KV_CUDA(cudaGetLastError());
  size_t tb = l.temp_bytes;
  KV_CUDA(cub::DeviceRadixSort::SortKeys(ws + l.temp, tb, comp, sorted, static_cast<int>(total), 0,
                                         id_bits + item_bits, stream));
  tb = l.temp_bytes;
  KV_CUDA(cub::DeviceSelect::Unique(ws + l.temp, tb, sorted, uniq, count, static_cast<int>(total),
                                    stream));
  retain_bounds_kernel<<<(nitems + 1 + 127) / 128, 128, 0, stream>>>(uniq, count, nitems, id_bits, d_off);
  KV_CUDA(cudaGetLastError());
}

void LaunchRetainBatch(int nitems, int64_t total, int id_bits, const int64_t* d_off, void* workspace,
                       cudaStream_t stream) {
  const RetainLayout l = LayoutRetain(nitems, total, id_bits);
  char* ws = static_cast<char*>(workspace);
  const RetainItem* items = reinterpret_cast<const RetainItem*>(ws + l.items);
  const int64_t* uniq = reinterpret_cast<const int64_t*>(ws + l.uniq);
  const int blocks = static_cast<int>(std::min<int64_t>((total + kWarpsPerBlock - 1) / kWarpsPerBlock, kNumSMs * 8));
  retain_kernel<<<blocks, kWarpsPerBlock * 32, 0, stream>>>(items, nitems, total, id_bits, uniq, d_off);
  KV_CUDA(cudaGetLastError());
}

void LaunchRowMap(const int64_t* gidx, int64_t nnr, int64_t table_rows, int32_t* row_map,
                  cudaStream_t stream) {
  if (table_rows <= 0) return;
  KV_CHECK(nnr < (1LL << 31));
  KV_CUDA(cudaMemsetAsync(row_map, 0xff, static_cast<size_t>(table_rows) * sizeof(int32_t), stream));
  if (nnr > 0) {
    row_map_scatter_kernel<<<GridFor(nnr, 256), 256, 0, stream>>>(gidx, nnr, row_map);
    KV_CUDA(cudaGetLastError());
  }
}

size_t NonzeroRowsWorkspaceBytes(int64_t rows) {
  size_t t = 0;
  cub::DeviceSelect::Flagged(nullptr, t, cub::CountingInputIterator<int64_t>(0),
                             static_cast<const uint8_t*>(nullptr), static_cast<int64_t*>(nullptr),
                             static_cast<int64_t*>(nullptr), static_cast<int>(std::max<int64_t>(rows, 1)));
  return ((static_cast<size_t>(std::max<int64_t>(rows, 1)) + 255) & ~static_cast<size_t>(255)) + t + 256;
}

void LaunchNonzeroRows(const float* data, int64_t rows, int64_t row_len, int64_t* out_idx,
                       int64_t* d_count, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  KV_CHECK(rows > 0 && rows < (1LL << 31));
  KV_CHECK(workspace_bytes >= NonzeroRowsWorkspaceBytes(rows));
  uint8_t* flags = static_cast<uint8_t*>(workspace);
  const size_t off = (static_cast<size_t>(rows) + 255) & ~static_cast<size_t>(255);
  const int blocks = static_cast<int>((rows + kWarpsPerBlock - 1) / kWarpsPerBlock);
  row_nonzero_flag_kernel<<<blocks, kWarpsPerBlock * 32, 0, stream>>>(data, rows, row_len, flags);
  KV_CUDA(cudaGetLastError());
  size_t tb = workspace_bytes - off;
  KV_CUDA(cub::DeviceSelect::Flagged(static_cast<char*>(workspace) + off, tb,
                                     cub::CountingInputIterator<int64_t>(0), flags, out_idx, d_count,
                                     static_cast<int>(rows), stream));
}

void LaunchRspScatterRows(const int64_t* idx, const float* val, int64_t nnr, int64_t row_len,
                          float* dense, cudaStream_t stream) {
  if (nnr <= 0 || row_len <= 0) return;
  const int blocks = static_cast<int>((nnr + kWarpsPerBlock - 1) / kWarpsPerBlock);
  rsp_scatter_rows_kernel<<<blocks, kWarpsPerBlock * 32, 0, stream>>>(idx, val, nnr, row_len, dense);
  KV_CUDA(cudaGetLastError());
}

void LaunchRspBroadcast(const RspBroadcastLaunch& p, cudaStream_t stream) {
  const int64_t domain = p.n_dns > 0 ? p.rows : p.nnr;
  if (domain <= 0 || p.row_bytes <= 0 || p.n_dns + p.n_rsp == 0) return;
  KV_CHECK(p.n_dns <= kMaxDst && p.n_rsp <= kMaxDst);
  uintptr_t bits = reinterpret_cast<uintptr_t>(p.src_val) | static_cast<uintptr_t>(p.row_bytes);
  for (int t = 0; t < p.n_dns; ++t) bits |= reinterpret_cast<uintptr_t>(p.dns[t]);
  for (int t = 0; t < p.n_rsp; ++t) bits |= reinterpret_cast<uintptr_t>(p.rsp_val[t]);
  const int blocks = static_cast<int>(std::min<int64_t>((domain + kWarpsPerBlock - 1) / kWarpsPerBlock, kNumSMs * 8));
  const int threads = kWarpsPerBlock * 32;
  if ((bits & 15) == 0) {
    rsp_broadcast_kernel<uint4><<<blocks, threads, 0, stream>>>(p);
  } else if ((bits & 3) == 0) {
    rsp_broadcast_kernel<uint32_t><<<blocks, threads, 0, stream>>>(p);
  } else {
    rsp_broadcast_kernel<uint8_t><<<blocks, threads, 0, stream>>>(p);
  }
  KV_CUDA(cudaGetLastError());
}

}  // namespace b200kv
