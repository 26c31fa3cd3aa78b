// kernels.h -- host-side launch interface of the hand-written sm_90a kernels (plain structs, no
// CUDA types beyond cudaStream_t) so the runtime (.cc) and the kernels (.cu) compile separately.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <climits>

namespace b200kv {

constexpr int kMaxSrc = 16;  // values of one key per push (devices / ranks)
constexpr int kMaxDst = 16;  // outs of one key per pull
constexpr int kChunkElems = 4096;   // work item: <= 4096 consecutive elements of one key
constexpr int kBlockElems = 32768;  // ownership stripe in the store-global element space
constexpr int kKeyAlignElems = 128; // every key starts on a 128-element boundary of that space

// What the update step computes from (w, merged gradient, state). Expression trees are the
// reference's, see dense_kernels.cu.
enum OptKind : int {
  kOptAssign = 0,     // stored = merged            (push without updater, kvstore_local.h:237-243)
  kOptSGD = 1,        // multi_sgd[_mom]_update     (optimizer_op-inl.h:225-258)
  kOptSGDSingle = 2,  // sgd_update / mp_sgd_update (optimizer_op-inl.h:388-397, 661-674)
  kOptAdam = 3,       // adam_update                (optimizer_op-inl.h:1302-1312)
  kOptTest = 4,       // mx.optimizer.Test          (optimizer.py:2044-2046)
  kOptPullOnly = 5,   // no gradient: broadcast the stored value
};

enum SumOrder : int {
  kOrderDevice = 0,  // left fold             (ndarray_function-inl.h:402-431, CommDevice)
  kOrderLocal = 1,   // g0 + groups of four   (comm.h:357-392, CommCPU)
};

// One key of a fused launch, as seen by ONE device. 16-byte aligned so it can be fetched as uint4.
struct alignas(16) KeyDesc {
  const void* src[kMaxSrc];  // gradient of every source (local or peer-mapped), dtype = key dtype
  void* out[kMaxDst];        // pull targets (local or peer-mapped), dtype = key dtype
  void* w;                   // stored value on this device, written (key dtype)
  // stored value on this device, read: w itself, except on the step that moves the value between
  // the store's own buffer and a pull anchor (kvstore.h, DevState)
  const void* w_in;
  float* w32;                // fp32 master weights (16-bit keys under multi_precision) or null
  float* s1;                 // momentum / Adam mean (fp32) or null
  float* s2;                 // Adam var (fp32) or null
  float lr_unused;           // per-key (lr, wd) travel in DenseLaunch::hyper so a plan's tables
  float wd_unused;           // stay constant across steps
  int32_t n_src;
  int32_t n_out;
  uint32_t vec_ok;           // all pointers 16-byte aligned -> vector path
  // NVLS (one rank per GPU, NVSwitch multicast mapping of the arenas): 0 = off, else 1 + number of
  // multicast pull targets. src[kMaxSrc-1] is then the MULTICAST address of the gradient (a
  // multimem.ld_reduce returns the sum over all ranks, added inside the switch) and
  // out[kMaxDst-2], out[kMaxDst-1] the multicast addresses of the pull targets (one multimem.st
  // reaches every rank). The unicast src[]/out[] entries stay valid for the scalar tail path.
  uint32_t nvls;
};
static_assert(sizeof(KeyDesc) == 320, "KeyDesc: 20 uint4 words");

struct alignas(16) ChunkDesc {
  uint32_t key;  // index into the KeyDesc table
  uint32_t off;  // first element (multiple of kKeyAlignElems unless the key is unaligned)
  uint32_t len;  // 1..kChunkElems
  uint32_t pad_;
};

struct DenseLaunch {
  const KeyDesc* keys = nullptr;      // device memory
  const ChunkDesc* chunks = nullptr;  // device memory
  const float* hyper = nullptr;       // device memory: (lr, wd) float pairs, one per key
  const float* lrs = nullptr;         // preloaded_multi_* operators: per-key lr and wd in two
  const float* wds = nullptr;         // device arrays (override hyper when set)
  int n_chunks = 0;
  int max_src = 0;     // max n_src over the keys (selects the unroll variant)
  bool nvls = false;   // every key of the launch carries NVSwitch multicast addresses (KeyDesc::nvls)
  int dtype = 0;       // key dtype: kFloat32 / kFloat16 / kBfloat16
  int opt = kOptAssign;
  int order = kOrderDevice;
  float momentum = 0.f, rescale = 1.f, clip = -1.f, beta1 = 0.9f, beta2 = 0.999f, eps = 1e-8f;
  // cross-process launches (one rank per GPU): signal pads for the in-kernel start/end barriers
  uint32_t* const* signal_pads = nullptr;  // device array [world] of peer-mapped pads, or null
  uint32_t* counter = nullptr;             // this rank's finished-CTA counter
  int rank = 0, world = 1;
  uint32_t epoch = 0;
  // a rank that waits longer than timeout_ns for a peer writes (peer + 1, phase/epoch) into the
  // host-visible err_word, stops waiting and lets the kernel finish: the host raises a recoverable
  // error at its next wait instead of the context dying in a __trap
  uint32_t* err_word = nullptr;
  unsigned long long timeout_ns = 0;
  int barrier_mask = 3;  // bit 0: start barrier inside this launch, bit 1: end barrier
};

// Fused reduce (+scale/clip +optimizer step) (+broadcast) over a list of chunks, one CTA per chunk.
void LaunchDenseFused(const DenseLaunch& p, cudaStream_t stream);

// ---- small elementwise helpers for the imperative-op surface (updaters written in Python) ----
enum EwOp : int { kEwCopy = 0, kEwAdd, kEwSub, kEwMul, kEwAddScalar, kEwMulScalar, kEwFill, kEwSqrt };
void LaunchElementwise(int op, int dtype, void* out, const void* a, const void* b, float scalar,
                       size_t n, cudaStream_t stream);
void LaunchCast(void* out, int out_dtype, const void* in, int in_dtype, size_t n, cudaStream_t stream);

// ---- row_sparse (rowsparse_kernels.cu) ----
// lazy row updates over the rows listed in a row_sparse gradient (optimizer_op-inl.h:426-450,
// 776-801, 1383-1408); opt is kOptSGDSingle (sgd_update), kOptSGD (sgd_mom_update), kOptAdam
struct RspUpdateLaunch {
  float* w = nullptr; float* s1 = nullptr; float* s2 = nullptr;
  const int64_t* gidx = nullptr; const float* gval = nullptr;
  int64_t nrows = 0, row_len = 0;
  const int64_t* d_nrows = nullptr;  // when set: the row count lives on the device, nrows bounds it
  int opt = kOptSGDSingle;
  float lr = 0.f, wd = 0.f, momentum = 0.f, rescale = 1.f, clip = -1.f, beta1 = 0.9f,
        beta2 = 0.999f, eps = 1e-8f;
};
void LaunchRspUpdate(const RspUpdateLaunch& p, cudaStream_t stream);

// standard (non-lazy) update over ALL `table_rows` rows of a dense weight; rows missing from the
// row_sparse gradient (gidx / gval / nrows or d_nrows of `p`) use grad = 0. row_map: int32[table_rows]
void LaunchRspStdUpdate(const RspUpdateLaunch& p, int64_t table_rows, int32_t* row_map,
                        cudaStream_t stream);
// storage casts: ids of the rows with any non-zero element (ascending) + count; scatter rows
size_t NonzeroRowsWorkspaceBytes(int64_t rows);
void LaunchNonzeroRows(const float* data, int64_t rows, int64_t row_len, int64_t* out_idx,
                       int64_t* d_count, void* workspace, size_t workspace_bytes, cudaStream_t stream);
void LaunchRspScatterRows(const int64_t* idx, const float* val, int64_t nnr, int64_t row_len,
                          float* dense, cudaStream_t stream);

// union of row ids + in-order accumulation (ndarray_function.cc:59-175 semantics), one call:
//   tag      keys[i] = id, vals[i] = i over the concatenation of the sources' id lists
//   sort     stable radix sort of (key, val) on the low `id_bits` bits only
//   heads    positions where the sorted id changes -> segment starts, count -> *d_nnr
//   sum      one warp per segment: out_idx[r] = id, out_val[r] = 0.0f + rows in SOURCE ORDER
//            (the stable sort keeps equal ids in concatenation = source order)
// No binary searches, no host read of the count: the sum grid covers `total` rows and warps
// beyond *d_nnr exit. With `fused_update` the summed row is never written: the same warp applies
// the lazy optimizer step to row `id` of w / state (out_idx, out_val unused).
struct RspSources {
  const int64_t* idx[kMaxSrc];
  const float* val[kMaxSrc];
  int64_t start[kMaxSrc + 1];  // prefix of the row counts; start[nsrc] = total
  int nsrc = 0;
};
// id_bits / nsrc / [lo, hi) as passed to LaunchRspMerge: they decide between the bitmap union
// (tables of up to 8 M rows per range) and the radix-sort union
size_t RspMergeWorkspaceBytes(int64_t total_ids, int id_bits, int nsrc, int64_t lo = 0, int64_t hi = INT64_MAX);
void LaunchRspMerge(const RspSources& srcs, int id_bits, int64_t row_len, int64_t* out_idx,
                    float* out_val, int64_t* d_nnr, void* workspace, size_t workspace_bytes,
                    cudaStream_t stream, const RspUpdateLaunch* fused_update = nullptr,
                    int64_t lo = 0, int64_t hi = INT64_MAX);  // [lo, hi): only ids of this row range

// row_sparse_pull for a batch of (row_ids, out) pairs that share an owner GPU
// (kvstore_local.h:263-283 + kvstore_utils.cu:43-97 Unique + sparse_retain-inl.h:121-150,262-323):
//   gather   comp[i] = item << id_bits | id over the concatenation of all items' row_ids
//   sort + unique of comp (one radix sort for the whole batch, id_bits + item_bits bits)
//   bounds   off[k] = first unique entry of item k (off[nitems] = total unique) -> device + host
//   retain   one warp per (item, unique id): out_idx = id, row copied where present else zeros
struct RetainItem {
  const void* ids; int ids_dtype; int64_t n; int64_t start;  // start: prefix of n over the batch
  const int64_t* src_idx; const float* src_val; int64_t src_nnr; int src_dense_rows;
  int64_t row_len;
  int64_t* out_idx; float* out_val;
  // table sharded by row range over several GPUs: device array of "virtual bases"
  // (shard base - first_row*row_len, so that vbase[id / rows_per_shard] + id*row_len is row id)
  const float* const* shard_vbase; int64_t rows_per_shard;
};
size_t RetainBatchWorkspaceBytes(int nitems, int64_t total_ids, int id_bits);
// d_items: device copy of `nitems` RetainItem (inside the workspace, filled by the callee from
// h_items); d_off: device int64[nitems + 1]
void LaunchUniqueBatch(const RetainItem* h_items, int nitems, int64_t total_ids, int id_bits,
                       int64_t* d_off, void* workspace, size_t workspace_bytes, cudaStream_t stream);
void LaunchRetainBatch(int nitems, int64_t total_ids, int id_bits, const int64_t* d_off,
                       void* workspace, cudaStream_t stream);

// whole-value pull of a row_sparse value (CopyFromTo with storage casts, ndarray.cc:1076-1093,
// cast_storage-inl.h:74-140), every target in one pass: row_sparse targets get the nnr ids and
// rows, dense targets every table row (the stored row or zeros). Rows move in 16-byte units when
// row_bytes and every base are 16-byte aligned, else in 4- or 1-byte units; any dtype.
struct RspBroadcastLaunch {
  const int64_t* src_idx = nullptr;  // nnr ascending ids
  const void* src_val = nullptr;     // nnr rows of row_bytes
  int64_t nnr = 0, rows = 0, row_bytes = 0;
  int n_rsp = 0, n_dns = 0;
  int64_t* rsp_idx[kMaxDst] = {};    // row_sparse targets with room for nnr rows
  void* rsp_val[kMaxDst] = {};
  void* dns[kMaxDst] = {};           // dense targets of rows x row_bytes
};
void LaunchRspBroadcast(const RspBroadcastLaunch& p, cudaStream_t stream);

// ---- multi-tensor optimizer operators (multi_tensor_kernels.cu; SURVEY 8f-f1) ----
constexpr int kMTChunk = 8192;      // elements per CTA
constexpr int kMTMaxTensors = 64;   // tensors per launch (their scalars travel by value)
struct MTTensor {
  void* p[6];            // op-specific: w, g, mean, var, w32, out / temp_g (see each functor)
  uint32_t size;         // elements
  uint32_t vec_ok;       // every pointer 16-byte aligned (8 for 16-bit types): vector path allowed
  uint32_t first_chunk;  // index of the tensor's first chunk partial
  uint32_t aux;          // position of the tensor in the op's per-tensor outputs (sums of squares)
};
struct MTChunk { uint32_t tensor, off, len, pad; };
struct MTScalars {
  float4 t[kMTMaxTensors];  // per tensor, e.g. (lr, wd, eta, -)
  float f[12];              // per launch
  const float* d0;          // device scalars / arrays (rescale_grad, r1, sums of squares ...)
  const float* d1;
};
enum MTOp : int { kMTSumSq = 0, kMTAdamW, kMTMultiAdamW, kMTLambPhase1, kMTLambPhase2,
                  kMTMultiLambStep1, kMTMultiLambStep2 };
struct MTLaunch {
  int op = kMTSumSq;
  int dtype = 0;         // DType (common.h) of the weight / gradient arrays; 0 = float32
  bool mp = false;       // fp32 master copies present (16-bit weights)
  const MTTensor* tensors = nullptr;
  const MTChunk* chunks = nullptr;
  int n_chunks = 0;
  MTScalars s;
  float* part0 = nullptr;  // per-chunk partial sums (reducing ops)
  float* part1 = nullptr;
};
void LaunchMultiTensor(const MTLaunch& L, cudaStream_t stream);
// out0[t.aux] (and out1) = the tensor's chunk partials summed in a fixed tree
void LaunchMultiTensorFinalize(const MTTensor* tensors, int n_tensors, const float* part0,
                               const float* part1, float* out0, float* out1, cudaStream_t stream);
void LaunchMultiLars(int n, float* out, const float* lrs, const float* wsq, const float* gsq,
                     const float* wds, float eta, float eps, float rescale, cudaStream_t stream);

// ---- single-tensor optimizer operators of the callback route (update_kernels.cu) ----
// nag_mom_update, mp_nag_mom_update, signsgd_update, signum_update, rmsprop_update,
// rmspropalex_update, ftml_update, ftrl_update (optimizer_op-inl.h:1061-1222, 1953-2158, 2344-2431)
enum UpdOp : int { kUpdNAG = 0, kUpdMPNAG, kUpdSignSGD, kUpdSignum, kUpdRMSProp, kUpdRMSPropAlex,
                   kUpdFTML, kUpdFtrl, kUpdAdaGrad, kUpdGroupAdaGrad };
struct UpdateLaunch {
  int op = kUpdNAG;
  int dtype = 0;                 // of w / g / out: kFloat32, or kFloat16 / kBfloat16 for kUpdMPNAG
  const void* w = nullptr;       // weight (read; may be the same storage as out)
  const void* g = nullptr;
  void* out = nullptr;
  float* s[3] = {nullptr, nullptr, nullptr};  // fp32 states in the operator's input order
                                              // (mp_nag: mom, weight32)
  size_t n = 0;
  bool out_is_w = false;  // nag_mom_update reads the weight again after storing out
  // hyper-parameters, by value (FTML: p1 = powf(beta1, t), p2 = powf(beta2, t) from the host)
  float lr = 0.f, wd = 0.f, rescale = 1.f, clip = -1.f, momentum = 0.f, wd_lh = 0.f, gamma1 = 0.f,
        gamma2 = 0.f, eps = 0.f, clip_weights = -1.f, beta1 = 0.f, beta2 = 0.f, p1 = 0.f, p2 = 0.f,
        lamda1 = 0.f, beta = 0.f;
  // row_sparse forms (LaunchRspRowUpdateOp): w / out / s hold every row of the table, g holds
  // `nnr` rows of `row_len` elements, and gradient row r updates table row gidx[r]
  const int64_t* gidx = nullptr;
  int64_t nnr = 0, row_len = 0;
};
void LaunchUpdateOp(const UpdateLaunch& L, cudaStream_t stream);
// row_sparse forms of ftrl_update and _sparse_adagrad_update (rowsparse_kernels.cu;
// FtrlDnsRspDnsKernel, AdagradDnsRspDnsKernel: optimizer_op-inl.h:2186-2219, 2507-2531): float32,
// one warp per gradient row, the same Step<OP> as the dense kernel. Rows not in gidx stay untouched.
// kUpdGroupAdaGrad (_contrib_group_adagrad_update, GroupAdagradDnsRspKernel: contrib/
// optimizer_op-inl.h:96-139): s[0] is the history, one float per table row; each row's sum of
// squares is folded strictly left to right, as the reference's CPU loop rounds it.
void LaunchRspRowUpdateOp(const UpdateLaunch& L, cudaStream_t stream);
// FillDnsZerosRspImpl's id half (init_op.h:474-487): ids[i] = i for i < rows
void LaunchFillRowIds(int64_t* ids, int64_t rows, cudaStream_t stream);

// ---- 2-bit gradient compression with residual (compress_kernels.cu;
// src/kvstore/gradient_compression-inl.h:40-132, comm.h:552-596 ReduceCompressed) ----
// residual += grad; >= +t -> code 11, residual -= t; <= -t -> code 10, residual += t; else 00.
// 16 values per 32-bit word, value i in byte (i%16)/4, bit pair 6-2*(i%4).
void LaunchQuantize2Bit(const float* grad, float* residual, uint32_t* compressed, size_t n,
                        float threshold, cudaStream_t stream);
// merged[i] = deq(comp[0])[i] + deq(comp[1])[i] + ...   (left fold, ElementwiseSum order)
void LaunchDequantizeSum2Bit(const uint32_t* const* d_compressed /* device array [nsrc] */, int nsrc,
                             float* merged, size_t n, float threshold, cudaStream_t stream);

// ---- TMA bulk-copy packing of many small arrays into one fusion buffer (pack_kernels.cu) ----
constexpr int kPackTileBytes = 16384;  // one TMA bulk copy; items passed to the kernel are <= this
struct PackItem { const void* src; void* dst; uint64_t bytes; };
void LaunchPackBulk(const PackItem* d_items, int n_items, uint64_t max_bytes, cudaStream_t stream,
                    int max_ctas = 0);

}  // namespace b200kv
