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
// float16, bfloat16, float32, float64, int32 and int64. `scalar` is the operator's double; the kernel
// converts it once to the array's dtype, as the reference's DType(alpha) / static_cast<DType>(value).
// kEwClip takes its float bounds a_min, a_max as `scalar`, `scalar2` and compares them with each
// element as the reference's clip kernel does. kEwDiv, kEwDivScalar and kEwRDivScalar (scalar / a)
// divide floating types only.
// b_row > 0 makes `b` one value per row of b_row elements (b[i / b_row]); 0: b has n elements.
enum EwOp : int {
  kEwCopy = 0, kEwAdd, kEwSub, kEwMul, kEwAddScalar, kEwMulScalar, kEwFill, kEwSqrt,
  kEwDiv, kEwMax, kEwDivScalar, kEwAbs, kEwClip, kEwSquare, kEwRDivScalar
};
bool ElementwiseDTypeOk(int dtype);
void LaunchElementwise(int op, int dtype, void* out, const void* a, const void* b, double scalar,
                       size_t n, cudaStream_t stream, double scalar2 = 0.0, size_t b_row = 0);

// out[r] = the mean of row r of `in`, `rows` rows of `cols` elements each (cols >= 1): each row
// folded left to right with red::sum's Kahan step in the dtype, then divided by DType(cols), as the
// reference's mean over the trailing axis (broadcast_reduce-inl.h:161-175, broadcast_reduce_op.h:
// 630-633). float16, bfloat16, float32 and float64 (reduce_kernels.cu).
void LaunchRowMean(int dtype, void* out, const void* in, int64_t rows, int64_t cols, cudaStream_t stream);
void LaunchCast(void* out, int out_dtype, const void* in, int in_dtype, size_t n, cudaStream_t stream);

// ---- row_sparse (rowsparse_kernels.cu) ----
// the lazy optimizer step that LaunchRspMerge fuses into its row sum (optimizer_op-inl.h:426-450,
// 776-801, 1383-1408): row `id` of the table w (+ states) takes the summed gradient row; opt is
// kOptSGDSingle (sgd_update), kOptSGD (sgd_mom_update) or kOptAdam
struct RspUpdateLaunch {
  float* w = nullptr; float* s1 = nullptr; float* s2 = nullptr;
  int opt = kOptSGDSingle;
  float lr = 0.f, wd = 0.f, momentum = 0.f, rescale = 1.f, clip = -1.f, beta1 = 0.9f,
        beta2 = 0.999f, eps = 1e-8f;
};

// row_map[r] = position of table row r among the `nnr` ascending ids `gidx`, or -1: a memset of
// int32[table_rows] to -1, then row_map_scatter_kernel when nnr > 0
void LaunchRowMap(const int64_t* gidx, int64_t nnr, int64_t table_rows, int32_t* row_map,
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

// all_finite / multi_all_finite (contrib/all_finite.cc): *out = 0.0f when any element of any array
// is non-finite, else *out is not written. One launch for up to kAFMaxArrays arrays; the list
// travels by value in the kernel parameters, so no device table and no host-to-device copy.
// Work is tiled by bytes (kAFTileBytes per CTA) so that every dtype gives a CTA the same work.
constexpr int kAFMaxArrays = 200;  // MultiAllFiniteKernelParam::N of the reference
constexpr int kAFTileBytes = 16384;
struct AllFiniteArrays {
  const void* p[kAFMaxArrays];               // dtype of the launch; any alignment
  uint64_t n[kAFMaxArrays];                  // elements
  uint32_t first_tile[kAFMaxArrays + 1];     // prefix of the tile counts (filled by the launcher)
  int32_t count;
};
static_assert(sizeof(AllFiniteArrays) <= 32764, "kernel parameters are limited to 32764 bytes");
// dtype: kFloat16, kBfloat16, kFloat32 or kFloat64. Always exactly one launch.
void LaunchAllFinite(int dtype, AllFiniteArrays& arrays, float* out, cudaStream_t stream);

// _b200kv_clip_global_norm / _b200kv_multi_scale (gluon.utils.clip_global_norm, amp.unscale): float32
// arrays of one GPU, listed by value like AllFiniteArrays and tiled by bytes the same way. A call
// with more than kCNMaxArrays arrays goes group by group; nothing here waits on the host.
constexpr int kCNMaxArrays = 200;
constexpr int kCNTileBytes = 16384;
struct ClipNormArrays {
  float* p[kCNMaxArrays];                    // any 4-byte alignment
  uint32_t n[kCNMaxArrays];                  // elements (stored rows x row length for row_sparse)
  uint32_t first_tile[kCNMaxArrays + 1];     // prefix of the tile counts (filled by ClipNormTiles)
  int32_t count;
};
// Fills first_tile; returns the group's number of tiles (0: nothing to launch for it).
uint32_t ClipNormTiles(ClipNormArrays& arrays);
// clip_norm_partial: part[0 .. tiles) = each tile's sum of squares. One launch.
void LaunchClipNormPartial(const ClipNormArrays& arrays, uint32_t tiles, float* part, cudaStream_t stream);
// clip_norm_fold: ss = part[0] + ... + part[n_part - 1] in one fixed association; *total_norm =
// sqrtf(ss); *scale = min(max_norm / (total_norm + 1e-8f), 1), and 1 when total_norm is inf / nan.
void LaunchClipNormFold(const float* part, uint32_t n_part, float max_norm, float* total_norm,
                        float* scale, cudaStream_t stream);
// clip_norm_scale: x *= s in place, s = *scale_dev when given, else scale. Returns without reading
// or writing the arrays when s == 1. One launch.
void LaunchClipNormScale(const ClipNormArrays& arrays, uint32_t tiles, const float* scale_dev, float scale,
                         cudaStream_t stream);

// reset_arrays (contrib/reset_arrays.cc, ParameterDict.zero_grad): every byte of every array set to
// 0x00, which is +0.0 in each floating dtype, so arrays of different dtypes share a launch. Listed
// by value like AllFiniteArrays, tiled by bytes the same way; no byte outside [p, p + bytes) is
// written. A call with more than kRAMaxArrays arrays goes group by group.
constexpr int kRAMaxArrays = 200;
constexpr int kRATileBytes = 16384;
struct ResetArraysList {
  void* p[kRAMaxArrays];                     // any alignment
  uint64_t bytes[kRAMaxArrays];
  uint32_t first_tile[kRAMaxArrays + 1];     // prefix of the tile counts (filled by the launcher)
  int32_t count;
};
static_assert(sizeof(ResetArraysList) <= 32764, "kernel parameters are limited to 32764 bytes");
// reset_arrays_kernel: one launch, none when every array is empty. Returns the number of launches.
int LaunchResetArrays(ResetArraysList& arrays, cudaStream_t stream);

// add_n / ElementWiseSum on dense arrays (tensor/elemwise_sum.h:48-98, ElementWiseSumCompute_):
// out = in[0] + (in[1] + (in[2] + in[3])) for 2-4 inputs, else the left chain out = in[0], then
// out = out + in[i]. Every + is in the dtype: the 16-bit types add in float and round once, integers
// wrap. zero_first starts the chain at +0 (out = 0 + in[0] + ...: ElementwiseSumContainsDnsImpl
// with a row_sparse in[0]). The input list travels by value, up to kAddNMaxArrays per launch; past
// that the chain continues in the next launch from out. Any alignment; out may be in[0] itself.
// float16, bfloat16, float32, float64, uint8, int8, int32 and int64 (sum_kernels.cu). Returns the
// number of launches: none for an empty out, else ceil((n_in - 1) / (kAddNMaxArrays - 1)), at least 1.
constexpr int kAddNMaxArrays = 200;
int LaunchAddN(int dtype, const void* const* in, int n_in, bool zero_first, void* out, uint64_t n,
               cudaStream_t stream);

// ---- the reference's GPU parallel sampler (random_kernels.cu; common/random_generator.cu,
// random/sampler.h) ----
// One generator copy is kRandStates curandStatePhilox4_32_10_t states of kRandStateBytes each.
constexpr int kRandStates = 32768;
constexpr int kRandMinPerThread = 64;
constexpr int kRandStateBytes = 64;
// state id = curand_init(seed, id, 0) for every id of the copy (one launch)
void LaunchRandSeed(void* states, uint32_t seed, cudaStream_t stream);
// out[i] = dtype(normal() * scale + loc) over n elements in LaunchRNG's state-to-element mapping,
// advancing the copy's states (float16, bfloat16, float32, float64; any alignment). staged = false
// stores as each thread draws, the reference's store order (for measurement only). No launch when
// n == 0.
void LaunchRandNormal(int dtype, void* states, void* out, uint64_t n, float loc, float scale, bool staged,
                      cudaStream_t stream);
// The scalar-parameter samplers of random/sampler.h, in the same mapping and staged store:
//   kRandUniform      a + (b - a) * uniform()                  (low a, high b)
//   kRandExponential  -log(1 - uniform()) / a                   (lam a)
//   kRandGamma        Marsaglia-Tsang, shape a, scale b
//   kRandInt          lo + rand_int64() % (hi - lo), hi > lo    (int32, int64)
// The first three write float16, bfloat16, float32 or float64. No launch when n == 0.
// (kRandNormal is the multi-sample normal; the scalar normal is LaunchRandNormal.)
enum RandDist { kRandUniform, kRandExponential, kRandGamma, kRandInt, kRandNormal };
struct RandParams {
  float a = 0.0f, b = 0.0f;
  int64_t lo = 0, hi = 0;
};
void LaunchRandSample(int dist, int dtype, void* states, void* out, uint64_t n, const RandParams& p,
                      cudaStream_t stream);
// The multi-sample samplers of multisample_op.h in the same mapping and staged store: element i of
// out[0, n) draws kRandUniform (low a, high b), kRandNormal (mu a, sigma b), kRandExponential (lam
// a; b unused) or kRandGamma (alpha a, beta b) with parameters a[i / nBatch], b[i / nBatch], nBatch
// = n / nparm. ptype (the parameter arrays) and otype (out): float16, float32 or float64. A gamma
// element that exhausts its attempt budget is NaN. out may be a (the same bytes) when nparm == n.
// No launch when n == 0.
void LaunchRandSampleParams(int dist, int ptype, int otype, void* states, const void* a, const void* b,
                            uint64_t nparm, void* out, uint64_t n, cudaStream_t stream);

// ---- single-tensor optimizer operators of the callback route (update_kernels.cu) ----
// nag_mom_update, mp_nag_mom_update, signsgd_update, signum_update, rmsprop_update,
// rmspropalex_update, ftml_update, ftrl_update (optimizer_op-inl.h:1061-1222, 1953-2158, 2344-2431).
// The row_sparse-gradient forms of sgd_update, sgd_mom_update and adam_update: kUpdSGD, kUpdAdamLazy
// lazy (only the gradient's rows), kUpdSGDStd, kUpdAdamStd standard (every row), kUpdSGDMom both.
enum UpdOp : int { kUpdNAG = 0, kUpdMPNAG, kUpdSignSGD, kUpdSignum, kUpdRMSProp, kUpdRMSPropAlex,
                   kUpdFTML, kUpdFtrl, kUpdAdaGrad, kUpdGroupAdaGrad,
                   kUpdSGD, kUpdSGDStd, kUpdSGDMom, kUpdAdamLazy, kUpdAdamStd };
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
  // a row_sparse gradient of a dense float32 weight (LaunchRspGradUpdateOp): g holds the stored rows of
  // `row_len` elements, row_map[r] is table row r's position among them or -1 (LaunchRowMap), and
  // all `n` elements are updated, those of absent rows with g = +0.0f
  const int32_t* row_map = nullptr;
};
void LaunchUpdateOp(const UpdateLaunch& L, cudaStream_t stream);
// the float32 operators but mp_nag with a row_sparse gradient (update_rsp_grad_kernels.cu): every
// element of the dense weight and states moves, absent rows with g = +0.0f; also the standard forms
// of sgd_update, sgd_mom_update and adam_update (kUpdSGDStd, kUpdSGDMom, kUpdAdamStd)
void LaunchRspGradUpdateOp(const UpdateLaunch& L, cudaStream_t stream);
// row_sparse forms of ftrl_update and _sparse_adagrad_update (rowsparse_kernels.cu;
// FtrlDnsRspDnsKernel, AdagradDnsRspDnsKernel: optimizer_op-inl.h:2186-2219, 2507-2531) and the lazy
// forms of sgd_update, sgd_mom_update and adam_update (kUpdSGD, kUpdSGDMom, kUpdAdamLazy): float32,
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
// host_io: the list has a pinned-host side (SM-issued 16-byte copies); otherwise TMA bulk copies
void LaunchPackBulk(const PackItem* d_items, int n_items, cudaStream_t stream, bool host_io);

}  // namespace b200kv
