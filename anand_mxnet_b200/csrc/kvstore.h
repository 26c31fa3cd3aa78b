// kvstore.h -- the store behind MXKVStore*: key table, value grouping, placement, the fused
// optimizer's host state and the launch plans of the dense path.
//
// Reference roles covered (and replaced): KVStoreLocal (src/kvstore/kvstore_local.h:69-490),
// CommCPU / CommDevice (src/kvstore/comm.h:103-797), the Python Updater + Optimizer bookkeeping
// for SGD / Adam (python/mxnet/optimizer/optimizer.py:104-140,400-509,603-659,1610-1629,2079-2128).
//
// Placement (replaces CommDevice::InitMergeBuffer's per-key owner GPU): every key
// gets an offset in a store-global element space (aligned to 128 elements); that space is cut into
// stripes of 32768 elements owned round-robin by the participating GPUs. Each GPU reduces, updates
// and broadcasts the stripes it owns (reduce-scatter + update + all-gather in ONE kernel per GPU,
// peers' gradients read and peers' weights written through NVLink-mapped pointers), and keeps the
// optimizer state of exactly those stripes. With one GPU this degenerates to one fused kernel.
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "common.h"
#include "kernels.h"
#include "ndarray.h"

namespace b200kv {

typedef void (*UpdaterFn)(int key, void* recv, void* local, void* handle);
typedef void (*StrUpdaterFn)(const char* key, void* recv, void* local, void* handle);

struct OptConfig {
  bool enabled = false;
  int kind = kOptAssign;  // kOptSGD / kOptAdam / kOptTest
  double lr = 0.01, wd = 0.0, momentum = 0.0, rescale = 1.0, clip = 0.0 /* falsy: no clipping */;
  double beta1 = 0.9, beta2 = 0.999, eps = 1e-8;
  bool multi_precision = false;
  bool lazy_update = true;
  int begin_num_update = 0;
  int num_update = 0;
  std::unordered_map<int, double> lr_mult, wd_mult;
  std::unordered_map<int, int> count;  // Optimizer._index_update_count
};

// Pull anchors. After a pushpull writes a key's new value into a pull target `out`, the store and
// the caller hold the same bits. The value may then simply LIVE in `out` (the key's anchor): the
// next step reads gradient, `out` and state and writes `out` and state -- the copy in the store's
// own buffer is neither written nor read again (20 instead of 24 bytes per element for SGD with
// momentum). Invariant: the anchor holds the stored value bit for bit, or the key has no anchor.
// Only whole, never-escaped GPU arrays on the key's home GPU anchor, in a single-process store, for
// unstriped float32 keys and float16 / bfloat16 keys not under SGD / Adam (which keep fp32 master
// weights), and only an `out` that no other operand of the call touches. Any other write to the
// anchor's storage (engine.h, detach_anchor) first copies the value back into `own`.
// B200KV_PULL_ANCHOR=0 (read whenever a call is planned) forms no anchor and ends existing ones.
struct DevState {
  NDArray w;    // stored value replica (key dtype): `own`, or a view of the anchor
  NDArray own;  // the store's buffer while `w` is an anchor (kept, so a detach never allocates)
  bool anchored = false;
  NDArray w32;  // fp32 master (16-bit keys + multi_precision)
  NDArray s1;   // momentum / Adam mean
  NDArray s2;   // Adam var
};

struct KeyEntry {
  int key = 0;
  std::vector<int64_t> shape;
  int dtype = kFloat32;
  int stype = kDefaultStorage;   // as initialised
  // storage type of the current value: a dense key holds a row_sparse value (in `rsp`) after a
  // row_sparse push without an updater (kvstore_local.h:237-243), until its next dense push
  int vstype = kDefaultStorage;
  size_t size = 0;
  uint64_t goff = 0;    // offset in the store-global element space
  NDArray host;         // value as initialised, pinned host (kvstore_local.h:202) until first GPU use
  int home = -1;        // GPU holding the whole authoritative value (-1: still on host)
  bool striped = false; // authoritative value is striped over the store's device set
  std::map<int, DevState> dev;
  uint8_t queued = 0;   // deferred bucket execution: bit 0 = a push of this key is queued, bit 1 = a pull
  NDArray merged;       // reduce target of the updater-callback path (on `home`)
  NDArray rsp;          // row_sparse stored value (on `home` or host), see vstype
  // Row-range sharding of a row_sparse table whose stored value holds every row and whose
  // optimizer runs fused on the store (the embedding-training case, SURVEY 8e): GPU rsp_devs[j]
  // owns rows [j*rsp_rows_per, (j+1)*rsp_rows_per) of the weight and of the optimizer state.
  // While sharded, `rsp` is stale; UnshardRsp() folds everything back onto `home`.
  std::vector<int> rsp_devs;
  std::vector<NDArray> rsp_shards;          // dense [rows_j, row_len]
  std::vector<DevState> rsp_shard_state;    // s1 / s2 per shard
  int64_t rsp_rows_per = 0;
  std::map<int, NDArray> rsp_vbase;         // per launching GPU: device table of shard virtual bases
  bool rsp_group = false;                   // one rank per GPU: rsp_shards holds THIS rank's shard only
  std::vector<int64_t> rsp_peer_off;        // arena offset of every rank's shard (group mode)
  std::vector<NDArray> stage_src, stage_out;  // device staging of host-resident values / outs
  // 2-bit gradient compression: per source slot residual (fp32) and compressed words, both on the
  // source's GPU; decoded sum on `home`
  std::vector<NDArray> gc_residual, gc_compressed;
  NDArray gc_merged;
};

struct DenseOp {
  KeyEntry* e = nullptr;
  std::vector<NDArray> srcs;  // empty: pull only
  std::vector<NDArray> outs;  // empty: push only
  // where the kernel reads the stored value when the call moves it between `own` and an anchor
  // (none: the stored value `w` of the owner)
  NDArray w_in;
};

// Device-resident descriptor tables of one fused launch, cached by call signature.
struct Plan {
  struct PerDev {
    int dev = -1;
    void* d_keys = nullptr;
    void* d_chunks = nullptr;
    void* d_hyper = nullptr;
    int n_chunks = 0;
    std::vector<float> hyper;  // last uploaded (lr, wd) per key
    size_t bytes_keys = 0, bytes_chunks = 0, bytes_hyper = 0;
  };
  std::vector<PerDev> per_dev;
  int n_keys = 0;
  int max_src = 0;
  bool nvls = false;  // the launch uses NVSwitch multicast reduce / broadcast
  uint64_t algorithmic_bytes = 0;
  ~Plan();
};

// Same-GPU staging copies of one prepared launch, executed as ONE TMA bulk-copy kernel
// (pack_kernels.cu) instead of one cudaMemcpyAsync per array.
struct PackList {
  int dev = -1;
  std::vector<std::pair<NDArray, NDArray>> pairs;  // (from, to), both on `dev`
  void* d_items = nullptr;                          // PackItem[n] on the device (tiles <= 16 KB)
  size_t bytes_items = 0;
  int n_items = 0;
  uint64_t total_bytes = 0;
  // engine lane the launch runs on: the compute lane for device-to-device lists; lists with a
  // pinned-host side run on the H2D / D2H copy lane (ordering comes from the arrays' dependencies)
  int lane = -1;
  bool host_io = false;
  ~PackList();
};

std::shared_ptr<PackList> BuildPackList(std::vector<std::pair<NDArray, NDArray>>* pairs, size_t dma_min_bytes = 0);
void RunPackList(PackList& pl);

// Everything one fused launch group needs at run time, computed once per distinct call signature:
// placement done, state allocated, plan built, the arrays whose dependencies must be tracked, the
// host<->device staging copies to issue around the launch.
struct Prepared {
  int opt_kind = kOptAssign;
  int dtype = kFloat32;
  bool is_push = false;
  bool group = false;                                    // one-rank-per-GPU launch (group.h)
  // NCCL fallback (kvstore 'nccl', or a peer group without peer memory): the sources were packed
  // into `nccl_bucket`, which is all-reduced in place before the (local, one-source) fused kernel
  NDArray nccl_bucket;
  std::vector<DenseOp> ops;                              // device-side operands
  std::vector<std::pair<NDArray, NDArray>> stage_in;     // (host source, device staging buffer)
  std::vector<std::pair<NDArray, NDArray>> stage_out;    // (device staging buffer, host out)
  std::shared_ptr<PackList> pack_in, pack_out;           // same-GPU staging: one TMA pack launch
  std::vector<int> owners, parts;
  std::shared_ptr<Plan> plan;
  std::vector<float> hyper;                              // per key (lr, wd)
  uint64_t hyper_version = 0;
  DenseLaunch scalars;                                   // momentum / rescale / clip / betas
};

struct CachedCall {
  std::vector<uint64_t> sig;       // keys + storage identities of every operand of the C call
  std::vector<Prepared> launches;
  uint64_t epoch = 0;
};

class KVStore {
 public:
  explicit KVStore(const std::string& type);
  ~KVStore();

  const std::string& type() const { return type_; }
  int rank() const { return rank_; }              // 0 / 1 unless created inside a peer group
  int group_size() const { return group_size_; }

  void Init(const std::vector<int>& keys, const std::vector<NDArray>& values);
  void InitStr(const std::vector<std::string>& keys, const std::vector<NDArray>& values);
  // (operand vectors by value: the C entry points hand over temporaries, a queued call keeps them)
  void Push(std::vector<int> keys, std::vector<NDArray> values, int priority);
  void Pull(std::vector<int> keys, std::vector<NDArray> outs, int priority,
            bool ignore_sparse);
  void PushPull(std::vector<int> vkeys, std::vector<int> okeys, std::vector<NDArray> values,
                std::vector<NDArray> outs, int priority);
  void PullRowSparse(const std::vector<int>& keys, const std::vector<NDArray>& outs,
                     const std::vector<NDArray>& row_ids, int priority);
  std::vector<int> LookupKeys(const std::vector<std::string>& str_keys);
  void SetKeyTypeInt();
  void SetKeyTypeStr();

  void SetUpdater(UpdaterFn fn, StrUpdaterFn sfn, void* handle);
  void SetGradientCompression(const std::vector<std::pair<std::string, std::string>>& kw);

  // ---- fused optimizer (extension)
  void SetOptimizer(const std::string& name,
                    const std::vector<std::pair<std::string, std::string>>& kw);
  OptConfig& opt() { Flush(); return opt_; }  // queued calls run with the old hyper-parameters first
  const OptConfig& opt_view() const { return opt_; }
  // Optimizer._index_update_count[key] / Optimizer.num_update as they stand once the queued calls
  // have run (a queued push counts), without running them
  int UpdateCount(int key) const;
  int NumUpdate() const;
  void TouchOpt() { ++opt_version_; }  // call after changing opt() scalars / multipliers
  NDArray GetOptimizerState(int key, int state_id);
  void SetOptimizerState(int key, int state_id, const NDArray& v);
  // deferred bucket execution (see kvstore_core.cc)
  void SetBucketBytes(size_t n);
  void Flush();
  static void FlushAll();
  // engine.h detach_anchor: a write to the anchor `v` of one of this store's keys is about to be
  // declared
  void DetachVar(Var* v);
  std::string DescribePlan(const std::vector<int>& keys, int num_devices);

 private:
  KeyEntry& Entry(int key);
  void InitImpl(const std::vector<int>& keys, const std::vector<NDArray>& values);
  void PushImpl(const std::vector<int>& keys, const std::vector<NDArray>& values,
                const std::vector<int>* okeys, const std::vector<NDArray>* outs);
  void PullImpl(const std::vector<int>& keys, const std::vector<NDArray>& outs, bool ignore_sparse);

  // dense machinery
  void ExecDense(std::vector<DenseOp>& ops, int opt_kind, bool allow_stripe = true);
  void PrepareDense(std::vector<DenseOp>& ops, int opt_kind, bool allow_stripe,
                    std::vector<Prepared>* out);
  void RunPrepared(Prepared& p);
  void PrepareDenseGroup(std::vector<DenseOp>& ops, int opt_kind, std::vector<Prepared>* out);
  void PrepareDenseNccl(std::vector<DenseOp>& ops, int opt_kind, std::vector<Prepared>* out);
  void BroadcastInitNccl(const std::vector<int>& keys);
  std::shared_ptr<Plan> GetPlanGroup(const std::vector<DenseOp>& ops, int opt_kind, int fixed_owner = -1);
  void BroadcastInitGroup(const std::vector<int>& keys);
  // call-level cache: a repeated C call (same keys, same arrays) skips grouping/validation/planning
  bool CallSignature(int tag, const std::vector<int>& vkeys, const std::vector<NDArray>& values,
                     const std::vector<int>* okeys, const std::vector<NDArray>* outs,
                     std::vector<uint64_t>* sig);
  bool RunCachedCall(const std::vector<uint64_t>& sig);
  void StoreCachedCall(const std::vector<uint64_t>& sig, std::vector<Prepared>&& launches);
  void ExecCallbackPush(KeyEntry& e, const std::vector<NDArray>& srcs);
  // pull anchors (DevState): settled for a call before it is planned; true when one formed or ended.
  // `moves` records what formed or ended, so that a call refused while it is planned -- before any
  // launch -- leaves every value where it was (UndoAnchorMoves).
  struct AnchorMove {
    KeyEntry* e;
    NDArray anchor;
    bool formed;
  };
  bool ResolveAnchors(std::vector<DenseOp>* fused, std::vector<DenseOp>* pulls, std::vector<AnchorMove>* moves);
  void UndoAnchorMoves(const std::vector<AnchorMove>& moves);
  bool AnchorEligible(const KeyEntry& e) const;
  void DetachAnchor(KeyEntry& e);                       // the value back into `own` (a copy)
  std::unordered_map<const Var*, KeyEntry*> anchors_;
  void DensifyValue(KeyEntry& e);                       // dense key: row_sparse value -> dense weight
  NDArray RowSparseValue(KeyEntry& e, const std::vector<NDArray>& outs);  // whole, on a GPU
  void EnsureOnDevice(KeyEntry& e, int dev);            // HOST -> WHOLE(dev)
  void EnsureStriped(KeyEntry& e);                      // WHOLE -> STRIPED(devset_)
  void EnsureWhole(KeyEntry& e, int dev);               // STRIPED -> WHOLE(dev)
  DevState& StateOn(KeyEntry& e, int dev, int opt_kind);
  int OwnerOf(const KeyEntry& e, uint64_t global_elem) const;
  void SetDeviceSet(const std::vector<int>& devs);
  NDArray StageSrc(KeyEntry& e, size_t slot, const NDArray& host_src, int dev);
  NDArray StageOut(KeyEntry& e, size_t slot, const NDArray& host_out, int dev);
  void KeyHyper(const KeyEntry& e, int opt_kind, float* lr, float* wd);
  std::shared_ptr<Plan> GetPlan(const std::vector<DenseOp>& ops, int opt_kind,
                                const std::vector<int>& devs, bool striped);

  NDArray CompressedReduce(KeyEntry& e, const std::vector<NDArray>& srcs);  // compress.cc
  void CompressedReduceGroup(const std::vector<KeyEntry*>& es, std::vector<std::vector<NDArray>>* srcs);
  bool force_local_ = false;  // the launch being prepared needs no cross-rank step (operands already merged)
  float gc_threshold_ = 0.5f;

  // row_sparse machinery (rowsparse.cc)
  void PushRowSparse(KeyEntry& e, const std::vector<NDArray>& srcs);
  bool PushRowSparseSharded(KeyEntry& e, const std::vector<NDArray>& srcs, const std::vector<int>& parts,
                            RspUpdateLaunch U);
  // one rank per GPU: every rank owns a row range; gradients of the peers are read through IPC
  void PushRowSparseGroup(KeyEntry& e, const NDArray& src, RspUpdateLaunch U);
  NDArray MergeRowSparseGroup(KeyEntry& e, const NDArray& src);   // no fused optimizer: replicated merge
  void GroupBarrier();   // cross-rank barrier on this rank's compute lane (signal pads)
  void ShardRsp(KeyEntry& e, const std::vector<int>& devs);
  void UnshardRsp(KeyEntry& e);
  const float* const* RspShardTable(KeyEntry& e, int dev);
  // launches one owner's batch; the returned closure waits for the counts and finishes the outputs
  std::function<void()> PullRowSparseGroup(int home, const std::vector<size_t>& which,
                                           const std::vector<int>& keys, const std::vector<NDArray>& outs,
                                           const std::vector<NDArray>& row_ids);

  std::string type_;
  bool dist_ = false;         // created inside a one-rank-per-GPU peer group
  bool nccl_ = false;         // cross-rank sums go through ncclAllReduce (type 'nccl', or no peer memory)
  bool nccl_type_ = false;    // created as 'nccl': dense values only (src/kvstore/kvstore_nccl.h:62-70)
  int rank_ = 0, group_size_ = 1;
  bool order_local_ = true;   // 'local' => CommCPU association, 'device' => left fold
  int key_type_ = -1;         // -1 undefined, 0 string, 1 int (kvstore_local.h:60-64)
  std::unordered_map<int, std::unique_ptr<KeyEntry>> local_;
  std::unordered_map<std::string, int> str_key_dict_;
  std::unordered_map<int, std::string> reverse_str_key_dict_;
  int next_str_key_ = 0;
  std::unordered_set<int> warnings_printed_;
  uint64_t next_goff_ = 0;
  std::vector<int> devset_;   // GPUs the striped values live on, in first-push order
  UpdaterFn updater_ = nullptr;
  StrUpdaterFn str_updater_ = nullptr;
  void* updater_handle_ = nullptr;
  OptConfig opt_;
  std::unordered_map<uint64_t, std::shared_ptr<Plan>> plans_;
  std::unordered_map<uint64_t, std::shared_ptr<CachedCall>> call_cache_;
  struct PendingOp {
    std::vector<int> vkeys, okeys;
    std::vector<NDArray> vals, outs;
    int priority = 0;
  };
  // queues the call and takes the vectors' contents when it returns true; leaves them alone otherwise
  bool TryDefer(int kind, std::vector<int>& vkeys, std::vector<NDArray>& values, std::vector<int>& okeys,
                std::vector<NDArray>& outs, int priority);
  std::vector<PendingOp> pending_;
  std::vector<KeyEntry*> pending_entries_;      // keys with a queued push (KeyEntry::queued bit 0) / pull (bit 1)
  size_t pending_bytes_ = 0, bucket_bytes_ = 0;
  bool bucket_auto_ = true;                      // queue single-key calls (see the constructor)
  size_t auto_bucket_bytes_ = static_cast<size_t>(256) << 20;
  uint64_t opt_version_ = 1;   // bumped whenever a hyper-parameter / multiplier changes
  uint64_t layout_epoch_ = 1;  // bumped whenever placement / optimizer kind / updater changes
  std::string gc_type_ = "none";
  friend struct PlanBuilder;
};

}  // namespace b200kv
