// rowsparse.cc -- host side of row_sparse push / row_sparse_pull (KVStore members).
//
// Reference flow: CommDevice::ReduceRowSparse (src/kvstore/comm.h:478-501) copies every source to
// the owner GPU and sums there; KVStoreLocal::PullRowSparseImpl / Unique (kvstore_local.h:263-283,
// 428-472) sort+unique the requested ids and CommDevice::BroadcastRowSparse (comm.h:618-674)
// retains those rows. Here the owner GPU reads the peers' rows directly over NVLink (no staging
// copies of values), and the union works on the ids present, not on a table-high flag array.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <iostream>
#include <map>

#include "group.h"
#include "kvstore.h"
#include "rowsparse.h"
#include "scalar_parse.h"

namespace b200kv {

namespace {

// The device produces row counts; the host needs them only to set an array's aux shape (the
// reference blocks on the same values: ndarray_function.cu:158-166, kvstore_utils.cu:77-85).
// Counts are copied into pinned memory behind an event, so kernels queued after the copy are
// already running while the host waits for the numbers.
struct CountFence {
  int dev;
  int64_t* host;
  size_t n;
  cudaEvent_t ev = nullptr;
  CountFence(int d, size_t count) : dev(d), n(count) {
    host = static_cast<int64_t*>(Engine::Get()->AllocPinned(n * sizeof(int64_t)));
  }
  ~CountFence() {
    if (ev) cudaEventDestroy(ev);
    Engine::Get()->FreePinned(host, n * sizeof(int64_t));
  }
  void Post(const int64_t* d_counts, cudaStream_t st) {
    DeviceGuard g(dev);
    KV_CUDA(cudaMemcpyAsync(host, d_counts, n * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    KV_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    KV_CUDA(cudaEventRecord(ev, st));
  }
  const int64_t* Wait() {
    KV_CUDA(cudaEventSynchronize(ev));
    return host;
  }
};

int BitsFor(int64_t n) {  // bits that hold every id in [0, n)
  int b = 1;
  while (b < 62 && (int64_t{1} << b) < n) ++b;
  return b;
}

// The union's inputs: the sources that hold rows, in the order given.
RspSources LocalSources(const std::vector<NDArray>& srcs) {
  RspSources S;
  int64_t total = 0;
  for (auto& s : srcs) {
    if (!s.storage_initialized()) continue;  // all-zero source
    S.idx[S.nsrc] = s.row_ids();
    S.val[S.nsrc] = static_cast<const float*>(s.data());
    S.start[S.nsrc] = total;
    total += s.nnr();
    ++S.nsrc;
  }
  S.start[S.nsrc] = total;
  return S;
}

// One rank per GPU: the union's inputs are every rank's gradient, read through IPC in rank order
// (the reference's value-list order). `*src` becomes this rank's gradient, copied into the IPC arena
// when the peers cannot address it where it is. Addresses and row counts change every step, so
// they travel by a host all-gather on every push.
RspSources RankSources(PeerGroup* g, int64_t key, const NDArray& src_in, NDArray* src) {
  *src = src_in;
  if (!src->on_gpu() || src->dev() != g->dev() ||
      (src->storage_initialized() && !(g->InArena(src->data()) && g->InArena(src->row_ids())))) {
    *src = src_in.Copy(Context::GPU(g->dev()));
  }
  const int64_t my_nnr = src->storage_initialized() ? src->nnr() : 0;
  if (my_nnr > 0) {
    KV_CHECK(g->InArena(src->data()) && g->InArena(src->row_ids()))
        << "IPC arena exhausted; raise B200KV_IPC_ARENA_MB";
  }
  const std::vector<int64_t> all = g->AllGatherI64(
      {my_nnr > 0 ? g->OffsetOf(src->row_ids()) : 0, my_nnr > 0 ? g->OffsetOf(src->data()) : 0, my_nnr, key});
  RspSources S;
  int64_t total = 0;
  for (int r = 0; r < g->world(); ++r) {
    KV_CHECK_EQ(all[4 * r + 3], key) << "one-rank-per-GPU store: rank " << r << " pushed a different row_sparse key";
    const int64_t n = all[4 * r + 2];
    if (n == 0) continue;
    S.idx[S.nsrc] = static_cast<const int64_t*>(g->PeerPtr(r, all[4 * r]));
    S.val[S.nsrc] = static_cast<const float*>(g->PeerPtr(r, all[4 * r + 1]));
    S.start[S.nsrc] = total;
    total += n;
    ++S.nsrc;
  }
  S.start[S.nsrc] = total;
  return S;
}

}  // namespace

// A dense key takes row_sparse values too (a dense weight with a sparse gradient: gluon's
// Embedding(sparse_grad=True) under Trainer). The merge is the same; the update target, its state
// and the callback's `local` are then the key's whole dense weight on `home`, which has the layout
// of a table holding every row. Without an updater the key's value becomes the merged row_sparse
// array (kvstore_local.h:237-243) until a dense push makes it dense again.
void KVStore::PushRowSparse(KeyEntry& e, const std::vector<NDArray>& srcs_in) {
  const bool dense_key = e.stype == kDefaultStorage;
  // every refusal comes before anything is enqueued: value and state stay as they were
  KV_CHECK_EQ(e.dtype, kFloat32) << (dense_key ? "row_sparse values pushed to a dense key are float32 on this path"
                                               : "row_sparse keys are float32 on this path");
  KV_CHECK(srcs_in.size() <= static_cast<size_t>(kMaxSrc));
  for (auto& s : srcs_in) {
    KV_CHECK(s.shape() == e.shape) << "push: shape mismatch for row_sparse key " << e.key;
    KV_CHECK_EQ(s.dtype(), e.dtype) << "push: dtype mismatch for key " << e.key;
  }
  if (dense_key) {
    KV_CHECK(!dist_) << "key " << e.key << " was initialised dense: the one-rank-per-GPU store takes "
                     << "dense values for it only";
    KV_CHECK(!nccl_type_) << "kvstore 'nccl' does not take row_sparse values (src/kvstore/kvstore_nccl.h:93-94)";
    KV_CHECK(!opt_.enabled || opt_.kind == kOptSGD || opt_.kind == kOptAdam)
        << "the store's fused optimizer takes row_sparse values for sgd and adam only";
  }
  Engine* eng = Engine::Get();
  DetachAnchor(e);  // the dense weight is updated, or replaced by a row_sparse value, below
  if (dist_ && e.home < 0) e.home = PeerGroup::Get()->dev();
  if (dense_key && e.striped) EnsureWhole(e, devset_[0]);   // state included; dense pushes restripe it
  if (e.home < 0) {
    int pick = 0;
    for (auto& s : srcs_in) {
      if (s.on_gpu()) { pick = s.dev(); break; }
    }
    if (dense_key) EnsureOnDevice(e, pick); else e.home = pick;
  }
  const int home = e.home;
  const bool callback = updater_ != nullptr && !opt_.enabled;
  if (dense_key && (opt_.enabled || callback)) DensifyValue(e);   // the update reads the dense weight
  if (!dense_key && !e.rsp.on_gpu()) e.rsp = e.rsp.Copy(Context::GPU(home));
  // the update target: the row_sparse table, or the dense weight
  const NDArray W = dense_key ? e.dev[home].w : e.rsp;
  std::vector<NDArray> srcs;
  std::vector<int> parts{home};
  for (auto& s : srcs_in) {
    if (!s.on_gpu()) {
      srcs.push_back(s.Copy(Context::GPU(home)));
    } else {
      srcs.push_back(s);
      if (std::find(parts.begin(), parts.end(), s.dev()) == parts.end()) parts.push_back(s.dev());
    }
  }
  eng->RequirePeerAccess(parts);
  // ---- union of ids + ordered sum, all on the owner's stream, row count left on the device
  const RspSources S = LocalSources(srcs);
  int64_t total = S.start[S.nsrc];
  NDArray merged = NDArray::RowSparse(e.shape, Context::GPU(home), e.dtype);
  const int64_t row_len = static_cast<int64_t>(W.RowLength());
  const bool on_store = opt_.enabled && (opt_.kind == kOptSGD || opt_.kind == kOptAdam);
  // lazy: the optimizer step is fused into the row-sum kernel. standard (lazy_update=False): the
  // merged gradient is materialised, then every row of the table is updated (SgdAdamRspUpdate).
  const bool fused = on_store && opt_.lazy_update;
  RspUpdateLaunch U;
  if (on_store) {
    KV_CHECK(dense_key || !e.rsp_devs.empty() || e.rsp_group || e.rsp.nnr() == e.shape[0])
        << "key " << e.key << ": the stored row_sparse weight must hold every row for sparse "
        << "optimizer updates (initialise it from a dense weight, as gluon does)";
    // Optimizer._update_count, then SGD._update_impl's non-aggregated branch / Adam.update
    auto it = opt_.count.find(e.key);
    int c = (it == opt_.count.end() ? opt_.begin_num_update : it->second) + 1;
    opt_.count[e.key] = c;
    opt_.num_update = std::max(opt_.num_update, c);
    if (total == 0 && fused && !dist_) return;   // a lazy update with an all-zero gradient touches nothing
    auto lm = opt_.lr_mult.find(e.key);
    auto wm = opt_.wd_mult.find(e.key);
    double lrd = opt_.lr * (lm == opt_.lr_mult.end() ? 1.0 : lm->second);
    double wdd = opt_.wd * (wm == opt_.wd_mult.end() ? 1.0 : wm->second);
    DevState& s = e.dev[home];
    const bool sharded_now = !e.rsp_devs.empty() || e.rsp_group || (dist_ && fused);   // state lives with the shards
    auto zero_state = [&](NDArray* a) {
      if (a->is_none() && !sharded_now) *a = ZerosOn(e.shape, home, kFloat32);
    };
    if (opt_.kind == kOptSGD) {
      U.opt = opt_.momentum != 0.0 ? kOptSGD : kOptSGDSingle;  // sgd_mom_update / sgd_update
      if (opt_.momentum != 0.0) zero_state(&s.s1);
      U.momentum = opt_.momentum > 0 ? ScalarParam(opt_.momentum) : 0.f;
    } else {
      U.opt = kOptAdam;
      zero_state(&s.s1);
      zero_state(&s.s2);
      const double coef1 = 1.0 - std::pow(opt_.beta1, c), coef2 = 1.0 - std::pow(opt_.beta2, c);
      lrd *= std::sqrt(coef2) / coef1;
      U.beta1 = ScalarParam(opt_.beta1);
      U.beta2 = ScalarParam(opt_.beta2);
      U.eps = ScalarParam(opt_.eps);
    }
    U.lr = ScalarParam(lrd);
    U.wd = ScalarParam(wdd);
    U.rescale = ScalarParam(opt_.rescale);
    U.clip = opt_.clip != 0.0 ? ScalarParam(opt_.clip) : -1.f;
    U.w = sharded_now ? nullptr : static_cast<float*>(W.data());
    U.s1 = s.s1.is_none() ? nullptr : static_cast<float*>(s.s1.data());
    U.s2 = s.s2.is_none() ? nullptr : static_cast<float*>(s.s2.data());
  }
  if (dist_) {
    KV_CHECK(!nccl_) << "kvstore 'nccl' handles dense keys only, as the reference's does "
                     << "(src/kvstore/kvstore_nccl.h:62-70); use kvstore 'device' for row_sparse keys";
    KV_CHECK_EQ(srcs.size(), 1u) << "one-rank-per-GPU store: push one row_sparse value per key and rank";
    if (fused) {
      PushRowSparseGroup(e, srcs[0], U);   // table and optimizer state sharded by row range
      return;
    }
    merged = MergeRowSparseGroup(e, srcs[0]);
    total = 0;   // the merge is done: skip the single-process union below
  }
  if (fused && !dense_key && total > 0 && parts.size() >= 2) {
    // sources on several GPUs: every GPU merges and updates its own row range of the table
    if (PushRowSparseSharded(e, srcs, parts, U)) return;
  }
  if (!e.rsp_devs.empty()) UnshardRsp(e);
  if (fused) {   // (re)bind the update to the whole table on `home`
    DevState& hs = e.dev[home];
    U.w = static_cast<float*>(W.data());
    U.s1 = hs.s1.is_none() ? nullptr : static_cast<float*>(hs.s1.data());
    U.s2 = hs.s2.is_none() ? nullptr : static_cast<float*>(hs.s2.data());
  }
  if (total > 0) {
    const int bits = BitsFor(e.shape[0]);
    NDArray d_nnr({1}, Context::GPU(home), kInt64);
    NDArray ws({static_cast<int64_t>(RspMergeWorkspaceBytes(total, bits, S.nsrc))}, Context::GPU(home), kUint8);
    // fused: the summed rows are consumed in registers by the optimizer step, nothing is stored
    if (!fused) merged.CheckAndAllocRows(total);  // upper bound; nnr is set once the count is known
    // the sources are read on their own lanes; the joins order those lanes around the home lane's work
    for (auto& s : srcs) eng->BeginRead(s.dev(), *s.var());
    LaneOp op(home);
    if (fused) op.Write(W).Write(e.dev[home].s1).Write(e.dev[home].s2);
    else op.Write(merged);
    op.Write(d_nnr).Write(ws);
    if (parts.size() > 1) eng->JoinStreams(parts);
    LaunchRspMerge(S, bits, row_len, fused ? nullptr : merged.row_ids(),
                   fused ? nullptr : static_cast<float*>(merged.data()),
                   static_cast<int64_t*>(d_nnr.data()), ws.data(), ws.ByteSize(), op.stream(), fused ? &U : nullptr);
    eng->CountLaunch("rsp_merge(tag, sort, heads)", total * 24);
    eng->CountLaunch(fused ? "rsp_sum+update" : "rsp_sum", static_cast<uint64_t>(total) * row_len * 4 * 2);
    if (parts.size() > 1) eng->JoinStreams(parts);
    const uint64_t seq = op.Issue();
    for (auto& s : srcs) {
      uint64_t sq = s.dev() == home ? seq : eng->Issue(s.dev());
      eng->MarkRead(s.dev(), sq, s.var());
    }
    if (!fused) {
      CountFence f(home, 1);
      f.Post(static_cast<const int64_t*>(d_nnr.data()), op.stream());
      merged.SetNnr(f.Wait()[0]);
    }
  }
  if (fused) return;
  if (on_store) {
    DevState& ds = e.dev[home];
    UpdateLaunch L;
    L.lr = U.lr;
    L.wd = U.wd;
    L.momentum = U.momentum;
    L.rescale = U.rescale;
    L.clip = U.clip;
    L.beta1 = U.beta1;
    L.beta2 = U.beta2;
    L.eps = U.eps;
    SgdAdamRspUpdate(U.opt, false, L, W, merged, {ds.s1, ds.s2});
    return;
  }
  if (callback) {
    NDArray* recv_h = new NDArray(merged);
    NDArray* local_h = new NDArray(dense_key ? W.Reshaped(e.shape) : W);
    if (key_type_ == 0 && str_updater_ != nullptr) {
      str_updater_(reverse_str_key_dict_[e.key].c_str(), recv_h, local_h, updater_handle_);
    } else {
      updater_(e.key, recv_h, local_h, updater_handle_);
    }
    return;
  }
  e.rsp = merged;  // no updater: local = merged (kvstore_local.h:237-243)
  if (e.vstype != kRowSparseStorage) {
    e.vstype = kRowSparseStorage;
    ++layout_epoch_;   // cached dense pulls of the key must not replay
  }
}

// row_sparse_pull (KVStoreLocal::PullRowSparseImpl kvstore_local.h:263-283, Unique :428-472,
// CommDevice::BroadcastRowSparse comm.h:618-674): every (key, out, row_ids) triple gets the
// ascending unique ids requested and the stored rows for them. All triples that share an owner
// GPU go through ONE sort/unique and ONE retain kernel; the per-output counts come back through
// a CountFence while the retain kernel is already running.
void KVStore::PullRowSparse(const std::vector<int>& keys, const std::vector<NDArray>& outs,
                            const std::vector<NDArray>& row_ids, int) {
  Flush();
  KV_CHECK_EQ(keys.size(), outs.size());
  KV_CHECK_EQ(keys.size(), row_ids.size());
  // GroupKVPairsPullRsp (kvstore_local.h:352-371): stable by key, storage types validated
  std::vector<size_t> order(keys.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return keys[a] < keys[b]; });
  for (size_t i : order) {
    KV_CHECK_EQ(outs[i].stype(), kRowSparseStorage)
        << "Expected row_sparse storage type for row_sparse_pull values, but detected storage type "
        << outs[i].stype();
    KV_CHECK_EQ(row_ids[i].stype(), kDefaultStorage)
        << "Expected default storage type for row_sparse_pull rowids, but detected storage type "
        << row_ids[i].stype();
  }
  Engine* eng = Engine::Get();
  std::map<int, std::vector<size_t>> by_home;  // owner GPU -> triples, in key order
  for (size_t i : order) {
    KeyEntry& e = Entry(keys[i]);
    KV_CHECK_EQ(e.vstype, kRowSparseStorage) << "PullRowSparse expects row_sparse src NDArray";
    const NDArray& out = outs[i];
    if (e.home < 0) e.home = out.on_gpu() ? out.dev() : (row_ids[i].on_gpu() ? row_ids[i].dev() : 0);
    const bool sharded = !e.rsp_devs.empty() || e.rsp_group;
    if (!sharded && !e.rsp.on_gpu()) e.rsp = e.rsp.Copy(Context::GPU(e.home));
    KV_CHECK(out.shape() == e.shape) << "row_sparse_pull: out shape mismatch for key " << e.key;
    KV_CHECK_EQ(out.dtype(), e.dtype) << "row_sparse_pull: out dtype mismatch for key " << e.key;
    if (out.SameStorage(e.rsp)) {
      std::cerr << "The output of row_sparse_pull() on key " << e.key << " refers to the same NDArray "
                << "as the one stored in KVStore. Consider a new NDArray buffer for the output.\n";
    }
    if (row_ids[i].Size() == 0 || (!sharded && !e.rsp.storage_initialized())) {
      // FillZerosRspImpl (sparse_retain-inl.h:271-275)
      eng->WaitToWrite(*out.var());
      out.SetNnr(0);
      continue;
    }
    // a sharded table has no single owner: the gather runs where the output lives
    by_home[sharded && out.on_gpu() ? out.dev() : e.home].push_back(i);
  }
  std::vector<std::function<void()>> finish;
  for (auto& kv : by_home) finish.push_back(PullRowSparseGroup(kv.first, kv.second, keys, outs, row_ids));
  for (auto& f : finish) f();
}

std::function<void()> KVStore::PullRowSparseGroup(int home, const std::vector<size_t>& which,
                                                  const std::vector<int>& keys,
                                                  const std::vector<NDArray>& outs,
                                                  const std::vector<NDArray>& row_ids) {
  Engine* eng = Engine::Get();
  const int nitems = static_cast<int>(which.size());
  std::vector<RetainItem> items(nitems);
  std::vector<NDArray> ids(nitems), targets(nitems);
  std::vector<int> parts{home};
  auto add_part = [&](int d) {
    if (std::find(parts.begin(), parts.end(), d) == parts.end()) parts.push_back(d);
  };
  int64_t total = 0;
  int id_bits = 1;
  for (int k = 0; k < nitems; ++k) {
    const size_t i = which[k];
    KeyEntry& e = Entry(keys[i]);
    const NDArray& out = outs[i];
    // ids are read in place when they live on a GPU (peer load), else copied to the owner
    ids[k] = row_ids[i].on_gpu() ? row_ids[i] : row_ids[i].Copy(Context::GPU(home));
    add_part(ids[k].dev());
    // rows go straight into `out` when it lives on a GPU (peer store over NVLink)
    targets[k] = out.on_gpu() ? out : NDArray::RowSparse(e.shape, Context::GPU(home), e.dtype);
    add_part(targets[k].dev());
    const int64_t n = static_cast<int64_t>(ids[k].Size());
    if (!targets[k].RowsFit(n)) eng->WaitToWrite(*targets[k].var());  // buffers get re-allocated
    targets[k].CheckAndAllocRows(n);       // upper bound; nnr is set once the count is known
    RetainItem& it = items[k];
    it.ids = ids[k].data();
    it.ids_dtype = ids[k].dtype();
    it.n = n;
    it.start = total;
    if (!e.rsp_devs.empty() || e.rsp_group) {
      it.src_idx = nullptr;
      it.src_val = nullptr;
      it.src_nnr = e.shape[0];
      it.src_dense_rows = 1;
      it.shard_vbase = RspShardTable(e, home);
      it.rows_per_shard = e.rsp_rows_per;
      it.row_len = static_cast<int64_t>(e.rsp_shards[0].RowLength());
      for (int d : e.rsp_devs) add_part(d);
    } else {
      it.src_idx = e.rsp.row_ids();
      it.src_val = static_cast<const float*>(e.rsp.data());
      it.src_nnr = e.rsp.nnr();
      it.src_dense_rows = e.rsp.nnr() == e.shape[0] ? 1 : 0;  // sparse_retain-inl.h:290
      it.row_len = static_cast<int64_t>(e.rsp.RowLength());
    }
    it.out_idx = targets[k].row_ids();
    it.out_val = static_cast<float*>(targets[k].data());
    total += n;
    id_bits = std::max(id_bits, BitsFor(e.shape[0]));
  }
  eng->RequirePeerAccess(parts);
  auto fence = std::make_shared<CountFence>(home, nitems + 1);
  NDArray d_off({nitems + 1}, Context::GPU(home), kInt64);
  NDArray ws({static_cast<int64_t>(RetainBatchWorkspaceBytes(nitems, total, id_bits))}, Context::GPU(home), kUint8);
  // every dependency is taken on the lane that runs the kernels (`home`): arrays on other GPUs are
  // reached through peer access, their writers / readers are waited for by events -- no stream
  // join, so groups that run on different GPUs do not serialise each other
  LaneOp op(home);
  for (int k = 0; k < nitems; ++k) {
    KeyEntry& ek = Entry(keys[which[k]]);
    op.Read(ids[k]);
    if (ek.rsp_devs.empty() && !ek.rsp_group) {
      op.Read(ek.rsp);
    } else {
      for (auto& sh : ek.rsp_shards) op.Read(sh);
    }
    op.Write(targets[k]);
  }
  op.Write(d_off).Write(ws);
  LaunchUniqueBatch(items.data(), nitems, total, id_bits, static_cast<int64_t*>(d_off.data()),
                    ws.data(), ws.ByteSize(), op.stream());
  eng->CountLaunch("unique_batch(gather, sort, unique, bounds)", total * 32);
  fence->Post(static_cast<const int64_t*>(d_off.data()), op.stream());
  LaunchRetainBatch(nitems, total, id_bits, static_cast<const int64_t*>(d_off.data()), ws.data(), op.stream());
  uint64_t bytes = 0;
  for (auto& it : items) bytes += static_cast<uint64_t>(it.n) * (it.row_len * 8 + 16);
  eng->CountLaunch("sparse_retain", bytes);
  op.Issue();
  // the counts are awaited by the caller AFTER every group of the call has been launched
  std::vector<NDArray> outs_k(nitems);
  for (int k = 0; k < nitems; ++k) outs_k[k] = outs[which[k]];
  return [fence, targets, outs_k, d_off, ws, nitems]() {
    const int64_t* off = fence->Wait();
    for (int k = 0; k < nitems; ++k) {
      targets[k].SetNnr(off[k + 1] - off[k]);
      if (!outs_k[k].on_gpu()) CopyFromTo(targets[k], outs_k[k]);
    }
  };
}

// =================================================================================================
// standard (non-lazy) updates and storage casts
// =================================================================================================
NDArray BuildRowMap(LaneOp& op, const NDArray& g, int64_t rows) {
  NDArray row_map({rows}, Context::GPU(g.dev()), kInt32);
  op.Write(row_map);
  const bool stored = g.storage_initialized();
  LaunchRowMap(stored ? g.row_ids() : nullptr, stored ? g.nnr() : 0, rows,
               static_cast<int32_t*>(row_map.data()), op.stream());
  return row_map;
}

namespace {

void SetStates(UpdateLaunch& L, const std::vector<NDArray>& states) {
  KV_CHECK(states.size() <= 3) << "an optimizer step takes at most three states";
  for (size_t i = 0; i < states.size(); ++i) {
    L.s[i] = states[i].is_none() ? nullptr : static_cast<float*>(states[i].data());
  }
}

}  // namespace

void RunRspRowUpdate(UpdateLaunch L, const NDArray& w, const NDArray& g, const std::vector<NDArray>& states,
                     const char* launch_name, int bytes_per_elem) {
  KV_CHECK(w.on_gpu() && g.on_gpu() && w.dev() == g.dev()) << "all operands must be on the same GPU";
  KV_CHECK_EQ(w.dtype(), kFloat32) << "row_sparse optimizer updates are float32";
  if (!g.storage_initialized()) return;  // an all-zero gradient changes nothing
  LaneOp op(w.dev());
  op.Read(g).Write(w);
  for (const NDArray& s : states) op.Write(s);
  L.dtype = kFloat32;
  L.w = w.data();
  L.out = w.data();
  L.g = g.data();
  L.gidx = g.row_ids();
  L.nnr = g.nnr();
  L.row_len = static_cast<int64_t>(w.RowLength());
  SetStates(L, states);
  LaunchRspRowUpdateOp(L, op.stream());
  // + 8 B of id per row, and GroupAdaGrad's history value read and written
  const int64_t per_row = L.op == kUpdGroupAdaGrad ? 16 : 8;
  Engine::Get()->CountLaunch(launch_name, static_cast<uint64_t>(L.nnr) * (bytes_per_elem * L.row_len + per_row));
  op.Issue();
}

void RunRspGradUpdate(UpdateLaunch L, const NDArray& w, const NDArray& g, const std::vector<NDArray>& states,
                      const NDArray& out, const char* launch_name, int bytes_per_elem) {
  KV_CHECK(w.on_gpu() && g.on_gpu() && w.dev() == g.dev()) << "all operands must be on the same GPU";
  KV_CHECK_EQ(w.dtype(), kFloat32) << "row_sparse optimizer updates are float32";
  KV_CHECK_EQ(g.stype(), kRowSparseStorage);
  const int64_t rows = w.shape()[0];
  if (w.stype() == kRowSparseStorage) {
    // CheckAllRowsPresent (optimizer_op-inl.h:532-536)
    KV_CHECK_EQ(w.nnr(), rows) << "standard sparse update: the row_sparse weight must hold every row";
  }
  const bool out_is_w = out.SameStorage(w);
  LaneOp op(w.dev());
  op.Read(g);
  if (!out_is_w) op.Read(w);
  op.Write(out);
  for (const NDArray& s : states) op.Write(s);
  // the stored rows through a row map, every element of the table updated; an empty gradient is
  // a full update with g = +0.0f
  const NDArray row_map = BuildRowMap(op, g, rows);
  L.dtype = kFloat32;
  L.w = w.data();
  L.out = out.data();
  L.out_is_w = out_is_w;
  L.n = w.Size();
  L.g = g.storage_initialized() ? g.data() : nullptr;
  L.nnr = g.nnr();
  L.row_len = static_cast<int64_t>(w.RowLength());
  L.row_map = static_cast<const int32_t*>(row_map.data());
  SetStates(L, states);
  LaunchRspGradUpdateOp(L, op.stream());
  // bytes: the scatter reads an 8 B id and writes 4 B per stored row; the update moves the dense
  // pass's bytes less the gradient's 4 B per element, reads the stored rows once, and counts the
  // row map's memset and read (4 B each per table row)
  if (L.nnr > 0) Engine::Get()->CountLaunch("update_op(row_map_scatter)", static_cast<uint64_t>(L.nnr) * 12);
  Engine::Get()->CountLaunch(launch_name, static_cast<uint64_t>(bytes_per_elem - 4) * L.n +
                                              static_cast<uint64_t>(L.nnr) * L.row_len * 4 +
                                              static_cast<uint64_t>(rows) * 8);
  op.Issue();
}

void SgdAdamRspUpdate(int kind, bool lazy, UpdateLaunch L, const NDArray& w, const NDArray& g,
                      const std::vector<NDArray>& states) {
  // g 4 + w 8, + 8 per state
  const int bytes = kind == kOptAdam ? 28 : kind == kOptSGD ? 20 : 12;
  if (kind == kOptSGD) {
    L.op = kUpdSGDMom;
  } else if (kind == kOptAdam) {
    L.op = lazy ? kUpdAdamLazy : kUpdAdamStd;
  } else {
    L.op = lazy ? kUpdSGD : kUpdSGDStd;
  }
  if (lazy) {
    RunRspRowUpdate(L, w, g, states, "rsp_update", bytes);
  } else {
    RunRspGradUpdate(L, w, g, states, w, "rsp_std_update", bytes);
  }
}

void SumRowSparse(const std::vector<NDArray>& in, const NDArray& out) {
  const int dev = out.dev();
  Engine* eng = Engine::Get();
  std::vector<NDArray> srcs;
  bool out_is_input = false;
  for (const NDArray& a : in) {
    out_is_input = out_is_input || a.SameStorage(out);
    if (a.storage_initialized()) srcs.push_back(a);
  }
  if (srcs.empty()) {  // every input is all zeros: out stores no rows, nothing is launched
    LaneOp op(dev);
    op.Write(out);
    op.Issue();
    out.SetNnr(0);
    return;
  }
  const int bits = BitsFor(out.shape()[0]);
  const int64_t row_len = static_cast<int64_t>(out.RowLength());
  NDArray acc;  // the sum so far
  for (size_t next = 0; next < srcs.size();) {
    std::vector<NDArray> group;
    if (!acc.is_none()) group.push_back(acc);
    while (group.size() < static_cast<size_t>(kMaxSrc) && next < srcs.size()) group.push_back(srcs[next++]);
    const bool last = next == srcs.size();
    const NDArray target = last && !out_is_input ? out : NDArray::RowSparse(out.shape(), Context::GPU(dev), kFloat32);
    const RspSources S = LocalSources(group);
    const int64_t total = S.start[S.nsrc];
    target.CheckAndAllocRows(total);  // upper bound; nnr is set once the count is known
    NDArray d_nnr({1}, Context::GPU(dev), kInt64);
    NDArray ws({static_cast<int64_t>(RspMergeWorkspaceBytes(total, bits, S.nsrc))}, Context::GPU(dev), kUint8);
    LaneOp op(dev);
    for (const NDArray& g : group) op.Read(g);
    op.Write(target).Write(d_nnr).Write(ws);
    LaunchRspMerge(S, bits, row_len, target.row_ids(), static_cast<float*>(target.data()),
                   static_cast<int64_t*>(d_nnr.data()), ws.data(), ws.ByteSize(), op.stream());
    eng->CountLaunch("rsp_merge(tag, sort, heads)", total * 24);
    eng->CountLaunch("rsp_sum", static_cast<uint64_t>(total) * row_len * 4 * 2);
    op.Issue();
    CountFence f(dev, 1);
    f.Post(static_cast<const int64_t*>(d_nnr.data()), op.stream());
    target.SetNnr(f.Wait()[0]);
    acc = target;
  }
  if (!acc.SameStorage(out)) CopyFromTo(acc, out);
}

void CastStorageCopy(const NDArray& from_in, const NDArray& to) {
  KV_CHECK(from_in.stype() == kDefaultStorage || to.stype() == kDefaultStorage)
      << "Copying ndarray of stype = " << from_in.stype() << " to stype = " << to.stype()
      << " is not supported";
  KV_CHECK_EQ(from_in.dtype(), kFloat32) << "storage casts are float32 on this path";
  KV_CHECK(from_in.shape() == to.shape()) << "CopyFromTo: operands shape mismatch";
  Engine* eng = Engine::Get();
  const int dev = from_in.on_gpu() ? from_in.dev() : (to.on_gpu() ? to.dev() : 0);
  NDArray from = from_in.on_gpu() && from_in.dev() == dev ? from_in : from_in.Copy(Context::GPU(dev));
  const int64_t rows = from.shape()[0];
  const int64_t row_len = static_cast<int64_t>(from.RowLength());
  DeviceGuard guard(dev);
  cudaStream_t st = eng->Stream(dev);
  if (to.stype() == kDefaultStorage) {
    // row_sparse -> dense (CastStorageRspDnsImpl): zeros, then the stored rows
    NDArray target = to.on_gpu() && to.dev() == dev ? to : NDArray(to.shape(), Context::GPU(dev), to.dtype());
    LaneOp op(dev);
    op.Read(from).Write(target);
    KV_CUDA(cudaMemsetAsync(target.data(), 0, target.ByteSize(), st));
    if (from.storage_initialized()) {
      LaunchRspScatterRows(from.row_ids(), static_cast<const float*>(from.data()), from.nnr(), row_len,
                           static_cast<float*>(target.data()), st);
    }
    eng->CountLaunch("cast_storage(rsp->dns)", target.ByteSize());
    op.Issue();
    if (!target.SameStorage(to)) CopyFromTo(target, to);
    return;
  }
  // dense -> row_sparse (CastStorageDnsRspImpl): rows with any element != 0, ascending
  NDArray target = to.on_gpu() && to.dev() == dev ? to : NDArray::RowSparse(to.shape(), Context::GPU(dev), to.dtype());
  if (rows == 0 || row_len == 0) {
    eng->WaitToWrite(*to.var());
    to.SetNnr(0);
    return;
  }
  NDArray ids({rows}, Context::GPU(dev), kInt64);
  NDArray cnt({1}, Context::GPU(dev), kInt64);
  NDArray ws({static_cast<int64_t>(NonzeroRowsWorkspaceBytes(rows))}, Context::GPU(dev), kUint8);
  {
    LaneOp op(dev);
    op.Read(from).Write(ids).Write(cnt).Write(ws);
    LaunchNonzeroRows(static_cast<const float*>(from.data()), rows, row_len,
                      static_cast<int64_t*>(ids.data()), static_cast<int64_t*>(cnt.data()), ws.data(),
                      ws.ByteSize(), st);
    eng->CountLaunch("cast_storage(nonzero rows)", from.ByteSize());
    op.Issue();
  }
  CountFence f(dev, 1);
  f.Post(static_cast<const int64_t*>(cnt.data()), st);
  const int64_t nnr = f.Wait()[0];
  eng->WaitToWrite(*target.var());
  if (nnr == 0) {
    target.SetNnr(0);
  } else {
    target.CheckAndAllocRows(nnr);
    // gather = retain with a source that holds every row
    RetainItem it{};
    it.ids = ids.data();
    it.ids_dtype = kInt64;
    it.n = nnr;
    it.start = 0;
    it.src_idx = nullptr;
    it.src_val = static_cast<const float*>(from.data());
    it.src_nnr = rows;
    it.src_dense_rows = 1;
    it.row_len = row_len;
    it.out_idx = target.row_ids();
    it.out_val = static_cast<float*>(target.data());
    NDArray off({2}, Context::GPU(dev), kInt64);
    const int id_bits = BitsFor(rows);
    NDArray rws({static_cast<int64_t>(RetainBatchWorkspaceBytes(1, nnr, id_bits))}, Context::GPU(dev), kUint8);
    LaneOp op(dev);
    op.Read(from).Read(ids).Write(target).Write(off).Write(rws);
    LaunchUniqueBatch(&it, 1, nnr, id_bits, static_cast<int64_t*>(off.data()), rws.data(), rws.ByteSize(), st);
    LaunchRetainBatch(1, nnr, id_bits, static_cast<const int64_t*>(off.data()), rws.data(), st);
    eng->CountLaunch("cast_storage(dns->rsp gather)", static_cast<uint64_t>(nnr) * row_len * 8);
    op.Issue();
  }
  if (!target.SameStorage(to)) CopyFromTo(target, to);
}

void BroadcastRspValue(const NDArray& src, const std::vector<NDArray>& outs) {
  KV_CHECK(src.on_gpu() && src.stype() == kRowSparseStorage);
  // the checks CopyFromTo and CastStorageCopy make, for every out before any is written
  for (auto& o : outs) {
    KV_CHECK(!o.is_none()) << "copy of an empty NDArray";
    KV_CHECK_EQ(src.dtype(), o.dtype()) << "CopyFromTo: dtype mismatch";
    if (o.stype() == kDefaultStorage) {
      KV_CHECK_EQ(src.dtype(), kFloat32) << "storage casts are float32 on this path";
      KV_CHECK(src.shape() == o.shape()) << "CopyFromTo: operands shape mismatch";
    } else {
      KV_CHECK_EQ(o.stype(), kRowSparseStorage) << "CopyFromTo: unsupported storage type " << o.stype();
      KV_CHECK(src.shape() == o.shape()) << "CopyFromTo: row_sparse shape mismatch";
    }
  }
  Engine* eng = Engine::Get();
  const int home = src.dev();
  const int64_t nnr = src.storage_initialized() ? src.nnr() : 0;
  for (size_t b = 0; b < outs.size(); b += kMaxDst) {
    const size_t e = std::min(outs.size(), b + kMaxDst);
    RspBroadcastLaunch L;
    L.src_idx = nnr > 0 ? src.row_ids() : nullptr;
    L.src_val = nnr > 0 ? src.data() : nullptr;
    L.nnr = nnr;
    L.rows = src.shape()[0];
    L.row_bytes = static_cast<int64_t>(src.RowLength() * DTypeSize(src.dtype()));
    std::vector<NDArray> targets, staged;   // staged[i]: host out of targets[i], or none
    std::vector<int> parts{home};
    for (size_t i = b; i < e; ++i) {
      const NDArray& o = outs[i];
      if (o.SameStorage(src)) continue;     // self-copy (ndarray.cc:1199-1203)
      const bool rsp = o.stype() == kRowSparseStorage;
      if (rsp && nnr == 0) {                // CopyFromToRspImpl of an all-zero value
        eng->WaitToWrite(*o.var());
        o.SetNnr(0);
        continue;
      }
      NDArray t = o.on_gpu() ? o
                 : rsp ? NDArray::RowSparse(o.shape(), Context::GPU(home), o.dtype())
                       : NDArray(o.shape(), Context::GPU(home), o.dtype());
      if (rsp) {
        if (!t.RowsFit(nnr)) eng->WaitToWrite(*t.var());  // buffers get re-allocated
        t.CheckAndAllocRows(nnr);
        L.rsp_idx[L.n_rsp] = t.row_ids();
        L.rsp_val[L.n_rsp++] = t.data();
      } else {
        L.dns[L.n_dns++] = t.data();
      }
      if (std::find(parts.begin(), parts.end(), t.dev()) == parts.end()) parts.push_back(t.dev());
      targets.push_back(t);
      staged.push_back(o.on_gpu() ? NDArray() : o);
    }
    if (targets.empty()) continue;
    eng->RequirePeerAccess(parts);
    LaneOp op(home);
    op.Read(src);
    for (auto& t : targets) op.Write(t);
    LaunchRspBroadcast(L, op.stream());
    eng->CountLaunch("rsp_broadcast", static_cast<uint64_t>(nnr) * L.row_bytes +
                                          static_cast<uint64_t>(L.n_rsp) * nnr * (L.row_bytes + 8) +
                                          static_cast<uint64_t>(L.n_dns) * L.rows * L.row_bytes);
    op.Issue();
    for (size_t k = 0; k < targets.size(); ++k) {
      if (!staged[k].is_none()) CopyFromTo(targets[k], staged[k]);
    }
  }
}

// =================================================================================================
// row-range sharding of a row_sparse table over the GPUs that push to it (SURVEY 8e)
// =================================================================================================
void KVStore::ShardRsp(KeyEntry& e, const std::vector<int>& devs) {
  Engine* eng = Engine::Get();
  const int64_t rows = e.shape[0];
  const int64_t row_len = static_cast<int64_t>(e.rsp.RowLength());
  const int n = static_cast<int>(devs.size());
  e.rsp_rows_per = (rows + n - 1) / n;
  e.rsp_devs = devs;
  e.rsp_shards.assign(n, NDArray());
  e.rsp_shard_state.assign(n, DevState());
  e.rsp_vbase.clear();
  DevState& hs = e.dev[e.home];
  const size_t rb = static_cast<size_t>(row_len) * sizeof(float);
  for (int j = 0; j < n; ++j) {
    const int64_t lo = j * e.rsp_rows_per, hi = std::min<int64_t>(rows, lo + e.rsp_rows_per);
    const int64_t cnt = std::max<int64_t>(hi - lo, 1);
    auto take = [&](const NDArray& whole, NDArray* shard) {
      *shard = NDArray({cnt, row_len}, Context::GPU(devs[j]), kFloat32);
      if (hi > lo) {
        RawCopy(shard->data(), shard->ctx(), shard->var(), static_cast<const char*>(whole.data()) + lo * rb,
                whole.ctx(), whole.var(), static_cast<size_t>(hi - lo) * rb);
      }
    };
    take(e.rsp, &e.rsp_shards[j]);
    if (!hs.s1.is_none()) take(hs.s1, &e.rsp_shard_state[j].s1);
    if (!hs.s2.is_none()) take(hs.s2, &e.rsp_shard_state[j].s2);
  }
  // the whole-table copies are stale from here on: release them (2 GB for a 1 M x 512 table)
  eng->WaitToWrite(*e.rsp.var());
  e.rsp = NDArray::RowSparse(e.shape, Context::GPU(e.home), e.dtype);
  hs.s1 = NDArray();
  hs.s2 = NDArray();
}

void KVStore::UnshardRsp(KeyEntry& e) {
  if (e.rsp_devs.empty()) return;
  const int64_t rows = e.shape[0];
  const int home = e.home;
  NDArray whole = NDArray::RowSparse(e.shape, Context::GPU(home), e.dtype);
  whole.CheckAndAllocRows(rows);
  const int64_t row_len = static_cast<int64_t>(whole.RowLength());
  const size_t rb = static_cast<size_t>(row_len) * sizeof(float);
  DevState& hs = e.dev[home];
  const bool has1 = !e.rsp_shard_state[0].s1.is_none(), has2 = !e.rsp_shard_state[0].s2.is_none();
  if (has1) hs.s1 = NDArray(e.shape, Context::GPU(home), kFloat32);
  if (has2) hs.s2 = NDArray(e.shape, Context::GPU(home), kFloat32);
  for (size_t j = 0; j < e.rsp_devs.size(); ++j) {
    const int64_t lo = static_cast<int64_t>(j) * e.rsp_rows_per, hi = std::min<int64_t>(rows, lo + e.rsp_rows_per);
    if (hi <= lo) continue;
    auto put = [&](const NDArray& shard, void* base, Var* var) {
      RawCopy(static_cast<char*>(base) + lo * rb, Context::GPU(home), var, shard.data(), shard.ctx(),
              shard.var(), static_cast<size_t>(hi - lo) * rb);
    };
    put(e.rsp_shards[j], whole.data(), whole.var());
    if (has1) put(e.rsp_shard_state[j].s1, hs.s1.data(), hs.s1.var());
    if (has2) put(e.rsp_shard_state[j].s2, hs.s2.data(), hs.s2.var());
  }
  // row ids 0..rows-1
  std::vector<int64_t> ids(rows);
  for (int64_t i = 0; i < rows; ++i) ids[i] = i;
  RawCopy(whole.row_ids(), whole.ctx(), whole.var(), ids.data(), Context::CPU(), nullptr,
          ids.size() * sizeof(int64_t));
  Engine::Get()->WaitToRead(*whole.var());  // `ids` goes out of scope
  e.rsp = whole;
  e.rsp_devs.clear();
  e.rsp_shards.clear();
  e.rsp_shard_state.clear();
  e.rsp_vbase.clear();
  e.rsp_rows_per = 0;
}

const float* const* KVStore::RspShardTable(KeyEntry& e, int dev) {
  auto it = e.rsp_vbase.find(dev);
  if (it == e.rsp_vbase.end()) {
    const int n = e.rsp_group ? static_cast<int>(e.rsp_peer_off.size()) : static_cast<int>(e.rsp_devs.size());
    const int64_t row_len = static_cast<int64_t>(e.rsp_shards[0].RowLength());
    std::vector<const float*> vb(n);
    for (int j = 0; j < n; ++j) {
      const float* base = e.rsp_group
          ? static_cast<const float*>(PeerGroup::Get()->PeerPtr(j, e.rsp_peer_off[j]))
          : static_cast<const float*>(e.rsp_shards[j].data());
      vb[j] = base - static_cast<int64_t>(j) * e.rsp_rows_per * row_len;
    }
    NDArray tbl({n}, Context::GPU(dev), kInt64);
    RawCopy(tbl.data(), tbl.ctx(), tbl.var(), vb.data(), Context::CPU(), nullptr, n * sizeof(void*));
    Engine::Get()->WaitToRead(*tbl.var());
    it = e.rsp_vbase.emplace(dev, tbl).first;
  }
  return static_cast<const float* const*>(it->second.data());
}

bool KVStore::PushRowSparseSharded(KeyEntry& e, const std::vector<NDArray>& srcs,
                                   const std::vector<int>& parts, RspUpdateLaunch U) {
  Engine* eng = Engine::Get();
  const int64_t rows = e.shape[0];
  if (e.rsp_devs.empty()) {
    if (e.rsp.nnr() != rows) return false;   // only tables that hold every row are sharded
    std::vector<int> devs = parts;
    std::sort(devs.begin(), devs.end());
    ShardRsp(e, devs);
  } else {
    for (int d : parts) {
      if (std::find(e.rsp_devs.begin(), e.rsp_devs.end(), d) == e.rsp_devs.end()) {
        UnshardRsp(e);       // pushed from a different GPU set: fold back and shard again
        return PushRowSparseSharded(e, srcs, parts, U);
      }
    }
  }
  const std::vector<int>& devs = e.rsp_devs;
  const int n = static_cast<int>(devs.size());
  const int64_t row_len = static_cast<int64_t>(e.rsp_shards[0].RowLength());
  const RspSources S = LocalSources(srcs);
  const int64_t total = S.start[S.nsrc];
  std::vector<int> lanes = devs;
  for (auto& s : srcs) {
    if (std::find(lanes.begin(), lanes.end(), s.dev()) == lanes.end()) lanes.push_back(s.dev());
  }
  eng->RequirePeerAccess(lanes);
  // optimizer state of a shard is created on first use (zeros), like Optimizer.create_state
  const bool need1 = U.opt == kOptSGD || U.opt == kOptAdam, need2 = U.opt == kOptAdam;
  for (int j = 0; j < n; ++j) {
    DevState& sj = e.rsp_shard_state[j];
    if (need1 && sj.s1.is_none()) sj.s1 = ZerosOn(e.rsp_shards[j].shape(), devs[j], kFloat32);
    if (need2 && sj.s2.is_none()) sj.s2 = ZerosOn(e.rsp_shards[j].shape(), devs[j], kFloat32);
  }
  const int id_bits = BitsFor(rows);
  for (int j = 0; j < n; ++j) {
    const int64_t lo = static_cast<int64_t>(j) * e.rsp_rows_per, hi = std::min<int64_t>(rows, lo + e.rsp_rows_per);
    if (hi <= lo) continue;
    const int dev = devs[j];
    DevState& sj = e.rsp_shard_state[j];
    NDArray d_nnr({1}, Context::GPU(dev), kInt64);
    NDArray ws({static_cast<int64_t>(RspMergeWorkspaceBytes(total, id_bits, S.nsrc, lo, hi))}, Context::GPU(dev), kUint8);
    // each shard's kernels depend on the sources through events on ITS lane (no global join: the
    // GPUs merge their row ranges concurrently and independently)
    LaneOp op(dev);
    for (auto& s : srcs) op.Read(s);
    op.Write(e.rsp_shards[j]).Write(d_nnr).Write(ws);
    if (need1) op.Write(sj.s1);
    if (need2) op.Write(sj.s2);
    RspUpdateLaunch Uj = U;
    // virtual bases: row `id` of the table is at base + id*row_len
    Uj.w = static_cast<float*>(e.rsp_shards[j].data()) - lo * row_len;
    Uj.s1 = need1 ? static_cast<float*>(sj.s1.data()) - lo * row_len : nullptr;
    Uj.s2 = need2 ? static_cast<float*>(sj.s2.data()) - lo * row_len : nullptr;
    LaunchRspMerge(S, id_bits, row_len, nullptr, nullptr, static_cast<int64_t*>(d_nnr.data()), ws.data(),
                   ws.ByteSize(), op.stream(), &Uj, lo, hi);
    eng->CountLaunch("rsp_merge(shard)", total * 24);
    eng->CountLaunch("rsp_sum+update(shard)", 0);
    op.Issue();
  }
  return true;
}

// =================================================================================================
// one rank per GPU (torchrun): row_sparse keys
// =================================================================================================
void KVStore::GroupBarrier() {
  PeerGroup* g = PeerGroup::Get();
  Engine* eng = Engine::Get();
  DenseLaunch L;
  g->FillLaunch(&L);
  L.n_chunks = 0;               // no work: the fused kernel's start + end barriers only
  L.dtype = kFloat32;
  L.opt = kOptAssign;
  DeviceGuard guard(g->dev());
  LaunchDenseFused(L, eng->Stream(g->dev()));
  eng->CountLaunch("group_barrier", 0);
}

// One rank per GPU, NO fused optimizer on the store (plain assignment, an updater callback, or a
// standard -- non-lazy -- update): what the reference does with the merged gradient happens on
// every rank alike, so every rank builds the SAME merged row_sparse gradient -- the union of all
// ranks' rows, summed in rank order, read through IPC -- and the caller carries on as the
// single-process store does (kvstore_local.h:208-245); the stored value stays replicated.
NDArray KVStore::MergeRowSparseGroup(KeyEntry& e, const NDArray& src_in) {
  PeerGroup* g = PeerGroup::Get();
  KV_CHECK(g != nullptr);
  Engine* eng = Engine::Get();
  const int dev = g->dev();
  KV_CHECK(!e.rsp_group) << "key " << e.key << " is sharded over the ranks by a fused optimizer; it "
                         << "cannot go back to a replicated value";
  NDArray src;
  const RspSources S = RankSources(g, e.key, src_in, &src);
  const int64_t total = S.start[S.nsrc];
  NDArray merged = NDArray::RowSparse(e.shape, Context::GPU(dev), e.dtype);
  const int64_t row_len = static_cast<int64_t>(src.RowLength());
  const int bits = BitsFor(e.shape[0]);
  NDArray d_nnr, ws;
  if (total > 0) {
    merged.CheckAndAllocRows(total);
    d_nnr = NDArray({1}, Context::GPU(dev), kInt64);
    ws = NDArray({static_cast<int64_t>(RspMergeWorkspaceBytes(total, bits, S.nsrc))}, Context::GPU(dev), kUint8);
  }
  // every wait is declared before the first barrier: none lands between the two
  LaneOp op(dev);
  op.Read(src).Write(merged).Write(d_nnr).Write(ws);
  GroupBarrier();   // every rank's gradient is complete before anybody reads it
  if (total > 0) {
    LaunchRspMerge(S, bits, row_len, merged.row_ids(), static_cast<float*>(merged.data()),
                   static_cast<int64_t*>(d_nnr.data()), ws.data(), ws.ByteSize(), op.stream());
    eng->CountLaunch("rsp_merge(replicated)", total * 24);
    eng->CountLaunch("rsp_sum(replicated)", static_cast<uint64_t>(total) * row_len * 8);
  }
  GroupBarrier();   // everybody has read the peers' gradients: they may be reused
  op.Issue();
  if (total > 0) {
    CountFence f(dev, 1);
    f.Post(static_cast<const int64_t*>(d_nnr.data()), op.stream());
    merged.SetNnr(f.Wait()[0]);
  }
  return merged;
}

void KVStore::PushRowSparseGroup(KeyEntry& e, const NDArray& src_in, RspUpdateLaunch U) {
  PeerGroup* g = PeerGroup::Get();
  KV_CHECK(g != nullptr);
  Engine* eng = Engine::Get();
  const int dev = g->dev(), W = g->world(), R = g->rank();
  const int64_t rows = e.shape[0];
  KV_CHECK_EQ(e.home, dev) << "key " << e.key << " lives on another GPU than this rank's";
  // ---- this rank's shard (rows [R*per, (R+1)*per)) and every rank's shard address, once
  if (!e.rsp_group) {
    KV_CHECK_EQ(e.rsp.nnr(), rows)
        << "key " << e.key << ": the stored row_sparse weight must hold every row (initialise it from "
        << "a dense weight, as gluon does)";
    e.rsp_rows_per = (rows + W - 1) / W;
    const int64_t lo = R * e.rsp_rows_per, hi = std::min<int64_t>(rows, lo + e.rsp_rows_per);
    const int64_t row_len = static_cast<int64_t>(e.rsp.RowLength());
    NDArray shard({std::max<int64_t>(hi - lo, 1), row_len}, Context::GPU(dev), kFloat32);
    KV_CHECK(g->InArena(shard.data())) << "IPC arena exhausted; raise B200KV_IPC_ARENA_MB";
    if (hi > lo) {
      RawCopy(shard.data(), shard.ctx(), shard.var(),
              static_cast<const char*>(e.rsp.data()) + lo * row_len * sizeof(float), e.rsp.ctx(), e.rsp.var(),
              static_cast<size_t>(hi - lo) * row_len * sizeof(float));
    }
    eng->WaitToWrite(*e.rsp.var());
    e.rsp = NDArray::RowSparse(e.shape, Context::GPU(dev), e.dtype);  // the full copy is released
    e.rsp_shards.assign(1, shard);
    e.rsp_shard_state.assign(1, DevState());
    const std::vector<int64_t> all = g->AllGatherI64({g->OffsetOf(shard.data()), rows, row_len});
    e.rsp_peer_off.resize(W);
    for (int r = 0; r < W; ++r) {
      KV_CHECK(all[3 * r + 1] == rows && all[3 * r + 2] == row_len)
          << "key " << e.key << " has a different shape on rank " << r;
      e.rsp_peer_off[r] = all[3 * r];
    }
    e.rsp_group = true;
    e.rsp_vbase.clear();
  }
  const int64_t row_len = static_cast<int64_t>(e.rsp_shards[0].RowLength());
  const int64_t lo = R * e.rsp_rows_per, hi = std::min<int64_t>(rows, lo + e.rsp_rows_per);
  // ---- every rank's gradient, addressable by the peers inside its rank's arena
  NDArray src;
  const RspSources S = RankSources(g, e.key, src_in, &src);
  const int64_t total = S.start[S.nsrc];
  // optimizer state of the shard
  const bool need1 = U.opt == kOptSGD || U.opt == kOptAdam, need2 = U.opt == kOptAdam;
  DevState& st8 = e.rsp_shard_state[0];
  if (need1 && st8.s1.is_none()) st8.s1 = ZerosOn(e.rsp_shards[0].shape(), dev, kFloat32);
  if (need2 && st8.s2.is_none()) st8.s2 = ZerosOn(e.rsp_shards[0].shape(), dev, kFloat32);
  const bool run = total > 0 && hi > lo;
  NDArray d_nnr, ws;
  if (run) {
    d_nnr = NDArray({1}, Context::GPU(dev), kInt64);
    ws = NDArray({static_cast<int64_t>(RspMergeWorkspaceBytes(total, BitsFor(rows), S.nsrc, lo, hi))}, Context::GPU(dev), kUint8);
  }
  // every wait is declared before barrier 1: none lands between the two barriers
  LaneOp op(dev);
  op.Read(src).Write(e.rsp_shards[0]).Write(d_nnr).Write(ws);
  if (need1) op.Write(st8.s1);
  if (need2) op.Write(st8.s2);
  // barrier 1: every rank's gradient is complete (its barrier kernel is stream-ordered behind the
  // producer) before anybody reads it through IPC
  GroupBarrier();
  if (run) {
    RspUpdateLaunch Uj = U;
    Uj.w = static_cast<float*>(e.rsp_shards[0].data()) - lo * row_len;
    Uj.s1 = need1 ? static_cast<float*>(st8.s1.data()) - lo * row_len : nullptr;
    Uj.s2 = need2 ? static_cast<float*>(st8.s2.data()) - lo * row_len : nullptr;
    LaunchRspMerge(S, BitsFor(rows), row_len, nullptr, nullptr, static_cast<int64_t*>(d_nnr.data()),
                   ws.data(), ws.ByteSize(), op.stream(), &Uj, lo, hi);
    eng->CountLaunch("rsp_merge(rank shard)", total * 24);
    eng->CountLaunch("rsp_sum+update(rank shard)", 0);
  }
  // barrier 2: every rank has finished reading the peers' gradients (they may now be reused) and
  // updating its shard (a pull that follows sees the new rows on every rank)
  GroupBarrier();
  op.Issue();
}

}  // namespace b200kv
