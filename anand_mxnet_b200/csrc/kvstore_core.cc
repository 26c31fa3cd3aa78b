// kvstore.cc -- see kvstore.h. Dense path, key table, fused-optimizer bookkeeping.
#include "kvstore.h"

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstring>
#include <iostream>
#include <set>

#include "group.h"
#include "nccl_dyn.h"
#include "rowsparse.h"
#include "scalar_parse.h"

namespace b200kv {

// =================================================================================================
// helpers
// =================================================================================================
static std::string Lower(std::string s) {
  for (auto& c : s) c = static_cast<char>(std::tolower(static_cast<unsigned char>(c)));
  return s;
}

static uint64_t RoundUp(uint64_t x, uint64_t m) { return (x + m - 1) / m * m; }

static bool Is16Bit(int dtype) { return dtype == kFloat16 || dtype == kBfloat16; }

static std::set<KVStore*>& LiveStores();  // stores with possibly queued work (FlushAll)

static void DetachAnchorOf(Var* v) { static_cast<KVStore*>(v->anchor)->DetachVar(v); }

// Chunk a key's elements for the device that owns them. A chunk never crosses a chunk boundary of
// the store-global element space, hence never an ownership stripe. owner_fixed >= 0: the whole key
// belongs to that slot (WHOLE placement); otherwise stripes rotate over ndev slots.
void PlanChunks(uint64_t goff, size_t size, uint32_t key_slot, int ndev, int owner_fixed,
                std::vector<std::vector<ChunkDesc>>* per_slot) {
  size_t pos = 0;
  while (pos < size) {
    const uint64_t g = goff + pos;
    const size_t room = kChunkElems - static_cast<size_t>(g % kChunkElems);
    const size_t len = std::min(room, size - pos);
    const int slot = owner_fixed >= 0 ? owner_fixed : static_cast<int>((g / kBlockElems) % ndev);
    ChunkDesc c;
    c.key = key_slot;
    c.off = static_cast<uint32_t>(pos);
    c.len = static_cast<uint32_t>(len);
    c.pad_ = 0;
    (*per_slot)[slot].push_back(c);
    pos += len;
  }
}

Plan::~Plan() {
  Engine* e = Engine::Get();
  for (auto& p : per_dev) {
    e->Free(p.dev, p.d_keys, p.bytes_keys);
    e->Free(p.dev, p.d_chunks, p.bytes_chunks);
    e->Free(p.dev, p.d_hyper, p.bytes_hyper);
  }
}

// =================================================================================================
// construction / key table
// =================================================================================================
KVStore::KVStore(const std::string& type) : type_(type) {
  // KVStore::Create (src/kvstore/kvstore.cc:40-77): substring match on the lower-cased name
  const std::string t = Lower(type);
  KV_CHECK(t.find("dist") == std::string::npos)
      << "kvstore type '" << type << "': multi-node parameter-server stores are outside this "
      << "library (single-node 'local' / 'device' / 'nccl' only)";
  order_local_ = !(t.find("device") != std::string::npos || t.find("nccl") != std::string::npos);
  nccl_type_ = t.find("nccl") != std::string::npos;
  Engine::Get()->NumDevices();  // fails loudly when there is no GPU
  if (PeerGroup* g = PeerGroup::Get()) {
    // one rank per GPU: this store is one worker of a group (the role dist_device_sync plays in
    // the reference, without servers: the ranks reduce among themselves over NVLink)
    dist_ = g->world() > 1;
    rank_ = g->rank();
    group_size_ = g->world();
    // KVStoreNCCL's role (src/kvstore/kvstore_nccl.h): asked for by name, or forced when the ranks
    // share no NVLink peer memory. Dense keys only, as in the reference.
    nccl_ = dist_ && (t.find("nccl") != std::string::npos || !g->ipc_ok() ||
                      std::getenv("B200KV_FORCE_NCCL") != nullptr);
    if (nccl_) Nccl::Get();   // fail at creation, with a clear message, when libnccl is missing
  }
  // Deferred bucket execution. Default ("auto"): calls that name ONE key -- the way Trainer and
  // tools/bandwidth/measure.py drive the store, one call per parameter -- are queued and fused into
  // one launch; calls that already carry a key list run at once. B200KV_BUCKET_MB=n queues every
  // call up to n MB, 0 switches queuing off.
  if (const char* b = std::getenv("B200KV_BUCKET_MB")) {
    bucket_bytes_ = static_cast<size_t>(std::max(0, std::atoi(b))) << 20;
    bucket_auto_ = false;
  }
  if (const char* b = std::getenv("B200KV_AUTO_BUCKET_MB")) {
    auto_bucket_bytes_ = static_cast<size_t>(std::max(1, std::atoi(b))) << 20;
  }
  LiveStores().insert(this);
  Engine::Get()->detach_anchor = &DetachAnchorOf;
}

KVStore::~KVStore() {
  LiveStores().erase(this);
  try {
    Flush();
    Engine::Get()->WaitAll();
  } catch (...) {
  }
  // the anchors keep the last value the caller pulled: theirs from now on
  for (auto& a : anchors_) const_cast<Var*>(a.first)->anchor = nullptr;
}

void KVStore::SetKeyTypeInt() {
  if (key_type_ == -1) key_type_ = 1;
  KV_CHECK_EQ(key_type_, 1) << "Mixed key types are not allowed";
}

void KVStore::SetKeyTypeStr() {
  if (key_type_ == -1) key_type_ = 0;
  KV_CHECK_EQ(key_type_, 0) << "Mixed key types are not allowed";
}

KeyEntry& KVStore::Entry(int key) {
  auto it = local_.find(key);
  KV_CHECK(it != local_.end()) << "key " << key << " has not been inited";
  return *it->second;
}

std::vector<int> KVStore::LookupKeys(const std::vector<std::string>& str_keys) {
  std::vector<int> keys(str_keys.size());
  for (size_t i = 0; i < str_keys.size(); ++i) {
    auto it = str_key_dict_.find(str_keys[i]);
    KV_CHECK(it != str_key_dict_.end()) << "key " << str_keys[i] << " doesn't exist. Did you init?";
    keys[i] = it->second;
  }
  return keys;
}

void KVStore::Init(const std::vector<int>& keys, const std::vector<NDArray>& values) {
  SetKeyTypeInt();
  InitImpl(keys, values);
}

void KVStore::InitStr(const std::vector<std::string>& str_keys, const std::vector<NDArray>& values) {
  SetKeyTypeStr();
  std::vector<int> keys(str_keys.size());
  for (size_t i = 0; i < str_keys.size(); ++i) {
    KV_CHECK(str_key_dict_.find(str_keys[i]) == str_key_dict_.end())
        << "duplicate init of key " << str_keys[i];
    int key = next_str_key_++;
    str_key_dict_[str_keys[i]] = key;
    reverse_str_key_dict_[key] = str_keys[i];
    keys[i] = key;
  }
  InitImpl(keys, values);
}

void KVStore::InitImpl(const std::vector<int>& keys, const std::vector<NDArray>& values) {
  Flush();
  KV_CHECK_EQ(keys.size(), values.size());
  for (size_t i = 0; i < keys.size(); ++i) {
    KV_CHECK(local_.find(keys[i]) == local_.end())
        << "duplicate init of key " << keys[i]
        << ". Please double check if you called kv.init or kv.broadcast with this key "
        << "multiple times";
    const NDArray& v = values[i];
    KV_CHECK(!v.is_none()) << "init with an empty NDArray";
    std::unique_ptr<KeyEntry> e(new KeyEntry());
    e->key = keys[i];
    e->shape = v.shape();
    e->dtype = v.dtype();
    e->stype = v.stype();
    e->vstype = v.stype();
    e->size = v.Size();
    e->goff = next_goff_;
    next_goff_ += RoundUp(std::max<size_t>(e->size, 1), kKeyAlignElems);
    if (v.stype() == kRowSparseStorage) {
      e->rsp = v.Copy(v.on_gpu() ? v.ctx() : Context::Pinned());
      if (v.on_gpu()) e->home = v.dev();
    } else if (v.on_gpu()) {
      // the reference parks the value in pinned host memory (kvstore_local.h:202) and migrates it
      // at the first push; a GPU-resident copy right away is observably identical and saves a hop
      e->home = v.dev();
      e->dev[e->home].w = v.Copy(v.ctx());
    } else {
      e->host = v.Copy(Context::Pinned());
    }
    local_[keys[i]] = std::move(e);
  }
  if (dist_) {
    if (nccl_) BroadcastInitNccl(keys); else BroadcastInitGroup(keys);
  }
}

void KVStore::SetUpdater(UpdaterFn fn, StrUpdaterFn sfn, void* handle) {
  Flush();  // queued calls were issued under the previous updater / optimizer
  updater_ = fn;
  str_updater_ = sfn;
  updater_handle_ = handle;
  ++layout_epoch_;
  // an explicit updater replaces a previously fused optimizer (set_optimizer -> _set_updater)
  if (fn != nullptr) opt_.enabled = false;
}

void KVStore::SetGradientCompression(const std::vector<std::pair<std::string, std::string>>& kw) {
  // GradientCompression::SetParams (src/kvstore/gradient_compression.cc:44-60): type in
  // {none, 2bit}, threshold > 0 (default 0.5)
  Flush();
  std::string type = gc_type_;
  float threshold = gc_threshold_;
  for (auto& kv : kw) {
    if (kv.first == "type") type = Lower(kv.second);
    else if (kv.first == "threshold") threshold = DmlcStof(kv.second);
    else KV_FATAL << "Cannot find argument '" << kv.first << "', Possible Arguments: type, threshold";
  }
  KV_CHECK(type == "none" || type == "2bit") << "Unknown type for gradient compression " << type;
  KV_CHECK(threshold > 0) << "threshold must be greater than 0";
  gc_type_ = type;
  gc_threshold_ = threshold;
  ++layout_epoch_;
}

// =================================================================================================
// fused optimizer bookkeeping (python/mxnet/optimizer/optimizer.py restated)
// =================================================================================================
static double ParseD(const std::string& s) {
  const std::string t = Lower(s);
  if (t == "none" || t.empty()) return 0.0;
  if (t == "true") return 1.0;
  if (t == "false") return 0.0;
  char* end = nullptr;
  double v = std::strtod(s.c_str(), &end);
  KV_CHECK(end != s.c_str() && *end == '\0') << "cannot parse optimizer parameter value '" << s << "'";
  return v;
}

void KVStore::SetOptimizer(const std::string& name,
                           const std::vector<std::pair<std::string, std::string>>& kw) {
  Flush();
  OptConfig o;
  const std::string n = Lower(name);
  if (n == "sgd") {
    o.kind = kOptSGD;
    o.lr = 0.01;
  } else if (n == "adam") {
    o.kind = kOptAdam;
    o.lr = 0.001;
  } else if (n == "test") {
    o.kind = kOptTest;
  } else {
    KV_FATAL << "optimizer '" << name << "' has no fused kernel (sgd, adam, test); use the "
             << "updater callback (MXKVStoreSetUpdaterEx) for it";
  }
  for (auto& kv : kw) {
    const std::string& k = kv.first;
    const double v = ParseD(kv.second);
    if (k == "learning_rate" || k == "lr") o.lr = v;
    else if (k == "wd") o.wd = v;
    else if (k == "momentum") o.momentum = v;
    else if (k == "rescale_grad") o.rescale = v;
    else if (k == "clip_gradient") o.clip = v;
    else if (k == "beta1") o.beta1 = v;
    else if (k == "beta2") o.beta2 = v;
    else if (k == "epsilon") o.eps = v;
    else if (k == "multi_precision") o.multi_precision = v != 0.0;
    else if (k == "lazy_update") o.lazy_update = v != 0.0;
    else if (k == "begin_num_update") o.begin_num_update = static_cast<int>(v);
    else KV_FATAL << "unknown optimizer parameter '" << k << "'";
  }
  o.num_update = o.begin_num_update;
  o.enabled = true;
  // keep multipliers / counts across a re-configuration of the same optimizer (Trainer re-sends
  // hyper-parameters when the learning rate changes)
  if (opt_.enabled && opt_.kind == o.kind) {
    o.lr_mult = opt_.lr_mult;
    o.wd_mult = opt_.wd_mult;
    o.count = opt_.count;
    o.num_update = std::max(o.num_update, opt_.num_update);
  }
  opt_ = o;
  ++layout_epoch_;
  ++opt_version_;
  updater_ = nullptr;
  str_updater_ = nullptr;
}

// Per-key (lr, wd) as float32, exactly as the reference's operator would receive them.
void KVStore::KeyHyper(const KeyEntry& e, int opt_kind, float* lr, float* wd) {
  *lr = 0.f;
  *wd = 0.f;
  if (opt_kind != kOptSGD && opt_kind != kOptAdam) return;
  auto lm = opt_.lr_mult.find(e.key);
  auto wm = opt_.wd_mult.find(e.key);
  double lrd = opt_.lr * (lm == opt_.lr_mult.end() ? 1.0 : lm->second);  // _get_lrs
  double wdd = opt_.wd * (wm == opt_.wd_mult.end() ? 1.0 : wm->second);  // _get_wds
  if (opt_kind == kOptSGD) {
    // multi_sgd*_update: lrs / wds are tuple parameters -> correctly rounded float
    *lr = TupleParam(lrd);
    *wd = TupleParam(wdd);
  } else {
    // Adam.update (optimizer.py:1610-1629): bias correction in python double, scalar parameters
    auto c = opt_.count.find(e.key);
    const int t = c == opt_.count.end() ? 0 : c->second;
    const double coef1 = 1.0 - std::pow(opt_.beta1, t);
    const double coef2 = 1.0 - std::pow(opt_.beta2, t);
    lrd *= std::sqrt(coef2) / coef1;
    *lr = ScalarParam(lrd);
    *wd = ScalarParam(wdd);
  }
}

// =================================================================================================
// grouping (KVStoreLocal::GroupKVPairs, kvstore_local.h:377-407)
// =================================================================================================
// The values of one key are reduced in the order the call lists them (a stable sort by key). The
// reference orders the (key, position) pairs with std::sort, which is not stable: identical for calls
// of at most 16 pairs -- every per-parameter call of gluon.Trainer / Module -- but in a bigger call
// (a key LIST with several values per key) the values of a key reach its reduce in whatever order
// libstdc++'s introsort leaves them, and a floating-point sum depends on that order.
// B200KV_GROUP_ORDER=reference reproduces it (same std::sort, same comparator, same libstdc++).
void SortKeyPairs(std::vector<std::pair<int, int>>* idx, bool reference_order) {
  auto by_key = [](const std::pair<int, int>& a, const std::pair<int, int>& b) { return a.first < b.first; };
  if (reference_order) {
    std::sort(idx->begin(), idx->end(), by_key);
  } else {
    std::stable_sort(idx->begin(), idx->end(), by_key);
  }
}

static bool ReferenceGroupOrder() {
  const char* e = std::getenv("B200KV_GROUP_ORDER");
  return e != nullptr && std::strcmp(e, "reference") == 0;
}

template <typename FValid>
static void GroupKVPairs(const std::vector<int>& keys, const std::vector<NDArray>& values,
                         std::vector<int>* uniq_keys, std::vector<std::vector<NDArray>>* grouped,
                         FValid is_valid) {
  KV_CHECK_EQ(keys.size(), values.size());
  if (keys.empty()) return;
  std::vector<std::pair<int, int>> idx(keys.size());
  for (size_t i = 0; i < keys.size(); ++i) idx[i] = {keys[i], static_cast<int>(i)};
  SortKeyPairs(&idx, ReferenceGroupOrder());
  bool have = false;
  int pre_key = 0;
  for (auto& i : idx) {
    if (!is_valid(i.first, values[i.second])) continue;
    if (!have || i.first != pre_key) {
      uniq_keys->push_back(i.first);
      grouped->push_back({values[i.second]});
      pre_key = i.first;
      have = true;
    } else {
      grouped->back().push_back(values[i.second]);
    }
  }
}

// =================================================================================================
// push / pull / pushpull
// =================================================================================================
// ---- deferred bucket execution ------------------------------------------------------------------
// The reference's callers issue one push / pull per parameter (gluon/trainer.py:371-396 with
// priority=-i; tools/bandwidth/measure.py:112-122). Executed one by one that is a kernel launch per
// key. With B200KVStoreSetBucketBytes(n > 0) the calls are queued -- they "return after enqueueing"
// exactly as the reference's asynchronous contract allows (kvstore.h:129-141,168-180) -- and fused
// into ONE launch per device when the queued bytes reach n, when any array is waited on / read,
// or on Flush(). Per-key order is preserved; higher priority values are issued first.
static std::set<KVStore*>& LiveStores() {
  static auto* s = new std::set<KVStore*>();
  return *s;
}

void KVStore::FlushAll() {
  for (KVStore* kv : LiveStores()) kv->Flush();
}

bool KVStore::TryDefer(int kind, std::vector<int>& vkeys, std::vector<NDArray>& values,
                       std::vector<int>& okeys, std::vector<NDArray>& outs, int priority) {
  if ((updater_ != nullptr && !opt_.enabled) || gc_type_ != "none") return false;
  size_t cap = bucket_bytes_;
  if (cap == 0) {
    if (!bucket_auto_) return false;
    // auto mode: only single-key calls (n values of one key count as one key)
    const int k0 = !vkeys.empty() ? vkeys[0] : (!okeys.empty() ? okeys[0] : 0);
    for (int k : vkeys) if (k != k0) return false;
    for (int k : okeys) if (k != k0) return false;
    if (vkeys.empty() && okeys.empty()) return false;
    // memory another framework owns (DLPack imports) can be read by its owner without any call
    // into this library, so nothing would ever flush the queue for it: run such calls at once
    for (auto& v : values) if (v.external()) return false;
    for (auto& o : outs) if (o.external()) return false;
    cap = auto_bucket_bytes_;
  }
  (void)kind;
  size_t bytes = 0;
  // a second push of a key, or a push after a queued pull of it, must not be merged with the
  // queued one: run what is queued first (KeyEntry::queued: bit 0 = push queued, bit 1 = pull)
  bool conflict = false;
  KeyEntry* last = nullptr;
  for (size_t i = 0; i < vkeys.size(); ++i) {
    KeyEntry& e = (last != nullptr && last->key == vkeys[i]) ? *last : Entry(vkeys[i]);  // un-initialised keys still fail synchronously
    last = &e;
    const NDArray& v = values[i];
    if (v.stype() != kDefaultStorage || e.vstype != kDefaultStorage) return false;
    KV_CHECK_EQ(v.Size(), e.size) << "push: shape mismatch for key " << e.key;
    KV_CHECK_EQ(v.dtype(), e.dtype) << "push: dtype mismatch for key " << e.key;
    bytes += v.ByteSize();
    conflict = conflict || e.queued != 0;
  }
  for (size_t i = 0; i < okeys.size(); ++i) {
    KeyEntry& e = (last != nullptr && last->key == okeys[i]) ? *last : Entry(okeys[i]);
    last = &e;
    const NDArray& o = outs[i];
    if (o.stype() != kDefaultStorage || e.vstype != kDefaultStorage) return false;
    KV_CHECK_EQ(o.Size(), e.size) << "pull: shape mismatch for key " << e.key;
    KV_CHECK_EQ(o.dtype(), e.dtype) << "pull: dtype mismatch for key " << e.key;
    bytes += o.ByteSize();
  }
  if (conflict) Flush();
  last = nullptr;
  auto mark = [&](int k, uint8_t bit) {
    KeyEntry& e = (last != nullptr && last->key == k) ? *last : Entry(k);
    last = &e;
    if (e.queued == 0) pending_entries_.push_back(&e);
    e.queued |= bit;
  };
  for (int k : vkeys) mark(k, 1);
  for (int k : okeys) mark(k, 2);
  pending_.emplace_back();
  PendingOp& op = pending_.back();
  op.vkeys = std::move(vkeys);
  op.vals = std::move(values);
  op.okeys = std::move(okeys);
  op.outs = std::move(outs);
  op.priority = priority;
  pending_bytes_ += bytes;
  if (pending_bytes_ >= cap) Flush();
  return true;
}

void KVStore::Flush() {
  if (pending_.empty()) return;
  std::vector<PendingOp> ops;
  ops.swap(pending_);
  for (KeyEntry* e : pending_entries_) e->queued = 0;
  pending_entries_.clear();
  pending_bytes_ = 0;
  // higher priority first; equal priorities (push i and pull i both carry -i) keep call order
  std::stable_sort(ops.begin(), ops.end(),
                   [](const PendingOp& a, const PendingOp& b) { return a.priority > b.priority; });
  std::vector<int> vkeys, okeys;
  std::vector<NDArray> vals, outs;
  for (auto& op : ops) {
    vkeys.insert(vkeys.end(), op.vkeys.begin(), op.vkeys.end());
    vals.insert(vals.end(), op.vals.begin(), op.vals.end());
    okeys.insert(okeys.end(), op.okeys.begin(), op.okeys.end());
    outs.insert(outs.end(), op.outs.begin(), op.outs.end());
  }
  if (!vkeys.empty()) {
    PushImpl(vkeys, vals, okeys.empty() ? nullptr : &okeys, okeys.empty() ? nullptr : &outs);
  } else {
    PullImpl(okeys, outs, true);
  }
}

int KVStore::UpdateCount(int key) const {
  auto it = opt_.count.find(key);
  const int c = it == opt_.count.end() ? opt_.begin_num_update : it->second;
  auto e = local_.find(key);
  return c + ((e != local_.end() && (e->second->queued & 1)) ? 1 : 0);
}

int KVStore::NumUpdate() const {
  int n = opt_.num_update;
  for (const KeyEntry* e : pending_entries_) {
    if (e->queued & 1) n = std::max(n, UpdateCount(e->key));
  }
  return n;
}

void KVStore::SetBucketBytes(size_t n) {
  Flush();
  bucket_bytes_ = n;
  bucket_auto_ = false;  // an explicit size (0 = off) replaces the automatic policy
}

void KVStore::Push(std::vector<int> keys, std::vector<NDArray> values, int priority) {
  std::vector<int> no_keys;
  std::vector<NDArray> no_outs;
  if (TryDefer(0, keys, values, no_keys, no_outs, priority)) return;
  Flush();
  PushImpl(keys, values, nullptr, nullptr);
}

void KVStore::PushPull(std::vector<int> vkeys, std::vector<int> okeys, std::vector<NDArray> values,
                       std::vector<NDArray> outs, int priority) {
  if (TryDefer(2, vkeys, values, okeys, outs, priority)) return;
  Flush();
  PushImpl(vkeys, values, &okeys, &outs);
}

void KVStore::Pull(std::vector<int> keys, std::vector<NDArray> outs, int priority, bool ignore_sparse) {
  std::vector<int> no_keys;
  std::vector<NDArray> no_vals;
  if (ignore_sparse && TryDefer(1, no_keys, no_vals, keys, outs, priority)) return;
  Flush();
  PullImpl(keys, outs, ignore_sparse);
}

void KVStore::PushImpl(const std::vector<int>& keys, const std::vector<NDArray>& values,
                       const std::vector<int>* okeys, const std::vector<NDArray>* outs) {
  // a repeated call (same keys, same arrays) replays its prepared launches
  const bool callback_mode = updater_ != nullptr && !opt_.enabled;
  std::vector<uint64_t> sig;
  const bool cacheable = !callback_mode && gc_type_ == "none" &&
      CallSignature(opt_.enabled ? 100 + opt_.kind : 1, keys, values, okeys, outs, &sig);
  if (cacheable && RunCachedCall(sig)) return;
  std::vector<int> uniq;
  std::vector<std::vector<NDArray>> grouped;
  GroupKVPairs(keys, values, &uniq, &grouped, [](int, const NDArray& nd) {
    KV_CHECK(nd.stype() == kDefaultStorage || nd.stype() == kRowSparseStorage)
        << "Unexpected storage type detected during kvstore push: " << nd.stype();
    return true;
  });
  // pull side of a pushpull: PullImpl(okeys, outs, ignore_sparse=true) (kvstore_local.h:296-303)
  std::vector<int> ouniq;
  std::vector<std::vector<NDArray>> ogrouped;
  if (okeys != nullptr) {
    GroupKVPairs(*okeys, *outs, &ouniq, &ogrouped, [this](int key, const NDArray& nd) {
      if (nd.stype() == kDefaultStorage) return true;
      if (warnings_printed_.insert(key).second) {
        std::cerr << "Warning: non-default weights detected during kvstore pull. This call has "
                     "been ignored. Please make sure to use kv.row_sparse_pull() or "
                     "module.prepare() with row_ids.\n";
      }
      return false;
    });
  }
  std::unordered_map<int, size_t> out_of;
  for (size_t i = 0; i < ouniq.size(); ++i) out_of[ouniq[i]] = i;

  std::vector<DenseOp> fused, pulls;
  std::set<int> pushed;
  const bool callback = updater_ != nullptr && !opt_.enabled;
  // 2-bit compression quantises a key's values before the per-key checks below, and every
  // quantise moves its value's residual: check every compressed key of the call first, so that a
  // refused call leaves all residuals where they were (and no kernel reads a value as float32
  // that is not one)
  if (gc_type_ == "2bit") {
    for (size_t i = 0; i < uniq.size(); ++i) {
      const std::vector<NDArray>& srcs = grouped[i];
      if (srcs[0].stype() != kDefaultStorage) continue;
      const KeyEntry& e = Entry(uniq[i]);
      KV_CHECK_EQ(e.stype, kDefaultStorage)
          << "key " << e.key << " was initialised row_sparse but a dense value was pushed";
      KV_CHECK_EQ(e.dtype, kFloat32) << "2-bit gradient compression needs float32 gradients";
      if (dist_) {
        KV_CHECK_EQ(srcs.size(), 1u) << "one-rank-per-GPU store: push one value per key and rank";
      } else {
        KV_CHECK(srcs.size() <= static_cast<size_t>(kMaxSrc))
            << "at most " << kMaxSrc << " values per key and push";
      }
      for (auto& s : srcs) {
        KV_CHECK_EQ(s.stype(), kDefaultStorage) << "mixed storage types in push";
        KV_CHECK_EQ(s.Size(), e.size) << "push: shape mismatch for key " << e.key;
        KV_CHECK_EQ(s.dtype(), e.dtype) << "push: dtype mismatch for key " << e.key;
      }
    }
  }
  // 2-bit compression in a peer group: all dense keys of the call are quantised, exchanged and
  // decoded in one batch (two cross-rank barriers per call, not per key); their merged gradients
  // are identical on every rank, so the rest of the push is a local, one-source launch
  const bool gc_group = gc_type_ == "2bit" && dist_;
  if (gc_group) {
    KV_CHECK(!nccl_) << "kvstore 'nccl' does not compress gradients (src/kvstore/kvstore_nccl.h:62-70)";
    std::vector<KeyEntry*> es;
    std::vector<std::vector<NDArray>> vals;
    std::vector<size_t> which;
    for (size_t i = 0; i < uniq.size(); ++i) {
      if (grouped[i][0].stype() != kDefaultStorage) continue;
      KeyEntry& e = Entry(uniq[i]);
      es.push_back(&e);
      vals.push_back(grouped[i]);
      which.push_back(i);
    }
    if (!es.empty()) CompressedReduceGroup(es, &vals);
    for (size_t j = 0; j < which.size(); ++j) grouped[which[j]] = vals[j];
  }
  struct LocalScope {   // launches prepared below skip the cross-rank plan when the sums are done
    bool* flag;
    bool old;
    LocalScope(bool* f, bool v) : flag(f), old(*f) { *f = v; }
    ~LocalScope() { *flag = old; }
  } local_scope(&force_local_, gc_group);
  for (size_t i = 0; i < uniq.size(); ++i) {
    KeyEntry& e = Entry(uniq[i]);
    std::vector<NDArray>& srcs = grouped[i];
    pushed.insert(e.key);
    if (gc_type_ == "2bit" && !gc_group && srcs[0].stype() == kDefaultStorage) {
      // CommDevice::Reduce -> ReduceCompressed (comm.h:507-509): quantise every value with its
      // residual, decode + sum on the owner; the optimizer then sees that merged gradient
      NDArray merged = CompressedReduce(e, srcs);
      srcs.assign(1, merged);
    }
    if (srcs[0].stype() == kRowSparseStorage) {
      for (auto& s : srcs) KV_CHECK_EQ(s.stype(), kRowSparseStorage) << "mixed storage types in push";
      PushRowSparse(e, srcs);   // one rank per GPU: PushRowSparseGroup (row-range shards per rank)
      // a dense key's pull side: the value left by the push, dense or row_sparse
      auto oit = out_of.find(e.key);
      if (e.stype == kDefaultStorage && oit != out_of.end()) {
        if (e.vstype == kRowSparseStorage) {
          BroadcastRspValue(RowSparseValue(e, ogrouped[oit->second]), ogrouped[oit->second]);
        } else {
          DenseOp p;
          p.e = &e;
          p.outs = ogrouped[oit->second];
          pulls.push_back(p);
        }
      }
      continue;
    }
    KV_CHECK_EQ(e.stype, kDefaultStorage)
        << "key " << e.key << " was initialised row_sparse but a dense value was pushed";
    KV_CHECK(srcs.size() <= static_cast<size_t>(kMaxSrc))
        << "at most " << kMaxSrc << " values per key and push";
    for (auto& s : srcs) {
      KV_CHECK_EQ(s.Size(), e.size) << "push: shape mismatch for key " << e.key;
      KV_CHECK_EQ(s.dtype(), e.dtype) << "push: dtype mismatch for key " << e.key;
    }
    auto oit = out_of.find(e.key);
    KV_CHECK(!(callback && dist_))
        << "the one-rank-per-GPU store runs fused optimizers only (sgd / adam / test) or no updater";
    DensifyValue(e);
    if (callback) {
      ExecCallbackPush(e, srcs);
      if (oit != out_of.end()) {
        DenseOp p;
        p.e = &e;
        p.outs = ogrouped[oit->second];
        pulls.push_back(p);
      }
    } else {
      DenseOp op;
      op.e = &e;
      op.srcs = srcs;
      if (oit != out_of.end()) op.outs = ogrouped[oit->second];
      fused.push_back(op);
    }
  }
  // keys that are pulled but were not pushed in this call
  for (size_t i = 0; i < ouniq.size(); ++i) {
    if (pushed.count(ouniq[i])) continue;
    KeyEntry& e = Entry(ouniq[i]);
    if (e.vstype == kRowSparseStorage) {
      BroadcastRspValue(RowSparseValue(e, ogrouped[i]), ogrouped[i]);
      continue;
    }
    DenseOp p;
    p.e = &e;
    p.outs = ogrouped[i];
    pulls.push_back(p);
  }
  // a call that anchors or detaches runs launches of its own; the next identical call is cached
  std::vector<AnchorMove> moves;
  const bool moved = ResolveAnchors(&fused, &pulls, &moves);
  std::vector<Prepared> launches;
  try {
    PrepareDense(fused, opt_.enabled ? opt_.kind : kOptAssign, true, &launches);
    PrepareDense(pulls, kOptPullOnly, true, &launches);
  } catch (...) {
    UndoAnchorMoves(moves);  // a refused call leaves every stored value where it was
    throw;
  }
  for (auto& p : launches) RunPrepared(p);
  if (cacheable && !moved) StoreCachedCall(sig, std::move(launches));
}

void KVStore::PullImpl(const std::vector<int>& keys, const std::vector<NDArray>& outs,
                       bool ignore_sparse) {
  std::vector<uint64_t> sig;
  const bool cacheable = CallSignature(2, std::vector<int>(), std::vector<NDArray>(), &keys, &outs, &sig);
  if (cacheable && RunCachedCall(sig)) return;
  bool cacheable_call = cacheable;
  std::vector<int> uniq;
  std::vector<std::vector<NDArray>> grouped;
  GroupKVPairs(keys, outs, &uniq, &grouped, [this, ignore_sparse](int key, const NDArray& nd) {
    if (nd.stype() == kDefaultStorage || !ignore_sparse) return true;
    if (warnings_printed_.insert(key).second) {
      std::cerr << "Warning: non-default weights detected during kvstore pull. This call has been "
                   "ignored. Please make sure to use kv.row_sparse_pull() or module.prepare() "
                   "with row_ids.\n";
    }
    return false;
  });
  std::vector<DenseOp> pulls;
  for (size_t i = 0; i < uniq.size(); ++i) {
    KeyEntry& e = Entry(uniq[i]);
    bool plain = e.vstype == kDefaultStorage;
    for (auto& o : grouped[i]) plain = plain && o.stype() == kDefaultStorage;
    if (!plain) {
      // a row_sparse key or a row_sparse target: Comm::Broadcast degenerates to CopyFromTo with a
      // storage cast (comm.h:598-616, ndarray.cc:1147-1196) -- the whole stored value travels
      cacheable_call = false;
      if (e.vstype == kRowSparseStorage) {
        BroadcastRspValue(RowSparseValue(e, grouped[i]), grouped[i]);
        continue;
      }
      const int dev = e.striped ? devset_[0] : (e.home >= 0 ? e.home : (devset_.empty() ? 0 : devset_[0]));
      EnsureWhole(e, dev);
      const NDArray local = e.dev[e.home].w;
      for (auto& o : grouped[i]) CopyFromTo(local, o);
      continue;
    }
    DenseOp p;
    p.e = &e;
    p.outs = grouped[i];
    pulls.push_back(p);
  }
  std::vector<AnchorMove> moves;  // pulls neither form nor end anchors
  if (ResolveAnchors(nullptr, &pulls, &moves)) cacheable_call = false;
  if (pulls.empty()) return;
  std::vector<Prepared> launches;
  PrepareDense(pulls, kOptPullOnly, true, &launches);
  for (auto& p : launches) RunPrepared(p);
  if (cacheable_call) StoreCachedCall(sig, std::move(launches));
}

// =================================================================================================
// placement transitions
// =================================================================================================
void KVStore::SetDeviceSet(const std::vector<int>& devs) {
  if (devs == devset_) return;
  // a different device list: fold every striped key back onto one GPU, then re-stripe lazily
  if (devset_.size() > 1) {
    for (auto& kv : local_) {
      if (kv.second->striped) EnsureWhole(*kv.second, devset_[0]);
    }
  }
  devset_ = devs;
  plans_.clear();
  ++layout_epoch_;
  if (devs.size() > 1) {
    int enabled = Engine::Get()->EnablePeerAccess(devs);
    const int want = static_cast<int>(devs.size() * (devs.size() - 1));
    KV_CHECK_EQ(enabled, want)
        << "only " << enabled << " out of " << want << " GPU pairs allow direct peer access; the "
        << "fused device path needs all of them";
  }
}

void KVStore::EnsureOnDevice(KeyEntry& e, int dev) {
  if (e.striped || e.home >= 0) return;
  KV_CHECK(!e.host.is_none()) << "key " << e.key << " has no value";
  DevState& s = e.dev[dev];
  s.w = NDArray(e.shape, Context::GPU(dev), e.dtype);
  CopyFromTo(e.host, s.w);
  e.home = dev;
}

static void CopyIfPresent(const NDArray& from, NDArray* to, const KeyEntry& e, int dev, int dtype) {
  if (from.is_none()) return;
  if (to->is_none()) *to = NDArray(e.shape, Context::GPU(dev), dtype);
  CopyFromTo(from, *to);
}

void KVStore::EnsureStriped(KeyEntry& e) {
  if (e.striped) return;
  KV_CHECK(devset_.size() >= 1);
  if (e.home < 0) EnsureOnDevice(e, devset_[0]);
  DetachAnchor(e);
  const DevState src = e.dev[e.home];
  for (int d : devset_) {
    if (d == e.home) continue;
    DevState& s = e.dev[d];
    CopyIfPresent(src.w, &s.w, e, d, e.dtype);
    CopyIfPresent(src.w32, &s.w32, e, d, kFloat32);
    CopyIfPresent(src.s1, &s.s1, e, d, kFloat32);
    CopyIfPresent(src.s2, &s.s2, e, d, kFloat32);
  }
  e.striped = devset_.size() > 1;
  if (!e.striped && e.home != devset_[0]) {
    // single-device set: the value simply lives on that device
    e.dev[devset_[0]] = e.dev[e.home];
    e.home = devset_[0];
  }
}

int KVStore::OwnerOf(const KeyEntry& e, uint64_t global_elem) const {
  if (!e.striped) return e.home;
  return devset_[(global_elem / kBlockElems) % devset_.size()];
}

void KVStore::EnsureWhole(KeyEntry& e, int dev) {
  if (!e.striped) {
    if (e.home < 0) EnsureOnDevice(e, dev);
    return;
  }
  // gather every stripe that another GPU owns (rare path: state save, device-set change, updater
  // callback after a fused optimizer) -- plain peer copies, one per stripe
  DevState& dst = e.dev[dev];
  KV_CHECK(!dst.w.is_none());
  const size_t esz = DTypeSize(e.dtype);
  size_t pos = 0;
  while (pos < e.size) {
    const uint64_t g = e.goff + pos;
    const size_t len = std::min<size_t>(kBlockElems - g % kBlockElems, e.size - pos);
    const int owner = OwnerOf(e, g);
    if (owner != dev) {
      DevState& src = e.dev[owner];
      auto cp = [&](const NDArray& a, NDArray& b, size_t es) {
        if (a.is_none()) return;
        if (b.is_none()) b = NDArray(e.shape, Context::GPU(dev), a.dtype());
        RawCopy(static_cast<char*>(b.data()) + pos * es, b.ctx(), b.var(),
                static_cast<const char*>(a.data()) + pos * es, a.ctx(), a.var(), len * es);
      };
      cp(src.w, dst.w, esz);
      cp(src.w32, dst.w32, 4);
      cp(src.s1, dst.s1, 4);
      cp(src.s2, dst.s2, 4);
    }
    pos += len;
  }
  e.striped = false;
  e.home = dev;
  ++layout_epoch_;
}

DevState& KVStore::StateOn(KeyEntry& e, int dev, int opt_kind) {
  DevState& s = e.dev[dev];
  if (s.w.is_none()) s.w = NDArray(e.shape, Context::GPU(dev), e.dtype);
  if (opt_kind == kOptSGD || opt_kind == kOptAdam) {
    const bool need_s1 = opt_kind == kOptAdam || opt_.momentum != 0.0;  // SGD.create_state
    if (need_s1 && s.s1.is_none()) s.s1 = ZerosOn(e.shape, dev, kFloat32);
    if (opt_kind == kOptAdam && s.s2.is_none()) s.s2 = ZerosOn(e.shape, dev, kFloat32);
    if (Is16Bit(e.dtype)) {
      KV_CHECK(opt_.multi_precision)
          << "16-bit key " << e.key << ": the fused optimizer keeps fp32 master weights; create "
          << "the optimizer with multi_precision=True (accumulating in 16 bit is not implemented)";
      if (s.w32.is_none()) {
        // create_state_multi_precision: weight_master_copy = weight.astype(float32)
        s.w32 = NDArray(e.shape, Context::GPU(dev), kFloat32);
        LaneOp op(dev);
        op.Read(s.w).Write(s.w32);
        LaunchCast(s.w32.data(), kFloat32, s.w.data(), e.dtype, e.size, op.stream());
        Engine::Get()->CountLaunch("cast", e.size * (4 + DTypeSize(e.dtype)));
        op.Issue();
      }
    }
  }
  return s;
}

// Host-resident values (CPU-context NDArrays) take part through per-key staging buffers on a GPU:
// the reference's 'local' store stages the other way round (GPU -> pinned host, comm.h:146-164).
NDArray KVStore::StageSrc(KeyEntry& e, size_t slot, const NDArray& host_src, int dev) {
  if (e.stage_src.size() <= slot) e.stage_src.resize(slot + 1);
  NDArray& st = e.stage_src[slot];
  if (st.is_none() || st.dev() != dev) st = NDArray(e.shape, Context::GPU(dev), e.dtype);
  (void)host_src;  // the H2D copy is issued every time the prepared launch runs
  return st;
}

NDArray KVStore::StageOut(KeyEntry& e, size_t slot, const NDArray&, int dev) {
  if (e.stage_out.size() <= slot) e.stage_out.resize(slot + 1);
  NDArray& st = e.stage_out[slot];
  if (st.is_none() || st.dev() != dev) st = NDArray(e.shape, Context::GPU(dev), e.dtype);
  return st;
}

// =================================================================================================
// pull anchors (kvstore.h, DevState)
// =================================================================================================
bool KVStore::AnchorEligible(const KeyEntry& e) const {
  if (dist_ || e.striped || e.home < 0 || e.stype != kDefaultStorage || e.vstype != kDefaultStorage) return false;
  if (e.dtype != kFloat32 && !Is16Bit(e.dtype)) return false;
  // 16-bit keys under SGD / Adam keep fp32 master weights (or the call is refused without them)
  if (Is16Bit(e.dtype) && opt_.enabled && (opt_.kind == kOptSGD || opt_.kind == kOptAdam)) return false;
  auto it = e.dev.find(e.home);
  return it != e.dev.end() && !it->second.w.is_none() && it->second.w32.is_none();
}

// The anchor of `s` ends: `w` is the store's own buffer again (whose contents the caller provides).
static void EndAnchor(DevState& s, std::unordered_map<const Var*, KeyEntry*>* anchors) {
  s.w.var()->anchor = nullptr;
  anchors->erase(s.w.var());
  s.w = s.own;
  s.anchored = false;
}

void KVStore::DetachAnchor(KeyEntry& e) {
  auto it = e.dev.find(e.home);
  if (e.home < 0 || it == e.dev.end() || !it->second.anchored) return;
  DevState& s = it->second;
  const NDArray anchor = s.w;
  EndAnchor(s, &anchors_);
  // ordered after the anchor's last writer; a write being declared on the anchor waits for it
  CopyFromTo(anchor, s.own);
  ++layout_epoch_;
}

void KVStore::DetachVar(Var* v) {
  auto it = anchors_.find(v);
  if (it == anchors_.end()) {
    v->anchor = nullptr;
    return;
  }
  DetachAnchor(*it->second);
}

void KVStore::UndoAnchorMoves(const std::vector<AnchorMove>& moves) {
  // nothing was launched: a formed anchor was never written and `own` still holds the value; an
  // ended anchor still holds it
  for (auto it = moves.rbegin(); it != moves.rend(); ++it) {
    DevState& s = it->e->dev[it->e->home];
    if (it->formed) {
      EndAnchor(s, &anchors_);
    } else {
      s.w = it->anchor;
      s.anchored = true;
      it->anchor.var()->anchor = this;
      anchors_[it->anchor.var()] = it->e;
    }
  }
  if (!moves.empty()) ++layout_epoch_;
}

bool KVStore::ResolveAnchors(std::vector<DenseOp>* fused, std::vector<DenseOp>* pulls,
                             std::vector<AnchorMove>* moves) {
  if (dist_) return false;
  const uint64_t epoch0 = layout_epoch_;
  // B200KV_PULL_ANCHOR=0, read whenever a call is planned: no anchor forms, and the store's
  // existing anchors end here
  const char* env = std::getenv("B200KV_PULL_ANCHOR");
  const bool form = env == nullptr || env[0] != '0';
  if (!form && !anchors_.empty()) {
    std::vector<KeyEntry*> anchored;
    for (auto& a : anchors_) anchored.push_back(a.second);
    for (KeyEntry* e : anchored) DetachAnchor(*e);
  }
  std::vector<DenseOp>* lists[2] = {fused, pulls};
  // operands of the whole call per storage: an anchor is an array nothing else in the call touches
  std::unordered_map<const Storage*, int> uses, out_uses;
  for (auto* l : lists) {
    if (l == nullptr) continue;
    for (auto& op : *l) {
      for (auto& a : op.srcs) ++uses[a.storage()];
      for (auto& a : op.outs) {
        ++uses[a.storage()];
        ++out_uses[a.storage()];
      }
    }
  }
  auto sole = [&](const NDArray& a) { return a.WholeStorage() && uses[a.storage()] == 1; };
  Engine* eng = Engine::Get();
  for (int li = 0; li < 2; ++li) {
    if (lists[li] == nullptr) continue;
    const bool push = li == 0;
    for (auto& op : *lists[li]) {
      KeyEntry& e = *op.e;
      bool local = true;  // a push with a value on another GPU stripes the key
      for (auto& a : op.srcs) local = local && (!a.on_gpu() || a.dev() == e.home);
      const bool ok = AnchorEligible(e) && local;
      if (!ok) DetachAnchor(e);
      DevState* s = ok ? &e.dev[e.home] : nullptr;
      // a target that is an anchor stays one only as this key's anchor, touched by nothing else
      bool into_anchor = false;
      for (auto& o : op.outs) {
        if (o.var()->anchor == nullptr) continue;
        if (s != nullptr && s->anchored && o.SameStorage(s->w) && sole(o)) into_anchor = true;
        else eng->detach_anchor(o.var());
      }
      if (s == nullptr) continue;
      if (s->anchored) {
        if (into_anchor) {
          // the step writes the value where it lives; the anchor is no target of its own
          op.outs.erase(std::remove_if(op.outs.begin(), op.outs.end(),
                                       [&](const NDArray& o) { return o.SameStorage(s->w); }),
                        op.outs.end());
        } else if (push && out_uses[s->w.storage()] == 0) {
          // push without a pull into the anchor: the caller's array keeps the value it last
          // pulled; this step reads the value from it and writes the new one into `own`
          moves->push_back(AnchorMove{&e, s->w, false});
          op.w_in = s->w;
          EndAnchor(*s, &anchors_);
          ++layout_epoch_;
        } else if (push) {
          // ... unless another key of the call writes that array in the same launch
          DetachAnchor(e);
        }
      } else if (push && form) {
        for (size_t i = 0; i < op.outs.size(); ++i) {
          const NDArray& o = op.outs[i];
          if (!o.on_gpu() || o.dev() != e.home || o.external() || o.storage()->escaped || !sole(o) ||
              o.dtype() != e.dtype || o.Size() != e.size || o.var()->anchor != nullptr) {
            continue;
          }
          // this step reads the value from `own` and writes the new one into the anchor only
          s->own = s->w;
          op.w_in = s->own;
          s->w = o.Reshaped(e.shape);
          s->anchored = true;
          o.var()->anchor = this;
          anchors_[o.var()] = &e;
          moves->push_back(AnchorMove{&e, s->w, true});
          op.outs.erase(op.outs.begin() + i);
          ++layout_epoch_;
          break;
        }
      }
    }
  }
  if (pulls != nullptr) {
    // a pull into the anchor alone moves no bytes
    pulls->erase(std::remove_if(pulls->begin(), pulls->end(), [](const DenseOp& op) { return op.outs.empty(); }),
                 pulls->end());
  }
  return layout_epoch_ != epoch0;
}

// =================================================================================================
// the fused dense launch
// =================================================================================================
static uint64_t HashMix(uint64_t h, uint64_t v) {
  h ^= v + 0x9e3779b97f4a7c15ULL + (h << 6) + (h >> 2);
  return h;
}

std::shared_ptr<Plan> KVStore::GetPlan(const std::vector<DenseOp>& ops, int opt_kind,
                                       const std::vector<int>& owners, bool) {
  uint64_t sig = HashMix(0x1234, static_cast<uint64_t>(opt_kind));
  for (auto& op : ops) {
    sig = HashMix(sig, static_cast<uint64_t>(op.e->key));
    sig = HashMix(sig, op.e->striped ? 1000 + devset_.size() : static_cast<uint64_t>(op.e->home));
    for (auto& s : op.srcs) sig = HashMix(sig, reinterpret_cast<uint64_t>(s.data()));
    sig = HashMix(sig, 0xabcdef);
    for (auto& o : op.outs) sig = HashMix(sig, reinterpret_cast<uint64_t>(o.data()));
    sig = HashMix(sig, reinterpret_cast<uint64_t>(op.w_in.is_none() ? nullptr : op.w_in.data()));
    for (int d : owners) {
      DevState& s = op.e->dev[d];
      sig = HashMix(sig, reinterpret_cast<uint64_t>(s.w.is_none() ? nullptr : s.w.data()));
      sig = HashMix(sig, reinterpret_cast<uint64_t>(s.s1.is_none() ? nullptr : s.s1.data()));
      sig = HashMix(sig, reinterpret_cast<uint64_t>(s.s2.is_none() ? nullptr : s.s2.data()));
      sig = HashMix(sig, reinterpret_cast<uint64_t>(s.w32.is_none() ? nullptr : s.w32.data()));
    }
  }
  auto it = plans_.find(sig);
  if (it != plans_.end()) return it->second;
  if (plans_.size() > 256) plans_.clear();

  auto plan = std::make_shared<Plan>();
  plan->n_keys = static_cast<int>(ops.size());
  const int nown = static_cast<int>(owners.size());
  std::vector<std::vector<KeyDesc>> kd(nown, std::vector<KeyDesc>(ops.size()));
  std::vector<std::vector<ChunkDesc>> chunks(nown);
  auto aligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  for (size_t k = 0; k < ops.size(); ++k) {
    const DenseOp& op = ops[k];
    KeyEntry& e = *op.e;
    plan->max_src = std::max<int>(plan->max_src, static_cast<int>(op.srcs.size()));
    const size_t esz = DTypeSize(e.dtype);
    for (int oi = 0; oi < nown; ++oi) {
      const int d = owners[oi];
      KeyDesc& K = kd[oi][k];
      std::memset(&K, 0, sizeof(K));
      bool ok = true;
      for (size_t i = 0; i < op.srcs.size(); ++i) {
        K.src[i] = op.srcs[i].data();
        ok = ok && aligned(K.src[i]);
      }
      for (size_t i = 0; i < op.outs.size(); ++i) {
        K.out[i] = op.outs[i].data();
        ok = ok && aligned(K.out[i]);
      }
      DevState& s = e.dev[d];
      K.w = s.w.is_none() ? nullptr : s.w.data();
      K.w_in = op.w_in.is_none() ? K.w : op.w_in.data();
      const bool use_state = opt_kind == kOptSGD || opt_kind == kOptAdam;
      K.w32 = (use_state && !s.w32.is_none()) ? static_cast<float*>(s.w32.data()) : nullptr;
      K.s1 = (use_state && !s.s1.is_none()) ? static_cast<float*>(s.s1.data()) : nullptr;
      K.s2 = (opt_kind == kOptAdam && !s.s2.is_none()) ? static_cast<float*>(s.s2.data()) : nullptr;
      ok = ok && aligned(K.w) && aligned(K.w_in) && aligned(K.w32) && aligned(K.s1) && aligned(K.s2);
      K.n_src = static_cast<int32_t>(op.srcs.size());
      K.n_out = static_cast<int32_t>(op.outs.size());
      K.vec_ok = ok ? 1u : 0u;
    }
    // chunk ownership: slot index into `owners`
    int fixed = -1;
    if (!e.striped) {
      for (int oi = 0; oi < nown; ++oi) {
        if (owners[oi] == e.home) fixed = oi;
      }
      KV_CHECK(fixed >= 0);
    } else {
      KV_CHECK_EQ(owners.size(), devset_.size());
    }
    PlanChunks(e.goff, e.size, static_cast<uint32_t>(k), nown, fixed, &chunks);
    // algorithmic bytes (SURVEY.md 8d): every array touched exactly once
    uint64_t per_elem = op.srcs.size() * esz + op.outs.size() * esz;
    if (opt_kind != kOptPullOnly) per_elem += esz;              // stored value written
    else per_elem += esz;                                       // stored value read
    DevState& s0 = e.dev[owners[0]];
    if (opt_kind == kOptSGD || opt_kind == kOptAdam || opt_kind == kOptSGDSingle ||
        opt_kind == kOptTest) {
      per_elem += s0.w32.is_none() ? esz : 8;                   // weight read (+ master rw)
      if (!s0.s1.is_none() && (opt_kind == kOptSGD || opt_kind == kOptAdam)) per_elem += 8;
      if (!s0.s2.is_none() && opt_kind == kOptAdam) per_elem += 8;
    }
    plan->algorithmic_bytes += per_elem * e.size;
  }
  Engine* eng = Engine::Get();
  for (int oi = 0; oi < nown; ++oi) {
    Plan::PerDev p;
    p.dev = owners[oi];
    p.n_chunks = static_cast<int>(chunks[oi].size());
    p.bytes_keys = ops.size() * sizeof(KeyDesc);
    p.bytes_chunks = std::max<size_t>(chunks[oi].size(), 1) * sizeof(ChunkDesc);
    p.bytes_hyper = ops.size() * 2 * sizeof(float);
    p.d_keys = eng->Alloc(p.dev, p.bytes_keys);
    p.d_chunks = eng->Alloc(p.dev, p.bytes_chunks);
    p.d_hyper = eng->Alloc(p.dev, p.bytes_hyper);
    DeviceGuard g(p.dev);
    cudaStream_t st = eng->Stream(p.dev);
    KV_CUDA(cudaMemcpyAsync(p.d_keys, kd[oi].data(), p.bytes_keys, cudaMemcpyHostToDevice, st));
    if (!chunks[oi].empty()) {
      KV_CUDA(cudaMemcpyAsync(p.d_chunks, chunks[oi].data(), chunks[oi].size() * sizeof(ChunkDesc),
                              cudaMemcpyHostToDevice, st));
    }
    // pageable sources: the runtime has staged the bytes when cudaMemcpyAsync returns
    plan->per_dev.push_back(std::move(p));
  }
  plans_[sig] = plan;
  return plan;
}

// =================================================================================================
// updater-callback path (kvstore_local.h:217-236): reduce, then call back into the host language
// =================================================================================================
void KVStore::ExecCallbackPush(KeyEntry& e, const std::vector<NDArray>& srcs_in) {
  std::vector<NDArray> srcs = srcs_in;
  DetachAnchor(e);  // the updater writes the stored value in place
  if (e.striped) EnsureWhole(e, devset_[0]);
  if (e.home < 0) {
    int pick = 0;
    for (auto& s : srcs) {
      if (s.on_gpu()) { pick = s.dev(); break; }
    }
    EnsureOnDevice(e, pick);
  }
  const int home = e.home;
  NDArray merged;
  if (srcs.size() == 1 && srcs[0].on_gpu()) {
    merged = srcs[0].Reshaped(e.shape);  // CommDevice::Reduce returns src[0] itself (comm.h:513-515)
  } else {
    if (e.merged.is_none() || e.merged.dev() != home) e.merged = NDArray(e.shape, Context::GPU(home), e.dtype);
    merged = e.merged;
    // Assign-kernel into the merge buffer: run the dense machinery on a shadow entry whose stored
    // value IS the merge buffer
    KeyEntry shadow;
    shadow.key = e.key;
    shadow.shape = e.shape;
    shadow.dtype = e.dtype;
    shadow.size = e.size;
    shadow.goff = e.goff;
    shadow.home = home;
    shadow.dev[home].w = merged;
    shadow.stage_src = e.stage_src;
    DenseOp op;
    op.e = &shadow;
    op.srcs = srcs;
    std::vector<DenseOp> ops{op};
    ExecDense(ops, kOptAssign, /*allow_stripe=*/false);  // a merge buffer is never striped
    e.stage_src = shadow.stage_src;
  }
  NDArray local = e.dev[home].w.Reshaped(e.shape);
  // the callee owns (and frees) both handles (include/mxnet/c_api.h:2871-2882)
  NDArray* recv_h = new NDArray(merged);
  NDArray* local_h = new NDArray(local);
  if (key_type_ == 0 && str_updater_ != nullptr) {
    const std::string& sk = reverse_str_key_dict_[e.key];
    str_updater_(sk.c_str(), recv_h, local_h, updater_handle_);
  } else {
    updater_(e.key, recv_h, local_h, updater_handle_);
  }
}

// A dense key whose value is row_sparse (a row_sparse push without an updater) takes it back into
// its dense weight -- zeros plus the stored rows -- before anything reads or updates that weight.
void KVStore::DensifyValue(KeyEntry& e) {
  if (e.vstype == kDefaultStorage) return;
  DetachAnchor(e);
  BroadcastRspValue(e.rsp, {e.dev[e.home].w});
  e.rsp = NDArray();
  e.vstype = kDefaultStorage;
  ++layout_epoch_;
}

// The row_sparse value of a key on a GPU, whole: a table sharded over this process's GPUs is folded
// back onto its home; a value still on the host is copied to the GPU of the first GPU out.
NDArray KVStore::RowSparseValue(KeyEntry& e, const std::vector<NDArray>& outs) {
  KV_CHECK(!e.rsp_group) << "key " << e.key << ": a whole-value pull of a row_sparse table that is "
                         << "sharded over the ranks is not supported; use row_sparse_pull";
  UnshardRsp(e);
  if (e.rsp.on_gpu()) return e.rsp;
  int dev = 0;
  for (auto& o : outs) {
    if (o.on_gpu()) { dev = o.dev(); break; }
  }
  return e.rsp.Copy(Context::GPU(dev));
}

// =================================================================================================
// optimizer state access / introspection
// =================================================================================================
NDArray KVStore::GetOptimizerState(int key, int state_id) {
  KeyEntry& e = Entry(key);
  if (e.stype == kRowSparseStorage) {
    // states of a row_sparse table are dense [rows, row_len] arrays; a table sharded by row range
    // over this process's GPUs is folded back onto its home GPU first
    KV_CHECK(!e.rsp_group) << "key " << key << ": the table is sharded over the ranks of a peer group; "
                           << "every rank holds the state of its own row range only";
    if (!e.rsp_devs.empty()) UnshardRsp(e);
  }
  int dev = e.striped ? devset_[0] : e.home;
  KV_CHECK(dev >= 0) << "key " << key << " has no optimizer state yet";
  if (e.striped) EnsureWhole(e, dev);
  DevState& s = e.dev[dev];
  const NDArray* a = state_id == 0 ? &s.s1 : state_id == 1 ? &s.s2 : &s.w32;
  KV_CHECK(!a->is_none()) << "key " << key << " has no optimizer state " << state_id;
  return a->Copy(a->ctx());
}

void KVStore::SetOptimizerState(int key, int state_id, const NDArray& v) {
  Flush();
  KeyEntry& e = Entry(key);
  if (!e.rsp_devs.empty()) UnshardRsp(e);
  int dev = e.striped ? devset_[0] : e.home;
  if (e.striped) EnsureWhole(e, dev);
  if (dev < 0) {
    dev = v.on_gpu() ? v.dev() : 0;
    EnsureOnDevice(e, dev);
  }
  KV_CHECK_EQ(v.Size(), e.size) << "optimizer state shape mismatch for key " << key;
  KV_CHECK_EQ(v.dtype(), kFloat32) << "optimizer states are float32";
  DetachAnchor(e);  // fp32 master weights (state 2) rule an anchor out
  DevState& s = e.dev[dev];
  NDArray* a = state_id == 0 ? &s.s1 : state_id == 1 ? &s.s2 : &s.w32;
  if (a->is_none()) *a = NDArray(e.shape, Context::GPU(dev), kFloat32);
  CopyFromTo(v.Reshaped(e.shape), *a);
  plans_.clear();
  ++layout_epoch_;
}

std::string KVStore::DescribePlan(const std::vector<int>& keys, int num_devices) {
  std::ostringstream os;
  std::vector<std::vector<ChunkDesc>> chunks(num_devices);
  uint32_t slot = 0;
  for (int k : keys) {
    KeyEntry& e = Entry(k);
    PlanChunks(e.goff, e.size, slot++, num_devices, num_devices > 1 ? -1 : 0, &chunks);
  }
  os << "{\"devices\":" << num_devices << ",\"chunks\":[";
  for (int d = 0; d < num_devices; ++d) {
    uint64_t elems = 0;
    for (auto& c : chunks[d]) elems += c.len;
    os << (d ? "," : "") << "{\"n\":" << chunks[d].size() << ",\"elems\":" << elems << "}";
  }
  os << "]}";
  return os.str();
}

}  // namespace b200kv
