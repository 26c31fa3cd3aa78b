// dense_exec.cc -- prepare / run split of the fused dense launch and the call-level cache.
//
// A training loop repeats the same C call every step (same keys, same arrays). Everything that
// does not change between steps -- grouping, validation, placement, state allocation, descriptor
// tables on the device, the list of arrays whose dependencies are tracked -- is computed once
// (PrepareDense) and cached by the call's signature; a repeated call only replays RunPrepared:
// staging copies (host-resident operands), update counts, (lr, wd) refresh when a hyper-parameter
// changed, dependency bookkeeping, ONE kernel launch per owner GPU. This is what keeps the host
// cost of a 157-key pushpull in the microseconds, below what the kernel itself takes.
#include <algorithm>
#include <cmath>
#include <map>
#include <set>

#include "group.h"
#include "nccl_dyn.h"
#include "kvstore.h"
#include "scalar_parse.h"

namespace b200kv {

static uint64_t Mix(uint64_t h, uint64_t v) {
  h ^= v + 0x9e3779b97f4a7c15ULL + (h << 6) + (h >> 2);
  return h;
}

// ---------------------------------------------------------------------------------------------
// same-GPU staging copies as one TMA bulk-copy launch
// ---------------------------------------------------------------------------------------------
PackList::~PackList() { Engine::Get()->Free(dev, d_items, bytes_items); }

// Moves the same-GPU pairs of `pairs` into a PackList (tiles of <= 16 KB uploaded once).
// dma_min_bytes > 0: pairs with a host side of at least that size are LEFT to the copy engines
// (CopyFromTo on the copy lanes). The copy engines move big arrays faster than SM-driven packing with
// both directions busy, but a DMA carries a fixed cost of microseconds -- so big arrays go by DMA and
// the many small ones by one pack launch.
std::shared_ptr<PackList> BuildPackList(std::vector<std::pair<NDArray, NDArray>>* pairs, size_t dma_min_bytes) {
  std::vector<std::pair<NDArray, NDArray>> rest;
  auto pl = std::make_shared<PackList>();
  std::vector<PackItem> items;
  for (auto& pr : *pairs) {
    const NDArray& from = pr.first;
    const NDArray& to = pr.second;
    // same-GPU pairs, or one side in kernel-visible pinned host memory (the SMs then drive the
    // PCIe transfer with TMA bulk copies: one launch instead of one cudaMemcpyAsync per array)
    int pdev = -1;
    if (from.on_gpu() && to.on_gpu() && from.dev() == to.dev()) pdev = from.dev();
    else if (from.on_gpu() && to.kernel_visible_host()) pdev = from.dev();
    else if (to.on_gpu() && from.kernel_visible_host()) pdev = to.dev();
    const bool host_side = !from.on_gpu() || !to.on_gpu();
    if (pdev < 0 || (pl->dev >= 0 && pdev != pl->dev) ||
        (host_side && dma_min_bytes > 0 && from.ByteSize() >= dma_min_bytes)) {
      rest.push_back(pr);
      continue;
    }
    pl->dev = pdev;
    if (!from.on_gpu()) { pl->host_io = true; pl->lane = Engine::CopyInLane(pdev); }
    if (!to.on_gpu()) { pl->host_io = true; pl->lane = Engine::CopyOutLane(pdev); }
    const char* s = static_cast<const char*>(from.data());
    char* d = static_cast<char*>(to.data());
    const uint64_t n = from.ByteSize();
    for (uint64_t off = 0; off < n; off += kPackTileBytes) {
      items.push_back(PackItem{s + off, d + off, std::min<uint64_t>(kPackTileBytes, n - off)});
    }
    pl->total_bytes += n;
    pl->pairs.push_back(pr);
  }
  *pairs = rest;
  if (items.empty()) return nullptr;
  Engine* eng = Engine::Get();
  if (pl->lane < 0) pl->lane = pl->dev;
  pl->n_items = static_cast<int>(items.size());
  pl->bytes_items = items.size() * sizeof(PackItem);
  pl->d_items = eng->Alloc(pl->dev, pl->bytes_items);
  DeviceGuard g(pl->dev);
  KV_CUDA(cudaMemcpyAsync(pl->d_items, items.data(), pl->bytes_items, cudaMemcpyHostToDevice,
                          eng->Stream(pl->dev)));
  if (pl->lane != pl->dev) {
    // the item table was uploaded on the compute lane; the copy lane must see it
    const uint64_t seq = eng->Issue(pl->dev);
    eng->StreamWait(pl->lane, Tag{pl->dev, seq});
  }
  return pl;
}

void RunPackList(PackList& pl) {
  LaneOp op(pl.lane);
  for (auto& pr : pl.pairs) op.Read(pr.first).Write(pr.second);
  LaunchPackBulk(static_cast<const PackItem*>(pl.d_items), pl.n_items, op.stream(), pl.host_io);
  Engine::Get()->CountLaunch("pack_bulk(tma)", 2 * pl.total_bytes);
  op.Issue();
}

// ---------------------------------------------------------------------------------------------
// call-level cache
// ---------------------------------------------------------------------------------------------
bool KVStore::CallSignature(int tag, const std::vector<int>& vkeys, const std::vector<NDArray>& values,
                            const std::vector<int>* okeys, const std::vector<NDArray>* outs,
                            std::vector<uint64_t>* sig) {
  sig->clear();
  sig->reserve(5 + 3 * vkeys.size() + (okeys ? 3 * okeys->size() : 0));
  sig->push_back(static_cast<uint64_t>(tag));
  sig->push_back(vkeys.size());
  for (size_t i = 0; i < vkeys.size(); ++i) {
    const NDArray& a = values[i];
    if (a.is_none() || a.stype() != kDefaultStorage) return false;  // row_sparse: slow path
    sig->push_back(static_cast<uint64_t>(static_cast<int64_t>(vkeys[i])));
    sig->push_back(reinterpret_cast<uint64_t>(a.storage()) ^ (reinterpret_cast<uint64_t>(a.data()) << 1));
    sig->push_back(static_cast<uint64_t>(a.Size()) * 16 + static_cast<uint64_t>(a.dtype()));  // a view of another length must not hit
  }
  sig->push_back(0xfeedULL);
  if (okeys != nullptr) {
    for (size_t i = 0; i < okeys->size(); ++i) {
      const NDArray& a = (*outs)[i];
      if (a.is_none() || a.stype() != kDefaultStorage) return false;
      sig->push_back(static_cast<uint64_t>(static_cast<int64_t>((*okeys)[i])));
      sig->push_back(reinterpret_cast<uint64_t>(a.storage()) ^ (reinterpret_cast<uint64_t>(a.data()) << 1));
      sig->push_back(static_cast<uint64_t>(a.Size()) * 16 + static_cast<uint64_t>(a.dtype()));
    }
  }
  return true;
}

static uint64_t HashSig(const std::vector<uint64_t>& sig) {
  uint64_t h = 0x51ed270b;
  for (uint64_t v : sig) h = Mix(h, v);
  return h;
}

bool KVStore::RunCachedCall(const std::vector<uint64_t>& sig) {
  auto it = call_cache_.find(HashSig(sig));
  if (it == call_cache_.end()) return false;
  CachedCall& c = *it->second;
  if (c.epoch != layout_epoch_ || c.sig != sig) {
    call_cache_.erase(it);
    return false;
  }
  for (auto& p : c.launches) RunPrepared(p);
  return true;
}

void KVStore::StoreCachedCall(const std::vector<uint64_t>& sig, std::vector<Prepared>&& launches) {
  // A cached call keeps its operand arrays alive. Training loops repeat a handful of signatures;
  // imperative use with fresh gradient arrays every step would otherwise pin one gradient set per
  // entry: first drop the entries nobody but the cache still holds operands of, then cap the size.
  if (call_cache_.size() >= 8) {
    for (auto it = call_cache_.begin(); it != call_cache_.end();) {
      bool orphan = false;
      for (auto& p : it->second->launches) {
        for (auto& op : p.ops) {
          for (auto& a : op.srcs) orphan = orphan || a.use_count() <= 1;
          for (auto& a : op.outs) orphan = orphan || a.use_count() <= 1;
        }
      }
      it = orphan ? call_cache_.erase(it) : std::next(it);
    }
  }
  if (call_cache_.size() > 32) call_cache_.clear();
  auto c = std::make_shared<CachedCall>();
  c->sig = sig;
  c->launches = std::move(launches);
  c->epoch = layout_epoch_;
  call_cache_[HashSig(sig)] = c;
}

// ---------------------------------------------------------------------------------------------
// prepare: placement, staging buffers, state, plan
// ---------------------------------------------------------------------------------------------
void KVStore::ExecDense(std::vector<DenseOp>& ops, int opt_kind, bool allow_stripe) {
  std::vector<Prepared> launches;
  PrepareDense(ops, opt_kind, allow_stripe, &launches);
  for (auto& p : launches) RunPrepared(p);
}

void KVStore::PrepareDense(std::vector<DenseOp>& ops, int opt_kind, bool allow_stripe,
                           std::vector<Prepared>* out) {
  if (ops.empty()) return;
  if (dist_ && !force_local_) {
    (void)allow_stripe;
    PrepareDenseGroup(ops, opt_kind, out);
    return;
  }
  const bool is_push = opt_kind != kOptPullOnly;
  // ---- 1. device set: a push with values on >= 2 GPUs (re)defines the stripe owners
  if (is_push && allow_stripe) {
    std::vector<int> devs;
    for (auto& s : ops[0].srcs) {
      if (s.on_gpu() && std::find(devs.begin(), devs.end(), s.dev()) == devs.end()) devs.push_back(s.dev());
    }
    if (devs.size() >= 2) SetDeviceSet(devs);
  }
  // ---- 2. placement of every key; foreign host memory gets device staging buffers
  // Launch groups: (dtype, striped?, home, bucket). Arrays in the library's own pinned+mapped host
  // memory are handed to the kernel as they are (it reads gradients / writes weights over PCIe
  // itself: one launch, no copies, both PCIe directions busy at once); foreign host memory is
  // staged through the GPU. A group with staged operands is cut into buckets of ~8 MB of staged
  // bytes so the H2D copy of bucket b+1, the kernel of bucket b and the D2H copy of bucket b-1 run
  // concurrently on the three lanes.
  constexpr size_t kStageBucketBytes = size_t{8} << 20;
  std::map<std::tuple<int, int, int, int>, Prepared> groups;
  std::map<std::tuple<int, int, int>, std::pair<int, size_t>> bucket_of;  // -> (bucket, bytes)
  for (auto& op : ops) {
    KeyEntry& e = *op.e;
    std::vector<int> sdev;
    for (auto& s : op.srcs) {
      if (s.on_gpu() && std::find(sdev.begin(), sdev.end(), s.dev()) == sdev.end()) sdev.push_back(s.dev());
    }
    if (is_push && allow_stripe && sdev.size() >= 2) {
      KV_CHECK(sdev == devset_) << "key " << e.key << ": values live on a different GPU list than "
                                << "the other keys of this push";
      EnsureStriped(e);
    } else if (!e.striped && e.home < 0) {
      int pick = -1;
      for (auto& s : op.srcs) if (pick < 0 && s.on_gpu()) pick = s.dev();
      for (auto& o : op.outs) if (pick < 0 && o.on_gpu()) pick = o.dev();
      if (pick < 0) pick = devset_.empty() ? 0 : devset_[0];
      EnsureOnDevice(e, pick);
    }
    KV_CHECK(op.outs.size() <= static_cast<size_t>(kMaxDst)) << "at most " << kMaxDst << " outs per key";
    const auto gkey = std::make_tuple(e.dtype, e.striped ? 1 : 0, e.striped ? -1 : e.home);
    size_t staged = 0;
    for (auto& s : op.srcs) if (!s.kernel_visible()) staged += s.ByteSize();
    for (auto& o : op.outs) if (!o.kernel_visible()) staged += o.ByteSize();
    auto& bk = bucket_of[gkey];
    if (staged > 0 && bk.second > 0 && bk.second + staged > kStageBucketBytes) {
      ++bk.first;
      bk.second = 0;
    }
    bk.second += staged;
    Prepared& P = groups[std::make_tuple(std::get<0>(gkey), std::get<1>(gkey), std::get<2>(gkey), bk.first)];
    const int stage_dev = e.striped ? devset_[0] : e.home;
    DenseOp dop = op;
    for (size_t i = 0; i < dop.srcs.size(); ++i) {
      if (!dop.srcs[i].kernel_visible()) {
        NDArray st = StageSrc(e, i, dop.srcs[i], stage_dev);
        P.stage_in.emplace_back(dop.srcs[i], st);
        dop.srcs[i] = st;
      }
    }
    for (size_t i = 0; i < dop.outs.size(); ++i) {
      KV_CHECK_EQ(dop.outs[i].Size(), e.size) << "pull: shape mismatch for key " << e.key;
      KV_CHECK_EQ(dop.outs[i].dtype(), e.dtype) << "pull: dtype mismatch for key " << e.key;
      if (!dop.outs[i].kernel_visible()) {
        NDArray st = StageOut(e, i, dop.outs[i], stage_dev);
        P.stage_out.emplace_back(st, dop.outs[i]);
        dop.outs[i] = st;
      }
    }
    P.ops.push_back(std::move(dop));
  }
  Engine* eng = Engine::Get();
  for (auto& kv : groups) {
    Prepared& P = kv.second;
    P.opt_kind = opt_kind;
    P.dtype = std::get<0>(kv.first);
    P.is_push = is_push;
    P.owners = P.ops[0].e->striped ? devset_ : std::vector<int>{P.ops[0].e->home};
    for (auto& op : P.ops) {
      for (int d : P.owners) StateOn(*op.e, d, opt_kind);
    }
    P.plan = GetPlan(P.ops, opt_kind, P.owners, P.ops[0].e->striped);
    std::set<int> part_set(P.owners.begin(), P.owners.end());
    for (auto& op : P.ops) {
      for (auto& s : op.srcs) if (s.on_gpu()) part_set.insert(s.dev());
      for (auto& o : op.outs) if (o.on_gpu()) part_set.insert(o.dev());
    }
    P.parts.assign(part_set.begin(), part_set.end());
    eng->RequirePeerAccess(P.parts);
    out->push_back(std::move(P));
  }
}

// ---------------------------------------------------------------------------------------------
// run: what happens on every step
// ---------------------------------------------------------------------------------------------
void KVStore::RunPrepared(Prepared& P) {
  Engine* eng = Engine::Get();
  const int opt_kind = P.opt_kind;
  const bool fused_opt = P.is_push && opt_.enabled && (opt_kind == kOptSGD || opt_kind == kOptAdam);
  if (P.pack_in) RunPackList(*P.pack_in);
  for (auto& io : P.stage_in) CopyFromTo(io.first, io.second);
  if (!P.nccl_bucket.is_none()) {
    // NCCL fallback: sum the packed gradients of all ranks in place, on the compute lane's stream
    PeerGroup* g = PeerGroup::Get();
    KV_CHECK(g != nullptr) << "the peer group was destroyed while a store still uses it";
    const int dev = g->dev();
    NcclComm comm = g->NcclCommunicator();
    LaneOp op(dev);
    op.Write(P.nccl_bucket);
    Nccl::Get()->AllReduceSum(P.nccl_bucket.data(), P.nccl_bucket.data(), P.nccl_bucket.Size(), P.dtype, comm,
                              op.stream());
    eng->CountLaunch("ncclAllReduce", P.nccl_bucket.ByteSize());
    op.Issue();
  }

  // ---- optimizer bookkeeping: update counts first (Optimizer._update_count, optimizer.py:412-430)
  if (fused_opt) {
    for (auto& op : P.ops) {
      auto it = opt_.count.find(op.e->key);
      const int c = (it == opt_.count.end() ? opt_.begin_num_update : it->second) + 1;
      if (it == opt_.count.end()) opt_.count[op.e->key] = c; else it->second = c;
      opt_.num_update = std::max(opt_.num_update, c);
    }
  }
  // per-key (lr, wd) and the scalar parameters: refreshed when a hyper-parameter changed (and on
  // every step for Adam, whose effective lr depends on the per-key update count)
  if (P.hyper_version != opt_version_ || opt_kind == kOptAdam) {
    P.hyper.resize(P.ops.size() * 2);
    for (size_t k = 0; k < P.ops.size(); ++k) {
      KeyHyper(*P.ops[k].e, opt_kind, &P.hyper[2 * k], &P.hyper[2 * k + 1]);
    }
    if (P.hyper_version != opt_version_) {
      DenseLaunch& L = P.scalars;
      L = DenseLaunch();
      if (opt_kind == kOptSGD) {
        // SGD._update_impl (optimizer.py:618-624): momentum only if > 0, clip only if truthy
        L.momentum = opt_.momentum > 0 ? ScalarParam(opt_.momentum) : 0.f;
        L.rescale = ScalarParam(opt_.rescale);
        L.clip = opt_.clip != 0.0 ? ScalarParam(opt_.clip) : -1.f;
      } else if (opt_kind == kOptAdam) {
        L.rescale = ScalarParam(opt_.rescale);
        L.clip = opt_.clip != 0.0 ? ScalarParam(opt_.clip) : -1.f;
        L.beta1 = ScalarParam(opt_.beta1);
        L.beta2 = ScalarParam(opt_.beta2);
        L.eps = ScalarParam(opt_.eps);
      } else if (opt_kind == kOptTest) {
        // Test.update's `grad * self.rescale_grad` is _mul_scalar: std::stod, then float32
        L.rescale = StodParam(opt_.rescale);
      }
      P.hyper_version = opt_version_;
    }
  }

  // ---- dependencies
  const bool multi = P.parts.size() > 1;
  const int host_lane = P.owners[0];  // kernel-visible host operands are touched by the owners' kernels
  auto lane_of = [&](const NDArray& a) { return a.on_gpu() ? a.dev() : host_lane; };
  // arrays the kernel reads besides the state: the sources, and `w_in` when the call moves the
  // stored value between the store's buffer and a pull anchor
  auto for_reads = [](const DenseOp& op, auto&& f) {
    for (auto& s : op.srcs) f(s);
    if (!op.w_in.is_none()) f(op.w_in);
  };
  for (auto& op : P.ops) {
    for_reads(op, [&](const NDArray& s) { eng->BeginRead(lane_of(s), *s.var()); });
    for (auto& o : op.outs) eng->BeginWrite(lane_of(o), *o.var());
    for (int d : P.owners) {
      DevState& s = op.e->dev[d];
      if (P.is_push) {
        Engine::AnchorWriteScope anchored_step;  // `w` may be the key's pull anchor
        eng->BeginWrite(d, *s.w.var());
      } else {
        eng->BeginRead(d, *s.w.var());
      }
    }
  }
  if (multi) eng->JoinStreams(P.parts);

  // ---- launch, one kernel per owner
  DenseLaunch L = P.scalars;
  L.max_src = P.plan->max_src;
  L.nvls = P.plan->nvls;
  L.dtype = P.dtype;
  L.opt = opt_kind;
  L.order = order_local_ ? kOrderLocal : kOrderDevice;
  for (auto& pd : P.plan->per_dev) {
    DeviceGuard g(pd.dev);
    cudaStream_t st = eng->Stream(pd.dev);
    if (pd.hyper != P.hyper) {
      KV_CUDA(cudaMemcpyAsync(pd.d_hyper, P.hyper.data(), P.hyper.size() * sizeof(float),
                              cudaMemcpyHostToDevice, st));
      pd.hyper = P.hyper;
    }
    if (pd.n_chunks == 0 && !P.group) continue;
    if (P.group) {
      // one rank per GPU: in-kernel start/end barriers on the IPC signal pads order the ranks
      PeerGroup* g = PeerGroup::Get();
      KV_CHECK(g != nullptr) << "the peer group was destroyed while a store still uses it";
      g->FillLaunch(&L);
      // gate launch: the start barrier runs in a one-CTA kernel ahead of the fused kernel (same
      // epoch, start flags only), so a rank whose peers are late -- a checkpoint, an evaluation
      // pass, a slow data loader on one rank -- waits with ONE resident CTA instead of a grid of
      // spinning ones, and the SMs stay free for whatever else its streams have queued.
      DenseLaunch G;
      G.signal_pads = L.signal_pads;
      G.counter = L.counter;
      G.rank = L.rank;
      G.world = L.world;
      G.epoch = L.epoch;
      G.err_word = L.err_word;
      G.timeout_ns = L.timeout_ns;
      G.n_chunks = 0;
      G.dtype = kFloat32;
      G.opt = kOptAssign;
      G.barrier_mask = 1;
      LaunchDenseFused(G, st);
      L.barrier_mask = 2;
    }
    L.keys = static_cast<const KeyDesc*>(pd.d_keys);
    L.chunks = static_cast<const ChunkDesc*>(pd.d_chunks);
    L.hyper = static_cast<const float*>(pd.d_hyper);
    L.n_chunks = pd.n_chunks;
    LaunchDenseFused(L, st);
    eng->CountLaunch(P.plan->nvls ? "dense_fused(nvls)" : "dense_fused",
                     P.plan->algorithmic_bytes / P.plan->per_dev.size());
  }
  if (multi) eng->JoinStreams(P.parts);

  // ---- mark results
  uint64_t seq[kMaxDevices] = {0};
  for (int d : P.parts) seq[d] = eng->Issue(d);
  for (auto& op : P.ops) {
    for_reads(op, [&](const NDArray& s) { eng->MarkRead(lane_of(s), seq[lane_of(s)], s.var()); });
    for (auto& o : op.outs) eng->MarkWrite(lane_of(o), seq[lane_of(o)], o.var());
    for (int d : P.owners) {
      DevState& s = op.e->dev[d];
      if (P.is_push) {
        eng->MarkWrite(d, seq[d], s.w.var());
        if (!s.w32.is_none()) eng->MarkWrite(d, seq[d], s.w32.var());
        if (!s.s1.is_none()) eng->MarkWrite(d, seq[d], s.s1.var());
        if (!s.s2.is_none()) eng->MarkWrite(d, seq[d], s.s2.var());
      } else {
        eng->MarkRead(d, seq[d], s.w.var());
      }
    }
  }
  if (P.pack_out) RunPackList(*P.pack_out);
  for (auto& io : P.stage_out) CopyFromTo(io.first, io.second);
}

}  // namespace b200kv
