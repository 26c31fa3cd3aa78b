// dense_group.cc -- the dense path when the store runs as one rank per GPU (group.h).
//
// Same fused kernel, different placement: the stripes of the store-global element space rotate over
// RANKS; rank r reduces the stripes it owns reading every rank's gradient through IPC-mapped
// pointers (its own included), updates them with its slice of the optimizer state, and writes the
// new weights into every rank's pull targets. Plan building is collective (one all-gather of
// arena offsets per distinct call signature); running a prepared launch involves no host
// communication at all -- the kernel's start / end barriers order the ranks.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <map>

#include "group.h"
#include "nccl_dyn.h"
#include "kvstore.h"

namespace b200kv {

void PlanChunks(uint64_t goff, size_t size, uint32_t key_slot, int ndev, int owner_fixed,
                std::vector<std::vector<ChunkDesc>>* per_slot);  // kvstore_core.cc

namespace {
constexpr int kMaxLocalOut = 2;   // pull targets per key per rank
constexpr int kFields = 5 + kMaxLocalOut;
uint64_t Mix(uint64_t h, uint64_t v) {
  h ^= v + 0x9e3779b97f4a7c15ULL + (h << 6) + (h >> 2);
  return h;
}
size_t RoundUp(size_t x, size_t m) { return (x + m - 1) / m * m; }
}  // namespace

// ---------------------------------------------------------------------------------------------
// NCCL fallback: pack -> ncclAllReduce -> local fused update (replicated state), no peer memory
// ---------------------------------------------------------------------------------------------
// KVStoreNCCL (src/kvstore/kvstore_nccl.h:267-316,383-420) reduces every key to a root GPU and
// broadcasts it back, <= 16 keys per NCCL group. Here all keys of a call (per dtype) are packed into
// ONE flat bucket by the TMA pack kernel and summed by ONE ncclAllReduce on the compute lane's
// stream -- no host synchronisation, the collective is ordered like any other kernel -- and every
// rank then runs the fused optimizer kernel over the whole bucket (the state is replicated, as with
// update_on_kvstore in the reference). The sum's association is NCCL's: results meet the 1e-6
// relative bound of the reference's own test, not bit equality.
void KVStore::PrepareDenseNccl(std::vector<DenseOp>& ops, int opt_kind, std::vector<Prepared>* out) {
  PeerGroup* g = PeerGroup::Get();
  KV_CHECK(g != nullptr);
  const int dev = g->dev();
  const bool is_push = opt_kind != kOptPullOnly;
  std::map<int, Prepared> groups;
  std::map<int, size_t> elems;
  for (auto& op : ops) {
    KeyEntry& e = *op.e;
    KV_CHECK(op.srcs.size() <= 1) << "one-rank-per-GPU store: push exactly one value per key on each rank";
    if (e.home < 0) EnsureOnDevice(e, dev);
    KV_CHECK_EQ(e.home, dev) << "key " << e.key << " lives on another GPU than this rank's";
    groups[e.dtype].ops.push_back(op);
    elems[e.dtype] += RoundUp(std::max<size_t>(e.size, 1), kKeyAlignElems);
  }
  for (auto& kv : groups) {
    Prepared& P = kv.second;
    P.opt_kind = opt_kind;
    P.dtype = kv.first;
    P.is_push = is_push;
    P.owners = {dev};
    P.parts = {dev};
    // the padding between keys is summed too: keep it finite
    if (is_push) P.nccl_bucket = ZerosOn({static_cast<int64_t>(elems[kv.first])}, dev, kv.first);
    size_t off = 0;
    for (auto& op : P.ops) {
      KeyEntry& e = *op.e;
      for (size_t i = 0; i < op.srcs.size(); ++i) {
        KV_CHECK_EQ(op.srcs[i].Size(), e.size) << "push: shape mismatch for key " << e.key;
        KV_CHECK_EQ(op.srcs[i].dtype(), e.dtype) << "push: dtype mismatch for key " << e.key;
        NDArray seg = P.nccl_bucket.Slice(static_cast<int64_t>(off), static_cast<int64_t>(off + e.size))
                          .Reshaped(e.shape);
        P.stage_in.emplace_back(op.srcs[i], seg);
        op.srcs[i] = seg;
      }
      off += RoundUp(std::max<size_t>(e.size, 1), kKeyAlignElems);
      for (size_t i = 0; i < op.outs.size(); ++i) {
        KV_CHECK_EQ(op.outs[i].Size(), e.size) << "pull: shape mismatch for key " << e.key;
        KV_CHECK_EQ(op.outs[i].dtype(), e.dtype) << "pull: dtype mismatch for key " << e.key;
        if (!op.outs[i].on_gpu() || op.outs[i].dev() != dev) {
          NDArray st = StageOut(e, i, op.outs[i], dev);
          P.stage_out.emplace_back(st, op.outs[i]);
          op.outs[i] = st;
        }
      }
      StateOn(e, dev, opt_kind);
    }
    P.pack_in = BuildPackList(&P.stage_in);     // same-GPU sources: one TMA pack launch
    P.plan = GetPlan(P.ops, opt_kind, P.owners, /*striped=*/false);
    out->push_back(std::move(P));
  }
}

// kv.init in NCCL mode: rank 0's value reaches every rank through ncclBroadcast
void KVStore::BroadcastInitNccl(const std::vector<int>& keys) {
  PeerGroup* g = PeerGroup::Get();
  const int dev = g->dev();
  NcclComm comm = g->NcclCommunicator();
  DeviceGuard guard(dev);
  for (int key : keys) {
    KeyEntry& e = Entry(key);
    if (e.stype != kDefaultStorage) continue;
    if (e.home < 0) EnsureOnDevice(e, dev);
    KV_CHECK_EQ(e.home, dev) << "one-rank-per-GPU store: initialise keys on this rank's GPU";
    NDArray& w = e.dev[dev].w;
    LaneOp op(dev);
    op.Write(w);
    Nccl::Get()->Broadcast(w.data(), w.data(), e.size, e.dtype, 0, comm, op.stream());
    op.Issue();
  }
}

void KVStore::PrepareDenseGroup(std::vector<DenseOp>& ops, int opt_kind, std::vector<Prepared>* out) {
  if (nccl_) {
    PrepareDenseNccl(ops, opt_kind, out);
    return;
  }
  PeerGroup* g = PeerGroup::Get();
  KV_CHECK(g != nullptr);
  const int dev = g->dev();
  const bool is_push = opt_kind != kOptPullOnly;
  // One launch group per dtype. Operands outside this rank's arena (host memory, a framework's own
  // tensors) are staged through arena buffers around the launch.
  std::map<int, Prepared> groups;
  auto arena_copy = [&](const NDArray& a) { return a.on_gpu() && a.dev() == dev && g->InArena(a.data()); };
  for (auto& op : ops) {
    KeyEntry& e = *op.e;
    KV_CHECK(op.srcs.size() <= 1)
        << "one-rank-per-GPU store: push exactly one value per key on each rank (key " << e.key << ")";
    KV_CHECK(op.outs.size() <= static_cast<size_t>(kMaxLocalOut))
        << "one-rank-per-GPU store: at most " << kMaxLocalOut << " pull targets per key per rank";
    if (e.home < 0) EnsureOnDevice(e, dev);
    KV_CHECK_EQ(e.home, dev) << "key " << e.key << " lives on another GPU than this rank's";
    Prepared& P = groups[e.dtype];
    DenseOp dop = op;
    for (size_t i = 0; i < dop.srcs.size(); ++i) {
      KV_CHECK_EQ(dop.srcs[i].Size(), e.size) << "push: shape mismatch for key " << e.key;
      if (!arena_copy(dop.srcs[i])) {  // not peer-addressable: stage through the IPC arena
        NDArray st = StageSrc(e, i, dop.srcs[i], dev);
        KV_CHECK(g->InArena(st.data())) << "IPC arena exhausted; raise B200KV_IPC_ARENA_MB";
        P.stage_in.emplace_back(dop.srcs[i], st);
        dop.srcs[i] = st;
      }
    }
    for (size_t i = 0; i < dop.outs.size(); ++i) {
      KV_CHECK_EQ(dop.outs[i].Size(), e.size) << "pull: shape mismatch for key " << e.key;
      KV_CHECK_EQ(dop.outs[i].dtype(), e.dtype) << "pull: dtype mismatch for key " << e.key;
      if (!arena_copy(dop.outs[i])) {
        NDArray st = StageOut(e, i, dop.outs[i], dev);
        KV_CHECK(g->InArena(st.data())) << "IPC arena exhausted; raise B200KV_IPC_ARENA_MB";
        P.stage_out.emplace_back(st, dop.outs[i]);
        dop.outs[i] = st;
      }
    }
    P.ops.push_back(std::move(dop));
  }
  for (auto& kv : groups) {
    Prepared& P = kv.second;
    P.opt_kind = opt_kind;
    P.dtype = kv.first;
    P.is_push = is_push;
    P.group = true;
    P.owners = {dev};
    P.parts = {dev};
    for (auto& op : P.ops) StateOn(*op.e, dev, opt_kind);
    // operands that live outside the IPC arena on this GPU (a framework's own tensors) are packed
    // into / unpacked from arena staging buffers by one pack launch each way; host arrays of 1 MB
    // and more go to the copy engines instead
    constexpr size_t kDmaMinBytes = size_t{1} << 20;
    P.pack_in = BuildPackList(&P.stage_in, kDmaMinBytes);
    P.pack_out = BuildPackList(&P.stage_out, kDmaMinBytes);
    P.plan = GetPlanGroup(P.ops, opt_kind);
    out->push_back(std::move(P));
  }
}

// kv.init in a group: "only the value supplied by worker with rank 0 is used" (kvstore.py:136-141,
// the dist stores' contract). One pull-only launch whose chunks all belong to rank 0 copies rank
// 0's stored value into every rank's stored value.
void KVStore::BroadcastInitGroup(const std::vector<int>& keys) {
  PeerGroup* g = PeerGroup::Get();
  const int dev = g->dev();
  std::map<int, Prepared> groups;
  for (int key : keys) {
    KeyEntry& e = Entry(key);
    if (e.stype != kDefaultStorage) continue;
    if (e.home < 0) EnsureOnDevice(e, dev);
    KV_CHECK_EQ(e.home, dev) << "one-rank-per-GPU store: initialise keys on this rank's GPU";
    KV_CHECK(g->InArena(e.dev[dev].w.data())) << "IPC arena exhausted; raise B200KV_IPC_ARENA_MB";
    Prepared& P = groups[e.dtype];
    DenseOp op;
    op.e = &e;
    op.outs = {e.dev[dev].w};
    P.ops.push_back(op);
  }
  for (auto& kv : groups) {
    Prepared& P = kv.second;
    P.opt_kind = kOptPullOnly;
    P.dtype = kv.first;
    P.is_push = false;
    P.group = true;
    P.owners = {dev};
    P.parts = {dev};
    P.plan = GetPlanGroup(P.ops, kOptPullOnly, /*fixed_owner=*/0);
    RunPrepared(P);
  }
}

std::shared_ptr<Plan> KVStore::GetPlanGroup(const std::vector<DenseOp>& ops, int opt_kind,
                                            int fixed_owner) {
  PeerGroup* g = PeerGroup::Get();
  const int dev = g->dev(), W = g->world(), R = g->rank();
  const bool is_push = opt_kind != kOptPullOnly;
  uint64_t sig = Mix(0x6702, static_cast<uint64_t>(opt_kind) * 131 + W + 7919 * (fixed_owner + 1));
  for (auto& op : ops) {
    sig = Mix(sig, static_cast<uint64_t>(op.e->key));
    for (auto& s : op.srcs) sig = Mix(sig, reinterpret_cast<uint64_t>(s.data()));
    sig = Mix(sig, 0xabcdef);
    for (auto& o : op.outs) sig = Mix(sig, reinterpret_cast<uint64_t>(o.data()));
    DevState& s = op.e->dev[dev];
    for (const NDArray* a : {&s.w, &s.s1, &s.s2, &s.w32}) {
      sig = Mix(sig, reinterpret_cast<uint64_t>(a->is_none() ? nullptr : a->data()));
    }
  }
  auto it = plans_.find(sig);
  if (it != plans_.end()) return it->second;
  if (plans_.size() > 256) plans_.clear();

  // ---- collective: first make sure every rank plans the SAME launch (same keys) -- a mismatch
  // would otherwise pair up all-gathers of different sizes or dead-lock the kernels' barriers
  {
    uint64_t kh = 0x9b;
    for (auto& op : ops) kh = Mix(kh, static_cast<uint64_t>(op.e->key));
    const std::vector<int64_t> hdr = g->AllGatherI64(
        {static_cast<int64_t>(ops.size()), static_cast<int64_t>(kh >> 1), static_cast<int64_t>(opt_kind)});
    for (int r = 0; r < W; ++r) {
      KV_CHECK(hdr[3 * r] == hdr[3 * R] && hdr[3 * r + 1] == hdr[3 * R + 1] && hdr[3 * r + 2] == hdr[3 * R + 2])
          << "one-rank-per-GPU store: rank " << r << " issued a different call than rank " << R << " ("
          << hdr[3 * r] << " vs " << hdr[3 * R] << " keys in this launch). Every rank must push / pull "
          << "the same keys in the same order";
    }
  }
  // ---- everybody's operand offsets inside its IPC arena
  std::vector<int64_t> mine(ops.size() * kFields, -1);
  for (size_t k = 0; k < ops.size(); ++k) {
    const DenseOp& op = ops[k];
    int64_t* f = &mine[k * kFields];
    f[0] = op.e->key;
    f[1] = static_cast<int64_t>(op.e->size);
    f[2] = static_cast<int64_t>(op.e->goff);
    f[3] = op.srcs.empty() ? -1 : g->OffsetOf(op.srcs[0].data());
    f[4] = static_cast<int64_t>(op.outs.size());
    for (size_t i = 0; i < op.outs.size(); ++i) f[5 + i] = g->OffsetOf(op.outs[i].data());
  }
  const std::vector<int64_t> all = g->AllGatherI64(mine);
  auto field = [&](int r, size_t k, int i) { return all[(static_cast<size_t>(r) * ops.size() + k) * kFields + i]; };

  auto plan = std::make_shared<Plan>();
  plan->n_keys = static_cast<int>(ops.size());
  plan->max_src = is_push ? W : 0;
  std::vector<KeyDesc> kd(ops.size());
  std::vector<std::vector<ChunkDesc>> chunks(W);
  auto aligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  for (size_t k = 0; k < ops.size(); ++k) {
    const DenseOp& op = ops[k];
    KeyEntry& e = *op.e;
    KeyDesc& K = kd[k];
    std::memset(&K, 0, sizeof(K));
    bool ok = true;
    int n_out = 0;
    for (int r = 0; r < W; ++r) {
      KV_CHECK(field(r, k, 0) == e.key && field(r, k, 1) == static_cast<int64_t>(e.size) &&
               field(r, k, 2) == static_cast<int64_t>(e.goff))
          << "rank " << r << " issued a different call (key/size/order mismatch at position " << k
          << "): every rank must init and push the same keys in the same order";
      if (is_push) {
        KV_CHECK(field(r, k, 3) >= 0) << "rank " << r << " pushed no value for key " << e.key;
        K.src[r] = g->PeerPtr(r, field(r, k, 3));
        ok = ok && aligned(K.src[r]);
      }
      for (int i = 0; i < field(r, k, 4); ++i) {
        KV_CHECK(n_out < kMaxDst) << "too many pull targets across ranks for key " << e.key;
        K.out[n_out] = g->PeerPtr(r, field(r, k, 5 + i));
        ok = ok && aligned(K.out[n_out]);
        ++n_out;
      }
    }
    DevState& s = e.dev[dev];
    const bool use_state = opt_kind == kOptSGD || opt_kind == kOptAdam;
    K.w = s.w.data();
    K.w_in = K.w;
    K.w32 = (use_state && !s.w32.is_none()) ? static_cast<float*>(s.w32.data()) : nullptr;
    K.s1 = (use_state && !s.s1.is_none()) ? static_cast<float*>(s.s1.data()) : nullptr;
    K.s2 = (opt_kind == kOptAdam && !s.s2.is_none()) ? static_cast<float*>(s.s2.data()) : nullptr;
    ok = ok && aligned(K.w) && aligned(K.w32) && aligned(K.s1) && aligned(K.s2);
    K.n_src = is_push ? W : 0;
    K.n_out = n_out;
    K.vec_ok = ok ? 1u : 0u;
    PlanChunks(e.goff, e.size, static_cast<uint32_t>(k), W, fixed_owner >= 0 ? fixed_owner : (W > 1 ? -1 : 0),
               &chunks);
    // bus bytes per GPU, as tools/bandwidth/measure.py:137-138 counts them
    plan->algorithmic_bytes += static_cast<uint64_t>(e.size) * DTypeSize(e.dtype) * 2 * (W - 1) / W;
  }
  // ---- NVLS: usable when the launcher gave us a multicast mapping, the keys are fp32 and every
  // rank's operands sit at the SAME arena offsets (symmetric allocation, the normal SPMD case);
  // then the switch sums the gradients and multicasts the weights. B200KV_NVLS = 1 / 0 forces it
  // on / off; unset or "auto" uses it from 8 ranks up, where it is expected to beat peer
  // loads/stores (the crossover rank count is not measured on H100). The
  // switch picks the summation order, so this mode meets the 1e-6 relative bound of the
  // reference's own test instead of bit equality with the CPU store.
  static const int nvls_env = []() {
    const char* z = std::getenv("B200KV_NVLS");
    if (z == nullptr || z[0] == '\0' || std::strcmp(z, "auto") == 0) return -1;
    return std::atoi(z) != 0 ? 1 : 0;
  }();
  const bool want_nvls = nvls_env < 0 ? W >= 8 : nvls_env == 1;
  bool nvls = want_nvls && g->has_multicast() && fixed_owner < 0 && W >= 2 && W < kMaxSrc;
  // why a launch that wanted the switch fell back to peer loads (B200KV_DEBUG_NVLS=1, rank 0)
  static const bool debug_nvls = std::getenv("B200KV_DEBUG_NVLS") != nullptr;
  auto reject = [&](size_t k, const char* why, int r, int64_t a, int64_t b) {
    if (debug_nvls && R == 0 && nvls) {
      std::fprintf(stderr, "b200kv: NVLS off for this launch: key position %zu (key %d, %zu elements): %s (rank %d: %lld vs rank 0: %lld)\n",
                   k, ops[k].e->key, ops[k].e->size, why, r, static_cast<long long>(a), static_cast<long long>(b));
    }
    nvls = false;
  };
  for (size_t k = 0; nvls && k < ops.size(); ++k) {
    if (ops[k].e->dtype != kFloat32) reject(k, "dtype is not float32", 0, ops[k].e->dtype, 0);
    const int64_t nout = field(0, k, 4);
    if (nvls && (nout > 2 || W * nout > kMaxDst - 2)) reject(k, "too many pull targets", 0, nout, 0);
    for (int r = 1; nvls && r < W; ++r) {
      if (field(r, k, 3) != field(0, k, 3)) reject(k, "gradient at a different arena offset", r, field(r, k, 3), field(0, k, 3));
      if (nvls && field(r, k, 4) != nout) reject(k, "different number of pull targets", r, field(r, k, 4), nout);
      for (int i = 0; nvls && i < nout; ++i) {
        if (field(r, k, 5 + i) != field(0, k, 5 + i)) reject(k, "pull target at a different arena offset", r, field(r, k, 5 + i), field(0, k, 5 + i));
      }
    }
  }
  if (nvls) {
    for (size_t k = 0; k < ops.size(); ++k) {
      KeyDesc& K = kd[k];
      const int nout = static_cast<int>(field(0, k, 4));
      if (is_push) K.src[kMaxSrc - 1] = g->McPtr(field(0, k, 3));
      for (int i = 0; i < nout; ++i) K.out[kMaxDst - 2 + i] = g->McPtr(field(0, k, 5 + i));
      K.nvls = 1u + static_cast<uint32_t>(nout);
    }
    plan->max_src = 1;  // the light instantiation: the switch does the N-way sum
    plan->nvls = true;
  }
  Engine* eng = Engine::Get();
  Plan::PerDev p;
  p.dev = dev;
  std::vector<ChunkDesc>& own = chunks[R];
  p.n_chunks = static_cast<int>(own.size());
  p.bytes_keys = ops.size() * sizeof(KeyDesc);
  // the tables come out of the arena too: size them alike on every rank (the chunk counts differ
  // by a few between ranks), or the ranks' later allocations drift apart and the NVLS mode -- one
  // offset in every rank's arena -- silently falls back to peer loads for everything allocated
  // afterwards
  size_t max_chunks = 1;
  for (auto& c : chunks) max_chunks = std::max(max_chunks, c.size());
  p.bytes_chunks = max_chunks * sizeof(ChunkDesc);
  p.bytes_hyper = ops.size() * 2 * sizeof(float);
  p.d_keys = eng->Alloc(dev, p.bytes_keys);
  p.d_chunks = eng->Alloc(dev, p.bytes_chunks);
  p.d_hyper = eng->Alloc(dev, p.bytes_hyper);
  {
    DeviceGuard guard(dev);
    cudaStream_t st = eng->Stream(dev);
    KV_CUDA(cudaMemcpyAsync(p.d_keys, kd.data(), p.bytes_keys, cudaMemcpyHostToDevice, st));
    if (!own.empty()) {
      KV_CUDA(cudaMemcpyAsync(p.d_chunks, own.data(), own.size() * sizeof(ChunkDesc),
                              cudaMemcpyHostToDevice, st));
    }
  }
  plan->per_dev.push_back(std::move(p));
  plans_[sig] = plan;
  return plan;
}

}  // namespace b200kv
