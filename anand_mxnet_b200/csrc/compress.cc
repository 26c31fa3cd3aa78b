// compress.cc -- KVStore::CompressedReduce: the 2-bit gradient-compression variant of the device
// reduce (reference: CommDevice::ReduceCompressed, src/kvstore/comm.h:552-596; parameters
// src/kvstore/gradient_compression.h:41-51: type='2bit', threshold=0.5).
#include <algorithm>

#include "group.h"
#include "kvstore.h"

namespace b200kv {

// One rank per GPU. Every rank quantises ITS gradient of every key of the call with its own residual
// (what crosses NVLink afterwards is 1/16 of the gradient), the ranks meet at one barrier, and every
// rank decodes and sums ALL ranks' words -- in rank order, the reference's ElementwiseSum order -- into
// its own merged gradient: identical bits everywhere, so the update that follows runs locally with a
// replicated state (the compressed traffic is so small that replicating the decode beats sharding
// it). A second barrier releases the word buffers for the next step.
void KVStore::CompressedReduceGroup(const std::vector<KeyEntry*>& es, std::vector<std::vector<NDArray>>* srcs) {
  PeerGroup* g = PeerGroup::Get();
  KV_CHECK(g != nullptr);
  Engine* eng = Engine::Get();
  const int dev = g->dev(), W = g->world();
  DeviceGuard guard(dev);
  std::vector<int64_t> mine;
  for (size_t k = 0; k < es.size(); ++k) {
    KeyEntry& e = *es[k];
    KV_CHECK_EQ(e.dtype, kFloat32) << "2-bit gradient compression needs float32 gradients";
    KV_CHECK_EQ((*srcs)[k].size(), 1u) << "one-rank-per-GPU store: push one value per key and rank";
    if (e.home < 0) EnsureOnDevice(e, dev);
    const size_t n = e.size;
    const int64_t words = static_cast<int64_t>((n + 15) / 16);
    if (e.gc_residual.empty()) {
      e.gc_residual.resize(1);
      e.gc_compressed.resize(1);
    }
    NDArray src = (*srcs)[k][0];
    if (!src.on_gpu() || src.dev() != dev) {
      NDArray stg = StageSrc(e, 0, src, dev);
      CopyFromTo(src, stg);
      src = stg;
    }
    NDArray& res = e.gc_residual[0];
    if (res.is_none()) {
      res = ZerosOn(e.shape, dev, kFloat32);
      e.gc_compressed[0] = NDArray({words}, Context::GPU(dev), kInt32);
      KV_CHECK(g->InArena(e.gc_compressed[0].data())) << "IPC arena exhausted; raise B200KV_IPC_ARENA_MB";
    }
    NDArray& comp = e.gc_compressed[0];
    LaneOp op(dev);
    op.Read(src).Write(res).Write(comp);
    LaunchQuantize2Bit(static_cast<const float*>(src.data()), static_cast<float*>(res.data()),
                       static_cast<uint32_t*>(comp.data()), n, gc_threshold_, op.stream());
    eng->CountLaunch("quantize_2bit", n * 12 + words * 4);
    op.Issue();
    mine.push_back(e.key);
    mine.push_back(static_cast<int64_t>(n));
    mine.push_back(g->OffsetOf(comp.data()));
  }
  const std::vector<int64_t> all = g->AllGatherI64(mine);
  GroupBarrier();   // every rank's words are complete before anybody decodes them
  for (size_t k = 0; k < es.size(); ++k) {
    KeyEntry& e = *es[k];
    std::vector<const uint32_t*> ptrs(W);
    for (int r = 0; r < W; ++r) {
      const int64_t* f = &all[(static_cast<size_t>(r) * es.size() + k) * 3];
      KV_CHECK(f[0] == e.key && f[1] == static_cast<int64_t>(e.size))
          << "one-rank-per-GPU store: rank " << r << " pushed a different key list (compression)";
      ptrs[r] = static_cast<const uint32_t*>(g->PeerPtr(r, f[2]));
    }
    if (e.gc_merged.is_none()) e.gc_merged = NDArray(e.shape, Context::GPU(dev), kFloat32);
    LaneOp op(dev);
    op.Write(e.gc_merged);
    LaunchDequantizeSum2Bit(ptrs.data(), W, static_cast<float*>(e.gc_merged.data()), e.size, gc_threshold_,
                            op.stream());
    eng->CountLaunch("dequantize_sum_2bit", e.size * 4 + static_cast<uint64_t>(W) * ((e.size + 15) / 16) * 4);
    op.Issue();
    (*srcs)[k].assign(1, e.gc_merged);
  }
  GroupBarrier();   // the peers have read my words: the next quantise may overwrite them
}

NDArray KVStore::CompressedReduce(KeyEntry& e, const std::vector<NDArray>& srcs_in) {
  KV_CHECK_EQ(e.dtype, kFloat32) << "2-bit gradient compression needs float32 gradients";
  KV_CHECK(!dist_) << "one-rank-per-GPU stores compress through CompressedReduceGroup";
  Engine* eng = Engine::Get();
  if (e.striped) EnsureWhole(e, devset_[0]);
  if (e.home < 0) {
    int pick = 0;
    for (auto& s : srcs_in) {
      if (s.on_gpu()) { pick = s.dev(); break; }
    }
    EnsureOnDevice(e, pick);
  }
  const int home = e.home;
  const size_t n = e.size;
  const int64_t words = static_cast<int64_t>((n + 15) / 16);
  const size_t nsrc = srcs_in.size();
  if (e.gc_residual.size() < nsrc) {
    e.gc_residual.resize(nsrc);
    e.gc_compressed.resize(nsrc);
  }
  std::vector<int> parts{home};
  std::vector<const uint32_t*> comp_ptrs(nsrc);
  for (size_t i = 0; i < nsrc; ++i) {
    NDArray src = srcs_in[i];
    if (!src.on_gpu()) src = StageSrc(e, i, src, home), CopyFromTo(srcs_in[i], src);
    const int d = src.dev();
    if (std::find(parts.begin(), parts.end(), d) == parts.end()) parts.push_back(d);
    NDArray& res = e.gc_residual[i];
    if (res.is_none() || res.dev() != d) {
      res = ZerosOn(e.shape, d, kFloat32);   // buf.residual[i] = 0 on the source's device (comm.h:569-571)
      e.gc_compressed[i] = NDArray({words}, Context::GPU(d), kInt32);
    }
    NDArray& comp = e.gc_compressed[i];
    // quantise where the gradient lives: what crosses NVLink afterwards is 1/16 of it
    LaneOp op(d);
    op.Read(src).Write(res).Write(comp);
    LaunchQuantize2Bit(static_cast<const float*>(src.data()), static_cast<float*>(res.data()),
                       static_cast<uint32_t*>(comp.data()), n, gc_threshold_, op.stream());
    eng->CountLaunch("quantize_2bit", n * 12 + words * 4);
    op.Issue();
    comp_ptrs[i] = static_cast<const uint32_t*>(comp.data());
  }
  if (parts.size() > 1) {
    eng->RequirePeerAccess(parts);
    eng->JoinStreams(parts);
  }
  if (e.gc_merged.is_none() || e.gc_merged.dev() != home) {
    e.gc_merged = NDArray(e.shape, Context::GPU(home), kFloat32);
  }
  {
    LaneOp op(home);
    for (size_t i = 0; i < nsrc; ++i) op.Read(e.gc_compressed[i]);
    op.Write(e.gc_merged);
    LaunchDequantizeSum2Bit(comp_ptrs.data(), static_cast<int>(nsrc),
                            static_cast<float*>(e.gc_merged.data()), n, gc_threshold_, op.stream());
    eng->CountLaunch("dequantize_sum_2bit", n * 4 + nsrc * words * 4);
    op.Issue();
  }
  if (parts.size() > 1) eng->JoinStreams(parts);
  return e.gc_merged;
}

}  // namespace b200kv
