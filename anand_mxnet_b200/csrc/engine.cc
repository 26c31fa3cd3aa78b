// engine.cc -- see engine.h.
#include "engine.h"

#include <algorithm>

#include "group.h"

namespace b200kv {

Engine* Engine::Get() {
  static Engine* inst = new Engine();  // intentionally leaked: no static-destruction-order races
  return inst;
}

Engine::Engine() {}

void Engine::Init() {
  if (inited_) return;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    cudaGetLastError();
    KV_FATAL << "libb200kv needs a CUDA device and found none (" << cudaGetErrorString(e)
             << "); there is no CPU fallback for the KVStore path";
  }
  ndev_ = std::min(n, kMaxDevices);
  lanes_.resize(kMaxStreams);
  mem_.resize(ndev_);
  inited_ = true;
}

int Engine::NumDevices() {
  Init();
  return ndev_;
}

cudaStream_t Engine::Stream(int sid) {
  Init();
  const int dev = DevOf(sid);
  KV_CHECK(sid >= 0 && sid < kMaxStreams && dev < ndev_) << "invalid gpu id " << dev;
  Lane& d = lanes_[sid];
  if (d.own == nullptr) {
    DeviceGuard g(dev);
    KV_CUDA(cudaStreamCreateWithFlags(&d.own, cudaStreamNonBlocking));
    d.ring.resize(16);
    for (auto& ev : d.ring) KV_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    if (d.cur == nullptr) d.cur = d.own;
  }
  return d.cur;
}

void Engine::SetStream(int dev, cudaStream_t s) {
  cudaStream_t old = Stream(dev);
  Lane& d = lanes_[dev];
  cudaStream_t next = s ? s : d.own;
  if (next == old) return;
  // work already issued on the old stream stays ordered before work on the new one
  DeviceGuard g(dev);
  ++d.issued;  // force a fresh event: the caller's framework may have enqueued work we never saw
  cudaEvent_t ev = RecordLatest(dev);
  KV_CUDA(cudaStreamWaitEvent(next, ev, 0));
  d.cur = next;
}

cudaEvent_t Engine::RecordLatest(int sid) {
  Stream(sid);
  Lane& d = lanes_[sid];
  if (d.latest == nullptr || d.recorded < d.issued) {
    DeviceGuard g(DevOf(sid));
    d.ring_pos = (d.ring_pos + 1) % d.ring.size();
    d.latest = d.ring[d.ring_pos];
    KV_CUDA(cudaEventRecord(d.latest, d.cur));
    d.recorded = d.issued;
  }
  return d.latest;
}

uint64_t Engine::Issue(int sid) {
  Stream(sid);
  return ++lanes_[sid].issued;
}

void Engine::StreamWait(int sid, Tag t) {
  if (t.dev < 0 || t.dev == sid) return;  // same lane: stream order
  Stream(sid);
  Lane& d = lanes_[sid];
  if (d.waited[t.dev] >= t.seq) return;
  if (lanes_[t.dev].completed >= t.seq) return;
  cudaEvent_t ev = RecordLatest(t.dev);
  DeviceGuard g(DevOf(sid));
  KV_CUDA(cudaStreamWaitEvent(d.cur, ev, 0));
  d.waited[t.dev] = lanes_[t.dev].recorded;
}

void Engine::HostWait(Tag t) {
  if (t.dev < 0) return;
  Init();
  Lane& d = lanes_[t.dev];
  if (d.completed >= t.seq) return;
  cudaEvent_t ev = RecordLatest(t.dev);
  uint64_t upto = d.recorded;
  KV_CUDA(cudaEventSynchronize(ev));
  d.completed = std::max(d.completed, upto);
}

void Engine::BeginRead(int sid, const Var& v) { StreamWait(sid, v.writer); }

void Engine::BeginWrite(int sid, const Var& v) {
  if (v.anchor != nullptr && anchor_writes_ok == 0) detach_anchor(const_cast<Var*>(&v));
  StreamWait(sid, v.writer);
  if (v.has_readers) {
    for (int e = 0; e < kMaxStreams; ++e) {
      if (v.reader_seq[e]) StreamWait(sid, Tag{e, v.reader_seq[e]});
    }
  }
}

void Engine::MarkRead(int sid, uint64_t seq, Var* v) {
  v->reader_seq[sid] = seq;
  v->has_readers = true;
}

void Engine::MarkWrite(int sid, uint64_t seq, Var* v) {
  v->writer = Tag{sid, seq};
  if (v->err) v->err.reset();  // a new writer supersedes the failed one
  if (v->has_readers) {
    for (int e = 0; e < kMaxStreams; ++e) v->reader_seq[e] = 0;
    v->has_readers = false;
  }
}

// Re-throw (once) the failure parked on `v`; mirrors ThreadedEngine::WaitForVar, which rethrows the
// var's exception and clears it (src/engine/threaded_engine.cc:375-420).
static void ThrowParked(const Var& v, std::shared_ptr<std::string>* global) {
  if (!v.err || v.err->empty()) return;
  const std::string msg = *v.err;
  v.err->clear();  // shared with every copy of the record: reported once
  if (*global && (*global)->empty()) global->reset();
  KV_FATAL << msg;
}

void Engine::WaitToRead(const Var& v) {
  HostWait(v.writer);
  CheckDeviceError();
  ThrowParked(v, &global_err_);
}

void Engine::WaitToWrite(const Var& v) {
  if (v.anchor != nullptr && anchor_writes_ok == 0) detach_anchor(const_cast<Var*>(&v));
  HostWait(v.writer);
  if (v.has_readers) {
    for (int e = 0; e < kMaxStreams; ++e) {
      if (v.reader_seq[e]) HostWait(Tag{e, v.reader_seq[e]});
    }
  }
  CheckDeviceError();
  ThrowParked(v, &global_err_);
}

void Engine::SetError(Var* v, const std::string& msg) {
  v->err = std::make_shared<std::string>(msg);
  if (!global_err_ || global_err_->empty()) global_err_ = v->err;
}

uint32_t* Engine::DeviceErrorWord() {
  if (dev_err_ == nullptr) {
    void* p = nullptr;
    KV_CUDA(cudaHostAlloc(&p, 64, cudaHostAllocMapped | cudaHostAllocPortable));
    dev_err_ = static_cast<volatile uint32_t*>(p);
    dev_err_[0] = 0;
    dev_err_[1] = 0;
  }
  void* d = nullptr;
  KV_CUDA(cudaHostGetDevicePointer(&d, const_cast<uint32_t*>(dev_err_), 0));
  return static_cast<uint32_t*>(d);
}

void Engine::CheckDeviceError() {
  if (dev_err_ == nullptr || dev_err_[0] == 0) return;
  const uint32_t code = dev_err_[0], info = dev_err_[1];
  dev_err_[0] = 0;
  dev_err_[1] = 0;
  KV_FATAL << "one-rank-per-GPU store: this rank waited longer than B200KV_PEER_TIMEOUT_S for rank "
           << (code - 1) << " inside a fused kernel (barrier phase " << (info >> 31) << ", epoch "
           << (info & 0x7fffffffu) << "): the peer never launched the matching call, or died. "
           << "Results of the affected call are undefined; the process itself stays usable";
}

void Engine::WaitAll() {
  if (!inited_) return;
  for (int e = 0; e < kMaxStreams; ++e) {
    Lane& d = lanes_[e];
    if (d.cur == nullptr) continue;
    DeviceGuard g(DevOf(e));
    uint64_t upto = d.issued;
    KV_CUDA(cudaStreamSynchronize(d.cur));
    d.completed = std::max(d.completed, upto);
  }
  CheckDeviceError();
  if (global_err_ && !global_err_->empty()) {   // WaitForAll rethrows any pending failure
    const std::string msg = *global_err_;
    global_err_->clear();
    global_err_.reset();
    KV_FATAL << msg;
  }
}

void Engine::JoinStreams(const std::vector<int>& sids) {
  if (sids.size() < 2) return;
  // hub = sids[0]: it waits for every other stream, then every other stream waits for it.
  // Issue() on every stream first so that a fresh event is recorded even when the only new work on
  // a (caller-provided) stream was enqueued by the caller's framework and never counted here.
  const int hub = sids[0];
  for (size_t i = 1; i < sids.size(); ++i) {
    uint64_t s = Issue(sids[i]);
    StreamWait(hub, Tag{sids[i], s});
  }
  uint64_t seq = Issue(hub);
  for (size_t i = 1; i < sids.size(); ++i) StreamWait(sids[i], Tag{hub, seq});
}

// ---------------------------------------------------------------------------------------------
size_t Engine::RoundSize(size_t bytes) {
  if (bytes == 0) bytes = 1;
  if (bytes <= (1u << 20)) return (bytes + 511) & ~static_cast<size_t>(511);
  return (bytes + (2u << 20) - 1) & ~static_cast<size_t>((2u << 20) - 1);
}

void* Engine::Alloc(int dev, size_t bytes, Var* fresh) {
  Init();
  KV_CHECK(dev >= 0 && dev < ndev_) << "invalid gpu id " << dev;
  DevMem& d = mem_[dev];
  size_t r = RoundSize(bytes);
  auto range = d.pool.equal_range(r);
  if (range.first != range.second) {
    // lowest address of the size class: which block an allocation gets then depends only on the SET
    // of free blocks, not on the order they were freed in -- ranks that released the same arrays in
    // a different order (garbage collection) still hand out the same arena offsets, which the NVLS
    // mode needs (a multicast address is one offset in every rank's arena)
    auto it = range.first;
    for (auto j = range.first; j != range.second; ++j) {
      if (j->second.p < it->second.p) it = j;
    }
    const Block b = it->second;
    d.pool.erase(it);
    if (fresh != nullptr) {
      // every pending op becomes a "reader" of the new array: its first writer waits for all
      auto carry = [&](Tag t) {
        if (t.dev < 0 || t.seq == 0 || lanes_[t.dev].completed >= t.seq) return;
        fresh->reader_seq[t.dev] = std::max(fresh->reader_seq[t.dev], t.seq);
        fresh->has_readers = true;
      };
      carry(b.pending.writer);
      if (b.pending.has_readers) {
        for (int e = 0; e < kMaxStreams; ++e) carry(Tag{e, b.pending.reader_seq[e]});
      }
    } else {
      BeginWrite(dev, b.pending);
    }
    return b.p;
  }
  if (PeerGroup* grp = PeerGroup::Get()) {
    // one-rank-per-GPU mode: allocations come out of the IPC arena so peers can address them
    if (grp->dev() == dev) {
      void* ap = grp->ArenaAlloc(r);
      if (ap != nullptr) return ap;
    }
  }
  DeviceGuard g(dev);
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, r);
  if (e != cudaSuccess) {
    cudaGetLastError();
    // release the cache and retry once
    WaitAll();
    for (auto& kv : d.pool) cudaFree(kv.second.p);
    d.pool.clear();
    KV_CUDA(cudaMalloc(&p, r));
  }
  d.bytes += r;
  return p;
}

void Engine::Free(int dev, void* p, size_t bytes, const Var* last_use) {
  if (p == nullptr || !inited_) return;
  Block b;
  b.p = p;
  if (last_use != nullptr) {
    b.pending = *last_use;
    b.pending.err.reset();
    b.pending.anchor = nullptr;
  } else {
    b.pending.writer = Tag{dev, lanes_[dev].issued};
  }
  mem_[dev].pool.emplace(RoundSize(bytes), b);
}

void* Engine::AllocPinned(size_t bytes) {
  Init();
  size_t r = RoundSize(bytes);
  auto it = pinned_pool_.find(r);
  if (it != pinned_pool_.end()) {
    void* p = it->second;
    pinned_pool_.erase(it);
    return p;
  }
  void* p = nullptr;
  // portable + mapped: every GPU's kernels can read/write it through the same (UVA) pointer
  KV_CUDA(cudaHostAlloc(&p, r, cudaHostAllocPortable | cudaHostAllocMapped));
  return p;
}

void Engine::FreePinned(void* p, size_t bytes) {
  if (p == nullptr) return;
  pinned_pool_.emplace(RoundSize(bytes), p);
}

size_t Engine::BytesAllocated(int dev) {
  Init();
  return mem_[dev].bytes;
}

int Engine::EnablePeerAccess(const std::vector<int>& devs) {
  Init();
  int enabled = 0;
  for (int a : devs) {
    for (int b : devs) {
      if (a == b) continue;
      if (peer_[a][b]) {
        ++enabled;
        continue;
      }
      DeviceGuard g(a);
      int can = 0;
      KV_CUDA(cudaDeviceCanAccessPeer(&can, a, b));
      if (!can) continue;
      cudaError_t e = cudaDeviceEnablePeerAccess(b, 0);
      if (e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled) {
        cudaGetLastError();
        peer_[a][b] = true;
        ++enabled;
      } else {
        cudaGetLastError();
      }
    }
  }
  return enabled;
}

void Engine::RequirePeerAccess(const std::vector<int>& devs) {
  if (devs.size() < 2) return;
  KV_CHECK_EQ(EnablePeerAccess(devs), static_cast<int>(devs.size() * (devs.size() - 1)))
      << "GPU peer access is not available between all participating devices";
}

bool Engine::PeerEnabled(int a, int b) { return a == b || peer_[a][b]; }

void Engine::CountLaunch(const char* name, uint64_t algorithmic_bytes) {
  ++launch_count;
  last_kernel = name;
  last_kernel_bytes = algorithmic_bytes;
}

void Engine::Shutdown() {
  if (!inited_) return;
  WaitAll();
}

}  // namespace b200kv
