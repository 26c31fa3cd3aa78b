// engine.h -- the stream/event scheduler that stands in for MXNet's dependency engine on this path.
//
// Reference contract (include/mxnet/engine.h:95-112,204-275; src/engine/threaded_engine_perdevice.cc):
// every operation declares the arrays it reads and the arrays it mutates; the engine guarantees
// read-after-write / write-after-read / write-after-write order per array, runs independent work
// concurrently, and lets the caller block with WaitForVar / WaitForAll. The reference realises that
// with worker threads that each own one CUDA stream (normal / priority / copy pools per GPU) and a
// `cudaStreamSynchronize` after every op.
//
// Design: no worker threads and no per-op host synchronisation. Each GPU has THREE in-order
// lanes -- compute (library-owned, or a caller-provided stream via B200KVEngineSetStream so KVStore
// work is ordered with the framework that produced the gradients), host-to-device copies, and
// device-to-host copies (the reference's kCopyToGPU / kCopyFromGPU pools) -- so PCIe traffic in
// both directions overlaps the kernels. A lane is identified by a stream id:
//     sid = dev (compute), kMaxDevices + dev (H2D), 2*kMaxDevices + dev (D2H).
// An array carries the tags (sid, sequence-number) of its last writer and last readers; same-lane
// order is stream order, cross-lane order is a cudaStreamWaitEvent on an event recorded lazily --
// only when some other lane (or the host) actually has to wait. Host waits are
// cudaEventSynchronize.
#pragma once
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "common.h"

namespace b200kv {

constexpr int kMaxStreams = 3 * kMaxDevices;

struct Tag {
  int dev = -1;      // stream id of the lane (-1: no pending device work)
  uint64_t seq = 0;  // position in that lane's issue order
};

// Per-array dependency record (the reference's engine::Var).
struct Var {
  Tag writer;
  uint64_t reader_seq[kMaxStreams] = {0};  // last read issued on each lane
  bool has_readers = false;
  // deferred failure of the asynchronous operation that last wrote the array: re-thrown by the
  // next wait on it (src/engine/threaded_engine.h:380-387, ThrowException / var_exception)
  std::shared_ptr<std::string> err;
  // the store that keeps a key's value in this array (a pull anchor, kvstore.h), or null
  void* anchor = nullptr;
};

class Engine {
 public:
  static Engine* Get();

  static int DevOf(int sid) { return sid % kMaxDevices; }
  static int CopyInLane(int dev) { return kMaxDevices + dev; }
  static int CopyOutLane(int dev) { return 2 * kMaxDevices + dev; }

  int NumDevices();
  cudaStream_t Stream(int sid);
  void SetStream(int dev, cudaStream_t s);  // compute lane; nullptr restores the library's stream

  // ---- dependency protocol: call BeginRead/BeginWrite before enqueueing an op on lane `sid`, then
  // Issue(sid) once the op is enqueued and Mark* the arrays with the returned sequence number.
  // An op on one lane uses LaneOp (ndarray.h), which names each array once for both steps.
  void BeginRead(int sid, const Var& v);   // lane waits for v's writer
  void BeginWrite(int sid, const Var& v);  // ... and for every reader
  // Copy-on-write of pull anchors: a write declared on an anchor (BeginWrite, WaitToWrite) first
  // calls detach_anchor, which hands the value back to the store -- a copy enqueued after the
  // anchor's last writer, so ahead of the new write. The store's own fused step writes its anchors
  // inside an AnchorWriteScope.
  void (*detach_anchor)(Var* v) = nullptr;
  int anchor_writes_ok = 0;
  struct AnchorWriteScope {
    AnchorWriteScope() { ++Get()->anchor_writes_ok; }
    ~AnchorWriteScope() { --Get()->anchor_writes_ok; }
  };
  uint64_t Issue(int sid);
  void MarkRead(int sid, uint64_t seq, Var* v);
  void MarkWrite(int sid, uint64_t seq, Var* v);

  void StreamWait(int sid, Tag t);  // lane `sid` waits for device work `t`
  void HostWait(Tag t);             // calling thread waits for device work `t`
  void WaitToRead(const Var& v);
  void WaitToWrite(const Var& v);
  void WaitAll();
  // ---- deferred errors. An asynchronous operation that fails cannot report to the call that
  // enqueued it; the failure is parked on the arrays it was to write and re-thrown (once) by the
  // next WaitToRead / WaitToWrite of such an array, or by WaitAll.
  void SetError(Var* v, const std::string& msg);
  // device-side failures (a peer-barrier time-out inside a kernel) land in a pinned host word the
  // kernels can write; every host wait checks it. Returns the device-visible pointer.
  uint32_t* DeviceErrorWord();
  void CheckDeviceError();
  // Full barrier among lanes: everything issued so far on any of them completes before anything
  // issued afterwards on any of them starts (2N event operations, not N^2).
  void JoinStreams(const std::vector<int>& sids);

  // ---- memory (pooled: blocks are cached per device and size class, never returned to the driver
  // before shutdown; the reference's GPUPooledStorageManager plays the same role)
  // A cached block remembers the device work that may still touch it (the dying array's last
  // writer / readers, or "everything issued so far on the device's compute lane" for raw blocks).
  // Re-use hands that record on: to the new array's Var (`fresh`: whichever lane -- copy lanes and
  // peer GPUs included -- first writes the array waits for it), or, for raw blocks, to the
  // compute lane of `dev` (raw blocks are tables / scratch of that lane's kernels).
  void* Alloc(int dev, size_t bytes, Var* fresh = nullptr);
  void Free(int dev, void* p, size_t bytes, const Var* last_use = nullptr);
  void* AllocPinned(size_t bytes);
  void FreePinned(void* p, size_t bytes);
  size_t BytesAllocated(int dev);

  // src/kvstore/comm.h:715-757 (EnableP2P): returns the number of ordered pairs enabled
  int EnablePeerAccess(const std::vector<int>& devs);
  // ... and fails unless every ordered pair of `devs` has peer access
  void RequirePeerAccess(const std::vector<int>& devs);
  bool PeerEnabled(int a, int b);

  std::recursive_mutex& mutex() { return mu_; }
  void Shutdown();

  // launch accounting (bench.py's gpu_launches, tests)
  void CountLaunch(const char* name, uint64_t algorithmic_bytes);
  uint64_t launch_count = 0;
  const char* last_kernel = "";
  uint64_t last_kernel_bytes = 0;

 private:
  Engine();
  void Init();
  cudaEvent_t RecordLatest(int sid);
  static size_t RoundSize(size_t bytes);

  struct Lane {
    cudaStream_t own = nullptr, cur = nullptr;
    std::vector<cudaEvent_t> ring;
    size_t ring_pos = 0;
    cudaEvent_t latest = nullptr;
    uint64_t issued = 0, recorded = 0, completed = 0;
    uint64_t waited[kMaxStreams] = {0};  // waited[e]: this lane already waits for e's seq <= value
  };
  struct Block {
    void* p = nullptr;
    Var pending;
  };
  struct DevMem {
    std::multimap<size_t, Block> pool;
    size_t bytes = 0;
  };
  std::vector<Lane> lanes_;
  std::vector<DevMem> mem_;
  int ndev_ = 0;
  std::multimap<size_t, void*> pinned_pool_;
  std::shared_ptr<std::string> global_err_;   // first unreported deferred failure (for WaitAll)
  volatile uint32_t* dev_err_ = nullptr;      // pinned + mapped
  bool peer_[kMaxDevices][kMaxDevices] = {{false}};
  bool inited_ = false;
  std::recursive_mutex mu_;
};

// RAII: switch the calling thread's current CUDA device.
struct DeviceGuard {
  explicit DeviceGuard(int dev) {
    KV_CUDA(cudaGetDevice(&prev_));
    if (prev_ != dev) KV_CUDA(cudaSetDevice(dev));
    dev_ = dev;
  }
  ~DeviceGuard() {
    if (prev_ != dev_) cudaSetDevice(prev_);
  }
  int prev_ = 0, dev_ = 0;
};

}  // namespace b200kv
