// ndarray.h -- the minimal NDArray the KVStore path needs: a ref-counted device (or pinned-host)
// buffer + shape/dtype/context/storage-type, with row_sparse support (values + int64 row ids).
// Mirrors the observable contract of include/mxnet/ndarray.h (Chunk sharing between handle copies,
// storage_initialized(), aux_shape) without any of its operator/autograd machinery.
#pragma once
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "common.h"
#include "engine.h"

namespace b200kv {

// DLPack ABI (3rdparty/dlpack/include/dlpack/dlpack.h, v0.2 layout -- stable across versions).
struct DLContextABI { int device_type; int device_id; };
struct DLDataTypeABI { uint8_t code; uint8_t bits; uint16_t lanes; };
struct DLTensorABI {
  void* data; DLContextABI ctx; int ndim; DLDataTypeABI dtype; int64_t* shape; int64_t* strides;
  uint64_t byte_offset;
};
struct DLManagedTensorABI {
  DLTensorABI dl_tensor; void* manager_ctx; void (*deleter)(DLManagedTensorABI*);
};

// Shared by every NDArray handle that aliases one value (the reference's NDArray::Chunk).
struct Storage {
  Context ctx;
  void* dptr = nullptr;
  size_t bytes = 0;
  void* aux = nullptr;  // row_sparse: int64 row ids, ascending & unique
  size_t aux_bytes = 0;
  int64_t nnr = 0;      // row_sparse: rows stored; 0 == storage not initialised == all zeros
  bool external = false;
  // a raw pointer to the memory went out (MXNDArrayGetData, DLPack export): writes through it are
  // invisible to the engine, so the array never becomes a pull anchor (kvstore.h)
  bool escaped = false;
  std::function<void()> deleter;
  Var var;
  ~Storage();
};

// Immutable shape shared between handle copies: copying an NDArray (the C API does it for every
// operand of every call) must not allocate.
class SharedShape {
 public:
  SharedShape() : p_(Empty()) {}
  SharedShape(const std::vector<int64_t>& v)  // NOLINT(runtime/explicit)
      : p_(std::make_shared<const std::vector<int64_t>>(v)) {}
  SharedShape& operator=(const std::vector<int64_t>& v) {
    p_ = std::make_shared<const std::vector<int64_t>>(v);
    return *this;
  }
  operator const std::vector<int64_t>&() const { return *p_; }  // NOLINT(runtime/explicit)
  const std::vector<int64_t>& get() const { return *p_; }

 private:
  static const std::shared_ptr<const std::vector<int64_t>>& Empty() {
    static const auto* e = new std::shared_ptr<const std::vector<int64_t>>(
        std::make_shared<const std::vector<int64_t>>());
    return *e;
  }
  std::shared_ptr<const std::vector<int64_t>> p_;
};

class NDArray {
 public:
  NDArray() {}
  // dense
  NDArray(const std::vector<int64_t>& shape, Context ctx, int dtype, bool delay_alloc = false);
  // row_sparse (always delay-allocated: no rows until CheckAndAllocRows)
  static NDArray RowSparse(const std::vector<int64_t>& shape, Context ctx, int dtype);
  static NDArray FromDLPack(DLManagedTensorABI* t, bool transient);

  bool is_none() const { return st_ == nullptr; }
  const std::vector<int64_t>& shape() const { return shape_.get(); }
  int dtype() const { return dtype_; }
  int stype() const { return stype_; }
  Context ctx() const { return st_ ? st_->ctx : Context(); }
  int dev() const { return st_->ctx.dev_id; }
  bool on_gpu() const { return st_ && st_->ctx.is_gpu(); }
  // host array in the library's own pinned+mapped memory: kernels can address it directly (UVA),
  // so the fused kernel reads gradients from / writes weights to it over PCIe without staging
  bool kernel_visible_host() const { return st_ && !st_->ctx.is_gpu() && !st_->external; }
  bool external() const { return st_ && st_->external; }  // memory owned by another framework (DLPack)
  bool kernel_visible() const { return on_gpu() || kernel_visible_host(); }
  size_t Size() const;        // product of shape
  size_t RowLength() const;   // product of shape[1:]
  size_t ByteSize() const { return Size() * DTypeSize(dtype_); }
  Var* var() const { return &st_->var; }
  Storage* storage() const { return st_.get(); }
  long use_count() const { return st_.use_count(); }   // holders of the underlying storage
  bool SameStorage(const NDArray& o) const { return st_ == o.st_; }
  // the view covers its storage's bytes exactly (offset 0, whole allocation)
  bool WholeStorage() const { return !aux_view_ && byte_offset_ == 0 && ByteSize() == st_->bytes; }
  // a raw pointer to the memory is handed out: a pull anchor in it ends, and it never becomes one
  void Escape() const;

  void Alloc() const;  // dense: allocate if delayed
  void* data() const;  // dense values / row_sparse value rows
  int64_t* row_ids() const { return static_cast<int64_t*>(st_->aux); }
  int64_t nnr() const { return st_->nnr; }
  bool storage_initialized() const { return stype_ == kDefaultStorage ? true : st_->nnr > 0; }
  // row_sparse: make room for `nnr` rows (contents undefined) and set aux_shape = nnr
  void CheckAndAllocRows(int64_t nnr) const;
  bool RowsFit(int64_t nnr) const;  // CheckAndAllocRows(nnr) would not re-allocate
  void SetNnr(int64_t nnr) const { st_->nnr = nnr; }

  // views used by MXNDArrayGetDataNDArray / GetAuxNDArray: dense arrays aliasing the blobs
  NDArray DataView() const;
  NDArray AuxView() const;
  NDArray Reshaped(const std::vector<int64_t>& shape) const;
  // rows [begin, end) of the first axis, sharing storage (NDArray::Slice, src/ndarray/ndarray.cc)
  NDArray Slice(int64_t begin, int64_t end) const;

  // NDArray::Save / Load (src/ndarray/ndarray.cc:1596-1670, 1672-1827): the V2 binary format --
  // magic 0xF993fac9, stype, [storage shape], shape (int32 ndim + int64 dims), context, type
  // flag, [aux type + shape], data, [aux data]. Load also accepts the V1 / legacy layouts.
  void SaveRaw(std::string* out) const;
  static NDArray LoadRaw(const char* buf, size_t size, size_t* consumed);

  // Deep copy into a fresh array on ctx (NDArray::Copy, src/ndarray/ndarray.cc:...)
  NDArray Copy(Context ctx) const;

 private:
  friend class LaneOp;
  std::shared_ptr<Storage> st_;
  SharedShape shape_;
  int dtype_ = kFloat32;
  int stype_ = kDefaultStorage;
  size_t byte_offset_ = 0;
  bool aux_view_ = false;
};

// CopyFromTo (src/ndarray/ndarray.cc:1198-1296): asynchronous copy as an engine op; self-copy and
// zero-size copies are skipped; handles every CPU/pinned/GPU/peer combination, dense and row_sparse.
void CopyFromTo(const NDArray& from, const NDArray& to);
// Raw async copy of `bytes` between two contexts on the right stream; used by CopyFromTo and the
// host<->device staging of MXNDArraySyncCopy*.
void RawCopy(void* dst, Context dctx, Var* dvar, const void* src, Context sctx, Var* svar,
             size_t bytes);

// One operation on one engine lane (the reference's Engine::PushAsync with its const and mutable
// var lists), with the lane's device current for its lifetime:
//     LaneOp op(lane);
//     op.Read(a).Write(b);   // the lane waits for a's writer, and for b's writer and readers
//     ... enqueue on op.stream() ...
//     op.Issue();            // marks a read and b written by this operation
// Each array is named once, so its wait and its mark cannot disagree. Issue() marks the reads
// before the writes: an array declared both ways ends as written. The declared arrays are held
// until the op is destroyed, so scratch arrays outlive their marks. An op destroyed without Issue()
// (an exception between declaring and enqueueing) marks nothing. A none array (an absent optional
// operand) is skipped.
class LaneOp {
 public:
  explicit LaneOp(int lane);
  LaneOp(const LaneOp&) = delete;
  LaneOp& operator=(const LaneOp&) = delete;

  LaneOp& Read(const NDArray& a) { return a.is_none() ? *this : Add(a.var(), false, a.st_); }
  LaneOp& Write(const NDArray& a) { return a.is_none() ? *this : Add(a.var(), true, a.st_); }
  LaneOp& Read(Var* v) { return Add(v, false, nullptr); }   // the caller keeps *v alive
  LaneOp& Write(Var* v) { return Add(v, true, nullptr); }
  int lane() const { return lane_; }
  cudaStream_t stream() const { return stream_; }
  uint64_t Issue();  // returns the operation's sequence number on the lane

 private:
  struct Use {
    Var* var = nullptr;
    bool write = false;
    std::shared_ptr<Storage> keep;
  };
  LaneOp& Add(Var* v, bool write, const std::shared_ptr<Storage>& keep);
  Use& At(int i) { return i < kInline ? inline_[i] : spill_[i - kInline]; }

  static constexpr int kInline = 8;  // no heap allocation for the common operation
  int lane_;
  cudaStream_t stream_;
  DeviceGuard guard_;
  Use inline_[kInline];
  std::vector<Use> spill_;
  int n_ = 0;
};

// A dense array of zeros on GPU `dev`, filled on that GPU's compute lane. The fill is the array's
// first writer, so it waits for whatever a recycled block's previous owner left pending.
NDArray ZerosOn(const std::vector<int64_t>& shape, int dev, int dtype);

}  // namespace b200kv
