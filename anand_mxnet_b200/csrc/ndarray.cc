// ndarray.cc -- see ndarray.h.
#include "ndarray.h"

#include "rowsparse.h"

#include <cstring>

namespace b200kv {

Storage::~Storage() {
  if (external) {
    if (deleter) deleter();
    return;
  }
  Engine* e = Engine::Get();
  try {
    if (ctx.is_gpu()) {
      e->Free(ctx.dev_id, dptr, bytes, &var);
      e->Free(ctx.dev_id, aux, aux_bytes, &var);
    } else {
      // a pinned host block may still be the target/source of an in-flight async copy
      e->WaitToWrite(var);
      e->FreePinned(dptr, bytes);
      e->FreePinned(aux, aux_bytes);
    }
  } catch (...) {
  }
}

static size_t Prod(const std::vector<int64_t>& s, size_t from = 0) {
  size_t n = 1;
  for (size_t i = from; i < s.size(); ++i) n *= static_cast<size_t>(s[i]);
  return n;
}

static void* AllocOn(Context ctx, size_t bytes, Var* var) {
  Engine* e = Engine::Get();
  if (ctx.is_gpu()) return e->Alloc(ctx.dev_id, bytes, var);
  return e->AllocPinned(bytes);  // every host-side array is pinned so H2D/D2H copies are async DMA
}

NDArray::NDArray(const std::vector<int64_t>& shape, Context ctx, int dtype, bool delay_alloc)
    : shape_(shape), dtype_(dtype), stype_(kDefaultStorage) {
  for (auto d : shape) KV_CHECK(d >= 0) << "negative dimension in shape";
  st_ = std::make_shared<Storage>();
  st_->ctx = ctx;
  if (ctx.is_gpu()) {
    KV_CHECK(ctx.dev_id >= 0 && ctx.dev_id < Engine::Get()->NumDevices())
        << "invalid gpu id " << ctx.dev_id;
  }
  if (!delay_alloc) Alloc();
}

NDArray NDArray::RowSparse(const std::vector<int64_t>& shape, Context ctx, int dtype) {
  KV_CHECK(shape.size() >= 1) << "row_sparse needs at least 1 dimension";
  NDArray a;
  a.shape_ = shape;
  a.dtype_ = dtype;
  a.stype_ = kRowSparseStorage;
  a.st_ = std::make_shared<Storage>();
  a.st_->ctx = ctx;
  a.st_->nnr = 0;
  return a;
}

size_t NDArray::Size() const { return Prod(shape_); }
size_t NDArray::RowLength() const { return Prod(shape_, 1); }

void NDArray::Alloc() const {
  if (st_->dptr != nullptr || stype_ != kDefaultStorage) return;
  size_t bytes = ByteSize();
  if (bytes == 0) return;
  st_->dptr = AllocOn(st_->ctx, bytes, &st_->var);
  st_->bytes = bytes;
}

void* NDArray::data() const {
  if (aux_view_) return st_->aux;
  if (stype_ == kDefaultStorage) Alloc();
  return static_cast<char*>(st_->dptr) + byte_offset_;
}

bool NDArray::RowsFit(int64_t nnr) const {
  return static_cast<size_t>(nnr) * RowLength() * DTypeSize(dtype_) <= st_->bytes &&
         static_cast<size_t>(nnr) * sizeof(int64_t) <= st_->aux_bytes;
}

void NDArray::CheckAndAllocRows(int64_t nnr) const {
  KV_CHECK_EQ(stype_, kRowSparseStorage);
  KV_CHECK(!st_->external) << "cannot re-allocate an external row_sparse array";
  Engine* e = Engine::Get();
  size_t need = static_cast<size_t>(nnr) * RowLength() * DTypeSize(dtype_);
  size_t need_aux = static_cast<size_t>(nnr) * sizeof(int64_t);
  if (need > st_->bytes) {
    if (st_->ctx.is_gpu()) e->Free(st_->ctx.dev_id, st_->dptr, st_->bytes, &st_->var);
    else { e->WaitToWrite(st_->var); e->FreePinned(st_->dptr, st_->bytes); }
    st_->dptr = AllocOn(st_->ctx, need, &st_->var);
    st_->bytes = need;
  }
  if (need_aux > st_->aux_bytes) {
    if (st_->ctx.is_gpu()) e->Free(st_->ctx.dev_id, st_->aux, st_->aux_bytes, &st_->var);
    else { e->WaitToWrite(st_->var); e->FreePinned(st_->aux, st_->aux_bytes); }
    st_->aux = AllocOn(st_->ctx, need_aux, &st_->var);
    st_->aux_bytes = need_aux;
  }
  st_->nnr = nnr;
}

NDArray NDArray::DataView() const {
  NDArray v = *this;
  v.stype_ = kDefaultStorage;
  if (stype_ == kRowSparseStorage) {
    std::vector<int64_t> s = shape_.get();
    s[0] = st_->nnr;
    v.shape_ = s;
  }
  return v;
}

NDArray NDArray::AuxView() const {
  KV_CHECK_EQ(stype_, kRowSparseStorage) << "only row_sparse arrays have aux data";
  NDArray v = *this;
  v.stype_ = kDefaultStorage;
  v.dtype_ = kInt64;
  v.shape_ = std::vector<int64_t>{st_->nnr};
  v.aux_view_ = true;
  return v;
}

void NDArray::Escape() const {
  if (st_ == nullptr) return;
  st_->escaped = true;
  Engine* e = Engine::Get();
  if (st_->var.anchor == nullptr) return;
  e->detach_anchor(&st_->var);
  // whoever writes through the pointer is not ordered by the engine: the copy that took the value
  // out of this array completes first
  e->WaitToWrite(st_->var);
}

NDArray NDArray::Reshaped(const std::vector<int64_t>& shape) const {
  KV_CHECK_EQ(Prod(shape), Size()) << "reshape size mismatch";
  NDArray v = *this;
  v.shape_ = shape;
  return v;
}

NDArray NDArray::Slice(int64_t begin, int64_t end) const {
  KV_CHECK_EQ(stype_, kDefaultStorage) << "Slice: only dense arrays can be sliced";
  KV_CHECK(!shape().empty() && begin >= 0 && begin <= end && end <= shape()[0])
      << "Slice: invalid range [" << begin << ", " << end << ") for axis of length "
      << (shape().empty() ? 0 : shape()[0]);
  NDArray v = *this;
  std::vector<int64_t> sh = shape();
  sh[0] = end - begin;
  v.shape_ = sh;
  v.byte_offset_ = byte_offset_ + static_cast<size_t>(begin) * RowLength() * DTypeSize(dtype_);
  return v;
}

NDArray NDArray::FromDLPack(DLManagedTensorABI* t, bool transient) {
  const DLTensorABI& d = t->dl_tensor;
  NDArray a;
  a.st_ = std::make_shared<Storage>();
  KV_CHECK(d.ctx.device_type == 1 || d.ctx.device_type == 2 || d.ctx.device_type == 3)
      << "unsupported DLPack device type " << d.ctx.device_type;
  a.st_->ctx = d.ctx.device_type == 2 ? Context::GPU(d.ctx.device_id)
                                       : Context{d.ctx.device_type == 3 ? kCPUPinned : kCPU, 0};
  KV_CHECK_EQ(d.dtype.lanes, 1);
  int dt = -1;
  if (d.dtype.code == 2 && d.dtype.bits == 32) dt = kFloat32;
  else if (d.dtype.code == 2 && d.dtype.bits == 64) dt = kFloat64;
  else if (d.dtype.code == 2 && d.dtype.bits == 16) dt = kFloat16;
  else if (d.dtype.code == 4 && d.dtype.bits == 16) dt = kBfloat16;
  else if (d.dtype.code == 0 && d.dtype.bits == 32) dt = kInt32;
  else if (d.dtype.code == 0 && d.dtype.bits == 64) dt = kInt64;
  else if (d.dtype.code == 0 && d.dtype.bits == 8) dt = kInt8;
  else if (d.dtype.code == 1 && d.dtype.bits == 8) dt = kUint8;
  KV_CHECK(dt >= 0) << "unsupported DLPack dtype code " << int(d.dtype.code) << " bits "
                    << int(d.dtype.bits);
  a.dtype_ = dt;
  a.shape_ = std::vector<int64_t>(d.shape, d.shape + d.ndim);
  if (d.strides != nullptr) {  // must be compact row-major
    int64_t expect = 1;
    for (int i = d.ndim - 1; i >= 0; --i) {
      KV_CHECK(d.shape[i] <= 1 || d.strides[i] == expect) << "DLPack tensor is not contiguous";
      expect *= d.shape[i];
    }
  }
  a.st_->dptr = static_cast<char*>(d.data) + d.byte_offset;
  a.st_->bytes = a.ByteSize();
  a.st_->external = true;
  if (!transient) a.st_->deleter = [t]() { if (t->deleter) t->deleter(t); };
  return a;
}

NDArray NDArray::Copy(Context ctx) const {
  NDArray out = stype_ == kRowSparseStorage ? RowSparse(shape_, ctx, dtype_)
                                            : NDArray(shape_, ctx, dtype_);
  CopyFromTo(*this, out);
  return out;
}

// ---------------------------------------------------------------------------------------------
void RawCopy(void* dst, Context dctx, Var* dvar, const void* src, Context sctx, Var* svar,
             size_t bytes) {
  if (bytes == 0 || dst == src) return;
  Engine* e = Engine::Get();
  Var none;
  if (dvar == nullptr) dvar = &none;
  if (svar == nullptr) svar = &none;
  if (!dctx.is_gpu() && !sctx.is_gpu()) {
    e->WaitToRead(*svar);
    e->WaitToWrite(*dvar);
    std::memcpy(dst, src, bytes);
    return;
  }
  // device<->device copies run on the destination GPU's compute lane; host->device and
  // device->host copies on that GPU's dedicated copy lanes, so both PCIe directions overlap the
  // kernels (the reference's kCopyToGPU / kCopyFromGPU worker pools)
  int lane;
  if (dctx.is_gpu() && sctx.is_gpu()) lane = dctx.dev_id;
  else if (dctx.is_gpu()) lane = Engine::CopyInLane(dctx.dev_id);
  else lane = Engine::CopyOutLane(sctx.dev_id);
  LaneOp op(lane);
  op.Read(svar).Write(dvar);
  if (dctx.is_gpu() && sctx.is_gpu() && dctx.dev_id != sctx.dev_id) {
    KV_CUDA(cudaMemcpyPeerAsync(dst, dctx.dev_id, src, sctx.dev_id, bytes, op.stream()));
  } else {
    KV_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, op.stream()));
  }
  op.Issue();
}

LaneOp::LaneOp(int lane)
    : lane_(lane), stream_(Engine::Get()->Stream(lane)), guard_(Engine::DevOf(lane)) {}

LaneOp& LaneOp::Add(Var* v, bool write, const std::shared_ptr<Storage>& keep) {
  Engine* e = Engine::Get();
  if (write) e->BeginWrite(lane_, *v);
  else e->BeginRead(lane_, *v);
  if (n_ >= kInline) spill_.emplace_back();
  Use& u = At(n_++);
  u.var = v;
  u.write = write;
  u.keep = keep;
  return *this;
}

uint64_t LaneOp::Issue() {
  Engine* e = Engine::Get();
  const uint64_t seq = e->Issue(lane_);
  for (int i = 0; i < n_; ++i) {
    if (!At(i).write) e->MarkRead(lane_, seq, At(i).var);
  }
  for (int i = 0; i < n_; ++i) {
    if (At(i).write) e->MarkWrite(lane_, seq, At(i).var);
  }
  return seq;
}

NDArray ZerosOn(const std::vector<int64_t>& shape, int dev, int dtype) {
  NDArray a(shape, Context::GPU(dev), dtype);
  if (a.Size() == 0) return a;
  LaneOp op(dev);
  op.Write(a);
  KV_CUDA(cudaMemsetAsync(a.data(), 0, a.ByteSize(), op.stream()));
  op.Issue();
  return a;
}

void CopyFromTo(const NDArray& from, const NDArray& to) {
  KV_CHECK(!from.is_none() && !to.is_none()) << "copy of an empty NDArray";
  if (from.SameStorage(to)) return;  // ndarray.cc:1199-1203
  KV_CHECK_EQ(from.dtype(), to.dtype()) << "CopyFromTo: dtype mismatch";
  if (from.stype() != to.stype()) {
    CastStorageCopy(from, to);  // rowsparse.cc: dense <-> row_sparse (ndarray.cc:1147-1196)
    return;
  }
  if (from.stype() == kDefaultStorage) {
    KV_CHECK_EQ(from.Size(), to.Size()) << "CopyFromTo: operands shape mismatch";
    if (from.Size() == 0) return;
    RawCopy(to.data(), to.ctx(), to.var(), from.data(), from.ctx(), from.var(), from.ByteSize());
    return;
  }
  // row_sparse (CopyFromToRspImpl, ndarray.cc:1076-1093)
  KV_CHECK(from.shape() == to.shape()) << "CopyFromTo: row_sparse shape mismatch";
  if (!from.storage_initialized()) {
    Engine::Get()->WaitToWrite(*to.var());
    to.SetNnr(0);
    return;
  }
  const int64_t nnr = from.nnr();
  to.CheckAndAllocRows(nnr);
  RawCopy(to.data(), to.ctx(), to.var(), from.data(), from.ctx(), from.var(),
          static_cast<size_t>(nnr) * from.RowLength() * DTypeSize(from.dtype()));
  RawCopy(to.row_ids(), to.ctx(), to.var(), from.row_ids(), from.ctx(), from.var(),
          static_cast<size_t>(nnr) * sizeof(int64_t));
}

// ---------------------------------------------------------------------------------------------
// serialization
// ---------------------------------------------------------------------------------------------
namespace {
constexpr uint32_t kV1Magic = 0xF993fac8, kV2Magic = 0xF993fac9, kV3Magic = 0xF993faca;

template <typename T> void Put(std::string* o, T v) { o->append(reinterpret_cast<const char*>(&v), sizeof(T)); }
void PutShape(std::string* o, const std::vector<int64_t>& s) {   // Tuple::Save (tuple.h:704-713)
  Put<int32_t>(o, static_cast<int32_t>(s.size()));
  for (int64_t d : s) Put<int64_t>(o, d);
}
struct Reader {
  const char* p;
  size_t left;
  template <typename T> T Get() {
    KV_CHECK(left >= sizeof(T)) << "Invalid NDArray file format";
    T v;
    std::memcpy(&v, p, sizeof(T));
    p += sizeof(T);
    left -= sizeof(T);
    return v;
  }
  std::vector<int64_t> Shape() {
    const int32_t nd = Get<int32_t>();
    KV_CHECK(nd >= 0 && nd <= 32) << "Invalid NDArray file format";
    std::vector<int64_t> s(nd);
    for (auto& d : s) d = Get<int64_t>();
    return s;
  }
  const char* Take(size_t n) {
    KV_CHECK(left >= n) << "Invalid NDArray file format";
    const char* q = p;
    p += n;
    left -= n;
    return q;
  }
};

// device (or pinned host) bytes -> host string, through the copy lanes
void AppendBytes(std::string* o, const void* src, Context ctx, Var* var, size_t bytes) {
  if (bytes == 0) return;
  const size_t at = o->size();
  o->resize(at + bytes);
  Var dst;
  RawCopy(&(*o)[at], Context::CPU(), &dst, src, ctx, var, bytes);
  Engine::Get()->WaitToRead(dst);
}
}  // namespace

void NDArray::SaveRaw(std::string* o) const {
  Put<uint32_t>(o, kV2Magic);
  Put<int32_t>(o, is_none() ? 0 : stype_);
  const bool rsp = !is_none() && stype_ == kRowSparseStorage;
  if (rsp) {
    std::vector<int64_t> ss = shape();
    ss[0] = nnr();
    PutShape(o, ss);
  }
  PutShape(o, is_none() ? std::vector<int64_t>() : shape());
  if (is_none()) return;
  // context: host-side arrays are plain cpu(0) to the outside (their pinning is an implementation detail)
  Put<int32_t>(o, st_->ctx.is_gpu() ? kGPU : kCPU);
  Put<int32_t>(o, st_->ctx.is_gpu() ? st_->ctx.dev_id : 0);
  Put<int32_t>(o, dtype_);
  if (rsp) {
    Put<int32_t>(o, kInt64);
    PutShape(o, {nnr()});
  }
  const size_t data_bytes = rsp ? static_cast<size_t>(nnr()) * RowLength() * DTypeSize(dtype_) : ByteSize();
  if (data_bytes) AppendBytes(o, data(), st_->ctx, &st_->var, data_bytes);
  if (rsp && nnr() > 0) AppendBytes(o, row_ids(), st_->ctx, &st_->var, static_cast<size_t>(nnr()) * sizeof(int64_t));
}

NDArray NDArray::LoadRaw(const char* buf, size_t size, size_t* consumed) {
  Reader r{buf, size};
  const uint32_t magic = r.Get<uint32_t>();
  KV_CHECK(magic != kV3Magic) << "ndarray was saved in np shape semantics, which this path does not use";
  int32_t stype = kDefaultStorage;
  std::vector<int64_t> sshape, shape;
  if (magic == kV2Magic) {
    stype = r.Get<int32_t>();
    KV_CHECK(stype == kDefaultStorage || stype == kRowSparseStorage) << "unsupported storage type " << stype;
    if (stype == kRowSparseStorage) sshape = r.Shape();
    shape = r.Shape();
  } else if (magic == kV1Magic) {
    shape = r.Shape();
  } else {
    // legacy TShape: the word just read is ndim, dims follow as uint32 (ndarray.cc:1672-1687)
    KV_CHECK(magic <= 32) << "Invalid NDArray file format";
    shape.resize(magic);
    for (auto& d : shape) d = r.Get<uint32_t>();
  }
  NDArray out;
  if (shape.empty()) {
    if (consumed) *consumed = size - r.left;
    return out;
  }
  const int32_t dev_type = r.Get<int32_t>(), dev_id = r.Get<int32_t>();
  const int32_t dtype = r.Get<int32_t>();
  int64_t nnr = 0;
  if (stype == kRowSparseStorage) {
    const int32_t aux_type = r.Get<int32_t>();
    KV_CHECK_EQ(aux_type, kInt64) << "row_sparse index type";
    const std::vector<int64_t> as = r.Shape();
    KV_CHECK(as.size() == 1 && !sshape.empty() && sshape[0] == as[0]) << "Invalid NDArray file format";
    nnr = as[0];
  }
  Context ctx = Context::CPU();
  if (dev_type == kGPU && dev_id < Engine::Get()->NumDevices()) ctx = Context::GPU(dev_id);
  auto fill = [&](void* dst, Var* var, size_t bytes) {
    if (bytes == 0) return;
    const char* src = r.Take(bytes);
    RawCopy(dst, ctx, var, src, Context::CPU(), nullptr, bytes);
    Engine::Get()->WaitToRead(*var);  // `buf` belongs to the caller
  };
  if (stype == kDefaultStorage) {
    out = NDArray(shape, ctx, dtype);
    fill(out.data(), out.var(), out.ByteSize());
  } else {
    out = NDArray::RowSparse(shape, ctx, dtype);
    if (nnr > 0) {
      out.CheckAndAllocRows(nnr);
      fill(out.data(), out.var(), static_cast<size_t>(nnr) * out.RowLength() * DTypeSize(dtype));
      fill(out.row_ids(), out.var(), static_cast<size_t>(nnr) * sizeof(int64_t));
    }
  }
  if (consumed) *consumed = size - r.left;
  return out;
}

}  // namespace b200kv
