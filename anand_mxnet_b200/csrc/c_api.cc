// c_api.cc -- the extern "C" boundary of libb200kv.so (include/b200kv_c_api.h).
//
// Same conventions as the reference's src/c_api/c_api.cc: every entry point is wrapped in a
// try/catch that turns an exception into `return -1` plus a thread-local message for
// MXGetLastError() (include/mxnet/c_api_error.h:36-58); handles are heap objects owned by the
// caller (NDArrayHandle = NDArray*, KVStoreHandle = KVStore*).
#include "b200kv_c_api.h"

#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "engine.h"
#include "group.h"
#include <cstdio>
#include <cstring>

#include <condition_variable>
#include <memory>
#include <mutex>
#include <stdexcept>

#include "kvstore.h"
#include "nccl_dyn.h"
#include "ndarray.h"
#include "ops.h"
#include "random_ops.h"
#include "scalar_parse.h"

using namespace b200kv;  // NOLINT

namespace {

thread_local std::string g_last_error;
thread_local std::vector<int> g_shape_buf;
thread_local std::vector<NDArrayHandle> g_out_handles;
thread_local std::vector<int> g_out_stypes;
thread_local std::string g_plan_buf;

int HandleException(const std::exception& e) {
  g_last_error = e.what();
  return -1;
}

#define API_BEGIN()                                                      \
  try {                                                                  \
    std::lock_guard<std::recursive_mutex> lock_(Engine::Get()->mutex());
#define API_END()                                      \
  }                                                    \
  catch (const std::exception& e_) {                   \
    return HandleException(e_);                        \
  }                                                    \
  catch (...) {                                        \
    g_last_error = "unknown error";                    \
    return -1;                                         \
  }                                                    \
  return 0;

NDArray& ND(NDArrayHandle h) {
  KV_CHECK(h != nullptr) << "null NDArrayHandle";
  return *static_cast<NDArray*>(h);
}

KVStore& KV(KVStoreHandle h) {
  KV_CHECK(h != nullptr) << "null KVStoreHandle";
  return *static_cast<KVStore*>(h);
}

std::vector<NDArray> NDVec(NDArrayHandle* v, size_t n) {
  std::vector<NDArray> out(n);
  for (size_t i = 0; i < n; ++i) out[i] = ND(v[i]);
  return out;
}

std::vector<std::string> StrVec(const char** v, size_t n) {
  std::vector<std::string> out(n);
  for (size_t i = 0; i < n; ++i) out[i] = v[i];
  return out;
}

Context MakeCtx(int dev_type, int dev_id) {
  KV_CHECK(dev_type == kCPU || dev_type == kGPU || dev_type == kCPUPinned || dev_type == kCPUShared)
      << "invalid device type " << dev_type;
  return Context{dev_type, dev_type == kGPU ? dev_id : 0};
}

}  // namespace

extern "C" {

const char* MXGetLastError(void) { return g_last_error.c_str(); }

int MXGetVersion(int* out) {
  *out = 10600;
  return 0;
}

int MXGetGPUCount(int* out) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    n = 0;
  }
  *out = n;
  return 0;
}

int MXNotifyShutdown(void) {
  API_BEGIN();
  Engine::Get()->Shutdown();
  API_END();
}

int MXRandomSeed(int seed) {
  API_BEGIN();
  RandomSeed(static_cast<uint32_t>(seed));
  API_END();
}

int MXRandomSeedContext(int seed, int dev_type, int dev_id) {
  API_BEGIN();
  RandomSeedContext(static_cast<uint32_t>(seed), MakeCtx(dev_type, dev_id));
  API_END();
}

// ------------------------------------------------------------------------------------------ NDArray
int MXNDArrayCreateNone(NDArrayHandle* out) {
  API_BEGIN();
  *out = new NDArray();
  API_END();
}

int MXNDArrayCreateEx64(const int64_t* shape, int ndim, int dev_type, int dev_id, int delay_alloc,
                        int dtype, NDArrayHandle* out) {
  API_BEGIN();
  std::vector<int64_t> s(shape, shape + ndim);
  DTypeSize(dtype);  // validates
  *out = new NDArray(s, MakeCtx(dev_type, dev_id), dtype, delay_alloc != 0);
  API_END();
}

int MXNDArrayCreateEx(const uint32_t* shape, uint32_t ndim, int dev_type, int dev_id, int delay_alloc,
                      int dtype, NDArrayHandle* out) {
  std::vector<int64_t> s(shape, shape + ndim);
  return MXNDArrayCreateEx64(s.data(), static_cast<int>(ndim), dev_type, dev_id, delay_alloc, dtype, out);
}

int MXNDArrayCreate(const uint32_t* shape, uint32_t ndim, int dev_type, int dev_id, int delay_alloc,
                    NDArrayHandle* out) {
  return MXNDArrayCreateEx(shape, ndim, dev_type, dev_id, delay_alloc, kFloat32, out);
}

int MXNDArrayCreateSparseEx(int storage_type, const uint32_t* shape, uint32_t ndim, int dev_type,
                            int dev_id, int, int dtype, uint32_t num_aux, int* aux_type,
                            uint32_t*, const uint32_t*, NDArrayHandle* out) {
  API_BEGIN();
  KV_CHECK_EQ(storage_type, kRowSparseStorage)
      << "only row_sparse sparse arrays are on the KVStore path (csr is not)";
  if (num_aux > 0) KV_CHECK_EQ(aux_type[0], kInt64) << "row ids are int64";
  std::vector<int64_t> s(shape, shape + ndim);
  *out = new NDArray(NDArray::RowSparse(s, MakeCtx(dev_type, dev_id), dtype));
  API_END();
}

int MXNDArrayFree(NDArrayHandle handle) {
  API_BEGIN();
  delete static_cast<NDArray*>(handle);
  API_END();
}

int MXNDArraySyncCopyFromCPU(NDArrayHandle handle, const void* data, size_t size) {
  API_BEGIN();
  KVStore::FlushAll();  // queued (bucketed) KVStore calls run before anything observes arrays
  NDArray& a = ND(handle);
  KV_CHECK_EQ(a.stype(), kDefaultStorage) << "SyncCopyFromCPU on a sparse array: copy the data and "
                                          << "aux arrays (MXNDArrayGetDataNDArray / GetAuxNDArray)";
  KV_CHECK_EQ(a.Size(), size) << "Memory size do not match";  // ndarray.cc:1876-1878
  if (size == 0) return 0;
  RawCopy(a.data(), a.ctx(), a.var(), data, Context::CPU(), nullptr, a.ByteSize());
  if (a.on_gpu()) {
    // the caller may reuse `data` immediately: pageable sources are staged by the runtime before
    // cudaMemcpyAsync returns; pinned sources need the copy to have completed
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, data) != cudaSuccess) cudaGetLastError();
    else if (attr.type == cudaMemoryTypeHost) Engine::Get()->WaitToRead(*a.var());
  }
  API_END();
}

int MXNDArraySyncCopyToCPU(NDArrayHandle handle, void* data, size_t size) {
  API_BEGIN();
  KVStore::FlushAll();  // queued (bucketed) KVStore calls run before anything observes arrays
  NDArray& a = ND(handle);
  KV_CHECK_EQ(a.stype(), kDefaultStorage) << "SyncCopyToCPU on a sparse array";
  KV_CHECK_EQ(a.Size(), size) << "Memory size do not match";
  if (size == 0) return 0;
  Var dst;
  RawCopy(data, Context::CPU(), &dst, a.data(), a.ctx(), a.var(), a.ByteSize());
  Engine::Get()->WaitToRead(dst);
  API_END();
}

int MXNDArraySyncCopyFromNDArray(NDArrayHandle handle_dst, const NDArrayHandle handle_src, const int i) {
  API_BEGIN();
  KVStore::FlushAll();  // queued (bucketed) KVStore calls run before anything observes arrays
  NDArray& dst = ND(handle_dst);
  NDArray& src = ND(handle_src);
  KV_CHECK_EQ(src.stype(), kDefaultStorage) << "source must be a dense array";
  if (dst.stype() == kRowSparseStorage) {
    // ndarray.cc SyncCopyFromNDArray: i = -1 data blob, i >= 0 aux blob; allocates for src's rows
    if (i >= 0) {
      const int64_t nnr = static_cast<int64_t>(src.Size());
      if (dst.nnr() != nnr) dst.CheckAndAllocRows(nnr);
      KV_CHECK_EQ(src.dtype(), kInt64) << "row ids must be int64";
      RawCopy(dst.row_ids(), dst.ctx(), dst.var(), src.data(), src.ctx(), src.var(), nnr * sizeof(int64_t));
    } else {
      const int64_t nnr = src.shape().empty() ? 0 : src.shape()[0];
      if (dst.nnr() != nnr) dst.CheckAndAllocRows(nnr);
      KV_CHECK_EQ(src.dtype(), dst.dtype());
      RawCopy(dst.data(), dst.ctx(), dst.var(), src.data(), src.ctx(), src.var(), src.ByteSize());
    }
  } else {
    CopyFromTo(src, dst);
  }
  Engine::Get()->WaitToRead(*dst.var());
  API_END();
}

int MXNDArrayWaitToRead(NDArrayHandle handle) {
  API_BEGIN();
  KVStore::FlushAll();  // queued (bucketed) KVStore calls run before anything observes arrays
  NDArray& a = ND(handle);
  if (!a.is_none()) Engine::Get()->WaitToRead(*a.var());
  API_END();
}

int MXNDArrayWaitToWrite(NDArrayHandle handle) {
  API_BEGIN();
  KVStore::FlushAll();  // queued (bucketed) KVStore calls run before anything observes arrays
  NDArray& a = ND(handle);
  if (!a.is_none()) Engine::Get()->WaitToWrite(*a.var());
  API_END();
}

int MXNDArrayWaitAll(void) {
  API_BEGIN();
  KVStore::FlushAll();  // queued (bucketed) KVStore calls run before anything observes arrays
  Engine::Get()->WaitAll();
  API_END();
}

int MXNDArrayGetStorageType(NDArrayHandle handle, int* out) {
  API_BEGIN();
  NDArray& a = ND(handle);
  *out = a.is_none() ? kUndefinedStorage : a.stype();
  API_END();
}

int MXNDArrayGetShapeEx(NDArrayHandle handle, int* out_dim, const int** out_pdata) {
  API_BEGIN();
  NDArray& a = ND(handle);
  if (a.is_none()) {
    *out_dim = -1;  // unknown shape, like an NDArray created by MXNDArrayCreateNone
    *out_pdata = nullptr;
  } else {
    g_shape_buf.assign(a.shape().begin(), a.shape().end());
    *out_dim = static_cast<int>(g_shape_buf.size());
    *out_pdata = g_shape_buf.data();
  }
  API_END();
}

int MXNDArrayGetData(NDArrayHandle handle, void** out_pdata) {
  API_BEGIN();
  KVStore::FlushAll();  // the caller is about to look at the memory
  NDArray& a = ND(handle);
  a.Escape();
  *out_pdata = a.is_none() ? nullptr : a.data();
  API_END();
}

int MXNDArrayGetDType(NDArrayHandle handle, int* out_dtype) {
  API_BEGIN();
  NDArray& a = ND(handle);
  *out_dtype = a.is_none() ? -1 : a.dtype();
  API_END();
}

int MXNDArrayGetAuxType(NDArrayHandle handle, uint32_t, int* out_type) {
  API_BEGIN();
  KV_CHECK_EQ(ND(handle).stype(), kRowSparseStorage) << "dense arrays have no aux data";
  *out_type = kInt64;
  API_END();
}

int MXNDArrayGetAuxNDArray(NDArrayHandle handle, uint32_t i, NDArrayHandle* out) {
  API_BEGIN();
  KV_CHECK_EQ(i, 0u) << "row_sparse arrays have exactly one aux array";
  *out = new NDArray(ND(handle).AuxView());
  API_END();
}

int MXNDArrayGetDataNDArray(NDArrayHandle handle, NDArrayHandle* out) {
  API_BEGIN();
  *out = new NDArray(ND(handle).DataView());
  API_END();
}

// ---- serialization (python pickling of optimizer states, mx.nd.save / load)
thread_local std::string g_raw_bytes;
thread_local std::vector<std::string> g_name_store;
thread_local std::vector<const char*> g_name_ptrs;

int MXNDArraySaveRawBytes(NDArrayHandle handle, size_t* out_size, const char** out_buf) {
  API_BEGIN();
  KVStore::FlushAll();
  g_raw_bytes.clear();
  ND(handle).SaveRaw(&g_raw_bytes);
  *out_size = g_raw_bytes.size();
  *out_buf = g_raw_bytes.data();
  API_END();
}

int MXNDArrayLoadFromRawBytes(const void* buf, size_t size, NDArrayHandle* out) {
  API_BEGIN();
  *out = new NDArray(NDArray::LoadRaw(static_cast<const char*>(buf), size, nullptr));
  API_END();
}

// list file: uint64 0x112, uint64 0, vector<NDArray>, vector<string> (ndarray.cc:1829-1857; dmlc
// serializes a vector as uint64 count + elements, a string as uint64 length + bytes)
int MXNDArraySave(const char* fname, uint32_t num_args, NDArrayHandle* args, const char** keys) {
  API_BEGIN();
  KVStore::FlushAll();
  std::string o;
  auto put64 = [&](uint64_t v) { o.append(reinterpret_cast<const char*>(&v), 8); };
  put64(0x112);
  put64(0);
  put64(num_args);
  for (uint32_t i = 0; i < num_args; ++i) ND(args[i]).SaveRaw(&o);
  put64(keys != nullptr ? num_args : 0);
  if (keys != nullptr) {
    for (uint32_t i = 0; i < num_args; ++i) {
      put64(std::strlen(keys[i]));
      o.append(keys[i]);
    }
  }
  FILE* f = std::fopen(fname, "wb");
  KV_CHECK(f != nullptr) << "cannot open " << fname << " for writing";
  const size_t w = std::fwrite(o.data(), 1, o.size(), f);
  std::fclose(f);
  KV_CHECK_EQ(w, o.size()) << "short write to " << fname;
  API_END();
}

int MXNDArrayLoad(const char* fname, uint32_t* out_size, NDArrayHandle** out_arr, uint32_t* out_name_size,
                  const char*** out_names) {
  API_BEGIN();
  FILE* f = std::fopen(fname, "rb");
  KV_CHECK(f != nullptr) << "cannot open " << fname;
  std::string buf;
  char tmp[1 << 16];
  size_t n;
  while ((n = std::fread(tmp, 1, sizeof(tmp), f)) > 0) buf.append(tmp, n);
  std::fclose(f);
  size_t pos = 0;
  auto get64 = [&]() {
    KV_CHECK(pos + 8 <= buf.size()) << "Invalid NDArray file format";
    uint64_t v;
    std::memcpy(&v, buf.data() + pos, 8);
    pos += 8;
    return v;
  };
  KV_CHECK_EQ(get64(), 0x112u) << "Invalid NDArray file format";
  get64();
  const uint64_t cnt = get64();
  g_out_handles.clear();
  for (uint64_t i = 0; i < cnt; ++i) {
    size_t used = 0;
    g_out_handles.push_back(new NDArray(NDArray::LoadRaw(buf.data() + pos, buf.size() - pos, &used)));
    pos += used;
  }
  const uint64_t nn = get64();
  KV_CHECK(nn == 0 || nn == cnt) << "Invalid NDArray file format";
  g_name_store.clear();
  g_name_ptrs.clear();
  for (uint64_t i = 0; i < nn; ++i) {
    const uint64_t len = get64();
    KV_CHECK(pos + len <= buf.size()) << "Invalid NDArray file format";
    g_name_store.emplace_back(buf.data() + pos, len);
    pos += len;
  }
  for (auto& sname : g_name_store) g_name_ptrs.push_back(sname.c_str());
  *out_size = static_cast<uint32_t>(cnt);
  *out_arr = g_out_handles.data();
  *out_name_size = static_cast<uint32_t>(nn);
  *out_names = g_name_ptrs.data();
  API_END();
}

int MXNDArraySlice(NDArrayHandle handle, uint32_t slice_begin, uint32_t slice_end, NDArrayHandle* out) {
  API_BEGIN();
  *out = new NDArray(ND(handle).Slice(slice_begin, slice_end));
  API_END();
}

int MXNDArrayGetContext(NDArrayHandle handle, int* out_dev_type, int* out_dev_id) {
  API_BEGIN();
  NDArray& a = ND(handle);
  if (a.is_none()) {
    *out_dev_type = 0;
    *out_dev_id = 0;
  } else {
    *out_dev_type = a.ctx().dev_type;
    *out_dev_id = a.ctx().dev_id;
  }
  API_END();
}

int MXNDArrayToDLPack(NDArrayHandle handle, DLManagedTensorHandle* out_dlpack) {
  API_BEGIN();
  KVStore::FlushAll();  // queued (bucketed) KVStore calls run before anything observes arrays
  NDArray& a = ND(handle);
  KV_CHECK_EQ(a.stype(), kDefaultStorage) << "only dense arrays export to DLPack";
  a.Escape();
  struct Holder {
    NDArray arr;
    std::vector<int64_t> shape;
    DLManagedTensorABI t;
  };
  Holder* h = new Holder{a, a.shape(), {}};
  std::memset(&h->t, 0, sizeof(h->t));
  h->t.dl_tensor.data = a.data();
  h->t.dl_tensor.ctx.device_type = a.on_gpu() ? 2 : (a.ctx().dev_type == kCPUPinned ? 3 : 1);
  h->t.dl_tensor.ctx.device_id = a.ctx().dev_id;
  h->t.dl_tensor.ndim = static_cast<int>(h->shape.size());
  uint8_t code = 2, bits = 32;
  switch (a.dtype()) {
    case kFloat32: code = 2; bits = 32; break;
    case kFloat64: code = 2; bits = 64; break;
    case kFloat16: code = 2; bits = 16; break;
    case kBfloat16: code = 4; bits = 16; break;
    case kInt32: code = 0; bits = 32; break;
    case kInt64: code = 0; bits = 64; break;
    case kInt8: code = 0; bits = 8; break;
    case kUint8: code = 1; bits = 8; break;
    default: KV_FATAL << "dtype not exportable to DLPack";
  }
  h->t.dl_tensor.dtype = DLDataTypeABI{code, bits, 1};
  h->t.dl_tensor.shape = h->shape.data();
  h->t.dl_tensor.strides = nullptr;
  h->t.dl_tensor.byte_offset = 0;
  h->t.manager_ctx = h;
  h->t.deleter = [](DLManagedTensorABI* t) { delete static_cast<Holder*>(t->manager_ctx); };
  *out_dlpack = &h->t;
  API_END();
}

int MXNDArrayFromDLPackEx(DLManagedTensorHandle dlpack, const bool transient_handle,
                          NDArrayHandle* out_handle) {
  API_BEGIN();
  *out_handle = new NDArray(NDArray::FromDLPack(static_cast<DLManagedTensorABI*>(dlpack), transient_handle));
  API_END();
}

int MXNDArrayCallDLPackDeleter(DLManagedTensorHandle dlpack) {
  API_BEGIN();
  DLManagedTensorABI* t = static_cast<DLManagedTensorABI*>(dlpack);
  if (t != nullptr && t->deleter != nullptr) t->deleter(t);
  API_END();
}

// ------------------------------------------------------------------------------------------ ops
int NNGetOpHandle(const char* op_name, AtomicSymbolCreator* op_out) {
  API_BEGIN();
  const OpInfo* op = FindOp(op_name);
  KV_CHECK(op != nullptr) << "Cannot find argument '" << op_name
                          << "': operator not registered in libb200kv (KVStore hot-path subset)";
  *op_out = const_cast<OpInfo*>(op);
  API_END();
}

int MXImperativeInvokeEx(AtomicSymbolCreator creator, int num_inputs, NDArrayHandle* inputs,
                         int* num_outputs, NDArrayHandle** outputs, int num_params,
                         const char** param_keys, const char** param_vals, const int** out_stypes) {
  API_BEGIN();
  KVStore::FlushAll();  // queued (bucketed) KVStore calls run before anything observes arrays
  const OpInfo* op = static_cast<const OpInfo*>(creator);
  KV_CHECK(op != nullptr) << "null operator handle";
  std::vector<NDArray> in = NDVec(inputs, num_inputs);
  std::vector<NDArray> out;
  const bool given = *outputs != nullptr && *num_outputs > 0;
  if (given) out = NDVec(*outputs, *num_outputs);
  std::vector<std::pair<std::string, std::string>> params(num_params);
  for (int i = 0; i < num_params; ++i) params[i] = {param_keys[i], param_vals[i]};
  InvokeOp(op, in, &out, params);
  if (!given) {
    g_out_handles.clear();
    for (auto& o : out) g_out_handles.push_back(new NDArray(o));
    *num_outputs = static_cast<int>(g_out_handles.size());
    *outputs = g_out_handles.data();
  }
  if (out_stypes != nullptr) {
    g_out_stypes.clear();
    for (auto& o : out) g_out_stypes.push_back(o.stype());
    *out_stypes = g_out_stypes.data();
  }
  API_END();
}

// ------------------------------------------------------------------------------------------ KVStore
int MXInitPSEnv(mx_uint, const char**, const char**) { return 0; }

// ------------------------------------------------------------------------------------------ engine ABI
// MXEnginePushAsyncND / MXEnginePushSyncND (include/mxnet/c_api.h:3323-3351, src/c_api/c_api.cc:
// 2396-2513): how an external scheduler (a Horovod-style plugin) joins the dependency graph. On
// the lane engine an external operation is ordered like the library's own: its reads wait for the
// arrays' writers, its writes for writers and readers; on a GPU context those waits are stream
// waits on the device's compute lane and the function receives that lane's stream in rctx->stream
// (work it enqueues there is ordered by the stream; on_complete may be called at once). On a CPU
// context the dependencies are awaited on the host before the function runs. The push returns once
// the function has signalled completion; a failure it reports (or throws) is parked on the arrays
// it was to write and surfaces at the next wait on them (threaded_engine.h:380-387).
namespace {
struct RunCtxABI {       // layout of mxnet::RunContext (include/mxnet/base.h:350-365)
  int32_t dev_type, dev_id;
  void* stream;          // the compute lane's cudaStream_t on a GPU context, else NULL
  void* aux_stream;
  bool is_bulk;
};
struct PendingExt {
  std::mutex m;
  std::condition_variable cv;
  bool done = false, failed = false;
  std::string msg;
};
struct OnCompleteABI {   // layout of mxnet::engine::CallbackOnComplete (include/mxnet/engine.h:73-90)
  void (*callback)(void* engine, void* param, const void* error);
  void* engine;
  void* param;
};
void ExtOnComplete(void*, void* param, const void* error) {
  PendingExt* p = static_cast<PendingExt*>(param);
  std::lock_guard<std::mutex> lk(p->m);
  if (error != nullptr) {  // const dmlc::Error* : a std::runtime_error
    p->failed = true;
    p->msg = static_cast<const std::exception*>(error)->what();
  }
  p->done = true;
  p->cv.notify_all();
}

int PushExternal(void (*async_fn)(void*, void*, void*), void (*sync_fn)(void*, void*), void* func_param,
                 EngineFuncParamDeleter deleter, ContextHandle ctx_handle, NDArrayHandle* const_nds,
                 int num_const, NDArrayHandle* mutable_nds, int num_mutable, const char* opr_name) {
  std::shared_ptr<void> keep(func_param, deleter ? deleter : [](void*) {});
  KVStore::FlushAll();
  KV_CHECK(ctx_handle != nullptr) << "MXEnginePush*: null context";
  const int32_t* c = static_cast<const int32_t*>(ctx_handle);
  const Context ctx = MakeCtx(c[0], c[1]);
  Engine* eng = Engine::Get();
  std::vector<Var*> rd, wr;
  for (int i = 0; i < num_const; ++i) if (!ND(const_nds[i]).is_none()) rd.push_back(ND(const_nds[i]).var());
  for (int i = 0; i < num_mutable; ++i) if (!ND(mutable_nds[i]).is_none()) wr.push_back(ND(mutable_nds[i]).var());
  // an operation that touches an array carrying a parked failure is not run; the failure moves to
  // everything it was to write (ThreadedEngine::OnStart: exceptions of const AND mutable vars
  // propagate, src/engine/threaded_engine.h:380-387)
  for (const std::vector<Var*>* set : {&rd, &wr}) {
    for (Var* v : *set) {
      if (v->err && !v->err->empty()) {
        const std::string msg = *v->err;
        for (Var* w : wr) if (w != v) eng->SetError(w, msg);
        return 0;
      }
    }
  }
  const bool gpu = ctx.dev_type == kGPU;
  RunCtxABI rctx{ctx.dev_type, ctx.dev_id, nullptr, nullptr, false};
  std::unique_ptr<LaneOp> op;
  if (gpu) {
    op.reset(new LaneOp(ctx.dev_id));
    for (Var* v : rd) op->Read(v);
    for (Var* v : wr) op->Write(v);
    rctx.stream = op->stream();
  } else {
    for (Var* v : rd) eng->WaitToRead(*v);
    for (Var* v : wr) eng->WaitToWrite(*v);
  }
  PendingExt pend;
  OnCompleteABI oc{ExtOnComplete, eng, &pend};
  try {
    if (async_fn != nullptr) {
      async_fn(&rctx, &oc, func_param);
      std::unique_lock<std::mutex> lk(pend.m);
      pend.cv.wait(lk, [&] { return pend.done; });
    } else {
      sync_fn(&rctx, func_param);
    }
  } catch (const std::exception& e) {
    pend.failed = true;
    pend.msg = e.what();
  }
  if (op) op->Issue();
  if (pend.failed) {
    const std::string msg = std::string("operator ") + (opr_name ? opr_name : "<external>") + ": " + pend.msg;
    for (Var* w : wr) eng->SetError(w, msg);
  }
  return 0;
}
}  // namespace

int MXEnginePushAsyncND(EngineAsyncFunc async_func, void* func_param, EngineFuncParamDeleter deleter,
                        ContextHandle ctx_handle, NDArrayHandle* const_nds_handle, int num_const_nds,
                        NDArrayHandle* mutable_nds_handle, int num_mutable_nds,
                        EngineFnPropertyHandle, int, const char* opr_name, bool) {
  API_BEGIN();
  KV_CHECK(async_func != nullptr);
  PushExternal(async_func, nullptr, func_param, deleter, ctx_handle, const_nds_handle, num_const_nds,
               mutable_nds_handle, num_mutable_nds, opr_name);
  API_END();
}

int MXEnginePushSyncND(EngineSyncFunc sync_func, void* func_param, EngineFuncParamDeleter deleter,
                       ContextHandle ctx_handle, NDArrayHandle* const_nds_handle, int num_const_nds,
                       NDArrayHandle* mutable_nds_handle, int num_mutable_nds, EngineFnPropertyHandle, int,
                       const char* opr_name) {
  API_BEGIN();
  KV_CHECK(sync_func != nullptr);
  PushExternal(nullptr, sync_func, func_param, deleter, ctx_handle, const_nds_handle, num_const_nds,
               mutable_nds_handle, num_mutable_nds, opr_name);
  API_END();
}

int B200KVEngineOnComplete(void* on_complete, const char* error) {
  API_BEGIN();
  KV_CHECK(on_complete != nullptr);
  const OnCompleteABI* oc = static_cast<const OnCompleteABI*>(on_complete);
  if (error != nullptr) {
    const std::runtime_error e(error);
    oc->callback(oc->engine, oc->param, &e);
  } else {
    oc->callback(oc->engine, oc->param, nullptr);
  }
  API_END();
}

int MXKVStoreCreate(const char* type, KVStoreHandle* out) {
  API_BEGIN();
  *out = new KVStore(type);
  API_END();
}

int MXKVStoreFree(KVStoreHandle handle) {
  API_BEGIN();
  delete static_cast<KVStore*>(handle);
  API_END();
}

int MXKVStoreSetGradientCompression(KVStoreHandle handle, mx_uint num_params, const char** keys,
                                    const char** vals) {
  API_BEGIN();
  std::vector<std::pair<std::string, std::string>> kw(num_params);
  for (mx_uint i = 0; i < num_params; ++i) kw[i] = {keys[i], vals[i]};
  KV(handle).SetGradientCompression(kw);
  API_END();
}

int MXKVStoreInit(KVStoreHandle handle, mx_uint num, const int* keys, NDArrayHandle* vals) {
  API_BEGIN();
  KV(handle).Init(std::vector<int>(keys, keys + num), NDVec(vals, num));
  API_END();
}

int MXKVStoreInitEx(KVStoreHandle handle, mx_uint num, const char** keys, NDArrayHandle* vals) {
  API_BEGIN();
  KV(handle).InitStr(StrVec(keys, num), NDVec(vals, num));
  API_END();
}

int MXKVStorePush(KVStoreHandle handle, mx_uint num, const int* keys, NDArrayHandle* vals, int priority) {
  API_BEGIN();
  KVStore& kv = KV(handle);
  kv.SetKeyTypeInt();
  kv.Push(std::vector<int>(keys, keys + num), NDVec(vals, num), priority);
  API_END();
}

int MXKVStorePushEx(KVStoreHandle handle, mx_uint num, const char** keys, NDArrayHandle* vals, int priority) {
  API_BEGIN();
  KVStore& kv = KV(handle);
  kv.SetKeyTypeStr();
  kv.Push(kv.LookupKeys(StrVec(keys, num)), NDVec(vals, num), priority);
  API_END();
}

int MXKVStorePullWithSparse(KVStoreHandle handle, mx_uint num, const int* keys, NDArrayHandle* vals,
                            int priority, bool ignore_sparse) {
  API_BEGIN();
  KVStore& kv = KV(handle);
  kv.SetKeyTypeInt();
  kv.Pull(std::vector<int>(keys, keys + num), NDVec(vals, num), priority, ignore_sparse);
  API_END();
}

int MXKVStorePullWithSparseEx(KVStoreHandle handle, mx_uint num, const char** keys,
                              NDArrayHandle* vals, int priority, bool ignore_sparse) {
  API_BEGIN();
  KVStore& kv = KV(handle);
  kv.SetKeyTypeStr();
  kv.Pull(kv.LookupKeys(StrVec(keys, num)), NDVec(vals, num), priority, ignore_sparse);
  API_END();
}

int MXKVStorePull(KVStoreHandle handle, mx_uint num, const int* keys, NDArrayHandle* vals, int priority) {
  return MXKVStorePullWithSparse(handle, num, keys, vals, priority, true);
}

int MXKVStorePullEx(KVStoreHandle handle, mx_uint num, const char** keys, NDArrayHandle* vals, int priority) {
  return MXKVStorePullWithSparseEx(handle, num, keys, vals, priority, true);
}

int MXKVStorePullRowSparse(KVStoreHandle handle, mx_uint num, const int* keys, NDArrayHandle* vals,
                           const NDArrayHandle* row_ids, int priority) {
  API_BEGIN();
  KVStore& kv = KV(handle);
  kv.SetKeyTypeInt();
  kv.PullRowSparse(std::vector<int>(keys, keys + num), NDVec(vals, num),
                   NDVec(const_cast<NDArrayHandle*>(row_ids), num), priority);
  API_END();
}

int MXKVStorePullRowSparseEx(KVStoreHandle handle, mx_uint num, const char** keys,
                             NDArrayHandle* vals, const NDArrayHandle* row_ids, int priority) {
  API_BEGIN();
  KVStore& kv = KV(handle);
  kv.SetKeyTypeStr();
  kv.PullRowSparse(kv.LookupKeys(StrVec(keys, num)), NDVec(vals, num),
                   NDVec(const_cast<NDArrayHandle*>(row_ids), num), priority);
  API_END();
}

int MXKVStorePushPull(KVStoreHandle handle, mx_uint vnum, const int* vkeys, mx_uint onum,
                      const int* okeys, NDArrayHandle* vals, NDArrayHandle* outs, int priority) {
  API_BEGIN();
  KVStore& kv = KV(handle);
  kv.SetKeyTypeInt();
  kv.PushPull(std::vector<int>(vkeys, vkeys + vnum), std::vector<int>(okeys, okeys + onum),
              NDVec(vals, vnum), NDVec(outs, onum), priority);
  API_END();
}

int MXKVStorePushPullEx(KVStoreHandle handle, mx_uint vnum, const char** vkeys, mx_uint onum,
                        const char** okeys, NDArrayHandle* vals, NDArrayHandle* outs, int priority) {
  API_BEGIN();
  KVStore& kv = KV(handle);
  kv.SetKeyTypeStr();
  kv.PushPull(kv.LookupKeys(StrVec(vkeys, vnum)), kv.LookupKeys(StrVec(okeys, onum)),
              NDVec(vals, vnum), NDVec(outs, onum), priority);
  API_END();
}

int MXKVStoreSetUpdater(KVStoreHandle handle, MXKVStoreUpdater updater, void* updater_handle) {
  API_BEGIN();
  KV(handle).SetUpdater(updater, nullptr, updater_handle);
  API_END();
}

int MXKVStoreSetUpdaterEx(KVStoreHandle handle, MXKVStoreUpdater updater,
                          MXKVStoreStrUpdater str_updater, void* updater_handle) {
  API_BEGIN();
  KV(handle).SetUpdater(updater, str_updater, updater_handle);
  API_END();
}

int MXKVStoreGetType(KVStoreHandle handle, const char** type) {
  API_BEGIN();
  *type = KV(handle).type().c_str();
  API_END();
}

int MXKVStoreGetRank(KVStoreHandle handle, int* ret) {
  API_BEGIN();
  *ret = KV(handle).rank();
  API_END();
}

int MXKVStoreGetGroupSize(KVStoreHandle handle, int* ret) {
  API_BEGIN();
  *ret = KV(handle).group_size();
  API_END();
}

// single-node stores: every process is a worker (kvstore.h:343-372 defaults)
int MXKVStoreIsWorkerNode(int* ret) { *ret = 1; return 0; }
int MXKVStoreIsServerNode(int* ret) { *ret = 0; return 0; }
int MXKVStoreIsSchedulerNode(int* ret) { *ret = 0; return 0; }

int MXKVStoreBarrier(KVStoreHandle handle) {
  API_BEGIN();
  KV(handle).Flush();
  API_END();
}

int MXKVStoreSetBarrierBeforeExit(KVStoreHandle, const int) { return 0; }

int MXKVStoreRunServer(KVStoreHandle, MXKVStoreServerController, void*) {
  g_last_error = "MXKVStoreRunServer: parameter-server roles exist only in dist_* stores";
  return -1;
}

int MXKVStoreSendCommmandToServers(KVStoreHandle, int, const char*) { return 0; }

int MXKVStoreGetNumDeadNode(KVStoreHandle, const int, int* number, const int) {
  *number = 0;
  return 0;
}

// ------------------------------------------------------------------------------------------ extensions
int B200KVStoreSetOptimizer(KVStoreHandle handle, const char* name, mx_uint num_params,
                            const char** keys, const char** vals) {
  API_BEGIN();
  std::vector<std::pair<std::string, std::string>> kw(num_params);
  for (mx_uint i = 0; i < num_params; ++i) kw[i] = {keys[i], vals[i]};
  KV(handle).SetOptimizer(name, kw);
  API_END();
}

int B200KVStoreSetLearningRate(KVStoreHandle handle, double lr) {
  API_BEGIN();
  if (KV(handle).opt_view().lr != lr) {   // re-sent every step by front-ends: only a change matters
    KV(handle).opt().lr = lr;
    KV(handle).TouchOpt();
  }
  API_END();
}

int B200KVStoreSetRescaleGrad(KVStoreHandle handle, double rescale_grad) {
  API_BEGIN();
  if (KV(handle).opt_view().rescale != rescale_grad) {
    KV(handle).opt().rescale = rescale_grad;
    KV(handle).TouchOpt();
  }
  API_END();
}

int B200KVStoreSetKeyMultipliers(KVStoreHandle handle, mx_uint num, const int* keys,
                                 const double* lr_mult, const double* wd_mult) {
  API_BEGIN();
  const OptConfig& cur = KV(handle).opt_view();
  bool changed = false;
  for (mx_uint i = 0; i < num && !changed; ++i) {
    auto differs = [&](const std::unordered_map<int, double>& m, const double* v) {
      if (v == nullptr) return false;
      auto it = m.find(keys[i]);
      return (it == m.end() ? 1.0 : it->second) != v[i];   // an absent multiplier is 1
    };
    changed = differs(cur.lr_mult, lr_mult) || differs(cur.wd_mult, wd_mult);
  }
  if (changed) {
    OptConfig& o = KV(handle).opt();
    for (mx_uint i = 0; i < num; ++i) {
      if (lr_mult) o.lr_mult[keys[i]] = lr_mult[i];
      if (wd_mult) o.wd_mult[keys[i]] = wd_mult[i];
    }
    KV(handle).TouchOpt();
  }
  API_END();
}

int B200KVStoreLookupKey(KVStoreHandle handle, const char* str_key, int* out_key) {
  API_BEGIN();
  *out_key = KV(handle).LookupKeys({std::string(str_key)})[0];
  API_END();
}

int B200KVStoreGetOptimizerState(KVStoreHandle handle, int key, int state_id, NDArrayHandle* out) {
  API_BEGIN();
  KVStore::FlushAll();  // queued (bucketed) KVStore calls run before anything observes arrays
  *out = new NDArray(KV(handle).GetOptimizerState(key, state_id));
  API_END();
}

int B200KVStoreSetOptimizerState(KVStoreHandle handle, int key, int state_id, NDArrayHandle value) {
  API_BEGIN();
  KV(handle).SetOptimizerState(key, state_id, ND(value));
  API_END();
}

int B200KVStoreGetUpdateCount(KVStoreHandle handle, int key, int* out) {
  API_BEGIN();
  *out = KV(handle).UpdateCount(key);
  API_END();
}

int B200KVStoreGetNumUpdate(KVStoreHandle handle, int* out) {
  API_BEGIN();
  *out = KV(handle).NumUpdate();
  API_END();
}

int B200KVStoreSetUpdateCount(KVStoreHandle handle, int key, int count) {
  API_BEGIN();
  OptConfig& o = KV(handle).opt();
  o.count[key] = count;
  o.num_update = std::max(o.num_update, count);
  KV(handle).TouchOpt();
  API_END();
}

int B200KVStoreSetBucketBytes(KVStoreHandle handle, size_t max_bytes) {
  API_BEGIN();
  KV(handle).SetBucketBytes(max_bytes);
  API_END();
}

int B200KVStoreFlush(KVStoreHandle handle) {
  API_BEGIN();
  KV(handle).Flush();
  API_END();
}

int B200KVFlushAll(void) {
  API_BEGIN();
  KVStore::FlushAll();
  API_END();
}

// One call PER KEY, issued from compiled code the way the reference's C++ callers do
// (cpp-package KVStore::Push/Pull loops; gluon Trainer._allreduce_grads is the python analogue):
// pattern 0 = pushpull(key i, priority -i) for every i; pattern 1 = push(key i, priority i) for
// every i, then pull(key i, priority i) for every i (tools/bandwidth/measure.py:112-122).
int B200KVIssuePerKey(KVStoreHandle handle, mx_uint num, const int* keys, NDArrayHandle* vals,
                      NDArrayHandle* outs, int pattern) {
  for (mx_uint i = 0; i < num; ++i) {
    const int pr = pattern == 0 ? -static_cast<int>(i) : static_cast<int>(i);
    const int rc = pattern == 0
        ? MXKVStorePushPull(handle, 1, keys + i, 1, keys + i, vals + i, outs + i, pr)
        : MXKVStorePush(handle, 1, keys + i, vals + i, pr);
    if (rc != 0) return rc;
  }
  if (pattern != 0) {
    for (mx_uint i = 0; i < num; ++i) {
      const int rc = MXKVStorePullWithSparse(handle, 1, keys + i, outs + i, static_cast<int>(i), true);
      if (rc != 0) return rc;
    }
  }
  return 0;
}

int B200KVEngineSetStream(int dev_id, void* cuda_stream) {
  API_BEGIN();
  KVStore::FlushAll();  // queued (bucketed) KVStore calls run before anything observes arrays
  Engine::Get()->SetStream(dev_id, static_cast<cudaStream_t>(cuda_stream));
  API_END();
}

int B200KVEngineGetStream(int dev_id, void** cuda_stream) {
  API_BEGIN();
  *cuda_stream = Engine::Get()->Stream(dev_id);
  API_END();
}

int B200KVGroupInit(int rank, int world_size, int dev_id, B200KVAllGatherFn allgather, void* ctx) {
  API_BEGIN();
  PeerGroup::Init(rank, world_size, dev_id, allgather, ctx);
  API_END();
}

int B200KVGroupInitExternal(int rank, int world_size, int dev_id, B200KVAllGatherFn allgather,
                            void* ctx, void* arena, size_t arena_bytes, void* const* peer_arenas,
                            void* multicast_arena) {
  API_BEGIN();
  KV_CHECK(arena != nullptr && peer_arenas != nullptr && arena_bytes > 0);
  PeerGroup::Init(rank, world_size, dev_id, allgather, ctx, arena, arena_bytes, peer_arenas,
                  multicast_arena);
  API_END();
}

int B200KVGroupDestroy(void) {
  API_BEGIN();
  PeerGroup::Destroy();
  API_END();
}

// test hook: copy n (src -> dst) array pairs with ONE TMA bulk-copy launch (pack_kernels.cu);
// pairs the pack path cannot take (different GPUs, foreign host memory) use CopyFromTo
B200KV_DLL int B200KVTestPackCopy(int n, NDArrayHandle* srcs, NDArrayHandle* dsts, int* n_packed) {
  API_BEGIN();
  std::vector<std::pair<NDArray, NDArray>> pairs;
  for (int i = 0; i < n; ++i) {
    KV_CHECK_EQ(ND(srcs[i]).ByteSize(), ND(dsts[i]).ByteSize());
    pairs.emplace_back(ND(srcs[i]), ND(dsts[i]));
  }
  std::shared_ptr<PackList> pl = BuildPackList(&pairs);
  *n_packed = pl ? static_cast<int>(pl->pairs.size()) : 0;
  if (pl) RunPackList(*pl);
  for (auto& pr : pairs) CopyFromTo(pr.first, pr.second);
  Engine::Get()->WaitAll();
  API_END();
}

// host-only hook: the rank-major int64 exchange plan building uses (runs under gloo on CPU)
B200KV_DLL int B200KVTestGatherI64(int world, B200KVAllGatherFn allgather, void* ctx,
                                   const int64_t* mine, int n, int64_t* out) {
  try {
    std::vector<int64_t> m(mine, mine + n);
    std::vector<int64_t> all = GatherI64(allgather, ctx, world, m);
    std::memcpy(out, all.data(), all.size() * sizeof(int64_t));
  } catch (const std::exception& e) {
    return HandleException(e);
  }
  return 0;
}

// host-only hook: the shared-memory mailbox between the ranks of a node (group.cc), no GPU needed
B200KV_DLL int B200KVTestMailbox(int rank, int world, B200KVAllGatherFn allgather, void* ctx,
                                 const int64_t* mine, int n, int rounds, int64_t* out, int* used_mailbox) {
  try {
    PeerGroup::TestMailbox(rank, world, allgather, ctx, mine, n, rounds, out, used_mailbox);
  } catch (const std::exception& e) {
    return HandleException(e);
  }
  return 0;
}

// host-only hook: can the NCCL fallback bind its library? (dlopen + dlsym only, no GPU, no communicator)
B200KV_DLL int B200KVTestNcclAvailable(int* available, char* version, size_t version_len) {
  try {
    *available = Nccl::Available() ? 1 : 0;
    if (*available && version != nullptr && version_len > 0) {
      std::snprintf(version, version_len, "%s", Nccl::Get()->version());
    }
  } catch (const std::exception& e) {
    return HandleException(e);
  }
  return 0;
}

int B200KVRandomStates(int dev_id, int copy, void* out, size_t bytes) {
  API_BEGIN();
  RandomStates(dev_id, copy, out, bytes);
  API_END();
}

int B200KVRandomNormalInto(NDArrayHandle out, float loc, float scale, int staged) {
  API_BEGIN();
  KVStore::FlushAll();
  RandNormalInto(ND(out), loc, scale, staged != 0);
  API_END();
}

int B200KVGetKernelLaunchCount(uint64_t* out) {
  *out = Engine::Get()->launch_count;
  return 0;
}

int B200KVResetKernelLaunchCount(void) {
  Engine::Get()->launch_count = 0;
  return 0;
}

int B200KVGetLastKernelInfo(const char** name, uint64_t* algorithmic_bytes) {
  *name = Engine::Get()->last_kernel;
  *algorithmic_bytes = Engine::Get()->last_kernel_bytes;
  return 0;
}

int B200KVStoreDescribePlan(KVStoreHandle handle, mx_uint num, const int* keys, int num_devices,
                            char* buf, size_t buf_len) {
  API_BEGIN();
  g_plan_buf = KV(handle).DescribePlan(std::vector<int>(keys, keys + num), num_devices);
  KV_CHECK(buf_len > g_plan_buf.size()) << "buffer too small";
  std::memcpy(buf, g_plan_buf.c_str(), g_plan_buf.size() + 1);
  API_END();
}

const char* B200KVBuildInfo(void) {
  return "libb200kv: sm_90a, -fmad=false, static cudart, chunk=4096 stripe=32768";
}

// test hooks for the scalar plumbing (pure host code, no GPU needed)
B200KV_DLL int B200KVTestPyFloatRepr(double v, char* buf, size_t buf_len) {
  std::string s = PyFloatRepr(v);
  if (buf_len <= s.size()) return -1;
  std::memcpy(buf, s.c_str(), s.size() + 1);
  return 0;
}

B200KV_DLL int B200KVTestDmlcStof(const char* s, float* out) {
  try {
    *out = DmlcStof(s);
  } catch (const std::exception& e) {
    return HandleException(e);
  }
  return 0;
}

// host-only planner hook: chunk/ownership layout of keys of the given sizes over n devices
B200KV_DLL int B200KVTestPlanChunks(const uint64_t* sizes, int nkeys, int ndev, uint64_t* out_counts,
                                    uint64_t* out_elems);

}  // extern "C"

namespace b200kv {
void PlanChunks(uint64_t goff, size_t size, uint32_t key_slot, int ndev, int owner_fixed,
                std::vector<std::vector<ChunkDesc>>* per_slot);
}

extern "C" int B200KVTestPlanChunks(const uint64_t* sizes, int nkeys, int ndev, uint64_t* out_counts,
                                    uint64_t* out_elems) {
  try {
    std::vector<std::vector<ChunkDesc>> chunks(ndev);
    uint64_t goff = 0;
    for (int k = 0; k < nkeys; ++k) {
      b200kv::PlanChunks(goff, sizes[k], static_cast<uint32_t>(k), ndev, ndev > 1 ? -1 : 0, &chunks);
      goff += (std::max<uint64_t>(sizes[k], 1) + kKeyAlignElems - 1) / kKeyAlignElems * kKeyAlignElems;
    }
    for (int d = 0; d < ndev; ++d) {
      out_counts[d] = chunks[d].size();
      out_elems[d] = 0;
      for (auto& c : chunks[d]) {
        out_elems[d] += c.len;
        if (c.len == 0 || c.len > static_cast<uint32_t>(kChunkElems)) return -1;
      }
    }
  } catch (const std::exception& e) {
    return HandleException(e);
  }
  return 0;
}

// host-only hook: the order in which the (key, position) pairs of one call are grouped
// (kvstore_core.cc SortKeyPairs): positions[] after the sort, for the call order (stable) or the
// reference's std::sort order (B200KV_GROUP_ORDER=reference)
namespace b200kv {
void SortKeyPairs(std::vector<std::pair<int, int>>* idx, bool reference_order);
}

extern "C" B200KV_DLL int B200KVTestGroupOrder(const int* keys, int n, int reference_order, int* positions) {
  try {
    std::vector<std::pair<int, int>> idx(static_cast<size_t>(n));
    for (int i = 0; i < n; ++i) idx[i] = {keys[i], i};
    b200kv::SortKeyPairs(&idx, reference_order != 0);
    for (int i = 0; i < n; ++i) positions[i] = idx[i].second;
  } catch (const std::exception& e) {
    return HandleException(e);
  }
  return 0;
}
