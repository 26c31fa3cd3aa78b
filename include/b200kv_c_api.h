/*
 * b200kv_c_api.h -- the C ABI of libb200kv.so, the H100-native drop-in for the KVStore hot path
 * of Apache MXNet 1.6 (reference: anandj91/anand-mxnet).
 *
 * Part A re-declares, with IDENTICAL names, argument lists and return conventions, the subset of
 * the reference's C API (include/mxnet/c_api.h) that its KVStore front-ends bind
 * (python/mxnet/kvstore/kvstore.py -> _LIB.MXKVStore*, and the same calls from the scala / R /
 * julia / perl / cpp-package bindings), plus the minimum of MXNDArray* / MXImperativeInvokeEx that
 * a caller needs to create the values it pushes and to run the reference's optimizer operators.
 * Each declaration cites the reference declaration it replaces.
 *
 * Part B holds the extensions (prefix B200KV) that have no counterpart in the reference: the
 * natively fused optimizer, external-stream interop, multi-process (one rank per GPU) peer groups
 * and introspection used by tests / bench.
 *
 * Conventions (reference: include/mxnet/c_api_error.h:36-58, src/c_api/c_api_error.cc):
 *   - every function returns 0 on success and -1 on failure; the message of the last failure on the
 *     calling thread is returned by MXGetLastError();
 *   - handles are opaque pointers; input NDArrayHandles are borrowed for the duration of the call;
 *   - push / pull / pushpull RETURN AFTER ENQUEUEING work on the owning device's stream; results
 *     are observable after MXNDArrayWaitToRead / MXNDArrayWaitAll / MXNDArraySyncCopyToCPU
 *     (reference contract: include/mxnet/kvstore.h:129-141,168-180).
 *
 * No torch / C++ types appear in any signature.
 */
#ifndef B200KV_C_API_H_
#define B200KV_C_API_H_

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200KV_DLL __attribute__((visibility("default")))

typedef uint32_t mx_uint;                 /* c_api.h:58 */
typedef void* NDArrayHandle;              /* c_api.h:67 */
typedef void* KVStoreHandle;              /* c_api.h:83 */
typedef void* AtomicSymbolCreator;        /* c_api.h:71 */
typedef void* DLManagedTensorHandle;      /* c_api.h:93 */

/* dev_type: 1 = CPU, 2 = GPU, 3 = CPUPinned (include/mxnet/base.h:104-109)
 * dtype:    0 f32, 1 f64, 2 f16, 3 u8, 4 i32, 5 i8, 6 i64 (3rdparty/mshadow/mshadow/base.h:307-314)
 *           12 = bf16 (extension; mshadow 1.6 has no bf16; value follows later MXNet kBfloat16)
 * storage_type: 0 default (dense), 1 row_sparse (include/mxnet/ndarray.h:61-66) */

/* ============================== Part A: reference C API subset ============================== */

/* c_api.h:228 */
B200KV_DLL const char* MXGetLastError(void);
/* c_api.h:519 -- returns 10600 (the reference's MXNET_VERSION, 1.6.0) */
B200KV_DLL int MXGetVersion(int* out);
/* c_api.h:493 */
B200KV_DLL int MXGetGPUCount(int* out);
/* c_api.h:270 */
B200KV_DLL int MXNotifyShutdown(void);

/* ---- NDArray: creation / inspection / host copies (c_api.h:567-1127) ---- */
B200KV_DLL int MXNDArrayCreateNone(NDArrayHandle* out);                               /* :567 */
B200KV_DLL int MXNDArrayCreate(const uint32_t* shape, uint32_t ndim, int dev_type, int dev_id,
                               int delay_alloc, NDArrayHandle* out);                  /* :579 */
B200KV_DLL int MXNDArrayCreateEx(const uint32_t* shape, uint32_t ndim, int dev_type, int dev_id,
                                 int delay_alloc, int dtype, NDArrayHandle* out);     /* :600 */
B200KV_DLL int MXNDArrayCreateEx64(const int64_t* shape, int ndim, int dev_type, int dev_id,
                                   int delay_alloc, int dtype, NDArrayHandle* out);   /* :622 */
B200KV_DLL int MXNDArrayCreateSparseEx(int storage_type, const uint32_t* shape, uint32_t ndim,
                                       int dev_type, int dev_id, int delay_alloc, int dtype,
                                       uint32_t num_aux, int* aux_type, uint32_t* aux_ndims,
                                       const uint32_t* aux_shape, NDArrayHandle* out); /* :649 */
B200KV_DLL int MXNDArrayFree(NDArrayHandle handle);                                   /* :837 */
/* `size` is an ELEMENT count checked against shape.Size() (src/ndarray/ndarray.cc:1874-1882) */
B200KV_DLL int MXNDArraySyncCopyFromCPU(NDArrayHandle handle, const void* data, size_t size); /* :773 */
B200KV_DLL int MXNDArraySyncCopyToCPU(NDArrayHandle handle, void* data, size_t size);         /* :787 */
/* i = -1 copies the data blob, i >= 0 the i-th aux blob (row ids) */
B200KV_DLL int MXNDArraySyncCopyFromNDArray(NDArrayHandle handle_dst, const NDArrayHandle handle_src,
                                            const int i);                             /* :798 */
B200KV_DLL int MXNDArrayWaitToRead(NDArrayHandle handle);                             /* :815 */
B200KV_DLL int MXNDArrayWaitToWrite(NDArrayHandle handle);                            /* :823 */
B200KV_DLL int MXNDArrayWaitAll(void);                                                /* :830 */
B200KV_DLL int MXNDArrayGetStorageType(NDArrayHandle handle, int* out_storage_type);  /* :898 */
B200KV_DLL int MXNDArrayGetShapeEx(NDArrayHandle handle, int* out_dim, const int** out_pdata); /* :948 */
B200KV_DLL int MXNDArrayGetData(NDArrayHandle handle, void** out_pdata);              /* :971 */
B200KV_DLL int MXNDArrayGetDType(NDArrayHandle handle, int* out_dtype);               /* :1034 */
B200KV_DLL int MXNDArrayGetAuxType(NDArrayHandle handle, uint32_t i, int* out_type);  /* :1046 */
B200KV_DLL int MXNDArrayGetAuxNDArray(NDArrayHandle handle, uint32_t i, NDArrayHandle* out); /* :1070 */
B200KV_DLL int MXNDArrayGetDataNDArray(NDArrayHandle handle, NDArrayHandle* out);     /* :1090 */
B200KV_DLL int MXNDArrayGetContext(NDArrayHandle handle, int* out_dev_type, int* out_dev_id); /* :1099 */
/* NDArray::Save binary format (src/ndarray/ndarray.cc:1596-1857): what python pickles of NDArrays --
 * hence Updater.get_states() optimizer checkpoints -- and mx.nd.save files contain */
B200KV_DLL int MXNDArrayLoadFromRawBytes(const void* buf, size_t size, NDArrayHandle* out);   /* :701 */
B200KV_DLL int MXNDArraySaveRawBytes(NDArrayHandle handle, size_t* out_size, const char** out_buf); /* :711 */
B200KV_DLL int MXNDArraySave(const char* fname, uint32_t num_args, NDArrayHandle* args,
                             const char** keys);                                               /* :722 */
B200KV_DLL int MXNDArrayLoad(const char* fname, uint32_t* out_size, NDArrayHandle** out_arr,
                             uint32_t* out_name_size, const char*** out_names);                /* :735 */
/* view of rows [slice_begin, slice_end) of the first axis, sharing memory (LARS slices its lr array) */
B200KV_DLL int MXNDArraySlice(NDArrayHandle handle, uint32_t slice_begin, uint32_t slice_end,
                              NDArrayHandle* out);                                      /* :849 */
/* zero-copy views of memory owned by another framework (torch) -- c_api.h:982-1026 */
B200KV_DLL int MXNDArrayToDLPack(NDArrayHandle handle, DLManagedTensorHandle* out_dlpack);     /* :982 */
B200KV_DLL int MXNDArrayFromDLPackEx(DLManagedTensorHandle dlpack, const bool transient_handle,
                                     NDArrayHandle* out_handle);                      /* :1017 */
B200KV_DLL int MXNDArrayCallDLPackDeleter(DLManagedTensorHandle dlpack);              /* :1026 */

/* ---- imperative operators the optimizer front-end calls (c_api.h:1251; nnvm/c_api.h NNGetOpHandle)
 * Registered ops: sgd_update, sgd_mom_update, mp_sgd_update, mp_sgd_mom_update, multi_sgd_update,
 * multi_sgd_mom_update, multi_mp_sgd_update, multi_mp_sgd_mom_update, adam_update
 * (src/operator/optimizer_op.cc:322-710) and the elementwise helpers updaters use
 * (_copyto, _plus, _minus, _mul, _plus_scalar, _mul_scalar, _set_value, _full, cast), the multi-tensor
 * operators (multi_sum_sq, multi_lars, preloaded_multi_*, AdamW, LAMB), the AMP overflow check
 * all_finite / multi_all_finite (src/operator/contrib/all_finite.cc), zero_grad's reset_arrays
 * (src/operator/contrib/reset_arrays.cc; inputs zeroed in place, no output) and zeros_like /
 * _sparse_zeros_like on row_sparse arrays, the single-tensor
 * operators of the other optimizers (ops.cc lists them all), and two extensions the reference
 * composes from NDArray arithmetic: _b200kv_clip_global_norm (inputs array_0 .. array_{n-1}, float32,
 * scaled in place; parameters num_arrays, max_norm; output total_norm, a (1,) float32 array) and
 * _b200kv_multi_scale (same inputs; parameters num_arrays, scalar; no output). Any other name fails
 * with "operator not registered". */
B200KV_DLL int NNGetOpHandle(const char* op_name, AtomicSymbolCreator* op_out);
B200KV_DLL int MXImperativeInvokeEx(AtomicSymbolCreator creator, int num_inputs,
                                    NDArrayHandle* inputs, int* num_outputs,
                                    NDArrayHandle** outputs, int num_params,
                                    const char** param_keys, const char** param_vals,
                                    const int** out_stypes);                          /* :1251 */

/* ---- KVStore (c_api.h:2645-3040; impl src/c_api/c_api.cc:1750-2131) ---- */
B200KV_DLL int MXInitPSEnv(mx_uint num_vars, const char** keys, const char** vals);   /* :2645 */
B200KV_DLL int MXKVStoreCreate(const char* type, KVStoreHandle* out);                 /* :2656 */
B200KV_DLL int MXKVStoreSetGradientCompression(KVStoreHandle handle, mx_uint num_params,
                                               const char** keys, const char** vals); /* :2667 */
B200KV_DLL int MXKVStoreFree(KVStoreHandle handle);                                   /* :2677 */
B200KV_DLL int MXKVStoreInit(KVStoreHandle handle, mx_uint num, const int* keys,
                             NDArrayHandle* vals);                                    /* :2686 */
B200KV_DLL int MXKVStoreInitEx(KVStoreHandle handle, mx_uint num, const char** keys,
                               NDArrayHandle* vals);                                  /* :2699 */
B200KV_DLL int MXKVStorePush(KVStoreHandle handle, mx_uint num, const int* keys,
                             NDArrayHandle* vals, int priority);                      /* :2713 */
B200KV_DLL int MXKVStorePushEx(KVStoreHandle handle, mx_uint num, const char** keys,
                               NDArrayHandle* vals, int priority);                    /* :2727 */
B200KV_DLL int MXKVStorePullWithSparse(KVStoreHandle handle, mx_uint num, const int* keys,
                                       NDArrayHandle* vals, int priority, bool ignore_sparse); /* :2745 */
B200KV_DLL int MXKVStorePullWithSparseEx(KVStoreHandle handle, mx_uint num, const char** keys,
                                         NDArrayHandle* vals, int priority, bool ignore_sparse); /* :2764 */
B200KV_DLL int MXKVStorePull(KVStoreHandle handle, mx_uint num, const int* keys,
                             NDArrayHandle* vals, int priority);                      /* :2779 */
B200KV_DLL int MXKVStorePullEx(KVStoreHandle handle, mx_uint num, const char** keys,
                               NDArrayHandle* vals, int priority);                    /* :2793 */
B200KV_DLL int MXKVStorePullRowSparse(KVStoreHandle handle, mx_uint num, const int* keys,
                                      NDArrayHandle* vals, const NDArrayHandle* row_ids,
                                      int priority);                                  /* :2811 */
B200KV_DLL int MXKVStorePullRowSparseEx(KVStoreHandle handle, mx_uint num, const char** keys,
                                        NDArrayHandle* vals, const NDArrayHandle* row_ids,
                                        int priority);                                /* :2829 */
B200KV_DLL int MXKVStorePushPull(KVStoreHandle handle, mx_uint vnum, const int* vkeys, mx_uint onum,
                                 const int* okeys, NDArrayHandle* vals, NDArrayHandle* outs,
                                 int priority);                                       /* :2847 */
B200KV_DLL int MXKVStorePushPullEx(KVStoreHandle handle, mx_uint vnum, const char** vkeys,
                                   mx_uint onum, const char** okeys, NDArrayHandle* vals,
                                   NDArrayHandle* outs, int priority);                /* :2867 */
/* The updater receives two freshly created handles and MUST free both (c_api.h:2871-2882). */
typedef void(MXKVStoreUpdater)(int key, NDArrayHandle recv, NDArrayHandle local, void* handle);
typedef void(MXKVStoreStrUpdater)(const char* key, NDArrayHandle recv, NDArrayHandle local,
                                  void* handle);
B200KV_DLL int MXKVStoreSetUpdater(KVStoreHandle handle, MXKVStoreUpdater updater,
                                   void* updater_handle);                             /* :2907 */
B200KV_DLL int MXKVStoreSetUpdaterEx(KVStoreHandle handle, MXKVStoreUpdater updater,
                                     MXKVStoreStrUpdater str_updater, void* updater_handle); /* :2918 */
B200KV_DLL int MXKVStoreGetType(KVStoreHandle handle, const char** type);             /* :2928 */
B200KV_DLL int MXKVStoreGetRank(KVStoreHandle handle, int* ret);                      /* :2940 */
B200KV_DLL int MXKVStoreGetGroupSize(KVStoreHandle handle, int* ret);                 /* :2951 */
B200KV_DLL int MXKVStoreIsWorkerNode(int* ret);                                       /* :2958 */
B200KV_DLL int MXKVStoreIsServerNode(int* ret);                                       /* :2966 */
B200KV_DLL int MXKVStoreIsSchedulerNode(int* ret);                                    /* :2973 */
B200KV_DLL int MXKVStoreBarrier(KVStoreHandle handle);                                /* :2980 */
B200KV_DLL int MXKVStoreSetBarrierBeforeExit(KVStoreHandle handle, const int barrier_before_exit); /* :2989 */
typedef void(MXKVStoreServerController)(int head, const char* body, void* controller_handle);
B200KV_DLL int MXKVStoreRunServer(KVStoreHandle handle, MXKVStoreServerController controller,
                                  void* controller_handle);                           /* :3010 */
B200KV_DLL int MXKVStoreSendCommmandToServers(KVStoreHandle handle, int cmd_id,
                                              const char* cmd_body);                  /* :3021 */
B200KV_DLL int MXKVStoreGetNumDeadNode(KVStoreHandle handle, const int node_id, int* number,
                                       const int timeout_sec);                        /* :3035 */

/* ---- engine ABI for external schedulers (include/mxnet/c_api.h:99-110, 3323-3351) -------------
 * An external operation joins the dependency graph by naming the arrays it reads (const) and the
 * arrays it writes (mutable). rctx points at {int32 dev_type; int32 dev_id; void* stream;
 * void* aux_stream; bool is_bulk} (mxnet::RunContext's layout; `stream` is the compute lane's
 * cudaStream_t on a GPU context -- the reference hands out an mshadow::Stream<gpu>* there);
 * on_complete points at {void (*callback)(void* engine, void* param, const void* error);
 * void* engine; void* param} (mxnet::engine::CallbackOnComplete's layout; `error` is a
 * const dmlc::Error* = std::runtime_error* or NULL). A C host completes with
 * B200KVEngineOnComplete. A reported failure is parked on the mutable arrays and surfaces as -1 /
 * MXGetLastError at the next MXNDArrayWaitToRead / WaitToWrite of one of them, or at
 * MXNDArrayWaitAll (src/engine/threaded_engine.h:380-387). */
typedef const void* ContextHandle;          /* -> {int32 dev_type; int32 dev_id} (mxnet::Context) */
typedef const void* EngineFnPropertyHandle;
typedef void (*EngineAsyncFunc)(void* rctx, void* on_complete, void* param);   /* c_api.h:105 */
typedef void (*EngineSyncFunc)(void* rctx, void* param);                       /* c_api.h:107 */
typedef void (*EngineFuncParamDeleter)(void* param);                           /* c_api.h:109 */
B200KV_DLL int MXEnginePushAsyncND(EngineAsyncFunc async_func, void* func_param,
                                   EngineFuncParamDeleter deleter, ContextHandle ctx_handle,
                                   NDArrayHandle* const_nds_handle, int num_const_nds,
                                   NDArrayHandle* mutable_nds_handle, int num_mutable_nds,
                                   EngineFnPropertyHandle prop_handle, int priority,
                                   const char* opr_name, bool wait);            /* c_api.h:3323 */
B200KV_DLL int MXEnginePushSyncND(EngineSyncFunc sync_func, void* func_param,
                                  EngineFuncParamDeleter deleter, ContextHandle ctx_handle,
                                  NDArrayHandle* const_nds_handle, int num_const_nds,
                                  NDArrayHandle* mutable_nds_handle, int num_mutable_nds,
                                  EngineFnPropertyHandle prop_handle, int priority,
                                  const char* opr_name);                        /* c_api.h:3345 */
/* completion entry for hosts that cannot call a C++ CallbackOnComplete: error == NULL = success */
B200KV_DLL int B200KVEngineOnComplete(void* on_complete, const char* error);

/* ============================== Part B: B200KV extensions =================================== */

/* Natively fused optimizer: replaces the per-key Python updater callback (kvstore.py:34-41 ->
 * optimizer.py:2079-2128) for the optimizers whose kernels are on the hot path. `name` is one of
 * "sgd", "adam", "test"; keys/vals are the reference's op-parameter strings (momentum, lr, wd,
 * rescale_grad, clip_gradient, beta1, beta2, epsilon, multi_precision, begin_num_update,
 * lazy_update). After this call push() = reduce + scale/clip + update in ONE kernel launch and
 * pushpull() additionally broadcasts the new weights to every `out`. */
B200KV_DLL int B200KVStoreSetOptimizer(KVStoreHandle handle, const char* name, mx_uint num_params,
                                       const char** keys, const char** vals);
/* per-step scalars (python double, as Optimizer.lr / rescale_grad are; nearest-float32 is taken at
 * the point the reference would format them into op parameters) */
B200KV_DLL int B200KVStoreSetLearningRate(KVStoreHandle handle, double lr);
B200KV_DLL int B200KVStoreSetRescaleGrad(KVStoreHandle handle, double rescale_grad);
/* per-key multipliers: Optimizer._get_lrs / _get_wds (optimizer.py:432-509). Keys are the int keys
 * (or the ints string keys were mapped to -- use B200KVStoreLookupKey). */
B200KV_DLL int B200KVStoreSetKeyMultipliers(KVStoreHandle handle, mx_uint num, const int* keys,
                                            const double* lr_mult, const double* wd_mult);
B200KV_DLL int B200KVStoreLookupKey(KVStoreHandle handle, const char* str_key, int* out_key);
/* optimizer-state checkpoint hooks (reference: Updater.get_states/set_states,
 * optimizer.py:2143-2161): state_id 0 = momentum / Adam mean, 1 = Adam var, 2 = fp32 master
 * weights; *out is a new NDArrayHandle (device copy gathered from the shards) the caller frees. */
B200KV_DLL int B200KVStoreGetOptimizerState(KVStoreHandle handle, int key, int state_id,
                                            NDArrayHandle* out);
B200KV_DLL int B200KVStoreSetOptimizerState(KVStoreHandle handle, int key, int state_id,
                                            NDArrayHandle value);
B200KV_DLL int B200KVStoreGetUpdateCount(KVStoreHandle handle, int key, int* out);
B200KV_DLL int B200KVStoreSetUpdateCount(KVStoreHandle handle, int key, int count);
/* Optimizer.num_update: the largest per-key update count so far (optimizer.py:412-430) */
B200KV_DLL int B200KVStoreGetNumUpdate(KVStoreHandle handle, int* out);

/* Deferred bucket execution: push/pull/pushpull calls are queued and fused into one launch per
 * device when the queued bytes reach the bucket size, when any array is waited on / read / exported,
 * when the store's configuration changes, or on B200KVStoreFlush. Default policy ("auto"): calls
 * that name ONE key are queued (bucket 256 MB, B200KV_AUTO_BUCKET_MB), calls carrying a key list run
 * at once as one fused launch. max_bytes > 0 queues every call up to max_bytes; 0 switches queuing
 * off. Env B200KV_BUCKET_MB=n sets the same at store creation. Results are identical either way:
 * queued calls of one key keep their order, higher priority keys are issued first. */
B200KV_DLL int B200KVStoreSetBucketBytes(KVStoreHandle handle, size_t max_bytes);
B200KV_DLL int B200KVStoreFlush(KVStoreHandle handle);
B200KV_DLL int B200KVFlushAll(void);   /* every store of the process; does not wait for the device */
/* Issues one call PER KEY from compiled code, as the reference's callers do: pattern 0 =
 * pushpull(key i, priority -i) (python/mxnet/gluon/trainer.py:385-396), pattern 1 = push of every
 * key then pull of every key with priority i (tools/bandwidth/measure.py:112-122). */
B200KV_DLL int B200KVIssuePerKey(KVStoreHandle handle, mx_uint num, const int* keys,
                                 NDArrayHandle* vals, NDArrayHandle* outs, int pattern);

/* Stream interop: make the engine issue all work for GPU `dev_id` on a caller-owned cudaStream_t
 * (e.g. torch.cuda.current_stream().cuda_stream) so KVStore work is ordered with the framework
 * that produced the gradients; stream == NULL restores the library's own stream. */
B200KV_DLL int B200KVEngineSetStream(int dev_id, void* cuda_stream);
B200KV_DLL int B200KVEngineGetStream(int dev_id, void** cuda_stream);

/* Multi-process peer group (one rank per GPU, NVLink peer memory through CUDA IPC). The library
 * never opens sockets: the host supplies an all-gather over its own process group
 * (torch.distributed) as a C callback: it must gather `nbytes` from every rank into
 * recv[rank*nbytes ...] and return 0. */
typedef int (*B200KVAllGatherFn)(const void* send, void* recv, size_t nbytes, void* ctx);
B200KV_DLL int B200KVGroupInit(int rank, int world_size, int dev_id, B200KVAllGatherFn allgather,
                               void* ctx);
/* Same, with an arena the launcher has already allocated and peer-mapped (e.g. torch symmetric
 * memory): peer_arenas[r] = rank r's arena as addressable from this rank (entry `rank` = arena);
 * multicast_arena = NVSwitch multicast mapping of all ranks' arenas or NULL. With a multicast
 * mapping and B200KV_NVLS=1 the fused kernel sums gradients in the switch (multimem.ld_reduce) and
 * multicasts the weights (multimem.st). */
B200KV_DLL int B200KVGroupInitExternal(int rank, int world_size, int dev_id,
                                       B200KVAllGatherFn allgather, void* ctx, void* arena,
                                       size_t arena_bytes, void* const* peer_arenas,
                                       void* multicast_arena);
B200KV_DLL int B200KVGroupDestroy(void);

/* Introspection for tests / bench / profiling. */
B200KV_DLL int B200KVGetKernelLaunchCount(uint64_t* out);    /* kernels launched by this library */
B200KV_DLL int B200KVResetKernelLaunchCount(void);
B200KV_DLL int B200KVGetLastKernelInfo(const char** name, uint64_t* algorithmic_bytes);
B200KV_DLL int B200KVStoreDescribePlan(KVStoreHandle handle, mx_uint num, const int* keys,
                                       int num_devices, char* buf, size_t buf_len);
B200KV_DLL const char* B200KVBuildInfo(void);

#ifdef __cplusplus
}
#endif

/* the random number generators (seeding, and the sampler's introspection) */
#include "b200kv_random_api.h"

#endif /* B200KV_C_API_H_ */
