/*
 * mxkv_b200.h -- C ABI of the H100-native KVStore engine.
 *
 * Drop-in boundary: every MX* symbol below has the signature, argument meaning and
 * error behaviour (0 = ok, -1 = error, message via MXGetLastError(), never throws) of
 * the function of the same name in the reference's include/mxnet/c_api.h, so a language
 * binding that today resolves these symbols in libmxnet.so can resolve them here
 * (INTEGRATION.md shows the ctypes side).  The reference line each one replaces is
 * cited next to it.  MXKVB200* symbols are extensions that have no reference
 * counterpart (fused optimizer registration, stream hand-off, one-process-per-GPU
 * bootstrap, symmetric allocation).
 *
 * Plain C: opaque handles, pointers and sizes only.
 *
 * Threading: every entry point may be called from any thread, like the reference's.  KVStore calls
 * are serialised per process first (the per-GPU streams, descriptor rings and staging slots are shared by all
 * stores) and per store second; they only ENQUEUE work and return -- results are ordered per array on the
 * engine's streams, and MXNDArrayWaitToRead / WaitAll (or the caller's own stream, see MXKVB200SetStream)
 * observe them.  The updater callback runs on the calling thread, inside the call.  The error string of
 * MXGetLastError is per thread.
 */
#ifndef MXKV_B200_H_
#define MXKV_B200_H_

#include <stddef.h>
#include <stdint.h>
#ifndef __cplusplus
#include <stdbool.h>
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define MXKV_DLL __attribute__((visibility("default")))

typedef void* NDArrayHandle;           /* c_api.h:67  */
typedef void* KVStoreHandle;           /* c_api.h:93  */
typedef void* DLManagedTensorHandle;   /* c_api.h:105 */
typedef uint32_t mx_uint;

/* ---- errors / library info ---------------------------------------------- */
MXKV_DLL const char* MXGetLastError(void);                           /* c_api.h:233 */
MXKV_DLL int MXGetGPUCount(int* out);                                /* c_api.h:502 */
MXKV_DLL int MXGetVersion(int* out);                                 /* c_api.h:528 */

/* ---- NDArray (the subset the KVStore path needs) ------------------------ */
/* dev_type: 1 cpu, 2 gpu, 3 cpu_pinned (include/mxnet/base.h:94-99); dtype: mshadow type flag
 * (3rdparty/mshadow/mshadow/base.h:352-366): 0 f32, 1 f64, 2 f16, 3 u8, 4 i32, 5 i8, 6 i64, 12 bf16 */
MXKV_DLL int MXNDArrayCreateNone(NDArrayHandle* out);                /* c_api.h:576 */
MXKV_DLL int MXNDArrayCreate(const uint32_t* shape, uint32_t ndim, int dev_type, int dev_id,
                             int delay_alloc, int dtype, NDArrayHandle* out);            /* c_api.h:592 */
MXKV_DLL int MXNDArrayCreate64(const int64_t* shape, int ndim, int dev_type, int dev_id,
                               int delay_alloc, int dtype, NDArrayHandle* out);          /* c_api.h:615 */
/* storage_type 1 = row_sparse (include/mxnet/ndarray.h:61-66); aux_shape[0] = row capacity */
MXKV_DLL int MXNDArrayCreateSparseEx64(int storage_type, const int64_t* shape, int ndim, int dev_type,
                                       int dev_id, int delay_alloc, int dtype, uint32_t num_aux,
                                       int* aux_type, int* aux_ndims, const int64_t* aux_shape,
                                       NDArrayHandle* out);                              /* c_api.h:674 */
MXKV_DLL int MXNDArrayFree(NDArrayHandle handle);                                        /* c_api.h:842 */
MXKV_DLL int MXNDArraySyncCopyFromCPU(NDArrayHandle handle, const void* data, size_t size); /* c_api.h:778 */
MXKV_DLL int MXNDArraySyncCopyToCPU(NDArrayHandle handle, void* data, size_t size);       /* c_api.h:792 */
/* i = -1: data, i >= 0: aux array i of a sparse source (c_api.h:803) */
MXKV_DLL int MXNDArraySyncCopyFromNDArray(NDArrayHandle handle_dst, const NDArrayHandle handle_src,
                                          const int i);
MXKV_DLL int MXNDArrayWaitToRead(NDArrayHandle handle);                                  /* c_api.h:820 */
MXKV_DLL int MXNDArrayWaitToWrite(NDArrayHandle handle);                                 /* c_api.h:828 */
MXKV_DLL int MXNDArrayWaitAll(void);                                                     /* c_api.h:835 */
MXKV_DLL int MXNDArrayGetStorageType(NDArrayHandle handle, int* out_storage_type);       /* c_api.h:903 */
MXKV_DLL int MXNDArrayGetShape(NDArrayHandle handle, int* out_dim, const int** out_pdata);       /* c_api.h:942 */
MXKV_DLL int MXNDArrayGetShape64(NDArrayHandle handle, int* out_dim, const int64_t** out_pdata); /* c_api.h:955 */
MXKV_DLL int MXNDArrayGetData(NDArrayHandle handle, void** out_pdata);                   /* c_api.h:965 */
MXKV_DLL int MXNDArrayToDLPack(NDArrayHandle handle, DLManagedTensorHandle* out_dlpack); /* c_api.h:976 */
MXKV_DLL int MXNDArrayFromDLPack(DLManagedTensorHandle dlpack, const bool transient_handle,
                                 NDArrayHandle* out_handle);                             /* c_api.h:993 */
MXKV_DLL int MXNDArrayCallDLPackDeleter(DLManagedTensorHandle dlpack);                   /* c_api.h:1002 */
MXKV_DLL int MXNDArrayGetDType(NDArrayHandle handle, int* out_dtype);                    /* c_api.h:1010 */
MXKV_DLL int MXNDArrayGetAuxType(NDArrayHandle handle, uint32_t i, int* out_type);       /* c_api.h:1022 */
MXKV_DLL int MXNDArrayGetAuxNDArray(NDArrayHandle handle, uint32_t i, NDArrayHandle* out); /* c_api.h:1046 */
MXKV_DLL int MXNDArrayGetDataNDArray(NDArrayHandle handle, NDArrayHandle* out);          /* c_api.h:1066 */
MXKV_DLL int MXNDArrayGetContext(NDArrayHandle handle, int* out_dev_type, int* out_dev_id); /* c_api.h:1075 */
MXKV_DLL int MXNDArrayReshape64(NDArrayHandle handle, int ndim, int64_t* dims, bool reverse,
                                NDArrayHandle* out);                                     /* c_api.h:927 */

/* ---- KVStore (c_api.h Part 6, :2391-2825; impl src/c_api/c_api.cc:2771-3204) --- */
MXKV_DLL int MXKVStoreCreate(const char* type, KVStoreHandle* out);                      /* c_api.h:2402 */
MXKV_DLL int MXKVStoreSetGradientCompression(KVStoreHandle handle, uint32_t num_params,
                                             const char** keys, const char** vals);      /* c_api.h:2412 */
MXKV_DLL int MXKVStoreFree(KVStoreHandle handle);                                        /* c_api.h:2422 */
MXKV_DLL int MXKVStoreInit(KVStoreHandle handle, uint32_t num, const int* keys, NDArrayHandle* vals);      /* :2431 */
MXKV_DLL int MXKVStoreInitEx(KVStoreHandle handle, uint32_t num, const char** keys, NDArrayHandle* vals);  /* :2444 */
MXKV_DLL int MXKVStorePush(KVStoreHandle handle, uint32_t num, const int* keys, NDArrayHandle* vals,
                           int priority);                                                /* c_api.h:2458 */
MXKV_DLL int MXKVStorePushEx(KVStoreHandle handle, uint32_t num, const char** keys, NDArrayHandle* vals,
                             int priority);                                              /* c_api.h:2472 */
MXKV_DLL int MXKVStorePullWithSparse(KVStoreHandle handle, uint32_t num, const int* keys,
                                     NDArrayHandle* vals, int priority, bool ignore_sparse);   /* :2487 */
MXKV_DLL int MXKVStorePullWithSparseEx(KVStoreHandle handle, uint32_t num, const char** keys,
                                       NDArrayHandle* vals, int priority, bool ignore_sparse); /* :2503 */
MXKV_DLL int MXKVStorePull(KVStoreHandle handle, uint32_t num, const int* keys, NDArrayHandle* vals,
                           int priority);                                                /* c_api.h:2518 */
MXKV_DLL int MXKVStorePullEx(KVStoreHandle handle, uint32_t num, const char** keys, NDArrayHandle* vals,
                             int priority);                                              /* c_api.h:2532 */
MXKV_DLL int MXKVStorePullRowSparse(KVStoreHandle handle, uint32_t num, const int* keys,
                                    NDArrayHandle* vals, const NDArrayHandle* row_ids, int priority);   /* :2550 */
MXKV_DLL int MXKVStorePullRowSparseEx(KVStoreHandle handle, uint32_t num, const char** keys,
                                      NDArrayHandle* vals, const NDArrayHandle* row_ids, int priority); /* :2568 */
MXKV_DLL int MXKVStoreBroadcast(KVStoreHandle handle, mx_uint vnum, const int* vkeys, mx_uint onum,
                                const int* okeys, NDArrayHandle* vals, NDArrayHandle* outs,
                                int priority);                                           /* c_api.h:2587 */
MXKV_DLL int MXKVStoreBroadcastEx(KVStoreHandle handle, mx_uint vnum, const char** vkeys, mx_uint onum,
                                  const char** okeys, NDArrayHandle* vals, NDArrayHandle* outs,
                                  int priority);                                         /* c_api.h:2608 */
MXKV_DLL int MXKVStorePushPull(KVStoreHandle handle, mx_uint vnum, const int* vkeys, mx_uint onum,
                               const int* okeys, NDArrayHandle* vals, NDArrayHandle* outs,
                               int priority);                                            /* c_api.h:2629 */
MXKV_DLL int MXKVStorePushPullEx(KVStoreHandle handle, mx_uint vnum, const char** vkeys, mx_uint onum,
                                 const char** okeys, NDArrayHandle* vals, NDArrayHandle* outs,
                                 int priority);                                          /* c_api.h:2650 */
/* updater callbacks: the callee must free both NDArray handles (c_api.h:2661) */
typedef void(MXKVStoreUpdater)(int key, NDArrayHandle recv, NDArrayHandle local, void* handle);
typedef void(MXKVStoreStrUpdater)(const char* key, NDArrayHandle recv, NDArrayHandle local, void* handle);
MXKV_DLL int MXKVStoreSetUpdater(KVStoreHandle handle, MXKVStoreUpdater updater, void* updater_handle);  /* :2690 */
MXKV_DLL int MXKVStoreSetUpdaterEx(KVStoreHandle handle, MXKVStoreUpdater updater,
                                   MXKVStoreStrUpdater str_updater, void* updater_handle);               /* :2701 */
MXKV_DLL int MXKVStoreGetType(KVStoreHandle handle, const char** type);                  /* c_api.h:2711 */
MXKV_DLL int MXKVStoreGetRank(KVStoreHandle handle, int* ret);                           /* c_api.h:2724 */
MXKV_DLL int MXKVStoreGetGroupSize(KVStoreHandle handle, int* ret);                      /* c_api.h:2736 */
MXKV_DLL int MXKVStoreIsWorkerNode(int* ret);                                            /* c_api.h:2744 */
MXKV_DLL int MXKVStoreIsServerNode(int* ret);                                            /* c_api.h:2752 */
MXKV_DLL int MXKVStoreIsSchedulerNode(int* ret);                                         /* c_api.h:2760 */
MXKV_DLL int MXKVStoreBarrier(KVStoreHandle handle);                                     /* c_api.h:2768 */
MXKV_DLL int MXKVStoreSetBarrierBeforeExit(KVStoreHandle handle, const int barrier_before_exit); /* :2777 */
MXKV_DLL int MXKVStoreGetNumDeadNode(KVStoreHandle handle, const int node_id, int* number,
                                     const int timeout_sec);                             /* c_api.h:2822 */
/* Server-side entry points: single-node stores take them as no-ops, exactly like KVStore::RunServer /
 * SendCommandToServers of the local store (include/mxnet/kvstore.h:432,466). */
typedef void (MXKVStoreServerController)(int head, const char* body, void* controller_handle); /* c_api.h:2786 */
MXKV_DLL int MXKVStoreRunServer(KVStoreHandle handle, MXKVStoreServerController controller,
                                void* controller_handle);                                /* c_api.h:2797 */
MXKV_DLL int MXKVStoreSendCommmandToServers(KVStoreHandle handle, int cmd_id, const char* cmd_body); /* :2808 */

/* ---- MXKVB200 extensions -------------------------------------------------- */
/* Fused optimizer: what Python's Updater + sgd_update/adam_update ops do per key in the
 * reference (python/mxnet/optimizer/updater.py:39-93) happens inside the reduce kernel.
 * name: "sgd" | "adam" | "adamw" | "test" | "lamb" | "lans" | "lars"; kwargs use the reference's
 * hyper-parameter names (learning_rate, wd, momentum, rescale_grad, clip_gradient, beta1, beta2,
 * epsilon, eta, multi_precision, lazy_update, correct_bias, lower_bound, upper_bound,
 * bias_correction).  lamb / lans / lars additionally take skip_nonfinite=True: when any merged
 * gradient of a push holds inf/nan, that push changes neither weights nor optimizer state (the AMP
 * overflow skip of gluon/trainer.py:445-448, decided on the device inside the same launch sequence). */
MXKV_DLL int MXKVB200SetOptimizer(KVStoreHandle handle, const char* name, uint32_t num_params,
                                  const char** keys, const char** vals);
MXKV_DLL int MXKVB200SetLearningRate(KVStoreHandle handle, double lr);
/* per-key multipliers (Optimizer.set_lr_mult / set_wd_mult); pass str_key = NULL for int keys */
MXKV_DLL int MXKVB200SetOptimizerMult(KVStoreHandle handle, int key, const char* str_key,
                                      float lr_mult, float wd_mult);
/* The native counterpart of the reference's per-device Updater (python/mxnet/optimizer/updater.py:
 * 39-93) and of the multi-tensor update operators it ends in when parameters are NOT updated on the
 * kvstore (multi_sgd_update / multi_sgd_mom_update / multi_mp_sgd_*, src/operator/optimizer_op-inl.h:
 * 207-375; multi_adamw, multi_lamb, multi_lans).  Create the handle with MXKVStoreCreate("updater"),
 * give it an optimizer with MXKVB200SetOptimizer, then every call updates all (weight, grad) pairs
 * IN PLACE with one launch (sequence) on their GPU.  Optimizer state of an index is created on first
 * sight and is reachable through MXKVB200GetState / SetState / Get|SetUpdateCount.  One handle serves
 * one device, like the reference's `Trainer._updaters[dev]`.  Never collective.  grads == NULL only
 * registers the indices with their weights (so that states can be loaded before the first update). */
MXKV_DLL int MXKVB200UpdaterStep(KVStoreHandle handle, uint32_t num, const int* keys,
                                 NDArrayHandle* weights, NDArrayHandle* grads);
MXKV_DLL int MXKVB200UpdaterStepEx(KVStoreHandle handle, uint32_t num, const char** keys,
                                   NDArrayHandle* weights, NDArrayHandle* grads);
/* Introspection: the per-key scalars the fused kernel would receive for the key's CURRENT update count
 * (learning rate with lr_mult and, for Adam, the host-side bias correction folded in; weight decay with
 * wd_mult; AdamW: operator lr = 1 and eta = the bias-corrected learning rate).  Host-only, no GPU needed. */
MXKV_DLL int MXKVB200GetKeyHyper(KVStoreHandle handle, int key, const char* str_key, float* lr, float* wd,
                                 float* eta);
/* per-key switch of a fused optimizer.  "no_trust_ratio" != 0: LARS keeps the plain learning rate
 * for this key (the reference does so for names ending in gamma / beta / bias, lars.py:121-123). */
MXKV_DLL int MXKVB200SetKeyFlag(KVStoreHandle handle, int key, const char* str_key, const char* name,
                                int value);
/* skip_nonfinite: *out = 1 if the last push met a non-finite gradient and was therefore skipped.
 * Waits for the engine streams, takes the skipped step back out of the update counts and clears the
 * flag (the next push does the same implicitly). */
MXKV_DLL int MXKVB200GetOverflow(KVStoreHandle handle, int* out);
/* multi_sum_sq (src/operator/contrib/multi_sum_sq-inl.h:83-96): out[i] = sum((scale * arrays[i])^2),
 * float32 [num] on the arrays' GPU; and multi_all_finite (src/operator/all_finite.cu:68-103):
 * out[0] = 0 if any element of any array is inf/nan (init_output != 0: out[0] is set to 1 first). */
MXKV_DLL int MXKVB200MultiSumSq(uint32_t num, NDArrayHandle* arrays, float scale, NDArrayHandle out);
MXKV_DLL int MXKVB200MultiAllFinite(uint32_t num, NDArrayHandle* arrays, int init_output, NDArrayHandle out);
/* which: 0 stored value, 1 fp32 master weight, 2 state0 (momentum | mean), 3 state1 (variance).
 * Returns a NEW handle aliasing engine memory (free it with MXNDArrayFree); *out = NULL when the
 * state does not exist. */
MXKV_DLL int MXKVB200GetState(KVStoreHandle handle, int key, const char* str_key, int which,
                              NDArrayHandle* out);
MXKV_DLL int MXKVB200SetState(KVStoreHandle handle, int key, const char* str_key, int which,
                              NDArrayHandle value);
MXKV_DLL int MXKVB200GetUpdateCount(KVStoreHandle handle, int key, const char* str_key, int64_t* out);
MXKV_DLL int MXKVB200SetUpdateCount(KVStoreHandle handle, int key, const char* str_key, int64_t count);

/* Wrap device/host memory owned by the embedding framework (no copy, no ownership). */
MXKV_DLL int MXKVB200NDArrayFromPtr(void* data, const int64_t* shape, int ndim, int dev_type, int dev_id,
                                    int dtype, NDArrayHandle* out);
/* Stream the embedding framework computes on for GPU dev_id (default: the legacy default
 * stream).  Engine work is ordered after what is queued there at call time. */
MXKV_DLL int MXKVB200SetStream(int dev_id, void* cuda_stream);
/* ---- engine ops (include/mxnet/c_api.h:3010-3127) ---------------------------------------------------------
 * Horovod-style plug-ins wrap their work in engine ops so that it is ordered with the framework's reads and writes
 * of the arrays involved.  This engine has no dependency graph -- ordering is by CUDA streams -- so the four entry
 * points are served conservatively: deferred calls are issued, every engine stream is drained (a superset of the
 * named dependencies), then the function runs on the calling thread; the Async flavours wait until the function
 * has called `on_complete`.  `ctx_handle` points at {int dev_type; int dev_id} (mxnet::Context's layout);
 * variable handles, `prop_handle`, `priority`, `opr_name` and `wait` are accepted and not interpreted. */
typedef void (*EngineAsyncFunc)(void* rctx, void* on_complete, void* param);
typedef void (*EngineSyncFunc)(void* rctx, void* param);
typedef void (*EngineFuncParamDeleter)(void* param);
typedef const void* ContextHandle;
typedef void* EngineVarHandle;
typedef const void* EngineFnPropertyHandle;
MXKV_DLL int MXEnginePushAsync(EngineAsyncFunc async_func, void* func_param, EngineFuncParamDeleter deleter,
                               ContextHandle ctx_handle, EngineVarHandle const_vars_handle, int num_const_vars,
                               EngineVarHandle mutable_vars_handle, int num_mutable_vars,
                               EngineFnPropertyHandle prop_handle, int priority, const char* opr_name, bool wait);
MXKV_DLL int MXEnginePushSync(EngineSyncFunc sync_func, void* func_param, EngineFuncParamDeleter deleter,
                              ContextHandle ctx_handle, EngineVarHandle const_vars_handle, int num_const_vars,
                              EngineVarHandle mutable_vars_handle, int num_mutable_vars,
                              EngineFnPropertyHandle prop_handle, int priority, const char* opr_name);
MXKV_DLL int MXEnginePushAsyncND(EngineAsyncFunc async_func, void* func_param, EngineFuncParamDeleter deleter,
                                 ContextHandle ctx_handle, NDArrayHandle* const_nds_handle, int num_const_nds,
                                 NDArrayHandle* mutable_nds_handle, int num_mutable_nds,
                                 EngineFnPropertyHandle prop_handle, int priority, const char* opr_name, bool wait);
MXKV_DLL int MXEnginePushSyncND(EngineSyncFunc sync_func, void* func_param, EngineFuncParamDeleter deleter,
                                ContextHandle ctx_handle, NDArrayHandle* const_nds_handle, int num_const_nds,
                                NDArrayHandle* mutable_nds_handle, int num_mutable_nds,
                                EngineFnPropertyHandle prop_handle, int priority, const char* opr_name);
/* The callback an EngineAsyncFunc receives as `on_complete`: call it once, from any thread, when the work is done
 * (the reference hands out an engine::CallbackOnComplete*; its one operation is this call). */
MXKV_DLL void MXKVB200EngineOnComplete(void* on_complete);

/* The engine's own CUDA stream for GPU dev_id (cudaStream_t), e.g. to record timing events on the
 * stream the kernels are launched on. */
MXKV_DLL int MXKVB200GetEngineStream(int dev_id, void** out);
/* auto_fence = 1 (default): after every call the framework stream waits for the engine stream.
 * 0: the caller issues MXKVB200Fence itself (one stream-wait per training step instead of one
 * per key; nothing blocks the host either way). */
MXKV_DLL int MXKVB200SetAutoFence(int auto_fence);
MXKV_DLL int MXKVB200Fence(int dev_id);
MXKV_DLL int MXKVB200GetLaunchCount(int64_t* out);
/* Dense reduce(+update) launches so far by kernel variant: 0 = per-thread (kv_dense_kernel), 1 = shared-memory
 * staged (kv_dense_bulk_kernel, cp.async.bulk + mbarrier), 2 = NVSwitch multicast (kv_dense_nvls_kernel),
 * 3 = tree order (kv_dense_tree_kernel / kv_sum_tree_f64_kernel, MXNET_KVSTORE_USETREE=1).
 * Test / bench instrumentation: proves which kernel a parity check has just exercised. */
MXKV_DLL int MXKVB200GetVariantLaunchCount(int variant, int64_t* out);
/* push / pushpull calls of this store served from a cached launch plan (a call whose keys and arrays repeat
 * while nothing else touched its keys replays its recorded work lists; MXKV_B200_PLAN=0 turns the cache off,
 * =2 builds every call both ways and aborts on a difference).  Instrumentation. */
MXKV_DLL int MXKVB200GetPlanHits(KVStoreHandle handle, int64_t* out);
/* Deferred issue -- what `priority` (include/mxnet/c_api.h:2592-2760) means on this engine.  The reference's
 * dependency engine runs the ops that are ready in priority order (src/engine/threaded_engine_perdevice.cc:97-279);
 * an in-order CUDA stream has no queue to reorder, so the store keeps one: with on = 1, MXKVStorePush /
 * MXKVStorePushPull calls with dense GPU values and integer keys are recorded instead of launched, and
 * MXKVB200Flush -- or any call that reads or changes the store, or waits for / copies an array -- issues them
 * highest priority first (never ahead of an earlier call on the same key) with neighbouring calls on disjoint keys
 * merged into one launch.  MXKVB200GetDeferredBatches: launches (sequences) issued that way so far. */
MXKV_DLL int MXKVB200SetDeferred(KVStoreHandle handle, int on);
MXKV_DLL int MXKVB200Flush(KVStoreHandle handle);
MXKV_DLL int MXKVB200GetDeferredBatches(KVStoreHandle handle, int64_t* out);
MXKV_DLL int MXKVB200SetTwoShotBytes(int64_t bytes);
/* Kernel scheduling knobs (also MXKV_B200_CHUNK / _THREADS / _MAX_BLOCKS / _BULK): elements per
 * scheduling chunk, block size (128/256/512), cap on the grid (0 = resident capacity), and the
 * shared-memory staged (cp.async.bulk) variant: 0 off, 1 auto (keys with <= 2 sources), 2 whenever
 * eligible, -1 keep.  Every rank of a process group must use the same values. */
MXKV_DLL int MXKVB200SetTuning(int64_t chunk_elems, int threads, int max_blocks, int bulk);

/* [begin, end) of the elements rank `rank` of `world` reduces and updates for a key of `size`
 * elements on the sharded (two-shot) path.  Pure host function. */
MXKV_DLL int MXKVB200ShardRange(int64_t size, int world, int rank, int64_t* begin, int64_t* end);

/* One process per GPU.  allgather(send, bytes, recv, ctx) must gather `bytes` from every rank
 * into recv (rank-major) on the host and return 0; it is used for bootstrap only (IPC handles,
 * allocation agreement), never on the data path. */
typedef int (*MXKVB200AllGatherFn)(const void* send, size_t bytes, void* recv, void* ctx);
MXKV_DLL int MXKVB200CommInit(int rank, int world, int dev_id, MXKVB200AllGatherFn allgather, void* ctx);
MXKV_DLL int MXKVB200CommDestroy(void);
/* Multi-node (kv.create('dist_device_sync'), the hierarchical form of KVStoreDist's synchronous mode,
 * src/kvstore/kvstore_dist.h:343-470): the group of MXKVB200CommInit is ONE node; `allreduce` sums `count`
 * elements of `dtype` (mshadow type flag) in place, on the device, over the ranks that have this rank's local
 * rank on every node, ordered on `cuda_stream` (e.g. ncclAllReduce on that stream).  Per push the engine runs
 * reduce-scatter inside the node -> ONE such call per dtype over this rank's packed shards -> fused update +
 * all-gather inside the node (row_sparse pushes: the node's merge, then a gather of the nodes' merged rows through
 * the same callback with dtype int64 / float32).  Returns non-zero on failure.  Call after MXKVB200CommInit, before creating stores. */
typedef int (*MXKVB200AllReduceFn)(void* dev_ptr, int64_t count, int dtype, void* cuda_stream, void* ctx);
MXKV_DLL int MXKVB200SetHierarchy(int node_rank, int num_nodes, MXKVB200AllReduceFn allreduce, void* ctx);
/* Collective: every rank calls it in the same order with the same shape.  The array lives in the
 * peer-mapped arena, so push/pushpull read and write it over NVLink without staging. */
MXKV_DLL int MXKVB200NDArrayCreateSymmetric(const int64_t* shape, int ndim, int dtype, NDArrayHandle* out);

/* 1 if the array has an NVSwitch multicast alias (arrays of MXKVB200NDArrayCreateSymmetric on a machine whose GPUs
 * support multicast: the arena is then built from CUDA VMM allocations bound to a multicast object, vmm_arena.cc;
 * arrays wrapped with a multicast pointer by MXKVB200NDArrayFromPeers), i.e. the NVLS kernel can serve it. */
MXKV_DLL int MXKVB200NDArrayHasMulticast(NDArrayHandle handle, int* out);

/* Wrap peer-mapped memory owned by the embedding framework (one process per GPU): peer_ptrs[r] is
 * the address of rank r's copy as mapped in THIS process, mc_ptr the NVSwitch multicast alias of all
 * copies (NULL when none).  With a multicast alias the exchange uses the NVLS kernel
 * (multimem.ld_reduce / multimem.st): the switch does the sum and the replication. */
MXKV_DLL int MXKVB200NDArrayFromPeers(void* const* peer_ptrs, int world, void* mc_ptr, const int64_t* shape,
                                      int ndim, int dtype, NDArrayHandle* out);
/* 0: never use the NVLS kernel; 1 (default): use it above 4 ranks when every array of a key has a
 * multicast alias; 2: whenever the arrays have one */
MXKV_DLL int MXKVB200SetNvls(int mode);
/* Scheduling of the NVLS kernel (also MXKV_B200_NVLS_U / _PIPE / _GRID / _THREADS): multimem.ld_reduce requests
 * in flight per thread (1, 2, 4, 8; <= 0 keeps), software pipelining of the reduce-scatter half (0 / 1; < 0
 * keeps), cap on the grid (0 = resident capacity; < 0 keeps), block size (128 / 256 / 512; anything else keeps).
 * Every rank of the process group must use the same values. */
MXKV_DLL int MXKVB200SetNvlsTuning(int unroll, int pipe, int grid, int threads);


/* ---- MXNET_KVSTORE_USETREE=1: the reduction trees of CommDeviceTree (src/kvstore/comm_tree.h:50-325) ----------
 * A store of a `device` type created with MXNET_KVSTORE_USETREE=1 adds the values of a key pairwise up the binary
 * trees the reference's solver builds from the GPUs' link matrix (src/kvstore/gpu_topology.h:1111-1157), slice by
 * slice for keys above MXNET_KVSTORE_TREE_ARRAY_BOUND elements (comm_tree.h:203-234) -- same bits as the reference's
 * tree mode; the transport stays this library's one-pass kernel.  MXNET_KVSTORE_TREE_BACKTRACK and
 * MXNET_KVSTORE_TREE_LINK_USAGE_PENALTY are read like the reference reads them (comm_tree.h:52-57).
 * The entry points below expose the pieces so that a test (or a maintainer) can compare them with the reference:
 * the link matrix GetP2PWeight would produce from the driver's answers (gpu_topology.h:137-253) ... */
MXKV_DLL int MXKVB200TopologyLinkWeights(int n, const int* perf_rank, const int* can_access, float* weights_out);
/* ... the same, querying the driver for the CUDA devices devs[0..n) (MXKV_B200_TREE_LINKS overrides) ... */
MXKV_DLL int MXKVB200TopologyQueryLinks(int n, const int* devs, float* weights_out);
/* ... ComputeTrees: n trees in array form, tree r at topo_out[r * *topo_len ...] (2^(depth+1) - 1 entries each),
 * level starts at scan_out[r * *scan_len ...] (depth + 2 entries each); caps are in entries ... */
MXKV_DLL int MXKVB200TopologyComputeTrees(const float* weights, int n, float alpha, int backtrack, uint64_t* topo_out,
                                          int topo_cap, int* topo_len, uint64_t* scan_out, int scan_cap, int* scan_len,
                                          int* depth);
/* ... one Kernighan-Lin pass (KernighanLin, gpu_topology.h:326-480) with std::mt19937(seed): returns *stop,
 * updates partition[0..n) and *num_partitions, writes (first, second) pairs ... */
MXKV_DLL int MXKVB200TopologyBisect(const float* weights, int n, int* partition, int* num_partitions, int* pairs_out,
                                    int pairs_cap, int* n_pairs, uint32_t seed, int* stop);
/* ... Postprocess (:746-770), ComputeTreeWeight (:778-813), IsValid (:727-791), IsConnected (:96-121) ... */
MXKV_DLL int MXKVB200TopologyFoldRepeats(int* leaves, int len, int n, int depth);
MXKV_DLL int MXKVB200TopologyTreeWeight(const float* weights, const int* leaves, int len, int n, int depth, int penalty,
                                        float* out);
MXKV_DLL int MXKVB200TopologyAdmissible(const float* weights, const int* state, int len, int n, int row, int depth,
                                        int* out);
MXKV_DLL int MXKVB200TopologyConnected(const float* weights, int n, int* out);
/* ... and the order in which the kernel adds the n values of an element for one tree (topology.h: ReduceProgram):
 * leaves_out[0..n) = participants in the order their values are taken, *prog_out = the add schedule. */
MXKV_DLL int MXKVB200TopologyReduceProgram(const uint64_t* topo, int topo_len, const uint64_t* scan, int scan_len, int n,
                                           int* leaves_out, uint32_t* prog_out);
/* Evaluates a reduce program on the host with the kernel's own code (csrc/tree_math.h compiled for the CPU):
 * out[e] = the tree sum of srcs[leaf k][e] taken in program order, float32.  Test instrumentation. */
MXKV_DLL int MXKVB200TopologyRunProgram(const float* const* srcs_in_leaf_order, int n, uint32_t prog, int64_t count,
                                        float* out);

#ifdef __cplusplus
}
#endif
#endif  /* MXKV_B200_H_ */
