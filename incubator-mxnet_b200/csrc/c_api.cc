// c_api.cc -- extern "C" shims: marshal C arrays into the engine and translate exceptions
// into the 0 / -1 + MXGetLastError() contract (API_BEGIN/API_END,
// include/mxnet/c_api_error.h:40-58; KVStore marshalling src/c_api/c_api.cc:2771-3204).
#include <condition_variable>
#include <mutex>
#include "../../include/mxkv_b200.h"
#include <algorithm>
#include <cstring>
#include "dlpack_abi.h"
#include "kvstore.h"
#include <random>
#include "topology.h"
#include "tree_math.h"

using namespace mxkv;

#define API_BEGIN() try {
#define API_END()                                                      \
  } catch (const std::exception& e) {                                  \
    ::mxkv::SetLastError(e.what());                                    \
    return -1;                                                         \
  } catch (...) {                                                      \
    ::mxkv::SetLastError("unknown C++ exception");                     \
    return -1;                                                         \
  }                                                                    \
  return 0;

namespace {
inline NDHandle* ND(NDArrayHandle h) {
  MXKV_CHECK(h != nullptr) << "null NDArrayHandle";
  return static_cast<NDHandle*>(h);
}
inline KVStore* KV(KVStoreHandle h) {
  MXKV_CHECK(h != nullptr) << "null KVStoreHandle";
  return static_cast<KVStore*>(h);
}
std::vector<NDArray> Vals(NDArrayHandle* vals, uint32_t n) {
  std::vector<NDArray> v(n);
  for (uint32_t i = 0; i < n; ++i) v[i] = *ND(vals[i]);
  return v;
}
std::vector<NDArray*> Outs(NDArrayHandle* vals, uint32_t n) {
  std::vector<NDArray*> v(n);
  for (uint32_t i = 0; i < n; ++i) v[i] = ND(vals[i]);
  return v;
}
std::vector<int> IKeys(const int* keys, uint32_t n) { return std::vector<int>(keys, keys + n); }
std::vector<std::string> SKeys(const char** keys, uint32_t n) {
  std::vector<std::string> v(n);
  for (uint32_t i = 0; i < n; ++i) v[i] = keys[i];
  return v;
}
}  // namespace

extern "C" {

const char* MXGetLastError(void) { return ::mxkv::GetLastError(); }

int MXGetGPUCount(int* out) {
  API_BEGIN();
  *out = Runtime::Get()->NumDevices();
  API_END();
}

int MXGetVersion(int* out) {
  API_BEGIN();
  *out = 20000;   // MXNET_VERSION of the reference snapshot (include/mxnet/base.h:62-68)
  API_END();
}

// ---------------------------------------------------------------------------
// NDArray
// ---------------------------------------------------------------------------
int MXNDArrayCreateNone(NDArrayHandle* out) {
  API_BEGIN();
  *out = new NDHandle();
  API_END();
}

int MXNDArrayCreate64(const int64_t* shape, int ndim, int dev_type, int dev_id, int delay_alloc, int dtype,
                      NDArrayHandle* out) {
  API_BEGIN();
  (void)delay_alloc;
  std::vector<int64_t> s(shape, shape + ndim);
  *out = new NDHandle(NDArray::Empty(s, Context{dev_type, dev_id}, dtype));
  API_END();
}

int MXNDArrayCreate(const uint32_t* shape, uint32_t ndim, int dev_type, int dev_id, int delay_alloc, int dtype,
                    NDArrayHandle* out) {
  std::vector<int64_t> s(shape, shape + ndim);
  return MXNDArrayCreate64(s.data(), static_cast<int>(ndim), dev_type, dev_id, delay_alloc, dtype, out);
}

int MXNDArrayCreateSparseEx64(int storage_type, const int64_t* shape, int ndim, int dev_type, int dev_id,
                              int delay_alloc, int dtype, uint32_t num_aux, int* aux_type, int* aux_ndims,
                              const int64_t* aux_shape, NDArrayHandle* out) {
  API_BEGIN();
  (void)delay_alloc;
  MXKV_CHECK(storage_type == kRowSparseStorage) << "only row_sparse sparse arrays are supported (got stype "
                                                << storage_type << ")";
  MXKV_CHECK(num_aux == 1) << "row_sparse has exactly one aux array";
  MXKV_CHECK(aux_type == nullptr || aux_type[0] == kInt64) << "row_sparse indices must be int64";
  std::vector<int64_t> s(shape, shape + ndim);
  int64_t cap = 0;
  if (aux_ndims != nullptr && aux_ndims[0] >= 1 && aux_shape != nullptr) cap = aux_shape[0];
  if (cap <= 0) cap = s.empty() ? 0 : s[0];
  *out = new NDHandle(NDArray::EmptyRowSparse(s, Context{dev_type, dev_id}, dtype, cap));
  API_END();
}

int MXNDArrayFree(NDArrayHandle handle) {
  API_BEGIN();
  delete static_cast<NDHandle*>(handle);
  API_END();
}

int MXNDArraySyncCopyFromCPU(NDArrayHandle handle, const void* data, size_t size) {
  API_BEGIN();
  FlushAllDeferred();      // deferred pushes may read or write this array
  ND(handle)->SyncCopyFromCPU(data, size);
  API_END();
}

int MXNDArraySyncCopyToCPU(NDArrayHandle handle, void* data, size_t size) {
  API_BEGIN();
  FlushAllDeferred();      // deferred pushes may read or write this array
  ND(handle)->SyncCopyToCPU(data, size);
  API_END();
}

int MXNDArraySyncCopyFromNDArray(NDArrayHandle handle_dst, const NDArrayHandle handle_src, const int i) {
  API_BEGIN();
  NDHandle* dst = ND(handle_dst);
  NDHandle* src = ND(handle_src);
  NDArray s = *src;
  if (src->stype() == kRowSparseStorage) s = (i < 0) ? src->data_nd() : src->aux_idx();
  NDArray d = *dst;
  if (dst->stype() == kRowSparseStorage) {
    // filling a row_sparse destination: i < 0 data, i >= 0 indices; the row count follows the source
    const int64_t rows = s.shape().empty() ? 0 : s.shape()[0];
    // row_sparse arrays are dynamically sized in the reference (CheckAndAlloc): grow on demand.  Growing
    // discards the contents, so fill the data (i < 0) before the indices, as the front-end does.
    if (rows > dst->cap_rows()) dst->ReserveRows(rows);
    dst->set_nnz(rows);
    d = (i < 0) ? dst->data_nd() : dst->aux_idx();
  }
  CopyFromTo(s.Reshape({s.size()}), d.Reshape({d.size()}));
  d.WaitToRead();
  API_END();
}

int MXNDArrayWaitToRead(NDArrayHandle handle) {
  API_BEGIN();
  FlushAllDeferred();      // deferred pushes may read or write this array
  ND(handle)->WaitToRead();
  API_END();
}

int MXNDArrayWaitToWrite(NDArrayHandle handle) {
  API_BEGIN();
  FlushAllDeferred();      // deferred pushes may read or write this array
  ND(handle)->WaitToWrite();
  API_END();
}

int MXNDArrayWaitAll(void) {
  API_BEGIN();
  FlushAllDeferred();      // deferred pushes may read or write this array
  Runtime::Get()->WaitAll();
  API_END();
}

int MXNDArrayGetStorageType(NDArrayHandle handle, int* out_storage_type) {
  API_BEGIN();
  NDHandle* a = ND(handle);
  *out_storage_type = a->is_none() ? kUndefinedStorage : a->stype();
  API_END();
}

int MXNDArrayGetShape64(NDArrayHandle handle, int* out_dim, const int64_t** out_pdata) {
  API_BEGIN();
  NDHandle* a = ND(handle);
  a->shape64 = a->shape();
  *out_dim = static_cast<int>(a->shape64.size());
  *out_pdata = a->shape64.data();
  API_END();
}

int MXNDArrayGetShape(NDArrayHandle handle, int* out_dim, const int** out_pdata) {
  API_BEGIN();
  NDHandle* a = ND(handle);
  a->shape32.assign(a->shape().begin(), a->shape().end());
  *out_dim = static_cast<int>(a->shape32.size());
  *out_pdata = a->shape32.data();
  API_END();
}

int MXNDArrayGetData(NDArrayHandle handle, void** out_pdata) {
  API_BEGIN();
  *out_pdata = ND(handle)->data();
  API_END();
}

int MXNDArrayToDLPack(NDArrayHandle handle, DLManagedTensorHandle* out_dlpack) {
  API_BEGIN();
  *out_dlpack = ND(handle)->ToDLPack();
  API_END();
}

int MXNDArrayFromDLPack(DLManagedTensorHandle dlpack, const bool transient_handle, NDArrayHandle* out_handle) {
  API_BEGIN();
  *out_handle = new NDHandle(NDArray::FromDLPack(static_cast<DLManagedTensor*>(dlpack), transient_handle));
  API_END();
}

int MXNDArrayCallDLPackDeleter(DLManagedTensorHandle dlpack) {
  API_BEGIN();
  DLManagedTensor* t = static_cast<DLManagedTensor*>(dlpack);
  if (t != nullptr && t->deleter != nullptr) t->deleter(t);
  API_END();
}

int MXNDArrayGetDType(NDArrayHandle handle, int* out_dtype) {
  API_BEGIN();
  NDHandle* a = ND(handle);
  *out_dtype = a->is_none() ? -1 : a->dtype();
  API_END();
}

int MXNDArrayGetAuxType(NDArrayHandle handle, uint32_t i, int* out_type) {
  API_BEGIN();
  MXKV_CHECK(ND(handle)->stype() == kRowSparseStorage && i == 0) << "no such aux array";
  *out_type = kInt64;
  API_END();
}

int MXNDArrayGetAuxNDArray(NDArrayHandle handle, uint32_t i, NDArrayHandle* out) {
  API_BEGIN();
  MXKV_CHECK(ND(handle)->stype() == kRowSparseStorage && i == 0) << "no such aux array";
  *out = new NDHandle(ND(handle)->aux_idx());
  API_END();
}

int MXNDArrayGetDataNDArray(NDArrayHandle handle, NDArrayHandle* out) {
  API_BEGIN();
  NDHandle* a = ND(handle);
  *out = new NDHandle(a->stype() == kRowSparseStorage ? a->data_nd() : *a);
  API_END();
}

int MXNDArrayGetContext(NDArrayHandle handle, int* out_dev_type, int* out_dev_id) {
  API_BEGIN();
  NDHandle* a = ND(handle);
  if (a->is_none()) { *out_dev_type = 0; *out_dev_id = 0; }
  else { *out_dev_type = a->ctx().dev_type; *out_dev_id = a->ctx().dev_id; }
  API_END();
}

int MXNDArrayReshape64(NDArrayHandle handle, int ndim, int64_t* dims, bool reverse, NDArrayHandle* out) {
  API_BEGIN();
  (void)reverse;
  std::vector<int64_t> s(dims, dims + ndim);
  NDHandle* a = ND(handle);
  int64_t known = 1, unknown = -1;
  for (int i = 0; i < ndim; ++i) {
    if (s[i] == -1) { MXKV_CHECK(unknown < 0) << "only one dimension can be inferred"; unknown = i; }
    else known *= s[i];
  }
  if (unknown >= 0) { MXKV_CHECK(known > 0 && a->size() % known == 0) << "cannot infer dimension"; s[unknown] = a->size() / known; }
  *out = new NDHandle(a->Reshape(s));
  API_END();
}

// ---------------------------------------------------------------------------
// KVStore
// ---------------------------------------------------------------------------
int MXKVStoreCreate(const char* type, KVStoreHandle* out) {
  API_BEGIN();
  MXKV_CHECK(type != nullptr) << "null kvstore type";
  *out = new KVStore(type);
  API_END();
}

int MXKVStoreSetGradientCompression(KVStoreHandle handle, uint32_t num_params, const char** keys,
                                    const char** vals) {
  API_BEGIN();
  std::vector<std::pair<std::string, std::string>> kw;
  for (uint32_t i = 0; i < num_params; ++i) kw.emplace_back(keys[i], vals[i]);
  KV(handle)->SetGradientCompression(kw);
  API_END();
}

int MXKVStoreFree(KVStoreHandle handle) {
  API_BEGIN();
  delete static_cast<KVStore*>(handle);
  API_END();
}

int MXKVStoreInit(KVStoreHandle handle, uint32_t num, const int* keys, NDArrayHandle* vals) {
  API_BEGIN();
  KV(handle)->Init(IKeys(keys, num), Vals(vals, num));
  API_END();
}

int MXKVStoreInitEx(KVStoreHandle handle, uint32_t num, const char** keys, NDArrayHandle* vals) {
  API_BEGIN();
  KV(handle)->Init(SKeys(keys, num), Vals(vals, num));
  API_END();
}

namespace {
// the fast path needs NDArray pointers; NDHandle IS an NDArray (ndarray.h)
inline NDArray* const* AsArrays(NDArrayHandle* h) { return reinterpret_cast<NDArray* const*>(h); }
struct PendingGuard { KVStore* kv; ~PendingGuard() { kv->ClearRawPending(); } };
}  // namespace

int MXKVStorePush(KVStoreHandle handle, uint32_t num, const int* keys, NDArrayHandle* vals, int priority) {
  API_BEGIN();
  KVStore* kv = KV(handle);
  // a repeated call replays its cached launch plan straight from the raw arguments (kvstore.h: CallPlan)
  if (kv->TryReplayRaw(0, num, keys, AsArrays(vals), 0, nullptr, nullptr)) return 0;
  PendingGuard guard{kv};
  kv->Push(IKeys(keys, num), Vals(vals, num), priority);
  API_END();
}

int MXKVStorePushEx(KVStoreHandle handle, uint32_t num, const char** keys, NDArrayHandle* vals, int priority) {
  API_BEGIN();
  KV(handle)->Push(SKeys(keys, num), Vals(vals, num), priority);
  API_END();
}

int MXKVStorePullWithSparse(KVStoreHandle handle, uint32_t num, const int* keys, NDArrayHandle* vals, int priority,
                            bool ignore_sparse) {
  API_BEGIN();
  KV(handle)->Pull(IKeys(keys, num), Outs(vals, num), priority, ignore_sparse);
  API_END();
}

int MXKVStorePullWithSparseEx(KVStoreHandle handle, uint32_t num, const char** keys, NDArrayHandle* vals,
                              int priority, bool ignore_sparse) {
  API_BEGIN();
  KV(handle)->Pull(SKeys(keys, num), Outs(vals, num), priority, ignore_sparse);
  API_END();
}

int MXKVStorePull(KVStoreHandle handle, uint32_t num, const int* keys, NDArrayHandle* vals, int priority) {
  return MXKVStorePullWithSparse(handle, num, keys, vals, priority, true);   // c_api.cc:2860-2875
}

int MXKVStorePullEx(KVStoreHandle handle, uint32_t num, const char** keys, NDArrayHandle* vals, int priority) {
  return MXKVStorePullWithSparseEx(handle, num, keys, vals, priority, true);
}

int MXKVStorePullRowSparse(KVStoreHandle handle, uint32_t num, const int* keys, NDArrayHandle* vals,
                           const NDArrayHandle* row_ids, int priority) {
  API_BEGIN();
  std::vector<std::pair<NDArray*, NDArray>> vr(num);
  for (uint32_t i = 0; i < num; ++i) vr[i] = {ND(vals[i]), *ND(row_ids[i])};
  KV(handle)->PullRowSparse(IKeys(keys, num), vr, priority);
  API_END();
}

int MXKVStorePullRowSparseEx(KVStoreHandle handle, uint32_t num, const char** keys, NDArrayHandle* vals,
                             const NDArrayHandle* row_ids, int priority) {
  API_BEGIN();
  std::vector<std::pair<NDArray*, NDArray>> vr(num);
  for (uint32_t i = 0; i < num; ++i) vr[i] = {ND(vals[i]), *ND(row_ids[i])};
  KV(handle)->PullRowSparse(SKeys(keys, num), vr, priority);
  API_END();
}

int MXKVStoreBroadcast(KVStoreHandle handle, mx_uint vnum, const int* vkeys, mx_uint onum, const int* okeys,
                       NDArrayHandle* vals, NDArrayHandle* outs, int priority) {
  API_BEGIN();
  KV(handle)->Broadcast(IKeys(vkeys, vnum), IKeys(okeys, onum), Vals(vals, vnum), Outs(outs, onum), priority);
  API_END();
}

int MXKVStoreBroadcastEx(KVStoreHandle handle, mx_uint vnum, const char** vkeys, mx_uint onum, const char** okeys,
                         NDArrayHandle* vals, NDArrayHandle* outs, int priority) {
  API_BEGIN();
  KV(handle)->Broadcast(SKeys(vkeys, vnum), SKeys(okeys, onum), Vals(vals, vnum), Outs(outs, onum), priority);
  API_END();
}

int MXKVStorePushPull(KVStoreHandle handle, mx_uint vnum, const int* vkeys, mx_uint onum, const int* okeys,
                      NDArrayHandle* vals, NDArrayHandle* outs, int priority) {
  API_BEGIN();
  KVStore* kv = KV(handle);
  if (kv->TryReplayRaw(1, vnum, vkeys, AsArrays(vals), onum, okeys, AsArrays(outs))) return 0;
  PendingGuard guard{kv};
  kv->PushPull(IKeys(vkeys, vnum), IKeys(okeys, onum), Vals(vals, vnum), Outs(outs, onum), priority);
  API_END();
}

int MXKVStorePushPullEx(KVStoreHandle handle, mx_uint vnum, const char** vkeys, mx_uint onum, const char** okeys,
                        NDArrayHandle* vals, NDArrayHandle* outs, int priority) {
  API_BEGIN();
  KV(handle)->PushPull(SKeys(vkeys, vnum), SKeys(okeys, onum), Vals(vals, vnum), Outs(outs, onum), priority);
  API_END();
}

int MXKVStoreSetUpdater(KVStoreHandle handle, MXKVStoreUpdater updater, void* updater_handle) {
  API_BEGIN();
  KV(handle)->SetUpdater(reinterpret_cast<UpdaterFn>(updater), nullptr, updater_handle);
  API_END();
}

int MXKVStoreSetUpdaterEx(KVStoreHandle handle, MXKVStoreUpdater updater, MXKVStoreStrUpdater str_updater,
                          void* updater_handle) {
  API_BEGIN();
  KV(handle)->SetUpdater(reinterpret_cast<UpdaterFn>(updater), reinterpret_cast<StrUpdaterFn>(str_updater),
                         updater_handle);
  API_END();
}

int MXKVStoreGetType(KVStoreHandle handle, const char** type) {
  API_BEGIN();
  *type = KV(handle)->type().c_str();   // borrowed, lives as long as the store (c_api.cc:3113-3118)
  API_END();
}

int MXKVStoreGetRank(KVStoreHandle handle, int* ret) {
  API_BEGIN();
  *ret = KV(handle)->rank();
  API_END();
}

int MXKVStoreGetGroupSize(KVStoreHandle handle, int* ret) {
  API_BEGIN();
  *ret = KV(handle)->group_size();
  API_END();
}

int MXKVStoreIsWorkerNode(int* ret) { *ret = 1; return 0; }       // kvstore.h:389-419: local stores are workers
int MXKVStoreIsServerNode(int* ret) { *ret = 0; return 0; }
int MXKVStoreIsSchedulerNode(int* ret) { *ret = 0; return 0; }

int MXKVStoreBarrier(KVStoreHandle handle) {
  API_BEGIN();
  KV(handle)->Barrier();
  API_END();
}

int MXKVStoreSetBarrierBeforeExit(KVStoreHandle handle, const int barrier_before_exit) {
  API_BEGIN();
  (void)KV(handle); (void)barrier_before_exit;
  API_END();
}

int MXKVStoreGetNumDeadNode(KVStoreHandle handle, const int node_id, int* number, const int timeout_sec) {
  API_BEGIN();
  (void)KV(handle); (void)node_id; (void)timeout_sec;
  *number = 0;   // kvstore.h:431-435: single-node stores have no dead nodes
  API_END();
}

int MXKVStoreRunServer(KVStoreHandle handle, MXKVStoreServerController controller, void* controller_handle) {
  API_BEGIN();
  (void)KV(handle); (void)controller; (void)controller_handle;   // kvstore.h:466: a no-op for single-node stores
  API_END();
}

int MXKVStoreSendCommmandToServers(KVStoreHandle handle, int cmd_id, const char* cmd_body) {
  API_BEGIN();
  (void)KV(handle); (void)cmd_id; (void)cmd_body;                // kvstore.h:432: a no-op for single-node stores
  API_END();
}

// ---------------------------------------------------------------------------
// extensions
// ---------------------------------------------------------------------------
int MXKVB200SetOptimizer(KVStoreHandle handle, const char* name, uint32_t num_params, const char** keys,
                         const char** vals) {
  API_BEGIN();
  std::vector<std::pair<std::string, std::string>> kw;
  for (uint32_t i = 0; i < num_params; ++i) kw.emplace_back(keys[i], vals[i]);
  KV(handle)->SetOptimizer(name, kw);
  API_END();
}

int MXKVB200SetLearningRate(KVStoreHandle handle, double lr) {
  API_BEGIN();
  KV(handle)->SetLearningRate(lr);
  API_END();
}

int MXKVB200SetOptimizerMult(KVStoreHandle handle, int key, const char* str_key, float lr_mult, float wd_mult) {
  API_BEGIN();
  KV(handle)->SetOptimizerMult(str_key != nullptr, key, str_key ? str_key : "", lr_mult, wd_mult);
  API_END();
}

int MXKVB200GetState(KVStoreHandle handle, int key, const char* str_key, int which, NDArrayHandle* out) {
  API_BEGIN();
  NDArray a = KV(handle)->GetState(str_key != nullptr, key, str_key ? str_key : "", which);
  *out = a.is_none() ? nullptr : new NDHandle(a);
  API_END();
}

int MXKVB200SetState(KVStoreHandle handle, int key, const char* str_key, int which, NDArrayHandle value) {
  API_BEGIN();
  KV(handle)->SetState(str_key != nullptr, key, str_key ? str_key : "", which, *ND(value));
  API_END();
}

int MXKVB200GetUpdateCount(KVStoreHandle handle, int key, const char* str_key, int64_t* out) {
  API_BEGIN();
  *out = KV(handle)->GetUpdateCount(str_key != nullptr, key, str_key ? str_key : "");
  API_END();
}

int MXKVB200SetUpdateCount(KVStoreHandle handle, int key, const char* str_key, int64_t count) {
  API_BEGIN();
  KV(handle)->SetUpdateCount(str_key != nullptr, key, str_key ? str_key : "", count);
  API_END();
}

int MXKVB200GetOptimizerScalar(KVStoreHandle handle, const char* name, double* out) {
  API_BEGIN();
  MXKV_CHECK(name != nullptr && out != nullptr) << "GetOptimizerScalar: null argument";
  *out = KV(handle)->GetOptimizerScalar(name);
  API_END();
}

int MXKVB200SetOptimizerScalar(KVStoreHandle handle, const char* name, double value) {
  API_BEGIN();
  MXKV_CHECK(name != nullptr) << "SetOptimizerScalar: null name";
  KV(handle)->SetOptimizerScalar(name, value);
  API_END();
}

int MXKVB200UpdaterStep(KVStoreHandle handle, uint32_t num, const int* keys, NDArrayHandle* weights,
                        NDArrayHandle* grads) {
  API_BEGIN();
  std::vector<int> k(keys, keys + num);
  std::vector<NDArray> w, g;
  for (uint32_t i = 0; i < num; ++i) {
    w.push_back(*ND(weights[i]));
    if (grads != nullptr) g.push_back(*ND(grads[i]));
  }
  KV(handle)->UpdaterStep(false, k, {}, w, g);
  API_END();
}

int MXKVB200UpdaterStepEx(KVStoreHandle handle, uint32_t num, const char** keys, NDArrayHandle* weights,
                          NDArrayHandle* grads) {
  API_BEGIN();
  std::vector<std::string> k;
  std::vector<NDArray> w, g;
  for (uint32_t i = 0; i < num; ++i) {
    k.emplace_back(keys[i]);
    w.push_back(*ND(weights[i]));
    if (grads != nullptr) g.push_back(*ND(grads[i]));
  }
  KV(handle)->UpdaterStep(true, {}, k, w, g);
  API_END();
}

int MXKVB200GetKeyHyper(KVStoreHandle handle, int key, const char* str_key, float* lr, float* wd, float* eta) {
  API_BEGIN();
  KV(handle)->GetKeyHyper(str_key != nullptr, key, str_key ? str_key : "", lr, wd, eta);
  API_END();
}

int MXKVB200SetKeyFlag(KVStoreHandle handle, int key, const char* str_key, const char* name, int value) {
  API_BEGIN();
  MXKV_CHECK(name != nullptr) << "flag name is null";
  KV(handle)->SetKeyFlag(str_key != nullptr, key, str_key ? str_key : "", name, value);
  API_END();
}

int MXKVB200GetOverflow(KVStoreHandle handle, int* out) {
  API_BEGIN();
  *out = KV(handle)->ResolveOverflow();
  API_END();
}

int MXKVB200MultiSumSq(uint32_t num, NDArrayHandle* arrays, float scale, NDArrayHandle out) {
  API_BEGIN();
  std::vector<NDArray> a;
  for (uint32_t i = 0; i < num; ++i) a.push_back(*ND(arrays[i]));
  NDArray o = *ND(out);
  MultiSumSq(a, scale, &o, nullptr, false);
  API_END();
}

int MXKVB200MultiAllFinite(uint32_t num, NDArrayHandle* arrays, int init_output, NDArrayHandle out) {
  API_BEGIN();
  std::vector<NDArray> a;
  for (uint32_t i = 0; i < num; ++i) a.push_back(*ND(arrays[i]));
  NDArray o = *ND(out);
  MultiSumSq(a, 1.0f, nullptr, &o, init_output != 0);
  API_END();
}

int MXKVB200NDArrayFromPtr(void* data, const int64_t* shape, int ndim, int dev_type, int dev_id, int dtype,
                           NDArrayHandle* out) {
  API_BEGIN();
  std::vector<int64_t> s(shape, shape + ndim);
  if (dev_type == kGPU) Runtime::Get()->Dev(dev_id);
  *out = new NDHandle(NDArray::FromExternal(data, s, Context{dev_type, dev_id}, dtype));
  API_END();
}

int MXKVB200NDArrayFromPeers(void* const* peer_ptrs, int world, void* mc_ptr, const int64_t* shape, int ndim,
                             int dtype, NDArrayHandle* out) {
  API_BEGIN();
  ProcessGroup* pg = Runtime::Get()->pg();
  MXKV_CHECK(pg != nullptr && pg->world() == world) << "MXKVB200NDArrayFromPeers needs a process group of " << world;
  std::vector<int64_t> s(shape, shape + ndim);
  *out = new NDHandle(NDArray::FromPeers(peer_ptrs, world, pg->rank(), mc_ptr, s, Context{kGPU, pg->dev()}, dtype));
  API_END();
}

int MXKVB200NDArrayHasMulticast(NDArrayHandle handle, int* out) {
  API_BEGIN();
  *out = ND(handle)->mc_data() != nullptr ? 1 : 0;
  API_END();
}

int MXKVB200SetNvls(int mode) {
  API_BEGIN();
  Runtime::Get()->nvls_mode = mode;
  Runtime::Get()->tuning_epoch++;
  API_END();
}

int MXKVB200SetNvlsTuning(int unroll, int pipe, int grid, int threads) {
  API_BEGIN();
  Runtime* rt = Runtime::Get();
  rt->WaitAll();
  rt->tuning_epoch++;
  if (unroll > 0) rt->nvls_unroll = unroll;
  if (pipe >= 0) rt->nvls_pipe = pipe != 0;
  if (grid >= 0) rt->nvls_grid = grid;
  if (threads == 128 || threads == 256 || threads == 512) rt->nvls_threads = threads;
  API_END();
}

// ---- engine ops: include/mxnet/c_api.h:3010-3127, served without a dependency graph (include/mxkv_b200.h) ----
namespace {
struct OnComplete {
  std::mutex mu;
  std::condition_variable cv;
  bool done = false;
};
void DrainForEngineOp() {
  FlushAllDeferred();
  Runtime::Get()->WaitAll();
}
int RunSync(EngineSyncFunc fn, void* param, EngineFuncParamDeleter deleter) {
  API_BEGIN();
  MXKV_CHECK(fn != nullptr) << "null engine function";
  DrainForEngineOp();
  fn(nullptr, param);
  if (deleter) deleter(param);
  API_END();
}
int RunAsync(EngineAsyncFunc fn, void* param, EngineFuncParamDeleter deleter) {
  API_BEGIN();
  MXKV_CHECK(fn != nullptr) << "null engine function";
  DrainForEngineOp();
  OnComplete oc;
  fn(nullptr, &oc, param);
  {
    std::unique_lock<std::mutex> lk(oc.mu);
    oc.cv.wait(lk, [&oc] { return oc.done; });
  }
  if (deleter) deleter(param);
  API_END();
}
}  // namespace

void MXKVB200EngineOnComplete(void* on_complete) {
  OnComplete* oc = static_cast<OnComplete*>(on_complete);
  if (oc == nullptr) return;
  std::lock_guard<std::mutex> lk(oc->mu);
  oc->done = true;
  oc->cv.notify_all();
}

int MXEnginePushAsync(EngineAsyncFunc async_func, void* func_param, EngineFuncParamDeleter deleter, ContextHandle,
                      EngineVarHandle, int, EngineVarHandle, int, EngineFnPropertyHandle, int, const char*, bool) {
  return RunAsync(async_func, func_param, deleter);
}
int MXEnginePushSync(EngineSyncFunc sync_func, void* func_param, EngineFuncParamDeleter deleter, ContextHandle,
                     EngineVarHandle, int, EngineVarHandle, int, EngineFnPropertyHandle, int, const char*) {
  return RunSync(sync_func, func_param, deleter);
}
int MXEnginePushAsyncND(EngineAsyncFunc async_func, void* func_param, EngineFuncParamDeleter deleter, ContextHandle,
                        NDArrayHandle*, int, NDArrayHandle*, int, EngineFnPropertyHandle, int, const char*, bool) {
  return RunAsync(async_func, func_param, deleter);
}
int MXEnginePushSyncND(EngineSyncFunc sync_func, void* func_param, EngineFuncParamDeleter deleter, ContextHandle,
                       NDArrayHandle*, int, NDArrayHandle*, int, EngineFnPropertyHandle, int, const char*) {
  return RunSync(sync_func, func_param, deleter);
}

int MXKVB200SetStream(int dev_id, void* cuda_stream) {
  API_BEGIN();
  Runtime::Get()->SetUserStream(dev_id, static_cast<cudaStream_t>(cuda_stream));
  API_END();
}

int MXKVB200GetEngineStream(int dev_id, void** out) {
  API_BEGIN();
  *out = Runtime::Get()->Dev(dev_id).stream;
  API_END();
}

int MXKVB200SetAutoFence(int auto_fence) {
  API_BEGIN();
  Runtime::Get()->auto_fence = auto_fence != 0;
  API_END();
}

int MXKVB200Fence(int dev_id) {
  API_BEGIN();
  FlushAllDeferred();      // deferred pushes may read or write this array
  Runtime::Get()->Fence(dev_id);
  API_END();
}

int MXKVB200GetLaunchCount(int64_t* out) {
  API_BEGIN();
  *out = Runtime::Get()->launches;
  API_END();
}

int MXKVB200SetDeferred(KVStoreHandle handle, int on) {
  API_BEGIN();
  KV(handle)->SetDeferred(on != 0);
  API_END();
}

int MXKVB200Flush(KVStoreHandle handle) {
  API_BEGIN();
  KV(handle)->Flush();
  API_END();
}

int MXKVB200GetDeferredBatches(KVStoreHandle handle, int64_t* out) {
  API_BEGIN();
  *out = KV(handle)->deferred_batches();
  API_END();
}

int MXKVB200GetPlanHits(KVStoreHandle handle, int64_t* out) {
  API_BEGIN();
  *out = static_cast<KVStore*>(handle)->plan_hits();
  API_END();
}

int MXKVB200GetVariantLaunchCount(int variant, int64_t* out) {
  API_BEGIN();
  MXKV_CHECK(variant >= 0 && variant < 4) << "variant: 0 per-thread, 1 staged (bulk), 2 multicast (NVLS), 3 tree order";
  *out = Runtime::Get()->variant_launches[variant];
  API_END();
}

int MXKVB200SetTuning(int64_t chunk_elems, int threads, int max_blocks, int bulk) {
  API_BEGIN();
  Runtime::Get()->SetTuning(chunk_elems, threads, max_blocks, bulk);
  API_END();
}

int MXKVB200SetTwoShotBytes(int64_t bytes) {
  API_BEGIN();
  Runtime::Get()->twoshot_bytes = bytes;
  Runtime::Get()->tuning_epoch++;
  API_END();
}

int MXKVB200ShardRange(int64_t size, int world, int rank, int64_t* begin, int64_t* end) {
  API_BEGIN();
  MXKV_CHECK(world >= 1 && rank >= 0 && rank < world && size >= 0) << "bad shard query";
  const int64_t L = ShardLen(size, world);
  *begin = std::min<int64_t>(size, L * rank);
  *end = std::min<int64_t>(size, L * (rank + 1));
  API_END();
}

int MXKVB200CommInit(int rank, int world, int dev_id, MXKVB200AllGatherFn allgather, void* ctx) {
  API_BEGIN();
  Runtime::Get()->InitProcessGroup(rank, world, dev_id, reinterpret_cast<AllGatherFn>(allgather), ctx);
  API_END();
}

int MXKVB200CommDestroy(void) {
  API_BEGIN();
  Runtime::Get()->DestroyProcessGroup();
  Runtime::Get()->hier = Hierarchy();
  API_END();
}

int MXKVB200SetHierarchy(int node_rank, int num_nodes, MXKVB200AllReduceFn allreduce, void* ctx) {
  API_BEGIN();
  MXKV_CHECK(num_nodes >= 1 && node_rank >= 0 && node_rank < num_nodes) << "bad node rank " << node_rank << " of "
                                                                        << num_nodes;
  MXKV_CHECK(allreduce != nullptr || num_nodes == 1) << "a multi-node hierarchy needs an all-reduce callback";
  Runtime* rt = Runtime::Get();
  MXKV_CHECK(rt->pg() != nullptr) << "MXKVB200CommInit (the node-local group) comes first";
  rt->tuning_epoch++;
  rt->hier.node_rank = node_rank;
  rt->hier.num_nodes = num_nodes;
  rt->hier.fn = reinterpret_cast<AllReduceFn>(allreduce);
  rt->hier.ctx = ctx;
  API_END();
}

int MXKVB200NDArrayCreateSymmetric(const int64_t* shape, int ndim, int dtype, NDArrayHandle* out) {
  API_BEGIN();
  ProcessGroup* pg = Runtime::Get()->pg();
  std::vector<int64_t> s(shape, shape + ndim);
  const int dev = pg ? pg->dev() : 0;
  *out = new NDHandle(NDArray::Empty(s, Context{kGPU, dev}, dtype, /*symmetric=*/pg != nullptr));
  API_END();
}


// ---- MXNET_KVSTORE_USETREE: the solver's pieces (topology.h) ------------------------------------------------
static std::vector<float> LinkMatrixArg(const float* w, int n) {
  MXKV_CHECK(n >= 1 && n <= 64 && w != nullptr) << "link matrix of " << n << " GPUs";
  return std::vector<float>(w, w + static_cast<size_t>(n) * n);
}

int MXKVB200TopologyLinkWeights(int n, const int* perf_rank, const int* can_access, float* out) {
  API_BEGIN();
  MXKV_CHECK(n >= 1 && n <= 64);
  const size_t nn = static_cast<size_t>(n) * n;
  const std::vector<float> W = topo::LinkWeights(n, std::vector<int>(perf_rank, perf_rank + nn),
                                                 std::vector<int>(can_access, can_access + nn));
  std::copy(W.begin(), W.end(), out);
  API_END();
}

int MXKVB200TopologyQueryLinks(int n, const int* devs, float* out) {
  API_BEGIN();
  MXKV_CHECK(n >= 1 && n <= 64);
  const std::vector<float> W = topo::QueryLinkWeights(std::vector<int>(devs, devs + n));
  std::copy(W.begin(), W.end(), out);
  API_END();
}

int MXKVB200TopologyComputeTrees(const float* weights, int n, float alpha, int backtrack, uint64_t* topo_out, int topo_cap,
                                 int* topo_len, uint64_t* scan_out, int scan_cap, int* scan_len, int* depth) {
  API_BEGIN();
  topo::TreeSet ts;
  topo::ComputeTrees(LinkMatrixArg(weights, n), n, alpha, backtrack != 0, &ts);
  const size_t tl = ts.topo[0].size(), sl = ts.scan[0].size();
  MXKV_CHECK(static_cast<size_t>(topo_cap) >= tl * n && static_cast<size_t>(scan_cap) >= sl * n) << "output too small";
  for (int r = 0; r < n; ++r) {
    MXKV_CHECK(ts.topo[r].size() == tl && ts.scan[r].size() == sl) << "trees of different depth";
    std::copy(ts.topo[r].begin(), ts.topo[r].end(), topo_out + r * tl);
    std::copy(ts.scan[r].begin(), ts.scan[r].end(), scan_out + r * sl);
  }
  *topo_len = static_cast<int>(tl);
  *scan_len = static_cast<int>(sl);
  *depth = ts.depth;
  API_END();
}

int MXKVB200TopologyBisect(const float* weights, int n, int* partition, int* num_partitions, int* pairs_out, int pairs_cap,
                           int* n_pairs, uint32_t seed, int* stop) {
  API_BEGIN();
  std::vector<int> color(partition, partition + n);
  std::vector<std::pair<int, int>> pairs;
  std::mt19937 gen(seed);
  *stop = topo::BisectClusters(LinkMatrixArg(weights, n), &color, num_partitions, &pairs, &gen) ? 1 : 0;
  MXKV_CHECK(static_cast<int>(pairs.size()) <= pairs_cap);
  std::copy(color.begin(), color.end(), partition);
  for (size_t i = 0; i < pairs.size(); ++i) { pairs_out[2 * i] = pairs[i].first; pairs_out[2 * i + 1] = pairs[i].second; }
  *n_pairs = static_cast<int>(pairs.size());
  API_END();
}

int MXKVB200TopologyFoldRepeats(int* leaves, int len, int n, int depth) {
  API_BEGIN();
  std::vector<int> r(leaves, leaves + len);
  topo::FoldRepeats(&r, n, depth);
  std::copy(r.begin(), r.end(), leaves);
  API_END();
}

int MXKVB200TopologyTreeWeight(const float* weights, const int* leaves, int len, int n, int depth, int penalty, float* out) {
  API_BEGIN();
  *out = topo::TreeWeight(LinkMatrixArg(weights, n), std::vector<int>(leaves, leaves + len), n, depth, penalty != 0);
  API_END();
}

int MXKVB200TopologyAdmissible(const float* weights, const int* state, int len, int n, int row, int depth, int* out) {
  API_BEGIN();
  *out = topo::Admissible(LinkMatrixArg(weights, n), std::vector<int>(state, state + len), n, row, depth) ? 1 : 0;
  API_END();
}

int MXKVB200TopologyConnected(const float* weights, int n, int* out) {
  API_BEGIN();
  *out = topo::LinksConnected(LinkMatrixArg(weights, n), n) ? 1 : 0;
  API_END();
}

int MXKVB200TopologyReduceProgram(const uint64_t* topo_row, int topo_len, const uint64_t* scan_row, int scan_len, int n,
                                  int* leaves_out, uint32_t* prog_out) {
  API_BEGIN();
  const topo::ReduceProgram rp = topo::ReduceProgramOf(std::vector<size_t>(topo_row, topo_row + topo_len),
                                                       std::vector<size_t>(scan_row, scan_row + scan_len), scan_len - 2, n);
  for (int i = 0; i < rp.n; ++i) leaves_out[i] = rp.leaf[i];
  *prog_out = rp.prog;
  API_END();
}

int MXKVB200TopologyRunProgram(const float* const* srcs, int n, uint32_t prog, int64_t count, float* out) {
  API_BEGIN();
  MXKV_CHECK(n >= 1 && n <= kMaxRanks);
  for (int64_t e = 0; e < count; ++e) {
    TreeSum<float, 1> ts;
    ts.begin(prog);
    for (int k = 0; k < n; ++k) {
      const float x[1] = {srcs[k][e]};
      ts.take(x, TreeAddF32());
    }
    float y[1];
    ts.result(y);
    out[e] = y[0];
  }
  API_END();
}

}  // extern "C"
