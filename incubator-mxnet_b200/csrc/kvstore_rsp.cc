// kvstore_rsp.cc -- row_sparse push / row_sparse_pull of KVStoreLocal on the H100 kernels.
//
// Reference: CommDevice::ReduceRowSparse (src/kvstore/comm.h:479-502) copies every row_sparse
// source to one GPU and calls the row_sparse ElementwiseSum; the updater then runs a sparse
// optimizer op; PullRowSparseImpl (src/kvstore/kvstore_local.h:316-336) = Unique(row_ids) +
// BroadcastRowSparse (comm.h:627-683: SparseRetain + copy).
//
// Here the stored value of a row_sparse key is a dense-backed table [num_rows x row_len] on
// every participating GPU (absent rows are zero rows, which is what SparseRetain returns for
// them).  A push runs the nnz-proportional union + gather-sum + lazy-update kernels
// (rsp_kernels.cu) on every replica's GPU, reading all sources in place (peer loads); nothing is
// copied to a root and nothing synchronises with the host.  row_sparse_pull sorts/uniques the ids
// in one block and gathers rows from the local replica.
#include <algorithm>
#include <cstring>
#include <set>
#include "kvstore.h"
#include "rsp_kernels.h"

namespace mxkv {

namespace {
inline bool Aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

void CheckLaunch(int rc, const char* what) {
  MXKV_CHECK(rc == 0) << what << " launch failed: " << cudaGetErrorString(static_cast<cudaError_t>(rc));
  Runtime::Get()->launches++;
}

}  // namespace

// make sure the device scalar of a row_sparse array mirrors its host-known row count
static void PublishNnz(const NDArray& a) {
  const int64_t n = a.nnz();   // host value (syncs only if it was device-only)
  const Context c = a.ctx();
  if (c.is_gpu()) {
    DeviceGuard g(c.dev_id);
    CheckLaunch(LaunchSetI64(a.d_nnz(), n, Runtime::Get()->Dev(c.dev_id).stream), "set_nnz");
  } else {
    *a.d_nnz() = n;
  }
}

void KVStore::InitRowSparseKey(KeyState& ks, const NDArray& v) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  MXKV_CHECK(v.dtype() == kFloat32) << "row_sparse keys support float32 only";
  MXKV_CHECK(!v.shape().empty()) << "row_sparse keys need at least 1 dimension";
  const Context c = v.ctx();
  const int dev = pg ? pg->dev() : (c.is_gpu() ? c.dev_id : DefaultDevice());
  if (c.is_gpu()) rt->AcquireUser(c.dev_id);
  Replica r;
  r.dev = dev;
  r.local = NDArray::Empty(ks.shape, Context{kGPU, dev}, kFloat32, pg != nullptr);
  DeviceGuard g(dev);
  cudaStream_t s = rt->Dev(dev).stream;
  CUDA_CALL(cudaMemsetAsync(r.local.data(), 0, r.local.nbytes(), s));
  const int64_t nnz = v.nnz();
  const int64_t L = v.row_len();
  if (nnz > 0) {
    const int64_t* idx = v.idx_ptr();
    const float* val = static_cast<const float*>(v.data());
    void* tmp_idx = nullptr; void* tmp_val = nullptr; int64_t* tmp_nnz = nullptr;
    CUDA_CALL(cudaMallocAsync(reinterpret_cast<void**>(&tmp_nnz), 16, s));
    CheckLaunch(LaunchSetI64(tmp_nnz, nnz, s), "set_nnz");
    if (!(c.is_gpu() && c.dev_id == dev)) {
      CUDA_CALL(cudaMallocAsync(&tmp_idx, nnz * 8, s));
      CUDA_CALL(cudaMallocAsync(&tmp_val, nnz * L * 4, s));
      CopyBytes(idx, c, tmp_idx, Context{kGPU, dev}, nnz * 8);
      CopyBytes(val, c, tmp_val, Context{kGPU, dev}, nnz * L * 4);
      idx = static_cast<const int64_t*>(tmp_idx);
      val = static_cast<const float*>(tmp_val);
    }
    CheckLaunch(LaunchRspScatter(static_cast<float*>(r.local.data()), idx, tmp_nnz, nnz, L, val, s), "rsp_scatter");
    if (tmp_idx) CUDA_CALL(cudaFreeAsync(tmp_idx, s));
    if (tmp_val) CUDA_CALL(cudaFreeAsync(tmp_val, s));
    CUDA_CALL(cudaFreeAsync(tmp_nnz, s));
  }
  ks.reps.push_back(r);
  if (pg && pg->world() > 1) BroadcastFromRank0(ks, ks.reps.back());
  if (pg && hier_) {              // every node adopts node 0's table (see InitImpl)
    Replica& me = ks.reps.back();
    if (rt->hier.node_rank != 0) CUDA_CALL(cudaMemsetAsync(me.local.data(), 0, me.local.nbytes(), s));
    InterNodeSum(me.local.data(), ks.size, kFloat32, dev);
  }
  rt->WaitDevice(dev);            // the host-side source may be released by the caller
  rt->ReleaseToUser(dev);
}

static void EnsureRspWorkspace(KeyState& ks, Replica& r, int n, int64_t cap) {
  if (r.rsp_n >= n && r.rsp_cap >= cap && !r.rsp_merged.is_none()) return;
  const Context ctx{kGPU, r.dev};
  n = std::max(n, r.rsp_n);
  cap = std::max<int64_t>(std::max<int64_t>(cap, r.rsp_cap), 16);
  r.rsp_first = NDArray::Empty({static_cast<int64_t>(n) * cap}, ctx, kInt32);
  r.rsp_pf = NDArray::Empty({static_cast<int64_t>(n) * (cap + 1)}, ctx, kInt32);
  r.rsp_merged = NDArray::EmptyRowSparse(ks.shape, ctx, kFloat32, static_cast<int64_t>(n) * cap);
  r.rsp_merged.set_nnz_device();
  r.rsp_n = n;
  r.rsp_cap = cap;
}

// source k of the row kernels on GPU dev: the value in place where dev can read it (after its own GPU's stream), else
// -- host-resident, or on a GPU without peer access -- staged on dev in cudaMallocAsync temporaries (ids, rows, device
// row count) that the caller frees after the launches
static void SourceOn(RspSources& S, int k, const NDArray& v, int64_t L, int dev, std::vector<void*>& temps) {
  Runtime* rt = Runtime::Get();
  const Context c = v.ctx();
  if (c.is_gpu() && (c.dev_id == dev || rt->PeerOK(dev, c.dev_id))) {
    if (c.dev_id != dev) rt->StreamWait(dev, c.dev_id);
    S.idx[k] = v.idx_ptr();
    S.val[k] = static_cast<const float*>(v.data());
    S.nnz[k] = v.d_nnz();
    return;
  }
  cudaStream_t s = rt->Dev(dev).stream;
  const int64_t nnz = v.nnz();
  void* ti = nullptr; void* tv = nullptr; int64_t* tn = nullptr;
  CUDA_CALL(cudaMallocAsync(&ti, std::max<int64_t>(nnz, 1) * 8, s));
  CUDA_CALL(cudaMallocAsync(&tv, std::max<int64_t>(nnz * L, 1) * 4, s));
  CUDA_CALL(cudaMallocAsync(reinterpret_cast<void**>(&tn), 16, s));
  if (nnz > 0) {
    CopyBytes(v.idx_ptr(), c, ti, Context{kGPU, dev}, nnz * 8);
    CopyBytes(v.data(), c, tv, Context{kGPU, dev}, nnz * L * 4);
  }
  CheckLaunch(LaunchSetI64(tn, nnz, s), "set_nnz");
  temps.push_back(ti); temps.push_back(tv); temps.push_back(tn);
  S.idx[k] = static_cast<const int64_t*>(ti);
  S.val[k] = static_cast<const float*>(tv);
  S.nnz[k] = tn;
}

// a key initialised dense that receives row_sparse values
void KVStore::RowSparseKeyFor(KeyState& ks) {
  if (ks.stype == kRowSparseStorage) return;
  MXKV_CHECK(ks.dtype == kFloat32 && !ks.shape.empty()) << "row_sparse values need a float32 key (key " << ks.key << ")";
  if (ks.local_world > 0) GatherLocal(ks);
  if (updater_ == nullptr && !opt_.enabled) {
    // Without an updater the stored value simply becomes the merged value, storage type included
    // (`local = merged.Copy(...)` on a storage-type mismatch, kvstore_local.h:268-276; the reference's
    // test_aggregator pushes row_sparse values to keys initialised dense).  The stored value is a
    // dense-backed table either way, so the key only changes its label.
    ks.stype = kRowSparseStorage;
    return;
  }
  // Dense weight, row_sparse gradient (gluon Parameter(grad_stype='row_sparse') updated on the store,
  // trainer.py:204-236; SGDUpdateDnsRspImpl / AdamLazyUpdate..., optimizer_op-inl.h:471-555,1305-1516):
  // the updater sees (merged row_sparse, stored dense) and the key stays dense.  The rows are updated
  // on every replica, each with its own complete optimizer state.
  if (opt_.enabled && updater_ == nullptr && ks.state_world > 0) {
    GatherState(ks);
    ks.state_world = 0;
    ks.state_devs.clear();
  }
}

// true: the store's optimizer updates the rows (no Python updater)
bool KVStore::RowSparseFused() const {
  const bool fused = opt_.enabled && updater_ == nullptr;
  if (fused)
    MXKV_CHECK(opt_.kind == OPT_SGD || opt_.kind == OPT_SGD_MOM || opt_.kind == OPT_ADAM)
        << "row_sparse gradients: only the lazy SGD / SGD-momentum / Adam updates are fused";
  return fused;
}

// One process per GPU: this rank's gradient v goes to r's symmetric staging area (allocated on first use), where every
// rank reads it; returns every rank's staging area as the sources.  Peers may still be reading the area of the previous
// push, so a barrier comes first unless that push ended with one (the fused kernel's: rsp_stage_guarded).  `fill`:
// copy v in and publish its row count behind a second barrier; otherwise the fused kernel does both.
RspSources KVStore::PublishRowSparse(const KeyState& ks, Replica& r, const NDArray& v, bool fill) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  const int64_t L = ks.size / ks.shape[0];
  const int64_t stage_rows = std::min<int64_t>(ks.shape[0], EnvInt("MXKV_B200_RSP_STAGE_ROWS", 131072));
  if (r.stage_idx.is_none()) {
    const Context ctx{kGPU, r.dev};
    r.stage_idx = NDArray::Empty({stage_rows}, ctx, kInt64, true);
    r.stage_val = NDArray::Empty({stage_rows * L}, ctx, kFloat32, true);
    r.stage_nnz = NDArray::Empty({2}, ctx, kInt64, true);
  }
  MXKV_CHECK(v.nnz() <= r.stage_idx.size())
      << "row_sparse gradient with " << v.nnz() << " rows exceeds the staging capacity of "
      << r.stage_idx.size() << " rows; raise MXKV_B200_RSP_STAGE_ROWS";
  DeviceGuard g(r.dev);
  cudaStream_t s = rt->Dev(r.dev).stream;
  SyncArgs sync = GroupSync(SYNC_WRITE_PEERS);
  sync.epoch = rt->NextSyncEpoch(pg);
  if (fill || !r.rsp_stage_guarded) CheckLaunch(LaunchBarrier(sync, s), "barrier");
  if (fill) {
    if (v.nnz() > 0) {
      CopyBytes(v.idx_ptr(), v.ctx(), r.stage_idx.data(), r.stage_idx.ctx(), v.nnz() * 8);
      CopyBytes(v.data(), v.ctx(), r.stage_val.data(), r.stage_val.ctx(), v.nnz() * L * 4);
    }
    CheckLaunch(LaunchSetI64(static_cast<int64_t*>(r.stage_nnz.data()), v.nnz(), s), "set_nnz");
    sync.epoch = rt->NextSyncEpoch(pg);
    CheckLaunch(LaunchBarrier(sync, s), "barrier");
  }
  r.rsp_stage_guarded = !fill;      // the fused kernel ends with a cross-GPU barrier
  RspSources S;
  std::memset(&S, 0, sizeof(S));
  S.n = pg->world();
  for (int q = 0; q < S.n; ++q) {
    S.idx[q] = static_cast<const int64_t*>(r.stage_idx.peer_data(q));
    S.val[q] = static_cast<const float*>(r.stage_val.peer_data(q));
    S.nnz[q] = static_cast<const int64_t*>(r.stage_nnz.peer_data(q));
  }
  return S;
}

// The row kernels' arguments on replica r over sources S.  `merge`: the union (and, unless the rows are updated lazily,
// the summed rows) goes to r's merge workspace.  `update`: the store's optimizer with r's state -- lazily on the touched
// rows (lazy_update), else afterwards over the whole table (MergeRows).  `assign`: the merged rows replace the table.
RspRowArgs KVStore::RowArgs(const KeyState& ks, const Replica& r, const RspSources& S, bool merge, bool update,
                            bool assign) const {
  const bool lazy = update && opt_.lazy_update;
  RspRowArgs A;
  std::memset(&A, 0, sizeof(A));
  if (merge) {
    A.out_idx = r.rsp_merged.idx_ptr();
    A.out_val = lazy ? nullptr : static_cast<float*>(r.rsp_merged.data());
    A.d_nnz_out = r.rsp_merged.d_nnz();
  }
  A.table = static_cast<float*>(r.local.data());
  A.row_len = ks.size / ks.shape[0];
  A.opt = lazy ? opt_.kind : OPT_NONE;
  A.assign = assign ? 1 : 0;
  A.rescale = opt_.rescale; A.clip = opt_.clip; A.momentum = opt_.momentum;
  A.beta1 = static_cast<float>(opt_.beta1); A.beta2 = static_cast<float>(opt_.beta2); A.eps = opt_.eps;
  if (update) {
    A.lr = ks.step.lr; A.wd = ks.step.wd;
    A.s0 = r.s0.is_none() ? nullptr : static_cast<float*>(r.s0.data());
    A.s1 = r.s1.is_none() ? nullptr : static_cast<float*>(r.s1.data());
  }
  bool vec = (A.row_len % 4 == 0) && Aligned16(A.table) && (A.out_val == nullptr || Aligned16(A.out_val)) &&
             (A.s0 == nullptr || Aligned16(A.s0)) && (A.s1 == nullptr || Aligned16(A.s1));
  for (int k = 0; k < S.n; ++k) vec = vec && Aligned16(S.val[k]);
  A.vec = vec ? 1 : 0;
  return A;
}

// The union + gather-sum kernels over sources S (up to `cap` rows each) on replica r, into its merge workspace, with
// RowArgs' update / assignment; an update without lazy_update then runs the reference's standard update.
void KVStore::MergeRows(KeyState& ks, Replica& r, const RspSources& S, int64_t cap, bool update, bool assign) {
  Runtime* rt = Runtime::Get();
  cudaStream_t s = rt->Dev(r.dev).stream;
  EnsureRspWorkspace(ks, r, S.n, cap);
  const RspRowArgs A = RowArgs(ks, r, S, true, update, assign);
  // push without updater: local = merged (kvstore_local.h:279-284) -- rows outside the union vanish
  if (assign) CUDA_CALL(cudaMemsetAsync(r.local.data(), 0, r.local.nbytes(), s));
  CheckLaunch(LaunchRspSum(S, A, static_cast<int32_t*>(r.rsp_first.data()), static_cast<int32_t*>(r.rsp_pf.data()),
                           r.rsp_cap, s), "rsp_sum");
  rt->launches += 3;
  r.rsp_merged.set_nnz_device();
  if (update && !opt_.lazy_update) {
    // densify the merged gradient (absent rows = 0) and run the dense kernel with the reference's
    // "Std" arithmetic over the whole table: O(table), as in the reference
    float* gd = nullptr;
    CUDA_CALL(cudaMallocAsync(reinterpret_cast<void**>(&gd), static_cast<size_t>(ks.size) * 4, s));
    CUDA_CALL(cudaMemsetAsync(gd, 0, static_cast<size_t>(ks.size) * 4, s));
    CheckLaunch(LaunchRspScatter(gd, r.rsp_merged.idx_ptr(), r.rsp_merged.d_nnz(), r.rsp_merged.cap_rows(), A.row_len,
                                 static_cast<const float*>(r.rsp_merged.data()), s), "rsp_scatter");
    TensorWork tw = ReplicaWork(ks, r, true, false, 0, ks.size);
    tw.src[0] = gd; tw.n_src = 1;
    tw.out[0] = r.local.data(); tw.n_out = 1;
    tw.flags = ks.size % 4 == 0 ? WorkFlags(tw, false) : 0;   // (tables of other sizes keep the scalar path)
    const int kind = opt_.kind == OPT_SGD ? OPT_SGD_STD : (opt_.kind == OPT_ADAM ? OPT_ADAM_STD : opt_.kind);
    LaunchLocal(LaunchClassKey{SYNC_NONE, kFloat32, 0}, tw, kind, r.dev);
    CUDA_CALL(cudaFreeAsync(gd, s));
  }
}

void KVStore::PushRowSparse(KeyState& ks, const std::vector<NDArray>& vals) {
  if (hier_) { HierPushRowSparse(ks, vals); return; }
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  const bool mp_mode = pg != nullptr;
  RowSparseKeyFor(ks);
  const int n_src = static_cast<int>(vals.size());
  MXKV_CHECK(n_src >= 1 && n_src <= kMaxSrc) << "push of " << n_src << " row_sparse values (max " << kMaxSrc << ")";
  const int64_t L = ks.size / ks.shape[0];
  int64_t cap = 0;
  for (auto& v : vals) {
    MXKV_CHECK(v.stype() == kRowSparseStorage) << "mixing dense and row_sparse values in one push is not supported";
    MXKV_CHECK(v.dtype() == kFloat32 && v.shape() == ks.shape) << "row_sparse push: shape/dtype mismatch";
    cap = std::max(cap, v.nnz());
  }
  const bool callback = updater_ != nullptr;
  const bool fused = RowSparseFused();

  // ---- which GPUs compute (each one redundantly, on its own replica) -------------------------
  std::vector<int> work_devs;
  std::set<int> touched;
  auto touch = [&](int dev) { if (dev >= 0 && touched.insert(dev).second) rt->AcquireUser(dev); };
  if (mp_mode) {
    MXKV_CHECK(n_src == 1) << "one-process-per-GPU mode: push exactly one value per key per rank";
    work_devs.push_back(pg->dev());
  } else {
    for (auto& r : ks.reps) work_devs.push_back(r.dev);
    for (auto& v : vals) {
      const Context c = v.ctx();
      if (c.is_gpu() && std::find(work_devs.begin(), work_devs.end(), c.dev_id) == work_devs.end())
        work_devs.push_back(c.dev_id);
    }
    if (work_devs.empty()) work_devs.push_back(DefaultDevice());
    rt->EnablePeerAccess(work_devs);
  }
  // One launch instead of nine when the merged value itself is not needed (lazy fused update): publish, union,
  // gather-sum and update in rsp_push_fused_kernel
  const bool fused_path = fused && opt_.lazy_update && EnvInt("MXKV_B200_RSP_FUSED", 1) != 0;
  for (auto& v : vals) {
    if (v.ctx().is_gpu()) touch(v.ctx().dev_id);
    if (!fused_path) PublishNnz(v);          // (the fused kernel takes the row counts by value)
  }
  for (int d : work_devs) { touch(d); EnsureReplica(ks, d); }
  if (fused) {
    // optimizer state of every computing replica, brought up to date BEFORE this update is counted or any
    // replica has run it (a replica whose GPU sat out earlier dense updates takes over a participant's state)
    for (int d : work_devs) {
      Replica& r = *FindReplica(ks, d);
      EnsureState(ks, r, false);
    }
    for (int d : work_devs) SyncState(ks, *FindReplica(ks, d));
    for (auto& r : ks.reps)
      if (std::find(work_devs.begin(), work_devs.end(), r.dev) == work_devs.end()) r.state_fresh = false;
  }

  if (fused) StepKey(ks);

  // ---- MP: publish this rank's gradient in the symmetric staging area ---------------------------
  const int world = mp_mode ? pg->world() : 1;
  RspSources staged{};
  if (world > 1) {
    Replica& r = *FindReplica(ks, pg->dev());
    staged = PublishRowSparse(ks, r, vals[0], !fused_path);
    cap = r.stage_idx.size();
  }

  // ---- per computing GPU: sources as seen from it, then the kernels ----------------------------
  for (int dev : work_devs) {
    Replica& r = *FindReplica(ks, dev);
    DeviceGuard g(dev);
    cudaStream_t s = rt->Dev(dev).stream;
    std::vector<void*> temps;
    RspSources S = staged;
    if (world == 1) {
      S.n = n_src;
      for (int k = 0; k < n_src; ++k) SourceOn(S, k, vals[k], L, dev, temps);
    }
    if (fused_path) {
      RspRowArgs A = RowArgs(ks, r, S, false, true, false);    // (no union is materialised)
      RspStage St;
      std::memset(&St, 0, sizeof(St));
      const SyncArgs sync = world > 1 ? GroupSync(SYNC_WRITE_PEERS) : LocalSync(dev);
      int64_t est_rows = 0;
      void* tmp_src[2] = {nullptr, nullptr};
      if (world > 1) {
        const NDArray& v = vals[0];
        St.publish = 1;
        St.src_idx = v.idx_ptr();
        St.src_val = static_cast<const float*>(v.data());
        St.src_nnz = v.nnz();
        if (!(v.ctx().is_gpu() && v.ctx().dev_id == dev) && v.nnz() > 0) {      // host-resident gradient: one hop first
          CUDA_CALL(cudaMallocAsync(&tmp_src[0], v.nnz() * 8, s));
          CUDA_CALL(cudaMallocAsync(&tmp_src[1], v.nnz() * L * 4, s));
          CopyBytes(v.idx_ptr(), v.ctx(), tmp_src[0], Context{kGPU, dev}, v.nnz() * 8);
          CopyBytes(v.data(), v.ctx(), tmp_src[1], Context{kGPU, dev}, v.nnz() * L * 4);
          St.src_idx = static_cast<const int64_t*>(tmp_src[0]);
          St.src_val = static_cast<const float*>(tmp_src[1]);
        }
        St.dst_idx = static_cast<int64_t*>(r.stage_idx.data());
        St.dst_val = static_cast<float*>(r.stage_val.data());
        St.dst_nnz = static_cast<int64_t*>(r.stage_nnz.data());
        St.localize = 1;
        est_rows = std::max<int64_t>(v.nnz(), 1) * world;
        A.vec = (A.vec && Aligned16(St.src_val) && Aligned16(St.dst_val)) ? 1 : 0;
      } else {
        St.nnz_by_value = 1;
        for (int k = 0; k < n_src; ++k) {
          const Context c = vals[k].ctx();
          if (c.is_gpu() && c.dev_id != dev && S.idx[k] == vals[k].idx_ptr()) St.localize = 1;
          St.nnz_val[k] = vals[k].nnz();
          est_rows += vals[k].nnz();
        }
      }
      if (St.localize) {
        const int64_t lcap = std::max<int64_t>(cap, 16);
        if (r.rsp_lidx.is_none() || r.rsp_lidx_n < S.n || r.rsp_lidx_cap < lcap) {
          r.rsp_lidx_n = std::max(r.rsp_lidx_n, S.n);
          r.rsp_lidx_cap = std::max(r.rsp_lidx_cap, lcap);
          r.rsp_lidx = NDArray::Empty({static_cast<int64_t>(r.rsp_lidx_n) * r.rsp_lidx_cap}, Context{kGPU, dev}, kInt64);
        }
        St.lidx = static_cast<int64_t*>(r.rsp_lidx.data());
        St.lcap = r.rsp_lidx_cap;
      }
      CheckLaunch(LaunchRspPushFused(dev, S, A, St, sync, est_rows, s), "rsp_push_fused");
      for (void* t : tmp_src) if (t) CUDA_CALL(cudaFreeAsync(t, s));
    } else {
      MergeRows(ks, r, S, cap, fused, !fused && !callback);
    }
    for (void* t : temps) CUDA_CALL(cudaFreeAsync(t, s));
    r.fresh = true;
  }
  if (world > 1) {
    // nobody may overwrite its staging area while a peer is still reading it: the rendezvous at the
    // start of the next push (PublishRowSparse) provides that ordering
  } else {
    // sources on other GPUs were read by this GPU's kernels: they must not be reused earlier
    for (auto& v : vals) {
      const Context c = v.ctx();
      if (!c.is_gpu()) continue;
      for (int dev : work_devs) if (dev != c.dev_id) rt->StreamWait(c.dev_id, dev);
    }
  }
  if (callback) {
    Replica& root = *FindReplica(ks, work_devs[0]);
    RunCallbackUpdater(ks, root, root.rsp_merged);
  }
  for (int d : touched) rt->ReleaseToUser(d);
}

// Multi-node row_sparse push (KVStoreDist pushes the rows to the servers, which merge them and run the sparse
// update, kvstore_dist.h:343-470 / kvstore_dist_server.h).  Here: (1) the node's sorted-union merge of its ranks'
// gradients, as in the single-node path, materialised on every rank; (2) the nodes' merged gradients are
// gathered -- row counts first (one tiny inter-node sum, read back by the host, as the reference reads its row
// counts), then ids and rows in buffers sized for the largest node, each node filling its section and the
// others contributing zeros to the inter-node sum; (3) the same four kernels again with one source per node,
// this time applying the lazy / standard update (or the assignment) to the rows of this rank's replica.
// Association per row: rank order inside a node, then node order.
void KVStore::HierPushRowSparse(KeyState& ks, const std::vector<NDArray>& vals) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  MXKV_CHECK(pg != nullptr) << "multi-node stores run in one-process-per-GPU mode";
  MXKV_CHECK(updater_ == nullptr) << "dist_device_sync: row_sparse values with a Python updater are not supported";
  const int nodes = rt->hier.num_nodes, node = rt->hier.node_rank;
  MXKV_CHECK(nodes <= kMaxSrc) << "row_sparse push over " << nodes << " nodes (max " << kMaxSrc << ")";
  MXKV_CHECK(vals.size() == 1) << "one-process-per-GPU mode: push exactly one value per key per rank";
  const NDArray& v = vals[0];
  RowSparseKeyFor(ks);
  MXKV_CHECK(v.stype() == kRowSparseStorage && v.dtype() == kFloat32 && v.shape() == ks.shape)
      << "row_sparse push: storage type / shape / dtype mismatch for key " << ks.key;
  const bool fused = RowSparseFused();
  const int dev = pg->dev();
  const int64_t L = ks.size / ks.shape[0];
  DeviceGuard g(dev);
  cudaStream_t s = rt->Dev(dev).stream;
  rt->AcquireUser(dev);
  MXKV_CHECK(!v.ctx().is_gpu() || v.ctx().dev_id == dev) << "value must live on GPU " << dev << " or on the host";
  PublishNnz(v);
  Replica& r = EnsureReplica(ks, dev);
  if (fused) { EnsureState(ks, r, false); SyncState(ks, r); StepKey(ks); }
  std::vector<void*> temps;

  // ---- (1) the node's merge ---------------------------------------------------------------------------------
  RspSources S;
  int64_t cap = std::max<int64_t>(v.nnz(), 1);
  if (pg->world() > 1) {
    S = PublishRowSparse(ks, r, v, true);
    cap = r.stage_idx.size();
  } else {
    std::memset(&S, 0, sizeof(S));
    S.n = 1;
    SourceOn(S, 0, v, L, dev, temps);
  }
  MergeRows(ks, r, S, cap, false, false);

  // ---- (2) gather the nodes' merged gradients ------------------------------------------------------------------
  int64_t* cnt = nullptr;                  // [nodes] row counts, device
  CUDA_CALL(cudaMallocAsync(reinterpret_cast<void**>(&cnt), static_cast<size_t>(nodes) * 8, s));
  temps.push_back(cnt);
  CUDA_CALL(cudaMemsetAsync(cnt, 0, static_cast<size_t>(nodes) * 8, s));
  CUDA_CALL(cudaMemcpyAsync(cnt + node, r.rsp_merged.d_nnz(), 8, cudaMemcpyDeviceToDevice, s));
  InterNodeSum(cnt, nodes, kInt64, dev);
  std::vector<int64_t> counts(nodes);
  CUDA_CALL(cudaMemcpyAsync(counts.data(), cnt, static_cast<size_t>(nodes) * 8, cudaMemcpyDeviceToHost, s));
  CUDA_CALL(cudaStreamSynchronize(s));
  int64_t cap2 = 1;
  for (int64_t c : counts) cap2 = std::max(cap2, c);
  int64_t* idx_all = nullptr; float* val_all = nullptr;
  const size_t idx_bytes = static_cast<size_t>(nodes) * cap2 * 8;
  const size_t val_bytes = static_cast<size_t>(nodes) * cap2 * L * 4;
  CUDA_CALL(cudaMallocAsync(reinterpret_cast<void**>(&idx_all), idx_bytes, s));
  CUDA_CALL(cudaMallocAsync(reinterpret_cast<void**>(&val_all), val_bytes, s));
  temps.push_back(idx_all); temps.push_back(val_all);
  CUDA_CALL(cudaMemsetAsync(idx_all, 0, idx_bytes, s));
  CUDA_CALL(cudaMemsetAsync(val_all, 0, val_bytes, s));
  if (counts[node] > 0) {
    CUDA_CALL(cudaMemcpyAsync(idx_all + static_cast<size_t>(node) * cap2, r.rsp_merged.idx_ptr(),
                              static_cast<size_t>(counts[node]) * 8, cudaMemcpyDeviceToDevice, s));
    CUDA_CALL(cudaMemcpyAsync(val_all + static_cast<size_t>(node) * cap2 * L, r.rsp_merged.data(),
                              static_cast<size_t>(counts[node]) * L * 4, cudaMemcpyDeviceToDevice, s));
  }
  InterNodeSum(idx_all, static_cast<int64_t>(nodes) * cap2, kInt64, dev);
  InterNodeSum(val_all, static_cast<int64_t>(nodes) * cap2 * L, kFloat32, dev);

  // ---- (3) merge the nodes and update this rank's replica --------------------------------------------------------
  RspSources S2;
  std::memset(&S2, 0, sizeof(S2));
  S2.n = nodes;
  for (int q = 0; q < nodes; ++q) {
    S2.idx[q] = idx_all + static_cast<size_t>(q) * cap2;
    S2.val[q] = val_all + static_cast<size_t>(q) * cap2 * L;
    S2.nnz[q] = cnt + q;
  }
  MergeRows(ks, r, S2, cap2, fused, !fused);
  for (void* t : temps) CUDA_CALL(cudaFreeAsync(t, s));
  r.fresh = true;
  ks.local_world = 0;
  rt->ReleaseToUser(dev);
}

void KVStore::PullDenseFromRowSparse(KeyState& ks, const std::vector<NDArray*>& outs) {
  Runtime* rt = Runtime::Get();
  std::set<int> touched;
  for (NDArray* o : outs) {
    if (o->stype() == kRowSparseStorage) {
      // pull(..., ignore_sparse=False) into a row_sparse array: the whole stored value (CopyFromTo
      // rsp -> rsp in CommDevice::Broadcast, comm.h:607-625).  The stored value is a dense-backed
      // table, so every row is delivered (rows the reference would not list arrive as zero rows: the
      // dense view is identical).
      NDArray ids = NDArray::Empty({ks.shape[0]}, Context{kCPU, 0}, kInt64);
      int64_t* p = static_cast<int64_t*>(ids.data());
      for (int64_t i = 0; i < ks.shape[0]; ++i) p[i] = i;
      PullRowSparseImpl({ks.key}, {{o, ids}}, 0);
      continue;
    }
    MXKV_CHECK(o->size() == ks.size && o->dtype() == ks.dtype) << "pull: output does not match key " << ks.key;
    const Context c = o->ctx();
    if (c.is_gpu() && touched.insert(c.dev_id).second) rt->AcquireUser(c.dev_id);
    const bool local_dev = c.is_gpu() && (rt->pg() == nullptr || c.dev_id == rt->pg()->dev());
    Replica& r = local_dev ? EnsureReplica(ks, c.dev_id) : FreshReplica(ks);
    CopyFromTo(r.local.Reshape(o->shape()), *o);      // storage-type cast of CopyFromTo (ndarray.cc:1301-1327)
  }
  for (int d : touched) rt->ReleaseToUser(d);
}

void KVStore::PullRowSparseImpl(const std::vector<int>& keys,
                                const std::vector<std::pair<NDArray*, NDArray>>& vr, int priority) {
  (void)priority;
  MXKV_CHECK(keys.size() == vr.size()) << keys.size() << " keys but " << vr.size() << " values";
  Runtime* rt = Runtime::Get();
  std::set<int> touched;
  auto touch = [&](int dev) { if (dev >= 0 && touched.insert(dev).second) rt->AcquireUser(dev); };
  for (size_t i = 0; i < keys.size(); ++i) {
    NDArray* out = vr[i].first;
    const NDArray& row_id = vr[i].second;
    // GroupKVPairsPullRsp validator, kvstore_local.h:421-431
    MXKV_CHECK(out->stype() == kRowSparseStorage)
        << "Expected row_sparse storage type for row_sparse_pull values, but detected storage type " << out->stype();
    MXKV_CHECK(row_id.stype() == kDefaultStorage)
        << "Expected default storage type for row_sparse_pull rowids, but detected storage type " << row_id.stype();
    KeyState& ks = GetKey(keys[i]);
    MXKV_CHECK(ks.stype == kRowSparseStorage) << "PullRowSparse expects row_sparse src NDArray";
    MXKV_CHECK(row_id.dtype() == kInt64 || row_id.dtype() == kInt32 || row_id.dtype() == kFloat32 ||
               row_id.dtype() == kFloat64) << "row_ids must be int64, int32, float32 or float64";
    const int64_t n = row_id.size();
    const int64_t L = ks.size / ks.shape[0];
    const Context oc = out->ctx();
    const Context rc = row_id.ctx();
    int dev;
    if (rt->pg()) dev = rt->pg()->dev();
    else if (oc.is_gpu()) dev = oc.dev_id;
    else if (rc.is_gpu()) dev = rc.dev_id;
    else dev = FreshReplica(ks).dev;
    touch(dev);
    if (oc.is_gpu()) touch(oc.dev_id);
    if (rc.is_gpu()) touch(rc.dev_id);
    Replica& r = EnsureReplica(ks, dev);
    DeviceGuard g(dev);
    cudaStream_t s = rt->Dev(dev).stream;
    // ids on this GPU, as int64
    const int64_t* ids = static_cast<const int64_t*>(row_id.data());
    void* tmp_ids = nullptr;
    void* tmp_cast = nullptr;
    if (!(rc.is_gpu() && rc.dev_id == dev) && n > 0) {
      CUDA_CALL(cudaMallocAsync(&tmp_ids, row_id.nbytes(), s));
      CopyBytes(row_id.data(), rc, tmp_ids, Context{kGPU, dev}, row_id.nbytes());
      ids = static_cast<const int64_t*>(tmp_ids);
    }
    if (row_id.dtype() != kInt64 && n > 0) {
      CUDA_CALL(cudaMallocAsync(&tmp_cast, n * 8, s));
      CheckLaunch(LaunchCastIdsToI64(ids, row_id.dtype(), static_cast<int64_t*>(tmp_cast), n, s), "rsp_cast_ids");
      ids = static_cast<const int64_t*>(tmp_cast);
    }
    const bool direct = oc.is_gpu() && oc.dev_id == dev;
    if (direct && out->cap_rows() < n) out->ReserveRows(n);
    NDArray target = *out;
    if (!direct) target = NDArray::EmptyRowSparse(ks.shape, Context{kGPU, dev}, kFloat32, std::max<int64_t>(n, 1));
    MXKV_CHECK(target.cap_rows() >= n) << "row_sparse_pull: output holds " << target.cap_rows() << " rows, "
                                       << n << " row ids requested";
    MXKV_CHECK(target.dtype() == kFloat32) << "row_sparse_pull: float32 outputs only";
    const int vec = (L % 4 == 0 && Aligned16(r.local.data()) && Aligned16(target.data())) ? 1 : 0;
    if (n >= 1 && n <= RspUniqueMax() && EnvInt("MXKV_B200_RSP_FUSED", 1) != 0) {
      // unique | grid barrier | gather in one launch
      CheckLaunch(LaunchRspPullFused(dev, static_cast<const float*>(r.local.data()), ids, n, target.idx_ptr(),
                                     target.d_nnz(), L, static_cast<float*>(target.data()), vec, LocalSync(dev), s),
                  "rsp_pull_fused");
    } else {
      CheckLaunch(LaunchRspUnique(ids, n, target.idx_ptr(), target.d_nnz(), s), "rsp_unique");
      CheckLaunch(LaunchRspGather(static_cast<const float*>(r.local.data()), target.idx_ptr(), target.d_nnz(),
                                  std::max<int64_t>(n, 1), L, static_cast<float*>(target.data()), target.idx_ptr(),
                                  vec, s), "rsp_gather");
    }
    target.set_nnz_device();
    if (tmp_ids) CUDA_CALL(cudaFreeAsync(tmp_ids, s));
    if (tmp_cast) CUDA_CALL(cudaFreeAsync(tmp_cast, s));
    if (!direct) {
      const int64_t cnt = target.nnz();      // one sync: the destination lives elsewhere
      if (out->cap_rows() < cnt) out->ReserveRows(cnt);
      if (cnt > 0) {
        CopyBytes(target.idx_ptr(), target.ctx(), out->idx_ptr(), oc, cnt * 8);
        CopyBytes(target.data(), target.ctx(), out->data(), oc, cnt * L * 4);
      }
      out->set_nnz(cnt);
      if (oc.is_gpu()) PublishNnz(*out);
      rt->WaitDevice(dev);
    }
  }
  for (int d : touched) rt->ReleaseToUser(d);
}

}  // namespace mxkv
