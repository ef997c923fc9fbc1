// kvstore.h -- KVStoreLocal semantics (src/kvstore/kvstore_local.h:70-552) on top of
// the fused sm_90a reduce/update/broadcast kernel.
//
// What is kept from the reference: the API and its observable behaviour -- key
// bookkeeping (int or str keys, never mixed, :344-347), duplicate-init check (:230-233),
// sort-and-group of (key, value) pairs (:440-469), push = reduce (+ updater) into the
// stored value (:240-286), pull = copy the stored value out (:288-314), pushpull = push
// then pull (:358-365), broadcast = init then pull (:349-356), row_sparse_pull = unique +
// retain (:316-336), updater callback contract (c_api.cc:3066-3111).
//
// What is redesigned: instead of one merge buffer per key on a load-balanced root GPU
// (CommDevice::InitMergeBuffer, comm.h:687-725) fed by n peer copies, every participating
// GPU keeps a replica of the stored value and the reduce(+update)(+broadcast) of a whole
// list of keys is ONE kernel launch per GPU (kernels.cu).  Large keys are sharded across the
// GPUs (each reduces and updates 1/n and stores it to all replicas), small keys are reduced
// redundantly by everyone (one-shot).
#pragma once
#include <functional>
#include <map>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include "ndarray.h"
#include "rsp_kernels.h"
#include "topology.h"

namespace mxkv {

typedef void (*UpdaterFn)(int key, void* recv, void* local, void* handle);
typedef void (*StrUpdaterFn)(const char* key, void* recv, void* local, void* handle);

struct OptimizerConfig {
  int kind = OPT_NONE;
  bool enabled = false;
  // kept in double: the reference computes lr/wd multipliers and Adam's bias correction in
  // Python doubles and rounds to float once, when the value becomes an op attribute
  double lr = 0.01, wd = 0.0, beta1 = 0.9, beta2 = 0.999;
  float momentum = 0.f, eps = 1e-8f, eta = 1.f;
  double eta_d = 1.0;          // eta as given (AdamW multiplies it with the learning rate in double)
  float rescale = 1.f, clip = -1.f;
  bool multi_precision = false;
  bool lazy_update = false;   // row_sparse gradients: touch only the rows present (sgd.py:78, adam.py:77 default False)
  bool correct_bias = true;   // AdamW, AdaBelief (python/mxnet/optimizer/adamW.py:80-88, adabelief.py:79-87)
  float rho = 0.9f, clip_weights = -1.f;   // RMSProp (rmsprop.py:70-71); clip_weights < 0: off
  double rho_d = 0.9;         // rho as given (AdaDelta's 1 - rho is computed in double)
  double wd_lh = 0.0;         // Signum's decoupled weight decay (signum.py:67); double: signSGD adds it to wd in double
  // Nadam (nadam.py:58-67): the schedule decay, and the optimizer's ONE momentum-schedule product, which every fused
  // key update multiplies in call order (KVStore::StepKey)
  double schedule_decay = 0.004, m_schedule = 1.0;
  // LAMB / LANS / LARS (python/mxnet/optimizer/{lamb,lans,lars}.py)
  float lower_bound = -1.f, upper_bound = -1.f;   // bounds on the weight norm, < 0: not set
  bool bias_correction = true;                     // LAMB
  float lars_eta = 0.001f, lars_eps = 1e-8f;       // LARS trust coefficient and epsilon
  bool skip_nonfinite = false;   // leave weight/state untouched when a merged gradient of the call is not finite
  std::unordered_set<int> no_trust;   // LARS: keys named *gamma / *beta / *bias keep the plain learning rate
  std::unordered_map<int, double> lr_mult, wd_mult;
};

struct Replica {
  int dev = -1;
  NDArray local;     // the stored value, key dtype
  NDArray w32;       // fp32 master (multi precision)
  NDArray s0, s1, s2;  // optimizer state (kernels.h: OptHasS0 / OptHasS1 / OptHasS2)
  NDArray stage;     // MP mode: symmetric staging for non-symmetric gradients
  NDArray merged;    // updater-callback path: reduce target
  NDArray aux0, aux1;  // LAMB/LANS/LARS: fp32 temporaries between the phases (update direction / merged gradient)
  NDArray nrm;         // LAMB/LANS/LARS: this replica's per-key sums of squares (peer-visible)
  bool fresh = true;
  bool state_fresh = true;   // optimizer state (kReplicaState) reflects every update so far
  // row_sparse keys: `local` is the dense-backed table [num_rows x row_len]
  NDArray rsp_merged;            // union ids + summed rows of the last push (capacity n * rsp_cap rows)
  NDArray rsp_first, rsp_pf;     // int32 workspaces of the union kernels
  NDArray rsp_lidx;              // fused push: local copies of the sources' id lists [rsp_lidx_n x rsp_lidx_cap]
  int64_t rsp_lidx_cap = 0;
  int rsp_lidx_n = 0;
  bool rsp_stage_guarded = false;   // MP: the last push ended with a cross-GPU barrier (nobody reads the staging area)
  int64_t rsp_cap = 0;           // rows per source the workspaces are sized for
  int rsp_n = 0;
  NDArray stage_idx, stage_val, stage_nnz;   // MP mode: symmetric staging of this rank's gradient
};

// A replica's optimizer-state arrays in the numbering of MXKVB200GetState / SetState (which = 1 + index): the fp32
// master, state0, state1, state2.  Every copy, gather, reset and presence check of the state walks this one list.
typedef NDArray Replica::*ReplicaArray;
inline constexpr ReplicaArray kReplicaState[] = {&Replica::w32, &Replica::s0, &Replica::s1, &Replica::s2};
constexpr int kNumReplicaState = static_cast<int>(sizeof(kReplicaState) / sizeof(kReplicaState[0]));

// Every scalar one fused update of a key hands its kernels (KVStore::KeyScalars): TensorWork's lr / wd / eta,
// NormWork's lr_d and bias corrections c1 / c2, and Nadam's DenseLaunch::nadam entry (1 - m_schedule,
// 1 - m_schedule_next, momentum_t_1, 1 - momentum_t).
struct KeyStep {
  float lr = 0.f, wd = 0.f, eta = 0.f, c1 = 0.f, c2 = 0.f;
  double lr_d = 0.0;
  float4 nadam{1.f, 1.f, 0.f, 0.f};
};

struct KeyState {
  int key = 0;
  std::vector<int64_t> shape;
  int dtype = kFloat32;
  int stype = kDefaultStorage;
  int64_t size = 0;
  NDArray init_value;            // value handed to Init until a GPU replica exists (host memory)
  std::vector<Replica> reps;
  int64_t count = 0;             // Optimizer._index_update_count
  int state_world = 0;           // number of shards the optimizer state is laid out for (0: replicated/none)
  int local_world = 0;           // > 0: the stored value is valid shard-wise only (shard p on shard_devs[p])
  std::vector<int> shard_devs;   // devices (SP) / placeholder per rank (MP) of the shard owners
  std::vector<int> state_devs;   // the same for the optimizer-state shards (state_world entries)
  bool has_state = false;
  KeyStep step;                  // the scalars of this key's latest fused update, set when its count advances
  // Bumped by every access through KVStore::GetKey, i.e. by every operation that may change this key's
  // replicas / layout / state flags; a cached launch plan (kvstore.h: CallPlan) is valid only while the
  // epochs of its keys are the ones it was recorded with.
  uint64_t epoch = 0;
  // gradient compression: per pushed-value slot, error-feedback residual and the code stream
  std::vector<NDArray> gc_residual, gc_packed;
};

int64_t ShardLen(int64_t size, int world);

struct LaunchClassKey {
  int sync_mode, dtype, mp;
  int nvls = 0;      // 1: multicast (multimem) kernel
  int tree = 0;      // 1: sums in the order of a reduction tree (MXNET_KVSTORE_USETREE; tree_kernels.cu)
  bool operator<(const LaunchClassKey& o) const {
    if (sync_mode != o.sync_mode) return sync_mode < o.sync_mode;
    if (dtype != o.dtype) return dtype < o.dtype;
    if (mp != o.mp) return mp < o.mp;
    if (nvls != o.nvls) return nvls < o.nvls;
    return tree < o.tree;
  }
};

class KVStore {
 public:
  explicit KVStore(const std::string& type);
  ~KVStore();
  const std::string& type() const { return type_; }
  int rank() const;
  int group_size() const;

  void Init(const std::vector<int>& keys, const std::vector<NDArray>& vals);
  void Init(const std::vector<std::string>& keys, const std::vector<NDArray>& vals);
  void Push(const std::vector<int>& keys, const std::vector<NDArray>& vals, int priority);
  void Push(const std::vector<std::string>& keys, const std::vector<NDArray>& vals, int priority);
  void Pull(const std::vector<int>& keys, const std::vector<NDArray*>& outs, int priority, bool ignore_sparse);
  void Pull(const std::vector<std::string>& keys, const std::vector<NDArray*>& outs, int priority, bool ignore_sparse);
  void PushPull(const std::vector<int>& vkeys, const std::vector<int>& okeys, const std::vector<NDArray>& vals,
                const std::vector<NDArray*>& outs, int priority);
  void PushPull(const std::vector<std::string>& vkeys, const std::vector<std::string>& okeys,
                const std::vector<NDArray>& vals, const std::vector<NDArray*>& outs, int priority);
  void Broadcast(const std::vector<int>& vkeys, const std::vector<int>& okeys, const std::vector<NDArray>& vals,
                 const std::vector<NDArray*>& outs, int priority);
  void Broadcast(const std::vector<std::string>& vkeys, const std::vector<std::string>& okeys,
                 const std::vector<NDArray>& vals, const std::vector<NDArray*>& outs, int priority);
  void PullRowSparse(const std::vector<int>& keys, const std::vector<std::pair<NDArray*, NDArray>>& val_rowids,
                     int priority);
  void PullRowSparse(const std::vector<std::string>& keys,
                     const std::vector<std::pair<NDArray*, NDArray>>& val_rowids, int priority);

  // ---- deferred issue: what `priority` means on this engine -------------------------------------------------
  // The reference's engine runs the ops that are ready in priority order (threaded_engine_perdevice.cc:97-279;
  // the Trainer pushes parameter i with priority -i, gluon/trainer.py:386-409).  An in-order stream has no queue
  // to reorder, so the queue is kept here: with deferral on, push / pushpull calls (dense GPU values, integer
  // keys) are recorded instead of launched; Flush() -- explicit, or implied by any call that reads or changes
  // the store or waits for an array -- issues them highest priority first, never moving a call ahead of an
  // earlier one that shares a key with it (the engine's write-after-write order), and merges calls that are
  // adjacent in that order and touch disjoint keys into ONE launch (sequence).
  void SetDeferred(bool on);
  void Flush();
  int64_t deferred_batches() const { return deferred_batches_; }

  void SetUpdater(UpdaterFn fn, StrUpdaterFn sfn, void* handle);
  void SetGradientCompression(const std::vector<std::pair<std::string, std::string>>& kwargs);
  void Barrier();

  // fused optimizer (MXKVB200 extension; replaces the Python Updater round trip)
  void SetOptimizer(const std::string& name, const std::vector<std::pair<std::string, std::string>>& kwargs);
  void SetOptimizerMult(bool str_key, int ikey, const std::string& skey, float lr_mult, float wd_mult);
  // type 'updater' only: in-place fused update of caller-owned (weight, grad) pairs (kvstore.cc)
  void UpdaterStep(bool str_keys, const std::vector<int>& ikeys, const std::vector<std::string>& skeys,
                   const std::vector<NDArray>& weights, const std::vector<NDArray>& grads);
  void SetLearningRate(double lr);
  bool has_fused_optimizer() const { return opt_.enabled; }
  // which: 0 stored value, 1 + i kReplicaState[i] (fp32 master, state0, state1, state2); gathers shards so the
  // result is complete
  NDArray GetState(bool str_key, int ikey, const std::string& skey, int which);
  void SetState(bool str_key, int ikey, const std::string& skey, int which, const NDArray& v);
  // per-key switches of the fused optimizers; "no_trust_ratio": LARS skips the layer-wise ratio (lars.py:121-123)
  void SetKeyFlag(bool str_key, int ikey, const std::string& skey, const std::string& name, int value);
  // 1 if the last push with skip_nonfinite met a non-finite gradient (and therefore changed nothing);
  // waits for the engine streams, undoes that push's update counts, clears the flag
  int ResolveOverflow();
  void GetKeyHyper(bool str_key, int ikey, const std::string& skey, float* lr, float* wd, float* eta);
  int64_t GetUpdateCount(bool str_key, int ikey, const std::string& skey);
  // store-wide scalars of the fused optimizer: "m_schedule" (Nadam's momentum-schedule product)
  double GetOptimizerScalar(const std::string& name);
  void SetOptimizerScalar(const std::string& name, double value);
  void SetUpdateCount(bool str_key, int ikey, const std::string& skey, int64_t c);

 private:
  enum KeyType { kUndefinedKey = -1, kStringKey = 0, kIntKey = 1 };
  void SetKeyType(KeyType t);
  void LookupKeys(const std::vector<std::string>& str_keys, std::vector<int>* keys);
  void NewStrKeys(const std::vector<std::string>& str_keys, std::vector<int>* keys);
  int ResolveKey(bool str_key, int ikey, const std::string& skey);

  void InitImpl(const std::vector<int>& keys, const std::vector<NDArray>& vals);
  void PushImpl(const std::vector<int>& keys, const std::vector<NDArray>& vals, int priority);
  void PullImpl(const std::vector<int>& keys, const std::vector<NDArray*>& outs, int priority, bool ignore_sparse);
  void PushPullImpl(const std::vector<int>& vkeys, const std::vector<int>& okeys, const std::vector<NDArray>& vals,
                    const std::vector<NDArray*>& outs, int priority);
  void PullRowSparseImpl(const std::vector<int>& keys, const std::vector<std::pair<NDArray*, NDArray>>& vr,
                         int priority);

  struct Group {                       // one unique key of a call
    int key;
    std::vector<NDArray> vals;         // pushed values (dense)
    std::vector<NDArray*> outs;        // pull destinations (may be empty)
  };
  // the fused reduce(+update)(+broadcast) over a list of dense key groups: builds the call's CallPlan key by key
  // (the stages below, none of which launches or touches a caller array), then IssuePlan
  void ReduceUpdate(std::vector<Group>& groups, bool write_outs);
  void PlaceKey(const Group& g, KeyState& ks, std::vector<int>* devs, std::vector<int>* key_part, bool* key_collective);
  struct CallPlan;
  struct KeyBuild;                     // one key of the call being built (kvstore.cc)
  struct Dest;
  void KeyReplicas(CallPlan& p, KeyBuild& k);
  std::vector<std::vector<const void*>> KeySources(CallPlan& p, KeyBuild& k);
  void KeyTree(const CallPlan& p, KeyBuild& k);
  std::vector<Dest> KeyDests(CallPlan& p, KeyBuild& k);
  void KeyWorks(CallPlan& p, const KeyBuild& k, const std::vector<std::vector<const void*>>& srcptr,
                const std::vector<Dest>& dests);
  // an entry that updates replica r of ks over [begin, end) (weight, fp32 master, optimizer state; a fused call's
  // ks.step scalars, else zeros, which no OPT_NONE kernel reads and which keep unfused lists byte-equal); sources,
  // destinations and flags are the caller's
  TensorWork ReplicaWork(const KeyState& ks, const Replica& r, bool fused, bool mp, int64_t begin, int64_t end) const;
  // busiest[i]: number of elements the busiest rank processes for entry i (fixes the common grid)
  void LaunchWorks(const LaunchClassKey& ck, std::vector<std::vector<TensorWork>>& per_part,
                   const std::vector<int64_t>& busiest, int opt_kind, const std::vector<int>& part_dev);
  void LaunchLocal(const LaunchClassKey& ck, const TensorWork& tw, int opt_kind, int dev);
  // LAMB / LANS / LARS: the same work lists as a first / finalize / (mid) / apply launch sequence
  struct NormClass {
    LaunchClassKey ck;
    std::vector<std::vector<TensorWork>>* per_part;
    const std::vector<int64_t>* busiest;
  };
  void LaunchNormWorks(std::vector<NormClass>& classes, int opt_kind, const std::vector<int>& part_dev);
  void GatherLocal(KeyState& ks);
  bool HostPipelined(std::vector<Group>& groups, bool write_outs);
  // quantize_only: quantise every pushed value (its residual advances) and count the update, nothing else
  void ReduceUpdateCompressed(std::vector<Group>& groups, bool write_outs, bool quantize_only = false);
  // a step that SkipsOnRescale: counted, weights and state untouched; under compression still quantised
  void SkipStep(std::vector<Group>& groups);
  // the Python updater on (merged, root's stored value)
  void RunCallbackUpdater(KeyState& ks, Replica& root, const NDArray& merged);
  // rendezvous arguments (epoch left 0): the process group's ranks in `mode`, or one GPU alone (SYNC_NONE: the grid
  // barrier of the fused row_sparse kernels)
  SyncArgs GroupSync(int mode) const;
  static SyncArgs LocalSync(int dev);
  // row_sparse push (kvstore_rsp.cc): the single-node and the multi-node form share the stages below
  void PushRowSparse(KeyState& ks, const std::vector<NDArray>& vals);
  void RowSparseKeyFor(KeyState& ks);
  bool RowSparseFused() const;
  RspSources PublishRowSparse(const KeyState& ks, Replica& r, const NDArray& v, bool fill);
  RspRowArgs RowArgs(const KeyState& ks, const Replica& r, const RspSources& S, bool merge, bool update,
                     bool assign) const;
  void MergeRows(KeyState& ks, Replica& r, const RspSources& S, int64_t cap, bool update, bool assign);
  void InitRowSparseKey(KeyState& ks, const NDArray& v);
  void PullDenseFromRowSparse(KeyState& ks, const std::vector<NDArray*>& outs);
  void BroadcastFromRank0(KeyState& ks, Replica& r);

  KeyState& GetKey(int key);
  KeyState& PeekKey(int key);
  Replica& EnsureReplica(KeyState& ks, int dev);
  Replica* FindReplica(KeyState& ks, int dev);
  Replica& FreshReplica(KeyState& ks);
  void EnsureState(KeyState& ks, Replica& r, bool mp);
  void SyncState(KeyState& ks, Replica& r);
  void GatherState(KeyState& ks);
  int DefaultDevice();
  bool SkipsOnRescale() const;
  // every scalar of a fused update of ks at its current count (and Nadam's current schedule product)
  KeyStep KeyScalars(const KeyState& ks) const;
  // the one place a fused update is counted (Optimizer._update_count, in call order; Nadam's schedule product
  // advances with it), run or skipped: derives the update's scalars into ks.step
  void StepKey(KeyState& ks);

  // ---- multi-node ('dist_device_sync' over a configured Hierarchy, runtime.h) --------------------------
  // A push runs as: phase 1 = reduce(-scatter) of the node's values into this rank's staging slices; ONE
  // inter-node sum per dtype over the packed slices; phase 2 = fused update (+ all-gather) inside the node with
  // the slice as the only source.  Every node computes the same update, so no parameter server is involved.
  void HierReduceUpdate(std::vector<Group>& groups, bool write_outs);
  void HierPushRowSparse(KeyState& ks, const std::vector<NDArray>& vals);
  void InterNodeSum(void* ptr, int64_t count, int dtype, int dev);
  bool hier_ = false;
  int hier_phase_ = 0;                       // 0: not inside a hierarchical push
  bool hier_whole_keys_ = false;             // phase 1 for a Python updater: no sharding, every rank gets the sum
  struct HierBuf { void* ptr = nullptr; size_t bytes = 0; int dev = -1; };
  std::map<int, HierBuf> hier_buf_;          // per dtype: packed staging slices of one call
  std::unordered_map<int, void*> hier_base_; // per key: slice address minus the byte offset of this rank's range

  // ---- cached launch plans (what replaces the per-call bookkeeping for the training loop's repeated calls) ----
  // The reference's engine re-derives nothing per step either: its per-key merge buffers and copy ops are set up
  // once (comm.h:452-520) and each step only pushes ops.  Here a push / pushpull whose signature (keys, value
  // and output arrays) repeats while nothing else has touched its keys replays the recorded work lists: only
  // the update counts and the per-key lr / wd / eta scalars are patched in.
  struct PlanLaunch {
    LaunchClassKey ck;
    std::vector<std::vector<TensorWork>> per_part;
    std::vector<int64_t> busiest;
    std::vector<std::vector<int>> key_idx;     // per entry of per_part: index of its key in CallPlan::keys
  };
  // What one dense call issues (IssuePlan).  ReduceUpdate builds it; a repeated call keeps it (plans_).
  struct StagedValue { NDArray src; void* tmp; int dev; };   // a value copied into a cudaMallocAsync temporary
  struct CallPlan {
    std::vector<uint64_t> sig;                 // keys, array addresses / sizes / devices, flags
    std::vector<int> keys;                     // group order
    std::vector<uint64_t> epochs;              // KeyState::epoch of `keys` right after the recorded call
    std::vector<PlanLaunch> launches;          // sorted by class key: the launch order of every rank
    std::vector<int> part_dev;                 // device of participant p (SP) / own device at index rank (MP)
    std::vector<int> touched;                  // (sorted) devices acquired from / released to the framework stream
    std::vector<std::pair<int, int>> pre_waits;                 // StreamWait(waiter, signaler) before the launches
    std::vector<std::pair<NDArray, NDArray>> pre_copies;        // staging copies (src, dst) before the launches
    std::vector<std::pair<NDArray, NDArray>> post_copies;       // outputs copied out of a replica afterwards
    int opt_kind = OPT_NONE;
    bool fused = false, collective = false;
    int root_dev = -1;
    uint64_t cfg_epoch = 0, tuning_epoch = 0;
    bool recorded = false;                     // false: only `sig` / `epochs` of the last identical slow call
    // per-call work a replay never repeats; a plan that has any is not kept
    std::vector<StagedValue> staged;           // host values / values without P2P, freed after the launches
    std::vector<KeyState*> callback_keys;      // keys whose Python updater runs after the launches
    bool repeatable = true;                    // false: the build gathered a sharded value or optimizer state
  };
  void IssuePlan(CallPlan& p);
  bool SamePlan(const CallPlan& a, const CallPlan& b) const;
  // The signature is taken from the call's raw arguments (TryReplayRaw, below) so that a hit costs no grouping,
  // no NDArray copies and no allocation; ReduceUpdate records under it when the call reached it as ONE fused
  // reduce over all of its keys (raw_single_).
  std::vector<uint64_t> raw_sig_;
  uint64_t raw_hash_ = 0;
  bool raw_pending_ = false, raw_single_ = false;
  bool PlanEpochsMatch(const CallPlan& p) const;
  void PlanPatch(CallPlan& p, bool commit_counts);
  struct Deferred {
    int kind;                               // 0 push, 1 pushpull
    std::vector<int> vkeys, okeys;
    std::vector<NDArray> vals, outs;
    int priority;
  };
  std::vector<Deferred> pending_;
  void FlushIfPending(int key);
  bool deferred_ = false;
  int64_t deferred_batches_ = 0;            // launches (sequences) issued by Flush so far
  bool Defer(int kind, const std::vector<int>& vkeys, const std::vector<int>& okeys, const std::vector<NDArray>& vals,
             const std::vector<NDArray*>& outs, int priority);
  std::unordered_map<uint64_t, CallPlan> plans_;       // by hash of the signature
  uint64_t cfg_epoch_ = 0;                   // optimizer kind / updater / compression / hierarchy changes
  int plan_mode_ = 1;                        // MXKV_B200_PLAN: 0 off, 1 on, 2 verify (build both ways, compare, abort on a difference)
  int64_t plan_hits_ = 0;
 public:
  int64_t plan_hits() const { return plan_hits_; }
  // C-API fast path of push (kind 0) / pushpull (kind 1) with integer keys: replays the cached plan of an identical
  // earlier call and returns true, or leaves the signature for the full path to record under and returns false
  bool TryReplayRaw(int kind, uint32_t vnum, const int* vkeys, NDArray* const* vals, uint32_t onum, const int* okeys,
                    NDArray* const* outs);
  void ClearRawPending() { raw_pending_ = false; raw_single_ = false; }
 private:

  // ---- MXNET_KVSTORE_USETREE=1 (CommDeviceTree, src/kvstore/comm_tree.h:50-325; topology.h) -----------------
  // The trees are built once per set of GPUs a key is pushed from (the reference builds them for the devices of
  // its first push, comm_tree.h:66-82) and turned into the add schedules the tree kernel executes.
  struct TreePlan {
    topo::TreeSet trees;
    std::vector<topo::ReduceProgram> prog;   // per root
  };
  bool tree_ = false;
  int64_t tree_bound_ = 10000000;            // MXNET_KVSTORE_TREE_ARRAY_BOUND: keys above it are summed slice by slice
  bool tree_backtrack_ = false;              // MXNET_KVSTORE_TREE_BACKTRACK
  float tree_penalty_ = 0.7f;                // MXNET_KVSTORE_TREE_LINK_USAGE_PENALTY
  std::map<std::vector<int>, TreePlan> tree_plans_;
  const TreePlan& TreePlanFor(const std::vector<int>& devs);
  void AppendTreeWorks(const TensorWork& tw, const TreePlan& tp, bool sliced, const KeyState& ks, int n_part,
                       std::vector<TensorWork>* out);

  ProcessGroup* PG() const;     // the process group this store exchanges over (none for 'updater' stores)
  std::string type_;
  bool device_mode_ = false;
  bool solo_ = false;
  int order_ = ORDER_DEVICE;
  std::unordered_map<int, KeyState> keys_;
  std::unordered_map<std::string, int> str_key_dict_;
  std::unordered_map<int, std::string> reverse_str_key_dict_;
  int next_str_key_ = 0;
  KeyType key_type_ = kUndefinedKey;
  std::unordered_set<int> warnings_printed_;
  UpdaterFn updater_ = nullptr;
  StrUpdaterFn str_updater_ = nullptr;
  void* updater_handle_ = nullptr;
  OptimizerConfig opt_;
  std::string gc_type_ = "none";
  float gc_threshold_ = 0.5f;
  int gc_bits_ = 0;
  int* overflow_flag_ = nullptr;        // host-mapped word written by the apply kernel
  std::vector<int> last_norm_keys_;     // keys of the last skip_nonfinite push (count roll-back)
  std::recursive_mutex mu_;
};

// issues the deferred calls of every store that has some (array reads and waits are flush points)
void FlushAllDeferred();

// multi_sum_sq / multi_all_finite over a list of dense arrays on one GPU (kvstore_norm.cc)
void MultiSumSq(const std::vector<NDArray>& arrays, float scale, NDArray* out_sumsq, NDArray* all_finite,
                bool init_output);

}  // namespace mxkv
