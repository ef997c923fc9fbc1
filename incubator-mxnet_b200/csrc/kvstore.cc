// kvstore.cc -- see kvstore.h for the reference mapping.
#include "kvstore.h"
#include "rsp_kernels.h"
#include "norm_kernels.h"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>

namespace mxkv {

static std::set<KVStore*>& DeferredStores();

static std::string Lower(std::string s) {
  std::transform(s.begin(), s.end(), s.begin(), ::tolower);
  return s;
}

// KVStore::Create, src/kvstore/kvstore.cc:42-85: substring dispatch on the lower-cased
// type.  'device' selects the on-GPU reduce (CommDevice association order); the other
// local types select CommCPU's association order -- the arithmetic still runs on the GPU.
KVStore::KVStore(const std::string& type) : type_(Lower(type)) {   // kvstore.cc:43-44,83: the type is kept lower-cased
  const std::string t = Lower(type);
  const bool dist = t.find("dist") != std::string::npos;
  if (dist) {
    // KVStoreDist's synchronous mode (src/kvstore/kvstore_dist.h:343-470) is served hierarchically, without
    // servers, once the embedding job has described the nodes; the parameter-server machinery itself
    // (ps-lite, asynchronous mode, server-side profiler commands) is out of scope of this library
    Runtime* rt = Runtime::Get();
    MXKV_CHECK(rt->hier.configured() && rt->pg() != nullptr)
        << "distributed kvstore types ('" << type << "') are out of scope of this library unless a node hierarchy "
           "is configured (MXKVB200SetHierarchy; mx.dist.init_process_group(local_world=...))";
    MXKV_CHECK(t.find("async") == std::string::npos)
        << "asynchronous distributed stores ('" << type << "') are out of scope of this library";
    hier_ = rt->hier.num_nodes > 1;
  }
  // 'nccl' (KVStoreNCCL, src/kvstore/kvstore_nccl.h:62-551: rooted ncclReduce + ncclBcast per key) is
  // served by the same engine: NCCL leaves its summation order unspecified, so the device order is a
  // conforming result for that name ("parity unpinned" for this one type).
  // 'updater': not a store of the reference -- the native counterpart of its per-device Updater
  // (python/mxnet/optimizer/updater.py:30-127): optimizer state + fused multi-tensor updates of
  // caller-owned weights (UpdaterStep), never collective even in one-process-per-GPU mode
  solo_ = t.find("updater") != std::string::npos;
  device_mode_ = solo_ || dist || t.find("device") != std::string::npos || t.find("nccl") != std::string::npos;
  order_ = device_mode_ ? ORDER_DEVICE : ORDER_COMMCPU;
  plan_mode_ = static_cast<int>(EnvInt("MXKV_B200_PLAN", 1));
  // kvstore_local.h:74-82: a store with device-side reduction takes CommDeviceTree instead of CommDevice when
  // MXNET_KVSTORE_USETREE is set; its knobs are read once, where the reference's constructor reads them
  // (comm_tree.h:52-57).  Multi-node stores keep their own two-phase sum (DESIGN.md section 1, row a18).
  if (!solo_ && !hier_ && t.find("device") != std::string::npos && EnvInt("MXNET_KVSTORE_USETREE", 0) != 0) {
    tree_ = true;
    tree_bound_ = EnvInt("MXNET_KVSTORE_TREE_ARRAY_BOUND", 10000000);
    tree_backtrack_ = EnvInt("MXNET_KVSTORE_TREE_BACKTRACK", 0) != 0;
    if (const char* v = std::getenv("MXNET_KVSTORE_TREE_LINK_USAGE_PENALTY")) tree_penalty_ = static_cast<float>(std::atof(v));
  }
}

const KVStore::TreePlan& KVStore::TreePlanFor(const std::vector<int>& devs) {
  auto it = tree_plans_.find(devs);
  if (it != tree_plans_.end()) return it->second;
  const int n = static_cast<int>(devs.size());
  TreePlan plan;
  const std::vector<float> W = topo::QueryLinkWeights(devs);
  topo::ComputeTrees(W, n, tree_penalty_, tree_backtrack_, &plan.trees);
  uint64_t digest = 1469598103934665603ull;
  auto mix = [&](uint64_t v) { digest = (digest ^ v) * 1099511628211ull; };
  for (int r = 0; r < n; ++r) {
    plan.prog.push_back(topo::ReduceProgramOf(plan.trees.topo[r], plan.trees.scan[r], plan.trees.depth, n));
    for (int k = 0; k < n; ++k) mix(static_cast<uint64_t>(plan.prog[r].leaf[k]));
    mix(plan.prog[r].prog);
  }
  if (EnvInt("MXNET_KVSTORE_LOGTREE", 0) != 0) {     // gpu_topology.h:46: print what was built
    for (int r = 0; r < n; ++r) {
      std::string line = "mxkv_b200: tree " + std::to_string(r) + ":";
      for (size_t v : plan.trees.topo[r]) line += " " + std::to_string(v);
      line += "  | add order";
      for (int k = 0; k < n; ++k) line += " " + std::to_string(plan.prog[r].leaf[k]);
      fprintf(stderr, "%s  (schedule 0x%x)\n", line.c_str(), plan.prog[r].prog);
    }
  }
  if (ProcessGroup* pg = PG()) {
    // one process per GPU: every rank must add in the same order, i.e. must have seen the same link matrix
    std::vector<uint64_t> all(pg->world());
    pg->AllGather(&digest, sizeof(digest), all.data());
    for (uint64_t d : all)
      MXKV_CHECK(d == digest) << "MXNET_KVSTORE_USETREE: the ranks derived different reduction trees (do they all see the "
                                 "same GPUs, in the same order?)";
  }
  return tree_plans_.emplace(devs, std::move(plan)).first->second;
}

// One work entry of a key, cut where the tree changes: a key above MXNET_KVSTORE_TREE_ARRAY_BOUND elements with
// at least 2n rows is n row slices, slice i summed up the tree rooted at GPU i (comm_tree.h:203-234: slice_size =
// rows / n, the last slice takes the remainder); any other key goes up tree 0 whole (:236-240).  The sources are
// handed to the kernel in the tree's leaf order.
void KVStore::AppendTreeWorks(const TensorWork& tw, const TreePlan& tp, bool sliced, const KeyState& ks, int n_part,
                              std::vector<TensorWork>* out) {
  const size_t before = out->size();
  auto emit = [&](int64_t pb, int64_t pe, int root) {
    const topo::ReduceProgram& rp = tp.prog[root];
    TensorWork t = tw;
    for (int k = 0; k < rp.n; ++k) t.src[k] = tw.src[rp.leaf[k]];
    t.tree_prog = rp.prog;
    t.flags &= ~kWorkStaged;
    // the vector path wants its first element on a packet boundary: a slice that begins inside a packet is led
    // in by a few scalar elements
    const int64_t aligned = std::min<int64_t>(pe, (pb + 7) / 8 * 8);
    if (pb < aligned) {
      TensorWork h = t;
      h.begin = pb; h.end = aligned;
      h.flags = WorkFlags(h, false);
      out->push_back(h);
      pb = aligned;
    }
    if (pb < pe) { t.begin = pb; t.end = pe; out->push_back(t); }
  };
  if (!sliced) {
    emit(tw.begin, tw.end, 0);
  } else {
    const int64_t rows = ks.shape[0], row_len = ks.size / rows, slice_rows = rows / n_part;
    for (int i = 0; i < n_part; ++i) {
      const int64_t lo = i * slice_rows * row_len, hi = i == n_part - 1 ? ks.size : (i + 1) * slice_rows * row_len;
      const int64_t pb = std::max(tw.begin, lo), pe = std::min(tw.end, hi);
      if (pb < pe) emit(pb, pe, i);
    }
  }
  if (out->size() == before) {          // an empty range still takes part in the launch's rendezvous
    TensorWork t = tw;
    t.tree_prog = tp.prog[0].prog;
    t.end = t.begin;
    out->push_back(t);
  }
}

ProcessGroup* KVStore::PG() const { return solo_ ? nullptr : Runtime::Get()->pg(); }

KVStore::~KVStore() {
  try { Flush(); } catch (...) {}
  DeferredStores().erase(this);
  try { Runtime::Get()->WaitAll(); } catch (...) {}
  for (auto& kv : hier_buf_) {
    if (kv.second.ptr == nullptr) continue;
    cudaSetDevice(kv.second.dev);
    cudaFree(kv.second.ptr);
  }
}

// workers are numbered node by node (kvstore_dist.h: get_rank = ps::MyRank)
int KVStore::rank() const {
  ProcessGroup* pg = PG();
  if (pg && hier_) return Runtime::Get()->hier.node_rank * pg->world() + pg->rank();
  return pg ? pg->rank() : 0;
}
int KVStore::group_size() const {
  ProcessGroup* pg = PG();
  if (pg && hier_) return Runtime::Get()->hier.num_nodes * pg->world();
  return pg ? pg->world() : 1;
}

void KVStore::Barrier() {
  std::lock_guard<std::recursive_mutex> rl(Runtime::Get()->mu());
  std::lock_guard<std::recursive_mutex> lk(mu_);
  if (!pending_.empty()) Flush();
  Runtime* rt = Runtime::Get();
  rt->WaitAll();
  ProcessGroup* pg = PG();
  if (pg) pg->Barrier();
  if (pg && hier_) {
    // every node's ranks have arrived; one element summed across the nodes completes the global barrier
    HierBuf& hb = hier_buf_[kFloat32];
    if (hb.ptr == nullptr) {
      DeviceGuard g(pg->dev());
      CUDA_CALL(cudaMalloc(&hb.ptr, 256));
      CUDA_CALL(cudaMemset(hb.ptr, 0, 256));
      hb.bytes = 256; hb.dev = pg->dev();
    }
    InterNodeSum(hb.ptr, 1, kFloat32, pg->dev());
    rt->WaitAll();
    pg->Barrier();
  }
}

void KVStore::InterNodeSum(void* ptr, int64_t count, int dtype, int dev) {
  Runtime* rt = Runtime::Get();
  MXKV_CHECK(rt->hier.fn != nullptr) << "no inter-node all-reduce configured";
  if (count <= 0) return;
  DeviceGuard g(dev);
  const int rc = rt->hier.fn(ptr, count, dtype, rt->Dev(dev).stream, rt->hier.ctx);
  MXKV_CHECK(rc == 0) << "the inter-node all-reduce callback failed (" << rc << ")";
}

// ---------------------------------------------------------------------------
// key bookkeeping (kvstore_local.h:95-116, 344-347, 471-479)
// ---------------------------------------------------------------------------
void KVStore::SetKeyType(KeyType t) {
  if (key_type_ == kUndefinedKey) key_type_ = t;
  MXKV_CHECK(key_type_ == t) << "Mixed key types are not allowed";
}

void KVStore::LookupKeys(const std::vector<std::string>& str_keys, std::vector<int>* keys) {
  keys->resize(str_keys.size());
  for (size_t i = 0; i < str_keys.size(); ++i) {
    auto it = str_key_dict_.find(str_keys[i]);
    MXKV_CHECK(it != str_key_dict_.end()) << "key " << str_keys[i] << " doesn't exist. Did you init?";
    (*keys)[i] = it->second;
  }
}

void KVStore::NewStrKeys(const std::vector<std::string>& str_keys, std::vector<int>* keys) {
  keys->resize(str_keys.size());
  for (size_t i = 0; i < str_keys.size(); ++i) {
    MXKV_CHECK(str_key_dict_.find(str_keys[i]) == str_key_dict_.end())
        << "duplicate init of key " << str_keys[i];
    const int key = next_str_key_++;
    str_key_dict_[str_keys[i]] = key;
    reverse_str_key_dict_[key] = str_keys[i];
    (*keys)[i] = key;
  }
}

int KVStore::ResolveKey(bool str_key, int ikey, const std::string& skey) {
  if (!str_key) return ikey;
  auto it = str_key_dict_.find(skey);
  MXKV_CHECK(it != str_key_dict_.end()) << "key " << skey << " doesn't exist. Did you init?";
  return it->second;
}

KeyState& KVStore::GetKey(int key) {
  auto it = keys_.find(key);
  MXKV_CHECK(it != keys_.end()) << "key " << key << " has not been inited";
  it->second.epoch++;          // whoever asks for a key may change it: cached launch plans of the key expire
  return it->second;
}

// for callers that only read the key's type / bump its update count (nothing a launch plan depends on)
KeyState& KVStore::PeekKey(int key) {
  auto it = keys_.find(key);
  MXKV_CHECK(it != keys_.end()) << "key " << key << " has not been inited";
  return it->second;
}

// ---------------------------------------------------------------------------
// public entry points: key-type handling then *Impl, as kvstore_local.h:95-219
// ---------------------------------------------------------------------------
// Entry points serialise on the runtime first (per-device streams, descriptor rings, peer tables and signal pads
// are shared by every store of the process), then on the store: callable from any thread, in this fixed order.
#define LOCK_ONLY()                                                             \
  std::lock_guard<std::recursive_mutex> rt_lk__(Runtime::Get()->mu());            \
  std::lock_guard<std::recursive_mutex> lk__(mu_)
// every entry point that reads or changes the store issues the deferred calls first
#define LOCK() LOCK_ONLY(); if (!pending_.empty()) Flush()

// ---------------------------------------------------------------------------
// deferred issue (kvstore.h)
// ---------------------------------------------------------------------------
static std::set<KVStore*>& DeferredStores() { static std::set<KVStore*> s; return s; }

void FlushAllDeferred() {
  std::lock_guard<std::recursive_mutex> rl(Runtime::Get()->mu());
  std::vector<KVStore*> stores(DeferredStores().begin(), DeferredStores().end());
  for (KVStore* s : stores) s->Flush();
}

void KVStore::SetDeferred(bool on) {
  LOCK();
  deferred_ = on;
  if (on) DeferredStores().insert(this); else DeferredStores().erase(this);
}

bool KVStore::Defer(int kind, const std::vector<int>& vkeys, const std::vector<int>& okeys,
                    const std::vector<NDArray>& vals, const std::vector<NDArray*>& outs, int priority) {
  if (!deferred_ || hier_ || updater_ != nullptr || gc_bits_ != 0) return false;
  // Nadam's momentum schedule is one product over every key update in call order: reordering calls by priority
  // would change it, so these calls are issued as they come
  if (opt_.enabled && opt_.kind == OPT_NADAM) return false;
  for (auto& v : vals) if (!v.ctx().is_gpu() || v.stype() != kDefaultStorage) return false;
  for (NDArray* o : outs) if (!o->ctx().is_gpu() || o->stype() != kDefaultStorage) return false;
  for (int k : vkeys) { auto it = keys_.find(k); if (it == keys_.end() || it->second.stype != kDefaultStorage) return false; }
  Deferred d;
  d.kind = kind; d.vkeys = vkeys; d.okeys = okeys; d.vals = vals; d.priority = priority;
  for (NDArray* o : outs) d.outs.push_back(*o);        // views of the caller's arrays (same memory)
  pending_.push_back(std::move(d));
  return true;
}

void KVStore::Flush() {
  LOCK_ONLY();
  if (pending_.empty()) return;
  std::vector<Deferred> calls;
  calls.swap(pending_);
  // issue order: highest priority first among the calls that no EARLIER pending call shares a key with
  std::vector<char> done(calls.size(), 0);
  std::vector<size_t> order;
  for (size_t n = 0; n < calls.size(); ++n) {
    int best = -1;
    std::unordered_set<int> blocked;         // keys of earlier calls that are still pending
    for (size_t i = 0; i < calls.size(); ++i) {
      if (done[i]) continue;
      bool free_ = true;
      for (int k : calls[i].vkeys) if (blocked.count(k)) { free_ = false; break; }
      if (free_ && (best < 0 || calls[i].priority > calls[best].priority)) best = static_cast<int>(i);
      for (int k : calls[i].vkeys) blocked.insert(k);
    }
    done[best] = 1;
    order.push_back(static_cast<size_t>(best));
  }
  // merge neighbours of that order with the same kind and disjoint keys into one call
  size_t i = 0;
  while (i < order.size()) {
    Deferred batch = calls[order[i]];
    std::unordered_set<int> keys(batch.vkeys.begin(), batch.vkeys.end());
    size_t j = i + 1;
    for (; j < order.size(); ++j) {
      const Deferred& c = calls[order[j]];
      bool disjoint = c.kind == batch.kind;
      for (int k : c.vkeys) if (keys.count(k)) { disjoint = false; break; }
      if (!disjoint) break;
      batch.vkeys.insert(batch.vkeys.end(), c.vkeys.begin(), c.vkeys.end());
      batch.okeys.insert(batch.okeys.end(), c.okeys.begin(), c.okeys.end());
      batch.vals.insert(batch.vals.end(), c.vals.begin(), c.vals.end());
      batch.outs.insert(batch.outs.end(), c.outs.begin(), c.outs.end());
      keys.insert(c.vkeys.begin(), c.vkeys.end());
    }
    i = j;
    deferred_batches_++;
    if (batch.kind == 0) {
      PushImpl(batch.vkeys, batch.vals, batch.priority);
    } else {
      std::vector<NDArray*> outs;
      for (auto& o : batch.outs) outs.push_back(&o);
      PushPullImpl(batch.vkeys, batch.okeys, batch.vals, outs, batch.priority);
    }
  }
}


void KVStore::Init(const std::vector<int>& keys, const std::vector<NDArray>& vals) {
  LOCK(); SetKeyType(kIntKey); InitImpl(keys, vals);
}
void KVStore::Init(const std::vector<std::string>& str_keys, const std::vector<NDArray>& vals) {
  LOCK(); SetKeyType(kStringKey);
  std::vector<int> keys; NewStrKeys(str_keys, &keys); InitImpl(keys, vals);
}
void KVStore::Push(const std::vector<int>& keys, const std::vector<NDArray>& vals, int priority) {
  LOCK_ONLY(); SetKeyType(kIntKey);
  if (Defer(0, keys, keys, vals, {}, priority)) return;
  if (!pending_.empty()) Flush();
  PushImpl(keys, vals, priority);
}
void KVStore::Push(const std::vector<std::string>& str_keys, const std::vector<NDArray>& vals, int priority) {
  LOCK(); SetKeyType(kStringKey);
  std::vector<int> keys; LookupKeys(str_keys, &keys); PushImpl(keys, vals, priority);
}
void KVStore::Pull(const std::vector<int>& keys, const std::vector<NDArray*>& outs, int priority, bool ignore_sparse) {
  LOCK(); SetKeyType(kIntKey); PullImpl(keys, outs, priority, ignore_sparse);
}
void KVStore::Pull(const std::vector<std::string>& str_keys, const std::vector<NDArray*>& outs, int priority,
                   bool ignore_sparse) {
  LOCK(); SetKeyType(kStringKey);
  std::vector<int> keys; LookupKeys(str_keys, &keys); PullImpl(keys, outs, priority, ignore_sparse);
}
void KVStore::PushPull(const std::vector<int>& vkeys, const std::vector<int>& okeys,
                       const std::vector<NDArray>& vals, const std::vector<NDArray*>& outs, int priority) {
  LOCK_ONLY(); SetKeyType(kIntKey);
  if (Defer(1, vkeys, okeys, vals, outs, priority)) return;
  if (!pending_.empty()) Flush();
  PushPullImpl(vkeys, okeys, vals, outs, priority);
}
void KVStore::PushPull(const std::vector<std::string>& svkeys, const std::vector<std::string>& sokeys,
                       const std::vector<NDArray>& vals, const std::vector<NDArray*>& outs, int priority) {
  LOCK(); SetKeyType(kStringKey);
  std::vector<int> vkeys, okeys; LookupKeys(svkeys, &vkeys); LookupKeys(sokeys, &okeys);
  PushPullImpl(vkeys, okeys, vals, outs, priority);
}
void KVStore::Broadcast(const std::vector<int>& vkeys, const std::vector<int>& okeys,
                        const std::vector<NDArray>& vals, const std::vector<NDArray*>& outs, int priority) {
  LOCK(); SetKeyType(kIntKey);
  InitImpl(vkeys, vals); PullImpl(okeys, outs, priority, true);   // kvstore_local.h:349-356
}
void KVStore::Broadcast(const std::vector<std::string>& svkeys, const std::vector<std::string>& sokeys,
                        const std::vector<NDArray>& vals, const std::vector<NDArray*>& outs, int priority) {
  LOCK(); SetKeyType(kStringKey);
  std::vector<int> vkeys, okeys; NewStrKeys(svkeys, &vkeys); LookupKeys(sokeys, &okeys);
  InitImpl(vkeys, vals); PullImpl(okeys, outs, priority, true);
}
void KVStore::PullRowSparse(const std::vector<int>& keys,
                            const std::vector<std::pair<NDArray*, NDArray>>& vr, int priority) {
  LOCK(); SetKeyType(kIntKey); PullRowSparseImpl(keys, vr, priority);
}
void KVStore::PullRowSparse(const std::vector<std::string>& str_keys,
                            const std::vector<std::pair<NDArray*, NDArray>>& vr, int priority) {
  LOCK(); SetKeyType(kStringKey);
  std::vector<int> keys; LookupKeys(str_keys, &keys); PullRowSparseImpl(keys, vr, priority);
}

void KVStore::SetUpdater(UpdaterFn fn, StrUpdaterFn sfn, void* handle) {
  LOCK();
  updater_ = fn; str_updater_ = sfn; updater_handle_ = handle;
  cfg_epoch_++;
}

void KVStore::SetGradientCompression(const std::vector<std::pair<std::string, std::string>>& kwargs) {
  LOCK();
  // GradientCompression::SetParams (src/kvstore/gradient_compression.cc:40-52): `type` (default "none") and
  // `threshold` (default 0.5) are read, other arguments are allowed and ignored (InitAllowUnknown), and a type
  // other than 1bit / 2bit is an error -- "none" included
  std::string type = "none";
  float threshold = 0.5f;
  for (auto& kv : kwargs) {
    if (kv.first == "type") type = kv.second;
    else if (kv.first == "threshold") threshold = std::stof(kv.second);
  }
  MXKV_CHECK(type == "1bit" || type == "2bit") << "Unknown type for gradient compression " << type;
  if (type == "2bit") MXKV_CHECK(threshold > 0) << "threshold must be greater than 0 for two bit compression";
  gc_type_ = type;
  gc_threshold_ = threshold;
  // only the device comm compresses (CommDevice::ReduceCompressed, comm.h:556-605); CommCPU sums what it is given
  gc_bits_ = !device_mode_ ? 0 : (type == "2bit" ? 2 : 1);
  cfg_epoch_++;
}

// ---------------------------------------------------------------------------
// optimizer registry
// ---------------------------------------------------------------------------
void KVStore::SetOptimizer(const std::string& name, const std::vector<std::pair<std::string, std::string>>& kwargs) {
  LOCK();
  OptimizerConfig c;
  const std::string n = Lower(name);
  c.enabled = true;
  bool reset_states = false, centered = false;
  if (n == "sgd") { c.kind = OPT_SGD; c.lr = 0.1; }                             // sgd.py:95
  else if (n == "adam") { c.kind = OPT_ADAM; c.lr = 0.001; }
  else if (n == "adamw") { c.kind = OPT_ADAMW; c.lr = 0.001; c.eps = 1e-6f; }  // adamW.py:80
  else if (n == "test") { c.kind = OPT_TEST; c.lr = 0.01; }
  else if (n == "lamb") { c.kind = OPT_LAMB; c.lr = 0.001; c.eps = 1e-6f; }    // lamb.py:66-68
  else if (n == "lans") { c.kind = OPT_LANS; c.lr = 0.001; c.eps = 1e-6f; }    // lans.py:61-63
  else if (n == "lars") { c.kind = OPT_LARS; c.lr = 0.1; }                     // lars.py:77-79
  else if (n == "nag") { c.kind = OPT_NAG; c.lr = 0.1; c.momentum = 0.9f; }     // nag.py:58
  else if (n == "adabelief") { c.kind = OPT_ADABELIEF; c.lr = 0.001; c.eps = 1e-6f; }   // adabelief.py:79
  else if (n == "rmsprop") { c.kind = OPT_RMSPROP; c.lr = 0.001; c.momentum = 0.9f; }    // rmsprop.py:70-71
  else if (n == "signum") { c.kind = OPT_SIGNUM; c.lr = 0.01; c.momentum = 0.9f; }      // signum.py:67
  else if (n == "ftml") { c.kind = OPT_FTML; c.lr = 0.0025; c.beta1 = 0.6; c.beta2 = 0.999; c.eps = 1e-8f; }  // ftml.py:66
  // adamax.py:61, adadelta.py:62.  Both keep the generic clip rule: `step` clips whenever clip_gradient is not None,
  // at 0 too.  A negative bound is off here, where `step` would clip to the inverted interval [-c, c]
  else if (n == "adamax") {
    c.kind = OPT_ADAMAX; c.lr = 0.002; c.beta1 = 0.9; c.beta2 = 0.999; c.eps = static_cast<float>(1e-8);
  } else if (n == "adadelta") {
    c.kind = OPT_ADADELTA; c.lr = 1.0; c.rho_d = 0.9; c.rho = static_cast<float>(0.9); c.eps = static_cast<float>(1e-6);
  } else if (n == "nadam") {      // nadam.py:58-67; clip as for Adamax
    c.kind = OPT_NADAM; c.lr = 0.001; c.beta1 = 0.9; c.beta2 = 0.999; c.eps = static_cast<float>(1e-8);
    c.schedule_decay = 0.004; c.m_schedule = 1.0;
  }
  else MXKV_FATAL() << "optimizer '" << name << "' has no fused kernel; register a Python updater instead";
  // Adamax, AdaDelta and Nadam restate their optimizer's Python `step`, where a scalar enters an NDArray operation as
  // float32(double): parse as double, then round once (std::stof may round the decimal string differently)
  const bool from_double = c.kind == OPT_ADAMAX || c.kind == OPT_ADADELTA || c.kind == OPT_NADAM;
  bool have_m_schedule = false;
  auto to_float = [from_double](const std::string& v) {
    return from_double ? static_cast<float>(std::stod(v)) : std::stof(v);
  };
  for (auto& kv : kwargs) {
    const std::string& k = kv.first;
    const std::string& v = kv.second;
    if (k == "learning_rate" || k == "lr") c.lr = std::stod(v);
    else if (k == "wd") c.wd = std::stod(v);
    else if (k == "momentum") c.momentum = std::stof(v);
    else if (k == "beta1") c.beta1 = std::stod(v);
    else if (k == "beta2") c.beta2 = std::stod(v);
    else if (k == "epsilon") { if (c.kind == OPT_LARS) c.lars_eps = std::stof(v); else c.eps = to_float(v); }
    else if (k == "eta") {
      if (c.kind == OPT_LARS) c.lars_eta = std::stof(v);
      else { c.eta = std::stof(v); c.eta_d = std::stod(v); }
    }
    else if (k == "lower_bound") c.lower_bound = (v == "None" || v.empty()) ? -1.f : std::stof(v);
    else if (k == "upper_bound") c.upper_bound = (v == "None" || v.empty()) ? -1.f : std::stof(v);
    else if (k == "bias_correction") c.bias_correction = (v == "True" || v == "true" || v == "1");
    else if (k == "skip_nonfinite") c.skip_nonfinite = (v == "True" || v == "true" || v == "1");
    else if (k == "rescale_grad") c.rescale = to_float(v);
    else if (k == "clip_gradient") c.clip = (v == "None" || v.empty()) ? -1.f : to_float(v);
    else if (k == "lazy_update") c.lazy_update = (v == "True" || v == "true" || v == "1");
    else if (k == "correct_bias") c.correct_bias = (v == "True" || v == "true" || v == "1");
    else if (k == "multi_precision") c.multi_precision = (v == "True" || v == "true" || v == "1");
    else if (k == "reset_states") reset_states = (v == "True" || v == "true" || v == "1");
    else if (k == "rho") { c.rho = to_float(v); c.rho_d = std::stod(v); }
    else if (k == "centered") centered = (v == "True" || v == "true" || v == "1");
    else if (k == "clip_weights") c.clip_weights = (v == "None" || v.empty()) ? -1.f : std::stof(v);
    else if (k == "wd_lh") c.wd_lh = std::stod(v);
    else if (k == "schedule_decay") c.schedule_decay = std::stod(v);
    else if (k == "m_schedule") { c.m_schedule = std::stod(v); have_m_schedule = true; }
    else MXKV_FATAL() << "unknown optimizer argument '" << k << "'";
  }
  if (c.kind == OPT_RMSPROP) {
    if (centered) c.kind = OPT_RMSPROP_CENTERED;                     // rmspropalex_update, rmsprop.py:175-181
    // RMSProp.fused_step hands clip_gradient / clip_weights to the operator only when they are truthy
    // (rmsprop.py:169-172): 0, a negative value or None turns either clip off for this optimizer
    if (!(c.clip > 0.f)) c.clip = -1.f;
    if (!(c.clip_weights > 0.f)) c.clip_weights = -1.f;
  }
  if (c.kind == OPT_SIGNUM) {
    // Signum.fused_step (signum.py:139-158): no state at momentum 0 -> signsgd_update; otherwise signum_update, handed
    // the momentum only when it is > 0 (a negative momentum creates the state and runs the operator at momentum 0)
    // and clip_gradient only when it is truthy (0, a negative value or None is off)
    if (c.momentum == 0.f) c.kind = OPT_SIGNSGD;
    if (!(c.momentum > 0.f)) c.momentum = 0.f;
    if (!(c.clip > 0.f)) c.clip = -1.f;
  }
  // FTML.fused_step hands clip_gradient to ftml_update only when it is truthy (ftml.py:152-153): 0, a negative value
  // or None is off
  if (c.kind == OPT_FTML && !(c.clip > 0.f)) c.clip = -1.f;
  if (c.kind == OPT_SGD && c.momentum != 0.f) c.kind = OPT_SGD_MOM;   // sgd.py:213-224
  if (c.kind == OPT_NAG && c.momentum == 0.f) c.kind = OPT_SGD;       // nag.py:59-63,141-154: no state, (mp_)sgd_update
  // Nadam's schedule product: set by an explicit m_schedule; without one, hyper-parameters re-sent to the current
  // Nadam (no reset_states) keep the product where the store's updates have taken it
  if (c.kind == OPT_NADAM && !have_m_schedule && !reset_states && opt_.enabled && opt_.kind == OPT_NADAM)
    c.m_schedule = opt_.m_schedule;
  MXKV_CHECK(!c.skip_nonfinite || IsNormOpt(c.kind)) << "skip_nonfinite is available for lamb / lans / lars";
  c.lr_mult = opt_.lr_mult;
  c.wd_mult = opt_.wd_mult;
  c.no_trust = opt_.no_trust;
  opt_ = c;
  // the reference's set_optimizer REPLACES the updater (python/mxnet/kvstore/kvstore.py:559-606): a callback
  // installed for an earlier optimizer must not keep running in front of the fused kernel
  updater_ = nullptr; str_updater_ = nullptr; updater_handle_ = nullptr;
  cfg_epoch_++;
  if (reset_states) {
    // a NEW optimizer starts from fresh state, like the new Updater the reference creates in set_optimizer
    // (kvstore.py:559-606); re-sending the hyper-parameters of the current one (rescale_grad per batch size,
    // a scheduled learning rate) keeps it
    Runtime::Get()->WaitAll();
    for (auto& kv : keys_) {
      KeyState& ks = kv.second;
      for (auto& r : ks.reps) {
        for (auto m : kReplicaState) r.*m = NDArray();
        r.aux0 = NDArray(); r.aux1 = NDArray();
        r.state_fresh = true;
      }
      ks.state_world = 0;
      ks.state_devs.clear();
      ks.has_state = false;
    }
  }
}

void KVStore::SetKeyFlag(bool str_key, int ikey, const std::string& skey, const std::string& name, int value) {
  LOCK();
  const int key = ResolveKey(str_key, ikey, skey);
  if (name == "no_trust_ratio") {
    if (value) opt_.no_trust.insert(key); else opt_.no_trust.erase(key);
  } else {
    MXKV_FATAL() << "unknown key flag '" << name << "'";
  }
}

void KVStore::SetLearningRate(double lr) {
  LOCK();                 // (deferred calls were made under the old learning rate)
  opt_.lr = lr;
}

// per-key scalars: only a deferred call on THAT key has to be issued first
void KVStore::FlushIfPending(int key) {
  for (auto& d : pending_)
    for (int k : d.vkeys) if (k == key) { Flush(); return; }
}

void KVStore::SetOptimizerMult(bool str_key, int ikey, const std::string& skey, float lr_mult, float wd_mult) {
  LOCK_ONLY();
  const int key = ResolveKey(str_key, ikey, skey);
  FlushIfPending(key);
  opt_.lr_mult[key] = lr_mult;
  opt_.wd_mult[key] = wd_mult;
}

// AdamW and AdaBelief: the reference's optimizer classes hand the operator lr = 1 and eta = the
// (bias-corrected) learning rate (`lrs=np.ones(...)`, `etas=lrs`, python/mxnet/optimizer/adamW.py:176-200,
// adabelief.py:171-220), which is how `w -= eta * (lr * m / (sqrt(v) + eps) + wd * w)`
// (contrib/adamw-inl.h:101-124) becomes the documented `w -= lr * (m / (sqrt(v) + eps) + wd * w)`.
// opt_.eta is an additional schedule multiplier of this engine's own (1 by default; the reference classes
// have none).
static bool EtaCarriesLR(int kind) { return kind == OPT_ADAMW || kind == OPT_ADABELIEF; }

// FTML: the two powers of the update count t that FTMLKernel evaluates per element (optimizer_op-inl.h:1171-1172),
// evaluated once per key as the operator's float arithmetic defines them -- t cast to float, beta^t, then
// (1 - beta1^t) / lr in float with lr the float attribute Python hands over.  The powers are correctly rounded
// (pow in double, rounded once), where the reference's device powf need not be.
static float FtmlPow(double beta, int64_t count) {
  const float t = static_cast<float>(count);
  return static_cast<float>(std::pow(static_cast<double>(static_cast<float>(beta)), static_cast<double>(t)));
}

// nadam.py:97-98, in double as Python computes it: the warming momentum schedule of update count t
static double NadamMomentum(const OptimizerConfig& o, double t) {
  return o.beta1 * (1. - 0.5 * std::pow(0.96, t * o.schedule_decay));
}

// `_adamw_update`, `_adabelief_update` and their multi / mp forms leave everything untouched when the
// rescale_grad scalar is 0, inf or nan (contrib/adamw-inl.h:455, contrib/adabelief-inl.h:454-466: the AMP
// loss-scale path); Optimizer._update_count has already run by then (adamW.py:158, adabelief.py:171).
bool KVStore::SkipsOnRescale() const {
  return opt_.enabled && updater_ == nullptr && EtaCarriesLR(opt_.kind) &&
         (!std::isfinite(opt_.rescale) || opt_.rescale == 0.f);
}

// The reference reduces every push before its updater runs (kvstore_local.h:240-280), so under compression a
// skipped step still quantises each pushed value against its residual (comm.h:556-605); only the operator then
// leaves weight and state alone.  Without compression there is nothing to reduce for: the step is only counted.
void KVStore::SkipStep(std::vector<Group>& groups) {
  if (gc_bits_ != 0) {
    ReduceUpdateCompressed(groups, false, true);
    return;
  }
  for (auto& g : groups) StepKey(PeekKey(g.key));
}

KeyStep KVStore::KeyScalars(const KeyState& ks) const {
  KeyStep s;
  // Optimizer._get_lr (optimizer.py) then, for Adam, the host-side bias correction of
  // adam.py:166-175 -- all in double like Python, rounded to float once.
  double lr = opt_.lr;
  auto it = opt_.lr_mult.find(ks.key);
  if (it != opt_.lr_mult.end()) lr *= it->second;
  // adamW.py:175-182, adabelief.py:174-181
  if (opt_.kind == OPT_ADAM || (EtaCarriesLR(opt_.kind) && opt_.correct_bias)) {
    const double t = static_cast<double>(ks.count);
    const double coef1 = 1. - std::pow(opt_.beta1, t);
    const double coef2 = 1. - std::pow(opt_.beta2, t);
    lr *= std::sqrt(coef2) / coef1;
  }
  // adamax.py:93: lr /= (1. - self.beta1**t)
  if (opt_.kind == OPT_ADAMAX) lr /= (1. - std::pow(opt_.beta1, static_cast<double>(ks.count)));
  s.lr_d = lr;
  double wd = opt_.wd;
  it = opt_.wd_mult.find(ks.key);
  if (it != opt_.wd_mult.end()) wd *= it->second;
  // signsgd_update is handed wd + wd_lh, summed in Python (double) and not multiplied by wd_mult (signum.py:156-158)
  if (opt_.kind == OPT_SIGNSGD) wd += opt_.wd_lh;
  s.wd = static_cast<float>(wd);
  s.lr = static_cast<float>(s.lr_d);
  s.eta = opt_.eta;
  if (EtaCarriesLR(opt_.kind)) {
    s.lr = 1.0f;
    s.eta = static_cast<float>(s.lr_d * opt_.eta_d);
  } else if (opt_.kind == OPT_FTML) {
    s.lr = (1.0f - FtmlPow(opt_.beta1, ks.count)) / static_cast<float>(s.lr_d);
    s.eta = 1.0f - FtmlPow(opt_.beta2, ks.count);
  } else if (opt_.kind == OPT_ADAMAX || opt_.kind == OPT_ADADELTA) {
    // the complement that `step` writes as `(1. - beta1) * grad` / `(1. - rho) * square(...)` -- computed in double,
    // then rounded once.  1.f - float(beta1) is a different number for most betas (0.1f against 0.100000024f at 0.9)
    s.eta = static_cast<float>(1.0 - (opt_.kind == OPT_ADAMAX ? opt_.beta1 : opt_.rho_d));
  } else if (opt_.kind == OPT_NADAM) {
    // nadam.py:95-101: coef2 = 1. - self.beta2**t, and the schedule at t and t + 1 with the optimizer-wide product
    // m_schedule that this update has multiplied (StepKey); in double as Python computes them, each rounded once
    const double t = static_cast<double>(ks.count);
    s.eta = static_cast<float>(1. - std::pow(opt_.beta2, t));
    const double mom_t = NadamMomentum(opt_, t), mom_t1 = NadamMomentum(opt_, t + 1.);
    const double m_next = opt_.m_schedule * mom_t1;
    s.nadam = make_float4(static_cast<float>(1. - opt_.m_schedule), static_cast<float>(1. - m_next),
                          static_cast<float>(mom_t1), static_cast<float>(1. - mom_t));
  }
  if (IsNormOpt(opt_.kind)) {
    // bias correction denominators: power::Map(beta, step) in float (multi_lamb.cc:64-69)
    const float tcount = static_cast<float>(ks.count);
    s.c1 = 1.0f - std::pow(static_cast<float>(opt_.beta1), tcount);
    s.c2 = 1.0f - std::pow(static_cast<float>(opt_.beta2), tcount);
  }
  return s;
}

void KVStore::StepKey(KeyState& ks) {
  ks.count += 1;
  if (opt_.kind == OPT_NADAM) opt_.m_schedule = opt_.m_schedule * NadamMomentum(opt_, static_cast<double>(ks.count));
  ks.step = KeyScalars(ks);
}

// ---------------------------------------------------------------------------
// replicas
// ---------------------------------------------------------------------------
int KVStore::DefaultDevice() {
  Runtime* rt = Runtime::Get();
  if (rt->pg()) return rt->pg()->dev();
  MXKV_CHECK(rt->NumDevices() > 0)
      << "no CUDA device is visible: this KVStore has no CPU fallback (build/run it on a GPU box)";
  return 0;
}

static bool HoldsState(const Replica& r) {
  for (auto m : kReplicaState) if (!(r.*m).is_none()) return true;
  return false;
}

Replica* KVStore::FindReplica(KeyState& ks, int dev) {
  for (auto& r : ks.reps) if (r.dev == dev) return &r;
  return nullptr;
}

Replica& KVStore::FreshReplica(KeyState& ks) {
  for (auto& r : ks.reps) if (r.fresh) return r;
  MXKV_FATAL() << "key " << ks.key << " has no valid replica";
}

Replica& KVStore::EnsureReplica(KeyState& ks, int dev) {
  if (Replica* r = FindReplica(ks, dev)) {
    if (!r->fresh) {
      if (ks.local_world > 0) GatherLocal(ks);
      if (r->fresh) return *r;
      Replica& src = FreshReplica(ks);
      CopyFromTo(src.local, r->local);
      r->fresh = true;
    }
    return *r;
  }
  Runtime* rt = Runtime::Get();
  if (rt->pg()) MXKV_CHECK(dev == rt->pg()->dev()) << "in one-process-per-GPU mode arrays must live on GPU "
                                                   << rt->pg()->dev();
  Replica nr;
  nr.dev = dev;
  nr.local = NDArray::Empty(ks.shape, Context{kGPU, dev}, ks.dtype, /*symmetric=*/PG() != nullptr);
  if (!ks.reps.empty()) {
    if (ks.local_world > 0) GatherLocal(ks);
    if (ks.has_state) GatherState(ks);   // make every existing replica's optimizer state complete
    CopyFromTo(FreshReplica(ks).local, nr.local);
    // a GPU joining later (e.g. states were loaded before the first multi-GPU push) inherits the state
    Replica* holder = nullptr;
    for (auto& cand : ks.reps) if (cand.state_fresh && HoldsState(cand)) { holder = &cand; break; }
    Replica& src = holder ? *holder : FreshReplica(ks);
    const Context nctx{kGPU, dev};
    const bool sym = PG() != nullptr;
    for (auto m : kReplicaState) {
      if ((src.*m).is_none()) continue;
      nr.*m = NDArray::Empty(ks.shape, nctx, kFloat32, sym);
      CopyFromTo(src.*m, nr.*m);
    }
  } else {
    MXKV_CHECK(!ks.init_value.is_none()) << "key " << ks.key << " has no initial value";
    CopyFromTo(ks.init_value, nr.local);
    // the pageable H2D copy above is synchronous w.r.t. the host buffer; safe to drop it
    rt->WaitDevice(dev);
    ks.init_value = NDArray();
  }
  ks.reps.push_back(nr);
  return ks.reps.back();
}

// Bring the optimizer state of a replica up to date from a replica whose state is (replicated layout only;
// a sharded layout is made complete everywhere by GatherState first).
void KVStore::SyncState(KeyState& ks, Replica& r) {
  if (r.state_fresh) return;
  for (auto& s : ks.reps) {
    if (&s == &r || !s.state_fresh || !HoldsState(s)) continue;
    for (auto m : kReplicaState)
      if (!(s.*m).is_none() && !(r.*m).is_none()) CopyFromTo(s.*m, r.*m);
    r.state_fresh = true;
    return;
  }
  r.state_fresh = true;     // nobody holds newer state (first use)
}

void KVStore::EnsureState(KeyState& ks, Replica& r, bool mp) {
  Runtime* rt = Runtime::Get();
  const bool sym = PG() != nullptr;
  const Context ctx{kGPU, r.dev};
  DeviceGuard g(r.dev);
  cudaStream_t s = rt->Dev(r.dev).stream;
  const bool need_s0 = OptHasS0(opt_.kind) || opt_.kind == OPT_LAMB || opt_.kind == OPT_LANS ||
                       (opt_.kind == OPT_LARS && opt_.momentum != 0.f);      // lars.py:96-101
  const bool need_s1 = OptHasS1(opt_.kind) || opt_.kind == OPT_LAMB || opt_.kind == OPT_LANS;
  if (IsNormOpt(opt_.kind)) {
    // temporaries between the phases and the per-key totals the peers read (allocated collectively
    // in one-process-per-GPU mode: every rank reaches this point for the same keys in the same order)
    if (r.aux0.is_none()) r.aux0 = NDArray::Empty(ks.shape, ctx, kFloat32, false);
    if (opt_.kind == OPT_LANS && r.aux1.is_none()) r.aux1 = NDArray::Empty(ks.shape, ctx, kFloat32, false);
    if (r.nrm.is_none()) {
      r.nrm = NDArray::Empty({kNrmFloats}, ctx, kFloat32, sym);
      CUDA_CALL(cudaMemsetAsync(r.nrm.data(), 0, r.nrm.nbytes(), s));
    }
  }
  bool created = false;
  if (mp && r.w32.is_none()) {
    created = true;
    r.w32 = NDArray::Empty(ks.shape, ctx, kFloat32, sym);
    // create_state_multi_precision: weight_master_copy = weight.astype(float32) (optimizer.py:341-352)
    MXKV_CHECK(ks.dtype == kFloat32 || ks.dtype == kFloat16 || ks.dtype == kBfloat16)
        << "multi_precision needs a floating-point key";
    const int rc = LaunchCastToF32(r.local.data(), ks.dtype, static_cast<float*>(r.w32.data()), ks.size, s);
    MXKV_CHECK(rc == 0) << "cast kernel launch failed: " << cudaGetErrorString(static_cast<cudaError_t>(rc));
    rt->launches++;
  }
  if (need_s0 && r.s0.is_none()) {
    created = true;
    r.s0 = NDArray::Empty(ks.shape, ctx, kFloat32, sym);
    CUDA_CALL(cudaMemsetAsync(r.s0.data(), 0, r.s0.nbytes(), s));
  }
  if (need_s1 && r.s1.is_none()) {
    created = true;
    r.s1 = NDArray::Empty(ks.shape, ctx, kFloat32, sym);
    CUDA_CALL(cudaMemsetAsync(r.s1.data(), 0, r.s1.nbytes(), s));
  }
  if (OptHasS2(opt_.kind) && r.s2.is_none()) {
    created = true;
    r.s2 = NDArray::Empty(ks.shape, ctx, kFloat32, sym);
    CUDA_CALL(cudaMemsetAsync(r.s2.data(), 0, r.s2.nbytes(), s));
  }
  // state arrays that come into being after updates have already happened elsewhere start out stale:
  // SyncState fills them from a replica that took part (zeros / a cast of the weight are only right for
  // the very first update)
  if (created && ks.count > 0 && ks.reps.size() > 1) r.state_fresh = false;
  ks.has_state = true;
}

// ---------------------------------------------------------------------------
// Init (kvstore_local.h:227-238).  The reference parks the value in pinned host memory
// until the first push reveals the devices; so do we, except that a GPU-resident value
// immediately becomes the first replica.  One-process-per-GPU mode: rank 0's value wins
// (the contract of KVStoreBase.broadcast, python/mxnet/kvstore/base.py:77-96).
// ---------------------------------------------------------------------------
void KVStore::InitImpl(const std::vector<int>& keys, const std::vector<NDArray>& vals) {
  MXKV_CHECK(keys.size() == vals.size()) << "Init: " << keys.size() << " keys but " << vals.size() << " values";
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  for (size_t i = 0; i < keys.size(); ++i) {
    MXKV_CHECK(keys_.find(keys[i]) == keys_.end())
        << "duplicate init of key " << keys[i]
        << ". Please double check if you called kv.init or kv.broadcast with this key multiple times";
    const NDArray& v = vals[i];
    MXKV_CHECK(!v.is_none()) << "Init: empty value for key " << keys[i];
    KeyState ks;
    ks.key = keys[i];
    ks.shape = v.shape();
    ks.dtype = v.dtype();
    ks.stype = v.stype();
    ks.size = v.size();
    if (v.stype() == kRowSparseStorage) {
      keys_[keys[i]] = ks;
      InitRowSparseKey(keys_[keys[i]], v);
      continue;
    }
    MXKV_CHECK(v.stype() == kDefaultStorage) << "Init: unsupported storage type " << v.stype();
    const Context c = v.ctx();
    if (c.is_gpu() || pg != nullptr) {
      const int dev = pg ? pg->dev() : c.dev_id;
      if (c.is_gpu()) rt->AcquireUser(c.dev_id);
      ks.init_value = v;   // EnsureReplica copies from it (D2D / H2D / peer)
      keys_[keys[i]] = ks;
      KeyState& k2 = keys_[keys[i]];
      Replica& r = EnsureReplica(k2, dev);
      if (pg && pg->world() > 1) BroadcastFromRank0(k2, r);
      if (pg && hier_) {
        // ... and every node adopts node 0's value (rank 0 of the job initialises, kvstore_dist.h:196-223):
        // the other nodes contribute zeros to an inter-node sum
        if (rt->hier.node_rank != 0) {
          DeviceGuard g(dev);
          CUDA_CALL(cudaMemsetAsync(r.local.data(), 0, r.local.nbytes(), rt->Dev(dev).stream));
        }
        InterNodeSum(r.local.data(), k2.size, k2.dtype, dev);
      }
      rt->ReleaseToUser(dev);
    } else {
      // host value, devices unknown yet: keep a private host copy (values[i].Copy(pinned_ctx_))
      rt->WaitAll();
      ks.init_value = NDArray::Empty(v.shape(), Context{kCPU, 0}, v.dtype());
      std::memcpy(ks.init_value.data(), v.data(), v.nbytes());
      keys_[keys[i]] = ks;
    }
  }
}

// one-process-per-GPU mode: every rank adopts rank 0's stored value (one-shot read of rank 0's
// replica; rank 0 copies onto itself).  Collective.
void KVStore::BroadcastFromRank0(KeyState& ks, Replica& r) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  if (pg == nullptr || pg->world() <= 1) return;
  TensorWork tw;
  std::memset(&tw, 0, sizeof(tw));
  tw.src[0] = r.local.peer_data(0);
  tw.n_src = 1;
  tw.out[0] = r.local.data();
  tw.n_out = 1;
  tw.begin = 0; tw.end = r.local.size();
  tw.flags = WorkFlags(tw, r.local.dtype() == kFloat32 && r.local.size() % 4 == 0);
  std::vector<int> part_dev(pg->world(), pg->dev());
  std::vector<std::vector<TensorWork>> per_part(pg->world());
  per_part[pg->rank()].push_back(tw);
  LaunchClassKey ck{SYNC_READ_PEERS, r.local.dtype(), 0};
  LaunchWorks(ck, per_part, {r.local.size()}, OPT_NONE, part_dev);
}

// ---------------------------------------------------------------------------
// GroupKVPairs (kvstore_local.h:440-469): std::sort on the key only, then group
// ---------------------------------------------------------------------------
template <typename V>
static void GroupPairs(const std::vector<int>& keys, const std::vector<V>& vals,
                       std::vector<int>* uniq, std::vector<std::vector<V>>* grouped,
                       const std::function<bool(int, const V&)>& valid) {
  MXKV_CHECK(keys.size() == vals.size()) << keys.size() << " keys but " << vals.size() << " values";
  std::vector<std::pair<int, int>> idx(keys.size());
  for (size_t i = 0; i < keys.size(); ++i) idx[i] = {keys[i], static_cast<int>(i)};
  std::stable_sort(idx.begin(), idx.end(),
                   [](const std::pair<int, int>& a, const std::pair<int, int>& b) { return a.first < b.first; });
  bool have = false;
  int pre = 0;
  for (auto& p : idx) {
    if (!valid(p.first, vals[p.second])) continue;
    if (!have || p.first != pre) {
      uniq->push_back(p.first);
      grouped->push_back({vals[p.second]});
      pre = p.first; have = true;
    } else {
      grouped->back().push_back(vals[p.second]);
    }
  }
}

void KVStore::PushImpl(const std::vector<int>& keys, const std::vector<NDArray>& vals, int priority) {
  (void)priority;      // consumed by the deferred queue (Flush): by the time a call gets here its turn has come
  std::vector<int> uniq;
  std::vector<std::vector<NDArray>> grouped;
  GroupPairs<NDArray>(keys, vals, &uniq, &grouped, [](int, const NDArray& nd) {
    MXKV_CHECK(nd.stype() == kDefaultStorage || nd.stype() == kRowSparseStorage)
        << "Unexpected storage type detected during kvstore push: " << nd.stype();
    return true;
  });
  std::vector<Group> dense, skipped;
  for (size_t i = 0; i < uniq.size(); ++i) {
    KeyState& ks = PeekKey(uniq[i]);
    if (grouped[i][0].stype() == kRowSparseStorage || ks.stype == kRowSparseStorage) {
      PushRowSparse(GetKey(uniq[i]), grouped[i]);
      continue;
    }
    if (SkipsOnRescale()) {
      Group g;
      g.key = uniq[i];
      g.vals = grouped[i];
      skipped.push_back(g);
      continue;
    }
    // BASELINE configs[0], the reference's CPU-runnable case: ONE host-resident value pushed to a key that has
    // never met a GPU, nothing to run on it (no updater, no optimizer, no compression).  The reference does no
    // arithmetic here either -- Reduce hands a single value back as it is (comm.h:128-131) and the store copies it
    // over the stored value (kvstore_local.h:279-284) -- so this is plumbing, served without a device.  Anything
    // that would need a sum or an update still fails loudly without a GPU (DefaultDevice).
    if (grouped[i].size() == 1 && !grouped[i][0].ctx().is_gpu() && ks.reps.empty() && !ks.init_value.is_none() &&
        !ks.init_value.ctx().is_gpu() && updater_ == nullptr && !opt_.enabled && gc_bits_ == 0 && !hier_ &&
        PG() == nullptr && Runtime::Get()->NumDevices() == 0) {
      const NDArray& v = grouped[i][0];
      MXKV_CHECK(v.size() == ks.size) << "push: value has " << v.size() << " elements, key " << ks.key
                                      << " was initialised with " << ks.size;
      MXKV_CHECK(v.dtype() == ks.dtype) << "push: dtype mismatch for key " << ks.key
                                        << " (Only support input/output with the same data type)";
      GetKey(uniq[i]);                               // (a change of the key: cached plans of it expire)
      std::memcpy(ks.init_value.data(), v.data(), v.nbytes());
      continue;
    }
    Group g;
    g.key = uniq[i];
    g.vals = grouped[i];
    dense.push_back(g);
  }
  if (!skipped.empty()) SkipStep(skipped);
  raw_single_ = dense.size() == uniq.size();        // the whole call as ONE reduce: a launch plan may be recorded
  if (!dense.empty()) ReduceUpdate(dense, false);
  raw_single_ = false;
}

void KVStore::PullImpl(const std::vector<int>& keys, const std::vector<NDArray*>& outs, int priority,
                       bool ignore_sparse) {
  (void)priority;
  std::vector<int> uniq;
  std::vector<std::vector<NDArray*>> grouped;
  GroupPairs<NDArray*>(keys, outs, &uniq, &grouped, [this, ignore_sparse](int key, NDArray* const& nd) {
    if (nd->stype() == kDefaultStorage || !ignore_sparse) return true;
    if (warnings_printed_.insert(key).second) {
      fprintf(stderr, "Warning: non-default weights detected during kvstore pull. This call has been "
                      "ignored. Please make sure to use kv.row_sparse_pull() or module.prepare() with row_ids.\n");
    }
    return false;
  });
  Runtime* rt = Runtime::Get();
  std::set<int> touched;
  for (size_t i = 0; i < uniq.size(); ++i) {
    KeyState& ks = GetKey(uniq[i]);
    if (ks.stype == kRowSparseStorage) {
      PullDenseFromRowSparse(ks, grouped[i]);
      continue;
    }
    if (ks.local_world > 0) GatherLocal(ks);       // the all-gather half of a sharded push
    for (NDArray* o : grouped[i]) {
      MXKV_CHECK(o->stype() == kDefaultStorage) << "pull into a sparse array is not supported for dense keys";
      MXKV_CHECK(o->size() == ks.size) << "pull: output has " << o->size() << " elements, key " << ks.key
                                       << " has " << ks.size;
      MXKV_CHECK(o->dtype() == ks.dtype) << "pull: dtype mismatch for key " << ks.key;
      const Context c = o->ctx();
      if (c.is_gpu()) {
        if (touched.insert(c.dev_id).second) rt->AcquireUser(c.dev_id);
        if (rt->pg() == nullptr || c.dev_id == rt->pg()->dev()) {
          Replica& r = EnsureReplica(ks, c.dev_id);   // comm.h:607-625, but from the local replica
          CopyFromTo(r.local, *o);
          continue;
        }
      }
      if (ks.reps.empty()) {
        if (!c.is_gpu()) {            // never touched a GPU: host -> host
          CopyFromTo(ks.init_value, *o);
          continue;
        }
        EnsureReplica(ks, DefaultDevice());
      }
      CopyFromTo(FreshReplica(ks).local, *o);
    }
  }
  for (int d : touched) rt->ReleaseToUser(d);
}

void KVStore::PushPullImpl(const std::vector<int>& vkeys, const std::vector<int>& okeys,
                           const std::vector<NDArray>& vals, const std::vector<NDArray*>& outs, int priority) {
  // fused path when the pushed and the pulled key sets coincide and everything is dense;
  // otherwise literally Push then Pull (kvstore_local.h:358-365).
  std::vector<int> vu, ou;
  std::vector<std::vector<NDArray>> vg;
  std::vector<std::vector<NDArray*>> og;
  bool dense = true;
  GroupPairs<NDArray>(vkeys, vals, &vu, &vg, [&dense](int, const NDArray& nd) {
    if (nd.stype() != kDefaultStorage) dense = false;
    return true;
  });
  GroupPairs<NDArray*>(okeys, outs, &ou, &og, [&dense](int, NDArray* const& nd) {
    if (nd->stype() != kDefaultStorage) dense = false;
    return true;
  });
  bool fusable = dense && vu == ou && updater_ == nullptr;
  if (fusable) {
    for (int k : vu) if (PeekKey(k).stype != kDefaultStorage) fusable = false;
  }
  // no device at all: literally push then pull, so that the one case that is pure plumbing (PushImpl) is served
  if (fusable && PG() == nullptr && Runtime::Get()->NumDevices() == 0) fusable = false;
  if (!fusable) {
    PushImpl(vkeys, vals, priority);
    PullImpl(okeys, outs, priority, true);
    return;
  }
  std::vector<Group> groups(vu.size());
  for (size_t i = 0; i < vu.size(); ++i) {
    groups[i].key = vu[i];
    groups[i].vals = vg[i];
    groups[i].outs = og[i];
  }
  if (SkipsOnRescale()) {
    SkipStep(groups);
    PullImpl(okeys, outs, priority, true);
    return;
  }
  raw_single_ = true;
  ReduceUpdate(groups, true);
  raw_single_ = false;
}

// ---------------------------------------------------------------------------
// the hot path
// ---------------------------------------------------------------------------
// two-shot partition: rank p owns elements [p*L, (p+1)*L) clipped to the key, L = ceil(size/n)
// rounded up to 128 elements so that every shard starts 16-byte aligned for any dtype
int64_t ShardLen(int64_t size, int world) {
  int64_t shard = (size + world - 1) / world;
  return (shard + 127) / 128 * 128;
}

struct KVStore::Dest {
  void* ptr[kMaxRanks];   // address as seen by participant p (MP: peer mapping; SP: same everywhere)
  int owner;              // participant index that owns the memory, -1: none, -2: one copy per rank (MP)
  bool own_only = false;  // two-shot: only the owning participant writes (its own shard of its own copy)
  void* mc = nullptr;     // NVSwitch multicast alias of all copies (one store reaches every rank)
};

namespace {
struct PostCopy { NDArray src; NDArray dst; };
inline bool Overlap(const void* a, size_t an, const void* b, size_t bn) {
  const char* x = static_cast<const char*>(a);
  const char* y = static_cast<const char*>(b);
  return x < y + bn && y < x + an;
}
inline bool Aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
}  // namespace

// Outputs of one key that alias the pushed values of ANOTHER key of the same call (the reference's
// tests do this: the same arrays are pushed for every key and pulled in place).  The reference runs
// every reduce of a call before any pull (PushImpl then PullImpl, kvstore_local.h:358-365), so such
// outputs must not be written by the fused kernel -- they are copied out after all kernels.
namespace {
class AliasIndex {
 public:
  template <typename Groups>
  explicit AliasIndex(const Groups& groups) {
    for (size_t gi = 0; gi < groups.size(); ++gi)
      for (auto& v : groups[gi].vals) {
        const char* b = static_cast<const char*>(v.data());
        if (b != nullptr && v.nbytes() > 0) iv_.push_back({b, b + v.nbytes(), static_cast<int>(gi)});
      }
    std::sort(iv_.begin(), iv_.end(), [](const Iv& a, const Iv& b) { return a.b < b.b; });
    // running maximum of interval ends for the overlap query
    maxe_.resize(iv_.size());
    const char* m = nullptr;
    for (size_t i = 0; i < iv_.size(); ++i) { if (i == 0 || iv_[i].e > m) m = iv_[i].e; maxe_[i] = m; }
  }
  // does [p, p+n) overlap a pushed value of a group other than `gi`?
  bool OverlapsOther(const void* p, size_t n, int gi) const {
    if (iv_.empty() || p == nullptr || n == 0) return false;
    const char* b = static_cast<const char*>(p);
    const char* e = b + n;
    // intervals with begin < e
    size_t hi = std::lower_bound(iv_.begin(), iv_.end(), e, [](const Iv& a, const char* x) { return a.b < x; }) - iv_.begin();
    for (size_t i = hi; i-- > 0;) {
      if (maxe_[i] <= b) break;                 // nothing at or before i reaches into [b, e)
      if (iv_[i].e > b && iv_[i].g != gi) return true;
    }
    return false;
  }
 private:
  struct Iv { const char* b; const char* e; int g; };
  std::vector<Iv> iv_;
  std::vector<const char*> maxe_;
};
}  // namespace

// Host-resident values and outputs (kv.create('local')-style use, and the end-to-end benchmark):
// instead of "copy everything in, run, copy everything out" on one stream, every key is cut into
// segments that flow through a three-stage pipeline on three streams -- H2D of segment i+1, the
// fused kernel on segment i and D2H of segment i-1 overlap, so PCIe runs full duplex and the
// kernel is hidden.  The kernel is the same work-list kernel, launched on an element range.
bool KVStore::HostPipelined(std::vector<Group>& groups, bool write_outs) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  // one process per GPU: every rank streams ITS host value through its own PCIe link into a peer-mapped slot, and
  // every rank's kernel sums all ranks' slots for the segment (one-shot: NVLink carries (n-1) x the segment, which
  // is still several times faster than the PCIe copy it hides behind) and updates its own complete replica -- the
  // optimizer state stays replicated, nothing is written across GPUs.  The decision below must come out the same
  // on every rank (the same call with host-resident values everywhere), like every other collective call.
  const bool coll = pg != nullptr && pg->world() > 1;
  if (coll && (hier_ || EnvInt("MXKV_B200_HOST_PIPELINE_MP", 1) == 0)) return false;
  if (updater_ != nullptr) return false;
  if (opt_.enabled && IsNormOpt(opt_.kind)) return false;   // per-key norms need the whole key in one launch
  if (EnvInt("MXKV_B200_HOST_PIPELINE", 1) == 0) return false;
  int64_t total_bytes = 0;
  for (auto& g : groups) {
    KeyState& ks = GetKey(g.key);
    if (ks.stype != kDefaultStorage) return false;
    if (static_cast<int>(g.vals.size()) > kMaxSrc) return false;
    if (coll && g.vals.size() != 1) return false;
    for (auto& v : g.vals) {
      if (v.ctx().is_gpu()) return false;
      if (v.size() != ks.size || v.dtype() != ks.dtype) return false;   // let the generic path report it
    }
    if (write_outs) {
      for (NDArray* o : g.outs) {
        if (o->ctx().is_gpu()) return false;
        if (o->size() != ks.size || o->dtype() != ks.dtype) return false;
      }
    }
    total_bytes += static_cast<int64_t>(ks.size) * DTypeSize(ks.dtype) * g.vals.size();
  }
  if (total_bytes < (int64_t(1) << 20)) return false;      // latency-bound: the simple path is fine
  if (write_outs && groups.size() > 1) {
    AliasIndex alias(groups);
    for (size_t gi = 0; gi < groups.size(); ++gi)
      for (NDArray* o : groups[gi].outs)
        if (alias.OverlapsOther(o->data(), o->nbytes(), static_cast<int>(gi))) return false;
  }

  const bool fused = opt_.enabled;
  const int opt_kind = fused ? opt_.kind : OPT_NONE;
  int dev = -1;
  for (auto& g : groups) {
    KeyState& ks = GetKey(g.key);
    if (!ks.reps.empty()) { dev = ks.reps[0].dev; break; }
  }
  if (dev < 0) dev = DefaultDevice();
  if (coll) dev = pg->dev();
  const int world = coll ? pg->world() : 1;
  const int me = coll ? pg->rank() : 0;
  DeviceState& d = rt->Dev(dev);
  DeviceGuard dg(dev);
  const int64_t seg_elems = std::max<int64_t>(rt->chunk_elems, EnvInt("MXKV_B200_HOST_SEG_ELEMS", 4 << 20)) /
                            rt->chunk_elems * rt->chunk_elems;
  // staging slots: kMaxSrc is the worst case, size for what this call needs
  size_t need = 0;
  for (auto& g : groups) {
    KeyState& ks = GetKey(g.key);
    const size_t seg_bytes = static_cast<size_t>(std::min<int64_t>(seg_elems, ks.size)) * DTypeSize(ks.dtype);
    need = std::max(need, ((seg_bytes + 255) / 256 * 256) * g.vals.size());
  }
  if (coll) {
    if (need > d.host_stage_peer_bytes) {          // collective allocation: `need` follows from the key sizes alone
      for (int i = 0; i < DeviceState::kHostSlots; ++i) {
        SymPtr sp = pg->SymAlloc(need);
        for (int q = 0; q < world; ++q) d.host_stage_peer[i][q] = sp.ptr[q];
      }
      d.host_stage_peer_bytes = need;
    }
  } else if (need > d.host_stage_bytes) {
    rt->WaitDevice(dev);
    CUDA_CALL(cudaStreamSynchronize(d.copy_in));
    CUDA_CALL(cudaStreamSynchronize(d.copy_out));
    for (int i = 0; i < DeviceState::kHostSlots; ++i) {
      if (d.host_stage[i]) CUDA_CALL(cudaFree(d.host_stage[i]));
      CUDA_CALL(cudaMalloc(&d.host_stage[i], need));
    }
    d.host_stage_bytes = need;
  }
  // outputs of the previous call may still be streaming out of the replicas
  CUDA_CALL(cudaStreamWaitEvent(d.stream, d.ev_d2h_all, 0));
  // the staging slots may still be read by kernels of the previous call
  for (int i = 0; i < DeviceState::kHostSlots; ++i) CUDA_CALL(cudaStreamWaitEvent(d.copy_in, d.ev_kern[i], 0));

  int64_t seq = 0;
  std::vector<int> part_dev(world, dev);
  for (auto& g : groups) {
    KeyState& ks = GetKey(g.key);
    const size_t esize = DTypeSize(ks.dtype);
    Replica* r = &EnsureReplica(ks, dev);
    if (ks.local_world > 0) GatherLocal(ks);
    const bool lowp = ks.dtype == kFloat16 || ks.dtype == kBfloat16;
    const bool mp = fused && (opt_.multi_precision || lowp);
    if (fused) {
      MXKV_CHECK(ks.dtype == kFloat32 || lowp) << "fused optimizers need float32/float16/bfloat16 keys";
      if (ks.has_state) GatherState(ks);
      EnsureState(ks, *r, mp);
      ks.state_world = 0;
      StepKey(ks);
    }
    r = FindReplica(ks, dev);
    if (fused) SyncState(ks, *r);
    for (auto& o : ks.reps) {
      o.fresh = (&o == r);
      if (fused && &o != r) o.state_fresh = false;
    }
    const int n_src = static_cast<int>(g.vals.size());
    const size_t slot_stride = ((static_cast<size_t>(std::min<int64_t>(seg_elems, ks.size)) * esize + 255) / 256) * 256;
    for (int64_t b = 0; b < ks.size || (ks.size == 0 && b == 0); b += seg_elems) {
      const int64_t e = std::min<int64_t>(ks.size, b + seg_elems);
      if (e <= b) break;
      const int slot = static_cast<int>(seq % DeviceState::kHostSlots);
      const size_t bytes = static_cast<size_t>(e - b) * esize;
      // stage 1: H2D (the slot is free once the kernel that last read it has finished)
      if (seq >= DeviceState::kHostSlots) CUDA_CALL(cudaStreamWaitEvent(d.copy_in, d.ev_kern[slot], 0));
      for (int k = 0; k < n_src; ++k) {
        char* dst = coll ? static_cast<char*>(d.host_stage_peer[slot][me])
                         : static_cast<char*>(d.host_stage[slot]) + k * slot_stride;
        const char* src = static_cast<const char*>(g.vals[k].data()) + static_cast<size_t>(b) * esize;
        CUDA_CALL(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, d.copy_in));
      }
      CUDA_CALL(cudaEventRecord(d.ev_h2d[slot], d.copy_in));
      // stage 2: fused reduce(+update) on the element range [b, e)
      CUDA_CALL(cudaStreamWaitEvent(d.stream, d.ev_h2d[slot], 0));
      TensorWork tw = ReplicaWork(ks, *r, fused, mp, b, e);
      if (coll) {               // rank q's slot as mapped here; the start rendezvous orders it after q's H2D
        tw.n_src = world;
        for (int q = 0; q < world; ++q)
          tw.src[q] = static_cast<char*>(d.host_stage_peer[slot][q]) - static_cast<size_t>(b) * esize;
      } else {
        tw.n_src = n_src;
        for (int k = 0; k < n_src; ++k)
          tw.src[k] = static_cast<char*>(d.host_stage[slot]) + k * slot_stride - static_cast<size_t>(b) * esize;
      }
      tw.out[tw.n_out++] = r->local.data();
      tw.flags = WorkFlags(tw, esize == 4 && ks.size % 4 == 0);
      std::vector<std::vector<TensorWork>> per_part(world);
      per_part[me].push_back(tw);
      // (the end rendezvous of a collective launch also tells this rank that no peer still reads its slot)
      LaunchClassKey ck{coll ? SYNC_WRITE_PEERS : SYNC_NONE, ks.dtype, mp ? 1 : 0};
      LaunchWorks(ck, per_part, {e - b}, opt_kind, part_dev);
      CUDA_CALL(cudaEventRecord(d.ev_kern[slot], d.stream));
      // stage 3: D2H of the freshly written range of the replica
      if (write_outs && !g.outs.empty()) {
        CUDA_CALL(cudaStreamWaitEvent(d.copy_out, d.ev_kern[slot], 0));
        for (NDArray* o : g.outs) {
          char* dst = static_cast<char*>(o->data()) + static_cast<size_t>(b) * esize;
          const char* src = static_cast<const char*>(r->local.data()) + static_cast<size_t>(b) * esize;
          CUDA_CALL(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, d.copy_out));
        }
      }
      ++seq;
    }
  }
  CUDA_CALL(cudaEventRecord(d.ev_d2h_all, d.copy_out));
  // WaitToRead / WaitAll synchronise the engine stream: make it cover the copies as well
  CUDA_CALL(cudaStreamWaitEvent(d.stream, d.ev_d2h_all, 0));
  return true;
}

// CommDevice::ReduceCompressed (src/kvstore/comm.h:556-605): every pushed value is quantised on its
// own GPU against a per-source residual (error feedback), the 16x / 32x smaller code stream is what
// crosses the interconnect, and the consumer dequantises and sums.  Here every participating GPU is
// a consumer: it reads all n code streams (peer loads), dequantises them into local scratch and
// runs the ordinary fused reduce(+update) kernel on its own replica -- no root, no broadcast.
void KVStore::ReduceUpdateCompressed(std::vector<Group>& groups, bool write_outs, bool quantize_only) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  const bool mp_mode = pg != nullptr;
  const bool callback = updater_ != nullptr;
  MXKV_CHECK(!callback) << "gradient compression together with a Python updater callback is not supported; "
                           "use a fused optimizer or no optimizer";
  // multi-node phase 1 (HierReduceUpdate): quantise, exchange the codes inside the node, sum the dequantised
  // streams into the staging slice; nothing stored, nothing updated
  const bool stage_only = hier_phase_ == 1;
  const bool fused = opt_.enabled && !stage_only;
  const int opt_kind = fused ? opt_.kind : OPT_NONE;
  const int world = mp_mode ? pg->world() : 1;
  std::set<int> touched;
  auto touch = [&](int dev) { if (dev >= 0 && touched.insert(dev).second) rt->AcquireUser(dev); };
  std::vector<PostCopy> post;
  std::vector<std::pair<void*, int>> temps;
  const AliasIndex alias(groups);

  for (size_t gi = 0; gi < groups.size(); ++gi) {
    auto& g = groups[gi];
    KeyState& ks = GetKey(g.key);
    MXKV_CHECK(ks.dtype == kFloat32) << "Gradient compression is only supported for float32";   // gradient_compression.cc
    const int n_src = static_cast<int>(g.vals.size());
    MXKV_CHECK(n_src >= 1 && n_src <= kMaxSrc) << "push of " << n_src << " values for one key";
    if (mp_mode) MXKV_CHECK(n_src == 1) << "one-process-per-GPU mode: push exactly one value per key per rank";
    const int per_word = 32 / gc_bits_;
    const int64_t nwords = (ks.size + per_word - 1) / per_word;
    // ---- 1. quantise every value where it lives ---------------------------------------------
    if (static_cast<int>(ks.gc_residual.size()) < n_src) { ks.gc_residual.resize(n_src); ks.gc_packed.resize(n_src); }
    std::vector<int> src_dev(n_src);
    for (int k = 0; k < n_src; ++k) {
      const NDArray& v = g.vals[k];
      MXKV_CHECK(v.size() == ks.size && v.dtype() == ks.dtype) << "push: value does not match key " << ks.key;
      const Context c = v.ctx();
      const int dev = mp_mode ? pg->dev() : (c.is_gpu() ? c.dev_id : (ks.reps.empty() ? DefaultDevice() : ks.reps[0].dev));
      src_dev[k] = dev;
      touch(dev);
      if (ks.gc_residual[k].is_none()) {
        ks.gc_residual[k] = NDArray::Empty(ks.shape, Context{kGPU, dev}, kFloat32);
        ks.gc_packed[k] = NDArray::Empty({nwords}, Context{kGPU, dev}, kInt32, mp_mode);
        DeviceGuard dg(dev);
        CUDA_CALL(cudaMemsetAsync(ks.gc_residual[k].data(), 0, ks.gc_residual[k].nbytes(), rt->Dev(dev).stream));
      } else if (ks.gc_residual[k].dev() != dev) {
        // value slot k is now pushed from another GPU: its error feedback moves along (the reference
        // allocates the residuals on the contexts of the first push and has no answer for a later change)
        touch(ks.gc_residual[k].dev());
        NDArray moved = NDArray::Empty(ks.shape, Context{kGPU, dev}, kFloat32);
        CopyFromTo(ks.gc_residual[k], moved);
        ks.gc_residual[k] = moved;
        ks.gc_packed[k] = NDArray::Empty({nwords}, Context{kGPU, dev}, kInt32, mp_mode);
      }
      DeviceGuard dg(dev);
      cudaStream_t s = rt->Dev(dev).stream;
      const float* gptr = static_cast<const float*>(v.data());
      if (!(c.is_gpu() && c.dev_id == dev)) {     // host value: stage it
        void* t = nullptr;
        CUDA_CALL(cudaMallocAsync(&t, std::max<size_t>(v.nbytes(), 16), s));
        CopyBytes(v.data(), c, t, Context{kGPU, dev}, v.nbytes());
        temps.push_back({t, dev});
        gptr = static_cast<const float*>(t);
      }
      const int rc = LaunchQuantize(gc_bits_, gptr, static_cast<float*>(ks.gc_residual[k].data()),
                                    static_cast<uint32_t*>(ks.gc_packed[k].data()), ks.size, gc_threshold_, s);
      MXKV_CHECK(rc == 0) << "quantize launch failed: " << cudaGetErrorString(static_cast<cudaError_t>(rc));
      rt->launches++;
    }
    // a skipped step (SkipStep): the residuals have advanced, nobody reads these codes (the next call's quantise
    // is ordered after this call's on the same stream, and after every earlier call's reads by its end waits)
    if (quantize_only) { StepKey(ks); continue; }
    // ---- 2. consumers: every GPU that holds (or must hold) a replica ----------------------------
    std::vector<int> consumers;
    if (mp_mode) consumers.push_back(pg->dev());
    else {
      for (int d : src_dev) if (std::find(consumers.begin(), consumers.end(), d) == consumers.end()) consumers.push_back(d);
      for (auto& r : ks.reps) if (std::find(consumers.begin(), consumers.end(), r.dev) == consumers.end()) consumers.push_back(r.dev);
      rt->EnablePeerAccess(consumers);
    }
    SyncArgs sync{};
    if (world > 1) {
      sync = GroupSync(SYNC_WRITE_PEERS);
      DeviceGuard dg(pg->dev());
      sync.epoch = rt->NextSyncEpoch(pg);
      MXKV_CHECK(LaunchBarrier(sync, rt->Dev(pg->dev()).stream) == 0) << "barrier launch failed";   // codes published
      rt->launches++;
    }
    const int n_total = mp_mode ? world : n_src;
    const bool mp = fused && opt_.multi_precision;
    std::set<NDArray*> written;
    if (fused) StepKey(ks);
    // every consumer's replica, master and state are made current before the first consumer updates its own: one
    // made (or refreshed) afterwards would be copied from an updated replica and take the step twice
    for (int dev : consumers) {
      touch(dev);
      EnsureReplica(ks, dev);
      if (!stage_only && ks.local_world > 0) GatherLocal(ks);
      Replica& r = *FindReplica(ks, dev);
      if (fused) { if (ks.has_state) GatherState(ks); EnsureState(ks, r, mp); ks.state_world = 0; }
    }
    for (int dev : consumers) {
      Replica& r = *FindReplica(ks, dev);
      DeviceGuard dg(dev);
      cudaStream_t s = rt->Dev(dev).stream;
      float* deq = nullptr;
      CUDA_CALL(cudaMallocAsync(reinterpret_cast<void**>(&deq), static_cast<size_t>(n_total) * std::max<int64_t>(ks.size, 4) * 4, s));
      temps.push_back({deq, dev});
      TensorWork tw = ReplicaWork(ks, r, fused, mp, 0, ks.size);
      tw.n_src = n_total;
      for (int k = 0; k < n_total; ++k) {
        const uint32_t* codes;
        if (mp_mode) {
          codes = static_cast<const uint32_t*>(world > 1 ? ks.gc_packed[0].peer_data(k) : ks.gc_packed[0].data());
        } else {
          if (src_dev[k] != dev) {
            MXKV_CHECK(rt->PeerOK(dev, src_dev[k])) << "gradient compression needs peer access between GPU " << dev
                                                    << " and GPU " << src_dev[k];
            rt->StreamWait(dev, src_dev[k]);
          }
          codes = static_cast<const uint32_t*>(ks.gc_packed[k].data());
        }
        float* out = deq + static_cast<size_t>(k) * ks.size;
        const int rc = LaunchDequantize(gc_bits_, codes, out, ks.size, gc_threshold_, s);
        MXKV_CHECK(rc == 0) << "dequantize launch failed: " << cudaGetErrorString(static_cast<cudaError_t>(rc));
        rt->launches++;
        tw.src[k] = out;
      }
      tw.out[tw.n_out++] = stage_only ? hier_base_.at(ks.key) : r.local.data();
      if (write_outs) {
        for (NDArray* o : g.outs) {
          MXKV_CHECK(o->size() == ks.size && o->dtype() == ks.dtype) << "pushpull: output does not match key " << ks.key;
          const Context oc = o->ctx();
          if (oc.is_gpu() && oc.dev_id == dev && tw.n_out < kMaxOut &&
              !(groups.size() > 1 && alias.OverlapsOther(o->data(), o->nbytes(), static_cast<int>(gi)))) {
            tw.out[tw.n_out++] = o->data();
            written.insert(o);
          }
        }
      }
      tw.flags = ks.size % 4 == 0 ? WorkFlags(tw, true) : 0;   // (other sizes keep the scalar path)
      LaunchLocal(LaunchClassKey{SYNC_NONE, ks.dtype, mp ? 1 : 0}, tw, opt_kind, dev);
      if (!stage_only) r.fresh = true;
    }
    if (world > 1) {
      DeviceGuard dg(pg->dev());
      sync.epoch = rt->NextSyncEpoch(pg);
      MXKV_CHECK(LaunchBarrier(sync, rt->Dev(pg->dev()).stream) == 0) << "barrier launch failed";   // codes consumed
      rt->launches++;
    } else {
      for (int k = 0; k < n_src; ++k)
        for (int dev : consumers) if (dev != src_dev[k]) rt->StreamWait(src_dev[k], dev);
    }
    for (auto& r : ks.reps) {
      if (!stage_only && std::find(consumers.begin(), consumers.end(), r.dev) == consumers.end()) r.fresh = false;
    }
    if (write_outs) {
      for (NDArray* o : g.outs) {
        if (written.count(o)) continue;          // the kernel on that GPU wrote it
        const Context oc = o->ctx();
        if (oc.is_gpu()) touch(oc.dev_id);
        PostCopy pc;
        pc.dst = *o;
        Replica* src = (oc.is_gpu() && FindReplica(ks, oc.dev_id) && FindReplica(ks, oc.dev_id)->fresh)
                           ? FindReplica(ks, oc.dev_id) : &FreshReplica(ks);
        pc.src = src->local;
        post.push_back(pc);
      }
    }
  }
  for (auto& t : temps) {
    DeviceGuard dg(t.second);
    CUDA_CALL(cudaFreeAsync(t.first, rt->Dev(t.second).stream));
  }
  for (auto& pc : post) CopyFromTo(pc.src, pc.dst);
  for (int dev : touched) rt->ReleaseToUser(dev);
}

// Multi-node push (see kvstore.h).  The staging slices of one call are packed per dtype so that the exchange
// between the nodes is ONE all-reduce per dtype, whatever the number of keys; a slice starts on a 256-byte
// boundary and is addressed through a base pointer shifted back by the byte offset of this rank's range, so the
// kernels index it like any other array of the key (and keep their 16-byte vector paths).
void KVStore::HierReduceUpdate(std::vector<Group>& groups, bool write_outs) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  MXKV_CHECK(pg != nullptr) << "multi-node stores run in one-process-per-GPU mode";
  // Gradient compression: every worker quantises against its own residual and the values that are summed are
  // the dequantised ones, as on KVStoreDist's servers (kvstore_dist_server.h:346-398).  The codes travel inside
  // the node; what crosses the network is the node's float32 sum (a sum of codes is not a code), whole keys.
  const bool compressed = gc_bits_ != 0;
  const int n = pg->world(), me = pg->rank(), dev = pg->dev();
  if (updater_ != nullptr) {
    // A Python updater (a user-defined optimizer; on KVStoreDist it runs on the servers from a pickled copy,
    // kvstore_dist_server.h:346-398): every rank receives the whole sum of the job in its `merged` array and runs
    // the callback on its own replica, key by key -- the same update everywhere.
    MXKV_CHECK(!compressed) << "gradient compression together with a Python updater callback is not supported";
    hier_base_.clear();
    rt->AcquireUser(dev);
    for (auto& g : groups) {
      KeyState& ks = GetKey(g.key);
      MXKV_CHECK(ks.stype == kDefaultStorage) << "dist_device_sync: row_sparse keys are not supported (key " << g.key << ")";
      EnsureReplica(ks, dev);
      if (ks.local_world > 0) GatherLocal(ks);
      Replica& root = *FindReplica(ks, dev);
      if (root.merged.is_none()) root.merged = NDArray::Empty(ks.shape, Context{kGPU, dev}, ks.dtype, false);
      hier_base_[g.key] = root.merged.data();
    }
    struct PhaseGuard { int* p; bool* w; ~PhaseGuard() { *p = 0; *w = false; } } guard{&hier_phase_, &hier_whole_keys_};
    hier_whole_keys_ = true;                 // whole keys on every rank in this mode
    hier_phase_ = 1;
    ReduceUpdate(groups, false);
    hier_phase_ = 0;
    hier_whole_keys_ = false;
    for (auto& g : groups) {
      KeyState& ks = GetKey(g.key);
      Replica& root = *FindReplica(ks, dev);
      InterNodeSum(root.merged.data(), ks.size, ks.dtype, dev);
      RunCallbackUpdater(ks, root, root.merged);
      ks.local_world = 0;
    }
    rt->ReleaseToUser(dev);
    if (write_outs) {
      std::vector<int> okeys;
      std::vector<NDArray*> outs;
      for (auto& g : groups) for (NDArray* o : g.outs) { okeys.push_back(g.key); outs.push_back(o); }
      if (!outs.empty()) PullImpl(okeys, outs, 0, true);
    }
    return;
  }
  struct Slice { int key; int dtype; size_t off; int64_t begin; };
  std::vector<Slice> plan;
  std::map<int, size_t> total;
  for (auto& g : groups) {
    KeyState& ks = GetKey(g.key);
    MXKV_CHECK(ks.stype == kDefaultStorage) << "dist_device_sync: row_sparse keys are not supported (key " << g.key << ")";
    const size_t esize = DTypeSize(ks.dtype);
    const bool two_shot = !compressed && n > 1 && static_cast<int64_t>(ks.size * esize) >= rt->twoshot_bytes &&
                          ks.size >= static_cast<int64_t>(n) * 128;
    const int64_t shard = two_shot ? ShardLen(ks.size, n) : ks.size;
    const int64_t begin = two_shot ? std::min<int64_t>(ks.size, shard * me) : 0;
    const int64_t end = two_shot ? std::min<int64_t>(ks.size, shard * (me + 1)) : ks.size;
    size_t& t = total[ks.dtype];
    plan.push_back(Slice{g.key, ks.dtype, t, begin});
    t += (static_cast<size_t>(end - begin) * esize + 255) / 256 * 256;
  }
  for (auto& kv : total) {
    HierBuf& hb = hier_buf_[kv.first];
    if (hb.bytes >= kv.second) continue;
    DeviceGuard g(dev);
    rt->WaitDevice(dev);
    if (hb.ptr != nullptr) CUDA_CALL(cudaFree(hb.ptr));
    hb.bytes = kv.second + kv.second / 4;
    hb.dev = dev;
    CUDA_CALL(cudaMalloc(&hb.ptr, hb.bytes));
    CUDA_CALL(cudaMemset(hb.ptr, 0, hb.bytes));      // the gaps between slices take part in the sums
  }
  hier_base_.clear();
  for (auto& sl : plan)
    hier_base_[sl.key] = static_cast<char*>(hier_buf_[sl.dtype].ptr) + sl.off -
                         static_cast<size_t>(sl.begin) * DTypeSize(sl.dtype);
  struct PhaseGuard { int* p; ~PhaseGuard() { *p = 0; } } guard{&hier_phase_};
  hier_phase_ = 1;
  ReduceUpdate(groups, false);
  for (auto& kv : total)
    InterNodeSum(hier_buf_[kv.first].ptr, static_cast<int64_t>(kv.second / DTypeSize(kv.first)), kv.first, dev);
  hier_phase_ = 2;
  ReduceUpdate(groups, write_outs);
}

// Where a key of a call is reduced: collectively on the GPUs its values live on (distinct,
// P2P-reachable GPUs, single process), by every rank (one process per GPU), or on one root GPU that reads
// and writes wherever the arrays are.
// ---------------------------------------------------------------------------
// cached launch plans (kvstore.h: CallPlan)
// ---------------------------------------------------------------------------
static uint64_t HashSig(const std::vector<uint64_t>& v) {
  uint64_t h = 1469598103934665603ull;
  for (uint64_t x : v) { h ^= x; h *= 1099511628211ull; }
  return h;
}

// The call's raw arguments as a signature: keys in call order, array identities (address, bytes, device, dtype,
// peer-mapped / multicast).  Not eligible (returns false, nothing pending): host-resident or sparse arrays,
// string keys, stores with an updater callback / compression / a node hierarchy / a layer-wise optimizer.
bool KVStore::TryReplayRaw(int kind, uint32_t vnum, const int* vkeys, NDArray* const* vals, uint32_t onum,
                           const int* okeys, NDArray* const* outs) {
  std::lock_guard<std::recursive_mutex> rt_lk(Runtime::Get()->mu());
  std::lock_guard<std::recursive_mutex> lk(mu_);
  raw_pending_ = false;
  raw_single_ = false;
  if (deferred_ || !pending_.empty()) return false;      // the call joins (or must follow) the deferred queue
  if (plan_mode_ == 0 || key_type_ == kStringKey || hier_ || updater_ != nullptr || gc_bits_ != 0 ||
      (opt_.enabled && (IsNormOpt(opt_.kind) || SkipsOnRescale())))
    return false;
  std::vector<uint64_t>& sig = raw_sig_;
  sig.clear();
  sig.reserve(4 + 4 * (static_cast<size_t>(vnum) + onum));
  sig.push_back(static_cast<uint64_t>(kind));
  sig.push_back(vnum);
  sig.push_back(onum);
  auto add = [&sig](int key, const NDArray* a) -> bool {
    if (a == nullptr) return false;
    const Context c = a->ctx();
    if (!c.is_gpu() || a->stype() != kDefaultStorage) return false;
    sig.push_back(static_cast<uint64_t>(static_cast<uint32_t>(key)));
    sig.push_back(reinterpret_cast<uintptr_t>(a->data()));
    sig.push_back(static_cast<uint64_t>(a->nbytes()));
    sig.push_back(static_cast<uint64_t>(c.dev_id) | (a->symmetric() ? 1ull << 32 : 0) |
                  (a->mc_data() != nullptr ? 1ull << 33 : 0) | (static_cast<uint64_t>(a->dtype()) << 40));
    return true;
  };
  for (uint32_t i = 0; i < vnum; ++i) if (!add(vkeys[i], vals[i])) return false;
  for (uint32_t i = 0; i < onum; ++i) if (!add(okeys[i], outs[i])) return false;
  raw_hash_ = HashSig(sig);
  raw_pending_ = true;
  auto it = plans_.find(raw_hash_);
  if (plan_mode_ == 1 && it != plans_.end() && it->second.recorded && it->second.sig == sig &&
      PlanEpochsMatch(it->second)) {
    if (key_type_ == kUndefinedKey) key_type_ = kIntKey;
    PlanPatch(it->second, true);
    IssuePlan(it->second);
    plan_hits_++;
    raw_pending_ = false;
    return true;
  }
  return false;
}

bool KVStore::PlanEpochsMatch(const CallPlan& p) const {
  if (p.cfg_epoch != cfg_epoch_ || p.tuning_epoch != Runtime::Get()->tuning_epoch) return false;
  for (size_t i = 0; i < p.keys.size(); ++i) {
    auto it = keys_.find(p.keys[i]);
    if (it == keys_.end() || it->second.epoch != p.epochs[i]) return false;
  }
  return true;
}

// the only per-call data of a repeated call: update counts and the per-key scalars derived from them
void KVStore::PlanPatch(CallPlan& p, bool commit_counts) {
  if (!p.fused) return;
  std::vector<KeyStep> steps(p.keys.size());
  const double m_schedule = opt_.m_schedule;
  for (size_t i = 0; i < p.keys.size(); ++i) {
    KeyState& ks = keys_.find(p.keys[i])->second;    // (not GetKey: a replay does not expire its own plan)
    const KeyStep prev = ks.step;
    StepKey(ks);                                      // in the group order of the call, as a fresh build does
    steps[i] = ks.step;
    if (!commit_counts) { ks.count -= 1; ks.step = prev; }
  }
  if (!commit_counts) opt_.m_schedule = m_schedule;
  for (auto& l : p.launches)
    for (size_t q = 0; q < l.per_part.size(); ++q)
      for (size_t e = 0; e < l.per_part[q].size(); ++e) {
        TensorWork& tw = l.per_part[q][e];
        const KeyStep& st = steps[l.key_idx[q][e]];
        tw.lr = st.lr; tw.wd = st.wd; tw.eta = st.eta;
      }
}

// Everything a dense call enqueues, in this order; a fresh call runs it once its plan is built, a repeated call
// after PlanPatch.
void KVStore::IssuePlan(CallPlan& p) {
  Runtime* rt = Runtime::Get();
  for (int dev : p.touched) rt->AcquireUser(dev);
  for (auto& w : p.pre_waits) rt->StreamWait(w.first, w.second);
  for (auto& c : p.pre_copies) CopyFromTo(c.first, c.second);
  for (auto& s : p.staged) CopyBytes(s.src.data(), s.src.ctx(), s.tmp, Context{kGPU, s.dev}, s.src.nbytes());
  if (IsNormOpt(p.opt_kind)) {
    // all classes together: the phases of every class are interleaved so that the overflow check
    // covers the whole push
    std::vector<NormClass> all;
    for (auto& l : p.launches) all.push_back(NormClass{l.ck, &l.per_part, &l.busiest});
    LaunchNormWorks(all, p.opt_kind, p.part_dev);
  } else {
    for (auto& l : p.launches) LaunchWorks(l.ck, l.per_part, l.busiest, p.opt_kind, p.part_dev);
  }
  for (auto& s : p.staged) {
    DeviceGuard dg(s.dev);
    CUDA_CALL(cudaFreeAsync(s.tmp, rt->Dev(s.dev).stream));
  }
  // destinations on other GPUs were written by the root's kernel
  if (!p.collective)
    for (int dev : p.touched) if (dev != p.root_dev) rt->StreamWait(dev, p.root_dev);
  if (!p.callback_keys.empty()) {
    ProcessGroup* pg = PG();
    for (KeyState* ks : p.callback_keys) {
      Replica& root = *FindReplica(*ks, p.part_dev[pg ? pg->rank() : 0]);
      RunCallbackUpdater(*ks, root, root.merged);
    }
  }
  for (auto& c : p.post_copies) CopyFromTo(c.first, c.second);
  for (int dev : p.touched) rt->ReleaseToUser(dev);
}

// MXKV_B200_PLAN=2: the replay of a kept plan must issue exactly what the full path builds
bool KVStore::SamePlan(const CallPlan& a, const CallPlan& b) const {
  auto same_copies = [](const std::vector<std::pair<NDArray, NDArray>>& x,
                        const std::vector<std::pair<NDArray, NDArray>>& y) {
    if (x.size() != y.size()) return false;
    for (size_t i = 0; i < x.size(); ++i)
      if (x[i].first.data() != y[i].first.data() || x[i].second.data() != y[i].second.data()) return false;
    return true;
  };
  if (a.launches.size() != b.launches.size() || a.part_dev != b.part_dev || a.touched != b.touched ||
      a.pre_waits != b.pre_waits || !same_copies(a.pre_copies, b.pre_copies) ||
      !same_copies(a.post_copies, b.post_copies) || a.opt_kind != b.opt_kind || a.fused != b.fused ||
      a.collective != b.collective || a.root_dev != b.root_dev || a.repeatable != b.repeatable ||
      a.staged.size() != b.staged.size() || a.callback_keys.size() != b.callback_keys.size())
    return false;
  for (size_t i = 0; i < a.launches.size(); ++i) {
    const PlanLaunch& x = a.launches[i];
    const PlanLaunch& y = b.launches[i];
    if (x.ck < y.ck || y.ck < x.ck || x.busiest != y.busiest || x.per_part.size() != y.per_part.size()) return false;
    for (size_t q = 0; q < x.per_part.size(); ++q)
      if (x.per_part[q].size() != y.per_part[q].size() ||
          (!x.per_part[q].empty() &&
           std::memcmp(x.per_part[q].data(), y.per_part[q].data(), x.per_part[q].size() * sizeof(TensorWork)) != 0))
        return false;
  }
  return true;
}

void KVStore::PlaceKey(const Group& g, KeyState& ks, std::vector<int>* devs_out, std::vector<int>* key_part_out,
                       bool* key_collective_out) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  const bool mp_mode = pg != nullptr;
  const int n_src = static_cast<int>(g.vals.size());
  std::vector<int>& devs = *devs_out;
  std::vector<int>& key_part = *key_part_out;
  bool key_collective = false;
  devs.clear();
  key_part.clear();
  for (auto& v : g.vals) devs.push_back(v.ctx().is_gpu() ? v.ctx().dev_id : -1);
  if (mp_mode) {
    MXKV_CHECK(n_src == 1) << "one-process-per-GPU mode: push exactly one value per key per rank";
    MXKV_CHECK(devs[0] < 0 || devs[0] == pg->dev()) << "value must live on GPU " << pg->dev() << " or on the host";
    key_part.assign(pg->world(), pg->dev());
    key_collective = pg->world() > 1;
  } else {
    bool all_gpu = true, distinct = true;
    std::set<int> seen;
    for (int d : devs) {
      if (d < 0) { all_gpu = false; continue; }
      if (!seen.insert(d).second) distinct = false;
    }
    if (all_gpu && distinct && n_src >= 2 && n_src <= kMaxRanks) {
      rt->EnablePeerAccess(devs);
      bool p2p = true;
      for (int a : devs) for (int b : devs) if (!rt->PeerOK(a, b)) p2p = false;
      key_collective = p2p;
    }
    if (key_collective) {
      key_part = devs;
    } else {
      int rd = -1;
      for (int d : devs) if (d >= 0) { rd = d; break; }
      if (rd < 0) {
        for (NDArray* o : g.outs) if (o->ctx().is_gpu()) { rd = o->ctx().dev_id; break; }
      }
      if (rd < 0 && !ks.reps.empty()) rd = ks.reps[0].dev;
      if (rd < 0) rd = DefaultDevice();
      key_part.assign(1, rd);
    }
  }
  *key_collective_out = key_collective;
}

namespace {
void Touch(std::vector<int>* touched, int dev) {
  if (dev >= 0 && std::find(touched->begin(), touched->end(), dev) == touched->end()) touched->push_back(dev);
}
}  // namespace

// One key of a dense call while ReduceUpdate builds the call's plan: each stage fills in what the next needs.
struct KVStore::KeyBuild {
  const std::vector<Group>& groups;
  size_t gi;                        // this key's group (and its index in CallPlan::keys)
  bool write_outs;
  const AliasIndex& alias;
  KeyState& ks;
  int first = 0, last = 0;          // local participant slots
  std::vector<int> devs;            // per source: device, -1 = host (PlaceKey)
  std::vector<Replica*> rep;        // per participant slot, the local ones only (KeyReplicas)
  bool mp = false;                  // fp32 master weight
  bool two_shot = false;            // sharded over the participants
  const TreePlan* tree = nullptr;   // MXNET_KVSTORE_USETREE (KeyTree)
  bool tree_sliced = false;
  bool nvls = false;                // the switch sums and stores (KeyDests)
  const Group& g() const { return groups[gi]; }
};

// Ordering: nothing below issues an operation that reads or writes a caller array.  The build only enqueues work on
// engine-owned memory (EnsureReplica / EnsureState / SyncState / GatherLocal / GatherState); stream waits, staging
// copies (also those into temporaries) and the launches are plan steps that IssuePlan runs after it has acquired
// every device of the call, once.
void KVStore::ReduceUpdate(std::vector<Group>& groups, bool write_outs) {
  // an overflow of the previous step is settled before this step's update counts are taken
  if (hier_phase_ == 0 && opt_.enabled && updater_ == nullptr && opt_.skip_nonfinite) ResolveOverflow();
  if (hier_ && hier_phase_ == 0) { HierReduceUpdate(groups, write_outs); return; }
  // (multi-node with compression: phase 1 is the compressed reduce, phase 2 the ordinary update from the slices)
  if (gc_bits_ != 0 && hier_phase_ != 2) { ReduceUpdateCompressed(groups, write_outs); return; }

  // ---- a repeated call: the plan of the last identical call is kept (only counts and lr / wd / eta are new) ----
  CallPlan plan;
  bool rec_on = false, rec_repeat = false;
  uint64_t rec_hash = 0;
  std::unique_ptr<CallPlan> verify;     // MXKV_B200_PLAN=2: the plan as a replay would have patched it
  if (plan_mode_ != 0 && raw_pending_ && raw_single_ && hier_phase_ == 0 && !hier_ && updater_ == nullptr &&
      !(opt_.enabled && IsNormOpt(opt_.kind))) {
    raw_pending_ = false;               // (consumed: a recursive or later call must not record under it)
    rec_on = true;
    plan.sig = raw_sig_;
    rec_hash = raw_hash_;
    auto it = plans_.find(rec_hash);
    if (it != plans_.end() && it->second.sig == plan.sig && PlanEpochsMatch(it->second)) {
      if (it->second.recorded) {        // (MXKV_B200_PLAN=1 replays in TryReplayRaw and never gets here)
        // verify mode: build the plan below and compare
        verify.reset(new CallPlan(it->second));
        PlanPatch(*verify, false);
      }
      rec_repeat = true;                // nothing touched these keys since the last identical call: steady state
    }
  }
  if (hier_phase_ == 0 && HostPipelined(groups, write_outs)) return;
  ProcessGroup* pg = PG();
  const bool mp_mode = pg != nullptr;
  const bool callback = updater_ != nullptr && hier_phase_ != 1;
  // multi-node: phase 1 only sums the node's values into the staging slices; phase 2 is the ordinary path with
  // the (by then globally summed) slice as the only source
  plan.fused = opt_.enabled && !callback && hier_phase_ != 1;
  plan.opt_kind = plan.fused ? opt_.kind : OPT_NONE;

  // Keys of one call that reduce on different GPUs (e.g. host-resident values for keys whose stored
  // values live on different GPUs) are served group by group; the reference has no such restriction
  // because every key has its own merge buffer.  Reduce first, copy out afterwards: the order of
  // kvstore_local.h:358-365, which also keeps values that alias another key's outputs intact.
  if (!mp_mode && groups.size() > 1) {
    std::vector<std::pair<std::vector<int>, bool>> sig(groups.size());
    bool uniform = true;
    for (size_t gi = 0; gi < groups.size(); ++gi) {
      std::vector<int> devs;
      PlaceKey(groups[gi], GetKey(groups[gi].key), &devs, &sig[gi].first, &sig[gi].second);
      if (sig[gi] != sig[0]) uniform = false;
    }
    if (!uniform) {
      std::vector<char> done(groups.size(), 0);
      for (size_t gi = 0; gi < groups.size(); ++gi) {
        if (done[gi]) continue;
        std::vector<Group> bucket;
        for (size_t gj = gi; gj < groups.size(); ++gj) {
          if (done[gj] || sig[gj] != sig[gi]) continue;
          done[gj] = 1;
          Group c = groups[gj];
          c.outs.clear();
          bucket.push_back(c);
        }
        ReduceUpdate(bucket, false);
      }
      if (write_outs) {
        std::vector<int> okeys;
        std::vector<NDArray*> outs;
        for (auto& g : groups) for (NDArray* o : g.outs) { okeys.push_back(g.key); outs.push_back(o); }
        if (!outs.empty()) PullImpl(okeys, outs, 0, true);
      }
      return;
    }
  }

  const AliasIndex alias(groups);
  for (size_t gi = 0; gi < groups.size(); ++gi) {
    Group& g = groups[gi];
    KeyState& ks = GetKey(g.key);
    MXKV_CHECK(ks.stype == kDefaultStorage) << "key " << g.key << " is row_sparse; dense push not allowed";
    const int n_src = static_cast<int>(g.vals.size());
    MXKV_CHECK(n_src >= 1 && n_src <= kMaxSrc) << "push of " << n_src << " values for one key (max " << kMaxSrc << ")";
    for (auto& v : g.vals) {
      MXKV_CHECK(v.size() == ks.size) << "push: value has " << v.size() << " elements, key " << ks.key
                                      << " was initialised with " << ks.size;
      MXKV_CHECK(v.dtype() == ks.dtype) << "push: dtype mismatch for key " << ks.key
                                        << " (Only support input/output with the same data type)";
    }
    KeyBuild k{groups, gi, write_outs, alias, ks};
    std::vector<int> key_part;    // participant devices for this key
    bool key_collective = false;
    PlaceKey(g, ks, &k.devs, &key_part, &key_collective);
    if (gi == 0) {
      plan.part_dev = key_part; plan.collective = key_collective; plan.root_dev = key_part[0];
    } else {
      MXKV_CHECK(key_part == plan.part_dev && key_collective == plan.collective)
          << "all keys of one push/pushpull call must use the same set of devices";
    }
    k.first = mp_mode ? pg->rank() : 0;
    k.last = mp_mode ? pg->rank() : static_cast<int>(plan.part_dev.size()) - 1;
    KeyReplicas(plan, k);
    const std::vector<std::vector<const void*>> srcptr = KeySources(plan, k);
    KeyTree(plan, k);
    const std::vector<Dest> dests = KeyDests(plan, k);
    KeyWorks(plan, k, srcptr, dests);
    plan.keys.push_back(g.key);
  }
  std::sort(plan.touched.begin(), plan.touched.end());
  if (verify) {
    MXKV_CHECK(SamePlan(*verify, plan)) << "MXKV_B200_PLAN=2: the cached launch plan differs from the one the full path builds";
    plan_hits_++;
  }
  IssuePlan(plan);

  // ---- remember this call: the second identical call in a row (nothing else touched its keys in between)
  // leaves a plan behind, the third and later ones replay it
  if (rec_on && plan.repeatable && plan.staged.empty() && plan.callback_keys.empty()) {
    for (int key : plan.keys) plan.epochs.push_back(keys_.find(key)->second.epoch);
    plan.cfg_epoch = cfg_epoch_;
    plan.tuning_epoch = Runtime::Get()->tuning_epoch;
    plan.recorded = rec_repeat;
    if (!plan.recorded) { plan.launches.clear(); plan.pre_copies.clear(); plan.post_copies.clear(); }
    if (plans_.size() > 256) plans_.clear();          // (a training loop has a handful of distinct calls)
    plans_[rec_hash] = std::move(plan);
  }
}

// ---- replicas and optimizer state, laid out for this call's participants -------------------------------
void KVStore::KeyReplicas(CallPlan& plan, KeyBuild& k) {
  Runtime* rt = Runtime::Get();
  KeyState& ks = k.ks;
  const std::vector<int>& part_dev = plan.part_dev;
  const int n_part = static_cast<int>(part_dev.size());
  const bool callback = updater_ != nullptr && hier_phase_ != 1;
  k.rep.assign(n_part, nullptr);
  for (int p = k.first; p <= k.last; ++p) {
    Touch(&plan.touched, part_dev[p]);
    EnsureReplica(ks, part_dev[p]);
  }
  // EnsureReplica may reallocate ks.reps: resolve pointers afterwards
  for (int p = k.first; p <= k.last; ++p) k.rep[p] = FindReplica(ks, part_dev[p]);

  const bool lowp = ks.dtype == kFloat16 || ks.dtype == kBfloat16;
  k.mp = plan.fused && (opt_.multi_precision || lowp);
  if (plan.fused) {
    MXKV_CHECK(ks.dtype == kFloat32 || lowp) << "fused optimizers need float32/float16/bfloat16 keys";
    for (int p = k.first; p <= k.last; ++p) EnsureState(ks, *k.rep[p], k.mp);
  }

  k.two_shot = plan.collective && !hier_whole_keys_ &&
               static_cast<int64_t>(ks.size * DTypeSize(ks.dtype)) >= rt->twoshot_bytes &&
               ks.size >= static_cast<int64_t>(n_part) * 128;
  if (hier_phase_ != 1 && ks.local_world > 0 &&
      (callback || !(k.two_shot && ks.local_world == n_part && ks.shard_devs == part_dev))) {
    GatherLocal(ks);
    plan.repeatable = false;
    for (int p = k.first; p <= k.last; ++p) EnsureReplica(ks, part_dev[p]);
    for (int p = k.first; p <= k.last; ++p) k.rep[p] = FindReplica(ks, part_dev[p]);
  }
  if (plan.fused) {
    // the optimizer state is laid out for this call's shape: sharded over the n participants of a
    // two-shot push, complete on every replica otherwise (also when a key that used to be sharded is
    // now pushed from one GPU only)
    const int want = (plan.collective && k.two_shot) ? n_part : 0;
    const bool same = ks.state_world == want && (want == 0 || ks.state_devs == part_dev);
    if (ks.count > 0 && !same) { GatherState(ks); plan.repeatable = false; }
    ks.state_world = want;
    if (want > 0) ks.state_devs = part_dev; else ks.state_devs.clear();
    // a replica that sat out earlier updates (its GPU did not take part) first takes over the state of
    // one that did; after this call only the participants' state is current
    for (int p = k.first; p <= k.last; ++p) SyncState(ks, *k.rep[p]);
    for (auto& r : ks.reps) {
      bool part = false;
      for (int p = k.first; p <= k.last; ++p) part = part || (&r == k.rep[p]);
      if (!part) r.state_fresh = false;
    }
  }
}

// ---- sources as addressable pointers: srcptr[p][k] is the address of source k for the kernel running as
// participant p.  Values the kernel cannot read where they are get a staging step into the plan.
std::vector<std::vector<const void*>> KVStore::KeySources(CallPlan& plan, KeyBuild& k) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  const Group& g = k.g();
  const int n_part = static_cast<int>(plan.part_dev.size());
  const int n_src = static_cast<int>(g.vals.size());
  const int root_dev = plan.root_dev;
  std::vector<std::vector<const void*>> srcptr(n_part, std::vector<const void*>(plan.collective ? n_part : n_src));
  auto stage = [&](const NDArray& v, int dev) -> const void* {   // a temporary on `dev`, filled by IssuePlan
    void* t = nullptr;
    DeviceGuard dg(dev);
    CUDA_CALL(cudaMallocAsync(&t, v.nbytes() ? v.nbytes() : 16, rt->Dev(dev).stream));
    plan.staged.push_back(StagedValue{v, t, dev});
    return t;
  };
  if (pg != nullptr && hier_phase_ == 2) {
    srcptr[pg->rank()].assign(1, hier_base_.at(k.ks.key));
  } else if (pg != nullptr) {
    const NDArray& v = g.vals[0];
    if (plan.collective) {
      NDArray sym_src = v;
      if (!v.symmetric()) {
        Replica& r = *k.rep[pg->rank()];
        if (r.stage.is_none()) r.stage = NDArray::Empty(k.ks.shape, Context{kGPU, pg->dev()}, k.ks.dtype, true);
        plan.pre_copies.emplace_back(v, r.stage);   // D2D or H2D
        sym_src = r.stage;
      }
      for (int q = 0; q < n_part; ++q) srcptr[pg->rank()][q] = sym_src.peer_data(q);
    } else {
      srcptr[pg->rank()][0] = k.devs[0] < 0 ? stage(v, pg->dev()) : v.data();
    }
  } else if (plan.collective) {
    for (int p = 0; p < n_part; ++p)
      for (int q = 0; q < n_part; ++q) srcptr[p][q] = g.vals[q].data();
  } else {
    for (int s = 0; s < n_src; ++s) {
      const int dev = k.devs[s];
      const bool direct = dev == root_dev || (dev >= 0 && (rt->EnablePeerAccess({root_dev, dev}),
                                                           rt->PeerOK(root_dev, dev)));
      Touch(&plan.touched, dev);
      if (direct && dev != root_dev) plan.pre_waits.emplace_back(root_dev, dev);   // foreign GPU read by the root kernel
      // a host value, or no P2P: staged on the root
      srcptr[0][s] = direct ? g.vals[s].data() : stage(g.vals[s], root_dev);
    }
  }
  return srcptr;
}

// ---- MXNET_KVSTORE_USETREE: which tree(s) this key's sum goes up ------------------------------------
// Two values add the same way in any order, and the integer dtypes wrap: only three or more floating-point
// values are order-sensitive.  Host-resident values and multi-node stores keep the plain order (the
// reference's tree needs every value on its own GPU, comm_tree.h:108-121).
void KVStore::KeyTree(const CallPlan& plan, KeyBuild& k) {
  const KeyState& ks = k.ks;
  const int n_part = static_cast<int>(plan.part_dev.size());
  if (!(tree_ && plan.collective && n_part >= 3 && hier_phase_ == 0 &&
        (ks.dtype == kFloat32 || ks.dtype == kFloat16 || ks.dtype == kBfloat16 || ks.dtype == kFloat64)))
    return;
  MXKV_CHECK(!(plan.fused && IsNormOpt(opt_.kind)))
      << "MXNET_KVSTORE_USETREE=1: the layer-wise optimizers (LAMB / LANS / LARS) are not served in tree order";
  MXKV_CHECK(TreeKernelAvailable(ks.dtype, plan.fused ? opt_.kind : OPT_NONE, k.mp ? 1 : 0))
      << "MXNET_KVSTORE_USETREE=1: no tree kernel for dtype " << ks.dtype << " with optimizer kind " << opt_.kind;
  ProcessGroup* pg = PG();
  k.tree = &TreePlanFor(pg != nullptr ? pg->rank_devs() : plan.part_dev);
  const int64_t rows = ks.shape.empty() ? 1 : ks.shape[0];
  k.tree_sliced = ks.size > tree_bound_ && rows >= 2 * static_cast<int64_t>(n_part);
}

// ---- destinations: what the kernels write (replicas, the updater's merge buffer, the outputs they can write
// themselves), the NVLS choice, the copies out of a replica afterwards, and which replicas are fresh after the call
std::vector<KVStore::Dest> KVStore::KeyDests(CallPlan& plan, KeyBuild& k) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  const bool mp_mode = pg != nullptr;
  const bool callback = updater_ != nullptr && hier_phase_ != 1;
  const Group& g = k.g();
  KeyState& ks = k.ks;
  const std::vector<int>& part_dev = plan.part_dev;
  const int n_part = static_cast<int>(part_dev.size());
  const bool collective = plan.collective, two_shot = k.two_shot;
  const int root_dev = plan.root_dev;
  std::vector<Dest> dests;
  auto add_dest_sp = [&](void* ptr, int dev) {
    Dest d;
    for (int p = 0; p < kMaxRanks; ++p) d.ptr[p] = ptr;
    d.owner = -1;
    for (int p = 0; p < n_part; ++p) if (part_dev[p] == dev) d.owner = p;
    dests.push_back(d);
  };
  if (callback) {
    Replica& root = *k.rep[k.first];
    if (root.merged.is_none())
      root.merged = NDArray::Empty(ks.shape, Context{kGPU, root.dev}, ks.dtype, mp_mode);
    if (mp_mode && collective) {
      Dest d; d.owner = -2;   // every rank owns its own copy
      for (int p = 0; p < n_part; ++p) d.ptr[p] = root.merged.peer_data(p);
      dests.push_back(d);
    } else {
      add_dest_sp(root.merged.data(), root.dev);
    }
    plan.callback_keys.push_back(&ks);
  } else {
    // which outputs can be written by the kernel itself?
    std::vector<char> out_direct(g.outs.size(), 0);
    bool need_post = false;
    if (k.write_outs) {
      int budget = kMaxOut - 1 - (mp_mode ? 1 : static_cast<int>(ks.reps.size()));
      for (size_t oi = 0; oi < g.outs.size(); ++oi) {
        NDArray* o = g.outs[oi];
        MXKV_CHECK(o->size() == ks.size && o->dtype() == ks.dtype)
            << "pushpull: output does not match key " << ks.key;
        const Context oc = o->ctx();
        bool direct = false;
        if (oc.is_gpu() && budget > 0) {
          if (mp_mode) {
            direct = collective ? o->symmetric() : (oc.dev_id == pg->dev());
          } else {
            for (int p = 0; p < n_part; ++p) if (part_dev[p] == oc.dev_id) direct = true;
          }
          // one-shot in-place allreduce: peers still read this buffer while we would write it
          if (direct && collective && !two_shot) {
            for (auto& v : g.vals)
              if (Overlap(o->data(), o->nbytes(), v.data(), v.nbytes())) direct = false;
          }
          if (direct && !Aligned16(o->data())) direct = false;
          if (direct && k.groups.size() > 1 && k.alias.OverlapsOther(o->data(), o->nbytes(), static_cast<int>(k.gi)))
            direct = false;
        }
        out_direct[oi] = direct ? 1 : 0;
        if (direct) --budget; else need_post = true;
      }
    }
    // Two-shot keys keep the stored value sharded (rank p owns shard p of its own replica) unless
    // an output has to be copied out of a complete replica afterwards: the all-gather then moves
    // each shard over NVLink once per peer (into the outputs) instead of twice.
    // NVLS: every array of the key is bound to a multicast object (and nothing has to be copied
    // out of a complete replica afterwards)
    // (auto: above 4 ranks.  Per direction the switch path moves S(1 + 1/n) against 2S(n-1)/n of
    // the peer path: 1.5x more at n=2, 1.2x less at n=4 -- where the peer path is still kept because
    // it is bit-exact --, 1.56x less at n=8)
    if (mp_mode && collective && !hier_ && k.tree == nullptr &&
        (rt->nvls_mode >= 2 || (rt->nvls_mode == 1 && n_part > 4)) &&
        !(plan.fused && IsNormOpt(opt_.kind)) && ks.dtype == kFloat32 && ks.size % 4 == 0 &&
        g.vals[0].mc_data() != nullptr && Aligned16(g.vals[0].mc_data()) && !(two_shot && need_post)) {
      k.nvls = true;
      if (k.write_outs)
        for (size_t oi = 0; oi < g.outs.size(); ++oi)
          if (out_direct[oi] && g.outs[oi]->mc_data() == nullptr) k.nvls = false;
    }
    const bool shard_local = two_shot && !need_post;
    if (hier_phase_ == 1) {
      // the node's sum of this rank's range (the whole key when it is not sharded) goes to the staging slice
      Dest d; d.owner = collective ? -2 : -1; d.own_only = shard_local;
      for (int p = 0; p < kMaxRanks; ++p) d.ptr[p] = hier_base_.at(ks.key);
      if (!collective) d.owner = 0;
      dests.push_back(d);
    } else if (mp_mode && collective) {
      Dest d; d.owner = -2; d.own_only = shard_local;
      for (int p = 0; p < n_part; ++p) d.ptr[p] = k.rep[pg->rank()]->local.peer_data(p);
      dests.push_back(d);
    } else {
      for (auto& r : ks.reps) {
        const bool reachable = r.dev == root_dev || collective ||
                               (rt->EnablePeerAccess({root_dev, r.dev}), rt->PeerOK(root_dev, r.dev));
        bool is_part = false;
        for (int p = 0; p < n_part; ++p) if (part_dev[p] == r.dev) is_part = true;
        if (is_part || (reachable && !collective)) {
          if (!is_part) { Touch(&plan.touched, r.dev); plan.pre_waits.emplace_back(root_dev, r.dev); }
          add_dest_sp(r.local.data(), r.dev);
          dests.back().own_only = shard_local;
          r.fresh = true;
        } else {
          r.fresh = false;          // refreshed lazily by EnsureReplica
        }
      }
    }
    if (hier_phase_ == 1) {
      // the stored value is not touched in this phase
    } else if (shard_local) { ks.local_world = n_part; ks.shard_devs = part_dev; }
    else ks.local_world = 0;
    if (k.write_outs) {
      for (size_t oi = 0; oi < g.outs.size(); ++oi) {
        NDArray* o = g.outs[oi];
        const Context oc = o->ctx();
        if (oc.is_gpu()) Touch(&plan.touched, oc.dev_id);
        if (out_direct[oi]) {
          if (mp_mode && collective) {
            Dest d; d.owner = -2;
            for (int p = 0; p < n_part; ++p) d.ptr[p] = o->peer_data(p);
            d.mc = o->mc_data();
            dests.push_back(d);
          } else {
            add_dest_sp(o->data(), oc.dev_id);
          }
        } else {
          // copy out of a replica this call has just written: a replica on the output's own GPU only if
          // that GPU took part (a replica left over from an earlier device set is stale now)
          Replica* near = oc.is_gpu() ? FindReplica(ks, oc.dev_id) : nullptr;
          const int sdev = (near != nullptr && near->fresh) ? oc.dev_id : part_dev[k.first];
          plan.post_copies.emplace_back(FindReplica(ks, sdev)->local, *o);
        }
      }
    }
  }
  MXKV_CHECK(static_cast<int>(dests.size()) <= kMaxOut) << "too many destinations for key " << ks.key;
  return dests;
}

// ---- work entries: one per local participant (per tree slice with MXNET_KVSTORE_USETREE), in the key's launch
// class.  One launch (one pair of rendezvous) serves the one-shot and the two-shot keys of a call: the
// release/acquire flavour of the end barrier covers both.
void KVStore::KeyWorks(CallPlan& plan, const KeyBuild& k, const std::vector<std::vector<const void*>>& srcptr,
                       const std::vector<Dest>& dests) {
  KeyState& ks = k.ks;
  const int n_part = static_cast<int>(plan.part_dev.size());
  const bool collective = plan.collective, two_shot = k.two_shot;
  if (plan.fused) StepKey(ks);     // Optimizer._update_count
  LaunchClassKey ck{collective ? SYNC_WRITE_PEERS : SYNC_NONE, ks.dtype, k.mp ? 1 : 0};
  ck.nvls = k.nvls ? 1 : 0;
  ck.tree = k.tree != nullptr ? 1 : 0;
  auto it = std::lower_bound(plan.launches.begin(), plan.launches.end(), ck,
                             [](const PlanLaunch& l, const LaunchClassKey& c) { return l.ck < c; });
  if (it == plan.launches.end() || ck < it->ck)
    it = plan.launches.insert(it, PlanLaunch{ck, std::vector<std::vector<TensorWork>>(n_part), {},
                                             std::vector<std::vector<int>>(n_part)});
  PlanLaunch& l = *it;
  const int64_t shard = two_shot ? ShardLen(ks.size, n_part) : ks.size;
  l.busiest.push_back(std::min<int64_t>(ks.size, shard));
  for (int p = k.first; p <= k.last; ++p) {
    TensorWork tw = two_shot ? ReplicaWork(ks, *k.rep[p], plan.fused, k.mp, std::min<int64_t>(ks.size, shard * p),
                                           std::min<int64_t>(ks.size, shard * (p + 1)))
                             : ReplicaWork(ks, *k.rep[p], plan.fused, k.mp, 0, ks.size);
    if (k.nvls) {                  // the switch sums the replicas: one multicast "source"
      tw.n_src = 1;
      tw.src[0] = k.g().vals[0].mc_data();
    } else {
      tw.n_src = static_cast<int>(srcptr[p].size());
      for (int s = 0; s < tw.n_src; ++s) tw.src[s] = srcptr[p][s];
    }
    std::vector<void*> mc_outs;
    for (auto& d : dests) {
      if (d.owner == -2) {           // MP: one copy per rank
        if (two_shot && !d.own_only) {
          if (k.nvls) { mc_outs.push_back(d.mc); continue; }
          for (int q = 0; q < n_part; ++q) tw.out[tw.n_out++] = d.ptr[q];
        } else {
          tw.out[tw.n_out++] = d.ptr[p];
        }
        continue;
      }
      const bool mine = !collective || (two_shot && !d.own_only) || d.owner == p || (d.owner == -1 && p == 0);
      if (mine) tw.out[tw.n_out++] = d.ptr[p];
    }
    for (void* m : mc_outs) { tw.out[tw.n_out++] = m; tw.n_mc++; }
    MXKV_CHECK(tw.n_out <= kMaxOut) << "too many destinations for key " << ks.key;
    tw.flags = WorkFlags(tw, DTypeSize(ks.dtype) == 4 && ks.size % 4 == 0);
    if (k.nvls) MXKV_CHECK(tw.flags & kWorkVec16) << "NVLS arrays must be 16-byte aligned";
    if (k.tree != nullptr) AppendTreeWorks(tw, *k.tree, k.tree_sliced, ks, n_part, &l.per_part[p]);
    else l.per_part[p].push_back(tw);
    l.key_idx[p].resize(l.per_part[p].size(), static_cast<int>(k.gi));
  }
}

// One kernel launch per local participant for a list of work entries that share dtype /
// precision mode / synchronisation mode.  The grid is derived from the busiest rank's chunk
// count, which every rank computes identically (paired blocks rendezvous across GPUs).
void KVStore::LaunchWorks(const LaunchClassKey& ck, std::vector<std::vector<TensorWork>>& per_part,
                          const std::vector<int64_t>& busiest, int opt_kind, const std::vector<int>& part_dev) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  const bool mp_mode = pg != nullptr;
  const int n_part = static_cast<int>(part_dev.size());
  const int my_first = mp_mode ? pg->rank() : 0;
  const int my_last = mp_mode ? pg->rank() : n_part - 1;
  if (IsNormOpt(opt_kind)) {
    std::vector<NormClass> one{NormClass{ck, &per_part, &busiest}};
    LaunchNormWorks(one, opt_kind, part_dev);
    return;
  }

  // ---- kernel variant: identical decision on every rank (it fixes the grid) --------------------
  // shared-memory staged (bulk-copy) variant: float32, every entry 16-byte aligned with a key size
  // that is a multiple of 4 elements (rank-independent facts only)
  int64_t chunk = rt->chunk_elems;
  int bulk = 0, bulk_stages = 0, bulk_arrays = 0, bulk_cap = 0;
  if (rt->bulk_mode != 0 && ck.dtype == kFloat32 && !ck.nvls && !ck.tree) {
    bool ok = true;
    int max_src = 1;
    for (int p = my_first; p <= my_last; ++p)
      for (auto& t : per_part[p]) { ok = ok && (t.flags & kWorkStaged); max_src = std::max(max_src, t.n_src); }
    const int extra = OptStreams(opt_kind);
    // the staged variant is taken (a) whenever sources are read over NVLink (more bytes in flight
    // against a ~2 us round trip) and (b) locally when a thread of the per-thread variant would have
    // few loads in flight (<= 2 sources, >= 3 streams).  With >= 3 local sources the per-thread variant
    // already keeps enough requests in flight.  bulk_mode 2 forces the staged variant wherever it is
    // eligible.
    const bool want = rt->bulk_mode >= 2 || ck.sync_mode != SYNC_NONE || (max_src <= 2 && max_src + extra >= 3);
    if (ok && want) {
      // n_src is the same for every entry of a collective class; take the max for safety
      int tile = 0, st = 0;
      const int cap = BulkPlan(part_dev[my_first], opt_kind, ck.mp, max_src + extra, ck.sync_mode == SYNC_NONE,
                               &tile, &st);
      if (cap > 0) { bulk = 1; bulk_stages = st; bulk_arrays = max_src + extra; bulk_cap = cap; chunk = tile; }
    }
  }
  int nvls_cap = 0;
  if (ck.nvls) {
    int ce = 0;
    nvls_cap = NvlsPlan(part_dev[my_first], opt_kind, ck.mp, rt->nvls_unroll, rt->nvls_pipe, rt->nvls_threads, &ce);
    MXKV_CHECK(nvls_cap > 0) << "no multicast kernel for optimizer kind " << opt_kind;
    chunk = ce;
    if (rt->nvls_grid > 0) nvls_cap = std::min(nvls_cap, rt->nvls_grid);
  }
  int64_t max_chunks = 0;
  for (int64_t len : busiest) max_chunks += (len + chunk - 1) / chunk;
  max_chunks = std::max<int64_t>(1, max_chunks);

  // one flag value for the rendezvous of this launch, the same on every participant (SyncArgs::epoch)
  const uint32_t sync_epoch = ck.sync_mode != SYNC_NONE ? rt->NextSyncEpoch(pg) : 0;
  for (int p = my_first; p <= my_last; ++p) {
    auto& w = per_part[p];
    if (w.empty()) continue;
    std::vector<int64_t> prefix(w.size() + 1);
    int64_t acc = 0;
    for (size_t i = 0; i < w.size(); ++i) {
      prefix[i] = acc;
      acc += (w[i].end - w[i].begin + chunk - 1) / chunk;
    }
    prefix[w.size()] = acc;
    const int dev = part_dev[p];
    DeviceState& d = rt->Dev(dev);
    // Nadam: the per-entry side array of the key scalars a TensorWork has no room for (DenseLaunch::nadam), in the
    // same upload, 16-byte aligned after the chunk prefix
    std::vector<float4> side;
    if (opt_kind == OPT_NADAM) {
      side.resize(w.size());
      for (size_t i = 0; i < w.size(); ++i) side[i] = keys_.find(w[i].key)->second.step.nadam;
    }
    const size_t wbytes = w.size() * sizeof(TensorWork);
    const size_t pbytes = prefix.size() * sizeof(int64_t);
    const size_t soff = wbytes + ((pbytes + 15) & ~static_cast<size_t>(15));
    const size_t sbytes = side.size() * sizeof(float4);
    const size_t bytes = side.empty() ? wbytes + pbytes : soff + sbytes;
    DeviceGuard dg(dev);
    // The upload is a copy on the engine stream between two kernels, a fixed cost of every launch: a list that is
    // byte-for-byte the resident one (the same keys pushed again with the same hyper-parameters) is read where it is.
    // Any other list that fits replaces it, in stream order, so every kernel that reads the old list is done first.
    const bool fits = bytes <= DeviceState::kResidentListBytes;
    const bool resident = fits && d.list_host.size() == bytes &&
                          std::memcmp(d.list_host.data(), w.data(), wbytes) == 0 &&
                          std::memcmp(d.list_host.data() + wbytes, prefix.data(), pbytes) == 0 &&
                          (side.empty() || std::memcmp(d.list_host.data() + soff, side.data(), sbytes) == 0);
    size_t off = 0;
    char* list = d.list_dev;
    if (!resident) {
      off = d.ring.Alloc(bytes);
      std::memcpy(d.ring.host(off), w.data(), wbytes);
      std::memcpy(d.ring.host(off) + wbytes, prefix.data(), pbytes);
      if (!side.empty()) {
        std::memset(d.ring.host(off) + wbytes + pbytes, 0, soff - wbytes - pbytes);
        std::memcpy(d.ring.host(off) + soff, side.data(), sbytes);
      }
      if (!fits) list = d.ring.dev(off);
      CUDA_CALL(cudaMemcpyAsync(list, d.ring.host(off), bytes, cudaMemcpyHostToDevice, d.stream));
      if (fits) d.list_host.assign(d.ring.host(off), d.ring.host(off) + bytes);
    }
    DenseLaunch L;
    std::memset(&L, 0, sizeof(L));
    L.works = reinterpret_cast<const TensorWork*>(list);
    L.chunk_prefix = reinterpret_cast<const int64_t*>(list + wbytes);
    L.nworks = static_cast<int>(w.size());
    L.total_chunks = prefix.back();
    L.dtype = ck.dtype;
    L.opt = opt_kind;
    L.multi_precision = ck.mp;
    // nag.py:137: mp_nag_mom_update where the optimizer asked for multi_precision on a 16-bit key
    L.mp_arith = (opt_kind != OPT_NONE && opt_.multi_precision &&
                  (ck.dtype == kFloat16 || ck.dtype == kBfloat16)) ? 1 : 0;
    L.order = ck.tree ? ORDER_TREE : order_;
    L.fp32_accum = (opt_kind != OPT_NONE || ck.dtype == kBfloat16 ||
                    EnvInt("MXKV_B200_FP16_FP32_ACCUM", 0) != 0) ? 1 : 0;
    L.rescale = opt_.rescale; L.clip = opt_.clip; L.momentum = opt_.momentum;
    L.beta1 = static_cast<float>(opt_.beta1); L.beta2 = static_cast<float>(opt_.beta2); L.eps = opt_.eps;
    L.rho = opt_.rho; L.clip_weights = opt_.clip_weights;
    L.wd_lh = static_cast<float>(opt_.wd_lh);
    if (!side.empty()) {
      L.nadam = reinterpret_cast<const float4*>(list + soff);
      L.one_minus_beta1 = static_cast<float>(1. - opt_.beta1);
      L.one_minus_beta2 = static_cast<float>(1. - opt_.beta2);
    }
    L.sync.mode = ck.sync_mode;
    L.sync.world = n_part;
    L.sync.rank = p;
    L.sync.self = d.signal_pad;
    L.sync.timeout = rt->spin_timeout_cycles;
    L.sync.epoch = sync_epoch;
    for (int q = 0; q < n_part; ++q)
      L.sync.peers[q] = mp_mode ? pg->signal_pad(q) : rt->Dev(part_dev[q]).signal_pad;
    L.grid = static_cast<int>(std::min<int64_t>(bulk ? std::min(bulk_cap, rt->max_blocks > 0 ? rt->max_blocks : bulk_cap)
                                                     : d.max_grid, max_chunks));
    L.chunk_elems = static_cast<int>(chunk);
    L.threads = rt->threads;
    L.bulk = bulk; L.bulk_stages = bulk_stages; L.bulk_arrays = bulk_arrays;
    // tile grouping pays where a block would otherwise meet hundreds of keys (BERT-base, ResNet-50: -4 %); on a few
    // large keys the plain strided walk streams DRAM best (the sweep: 0.945 of the HBM peak)
    L.bulk_group = (rt->bulk_group_forced || w.size() >= 32) ? rt->bulk_group : 1;
    L.nvls = ck.nvls;
    L.nvls_unroll = rt->nvls_unroll;
    L.nvls_pipe = rt->nvls_pipe;
    if (ck.nvls) { L.threads = rt->nvls_threads; L.grid = static_cast<int>(std::min<int64_t>(nvls_cap, max_chunks)); }
    int small_n = 1;
    for (auto& t : w) if (t.n_src > 2) small_n = 0;
    L.small_n = small_n;
    const int rc = LaunchDense(L, d.stream);
    MXKV_CHECK(rc == 0) << "kernel launch failed: " << cudaGetErrorString(static_cast<cudaError_t>(rc));
    rt->launches++;
    rt->variant_launches[ck.tree ? 3 : (L.nvls ? 2 : (L.bulk ? 1 : 0))]++;
    if (!resident) d.ring.Commit(off, bytes, d.stream);
  }
}

TensorWork KVStore::ReplicaWork(const KeyState& ks, const Replica& r, bool fused, bool mp, int64_t begin,
                                int64_t end) const {
  TensorWork tw;
  std::memset(&tw, 0, sizeof(tw));
  tw.w = r.local.data();
  tw.w32 = mp ? static_cast<float*>(r.w32.data()) : nullptr;
  tw.s0 = r.s0.is_none() ? nullptr : static_cast<float*>(r.s0.data());
  tw.s1 = r.s1.is_none() ? nullptr : static_cast<float*>(r.s1.data());
  tw.s2 = r.s2.is_none() ? nullptr : static_cast<float*>(r.s2.data());
  tw.begin = begin; tw.end = end;
  if (fused) { tw.lr = ks.step.lr; tw.wd = ks.step.wd; tw.eta = ks.step.eta; }
  tw.key = ks.key;
  return tw;
}

// A launch that involves one GPU only (no rendezvous), whatever the deployment shape.
void KVStore::LaunchLocal(const LaunchClassKey& ck, const TensorWork& tw, int opt_kind, int dev) {
  ProcessGroup* pg = PG();
  const int slots = pg ? pg->world() : 1;
  const int mine = pg ? pg->rank() : 0;
  std::vector<std::vector<TensorWork>> per_part(slots);
  per_part[mine].push_back(tw);
  std::vector<int> part_dev(slots, dev);
  LaunchClassKey local = ck;
  local.sync_mode = SYNC_NONE;
  LaunchWorks(local, per_part, {tw.end - tw.begin}, opt_kind, part_dev);
}

// All-gather of a key whose stored value is valid shard-wise only (after a two-shot push that did
// not have to deliver full outputs): participant p stores its shard into every replica.
void KVStore::GatherLocal(KeyState& ks) {
  const int n = ks.local_world;
  if (n <= 1) { ks.local_world = 0; return; }
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  const bool mp_mode = pg != nullptr;
  const std::vector<int> part_dev = ks.shard_devs;
  MXKV_CHECK(static_cast<int>(part_dev.size()) == n) << "inconsistent shard layout for key " << ks.key;
  const int64_t shard = ShardLen(ks.size, n);
  std::vector<std::vector<TensorWork>> per_part(n);
  const int my_first = mp_mode ? pg->rank() : 0;
  const int my_last = mp_mode ? pg->rank() : n - 1;
  for (int p = my_first; p <= my_last; ++p) {
    Replica* r = FindReplica(ks, part_dev[p]);
    MXKV_CHECK(r != nullptr) << "missing replica";
    TensorWork tw;
    std::memset(&tw, 0, sizeof(tw));
    tw.src[0] = r->local.data();
    tw.n_src = 1;
    for (int q = 0; q < n; ++q) {
      if (mp_mode) {
        tw.out[tw.n_out++] = r->local.peer_data(q);
      } else {
        Replica* rq = FindReplica(ks, part_dev[q]);
        tw.out[tw.n_out++] = rq->local.data();
      }
    }
    tw.begin = std::min<int64_t>(ks.size, shard * p);
    tw.end = std::min<int64_t>(ks.size, shard * (p + 1));
    tw.flags = WorkFlags(tw, ks.dtype == kFloat32 && ks.size % 4 == 0);
    per_part[p].push_back(tw);
  }
  LaunchClassKey ck{SYNC_WRITE_PEERS, ks.dtype, 0};
  LaunchWorks(ck, per_part, {std::min<int64_t>(ks.size, shard)}, OPT_NONE, part_dev);
  ks.local_world = 0;
  for (auto& r : ks.reps) {
    bool is_part = false;
    for (int d : part_dev) if (d == r.dev) is_part = true;
    r.fresh = is_part;
  }
}

SyncArgs KVStore::GroupSync(int mode) const {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  SyncArgs sync;
  std::memset(&sync, 0, sizeof(sync));
  sync.self = rt->Dev(pg->dev()).signal_pad;
  for (int q = 0; q < pg->world(); ++q) sync.peers[q] = pg->signal_pad(q);
  sync.world = pg->world(); sync.rank = pg->rank(); sync.mode = mode;
  sync.timeout = rt->spin_timeout_cycles;
  return sync;
}

SyncArgs KVStore::LocalSync(int dev) {
  Runtime* rt = Runtime::Get();
  SyncArgs sync;
  std::memset(&sync, 0, sizeof(sync));
  sync.self = rt->Dev(dev).signal_pad;
  sync.world = 1; sync.rank = 0; sync.mode = SYNC_NONE;
  sync.timeout = rt->spin_timeout_cycles;
  return sync;
}

// updater_(key, merged, &local) on the caller thread (kvstore_local.h:259-277); the callee owns and
// frees both handles (c_api.cc:3066-3080).  The embedding framework computes on its own stream:
// fence it on the reduce, then make the engine stream wait for whatever the callback enqueued.
void KVStore::RunCallbackUpdater(KeyState& ks, Replica& root, const NDArray& merged) {
  Runtime* rt = Runtime::Get();
  rt->Dev(root.dev).engine_dirty = true;
  rt->Fence(root.dev);
  NDHandle* recv = new NDHandle(merged);
  NDHandle* local = new NDHandle(root.local);
  if (key_type_ == kStringKey && str_updater_ != nullptr) {
    const std::string& sk = reverse_str_key_dict_[ks.key];
    str_updater_(sk.c_str(), recv, local, updater_handle_);
  } else {
    MXKV_CHECK(updater_ != nullptr) << "updater not set";
    updater_(ks.key, recv, local, updater_handle_);
  }
  rt->AcquireUser(root.dev);
  for (auto& r : ks.reps) r.fresh = (&r == &root);
}

// ---------------------------------------------------------------------------
// optimizer state access (save/load_optimizer_states; Updater.get_states/set_states,
// python/mxnet/optimizer/updater.py:108-127)
// ---------------------------------------------------------------------------
void KVStore::GatherState(KeyState& ks) {
  // sharded layout -> every replica complete.  Shard p of every kReplicaState array is valid on participant p.
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  const int n = ks.state_world;
  if (n <= 1) return;
  const int64_t shard = ShardLen(ks.size, n);
  auto gather = [&](ReplicaArray sel) {
    if (pg) {
      Replica& me = ks.reps[0];
      NDArray& mine = me.*sel;
      if (mine.is_none()) return;
      rt->WaitAll(); pg->Barrier();
      for (int p = 0; p < n; ++p) {
        if (p == pg->rank()) continue;
        const int64_t b = std::min(ks.size, shard * p), e = std::min(ks.size, shard * (p + 1));
        if (e <= b) continue;
        const char* src = static_cast<const char*>(mine.peer_data(p)) + b * 4;
        char* dst = static_cast<char*>(mine.data()) + b * 4;
        DeviceGuard dg(me.dev);
        CUDA_CALL(cudaMemcpyAsync(dst, src, (e - b) * 4, cudaMemcpyDeviceToDevice, rt->Dev(me.dev).stream));
      }
      rt->WaitAll(); pg->Barrier();
    } else {
      MXKV_CHECK(static_cast<int>(ks.state_devs.size()) == n) << "inconsistent state layout for key " << ks.key;
      for (size_t q = 0; q < ks.reps.size(); ++q) {
        for (int p = 0; p < n; ++p) {
          Replica* owner = FindReplica(ks, ks.state_devs[p]);      // shard p lives on participant p's GPU
          MXKV_CHECK(owner != nullptr) << "state shard " << p << " of key " << ks.key << " has no replica";
          if (owner == &ks.reps[q]) continue;
          NDArray& src = (*owner).*sel;
          NDArray& dst = ks.reps[q].*sel;
          if (src.is_none() || dst.is_none()) continue;
          const int64_t b = std::min(ks.size, shard * p), e = std::min(ks.size, shard * (p + 1));
          if (e <= b) continue;
          CopyFromTo(src.Reshape({ks.size}).Slice1D(b, e), dst.Reshape({ks.size}).Slice1D(b, e));
        }
      }
    }
  };
  for (auto m : kReplicaState) gather(m);
  ks.state_world = 0;
  ks.state_devs.clear();
  for (auto& r : ks.reps) r.state_fresh = HoldsState(r);      // every replica with state arrays holds every shard
}

// Updater.__call__ (python/mxnet/optimizer/updater.py:39-93) + the multi-tensor update operators it
// ends in (multi_sgd_update / multi_sgd_mom_update / multi_mp_sgd_* optimizer_op-inl.h:207-375,
// multi_adamw contrib/adamw-inl.h:329-464, multi_lamb / multi_lans): every (weight, grad) pair of
// the call is updated IN PLACE in one launch (sequence) on the arrays' GPU; the optimizer state of an
// index is created on first sight (create_state_multi_precision) and lives in this object.
void KVStore::UpdaterStep(bool str_keys, const std::vector<int>& ikeys, const std::vector<std::string>& skeys,
                          const std::vector<NDArray>& weights, const std::vector<NDArray>& grads) {
  LOCK();
  MXKV_CHECK(solo_) << "UpdaterStep needs a store created with type 'updater'";
  MXKV_CHECK(opt_.enabled && updater_ == nullptr) << "set a fused optimizer first (MXKVB200SetOptimizer)";
  const size_t n = weights.size();
  const bool bind_only = grads.empty() && n > 0;     // register the indices (e.g. before loading states)
  MXKV_CHECK((bind_only || grads.size() == n) && (str_keys ? skeys.size() : ikeys.size()) == n)
      << "UpdaterStep: keys / weights / grads differ in length";
  SetKeyType(str_keys ? kStringKey : kIntKey);
  std::vector<Group> groups;
  std::vector<std::pair<int, NDArray>> sparse;
  for (size_t i = 0; i < n; ++i) {
    int key;
    if (str_keys) {
      auto it = str_key_dict_.find(skeys[i]);
      if (it == str_key_dict_.end()) {
        key = next_str_key_++;
        str_key_dict_[skeys[i]] = key;
        reverse_str_key_dict_[key] = skeys[i];
      } else {
        key = it->second;
      }
    } else {
      key = ikeys[i];
    }
    const NDArray& w = weights[i];
    MXKV_CHECK(w.stype() == kDefaultStorage && w.ctx().is_gpu()) << "UpdaterStep: weights are dense GPU arrays";
    if (!bind_only) {
      // a row_sparse gradient updates the rows it holds (sgd / sgd-momentum / adam; lazy or standard
      // flavour as the optimizer says): the reference's per-device updater on Parameter(grad_stype='row_sparse')
      const NDArray& g = grads[i];
      MXKV_CHECK((g.stype() == kDefaultStorage || g.stype() == kRowSparseStorage) && g.ctx().is_gpu() &&
                 w.dev() == g.dev())
          << "UpdaterStep: weight and gradient of index " << key << " must be arrays on the same GPU";
    }
    auto it = keys_.find(key);
    if (it == keys_.end()) {
      KeyState ks;
      ks.key = key;
      ks.shape = w.shape();
      ks.dtype = w.dtype();
      ks.size = w.size();
      it = keys_.emplace(key, ks).first;
    }
    KeyState& ks = it->second;
    MXKV_CHECK(ks.size == w.size() && ks.dtype == w.dtype())
        << "UpdaterStep: weight of index " << key << " changed shape or dtype";
    Replica* r = FindReplica(ks, w.dev());
    if (r == nullptr) {
      MXKV_CHECK(ks.reps.empty()) << "an updater serves one device (index " << key << " was first seen on GPU "
                                  << ks.reps[0].dev << "); the reference keeps one Updater per device, too";
      Replica nr;
      nr.dev = w.dev();
      ks.reps.push_back(nr);
      r = &ks.reps.back();
    }
    r->local = w;          // alias of the caller's array: the kernel's store target
    r->fresh = true;
    ks.local_world = 0;
    if (bind_only) continue;
    if (SkipsOnRescale() && grads[i].stype() == kRowSparseStorage) { StepKey(ks); continue; }
    if (grads[i].stype() == kRowSparseStorage) { sparse.emplace_back(key, grads[i]); continue; }
    Group grp;
    grp.key = key;
    grp.vals = {grads[i]};
    groups.push_back(grp);
  }
  if (!groups.empty() && SkipsOnRescale()) SkipStep(groups);
  else if (!groups.empty()) ReduceUpdate(groups, false);
  for (auto& kg : sparse) PushRowSparse(GetKey(kg.first), {kg.second});
}

NDArray KVStore::GetState(bool str_key, int ikey, const std::string& skey, int which) {
  LOCK();
  KeyState& ks = GetKey(ResolveKey(str_key, ikey, skey));
  if (ks.reps.empty()) EnsureReplica(ks, DefaultDevice());
  if (ks.local_world > 0) GatherLocal(ks);
  GatherState(ks);
  if (which == 0) return FreshReplica(ks).local;
  // optimizer state: from a replica that took part in the latest update (the others may lag behind)
  Replica* holder = nullptr;
  for (auto& cand : ks.reps) if (cand.state_fresh && HoldsState(cand)) { holder = &cand; break; }
  Replica& r = holder ? *holder : FreshReplica(ks);
  MXKV_CHECK(which >= 1 && which <= kNumReplicaState) << "GetState: which must be 0.." << kNumReplicaState;
  return r.*kReplicaState[which - 1];
}

void KVStore::SetState(bool str_key, int ikey, const std::string& skey, int which, const NDArray& v) {
  LOCK();
  KeyState& ks = GetKey(ResolveKey(str_key, ikey, skey));
  if (ks.reps.empty()) EnsureReplica(ks, DefaultDevice());
  if (ks.local_world > 0) GatherLocal(ks);
  GatherState(ks);
  MXKV_CHECK(v.size() == ks.size) << "SetState: size mismatch";
  MXKV_CHECK(which >= 0 && which <= kNumReplicaState) << "SetState: which must be 0.." << kNumReplicaState;
  for (auto& r : ks.reps) {
    const bool lowp = ks.dtype == kFloat16 || ks.dtype == kBfloat16;
    if (which != 0) EnsureState(ks, r, opt_.multi_precision || lowp);
    NDArray* dst = which == 0 ? &r.local : &(r.*kReplicaState[which - 1]);
    MXKV_CHECK(!dst->is_none()) << "SetState: the active optimizer has no such state";
    CopyFromTo(v.Reshape(dst->shape()), *dst);
  }
}

void KVStore::GetKeyHyper(bool str_key, int ikey, const std::string& skey, float* lr, float* wd, float* eta) {
  LOCK();
  MXKV_CHECK(opt_.enabled) << "no fused optimizer is set";
  const KeyState& ks = GetKey(ResolveKey(str_key, ikey, skey));
  const KeyStep s = KeyScalars(ks);
  if (lr) *lr = s.lr;
  if (wd) *wd = s.wd;
  if (eta) *eta = s.eta;
}

int64_t KVStore::GetUpdateCount(bool str_key, int ikey, const std::string& skey) {
  LOCK();
  return GetKey(ResolveKey(str_key, ikey, skey)).count;
}
double KVStore::GetOptimizerScalar(const std::string& name) {
  LOCK();
  MXKV_CHECK(name == "m_schedule") << "unknown optimizer scalar '" << name << "'";
  return opt_.m_schedule;
}
void KVStore::SetOptimizerScalar(const std::string& name, double value) {
  LOCK();
  MXKV_CHECK(name == "m_schedule") << "unknown optimizer scalar '" << name << "'";
  opt_.m_schedule = value;
}

void KVStore::SetUpdateCount(bool str_key, int ikey, const std::string& skey, int64_t c) {
  LOCK_ONLY();
  const int key = ResolveKey(str_key, ikey, skey);
  FlushIfPending(key);
  PeekKey(key).count = c;          // (the count is read live by every launch: no plan depends on it)
}

}  // namespace mxkv
