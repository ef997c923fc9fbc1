// kvstore_norm.cc -- host side of the layer-wise adaptive optimizers (LAMB, LANS, LARS) and of the
// stand-alone multi_sum_sq / multi_all_finite reductions.  ReduceUpdate builds the same work lists
// as for the single-pass optimizers; LaunchNormWorks turns each list into the launch sequence of
// norm_kernels.h.  Every decision that shapes a launch (grid, chunking, which phases run) depends
// only on facts all ranks share, so paired blocks meet at every rendezvous.
#include "kvstore.h"
#include "norm_kernels.h"
#include <cstring>
#include <functional>
#include <map>

namespace mxkv {

// Entry points serialise on the runtime first (per-device streams, descriptor rings, peer tables and signal pads
// are shared by every store of the process), then on the store: callable from any thread, in this fixed order.
#define LOCK()                                                                  \
  std::lock_guard<std::recursive_mutex> rt_lock_(Runtime::Get()->mu());            \
  std::lock_guard<std::recursive_mutex> lock_(mu_)

void KVStore::LaunchNormWorks(std::vector<NormClass>& classes, int opt_kind, const std::vector<int>& part_dev) {
  Runtime* rt = Runtime::Get();
  ProcessGroup* pg = PG();
  const bool mp_mode = pg != nullptr;
  const int n_part = static_cast<int>(part_dev.size());
  const int my_first = mp_mode ? pg->rank() : 0;
  const int my_last = mp_mode ? pg->rank() : n_part - 1;
  const int kind = opt_kind == OPT_LAMB ? NORM_LAMB : (opt_kind == OPT_LANS ? NORM_LANS : NORM_LARS);
  const int64_t chunk = rt->chunk_elems;

  if (opt_.skip_nonfinite && overflow_flag_ == nullptr) {
    CUDA_CALL(cudaHostAlloc(reinterpret_cast<void**>(&overflow_flag_), sizeof(int),
                            cudaHostAllocMapped | cudaHostAllocPortable));
    *overflow_flag_ = 0;
  }

  struct Part {
    int dev = -1;
    bool collective = false;
    int cls = 0;                 // index of the launch class (one rendezvous value per class and phase)
    NormLaunch L;
    float* psum = nullptr;
    size_t off = 0, bytes = 0;
  };
  std::vector<Part> parts;
  // per device: where the non-finite counts of every key of the push live (as mapped on that device)
  std::map<int, std::vector<const float*>> bad_ptrs;

  int cls_index = -1;
  for (auto& cls : classes) {
    ++cls_index;
    const LaunchClassKey& ck = cls.ck;
    MXKV_CHECK(!ck.nvls) << "the multicast variant has no layer-wise optimizers";
    const bool collective = ck.sync_mode != SYNC_NONE;
    int64_t max_chunks = 0;
    for (int64_t len : *cls.busiest) max_chunks += (len + chunk - 1) / chunk;
    max_chunks = std::max<int64_t>(1, max_chunks);

    for (int p = my_first; p <= my_last; ++p) {
      auto& w = (*cls.per_part)[p];
      if (w.empty()) continue;
      const int dev = part_dev[p];
      DeviceState& d = rt->Dev(dev);
      DeviceGuard dg(dev);
      std::vector<int64_t> prefix(w.size() + 1);
      int64_t acc = 0;
      for (size_t i = 0; i < w.size(); ++i) {
        prefix[i] = acc;
        acc += (w[i].end - w[i].begin + chunk - 1) / chunk;
      }
      prefix[w.size()] = acc;
      Part part;
      part.dev = dev;
      part.collective = collective;
      part.cls = cls_index;
      CUDA_CALL(cudaMallocAsync(reinterpret_cast<void**>(&part.psum),
                                std::max<size_t>(16, static_cast<size_t>(acc) * kPsumStride * sizeof(float)), d.stream));

      std::vector<NormWork> nw(w.size());
      for (size_t i = 0; i < w.size(); ++i) {
        const TensorWork& t = w[i];
        KeyState& ks = GetKey(t.key);
        Replica* r = FindReplica(ks, dev);
        MXKV_CHECK(r != nullptr && !r->aux0.is_none() && !r->nrm.is_none())
            << "key " << ks.key << ": optimizer scratch missing";
        NormWork& n = nw[i];
        std::memset(&n, 0, sizeof(n));
        std::memcpy(n.src, t.src, sizeof(n.src));
        std::memcpy(n.out, t.out, sizeof(n.out));
        n.w = t.w; n.w32 = t.w32; n.s0 = t.s0; n.s1 = t.s1;
        n.aux0 = static_cast<float*>(r->aux0.data());
        n.aux1 = r->aux1.is_none() ? nullptr : static_cast<float*>(r->aux1.data());
        n.psum = part.psum + prefix[i] * kPsumStride;
        n.nrm = static_cast<float*>(r->nrm.data());
        n.begin = t.begin; n.end = t.end;
        n.lr_d = ks.step.lr_d;
        n.lr = t.lr; n.wd = t.wd;
        n.c1 = ks.step.c1; n.c2 = ks.step.c2;
        n.n_src = t.n_src; n.n_out = t.n_out;
        n.flags = (t.flags & kWorkVec16) | (opt_.no_trust.count(ks.key) ? 2 : 0);
        // a sharded (two-shot) key: every rank holds the sums of its shard only
        const bool sharded = collective && (t.end - t.begin) != ks.size;
        if (sharded) {
          n.norm_world = n_part;
          for (int q = 0; q < n_part; ++q) {
            if (mp_mode) {
              n.nrm_peer[q] = static_cast<const float*>(r->nrm.peer_data(q));
            } else {
              Replica* rq = FindReplica(ks, part_dev[q]);
              MXKV_CHECK(rq != nullptr && !rq->nrm.is_none()) << "key " << ks.key << ": peer scratch missing";
              n.nrm_peer[q] = static_cast<const float*>(rq->nrm.data());
            }
          }
        } else {
          n.norm_world = 1;
          n.nrm_peer[0] = n.nrm;
        }
        for (int q = 0; q < n.norm_world; ++q) bad_ptrs[dev].push_back(n.nrm_peer[q] + kNrmBad);
      }

      const size_t wbytes = nw.size() * sizeof(NormWork);
      const size_t pbytes = prefix.size() * sizeof(int64_t);
      part.bytes = wbytes + pbytes;
      part.off = d.ring.Alloc(part.bytes);
      std::memcpy(d.ring.host(part.off), nw.data(), wbytes);
      std::memcpy(d.ring.host(part.off) + wbytes, prefix.data(), pbytes);
      CUDA_CALL(cudaMemcpyAsync(d.ring.dev(part.off), d.ring.host(part.off), part.bytes, cudaMemcpyHostToDevice,
                                d.stream));

      NormLaunch& L = part.L;
      std::memset(&L, 0, sizeof(L));
      L.works = reinterpret_cast<const NormWork*>(d.ring.dev(part.off));
      L.chunk_prefix = reinterpret_cast<const int64_t*>(d.ring.dev(part.off) + wbytes);
      L.nworks = static_cast<int>(nw.size());
      L.total_chunks = acc;
      L.dtype = ck.dtype;
      L.kind = kind;
      L.multi_precision = ck.mp;
      L.order = order_;
      L.bias_correction = opt_.bias_correction ? 1 : 0;
      L.has_momentum = opt_.momentum != 0.f ? 1 : 0;
      L.rescale = opt_.rescale; L.clip = opt_.clip; L.momentum = opt_.momentum;
      L.beta1 = static_cast<float>(opt_.beta1); L.beta2 = static_cast<float>(opt_.beta2); L.eps = opt_.eps;
      L.lower_bound = opt_.lower_bound; L.upper_bound = opt_.upper_bound;
      L.lars_eta = opt_.lars_eta; L.lars_eps = opt_.lars_eps;
      L.skip_nonfinite = opt_.skip_nonfinite ? 1 : 0;
      L.overflow_flag = overflow_flag_;
      L.sync.world = n_part;
      L.sync.rank = p;
      L.sync.self = d.signal_pad;
      L.sync.timeout = rt->spin_timeout_cycles;
      for (int q = 0; q < n_part; ++q)
        L.sync.peers[q] = mp_mode ? pg->signal_pad(q) : rt->Dev(part_dev[q]).signal_pad;
      int cap = NormMaxGrid(dev);
      if (rt->max_blocks > 0) cap = std::min(cap, rt->max_blocks);
      L.grid = static_cast<int>(std::min<int64_t>(cap, max_chunks));
      L.chunk_elems = static_cast<int>(chunk);
      parts.push_back(part);
    }
  }
  if (parts.empty()) return;

  // upload the per-device lists of non-finite counters
  struct BadList { size_t off, bytes; };
  std::map<int, BadList> bad_alloc;
  if (opt_.skip_nonfinite) {
    for (auto& kv : bad_ptrs) {
      DeviceState& d = rt->Dev(kv.first);
      DeviceGuard dg(kv.first);
      BadList bl;
      bl.bytes = kv.second.size() * sizeof(const float*);
      bl.off = d.ring.Alloc(bl.bytes);
      std::memcpy(d.ring.host(bl.off), kv.second.data(), bl.bytes);
      CUDA_CALL(cudaMemcpyAsync(d.ring.dev(bl.off), d.ring.host(bl.off), bl.bytes, cudaMemcpyHostToDevice, d.stream));
      bad_alloc[kv.first] = bl;
    }
    for (auto& part : parts) {
      part.L.bad_list = reinterpret_cast<const float* const*>(rt->Dev(part.dev).ring.dev(bad_alloc[part.dev].off));
      part.L.n_bad = static_cast<int>(bad_ptrs[part.dev].size());
    }
  }

  // phase-major issue order: a rank's kernel spins until its peers' kernel of the same phase runs,
  // and no class may decide about an overflow before every class has counted
  auto phase = [&](int sync_mode, const std::function<int(const NormLaunch&, cudaStream_t)>& fn) {
    // one rendezvous value per launch class of this phase, the same on every participant (SyncArgs::epoch);
    // every rank walks the classes in the same order, so the counters advance alike
    std::map<int, uint32_t> epoch_of_class;
    if (sync_mode != SYNC_NONE)
      for (auto& part : parts)
        if (part.collective && !epoch_of_class.count(part.cls)) epoch_of_class[part.cls] = rt->NextSyncEpoch(pg);
    for (auto& part : parts) {
      DeviceGuard dg(part.dev);
      NormLaunch L = part.L;
      L.sync.mode = part.collective ? sync_mode : SYNC_NONE;
      L.sync.epoch = (part.collective && sync_mode != SYNC_NONE) ? epoch_of_class[part.cls] : 0;
      const int rc = fn(L, rt->Dev(part.dev).stream);
      MXKV_CHECK(rc == 0) << "kernel launch failed: " << cudaGetErrorString(static_cast<cudaError_t>(rc));
      rt->launches++;
    }
  };
  const bool lamb_direct = kind == NORM_LAMB && !opt_.skip_nonfinite;
  phase(SYNC_READ_PEERS, [&](const NormLaunch& L, cudaStream_t s) { return LaunchNormFirst(L, lamb_direct ? 0 : 1, s); });
  phase(SYNC_NONE, [&](const NormLaunch& L, cudaStream_t s) { return LaunchNormFinalize(L, 3, kNrmW, kNrmG, kNrmBad, s); });
  if (kind == NORM_LANS || (kind == NORM_LAMB && !lamb_direct)) {
    phase(SYNC_READ_PEERS, [&](const NormLaunch& L, cudaStream_t s) { return LaunchNormMid(L, s); });
    if (kind == NORM_LANS)
      phase(SYNC_NONE, [&](const NormLaunch& L, cudaStream_t s) { return LaunchNormFinalize(L, 2, kNrmM, kNrmG2, 0, s); });
    else
      phase(SYNC_NONE, [&](const NormLaunch& L, cudaStream_t s) { return LaunchNormFinalize(L, 2, kNrmW, kNrmG, 0, s); });
  }
  phase(SYNC_WRITE_PEERS, [&](const NormLaunch& L, cudaStream_t s) { return LaunchNormApply(L, s); });

  for (auto& part : parts) {
    DeviceGuard dg(part.dev);
    DeviceState& d = rt->Dev(part.dev);
    CUDA_CALL(cudaFreeAsync(part.psum, d.stream));
    d.ring.Commit(part.off, part.bytes, d.stream);
  }
  for (auto& kv : bad_alloc) {
    DeviceGuard dg(kv.first);
    DeviceState& d = rt->Dev(kv.first);
    d.ring.Commit(kv.second.off, kv.second.bytes, d.stream);
  }
  if (opt_.skip_nonfinite) {
    for (auto& cls : classes)
      for (auto& t : (*cls.per_part)[my_first]) last_norm_keys_.push_back(t.key);
  }
}

int KVStore::ResolveOverflow() {
  LOCK();
  if (overflow_flag_ == nullptr) { last_norm_keys_.clear(); return 0; }
  Runtime::Get()->WaitAll();
  const int flag = *overflow_flag_;
  if (flag != 0) {
    // the skipped step does not count (the reference returns before the updater runs,
    // gluon/trainer.py:445-448, so Optimizer._update_count never sees it)
    for (int key : last_norm_keys_) {
      auto it = keys_.find(key);
      if (it != keys_.end() && it->second.count > 0) it->second.count -= 1;
    }
    *overflow_flag_ = 0;
  }
  last_norm_keys_.clear();
  return flag;
}

// multi_sum_sq (contrib/multi_sum_sq-inl.h:83-96) and multi_all_finite (all_finite.cu:68-103) over
// a list of arrays on one GPU: out_sumsq[i] = sum((scale * x_i)^2); all_finite[0] = 0 if any element
// of any array is inf/nan (init_output: set it to 1 first).
void MultiSumSq(const std::vector<NDArray>& arrays, float scale, NDArray* out_sumsq, NDArray* all_finite,
                bool init_output) {
  MXKV_CHECK(!arrays.empty()) << "multi_sum_sq: no arrays";
  Runtime* rt = Runtime::Get();
  std::lock_guard<std::recursive_mutex> lk(rt->mu());
  const int dev = arrays[0].dev();
  MXKV_CHECK(dev >= 0) << "multi_sum_sq: arrays must live on a GPU";
  const int dtype = arrays[0].dtype();
  for (auto& a : arrays) {
    MXKV_CHECK(a.dev() == dev) << "multi_sum_sq: all arrays must be on GPU " << dev;
    MXKV_CHECK(a.dtype() == dtype) << "multi_sum_sq: all arrays must share one dtype";
    MXKV_CHECK(a.stype() == kDefaultStorage) << "multi_sum_sq: dense arrays only";
  }
  const int n = static_cast<int>(arrays.size());
  if (out_sumsq) MXKV_CHECK(out_sumsq->dev() == dev && out_sumsq->dtype() == kFloat32 && out_sumsq->size() == n)
      << "multi_sum_sq: output must be float32 [" << n << "] on GPU " << dev;
  if (all_finite) MXKV_CHECK(all_finite->dev() == dev && all_finite->dtype() == kFloat32 && all_finite->size() >= 1)
      << "multi_all_finite: output must be float32 [1] on GPU " << dev;
  DeviceState& d = rt->Dev(dev);
  DeviceGuard dg(dev);
  rt->AcquireUser(dev);
  const int64_t chunk = rt->chunk_elems;
  std::vector<SumSqItem> items(n);
  std::vector<int64_t> prefix(n + 1);
  int64_t acc = 0;
  for (int i = 0; i < n; ++i) {
    items[i].ptr = arrays[i].data();
    items[i].n = arrays[i].size();
    prefix[i] = acc;
    acc += (arrays[i].size() + chunk - 1) / chunk;
  }
  prefix[n] = acc;
  const size_t ibytes = items.size() * sizeof(SumSqItem);
  const size_t pbytes = prefix.size() * sizeof(int64_t);
  const size_t off = d.ring.Alloc(ibytes + pbytes);
  std::memcpy(d.ring.host(off), items.data(), ibytes);
  std::memcpy(d.ring.host(off) + ibytes, prefix.data(), pbytes);
  CUDA_CALL(cudaMemcpyAsync(d.ring.dev(off), d.ring.host(off), ibytes + pbytes, cudaMemcpyHostToDevice, d.stream));
  float* scratch = nullptr;   // [chunks x 2] partials, then [n] non-finite counts
  const size_t sbytes = (static_cast<size_t>(acc) * 2 + n + 4) * sizeof(float);
  CUDA_CALL(cudaMallocAsync(reinterpret_cast<void**>(&scratch), sbytes, d.stream));
  float* bad = scratch + acc * 2;
  int rc = LaunchMultiSumSq(reinterpret_cast<const SumSqItem*>(d.ring.dev(off)),
                            reinterpret_cast<const int64_t*>(d.ring.dev(off) + ibytes), n, acc, dtype, scale, scratch,
                            out_sumsq ? static_cast<float*>(out_sumsq->data()) : nullptr, all_finite ? bad : nullptr,
                            static_cast<int>(chunk), d.stream);
  MXKV_CHECK(rc == 0) << "kernel launch failed: " << cudaGetErrorString(static_cast<cudaError_t>(rc));
  rt->launches += 2;
  if (all_finite) {
    rc = LaunchAllFiniteFlag(bad, n, static_cast<float*>(all_finite->data()), init_output ? 1 : 0, d.stream);
    MXKV_CHECK(rc == 0) << "kernel launch failed: " << cudaGetErrorString(static_cast<cudaError_t>(rc));
    rt->launches++;
  }
  CUDA_CALL(cudaFreeAsync(scratch, d.stream));
  d.ring.Commit(off, ibytes + pbytes, d.stream);
  rt->ReleaseToUser(dev);
}

}  // namespace mxkv
