// runtime.cc -- streams, event edges, peer access, staging rings, process group.
#include "runtime.h"
#include <cstdlib>
#include <algorithm>
#include <cstring>

namespace mxkv {

static thread_local std::string g_last_error;
void SetLastError(const std::string& msg) { g_last_error = msg; }
const char* GetLastError() { return g_last_error.c_str(); }

int64_t EnvInt(const char* name, int64_t dflt) {
  const char* v = std::getenv(name);
  if (v == nullptr || *v == 0) return dflt;
  return std::strtoll(v, nullptr, 10);
}

// ---------------------------------------------------------------------------
// StagingRing
// ---------------------------------------------------------------------------
void StagingRing::Init(int dev, size_t cap) {
  DeviceGuard g(dev);
  cap_ = cap;
  CUDA_CALL(cudaMallocHost(reinterpret_cast<void**>(&host_), cap));
  CUDA_CALL(cudaMalloc(reinterpret_cast<void**>(&dev_), cap));
  head_ = 0;
}

void StagingRing::Destroy() {
  for (auto& f : inflight_) cudaEventDestroy(f.ev);
  for (auto e : pool_) cudaEventDestroy(e);
  inflight_.clear(); pool_.clear();
  if (host_) cudaFreeHost(host_);
  if (dev_) cudaFree(dev_);
  host_ = dev_ = nullptr;
}

size_t StagingRing::Alloc(size_t bytes) {
  bytes = (bytes + 255) & ~static_cast<size_t>(255);
  MXKV_CHECK(bytes <= cap_) << "descriptor table of " << bytes << " bytes exceeds the staging ring";
  if (head_ + bytes > cap_) head_ = 0;
  const size_t b = head_, e = head_ + bytes;
  // retire (and if necessary wait for) every in-flight region overlapping [b, e)
  while (!inflight_.empty()) {
    InFlight& f = inflight_.front();
    const bool overlap = f.b < e && b < f.e;
    if (!overlap) {
      if (cudaEventQuery(f.ev) != cudaSuccess) break;   // still running, but not in our way
    } else {
      CUDA_CALL(cudaEventSynchronize(f.ev));
    }
    pool_.push_back(f.ev);
    inflight_.pop_front();
  }
  // regions behind a still-running non-overlapping head may overlap: check the rest
  for (auto& f : inflight_) {
    if (f.b < e && b < f.e) CUDA_CALL(cudaEventSynchronize(f.ev));
  }
  head_ = e;
  return b;
}

void StagingRing::Commit(size_t off, size_t bytes, cudaStream_t s) {
  bytes = (bytes + 255) & ~static_cast<size_t>(255);
  cudaEvent_t ev;
  if (!pool_.empty()) { ev = pool_.back(); pool_.pop_back(); }
  else CUDA_CALL(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  CUDA_CALL(cudaEventRecord(ev, s));
  inflight_.push_back({off, off + bytes, ev});
}

// ---------------------------------------------------------------------------
// ProcessGroup
// ---------------------------------------------------------------------------
ProcessGroup::ProcessGroup(int rank, int world, int dev, AllGatherFn fn, void* ctx)
    : rank_(rank), world_(world), dev_(dev), fn_(fn), ctx_(ctx) {
  MXKV_CHECK(world >= 1 && world <= kMaxRanks) << "world size " << world << " not in [1," << kMaxRanks << "]";
  MXKV_CHECK(rank >= 0 && rank < world) << "bad rank " << rank;
  MXKV_CHECK(fn != nullptr || world == 1) << "an all-gather callback is required when world > 1";
  DeviceGuard g(dev);
  pads_ = SymAlloc(kSignalPadBytes);
  CUDA_CALL(cudaMemset(pads_.ptr[rank_], 0, kSignalPadBytes));
  CUDA_CALL(cudaDeviceSynchronize());
  // nobody may signal into a pad that has not been zeroed yet: this exchange (who sits on which GPU -- the link
  // matrix of MXNET_KVSTORE_USETREE is asked for by device ordinal) doubles as the barrier
  std::vector<int64_t> all(world_);
  const int64_t mine = dev_;
  AllGather(&mine, sizeof(mine), all.data());
  rank_devs_.assign(all.begin(), all.end());
}

ProcessGroup::~ProcessGroup() {
  for (auto& s : segs_) {
    if (s.vmm) { FreeSegmentVmm(s); continue; }
    for (int r = 0; r < world_; ++r) {
      if (s.base[r] == nullptr) continue;
      if (r == rank_) cudaFree(s.base[r]);
      else cudaIpcCloseMemHandle(s.base[r]);
    }
  }
}

void ProcessGroup::AllGather(const void* send, size_t bytes, void* recv) {
  if (world_ == 1) { std::memcpy(recv, send, bytes); return; }
  const int rc = fn_(send, bytes, recv, ctx_);
  MXKV_CHECK(rc == 0) << "bootstrap all-gather callback failed with code " << rc;
}

void ProcessGroup::Barrier() {
  int64_t x = rank_;
  std::vector<int64_t> all(world_);
  AllGather(&x, sizeof(x), all.data());
}

void ProcessGroup::NewSegment(size_t min_bytes) {
  DeviceGuard g(dev_);
  size_t bytes = static_cast<size_t>(EnvInt("MXKV_B200_ARENA_MB", 1024)) << 20;
  if (bytes < min_bytes) bytes = (min_bytes + (size_t(64) << 20) - 1) & ~((size_t(64) << 20) - 1);
  Segment s;
  std::memset(&s, 0, sizeof(s));
  if (world_ > 1 && vmm_mode_ != 0) {
    // engine-owned multicast memory (vmm_arena.cc); the first segment decides for the life of the group
    const bool want = vmm_mode_ == 1 || EnvInt("MXKV_B200_ARENA_VMM", 1) != 0;
    const bool got = want && NewSegmentVmm(bytes, &s);
    // a later segment that cannot be had (multicast objects are a finite resource) is an ordinary IPC segment:
    // its arrays simply have no multicast alias; no further attempts are made
    vmm_mode_ = got ? 1 : 0;
    if (got) { segs_.push_back(s); return; }
    std::memset(&s, 0, sizeof(s));
  }
  s.bytes = bytes; s.used = 0;
  char* mine = nullptr;
  CUDA_CALL(cudaMalloc(reinterpret_cast<void**>(&mine), bytes));
  s.base[rank_] = mine;
  if (world_ > 1) {
    struct Msg { cudaIpcMemHandle_t h; uint64_t bytes; };
    Msg m;
    std::memset(&m, 0, sizeof(m));
    CUDA_CALL(cudaIpcGetMemHandle(&m.h, mine));
    m.bytes = bytes;
    std::vector<Msg> all(world_);
    AllGather(&m, sizeof(Msg), all.data());
    for (int r = 0; r < world_; ++r) {
      if (r == rank_) continue;
      MXKV_CHECK(all[r].bytes == bytes) << "rank " << r << " created an arena segment of a different size";
      void* p = nullptr;
      CUDA_CALL(cudaIpcOpenMemHandle(&p, all[r].h, cudaIpcMemLazyEnablePeerAccess));
      s.base[r] = static_cast<char*>(p);
    }
  }
  segs_.push_back(s);
}

SymPtr ProcessGroup::SymAlloc(size_t bytes) {
  bytes = (bytes + 511) & ~static_cast<size_t>(511);
  if (segs_.empty() || segs_.back().used + bytes > segs_.back().bytes) NewSegment(bytes);
  Segment& s = segs_.back();
  const uint64_t off = s.used;
  s.used += bytes;
  used_total_ += bytes;
  // bump-only allocation is deterministic; verify that the ranks agree anyway
  if (world_ > 1) {
    uint64_t msg[3] = {static_cast<uint64_t>(segs_.size() - 1), off, bytes};
    std::vector<uint64_t> all(3 * world_);
    AllGather(msg, sizeof(msg), all.data());
    for (int r = 0; r < world_; ++r)
      MXKV_CHECK(all[3 * r] == msg[0] && all[3 * r + 1] == off && all[3 * r + 2] == bytes)
          << "symmetric allocation mismatch between rank " << rank_ << " and rank " << r
          << ": collective allocations must be issued in the same order with the same sizes";
  }
  SymPtr p;
  for (int r = 0; r < world_; ++r) p.ptr[r] = s.base[r] + off;
  p.mc = s.mc ? s.mc + off : nullptr;
  p.valid = true;
  return p;
}

// ---------------------------------------------------------------------------
// Runtime
// ---------------------------------------------------------------------------
Runtime::Runtime() {
  twoshot_bytes = EnvInt("MXKV_B200_TWOSHOT_BYTES", 256 * 1024);
  auto_fence = EnvInt("MXKV_B200_AUTO_FENCE", 1) != 0;
  chunk_elems = EnvInt("MXKV_B200_CHUNK", kChunkElems);
  if (chunk_elems < 128) chunk_elems = 128;
  chunk_elems = (chunk_elems + 127) / 128 * 128;
  bulk_mode = static_cast<int>(EnvInt("MXKV_B200_BULK", 1));
  bulk_group_forced = std::getenv("MXKV_B200_BULK_GROUP") != nullptr;
  bulk_group = static_cast<int>(EnvInt("MXKV_B200_BULK_GROUP", bulk_group));
  if (bulk_group < 1) bulk_group = 1;
  nvls_mode = static_cast<int>(EnvInt("MXKV_B200_NVLS", 1));
  nvls_unroll = static_cast<int>(EnvInt("MXKV_B200_NVLS_U", nvls_unroll));
  nvls_pipe = static_cast<int>(EnvInt("MXKV_B200_NVLS_PIPE", nvls_pipe));
  nvls_grid = static_cast<int>(EnvInt("MXKV_B200_NVLS_GRID", nvls_grid));
  nvls_threads = static_cast<int>(EnvInt("MXKV_B200_NVLS_THREADS", nvls_threads));
  if (nvls_threads != 128 && nvls_threads != 256 && nvls_threads != 512) nvls_threads = 512;
  spin_timeout_cycles = EnvInt("MXKV_B200_SPIN_TIMEOUT_S", 120) * 1900000000LL;   // ~1.9 GHz SM clock
  max_blocks = static_cast<int>(EnvInt("MXKV_B200_MAX_BLOCKS", 0));
  threads = static_cast<int>(EnvInt("MXKV_B200_THREADS", 512));
  if (threads != 128 && threads != 256 && threads != 512) threads = 512;
}

Runtime* Runtime::Get() {
  static Runtime* inst = new Runtime();   // intentionally leaked: CUDA may unload first at exit
  return inst;
}

int Runtime::NumDevices() {
  if (ndev_ < 0) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) { cudaGetLastError(); n = 0; }
    ndev_ = n;
  }
  return ndev_;
}

DeviceState& Runtime::Dev(int dev) {
  std::lock_guard<std::recursive_mutex> lk(mu_);
  auto it = devs_.find(dev);
  if (it != devs_.end()) return *it->second;
  MXKV_CHECK(dev >= 0 && dev < NumDevices())
      << "GPU " << dev << " requested but " << NumDevices()
      << " CUDA device(s) are visible; this library has no CPU fallback";
  std::unique_ptr<DeviceState> d(new DeviceState());
  d->dev = dev;
  DeviceGuard g(dev);
  int lo = 0, hi = 0;
  CUDA_CALL(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  CUDA_CALL(cudaStreamCreateWithPriority(&d->stream, cudaStreamNonBlocking, hi));
  CUDA_CALL(cudaEventCreateWithFlags(&d->ev_user, cudaEventDisableTiming));
  CUDA_CALL(cudaEventCreateWithFlags(&d->ev_engine, cudaEventDisableTiming));
  CUDA_CALL(cudaEventCreateWithFlags(&d->ev_xdev, cudaEventDisableTiming));
  CUDA_CALL(cudaStreamCreateWithFlags(&d->copy_in, cudaStreamNonBlocking));
  CUDA_CALL(cudaStreamCreateWithFlags(&d->copy_out, cudaStreamNonBlocking));
  for (int i = 0; i < DeviceState::kHostSlots; ++i) {
    CUDA_CALL(cudaEventCreateWithFlags(&d->ev_h2d[i], cudaEventDisableTiming));
    CUDA_CALL(cudaEventCreateWithFlags(&d->ev_kern[i], cudaEventDisableTiming));
  }
  CUDA_CALL(cudaEventCreateWithFlags(&d->ev_d2h_all, cudaEventDisableTiming));
  if (pg_ && pg_->dev() == dev) {
    d->signal_pad = pg_->signal_pad(pg_->rank());
  } else {
    CUDA_CALL(cudaMalloc(reinterpret_cast<void**>(&d->signal_pad), kSignalPadBytes));
    CUDA_CALL(cudaMemset(d->signal_pad, 0, kSignalPadBytes));
    CUDA_CALL(cudaDeviceSynchronize());
  }
  {
    // stream-ordered temporaries (host staging of CPU-resident values): keep the pool warm
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      uint64_t thr = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    cudaGetLastError();
  }
  d->ring.Init(dev, static_cast<size_t>(EnvInt("MXKV_B200_RING_MB", 8)) << 20);
  CUDA_CALL(cudaMalloc(reinterpret_cast<void**>(&d->list_dev), DeviceState::kResidentListBytes));
  d->max_grid = DenseMaxGrid(dev, threads);
  const int64_t cap = max_blocks_override_ > 0 ? max_blocks_override_ : EnvInt("MXKV_B200_MAX_BLOCKS", 0);
  if (cap > 0 && cap < d->max_grid) d->max_grid = static_cast<int>(cap);
  DeviceState& ref = *d;
  devs_[dev] = std::move(d);
  return ref;
}

bool Runtime::PeerOK(int a, int b) {
  if (a == b) return true;
  std::lock_guard<std::recursive_mutex> lk(mu_);
  auto it = peer_ok_.find((static_cast<int64_t>(a) << 32) | b);
  return it != peer_ok_.end() && it->second;
}

void Runtime::EnablePeerAccess(const std::vector<int>& devs) {
  std::lock_guard<std::recursive_mutex> lk(mu_);
  if (EnvInt("MXNET_ENABLE_GPU_P2P", 1) == 0) return;   // comm.h:473
  for (int a : devs) {
    for (int b : devs) {
      if (a == b) continue;
      const int64_t k = (static_cast<int64_t>(a) << 32) | b;
      if (peer_ok_.count(k)) continue;
      int can = 0;
      CUDA_CALL(cudaDeviceCanAccessPeer(&can, a, b));
      bool ok = false;
      if (can) {
        DeviceGuard g(a);
        cudaError_t e = cudaDeviceEnablePeerAccess(b, 0);
        if (e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled) ok = true;
        cudaGetLastError();
      }
      peer_ok_[k] = ok;
    }
  }
}

void Runtime::SetUserStream(int dev, cudaStream_t s) { Dev(dev).user_stream = s; }

void Runtime::AcquireUser(int dev) {
  DeviceState& d = Dev(dev);
  DeviceGuard g(dev);
  CUDA_CALL(cudaEventRecord(d.ev_user, d.user_stream));
  CUDA_CALL(cudaStreamWaitEvent(d.stream, d.ev_user, 0));
}

void Runtime::ReleaseToUser(int dev) {
  DeviceState& d = Dev(dev);
  d.engine_dirty = true;
  if (auto_fence) Fence(dev);
}

void Runtime::Fence(int dev) {
  {
    std::lock_guard<std::recursive_mutex> lk(mu_);
    if (devs_.find(dev) == devs_.end()) return;   // the engine never touched this GPU
  }
  DeviceState& d = Dev(dev);
  if (!d.engine_dirty) return;
  DeviceGuard g(dev);
  CUDA_CALL(cudaEventRecord(d.ev_engine, d.stream));
  CUDA_CALL(cudaStreamWaitEvent(d.user_stream, d.ev_engine, 0));
  d.engine_dirty = false;
}

void Runtime::StreamWait(int waiter_dev, int signaler_dev) {
  if (waiter_dev == signaler_dev) return;
  DeviceState& s = Dev(signaler_dev);
  DeviceState& w = Dev(waiter_dev);
  {
    DeviceGuard g(signaler_dev);
    CUDA_CALL(cudaEventRecord(s.ev_xdev, s.stream));
  }
  DeviceGuard g(waiter_dev);
  CUDA_CALL(cudaStreamWaitEvent(w.stream, s.ev_xdev, 0));
}

void Runtime::WaitDevice(int dev) {
  std::lock_guard<std::recursive_mutex> lk(mu_);
  auto it = devs_.find(dev);
  if (it == devs_.end()) return;
  DeviceGuard g(dev);
  CUDA_CALL(cudaStreamSynchronize(it->second->stream));
}

void Runtime::WaitAll() {
  std::lock_guard<std::recursive_mutex> lk(mu_);
  for (auto& kv : devs_) {
    DeviceGuard g(kv.first);
    CUDA_CALL(cudaStreamSynchronize(kv.second->stream));
  }
}

void Runtime::SetTuning(int64_t chunk, int nthreads, int max_blocks, int bulk) {
  tuning_epoch++;
  if (bulk >= 0) bulk_mode = bulk;
  std::lock_guard<std::recursive_mutex> lk(mu_);
  WaitAll();
  if (chunk > 0) chunk_elems = std::max<int64_t>(128, (chunk + 127) / 128 * 128);
  if (nthreads == 128 || nthreads == 256 || nthreads == 512) threads = nthreads;
  for (auto& kv : devs_) {
    int g = DenseMaxGrid(kv.first, threads);
    if (max_blocks > 0 && max_blocks < g) g = max_blocks;
    kv.second->max_grid = g;
  }
  max_blocks_override_ = max_blocks;
  this->max_blocks = max_blocks;
}

void Runtime::DrainForFree() noexcept {
  try {
    std::lock_guard<std::recursive_mutex> lk(mu_);
    int prev = -1;
    cudaGetDevice(&prev);
    for (auto& kv : devs_) {
      cudaSetDevice(kv.first);
      cudaStreamSynchronize(kv.second->stream);
    }
    if (prev >= 0) cudaSetDevice(prev);
    cudaGetLastError();
  } catch (...) {
  }
}

void Runtime::InitProcessGroup(int rank, int world, int dev, AllGatherFn fn, void* ctx) {
  tuning_epoch++;
  std::lock_guard<std::recursive_mutex> lk(mu_);
  MXKV_CHECK(!pg_) << "process group already initialised";
  MXKV_CHECK(devs_.find(dev) == devs_.end())
      << "MXKVB200CommInit must be called before the first use of GPU " << dev;
  MXKV_CHECK(dev >= 0 && dev < NumDevices()) << "GPU " << dev << " is not visible";
  pg_.reset(new ProcessGroup(rank, world, dev, fn, ctx));
}

void Runtime::DestroyProcessGroup() {
  tuning_epoch++;
  std::lock_guard<std::recursive_mutex> lk(mu_);
  WaitAll();
  if (pg_) {
    auto it = devs_.find(pg_->dev());
    if (it != devs_.end()) {   // the device's signal pad lived in the arena: give it a private one
      DeviceGuard g(pg_->dev());
      uint32_t* pad = nullptr;
      CUDA_CALL(cudaMalloc(reinterpret_cast<void**>(&pad), kSignalPadBytes));
      CUDA_CALL(cudaMemset(pad, 0, kSignalPadBytes));
      CUDA_CALL(cudaDeviceSynchronize());
      it->second->signal_pad = pad;
    }
  }
  pg_.reset();
}

}  // namespace mxkv
