// runtime.h -- the host side that replaces the reference's dependency engine and
// device plumbing for this path.
//
// Reference                                   | here
// --------------------------------------------+---------------------------------------------
// ThreadedEnginePerDevice worker pools, one   | one in-order, high-priority CUDA stream per GPU
//   mshadow stream per worker thread, host    |   (the "engine stream"); dependencies are CUDA
//   blocking stream->Wait() in every op       |   events between streams, the host never blocks
//   (src/engine/threaded_engine_perdevice.cc, |   except in WaitToRead/WaitAll
//    src/ndarray/ndarray.cc:1396-1412,1477)   |
// ThreadedVar read/write queues               | per-call event edges user-stream -> engine-stream
//   (src/engine/threaded_engine.cc:51-190)    |   -> user-stream (AcquireUser / ReleaseToUser)
// CommDevice::EnableP2P (comm.h:728-770)      | EnablePeerAccess + peer-mapped signal pads
// (no equivalent: single process only)        | ProcessGroup: one process per GPU, symmetric
//                                             |   arena exported with cudaIpc*, host all-gather
//                                             |   callback supplied by the embedding language
#pragma once
#include <deque>
#include <memory>
#include <mutex>
#include <unordered_map>
#include <vector>
#include "base.h"

namespace mxkv {

// Host all-gather used only for bootstrap (IPC handle / offset exchange).  Must
// gather `bytes` from every rank into recv[rank*bytes ...].  Returns 0 on success.
typedef int (*AllGatherFn)(const void* send, size_t bytes, void* recv, void* ctx);

class StagingRing {
 public:
  void Init(int dev, size_t cap);
  void Destroy();
  // reserve `bytes` (256-aligned) in the mirrored host/device rings; blocks only if
  // the region is still referenced by a launch that has not finished
  size_t Alloc(size_t bytes);
  void Commit(size_t off, size_t bytes, cudaStream_t s);   // call after the consuming launch
  char* host(size_t off) const { return host_ + off; }
  char* dev(size_t off) const { return dev_ + off; }
 private:
  struct InFlight { size_t b, e; cudaEvent_t ev; };
  char* host_ = nullptr;
  char* dev_ = nullptr;
  size_t cap_ = 0, head_ = 0;
  std::deque<InFlight> inflight_;
  std::vector<cudaEvent_t> pool_;
};

struct DeviceState {
  int dev = -1;
  cudaStream_t stream = nullptr;       // engine stream
  cudaStream_t user_stream = nullptr;  // stream the embedding framework computes on (legacy default)
  cudaEvent_t ev_user = nullptr;
  cudaEvent_t ev_engine = nullptr;
  cudaEvent_t ev_xdev = nullptr;
  uint32_t* signal_pad = nullptr;      // this device's pad (SP mode: cudaMalloc; MP mode: in the arena)
  StagingRing ring;
  // The dense work list (TensorWork[] + chunk prefix) last uploaded on `stream`, kept resident: a launch whose list is
  // byte-for-byte the same (a pushpull of the same keys with the same hyper-parameters) reads it without an upload.
  static constexpr size_t kResidentListBytes = 128 << 10;   // ResNet-50's and BERT-base's lists fit
  char* list_dev = nullptr;
  std::vector<char> list_host;         // what list_dev holds once the engine stream has reached this point
  int max_grid = 2 * kNumSms;
  bool engine_dirty = false;           // engine stream has work the user stream has not been fenced on
  // host-resident values: H2D / compute / D2H software pipeline (kvstore.cc: HostPipelined)
  static constexpr int kHostSlots = 3;
  cudaStream_t copy_in = nullptr, copy_out = nullptr;
  cudaEvent_t ev_h2d[kHostSlots] = {nullptr}, ev_kern[kHostSlots] = {nullptr};
  cudaEvent_t ev_d2h_all = nullptr;
  void* host_stage[kHostSlots] = {nullptr};
  size_t host_stage_bytes = 0;
  // one process per GPU: the slots live in the peer-mapped arena (every rank's kernel reads every rank's slot)
  void* host_stage_peer[kHostSlots][kMaxRanks] = {{nullptr}};
  size_t host_stage_peer_bytes = 0;
};

// Multi-node jobs (dist_device_sync): the process group above spans ONE node (the GPUs that share an NVSwitch
// domain and this library's peer-mapped arena); between the nodes the only thing the engine needs is a sum of a
// device buffer over the ranks that hold the same local rank on every node.  The embedding framework provides
// it (NCCL over the network in production), ordered on the CUDA stream it is handed.
typedef int (*AllReduceFn)(void* dev_ptr, int64_t count, int dtype, void* cuda_stream, void* ctx);
struct Hierarchy {
  int node_rank = 0;
  int num_nodes = 1;
  AllReduceFn fn = nullptr;
  void* ctx = nullptr;
  bool configured() const { return fn != nullptr; }
};

struct SymPtr {                 // one symmetric allocation as seen from this process
  void* ptr[kMaxRanks] = {nullptr};
  void* mc = nullptr;           // NVSwitch multicast alias of all copies (engine-owned VMM arena, vmm_arena.cc)
  bool valid = false;
};

class ProcessGroup {
 public:
  ProcessGroup(int rank, int world, int dev, AllGatherFn fn, void* ctx);
  ~ProcessGroup();
  int rank() const { return rank_; }
  int world() const { return world_; }
  int dev() const { return dev_; }
  const std::vector<int>& rank_devs() const { return rank_devs_; }   // CUDA device ordinal of every rank
  // collective: every rank must call with the same byte count, in the same order
  SymPtr SymAlloc(size_t bytes);
  void AllGather(const void* send, size_t bytes, void* recv);
  void Barrier();
  uint32_t* signal_pad(int r) const { return pads_.ptr[r] ? static_cast<uint32_t*>(pads_.ptr[r]) : nullptr; }
  size_t arena_used() const { return used_total_; }
  uint32_t NextSyncEpoch() { return ++sync_epoch_; }     // every rank issues the same collective launches in order
 private:
  uint32_t sync_epoch_ = 0;
  void NewSegment(size_t min_bytes);
  struct Segment { char* base[kMaxRanks]; size_t bytes; size_t used; char* mc; bool vmm; };
  // vmm_arena.cc: cuMemCreate + POSIX-fd exchange + cuMulticast*; collective, all ranks succeed or all fail
  bool NewSegmentVmm(size_t min_bytes, Segment* out);
  void FreeSegmentVmm(Segment& s);
  int vmm_mode_ = -1;           // -1 not decided yet, 0 cudaMalloc + cudaIpc from now on, 1 VMM + multicast so far
 public:
  bool has_multicast() const { for (auto& s : segs_) if (s.vmm) return true; return false; }
 private:
  int rank_, world_, dev_;
  std::vector<int> rank_devs_;
  AllGatherFn fn_;
  void* ctx_;
  std::vector<Segment> segs_;
  SymPtr pads_;
  size_t used_total_ = 0;
};

class Runtime {
 public:
  static Runtime* Get();
  DeviceState& Dev(int dev);                 // lazily creates streams, pad, ring
  int NumDevices();
  void EnablePeerAccess(const std::vector<int>& devs);   // SP mode, idempotent
  bool PeerOK(int a, int b);
  // ordering edges between the embedding framework's stream and the engine stream
  void AcquireUser(int dev);
  void ReleaseToUser(int dev);
  void Fence(int dev);                       // user stream waits for everything queued on the engine stream
  void StreamWait(int waiter_dev, int signaler_dev);
  void SetUserStream(int dev, cudaStream_t s);
  void WaitAll();
  void DrainForFree() noexcept;            // like WaitAll, never throws (used by destructors)
  void WaitDevice(int dev);
  void SetTuning(int64_t chunk, int nthreads, int max_blocks, int bulk = -1);

  // one-process-per-GPU mode
  void InitProcessGroup(int rank, int world, int dev, AllGatherFn fn, void* ctx);
  void DestroyProcessGroup();
  ProcessGroup* pg() { return pg_.get(); }
  Hierarchy hier;                            // MXKVB200SetHierarchy

  // the flag value of the next collective launch (kernels.h: SyncArgs::epoch): the group's counter in
  // one-process-per-GPU mode, a process-wide one for single-process launches over any subset of the GPUs
  uint32_t NextSyncEpoch(ProcessGroup* pg) { return pg != nullptr ? pg->NextSyncEpoch() : ++sync_epoch_; }
  std::recursive_mutex& mu() { return mu_; }
  bool auto_fence = true;
  int64_t launches = 0;                      // kernels launched by this library (bench "gpu_launches")
  uint64_t tuning_epoch = 0;                 // bumped by every change of a knob that shapes launches (cached plans expire)
  // dense launches by kernel variant: 0 per-thread (kv_dense_kernel / kv_sum_typed_kernel), 1 shared-memory
  // staged (kv_dense_bulk_kernel), 2 NVSwitch multicast (kv_dense_nvls_kernel) -- lets a parity test prove
  // which kernel it has just compared with the oracle (MXKVB200GetVariantLaunchCount)
  // 3: the tree-order kernels of MXNET_KVSTORE_USETREE (kv_dense_tree_kernel / kv_sum_tree_f64_kernel)
  int64_t variant_launches[4] = {0, 0, 0, 0};
  int64_t twoshot_bytes = 256 * 1024;
  int64_t chunk_elems = kChunkElems;         // MXKV_B200_CHUNK
  int threads = 512;                         // MXKV_B200_THREADS
  long long spin_timeout_cycles = 0;         // MXKV_B200_SPIN_TIMEOUT_S (default 120 s) in SM cycles
  int max_blocks = 0;                        // MXKV_B200_MAX_BLOCKS (0: resident capacity)
  int nvls_mode = 1;                         // MXKV_B200_NVLS: use multimem kernels for multicast-bound arrays
  int nvls_unroll = 2;                       // MXKV_B200_NVLS_U: ld_reduce requests in flight per thread (1 | 2 | 4 | 8)
  int nvls_pipe = 0;                         // MXKV_B200_NVLS_PIPE: issue the next chunk's ld_reduce before this chunk's update
  int nvls_grid = 48;                        // MXKV_B200_NVLS_GRID: cap on the multicast kernel's grid (0: resident capacity).
                                             // The switch, not the SMs, bounds this kernel: a small grid leaves most
                                             // SMs to whatever else is running (tools/tune_nvls.py sweeps it)
  int nvls_threads = 512;                    // MXKV_B200_NVLS_THREADS: its block size (128 | 256 | 512)
  int bulk_mode = 1;                         // MXKV_B200_BULK: 0 off, 1 auto (<= 2 sources), 2 whenever eligible
  int bulk_group = 4;                        // MXKV_B200_BULK_GROUP: consecutive tiles per block of the staged kernel,
  bool bulk_group_forced = false;            // for work lists of >= 32 keys (always when the variable is set)
 private:
  Runtime();
  std::recursive_mutex mu_;
  std::unordered_map<int, std::unique_ptr<DeviceState>> devs_;
  std::unordered_map<int64_t, bool> peer_ok_;
  std::unique_ptr<ProcessGroup> pg_;
  int ndev_ = -1;
  int max_blocks_override_ = 0;
  uint32_t sync_epoch_ = 0;
};

}  // namespace mxkv
