// fake_cudart.cc -- a stand-in for libcudart.so.12 that lets the engine's HOST code run on a machine
// without a GPU (test infrastructure only; see tests/sim/README.md).
//
// "Device" memory is host memory, every "GPU" lives in this process and can reach every other one,
// streams execute synchronously in issue order, events are no-ops.  A kernel launch is dispatched by the
// kernel's (demangled) name to a semantic emulator in sim_kernels.cc, which performs what the kernel is
// specified to do with the launch descriptor it was given -- using the very arithmetic headers the real
// kernels are compiled from (csrc/optim_math.h, csrc/norm_math.h), so results are bit-identical to the
// oracle.  What this exercises is everything AROUND the kernels: key bookkeeping, placement, replica and
// state management, work-list construction, aliasing rules, launch sequencing, the C ABI and the Python
// front-end.  It cannot find a bug inside a CUDA kernel; the `-m gpu` tests on real hardware do that.
//
// The number of simulated GPUs is MXKV_SIM_DEVICES (default 4).
#include <cuda_runtime_api.h>
#include <cxxabi.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include "sim.h"

namespace {

std::mutex g_mu;
std::map<const void*, std::string> g_kernels;     // host stub address -> demangled kernel name
thread_local int g_device = 0;
thread_local cudaError_t g_last = cudaSuccess;

struct CallConfig { dim3 grid, block; size_t smem; void* stream; };
thread_local CallConfig g_cfg;

int device_count() {
  const char* e = getenv("MXKV_SIM_DEVICES");
  const int n = (e && *e) ? atoi(e) : 4;
  return n < 1 ? 1 : (n > 8 ? 8 : n);
}

cudaError_t fail(cudaError_t e) { g_last = e; return e; }

// Allocations of 1 MiB and more are backed by named POSIX shared memory so that another simulated "GPU
// process" can map them (cudaIpcGetMemHandle / cudaIpcOpenMemHandle: the one-process-per-GPU mode).
struct Shm { std::string name; size_t bytes; bool owner; };
std::map<void*, Shm> g_shm;
int g_shm_counter = 0;

void unlink_owned_shm() {           // a process that exits without freeing must not leave /dev/shm entries behind
  for (auto& kv : g_shm)
    if (kv.second.owner) shm_unlink(kv.second.name.c_str());
}
constexpr size_t kShmThreshold = 1 << 20;

void* sim_alloc(size_t bytes) {
  if (bytes >= kShmThreshold) {
    char name[64];
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_shm_counter == 0) atexit(unlink_owned_shm);
    snprintf(name, sizeof(name), "/mxkvsim_%d_%d", static_cast<int>(getpid()), g_shm_counter++);
    const int fd = shm_open(name, O_CREAT | O_RDWR | O_EXCL, 0600);
    if (fd < 0) return nullptr;
    if (ftruncate(fd, static_cast<off_t>(bytes)) != 0) { close(fd); shm_unlink(name); return nullptr; }
    void* p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (p == MAP_FAILED) { shm_unlink(name); return nullptr; }
    g_shm[p] = Shm{name, bytes, true};
    return p;
  }
  void* p = nullptr;
  if (posix_memalign(&p, 512, bytes ? bytes : 16) != 0) return nullptr;
  return p;
}

void sim_free(void* p) {
  if (p == nullptr) return;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_shm.find(p);
    if (it != g_shm.end()) {
      munmap(p, it->second.bytes);
      if (it->second.owner) shm_unlink(it->second.name.c_str());
      g_shm.erase(it);
      return;
    }
  }
  free(p);
}

}  // namespace

#define API extern "C" __attribute__((visibility("default")))

// ---- registration of the kernels compiled into the engine -----------------------------------
API void** __cudaRegisterFatBinary(void*) { static void* h = nullptr; return &h; }
API void __cudaRegisterFatBinaryEnd(void**) {}
API void __cudaUnregisterFatBinary(void**) {}
API void __cudaRegisterFunction(void**, const char* hostFun, char*, const char* deviceName, int, uint3*, uint3*,
                                dim3*, dim3*, int*) {
  int status = 0;
  char* dem = abi::__cxa_demangle(deviceName, nullptr, nullptr, &status);
  std::lock_guard<std::mutex> lk(g_mu);
  g_kernels[hostFun] = (status == 0 && dem) ? dem : deviceName;
  free(dem);
}
API void __cudaRegisterVar(void**, char*, char*, const char*, int, size_t, int, int) {}
API unsigned __cudaPushCallConfiguration(dim3 grid, dim3 block, size_t smem, void* stream) {
  g_cfg = CallConfig{grid, block, smem, stream};
  return 0;
}
API cudaError_t __cudaPopCallConfiguration(dim3* grid, dim3* block, size_t* smem, void* stream) {
  *grid = g_cfg.grid; *block = g_cfg.block; *smem = g_cfg.smem;
  *static_cast<void**>(stream) = g_cfg.stream;
  return cudaSuccess;
}

API cudaError_t cudaLaunchKernel(const void* func, dim3 grid, dim3 block, void** args, size_t smem, cudaStream_t) {
  std::string name;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_kernels.find(func);
    if (it == g_kernels.end()) return fail(cudaErrorInvalidDeviceFunction);
    name = it->second;
  }
  static const bool noexec = getenv("MXKV_SIM_NOEXEC") != nullptr;   // host-overhead measurements: launch = no-op
  if (noexec) return cudaSuccess;
  sim::LaunchInfo info;
  info.name = name;
  info.grid = grid.x; info.grid_y = grid.y; info.block = block.x; info.smem = smem;
  info.device = g_device;
  if (!sim::Dispatch(info, args)) {
    fprintf(stderr, "[mxkv sim] no emulator for kernel: %s\n", name.c_str());
    return fail(cudaErrorNotSupported);
  }
  return cudaSuccess;
}

// ---- devices ------------------------------------------------------------------------------------
API cudaError_t cudaGetDeviceCount(int* n) { *n = device_count(); return cudaSuccess; }
API cudaError_t cudaGetDevice(int* d) { *d = g_device; return cudaSuccess; }
API cudaError_t cudaSetDevice(int d) {
  if (d < 0 || d >= device_count()) return fail(cudaErrorInvalidDevice);
  g_device = d;
  return cudaSuccess;
}
API cudaError_t cudaDeviceSynchronize(void) { return cudaSuccess; }
API cudaError_t cudaDeviceCanAccessPeer(int* can, int a, int b) { *can = (a != b) ? 1 : 0; return cudaSuccess; }
API cudaError_t cudaDeviceEnablePeerAccess(int, unsigned) { return cudaSuccess; }
// every pair behind one switch: performance rank 0 (what an NVSwitch machine reports)
API cudaError_t cudaDeviceGetP2PAttribute(int* value, cudaDeviceP2PAttr, int, int) { *value = 0; return cudaSuccess; }
API cudaError_t cudaDeviceGetStreamPriorityRange(int* lo, int* hi) { *lo = 0; *hi = -5; return cudaSuccess; }
API cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr attr, int) {
  switch (attr) {
    case cudaDevAttrMultiProcessorCount: *v = 132; break;
    case cudaDevAttrClockRate: *v = 1980000; break;
    case cudaDevAttrMaxSharedMemoryPerBlockOptin: *v = 227 * 1024; break;
    default: *v = 0; break;
  }
  return cudaSuccess;
}
API cudaError_t cudaDeviceGetDefaultMemPool(cudaMemPool_t* pool, int) { *pool = nullptr; return cudaSuccess; }
API cudaError_t cudaMemPoolSetAttribute(cudaMemPool_t, cudaMemPoolAttr, void*) { return cudaSuccess; }
API cudaError_t cudaFuncSetAttribute(const void*, cudaFuncAttribute, int) { return cudaSuccess; }
// the driver entry points of csrc/vmm_arena.cc (VMM allocations, multicast objects) are served by fake_driver.cc;
// anything else is "not found", as on a machine without a driver
namespace sim { void* DriverEntry(const char* name); }
API cudaError_t cudaGetDriverEntryPoint(const char* name, void** fn, unsigned long long, cudaDriverEntryPointQueryResult* status) {
  void* p = sim::DriverEntry(name);
  if (fn) *fn = p;
  if (status) *status = p ? cudaDriverEntryPointSuccess : cudaDriverEntryPointSymbolNotFound;
  return p ? cudaSuccess : cudaErrorNotSupported;
}

API cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags(int* n, const void*, int, size_t, unsigned) {
  *n = 2;
  return cudaSuccess;
}

// ---- errors ---------------------------------------------------------------------------------------
API cudaError_t cudaGetLastError(void) { const cudaError_t e = g_last; g_last = cudaSuccess; return e; }
API const char* cudaGetErrorString(cudaError_t e) {
  switch (e) {
    case cudaSuccess: return "no error";
    case cudaErrorNotSupported: return "operation not supported (simulated runtime)";
    case cudaErrorInvalidValue: return "invalid argument";
    case cudaErrorInvalidDevice: return "invalid device ordinal";
    case cudaErrorInvalidDeviceFunction: return "invalid device function";
    default: return "simulated CUDA error";
  }
}

// ---- memory -----------------------------------------------------------------------------------------
API cudaError_t cudaMalloc(void** p, size_t n) { *p = sim_alloc(n); return *p ? cudaSuccess : fail(cudaErrorMemoryAllocation); }
API cudaError_t cudaMallocAsync(void** p, size_t n, cudaStream_t) { return cudaMalloc(p, n); }
API cudaError_t cudaMallocHost(void** p, size_t n) { return cudaMalloc(p, n); }
API cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { return cudaMalloc(p, n); }
API cudaError_t cudaFree(void* p) { sim_free(p); return cudaSuccess; }
API cudaError_t cudaFreeAsync(void* p, cudaStream_t) { sim_free(p); return cudaSuccess; }
API cudaError_t cudaFreeHost(void* p) { sim_free(p); return cudaSuccess; }
API cudaError_t cudaMemcpyAsync(void* dst, const void* src, size_t n, cudaMemcpyKind, cudaStream_t) {
  if (n) memmove(dst, src, n);
  return cudaSuccess;
}
API cudaError_t cudaMemcpyPeerAsync(void* dst, int, const void* src, int, size_t n, cudaStream_t) {
  if (n) memmove(dst, src, n);
  return cudaSuccess;
}
API cudaError_t cudaMemset(void* p, int v, size_t n) { if (n) memset(p, v, n); return cudaSuccess; }
API cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { return cudaMemset(p, v, n); }
// IPC handle = name and size of the shared-memory object behind the allocation (64 bytes, like the real one)
API cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_shm.find(p);
  if (it == g_shm.end()) return fail(cudaErrorInvalidValue);
  memset(h, 0, sizeof(*h));
  snprintf(h->reserved, 48, "%s", it->second.name.c_str());
  memcpy(h->reserved + 48, &it->second.bytes, sizeof(size_t));
  return cudaSuccess;
}
API cudaError_t cudaIpcOpenMemHandle(void** out, cudaIpcMemHandle_t h, unsigned) {
  char name[49];
  memcpy(name, h.reserved, 48);
  name[48] = 0;
  size_t bytes = 0;
  memcpy(&bytes, h.reserved + 48, sizeof(size_t));
  const int fd = shm_open(name, O_RDWR, 0600);
  if (fd < 0) return fail(cudaErrorInvalidValue);
  void* p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (p == MAP_FAILED) return fail(cudaErrorMemoryAllocation);
  std::lock_guard<std::mutex> lk(g_mu);
  g_shm[p] = Shm{name, bytes, false};
  *out = p;
  return cudaSuccess;
}
API cudaError_t cudaIpcCloseMemHandle(void* p) { sim_free(p); return cudaSuccess; }

// ---- streams and events: everything has already happened -----------------------------------------
API cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) {
  *s = reinterpret_cast<cudaStream_t>(malloc(16));
  return cudaSuccess;
}
API cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, unsigned f, int) { return cudaStreamCreateWithFlags(s, f); }
API cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
API cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
API cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) {
  *e = reinterpret_cast<cudaEvent_t>(malloc(16));
  return cudaSuccess;
}
API cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
API cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
API cudaError_t cudaEventQuery(cudaEvent_t) { return cudaSuccess; }
API cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
