// device_utils.cuh -- device helpers shared by kernels.cu and norm_kernels.cu: 16-byte global
// accesses, flag loads/stores of the cross-GPU rendezvous, typed packets, the per-element
// arithmetic of the fused optimizers, and the work-entry lookup of the dense kernels.
#pragma once
#include "kernels.h"
#include "optim_math.h"
#include <cuda_fp16.h>
#include <cuda_bf16.h>
// MXKV_HOST_EMU (tests/sim/hostemu_tree.cc only): a kernel's own source compiled by g++ and run on the CPU -- the
// handful of PTX accesses below get plain C++ bodies, everything else in this file and in the kernel is the
// source the device executes.  Never defined in the product build.
#if defined(MXKV_HOST_EMU)
#include "host_emu.h"
#endif

namespace mxkv {

constexpr int kThreads = 512;

// ---------------------------------------------------------------------------
// memory helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint4 ld16(const void* p) {
#if defined(MXKV_HOST_EMU)
  return *static_cast<const uint4*>(hostemu::Aligned(p, 16));
#else
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
#endif
}
__device__ __forceinline__ void st16(void* p, const uint4& v) {
#if defined(MXKV_HOST_EMU)
  *static_cast<uint4*>(hostemu::Aligned(p, 16)) = v;
#else
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
#endif
}
__device__ __forceinline__ void st_flag_volatile(uint32_t* p, uint32_t v) {
#if defined(MXKV_HOST_EMU)
  __atomic_store_n(p, v, __ATOMIC_RELAXED);
#else
  asm volatile("st.volatile.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
#endif
}
__device__ __forceinline__ uint32_t ld_flag_volatile(const uint32_t* p) {
#if defined(MXKV_HOST_EMU)
  return hostemu::PoliteLoad(p, __ATOMIC_RELAXED);
#else
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
#endif
}
__device__ __forceinline__ void st_flag_release(uint32_t* p, uint32_t v) {
#if defined(MXKV_HOST_EMU)
  __atomic_store_n(p, v, __ATOMIC_RELEASE);
#else
  asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
#endif
}
__device__ __forceinline__ uint32_t ld_flag_acquire(const uint32_t* p) {
#if defined(MXKV_HOST_EMU)
  return hostemu::PoliteLoad(p, __ATOMIC_ACQUIRE);
#else
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
#endif
}

// ---------------------------------------------------------------------------
// cross-GPU rendezvous.  Block b of every rank pairs with block b of every other
// rank: thread i<world stores the block's next flag value into rank i's pad and
// spins on the slot rank i writes in ours.  Separate start/end slots so a fast
// rank's next start cannot overwrite a slow rank's pending end.
// ---------------------------------------------------------------------------
// A peer that never shows up (its launch failed, its process died) must not hang this GPU for
// ever: after `timeout` clock cycles the kernel traps and the host sees a CUDA error.
__device__ __forceinline__ void spin_check(long long t0, long long timeout) {
  if (timeout > 0 && clock64() - t0 > timeout) __trap();
}

__device__ __forceinline__ void barrier_start(const SyncArgs& s) {
  const uint32_t flag = s.epoch;
  if (threadIdx.x < s.world) {
    uint32_t* peer = s.peers[threadIdx.x] + kSigStartOff + blockIdx.x * kMaxRanks + s.rank;
    const uint32_t* mine = s.self + kSigStartOff + blockIdx.x * kMaxRanks + threadIdx.x;
    st_flag_volatile(peer, flag);
    const long long t0 = clock64();
    while (ld_flag_volatile(mine) != flag) spin_check(t0, s.timeout);
  }
  __syncthreads();
}

// release == true: this block stored into peer memory; make those stores visible
// system-wide before signalling (two-shot all-gather half).
__device__ __forceinline__ void barrier_end(const SyncArgs& s, bool release) {
  __syncthreads();
  const uint32_t flag = s.epoch;
  if (threadIdx.x < s.world) {
    uint32_t* peer = s.peers[threadIdx.x] + kSigEndOff + blockIdx.x * kMaxRanks + s.rank;
    const uint32_t* mine = s.self + kSigEndOff + blockIdx.x * kMaxRanks + threadIdx.x;
    const long long t0 = clock64();
    if (release) {
      st_flag_release(peer, flag);
      while (ld_flag_acquire(mine) != flag) spin_check(t0, s.timeout);
    } else {
      st_flag_volatile(peer, flag);
      while (ld_flag_volatile(mine) != flag) spin_check(t0, s.timeout);
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// Barrier over ALL blocks of the grid (the launcher sizes the grid to the resident capacity, so every block
// is on an SM) and, when `cross` and s.world > 1, over the grids of all ranks: blocks arrive on a counter in this GPU's
// signal pad; the last one to arrive exchanges an epoch with the other ranks (release / acquire at system
// scope: everything any block of any rank wrote before the barrier is visible to every block after it) and
// then opens the next generation for the blocks spinning locally.  Lets a kernel have phases that the
// reference (and round 1 of this engine) expressed as separate launches.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void grid_barrier(const SyncArgs& s, bool cross) {
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t* g = s.self + kSigGridOff;
    const uint32_t gen = ld_flag_volatile(g + kSigGridGen);
    __threadfence_system();                       // this block's writes, before it is counted
    const uint32_t arrived = atomicAdd(g + kSigGridCount, 1u);
    if (arrived == gridDim.x - 1) {
      g[kSigGridCount] = 0;
      if (cross && s.world > 1) {
        const uint32_t epoch = g[kSigGridEpoch] + 1;
        g[kSigGridEpoch] = epoch;
        const long long t0 = clock64();
        for (int q = 0; q < s.world; ++q)
          st_flag_release(s.peers[q] + kSigGridOff + kSigGridFlags + s.rank, epoch);
        for (int q = 0; q < s.world; ++q) {
          const uint32_t* mine = g + kSigGridFlags + q;
          // a fast rank may already have published its NEXT epoch: compare with >= (wrap-safe)
          while (static_cast<int32_t>(ld_flag_acquire(mine) - epoch) < 0) spin_check(t0, s.timeout);
        }
      }
      __threadfence_system();
      st_flag_release(g + kSigGridGen, gen + 1);
    } else {
      const long long t0 = clock64();
      // (relaxed polling -- hundreds of blocks spin here -- and one fence once the generation has moved)
      while (ld_flag_volatile(g + kSigGridGen) == gen) spin_check(t0, s.timeout);
      __threadfence_system();
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// packets: a 16-byte vector or a single element, exposed as N floats
// ---------------------------------------------------------------------------
template <typename T> struct Cvt;
template <> struct Cvt<float> {
  __device__ static __forceinline__ float to(float v) { return v; }
  __device__ static __forceinline__ float from(float v) { return v; }
};
template <> struct Cvt<__half> {
  __device__ static __forceinline__ float to(__half v) { return __half2float(v); }
  __device__ static __forceinline__ __half from(float v) { return __float2half_rn(v); }
};
template <> struct Cvt<__nv_bfloat16> {
  __device__ static __forceinline__ float to(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ static __forceinline__ __nv_bfloat16 from(float v) { return __float2bfloat16_rn(v); }
};
template <> struct Cvt<double> {          // multi_sum_sq squares float64 inputs in float (multi_sum_sq.cc:50)
  __device__ static __forceinline__ float to(double v) { return static_cast<float>(v); }
  __device__ static __forceinline__ double from(float v) { return static_cast<double>(v); }
};

__device__ __forceinline__ uint2 ld8(const void* p) {
#if defined(MXKV_HOST_EMU)
  return *static_cast<const uint2*>(hostemu::Aligned(p, 8));
#else
  uint2 v;
  asm volatile("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
#endif
}
__device__ __forceinline__ void st8(void* p, const uint2& v) {
#if defined(MXKV_HOST_EMU)
  *static_cast<uint2*>(hostemu::Aligned(p, 8)) = v;
#else
  asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" :: "l"(p), "r"(v.x), "r"(v.y) : "memory");
#endif
}

// Packet<T, N>: N consecutive elements (N*sizeof(T) in {16, 8} bytes, or N == 1)
template <typename T, int N, int BYTES = N * sizeof(T)> struct Packet;
template <typename T, int N_> struct Packet<T, N_, 16> {
  static constexpr int N = N_;
  uint4 raw;
  __device__ __forceinline__ void load(const void* base, int64_t elem) {
    raw = ld16(reinterpret_cast<const T*>(base) + elem);
  }
  __device__ __forceinline__ void unpack(float (&f)[N]) const {
    const T* t = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int i = 0; i < N; ++i) f[i] = Cvt<T>::to(t[i]);
  }
  __device__ static __forceinline__ void store(void* base, int64_t elem, const float (&f)[N]) {
    uint4 v;
    T* t = reinterpret_cast<T*>(&v);
#pragma unroll
    for (int i = 0; i < N; ++i) t[i] = Cvt<T>::from(f[i]);
    st16(reinterpret_cast<T*>(base) + elem, v);
  }
};
template <typename T, int N_> struct Packet<T, N_, 8> {
  static constexpr int N = N_;
  uint2 raw;
  __device__ __forceinline__ void load(const void* base, int64_t elem) {
    raw = ld8(reinterpret_cast<const T*>(base) + elem);
  }
  __device__ __forceinline__ void unpack(float (&f)[N]) const {
    const T* t = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int i = 0; i < N; ++i) f[i] = Cvt<T>::to(t[i]);
  }
  __device__ static __forceinline__ void store(void* base, int64_t elem, const float (&f)[N]) {
    uint2 v;
    T* t = reinterpret_cast<T*>(&v);
#pragma unroll
    for (int i = 0; i < N; ++i) t[i] = Cvt<T>::from(f[i]);
    st8(reinterpret_cast<T*>(base) + elem, v);
  }
};
template <typename T, int BYTES> struct Packet<T, 1, BYTES> {
  static constexpr int N = 1;
  T raw;
  __device__ __forceinline__ void load(const void* base, int64_t elem) {
    raw = reinterpret_cast<const T*>(base)[elem];
  }
  __device__ __forceinline__ void unpack(float (&f)[1]) const { f[0] = Cvt<T>::to(raw); }
  __device__ static __forceinline__ void store(void* base, int64_t elem, const float (&f)[1]) {
    reinterpret_cast<T*>(base)[elem] = Cvt<T>::from(f[0]);
  }
};

// fp32 packets for master weights / optimizer state (N floats, N in {1,4,8})
template <int N> __device__ __forceinline__ void ldf(const float* p, int64_t e, float (&f)[N]) {
  if (N == 1) {
    f[0] = p[e];
  } else {
#pragma unroll
    for (int i = 0; i < N; i += 4) {
      uint4 v = ld16(p + e + i);
      f[i] = __uint_as_float(v.x); f[i + 1] = __uint_as_float(v.y);
      f[i + 2] = __uint_as_float(v.z); f[i + 3] = __uint_as_float(v.w);
    }
  }
}
template <int N> __device__ __forceinline__ void stf(float* p, int64_t e, const float (&f)[N]) {
  if (N == 1) {
    p[e] = f[0];
  } else {
#pragma unroll
    for (int i = 0; i < N; i += 4) {
      uint4 v = make_uint4(__float_as_uint(f[i]), __float_as_uint(f[i + 1]),
                           __float_as_uint(f[i + 2]), __float_as_uint(f[i + 3]));
      st16(p + e + i, v);
    }
  }
}

// ---------------------------------------------------------------------------
// work entries of a dense launch
// ---------------------------------------------------------------------------
// chunk -> work entry (uniform across the block); the entry is staged in shared memory when it changes
__device__ __forceinline__ int find_work(const DenseLaunch& L, int64_t c, int* cur, TensorWork* tw) {
  int lo = 0, hi = L.nworks - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (L.chunk_prefix[mid] <= c) lo = mid; else hi = mid - 1;
  }
  if (lo != *cur) {
    __syncthreads();
    const uint4* src = reinterpret_cast<const uint4*>(L.works + lo);
    uint4* dst = reinterpret_cast<uint4*>(tw);
    for (int i = threadIdx.x; i < static_cast<int>(sizeof(TensorWork) / 16); i += blockDim.x) dst[i] = src[i];
    __syncthreads();
    *cur = lo;
  }
  return lo;
}

// the update's hyper-parameters for entry `idx`: lr / wd / eta are per key, the rest per launch.  Nadam's further
// per-key scalars come from the launch's side array (DenseLaunch::nadam); no other kind reads it
template <int OPT>
__device__ __forceinline__ Hyper make_hyper(const DenseLaunch& L, const TensorWork& tw, bool mp, int idx) {
  Hyper h;
  h.lr = tw.lr; h.wd = tw.wd; h.eta = tw.eta;
  h.rescale = L.rescale; h.clip = L.clip; h.momentum = L.momentum;
  h.beta1 = L.beta1; h.beta2 = L.beta2; h.eps = L.eps;
  h.rho = L.rho; h.clip_weights = L.clip_weights;
  h.wd_lh = L.wd_lh;
  h.mp = mp;
  if constexpr (OPT == OPT_NADAM) {
    const float4 s = L.nadam[idx];
    h.c1 = L.one_minus_beta1; h.c2 = L.one_minus_beta2;
    h.g_div = s.x; h.m_div = s.y; h.mom_t1 = s.z; h.c_mom_t = s.w;
  } else {
    (void)idx;
  }
  return h;
}

}  // namespace mxkv
