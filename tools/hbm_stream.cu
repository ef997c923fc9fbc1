// hbm_stream.cu -- the kernels of tools/hbm_stream.py: what one GPU can stream for the staged dense kernel's access
// pattern of three fp32 reads and three fp32 writes per element (g, w, mom in; stored w, mom, out of a fused
// SGD-momentum pushpull), set against the same bytes through plain per-thread vector loads, and against read-only and
// write-only streams.  Not part of the library: compiled by the probe into a temporary directory.
//
// Every kernel takes three input arrays a, b, c and three output arrays x, y, z of n floats (n a multiple of 4) and
// computes x = a + b, y = b + c, z = a + c: one add per output element, so arithmetic is never the limit.
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int kThreads = 256;
constexpr int kMaxStages = 8;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "W:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D;\n\tbra W;\n\tD:\n\t}"
      :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// The staged kernel's scheme: thread 0 requests the three input streams of a tile with cp.async.bulk into a ring of
// `stages` shared-memory buffers; every thread waits on the stage's mbarrier, computes out of shared memory and stores
// from registers.  EARLY = false releases the stage after the stores (one __syncthreads after them); EARLY = true
// copies the thread's operands of the tile into registers first, releases the stage, then computes and stores, so the
// next tile's loads are in flight during the stores.  Tiles are walked block-strided.
template <bool EARLY, int MAXV>
__global__ void __launch_bounds__(kThreads, 2)
hs_staged_kernel(const float* a, const float* b, const float* c, float* x, float* y, float* z, int64_t n, int tile,
                 int stages) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t full[kMaxStages];
  const uint32_t arr_bytes = static_cast<uint32_t>(tile) * 4u;
  const int64_t ntotal = (n + tile - 1) / tile;
  const int64_t ntiles = blockIdx.x < ntotal ? (ntotal - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) mbar_init(&full[s]);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int64_t i) {
    const int64_t cb = (blockIdx.x + i * gridDim.x) * static_cast<int64_t>(tile);
    const int64_t ce = cb + tile < n ? cb + tile : n;
    const uint32_t bytes = static_cast<uint32_t>(ce - cb) * 4u;
    const int s = static_cast<int>(i % stages);
    unsigned char* base = smem + static_cast<size_t>(s) * 3 * arr_bytes;
    mbar_expect_tx(&full[s], 3 * bytes);
    bulk_g2s(base, a + cb, bytes, &full[s]);
    bulk_g2s(base + arr_bytes, b + cb, bytes, &full[s]);
    bulk_g2s(base + 2 * arr_bytes, c + cb, bytes, &full[s]);
  };
  if (threadIdx.x == 0)
    for (int64_t i = 0; i < ntiles && i < stages; ++i) issue(i);
  for (int64_t i = 0; i < ntiles; ++i) {
    const int64_t cb = (blockIdx.x + i * gridDim.x) * static_cast<int64_t>(tile);
    const int64_t ce = cb + tile < n ? cb + tile : n;
    const int nvec = static_cast<int>((ce - cb) >> 2);
    const int s = static_cast<int>(i % stages);
    const float4* base = reinterpret_cast<const float4*>(smem + static_cast<size_t>(s) * 3 * arr_bytes);
    const int av = tile / 4;
    mbar_wait(&full[s], static_cast<uint32_t>((i / stages) & 1));
    if (EARLY) {
      float4 ra[MAXV], rb[MAXV], rc[MAXV];
#pragma unroll
      for (int u = 0; u < MAXV; ++u) {
        const int v = threadIdx.x + u * kThreads;
        if (v < nvec) { ra[u] = base[v]; rb[u] = base[av + v]; rc[u] = base[2 * av + v]; }
      }
      // the reads above must be performed before the bulk copy refills the stage (a write of the async proxy)
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();
      if (threadIdx.x == 0 && i + stages < ntiles) issue(i + stages);
#pragma unroll
      for (int u = 0; u < MAXV; ++u) {
        const int v = threadIdx.x + u * kThreads;
        if (v < nvec) {
          const int64_t e = cb / 4 + v;
          reinterpret_cast<float4*>(x)[e] = make_float4(ra[u].x + rb[u].x, ra[u].y + rb[u].y, ra[u].z + rb[u].z, ra[u].w + rb[u].w);
          reinterpret_cast<float4*>(y)[e] = make_float4(rb[u].x + rc[u].x, rb[u].y + rc[u].y, rb[u].z + rc[u].z, rb[u].w + rc[u].w);
          reinterpret_cast<float4*>(z)[e] = make_float4(ra[u].x + rc[u].x, ra[u].y + rc[u].y, ra[u].z + rc[u].z, ra[u].w + rc[u].w);
        }
      }
    } else {
      for (int v = threadIdx.x; v < nvec; v += kThreads) {
        const float4 ra = base[v], rb = base[av + v], rc = base[2 * av + v];
        const int64_t e = cb / 4 + v;
        reinterpret_cast<float4*>(x)[e] = make_float4(ra.x + rb.x, ra.y + rb.y, ra.z + rb.z, ra.w + rb.w);
        reinterpret_cast<float4*>(y)[e] = make_float4(rb.x + rc.x, rb.y + rc.y, rb.z + rc.z, rb.w + rc.w);
        reinterpret_cast<float4*>(z)[e] = make_float4(ra.x + rc.x, ra.y + rc.y, ra.z + rc.z, ra.w + rc.w);
      }
      __syncthreads();
      if (threadIdx.x == 0 && i + stages < ntiles) issue(i + stages);
    }
  }
}

// Plain grid-stride streaming: every thread issues U 16-byte loads of each input (3U requests in flight), then the U
// packets' stores.
template <int U>
__global__ void __launch_bounds__(kThreads)
hs_plain_kernel(const float4* a, const float4* b, const float4* c, float4* x, float4* y, float4* z, int64_t nv) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kThreads;
  for (int64_t v0 = blockIdx.x * static_cast<int64_t>(kThreads) + threadIdx.x; v0 < nv; v0 += stride * U) {
    float4 ra[U], rb[U], rc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t v = v0 + u * stride;
      if (v < nv) { ra[u] = a[v]; rb[u] = b[v]; rc[u] = c[v]; }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t v = v0 + u * stride;
      if (v < nv) {
        x[v] = make_float4(ra[u].x + rb[u].x, ra[u].y + rb[u].y, ra[u].z + rb[u].z, ra[u].w + rb[u].w);
        y[v] = make_float4(rb[u].x + rc[u].x, rb[u].y + rc[u].y, rb[u].z + rc[u].z, rb[u].w + rc[u].w);
        z[v] = make_float4(ra[u].x + rc[u].x, ra[u].y + rc[u].y, ra[u].z + rc[u].z, ra[u].w + rc[u].w);
      }
    }
  }
}

// Three reads, no writes: the sum of a packet is stored only when it equals a value the inputs never produce, so the
// loads cannot be dropped.
template <int U>
__global__ void __launch_bounds__(kThreads)
hs_read_kernel(const float4* a, const float4* b, const float4* c, float4* sink, int64_t nv) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kThreads;
  float acc = 0.f;
  for (int64_t v0 = blockIdx.x * static_cast<int64_t>(kThreads) + threadIdx.x; v0 < nv; v0 += stride * U) {
    float4 ra[U], rb[U], rc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t v = v0 + u * stride;
      if (v < nv) { ra[u] = a[v]; rb[u] = b[v]; rc[u] = c[v]; }
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (v0 + u * stride < nv) acc += ra[u].x + rb[u].y + rc[u].z + ra[u].w;
  }
  if (acc == -12345.f) sink[0] = make_float4(acc, acc, acc, acc);
}

// Three writes, no reads.
__global__ void __launch_bounds__(kThreads)
hs_write_kernel(float4* x, float4* y, float4* z, int64_t nv) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kThreads;
  const float4 k = make_float4(1.f, 2.f, 3.f, 4.f);
  for (int64_t v = blockIdx.x * static_cast<int64_t>(kThreads) + threadIdx.x; v < nv; v += stride) {
    x[v] = k; y[v] = k; z[v] = k;
  }
}

template <bool EARLY>
cudaError_t launch_staged(const float* a, const float* b, const float* c, float* x, float* y, float* z, int64_t n,
                          int tile, int stages, int grid, cudaStream_t s) {
  typedef void (*Fn)(const float*, const float*, const float*, float*, float*, float*, int64_t, int, int);
  Fn fn;
  switch (tile / (4 * kThreads)) {
    case 1: fn = hs_staged_kernel<EARLY, 1>; break;
    case 2: fn = hs_staged_kernel<EARLY, 2>; break;
    case 4: fn = hs_staged_kernel<EARLY, 4>; break;
    default: return cudaErrorInvalidValue;
  }
  if (stages < 1 || stages > kMaxStages) return cudaErrorInvalidValue;
  const int smem = stages * 3 * tile * 4;
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  fn<<<grid, kThreads, smem, s>>>(a, b, c, x, y, z, n, tile, stages);
  return cudaGetLastError();
}

}  // namespace

extern "C" {

// resident blocks per SM of the staged kernel at this tile / ring depth (0: does not fit)
int hs_staged_occupancy(int early, int tile, int stages) {
  const int smem = stages * 3 * tile * 4;
  const void* fn = nullptr;
  switch (tile / (4 * kThreads)) {
    case 1: fn = early ? (const void*)hs_staged_kernel<true, 1> : (const void*)hs_staged_kernel<false, 1>; break;
    case 2: fn = early ? (const void*)hs_staged_kernel<true, 2> : (const void*)hs_staged_kernel<false, 2>; break;
    case 4: fn = early ? (const void*)hs_staged_kernel<true, 4> : (const void*)hs_staged_kernel<false, 4>; break;
    default: return 0;
  }
  if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return 0;
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, kThreads, smem) != cudaSuccess) return 0;
  return occ;
}

int hs_staged(const float* a, const float* b, const float* c, float* x, float* y, float* z, long long n, int tile,
              int stages, int early, int grid, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return static_cast<int>(early ? launch_staged<true>(a, b, c, x, y, z, n, tile, stages, grid, s)
                                : launch_staged<false>(a, b, c, x, y, z, n, tile, stages, grid, s));
}

int hs_plain(const float* a, const float* b, const float* c, float* x, float* y, float* z, long long n, int unroll,
             int grid, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t nv = n / 4;
  const float4 *a4 = reinterpret_cast<const float4*>(a), *b4 = reinterpret_cast<const float4*>(b),
               *c4 = reinterpret_cast<const float4*>(c);
  float4 *x4 = reinterpret_cast<float4*>(x), *y4 = reinterpret_cast<float4*>(y), *z4 = reinterpret_cast<float4*>(z);
  switch (unroll) {
    case 1: hs_plain_kernel<1><<<grid, kThreads, 0, s>>>(a4, b4, c4, x4, y4, z4, nv); break;
    case 2: hs_plain_kernel<2><<<grid, kThreads, 0, s>>>(a4, b4, c4, x4, y4, z4, nv); break;
    case 4: hs_plain_kernel<4><<<grid, kThreads, 0, s>>>(a4, b4, c4, x4, y4, z4, nv); break;
    default: return static_cast<int>(cudaErrorInvalidValue);
  }
  return static_cast<int>(cudaGetLastError());
}

int hs_read(const float* a, const float* b, const float* c, float* sink, long long n, int grid, void* stream) {
  hs_read_kernel<4><<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(a), reinterpret_cast<const float4*>(b), reinterpret_cast<const float4*>(c),
      reinterpret_cast<float4*>(sink), n / 4);
  return static_cast<int>(cudaGetLastError());
}

int hs_write(float* x, float* y, float* z, long long n, int grid, void* stream) {
  hs_write_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<float4*>(x), reinterpret_cast<float4*>(y), reinterpret_cast<float4*>(z), n / 4);
  return static_cast<int>(cudaGetLastError());
}

}  // extern "C"
