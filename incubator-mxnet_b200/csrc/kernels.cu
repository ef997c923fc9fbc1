// kernels.cu -- sm_90a kernels of the KVStore gradient path.
//
// kv_dense_kernel: ONE kernel does what the reference spreads over
//   n x CopyFromTo (cudaMemcpyPeerAsync, src/ndarray/ndarray_function.cu:68-99)
//   + ElementwiseSum (src/ndarray/ndarray_function-inl.h:443-489)
//   + the Python updater -> sgd_update / sgd_mom_update / mp_sgd_* / adam_update /
//     _mp_adamw_update (src/operator/optimizer_op-inl.h, contrib/adamw-inl.h)
//   + n x CopyFromTo broadcast (src/kvstore/comm.h:607-625):
// every thread streams 16-byte vectors of the n gradient replicas straight from
// the GPUs that own them (NVLink peer loads), sums them in the reference's
// association order in fp32, applies the optimizer on the fp32 master and writes
// the new weight to every destination replica (local or peer stores).  Ranks
// rendezvous through flag words in peer-mapped signal pads; no host round trip,
// no intermediate buffer, no second pass over HBM.
//
// Arithmetic uses __fmul_rn/__fadd_rn/... so ptxas cannot contract a*b+c into an
// FMA: results are bit-identical to the CPU oracle (oracle/kv_oracle.c), which
// restates the reference source operation by operation.
#include "kernels.h"
#include "rsp_kernels.h"
#include "device_utils.cuh"
#include <cstdio>
#include <cstdlib>

namespace mxkv {

#if !defined(MXKV_HOST_EMU)
static int sm_count(int device);
#endif

// ---------------------------------------------------------------------------
// U packets per thread: gather n sources, sum in order, update, scatter.  All loads of a batch are
// issued before the first use so U * min(n, BATCH) 16-byte requests per thread are in flight
// (NVLink round trips are ~2 us: bytes in flight are what buys bandwidth).
// ---------------------------------------------------------------------------
template <typename T, int OPT, bool MP, int N, int BATCH, int U>
__device__ __forceinline__ void process_packets(const TensorWork& tw, const int64_t (&e)[U], const bool (&ok)[U],
                                                const Hyper& h, int order, bool native_half_add) {
  typedef Packet<T, N> P;
  float acc[U][N];
  // the CommCPU grouping only differs from left-to-right for n >= 3, i.e. never when BATCH == 2
  // (the small-n variant): no group registers there
  float grp[BATCH > 2 ? U : 1][N];
  const int n = tw.n_src;
  for (int k0 = 0; k0 < n; k0 += BATCH) {
    P buf[U][BATCH];
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
      for (int j = 0; j < BATCH; ++j)
        if (ok[u] && k0 + j < n) buf[u][j].load(tw.src[k0 + j], e[u]);
#pragma unroll
    for (int j = 0; j < BATCH; ++j) {
      const int k = k0 + j;
      if (k < n) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          float x[N];
          buf[u][j].unpack(x);
          if (k == 0) {
#pragma unroll
            for (int i = 0; i < N; ++i) acc[u][i] = x[i];
          } else if (order == ORDER_DEVICE || BATCH <= 2) {
#pragma unroll
            for (int i = 0; i < N; ++i) {
              float s = __fadd_rn(acc[u][i], x[i]);
              if (native_half_add) s = Cvt<T>::to(Cvt<T>::from(s));
              acc[u][i] = s;
            }
          } else {  // ORDER_COMMCPU: in0 += ((in1+in2)+in3)+in4 per group of four
            const int pos = (k - 1) & 3;
            constexpr int GU = BATCH > 2 ? 1 : 0;
#pragma unroll
            for (int i = 0; i < N; ++i) grp[u * GU][i] = (pos == 0) ? x[i] : __fadd_rn(grp[u * GU][i], x[i]);
            if (pos == 3 || k == n - 1) {
#pragma unroll
              for (int i = 0; i < N; ++i) acc[u][i] = __fadd_rn(acc[u][i], grp[u * GU][i]);
            }
          }
        }
      }
    }
  }

  float wnew[U][N];
  if (OPT == OPT_NONE) {
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
      for (int i = 0; i < N; ++i) wnew[u][i] = acc[u][i];
  } else {
    float w[U][N], s0[U][N], s1[U][N];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!ok[u]) continue;
      if (MP) {
        ldf<N>(tw.w32, e[u], w[u]);
      } else {
        P pw;
        pw.load(tw.w, e[u]);
        pw.unpack(w[u]);
      }
      if (OPT == OPT_SGD_MOM || OPT == OPT_ADAM || OPT == OPT_ADAMW || OPT == OPT_ADAM_STD) ldf<N>(tw.s0, e[u], s0[u]);
      if (OPT == OPT_ADAM || OPT == OPT_ADAMW || OPT == OPT_ADAM_STD) ldf<N>(tw.s1, e[u], s1[u]);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!ok[u]) continue;
#pragma unroll
      for (int i = 0; i < N; ++i) wnew[u][i] = update_one<OPT>(acc[u][i], w[u][i], s0[u][i], s1[u][i], h);
      if (OPT == OPT_SGD_MOM || OPT == OPT_ADAM || OPT == OPT_ADAMW || OPT == OPT_ADAM_STD) stf<N>(tw.s0, e[u], s0[u]);
      if (OPT == OPT_ADAM || OPT == OPT_ADAMW || OPT == OPT_ADAM_STD) stf<N>(tw.s1, e[u], s1[u]);
      if (MP) stf<N>(tw.w32, e[u], wnew[u]);
    }
  }
  const int m = tw.n_out;
#pragma unroll
  for (int u = 0; u < U; ++u) {
    if (!ok[u]) continue;
    for (int j = 0; j < m; ++j) P::store(tw.out[j], e[u], wnew[u]);
  }
}

template <typename T, int OPT, bool MP, bool SMALLN>
__global__ void __launch_bounds__(kThreads, 2)
kv_dense_kernel(DenseLaunch L) {
  __shared__ TensorWork tw;
  const bool sync = L.sync.mode != SYNC_NONE;
  if (sync) barrier_start(L.sync);

  // 16-bit gradients with fp32 master/state: 4-element packets (8 B of gradient against
  // 16 B of every fp32 stream) keep the kernel inside 64 registers.
  constexpr int NV = (OPT != OPT_NONE && sizeof(T) == 2) ? 4 : 16 / sizeof(T);
  constexpr int BATCH = SMALLN ? 2 : 4;
  constexpr int U = SMALLN ? 2 : 1;
  const bool native_half_add = (sizeof(T) == 2) && !L.fp32_accum && (OPT == OPT_NONE);
  int cur = -1;
  for (int64_t c = blockIdx.x; c < L.total_chunks; c += gridDim.x) {
    // chunk -> work entry (uniform across the block)
    int lo = 0, hi = L.nworks - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (L.chunk_prefix[mid] <= c) lo = mid; else hi = mid - 1;
    }
    if (lo != cur) {
      __syncthreads();
      const uint4* src = reinterpret_cast<const uint4*>(L.works + lo);
      uint4* dst = reinterpret_cast<uint4*>(&tw);
      for (int i = threadIdx.x; i < static_cast<int>(sizeof(TensorWork) / 16); i += blockDim.x)
        dst[i] = src[i];
      __syncthreads();
      cur = lo;
    }
    Hyper h;
    h.lr = tw.lr; h.wd = tw.wd; h.eta = tw.eta;
    h.rescale = L.rescale; h.clip = L.clip; h.momentum = L.momentum;
    h.beta1 = L.beta1; h.beta2 = L.beta2; h.eps = L.eps;

    const int64_t cb = tw.begin + (c - L.chunk_prefix[lo]) * L.chunk_elems;
    const int64_t ce = (cb + L.chunk_elems < tw.end) ? cb + L.chunk_elems : tw.end;
    int64_t scalar_from = cb;
    if (tw.pad_ & 1) {  // every pointer 16-byte aligned and begin % 8 == 0
      const int64_t nvec = (ce - cb) / NV;
      const int64_t nthr = blockDim.x;
      for (int64_t v = threadIdx.x; v < nvec; v += static_cast<int64_t>(U) * nthr) {
        int64_t e[U];
        bool ok[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t vv = v + static_cast<int64_t>(u) * nthr;
          ok[u] = vv < nvec;
          e[u] = cb + (ok[u] ? vv : v) * NV;
        }
        process_packets<T, OPT, MP, NV, BATCH, U>(tw, e, ok, h, L.order, native_half_add);
      }
      scalar_from = cb + nvec * NV;
    }
    for (int64_t s = scalar_from + threadIdx.x; s < ce; s += blockDim.x) {
      const int64_t e1[1] = {s};
      const bool ok1[1] = {true};
      process_packets<T, OPT, MP, 1, 4, 1>(tw, e1, ok1, h, L.order, native_half_add);
    }
  }

  if (sync) barrier_end(L.sync, L.sync.mode == SYNC_WRITE_PEERS);
}

// ---------------------------------------------------------------------------
// Shared-memory staged variant (float32): a bulk-copy engine pipeline instead of per-thread loads.
// One elected thread issues cp.async.bulk (the 1-D TMA path, SASS UBLKCP) for every input stream of
// a tile -- the n gradient replicas (local HBM or NVLink peers), the weight and the optimizer state
// -- into a ring of `stages` shared-memory buffers, arming an mbarrier with the byte count; all
// threads wait on the barrier, compute the tile out of shared memory and store results straight
// from registers.  Bytes in flight per SM are bounded by shared memory (up to ~200 KB) instead of by
// registers (48 KB for the per-thread variant), which is what a latency-bound stream needs.
// ---------------------------------------------------------------------------
constexpr int kBulkThreads = 256;
constexpr int kBulkMaxStages = 8;

#if defined(MXKV_HOST_EMU)     // tests/sim/host_emu.h: the same protocol on a CPU (phase, byte count, parity wait)
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t) { hostemu::MbarInit(bar); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { hostemu::MbarExpectTx(bar, bytes); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) { hostemu::MbarWait(bar, parity); }
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  hostemu::BulkCopy(dst_smem, src_gmem, bytes, bar);
}
#else
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

#endif

template <int OPT, bool MP>
__global__ void __launch_bounds__(kBulkThreads, 2)
kv_dense_bulk_kernel(DenseLaunch L) {
#if defined(MXKV_HOST_EMU)
  unsigned char* const bulk_smem = hostemu::DynamicSmem();
#else
  extern __shared__ __align__(128) unsigned char bulk_smem[];
#endif
  __shared__ TensorWork tw;        // descriptor of the tile being computed (all threads)
  __shared__ TensorWork twp;       // descriptor of the tile being requested (thread 0 only)
  __shared__ __align__(8) uint64_t full[kBulkMaxStages];
  int p_cur = -1;
  const bool sync = L.sync.mode != SYNC_NONE;
  const int stages = L.bulk_stages;
  const int tile = L.chunk_elems;
  const uint32_t arr_bytes = static_cast<uint32_t>(tile) * 4u;
  const uint32_t stage_bytes = arr_bytes * static_cast<uint32_t>(L.bulk_arrays);
  constexpr bool HAS_W = OPT != OPT_NONE;
  constexpr bool HAS_S0 = OPT == OPT_SGD_MOM || OPT == OPT_ADAM || OPT == OPT_ADAMW;
  constexpr bool HAS_S1 = OPT == OPT_ADAM || OPT == OPT_ADAMW;

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) mbar_init(&full[s], 1);
#if !defined(MXKV_HOST_EMU)
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
  }
  __syncthreads();
  if (sync) barrier_start(L.sync);     // no peer byte may be requested before the rendezvous

  // tiles of this block: groups of G consecutive tiles, block-cyclic -- tile(i) = ((i / G) * grid + block) * G + i % G.
  // G = 1 is the plain strided walk: all blocks stream through one narrow window of every array (best for DRAM on
  // large keys) but every block meets every key of the work list and reloads a 400-byte descriptor each time, which
  // costs a large share of the kernel on a model of hundreds of small keys (BERT-base).  A contiguous range per
  // block has the opposite profile.  Small groups keep the window narrow and divide the descriptor switches by G
  // (MXKV_B200_BULK_GROUP); the host groups only work lists of many keys (kvstore.cc: LaunchWorks) and keeps G = 1
  // for the rest.
  const int64_t G = L.bulk_group > 0 ? L.bulk_group : 1;
  int64_t ntiles;
  if (G == 1) {             // the plain strided walk, without the divisions of the grouped one
    ntiles = static_cast<int64_t>(blockIdx.x) < L.total_chunks ? (L.total_chunks - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  } else {
    const int64_t ngroups = (L.total_chunks + G - 1) / G;
    const int64_t my_groups = static_cast<int64_t>(blockIdx.x) < ngroups ? (ngroups - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    ntiles = my_groups * G;
    if (my_groups > 0) {      // the very last group of the list may be short
      const int64_t last_group = blockIdx.x + (my_groups - 1) * gridDim.x;
      if (last_group == ngroups - 1) ntiles -= ngroups * G - L.total_chunks;
    }
  }
  auto tile_of = [&](int64_t i) -> int64_t {
    return G == 1 ? blockIdx.x + i * gridDim.x : ((i / G) * gridDim.x + blockIdx.x) * G + i % G;
  };
  auto issue = [&](int64_t i) {       // thread 0 only: request every input stream of tile i
    const int64_t c = tile_of(i);
    int lo = 0, hi = L.nworks - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (L.chunk_prefix[mid] <= c) lo = mid; else hi = mid - 1;
    }
    if (lo != p_cur) {               // descriptor changes once per key: keep a private copy
      const uint4* src = reinterpret_cast<const uint4*>(L.works + lo);
      uint4* dst = reinterpret_cast<uint4*>(&twp);
      for (int t = 0; t < static_cast<int>(sizeof(TensorWork) / 16); ++t) dst[t] = src[t];
      p_cur = lo;
    }
    const TensorWork* w = &twp;
    const int64_t cb = w->begin + (c - L.chunk_prefix[lo]) * tile;
    const int64_t ce = (cb + tile < w->end) ? cb + tile : w->end;
    const uint32_t bytes = static_cast<uint32_t>(ce - cb) * 4u;
    const int n = w->n_src;
    const int narr = n + (HAS_W ? 1 : 0) + (HAS_S0 ? 1 : 0) + (HAS_S1 ? 1 : 0);
    const int s = static_cast<int>(i % stages);
    unsigned char* base = bulk_smem + static_cast<size_t>(s) * stage_bytes;
    mbar_expect_tx(&full[s], bytes * static_cast<uint32_t>(narr));
    int a = 0;
    for (int k = 0; k < n; ++k, ++a)
      bulk_g2s(base + static_cast<size_t>(a) * arr_bytes, static_cast<const float*>(w->src[k]) + cb, bytes, &full[s]);
    if (HAS_W) {
      const float* wp = MP ? w->w32 : static_cast<const float*>(w->w);
      bulk_g2s(base + static_cast<size_t>(a) * arr_bytes, wp + cb, bytes, &full[s]); ++a;
    }
    if (HAS_S0) { bulk_g2s(base + static_cast<size_t>(a) * arr_bytes, w->s0 + cb, bytes, &full[s]); ++a; }
    if (HAS_S1) { bulk_g2s(base + static_cast<size_t>(a) * arr_bytes, w->s1 + cb, bytes, &full[s]); ++a; }
  };

  if (threadIdx.x == 0) {
    for (int64_t i = 0; i < ntiles && i < stages; ++i) issue(i);
  }

  int cur = -1;
  for (int64_t i = 0; i < ntiles; ++i) {
    const int64_t c = tile_of(i);
    int lo = 0, hi = L.nworks - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (L.chunk_prefix[mid] <= c) lo = mid; else hi = mid - 1;
    }
    if (lo != cur) {
      __syncthreads();
      const uint4* src = reinterpret_cast<const uint4*>(L.works + lo);
      uint4* dst = reinterpret_cast<uint4*>(&tw);
      for (int t = threadIdx.x; t < static_cast<int>(sizeof(TensorWork) / 16); t += blockDim.x) dst[t] = src[t];
      __syncthreads();
      cur = lo;
    }
    Hyper h;
    h.lr = tw.lr; h.wd = tw.wd; h.eta = tw.eta;
    h.rescale = L.rescale; h.clip = L.clip; h.momentum = L.momentum;
    h.beta1 = L.beta1; h.beta2 = L.beta2; h.eps = L.eps;
    const int64_t cb = tw.begin + (c - L.chunk_prefix[lo]) * tile;
    const int64_t ce = (cb + tile < tw.end) ? cb + tile : tw.end;
    const int nvec = static_cast<int>((ce - cb) >> 2);
    const int n = tw.n_src;
    const int s = static_cast<int>(i % stages);
    const uint32_t parity = static_cast<uint32_t>((i / stages) & 1);
    const unsigned char* base = bulk_smem + static_cast<size_t>(s) * stage_bytes;
    mbar_wait(&full[s], parity);

    for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
      float acc[4], grp[4];
      for (int k = 0; k < n; ++k) {
        const float4 x4 = reinterpret_cast<const float4*>(base + static_cast<size_t>(k) * arr_bytes)[v];
        const float x[4] = {x4.x, x4.y, x4.z, x4.w};
        if (k == 0) {
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[j] = x[j];
        } else if (L.order == ORDER_DEVICE) {
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[j] = __fadd_rn(acc[j], x[j]);
        } else {
          const int pos = (k - 1) & 3;
#pragma unroll
          for (int j = 0; j < 4; ++j) grp[j] = (pos == 0) ? x[j] : __fadd_rn(grp[j], x[j]);
          if (pos == 3 || k == n - 1) {
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[j] = __fadd_rn(acc[j], grp[j]);
          }
        }
      }
      float wnew[4];
      const int64_t e = cb + static_cast<int64_t>(v) * 4;
      if (OPT == OPT_NONE) {
#pragma unroll
        for (int j = 0; j < 4; ++j) wnew[j] = acc[j];
      } else {
        int a = n;
        const float4 w4 = reinterpret_cast<const float4*>(base + static_cast<size_t>(a) * arr_bytes)[v]; ++a;
        float w[4] = {w4.x, w4.y, w4.z, w4.w};
        float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
        if (HAS_S0) {
          const float4 t4 = reinterpret_cast<const float4*>(base + static_cast<size_t>(a) * arr_bytes)[v]; ++a;
          s0[0] = t4.x; s0[1] = t4.y; s0[2] = t4.z; s0[3] = t4.w;
        }
        if (HAS_S1) {
          const float4 t4 = reinterpret_cast<const float4*>(base + static_cast<size_t>(a) * arr_bytes)[v]; ++a;
          s1[0] = t4.x; s1[1] = t4.y; s1[2] = t4.z; s1[3] = t4.w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) wnew[j] = update_one<OPT>(acc[j], w[j], s0[j], s1[j], h);
        if (HAS_S0) stf<4>(tw.s0, e, s0);
        if (HAS_S1) stf<4>(tw.s1, e, s1);
        if (MP) stf<4>(tw.w32, e, wnew);
      }
      const int m = tw.n_out;
      for (int j = 0; j < m; ++j) stf<4>(static_cast<float*>(tw.out[j]), e, wnew);
    }
    __syncthreads();                  // every thread is done reading stage s
    if (threadIdx.x == 0 && i + stages < ntiles) issue(i + stages);
  }

  if (sync) barrier_end(L.sync, L.sync.mode == SYNC_WRITE_PEERS);
}

typedef void (*BulkKernelFn)(DenseLaunch);
static BulkKernelFn pick_bulk(int opt, int mp) {
  switch (opt) {
    case OPT_NONE: return kv_dense_bulk_kernel<OPT_NONE, false>;
    case OPT_SGD: return mp ? kv_dense_bulk_kernel<OPT_SGD, true> : kv_dense_bulk_kernel<OPT_SGD, false>;
    case OPT_SGD_MOM: return mp ? kv_dense_bulk_kernel<OPT_SGD_MOM, true> : kv_dense_bulk_kernel<OPT_SGD_MOM, false>;
    case OPT_ADAM: return mp ? kv_dense_bulk_kernel<OPT_ADAM, true> : kv_dense_bulk_kernel<OPT_ADAM, false>;
    case OPT_ADAMW: return mp ? kv_dense_bulk_kernel<OPT_ADAMW, true> : kv_dense_bulk_kernel<OPT_ADAMW, false>;
    case OPT_TEST: return mp ? kv_dense_bulk_kernel<OPT_TEST, true> : kv_dense_bulk_kernel<OPT_TEST, false>;
    default: return nullptr;
  }
}

// ---------------------------------------------------------------------------
// NVLS variant (float32, one process per GPU, arrays bound to an NVSwitch multicast object):
// the reduce-scatter half is ONE multimem.ld_reduce per 16 bytes -- the switch adds the n replicas
// and returns the sum, so a GPU receives S/n instead of S(n-1)/n -- and the all-gather half is ONE
// multimem.st per 16 bytes that the switch replicates into every GPU's copy.  The optimizer runs in
// between on the shard this rank owns, exactly as in the peer-load variants.  The switch's
// summation order is not the reference's left-to-right order: results agree with the oracle to
// fp32 rounding (<= 1e-6 relative, the reference's own bound), not bit for bit, and every replica
// receives identical bits (each shard is produced by exactly one rank).
// ---------------------------------------------------------------------------
__device__ __forceinline__ float4 mm_ld_reduce(const void* p) {
#if defined(MXKV_HOST_EMU)     // tests/sim: the n copies behind a multicast address, added on the CPU
  return hostemu::MultimemLoadReduce(p);
#else
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
#endif
}
__device__ __forceinline__ void mm_st(void* p, const float4& v) {
#if defined(MXKV_HOST_EMU)
  hostemu::MultimemStore(p, v);
#else
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
#endif
}

// One scheduling chunk = ONE block iteration (blockDim * U 16-byte vectors), so `chunk c -> block c % grid`
// is an exactly balanced grid-stride walk over the concatenated shards of the whole work list.
//   U     multimem.ld_reduce requests (16 B each) a thread has in flight per iteration
//   PIPE  software pipeline: the ld_reduce requests of the block's NEXT chunk are issued before the current
//         chunk's state loads / update / multimem.st, so the reduce-scatter half never idles behind the
//         all-gather half (the two halves use opposite link directions)
// The SM side is never the limiter here (a GPU consumes ~80 GB/s of reduced data, i.e. < 1 KB/us per SM): what
// these knobs and the grid size change is the REQUEST PATTERN the switch sees (how many reduce requests queue
// in the fabric, how they interleave with the multicast stores).  tools/tune_nvls.py sweeps them.
struct NvlsChunk {
  const float* g;      // multicast address of the key's gradient
  int64_t cb, ce;      // element range of the chunk
  int lo;              // work entry
};

__device__ __forceinline__ NvlsChunk nvls_lookup(const DenseLaunch& L, int64_t c) {
  int lo = 0, hi = L.nworks - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (static_cast<int64_t>(__ldg(reinterpret_cast<const long long*>(L.chunk_prefix + mid))) <= c) lo = mid; else hi = mid - 1;
  }
  const TensorWork* w = L.works + lo;
  NvlsChunk k;
  k.lo = lo;
  k.g = reinterpret_cast<const float*>(__ldg(reinterpret_cast<const unsigned long long*>(&w->src[0])));
  const int64_t begin = static_cast<int64_t>(__ldg(reinterpret_cast<const long long*>(&w->begin)));
  const int64_t end = static_cast<int64_t>(__ldg(reinterpret_cast<const long long*>(&w->end)));
  k.cb = begin + (c - static_cast<int64_t>(__ldg(reinterpret_cast<const long long*>(L.chunk_prefix + lo)))) * L.chunk_elems;
  k.ce = (k.cb + L.chunk_elems < end) ? k.cb + L.chunk_elems : end;
  return k;
}

template <int U>
__device__ __forceinline__ void nvls_issue(const NvlsChunk& k, float4 (&g)[U]) {
  const int64_t nvec = (k.ce - k.cb) >> 2;           // host guarantees multiples of 4 elements
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int64_t vv = threadIdx.x + static_cast<int64_t>(u) * blockDim.x;
    if (vv < nvec) g[u] = mm_ld_reduce(k.g + k.cb + vv * 4);
  }
}

template <int OPT, bool MP, int U, bool PIPE>
__global__ void __launch_bounds__(kThreads, (U >= 4 || PIPE) ? 1 : 2)
kv_dense_nvls_kernel(DenseLaunch L) {
  __shared__ TensorWork tw;
  barrier_start(L.sync);
  constexpr bool HAS_S0 = OPT == OPT_SGD_MOM || OPT == OPT_ADAM || OPT == OPT_ADAMW;
  constexpr bool HAS_S1 = OPT == OPT_ADAM || OPT == OPT_ADAMW;
  int cur = -1;
  int64_t c = blockIdx.x;
  NvlsChunk k, kn;
  float4 g[U], gn[U];
  if (c < L.total_chunks) {
    k = nvls_lookup(L, c);
    if (PIPE) nvls_issue<U>(k, g);
  }
  while (c < L.total_chunks) {
    const int64_t cn = c + gridDim.x;
    if (cn < L.total_chunks) {
      kn = nvls_lookup(L, cn);
      if (PIPE) nvls_issue<U>(kn, gn);
    }
    if (!PIPE) nvls_issue<U>(k, g);
    if (k.lo != cur) {
      __syncthreads();
      const uint4* src = reinterpret_cast<const uint4*>(L.works + k.lo);
      uint4* dst = reinterpret_cast<uint4*>(&tw);
      for (int i = threadIdx.x; i < static_cast<int>(sizeof(TensorWork) / 16); i += blockDim.x) dst[i] = src[i];
      __syncthreads();
      cur = k.lo;
    }
    Hyper h;
    h.lr = tw.lr; h.wd = tw.wd; h.eta = tw.eta;
    h.rescale = L.rescale; h.clip = L.clip; h.momentum = L.momentum;
    h.beta1 = L.beta1; h.beta2 = L.beta2; h.eps = L.eps;
    const int64_t nvec = (k.ce - k.cb) >> 2;
    const int n_plain = tw.n_out - tw.n_mc;
    // state of all U packets first (independent HBM loads in flight together), then the arithmetic
    float w[U][4], s0[U][4], s1[U][4];
    if (OPT != OPT_NONE) {
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t vv = threadIdx.x + static_cast<int64_t>(u) * blockDim.x;
        if (vv >= nvec) continue;
        const int64_t e = k.cb + vv * 4;
        ldf<4>(MP ? tw.w32 : static_cast<const float*>(tw.w), e, w[u]);
        if (HAS_S0) ldf<4>(tw.s0, e, s0[u]);
        if (HAS_S1) ldf<4>(tw.s1, e, s1[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t vv = threadIdx.x + static_cast<int64_t>(u) * blockDim.x;
      if (vv >= nvec) continue;
      const int64_t e = k.cb + vv * 4;
      const float acc[4] = {g[u].x, g[u].y, g[u].z, g[u].w};
      float wnew[4];
      if (OPT == OPT_NONE) {
#pragma unroll
        for (int j = 0; j < 4; ++j) wnew[j] = acc[j];
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) wnew[j] = update_one<OPT>(acc[j], w[u][j], s0[u][j], s1[u][j], h);
        if (HAS_S0) stf<4>(tw.s0, e, s0[u]);
        if (HAS_S1) stf<4>(tw.s1, e, s1[u]);
        if (MP) stf<4>(tw.w32, e, wnew);
      }
      for (int j = 0; j < n_plain; ++j) stf<4>(static_cast<float*>(tw.out[j]), e, wnew);
      const float4 o = make_float4(wnew[0], wnew[1], wnew[2], wnew[3]);
      for (int j = n_plain; j < tw.n_out; ++j) mm_st(static_cast<float*>(tw.out[j]) + e, o);
    }
    c = cn;
    k = kn;
    if (PIPE) {
#pragma unroll
      for (int u = 0; u < U; ++u) g[u] = gn[u];
    }
  }
  barrier_end(L.sync, true);
}

typedef void (*NvlsKernelFn)(DenseLaunch);

template <int U, bool PIPE>
static NvlsKernelFn pick_nvls_opt(int opt, int mp) {
  switch (opt) {
    case OPT_NONE: return kv_dense_nvls_kernel<OPT_NONE, false, U, PIPE>;
    case OPT_SGD: return mp ? kv_dense_nvls_kernel<OPT_SGD, true, U, PIPE> : kv_dense_nvls_kernel<OPT_SGD, false, U, PIPE>;
    case OPT_SGD_MOM: return mp ? kv_dense_nvls_kernel<OPT_SGD_MOM, true, U, PIPE> : kv_dense_nvls_kernel<OPT_SGD_MOM, false, U, PIPE>;
    case OPT_ADAM: return mp ? kv_dense_nvls_kernel<OPT_ADAM, true, U, PIPE> : kv_dense_nvls_kernel<OPT_ADAM, false, U, PIPE>;
    case OPT_ADAMW: return mp ? kv_dense_nvls_kernel<OPT_ADAMW, true, U, PIPE> : kv_dense_nvls_kernel<OPT_ADAMW, false, U, PIPE>;
    case OPT_TEST: return mp ? kv_dense_nvls_kernel<OPT_TEST, true, U, PIPE> : kv_dense_nvls_kernel<OPT_TEST, false, U, PIPE>;
    default: return nullptr;
  }
}

// the instantiated (U, PIPE) points; anything else is rounded down to the nearest one
// (Adam / AdamW carry three state packets per gradient packet: 8 requests would spill at 128 registers)
static int nvls_round_unroll(int unroll, int opt) {
  if ((opt == OPT_ADAM || opt == OPT_ADAMW) && unroll > 4) unroll = 4;
  return unroll >= 8 ? 8 : (unroll >= 4 ? 4 : (unroll >= 2 ? 2 : 1));
}

static NvlsKernelFn pick_nvls(int opt, int mp, int unroll, int pipe) {
  switch (nvls_round_unroll(unroll, opt)) {
    case 8: return pipe ? pick_nvls_opt<8, true>(opt, mp) : pick_nvls_opt<8, false>(opt, mp);
    case 4: return pipe ? pick_nvls_opt<4, true>(opt, mp) : pick_nvls_opt<4, false>(opt, mp);
    case 2: return pipe ? pick_nvls_opt<2, true>(opt, mp) : pick_nvls_opt<2, false>(opt, mp);
    default: return pipe ? pick_nvls_opt<1, true>(opt, mp) : pick_nvls_opt<1, false>(opt, mp);
  }
}

#if !defined(MXKV_HOST_EMU)
int NvlsPlan(int device, int opt, int multi_precision, int unroll, int pipe, int threads, int* chunk_elems) {
  NvlsKernelFn fn = pick_nvls(opt, multi_precision, unroll, pipe);
  if (fn == nullptr) return 0;
  if (threads != 128 && threads != 256 && threads != 512) threads = kThreads;
  int prev = -1;
  cudaGetDevice(&prev);
  if (prev != device) cudaSetDevice(device);
  int occ = 0;
  const bool ok = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, threads, 0) == cudaSuccess && occ >= 1;
  if (!ok) cudaGetLastError();
  if (prev >= 0 && prev != device) cudaSetDevice(prev);
  if (!ok) return 0;
  *chunk_elems = threads * nvls_round_unroll(unroll, opt) * 4;
  const int g = occ * sm_count(device);
  return g > kMaxBlocks ? kMaxBlocks : g;
}
#endif

// ---------------------------------------------------------------------------
// plain typed sum for the dtypes the reference's ElementwiseSum also accepts
// (MSHADOW_TYPE_SWITCH: f64, u8, i32, i8, i64); native arithmetic, device order.
// ---------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads, 2)
kv_sum_typed_kernel(DenseLaunch L) {
  __shared__ TensorWork tw;
  const bool sync = L.sync.mode != SYNC_NONE;
  if (sync) barrier_start(L.sync);
  int cur = -1;
  for (int64_t c = blockIdx.x; c < L.total_chunks; c += gridDim.x) {
    int lo = 0, hi = L.nworks - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (L.chunk_prefix[mid] <= c) lo = mid; else hi = mid - 1;
    }
    if (lo != cur) {
      __syncthreads();
      const uint4* src = reinterpret_cast<const uint4*>(L.works + lo);
      uint4* dst = reinterpret_cast<uint4*>(&tw);
      for (int i = threadIdx.x; i < static_cast<int>(sizeof(TensorWork) / 16); i += blockDim.x)
        dst[i] = src[i];
      __syncthreads();
      cur = lo;
    }
    const int64_t cb = tw.begin + (c - L.chunk_prefix[lo]) * L.chunk_elems;
    const int64_t ce = (cb + L.chunk_elems < tw.end) ? cb + L.chunk_elems : tw.end;
    for (int64_t e = cb + threadIdx.x; e < ce; e += blockDim.x) {
      T acc = reinterpret_cast<const T*>(tw.src[0])[e];
      for (int k = 1; k < tw.n_src; ++k) acc = static_cast<T>(acc + reinterpret_cast<const T*>(tw.src[k])[e]);
      for (int j = 0; j < tw.n_out; ++j) reinterpret_cast<T*>(tw.out[j])[e] = acc;
    }
  }
  if (sync) barrier_end(L.sync, L.sync.mode == SYNC_WRITE_PEERS);
}

// ---------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------
typedef void (*DenseKernelFn)(DenseLaunch);

template <typename T, int OPT, bool MP>
static DenseKernelFn pick_n(bool small_n) {
  // the two-packet variant is only instantiated where it stays inside 64 registers
  if constexpr (OPT == OPT_NONE || OPT == OPT_SGD || OPT == OPT_TEST) {
    if (small_n) return kv_dense_kernel<T, OPT, MP, true>;
  }
  return kv_dense_kernel<T, OPT, MP, false>;
}

template <typename T>
static DenseKernelFn pick_opt(int opt, bool mp, bool small_n, bool allow_non_mp) {
  if (opt == OPT_NONE) return pick_n<T, OPT_NONE, false>(small_n);
  if (mp) {
    switch (opt) {
      case OPT_SGD: return pick_n<T, OPT_SGD, true>(small_n);
      case OPT_SGD_MOM: return pick_n<T, OPT_SGD_MOM, true>(small_n);
      case OPT_ADAM: return pick_n<T, OPT_ADAM, true>(small_n);
      case OPT_ADAMW: return pick_n<T, OPT_ADAMW, true>(small_n);
      case OPT_TEST: return pick_n<T, OPT_TEST, true>(small_n);
      default: return nullptr;
    }
  }
  if (!allow_non_mp) return nullptr;
  return nullptr;
}

static DenseKernelFn pick_kernel(const DenseLaunch& L) {
  const bool mp = L.multi_precision != 0;
  // the two-packet variant stays inside 64 registers (2 resident blocks/SM) only for these
  const bool sn = L.small_n != 0 && (L.opt == OPT_NONE || L.opt == OPT_SGD || L.opt == OPT_TEST);
  switch (L.dtype) {
    case kFloat32:
      if (mp || L.opt == OPT_NONE) return pick_opt<float>(L.opt, mp, sn, true);
      switch (L.opt) {
        case OPT_SGD: return pick_n<float, OPT_SGD, false>(sn);
        case OPT_SGD_MOM: return pick_n<float, OPT_SGD_MOM, false>(sn);
        case OPT_ADAM: return pick_n<float, OPT_ADAM, false>(sn);
        case OPT_ADAMW: return pick_n<float, OPT_ADAMW, false>(sn);
        case OPT_TEST: return pick_n<float, OPT_TEST, false>(sn);
        case OPT_SGD_STD: return kv_dense_kernel<float, OPT_SGD_STD, false, false>;
        case OPT_ADAM_STD: return kv_dense_kernel<float, OPT_ADAM_STD, false, false>;
        default: return nullptr;
      }
    case kFloat16: return pick_opt<__half>(L.opt, mp, sn, false);
    case kBfloat16: return pick_opt<__nv_bfloat16>(L.opt, mp, sn, false);
    case kFloat64: return L.opt == OPT_NONE ? kv_sum_typed_kernel<double> : nullptr;
    case kInt32: return L.opt == OPT_NONE ? kv_sum_typed_kernel<int32_t> : nullptr;
    case kInt64: return L.opt == OPT_NONE ? kv_sum_typed_kernel<int64_t> : nullptr;
    case kUint8: return L.opt == OPT_NONE ? kv_sum_typed_kernel<uint8_t> : nullptr;
    case kInt8: return L.opt == OPT_NONE ? kv_sum_typed_kernel<int8_t> : nullptr;
    default: return nullptr;
  }
}

#if !defined(MXKV_HOST_EMU)
static int g_num_sms[64] = {0};

static int sm_count(int device) {
  if (device < 0 || device >= 64) return kNumSms;
  if (g_num_sms[device] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0) n = kNumSms;
    g_num_sms[device] = n;
  }
  return g_num_sms[device];
}

int DenseMaxGrid(int device, int threads) {
  // __launch_bounds__(512, 2): 64 registers/thread, i.e. 1024 resident threads per SM for every
  // instantiation, whatever the block size
  if (threads != 128 && threads != 256 && threads != 512) threads = kThreads;
  int g = (1024 / threads) * sm_count(device);
  return g > kMaxBlocks ? kMaxBlocks : g;
}

// Function attributes are per device: opt in to large dynamic shared memory on the GPU a launch goes to -- and
// only there (a process that owns one GPU must not create contexts on the others).  The device must be current.
static bool EnsureBulkAttr(int device, int opt, int multi_precision) {
  static bool attr_done[64][16] = {{false}};
  if (device < 0 || device >= 64) return false;
  const int slot = (opt & 7) * 2 + (multi_precision ? 1 : 0);
  if (attr_done[device][slot]) return true;
  BulkKernelFn fn = pick_bulk(opt, multi_precision);
  if (fn == nullptr) return false;
  if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  attr_done[device][slot] = true;
  return true;
}

static int g_smem_budget = 0;   // MXKV_B200_BULK_SMEM_KB per block (default 100: two blocks per SM)

int BulkPlan(int device, int opt, int multi_precision, int arrays, int* tile_elems, int* stages) {
  BulkKernelFn fn = pick_bulk(opt, multi_precision);
  if (fn == nullptr || arrays < 1) return 0;
  if (g_smem_budget == 0) {
    const char* e = getenv("MXKV_B200_BULK_SMEM_KB");
    g_smem_budget = (e && *e) ? atoi(e) * 1024 : 100 * 1024;
    if (g_smem_budget < 16 * 1024) g_smem_budget = 16 * 1024;
    if (g_smem_budget > 200 * 1024) g_smem_budget = 200 * 1024;
  }
  // 2048-element tiles, two stages (MXKV_B200_BULK_TILE / _STAGES override them): with two blocks per SM
  // that is 2 x 100 KB of the 228 KB of shared memory an H100 SM has.  Wide work lists (many sources) fall
  // back to 1024-element tiles to keep two blocks per SM resident.
  int tile = 2048;
  int st = 2;
  if (st * arrays * tile * 4 > g_smem_budget) tile = 1024;
  if (st * arrays * tile * 4 > g_smem_budget) return 0;
  {
    static int env_tile = -1, env_st = -1;
    if (env_tile < 0) {
      const char* e1 = getenv("MXKV_B200_BULK_TILE");
      const char* e2 = getenv("MXKV_B200_BULK_STAGES");
      env_tile = (e1 && *e1) ? atoi(e1) : 0;
      env_st = (e2 && *e2) ? atoi(e2) : 0;
    }
    if (env_tile >= 256 && env_tile % 128 == 0) tile = env_tile;
    if (env_st >= 2) st = env_st;
    if (st * arrays * tile * 4 > 200 * 1024) return 0;
  }
  if (st < 2) return 0;
  if (st > kBulkMaxStages) st = kBulkMaxStages;
  const int smem = st * arrays * tile * 4;
  int prev = -1;
  cudaGetDevice(&prev);
  if (prev != device) cudaSetDevice(device);
  bool ok = EnsureBulkAttr(device, opt, multi_precision);
  int occ = 0;
  if (ok && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, kBulkThreads, smem) != cudaSuccess || occ < 1)) {
    cudaGetLastError();
    ok = false;
  }
  if (prev >= 0 && prev != device) cudaSetDevice(prev);
  if (!ok) return 0;
  *tile_elems = tile;
  *stages = st;
  int g = occ * sm_count(device);
  return g > kMaxBlocks ? kMaxBlocks : g;
}

int LaunchDense(const DenseLaunch& L, cudaStream_t stream) {
  if (L.order == ORDER_TREE) return LaunchDenseTree(L, stream);
  if (L.nvls) {
    NvlsKernelFn nf = pick_nvls(L.opt, L.multi_precision, L.nvls_unroll, L.nvls_pipe);
    if (nf == nullptr || L.dtype != kFloat32 || L.sync.mode == SYNC_NONE) return static_cast<int>(cudaErrorInvalidValue);
    int grid = L.grid < 1 ? 1 : (L.grid > kMaxBlocks ? kMaxBlocks : L.grid);
    int threads = L.threads;
    if (threads != 128 && threads != 256 && threads != 512) threads = kThreads;
    if (L.chunk_elems != threads * nvls_round_unroll(L.nvls_unroll, L.opt) * 4) return static_cast<int>(cudaErrorInvalidValue);
    nf<<<grid, threads, 0, stream>>>(L);
    return static_cast<int>(cudaGetLastError());
  }
  if (L.bulk) {
    BulkKernelFn bf = pick_bulk(L.opt, L.multi_precision);
    if (bf == nullptr || L.dtype != kFloat32) return static_cast<int>(cudaErrorInvalidValue);
    int cur = -1;                      // single process, several GPUs: the plan was made on the first participant
    cudaGetDevice(&cur);
    if (!EnsureBulkAttr(cur, L.opt, L.multi_precision)) return static_cast<int>(cudaErrorInvalidValue);
    int grid = L.grid < 1 ? 1 : (L.grid > kMaxBlocks ? kMaxBlocks : L.grid);
    const size_t smem = static_cast<size_t>(L.bulk_stages) * L.bulk_arrays * L.chunk_elems * 4;
    bf<<<grid, kBulkThreads, smem, stream>>>(L);
    return static_cast<int>(cudaGetLastError());
  }
  DenseKernelFn fn = pick_kernel(L);
  if (fn == nullptr) return static_cast<int>(cudaErrorInvalidValue);
  int grid = L.grid;
  if (grid < 1) grid = 1;
  if (grid > kMaxBlocks) grid = kMaxBlocks;
  int threads = L.threads;
  if (threads != 128 && threads != 256 && threads != 512) threads = kThreads;
  fn<<<grid, threads, 0, stream>>>(L);
  return static_cast<int>(cudaGetLastError());
}

template <typename T>
__global__ void kv_cast_f32_kernel(const T* __restrict__ src, float* __restrict__ dst, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = Cvt<T>::to(src[i]);
}

int LaunchCastToF32(const void* src, int dtype, float* dst, int64_t n, cudaStream_t s) {
  if (n == 0) return 0;
  const int threads = 256;
  int64_t blocks = (n + threads - 1) / threads;
  if (blocks > kMaxBlocks) blocks = kMaxBlocks;
  switch (dtype) {
    case kFloat32: kv_cast_f32_kernel<float><<<blocks, threads, 0, s>>>(static_cast<const float*>(src), dst, n); break;
    case kFloat16: kv_cast_f32_kernel<__half><<<blocks, threads, 0, s>>>(static_cast<const __half*>(src), dst, n); break;
    case kBfloat16: kv_cast_f32_kernel<__nv_bfloat16><<<blocks, threads, 0, s>>>(static_cast<const __nv_bfloat16*>(src), dst, n); break;
    default: return static_cast<int>(cudaErrorInvalidValue);
  }
  return static_cast<int>(cudaGetLastError());
}

// ---------------------------------------------------------------------------
// 1-bit / 2-bit gradient compression with error feedback
// (src/kvstore/gradient_compression-inl.h:44-227).  One thread per 32-bit code word (the reference
// uses one thread per byte): residual += grad; emit the code; keep the quantisation error in the
// residual.  Bit layout is the reference's: byte j of the stream holds values 4j..4j+3 (2-bit) or
// 8j..8j+7 (1-bit), first value in the most significant bits.
// ---------------------------------------------------------------------------
template <int BITS>
__global__ void kv_quantize_kernel(const float* __restrict__ grad, float* __restrict__ residual,
                                   uint32_t* __restrict__ out, int64_t n, float thr) {
  constexpr int PER_WORD = 32 / BITS;
  const int64_t nwords = (n + PER_WORD - 1) / PER_WORD;
  for (int64_t w = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; w < nwords;
       w += static_cast<int64_t>(gridDim.x) * blockDim.x)
    out[w] = quantize_word<BITS>(grad, residual, n, thr, w);
}

template <int BITS>
__global__ void kv_dequantize_kernel(const uint32_t* __restrict__ in, float* __restrict__ out, int64_t n, float thr) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    out[i] = dequantize_value<BITS>(in, thr, i);
}

int LaunchQuantize(int bits, const float* grad, float* residual, uint32_t* out, int64_t n, float thr, cudaStream_t s) {
  if (n == 0) return 0;
  const int per = 32 / bits;
  int64_t blocks = ((n + per - 1) / per + 255) / 256;
  if (blocks > kMaxBlocks) blocks = kMaxBlocks;
  if (blocks < 1) blocks = 1;
  if (bits == 2) kv_quantize_kernel<2><<<blocks, 256, 0, s>>>(grad, residual, out, n, thr);
  else if (bits == 1) kv_quantize_kernel<1><<<blocks, 256, 0, s>>>(grad, residual, out, n, thr);
  else return static_cast<int>(cudaErrorInvalidValue);
  return static_cast<int>(cudaGetLastError());
}

int LaunchDequantize(int bits, const uint32_t* in, float* out, int64_t n, float thr, cudaStream_t s) {
  if (n == 0) return 0;
  int64_t blocks = (n + 255) / 256;
  if (blocks > kMaxBlocks) blocks = kMaxBlocks;
  if (bits == 2) kv_dequantize_kernel<2><<<blocks, 256, 0, s>>>(in, out, n, thr);
  else if (bits == 1) kv_dequantize_kernel<1><<<blocks, 256, 0, s>>>(in, out, n, thr);
  else return static_cast<int>(cudaErrorInvalidValue);
  return static_cast<int>(cudaGetLastError());
}

__global__ void kv_barrier_kernel(SyncArgs sync) {
  barrier_start(sync);
  barrier_end(sync, true);
}

int LaunchBarrier(const SyncArgs& sync, cudaStream_t stream) {
  kv_barrier_kernel<<<1, 32, 0, stream>>>(sync);
  return static_cast<int>(cudaGetLastError());
}

int LaunchFill(void* ptr, int value_byte, size_t bytes, cudaStream_t s) {
  if (bytes == 0) return 0;
  return static_cast<int>(cudaMemsetAsync(ptr, value_byte, bytes, s));
}

#else   // MXKV_HOST_EMU
// tests/sim/hostemu_dense.cc: this file compiled by g++ -- the per-thread, the staged and the typed-sum kernels run
// as CPU threads from the source above.  The instantiation is chosen by the same pick_* code the device launch uses.
int LaunchDenseHostEmu(const DenseLaunch& L) {
  if (L.order == ORDER_TREE) return 1;
  const int grid = L.grid < 1 ? 1 : (L.grid > kMaxBlocks ? kMaxBlocks : L.grid);
  if (L.nvls) {      // a chunk is exactly blockDim * U vectors: this kernel needs the launch's own block size
    NvlsKernelFn nf = pick_nvls(L.opt, L.multi_precision, L.nvls_unroll, L.nvls_pipe);
    int threads = L.threads;
    if (threads != 128 && threads != 256 && threads != 512) threads = kThreads;
    if (nf == nullptr || L.dtype != kFloat32 || L.sync.mode == SYNC_NONE ||
        L.chunk_elems != threads * nvls_round_unroll(L.nvls_unroll, L.opt) * 4) return 1;
    hostemu::RunGridFibers(nf, dim3(static_cast<unsigned>(grid), 1, 1), threads, 0, L);
    return 0;
  }
  if (L.bulk) {
    BulkKernelFn bf = pick_bulk(L.opt, L.multi_precision);
    if (bf == nullptr || L.dtype != kFloat32) return 1;
    const size_t smem = static_cast<size_t>(L.bulk_stages) * L.bulk_arrays * L.chunk_elems * 4;
    hostemu::RunGrid(bf, L, grid, kBulkThreads, smem);
    return 0;
  }
  DenseKernelFn fn = pick_kernel(L);
  if (fn == nullptr) return 1;
  hostemu::RunGrid(fn, L, grid, L.threads);
  return 0;
}
#endif  // MXKV_HOST_EMU

}  // namespace mxkv
