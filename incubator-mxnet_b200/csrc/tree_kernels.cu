// tree_kernels.cu -- the dense kernel for stores created with MXNET_KVSTORE_USETREE=1 (reference: CommDeviceTree,
// src/kvstore/comm_tree.h:91-325).
//
// The reference reduces a key in log2(n) rounds of cudaMemcpyPeerAsync + ElementwiseSum over per-GPU merge buffers,
// then broadcasts down the same tree.  What a caller can observe of that is the association of the sum -- pairwise up
// a tree chosen from the link matrix, one tree per row slice for big keys -- so this kernel keeps the transport of
// kv_dense_kernel (kernels.cu: every thread streams 16-byte vectors of the n replicas straight from the GPUs that own
// them, updates, and stores to every destination; one pass, cross-GPU rendezvous in the kernel) and only changes the
// order of the additions: the sources of a work entry arrive in the tree's leaf order and TensorWork::tree_prog says
// when two partial sums meet (topology.h: ReduceProgram; tree_math.h: TreeSum).
//
// Separate translation unit on purpose: the kernels of kernels.cu are bit-for-bit what was profiled and validated
// on hardware; the tree path adds instantiations next to them, not branches inside them.
#include "kernels.h"
#include "device_utils.cuh"
#include "tree_math.h"

namespace mxkv {

namespace {

// rounds a float32 partial sum to T after every addition: what ElementwiseSum does on float16 arrays when no
// optimizer follows (the reference adds half_t values)
template <typename T>
struct AddRounded {
  bool round;
  __device__ __forceinline__ float operator()(float l, float r) const {
    float s = __fadd_rn(l, r);
    if (round) s = Cvt<T>::to(Cvt<T>::from(s));
    return s;
  }
};

// one packet of N elements at element offset e: gather the n sources four loads at a time (all of a batch are
// issued before the first is used), add them in program order, update, scatter
template <typename T, int OPT, bool MP, int N>
__device__ __forceinline__ void tree_packet(const TensorWork& tw, int64_t e, const Hyper& h, bool native_half_add) {
  typedef Packet<T, N> P;
  constexpr int BATCH = 4;
  TreeSum<float, N> sum;
  sum.begin(tw.tree_prog);
  const AddRounded<T> add{native_half_add};
  const int n = tw.n_src;
  for (int k0 = 0; k0 < n; k0 += BATCH) {
    P buf[BATCH];
#pragma unroll
    for (int j = 0; j < BATCH; ++j)
      if (k0 + j < n) buf[j].load(tw.src[k0 + j], e);
#pragma unroll
    for (int j = 0; j < BATCH; ++j) {
      if (k0 + j < n) {
        float x[N];
        buf[j].unpack(x);
        sum.take(x, add);
      }
    }
  }
  float acc[N];
  sum.result(acc);

  float wnew[N];
  if (OPT == OPT_NONE) {
#pragma unroll
    for (int i = 0; i < N; ++i) wnew[i] = acc[i];
  } else {
    constexpr bool HAS_S0 = OptHasS0(OPT);
    constexpr bool HAS_S1 = OptHasS1(OPT);
    constexpr bool HAS_S2 = OptHasS2(OPT);
    float w[N], s0[N], s1[N], s2[N];
    if (MP) {
      ldf<N>(tw.w32, e, w);
    } else {
      P pw;
      pw.load(tw.w, e);
      pw.unpack(w);
    }
    if (HAS_S0) ldf<N>(tw.s0, e, s0);
    if (HAS_S1) ldf<N>(tw.s1, e, s1);
    if (HAS_S2) ldf<N>(tw.s2, e, s2);
#pragma unroll
    for (int i = 0; i < N; ++i) wnew[i] = update_one<OPT>(acc[i], w[i], s0[i], s1[i], s2[i], h);
    if (HAS_S0) stf<N>(tw.s0, e, s0);
    if (HAS_S1) stf<N>(tw.s1, e, s1);
    if (HAS_S2) stf<N>(tw.s2, e, s2);
    if (MP) stf<N>(tw.w32, e, wnew);
  }
  const int m = tw.n_out;
  for (int j = 0; j < m; ++j) P::store(tw.out[j], e, wnew);
}

}  // namespace

template <typename T, int OPT, bool MP>
__global__ void __launch_bounds__(kThreads, 2)
kv_dense_tree_kernel(DenseLaunch L) {
  __shared__ TensorWork tw;
  const bool sync = L.sync.mode != SYNC_NONE;
  if (sync) barrier_start(L.sync);

  // 16-byte packets of float32, 8-byte packets (4 elements) of the 16-bit types: with three pending partial sums per
  // element next to a batch of loads, 8 elements per thread would not fit in the 64 registers that keep two blocks
  // of 512 threads resident (the residency the rendezvous grid is sized for)
  // (float32 keys of centered RMSProp and FTML, with three state arrays, take one element at a time for the same
  // reason; so do FTML's 16-bit keys, which spill 32 / 48 bytes at 64 registers with 4-element packets, and the
  // float32 keys of Adamax, AdaDelta and Nadam, which spill 12 / 16 / 16 bytes with them)
  constexpr bool kOneElem = OPT == OPT_ADAMAX || OPT == OPT_ADADELTA || OPT == OPT_NADAM;
  constexpr int NV = (sizeof(T) == 2 && OPT == OPT_FTML) ? 1
                   : (sizeof(T) == 2 ? 4 : ((OptHasS2(OPT) || kOneElem) ? 1 : 16 / sizeof(T)));
  const bool native_half_add = (sizeof(T) == 2) && !L.fp32_accum && (OPT == OPT_NONE);
  int cur = -1;
  for (int64_t c = blockIdx.x; c < L.total_chunks; c += gridDim.x) {
    const int lo = find_work(L, c, &cur, &tw);
    const Hyper h = make_hyper<OPT>(L, tw, sizeof(T) == 2 && L.mp_arith != 0, lo);

    const int64_t cb = tw.begin + (c - L.chunk_prefix[lo]) * L.chunk_elems;
    const int64_t ce = (cb + L.chunk_elems < tw.end) ? cb + L.chunk_elems : tw.end;
    int64_t scalar_from = cb;
    if (tw.flags & kWorkVec16) {  // every pointer 16-byte aligned and begin % 8 == 0
      const int64_t nvec = (ce - cb) / NV;
      for (int64_t v = threadIdx.x; v < nvec; v += blockDim.x)
        tree_packet<T, OPT, MP, NV>(tw, cb + v * NV, h, native_half_add);
      scalar_from = cb + nvec * NV;
    }
    for (int64_t s = scalar_from + threadIdx.x; s < ce; s += blockDim.x)
      tree_packet<T, OPT, MP, 1>(tw, s, h, native_half_add);
  }

  if (sync) barrier_end(L.sync, L.sync.mode == SYNC_WRITE_PEERS);
}

// float64 keys (no optimizer): native double additions in tree order.  The integer dtypes need no tree variant --
// their sums wrap and are associative -- and stay on kv_sum_typed_kernel.
struct AddF64 {
  __device__ __forceinline__ double operator()(double l, double r) const { return __dadd_rn(l, r); }
};

__global__ void __launch_bounds__(kThreads, 2)
kv_sum_tree_f64_kernel(DenseLaunch L) {
  __shared__ TensorWork tw;
  const bool sync = L.sync.mode != SYNC_NONE;
  if (sync) barrier_start(L.sync);
  int cur = -1;
  for (int64_t c = blockIdx.x; c < L.total_chunks; c += gridDim.x) {
    const int lo = find_work(L, c, &cur, &tw);
    const int64_t cb = tw.begin + (c - L.chunk_prefix[lo]) * L.chunk_elems;
    const int64_t ce = (cb + L.chunk_elems < tw.end) ? cb + L.chunk_elems : tw.end;
    for (int64_t e = cb + threadIdx.x; e < ce; e += blockDim.x) {
      TreeSum<double, 1> sum;
      sum.begin(tw.tree_prog);
      for (int k = 0; k < tw.n_src; ++k) {
        const double x[1] = {reinterpret_cast<const double*>(tw.src[k])[e]};
        sum.take(x, AddF64());
      }
      double acc[1];
      sum.result(acc);
      for (int j = 0; j < tw.n_out; ++j) reinterpret_cast<double*>(tw.out[j])[e] = acc[0];
    }
  }
  if (sync) barrier_end(L.sync, L.sync.mode == SYNC_WRITE_PEERS);
}

typedef void (*TreeKernelFn)(DenseLaunch);

template <typename T>
static TreeKernelFn pick_tree_opt(int opt, bool mp) {
  if (opt == OPT_NONE) return kv_dense_tree_kernel<T, OPT_NONE, false>;
  return ElementwiseOpts::Dispatch<TreeKernelFn>(opt, [&](auto k) -> TreeKernelFn {
    constexpr int K = decltype(k)::value;
    if (mp) return kv_dense_tree_kernel<T, K, true>;
    if constexpr (sizeof(T) == 4) return kv_dense_tree_kernel<T, K, false>;   // 16-bit keys: fp32 master only
    return nullptr;
  });
}

// 1 when a tree kernel exists for this dtype / optimizer / precision mode (the host decides per key whether the
// tree order can be honoured before it builds work entries)
int TreeKernelAvailable(int dtype, int opt, int multi_precision) {
  const bool mp = multi_precision != 0;
  switch (dtype) {
    case kFloat32: return pick_tree_opt<float>(opt, mp) != nullptr;
    case kFloat16: return pick_tree_opt<__half>(opt, mp) != nullptr;
    case kBfloat16: return pick_tree_opt<__nv_bfloat16>(opt, mp) != nullptr;
    case kFloat64: return opt == OPT_NONE;
    default: return 0;
  }
}

int LaunchDenseTree(const DenseLaunch& L, cudaStream_t stream) {
  const bool mp = L.multi_precision != 0;
  TreeKernelFn fn = nullptr;
  switch (L.dtype) {
    case kFloat32: fn = pick_tree_opt<float>(L.opt, mp); break;
    case kFloat16: fn = pick_tree_opt<__half>(L.opt, mp); break;
    case kBfloat16: fn = pick_tree_opt<__nv_bfloat16>(L.opt, mp); break;
    case kFloat64: fn = L.opt == OPT_NONE ? kv_sum_tree_f64_kernel : nullptr; break;
    default: break;
  }
  if (fn == nullptr || L.nvls || L.bulk) return static_cast<int>(cudaErrorInvalidValue);
  int grid = L.grid;
  if (grid < 1) grid = 1;
  if (grid > kMaxBlocks) grid = kMaxBlocks;
  int threads = L.threads;
  if (threads != 128 && threads != 256 && threads != 512) threads = kThreads;
#if defined(MXKV_HOST_EMU)       // tests/sim/hostemu_tree.cc: this file compiled by g++, blocks run as CPU threads
  (void)stream;
  hostemu::RunGrid(fn, L, grid, threads);
  return 0;
#else
  fn<<<grid, threads, 0, stream>>>(L);
  return static_cast<int>(cudaGetLastError());
#endif
}

}  // namespace mxkv
