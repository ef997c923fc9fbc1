// norm_kernels.cu -- sm_90a kernels of the layer-wise adaptive optimizers (see norm_kernels.h).
//
// Element arithmetic follows the reference's CPU kernels operation by operation
// (contrib/multi_lamb.cc:36-120, contrib/multi_lans.cc:36-130, optimizer_op-inl.h:377-390,590-606
// for LARS' sgd/sgd_mom step) with __f*_rn intrinsics so nothing is contracted into an FMA; the
// sums of squares are tree reductions with a fixed shape (per-thread strided partials -> warp
// shuffle -> warp order -> chunk order -> rank order), so a result is reproducible run to run and
// identical on every rank, but its rounding differs from the reference's sequential
// (CPU, multi_sum_sq.cc:42-62) or block-shaped (GPU, multi_sum_sq.cu:85-121) sums -- which also
// differ from each other.
#include "norm_kernels.h"
#include "device_utils.cuh"
#include "norm_math.h"

namespace mxkv {

constexpr int kNormThreads = 512;
constexpr int kNormWarps = kNormThreads / 32;

// chunk -> work entry (uniform across the block)
__device__ __forceinline__ int find_entry(const int64_t* prefix, int nworks, int64_t c) {
  int lo = 0, hi = nworks - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (prefix[mid] <= c) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ void load_work(NormWork* dst, const NormWork* src) {
  __syncthreads();
  const uint4* s = reinterpret_cast<const uint4*>(src);
  uint4* d = reinterpret_cast<uint4*>(dst);
  for (int i = threadIdx.x; i < static_cast<int>(sizeof(NormWork) / 16); i += blockDim.x) d[i] = s[i];
  __syncthreads();
}

// fixed-shape block reduction of K per-thread partials; thread j < K writes total j to dst[j]
template <int K>
__device__ __forceinline__ void block_sums(float (&p)[K], float* red, float* dst) {
#pragma unroll
  for (int k = 0; k < K; ++k) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) p[k] += __shfl_xor_sync(0xffffffffu, p[k], off);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) red[warp * K + k] = p[k];
  }
  __syncthreads();
  if (threadIdx.x < K) {
    float s = 0.f;
    const int nw = blockDim.x >> 5;
    for (int w = 0; w < nw; ++w) s += red[w * K + threadIdx.x];
    dst[threadIdx.x] = s;
  }
  __syncthreads();
}

// gather the n gradient replicas of N consecutive elements and add them in the reference's
// association order, fp32 accumulation (four 16-byte requests in flight per thread)
template <typename T, int N>
__device__ __forceinline__ void sum_sources(const NormWork& tw, int64_t e, int order, float (&acc)[N]) {
  typedef Packet<T, N> P;
  float grp[N];
  const int n = tw.n_src;
  for (int k0 = 0; k0 < n; k0 += 4) {
    P buf[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (k0 + j < n) buf[j].load(tw.src[k0 + j], e);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + j;
      if (k < n) {
        float x[N];
        buf[j].unpack(x);
        if (k == 0) {
#pragma unroll
          for (int i = 0; i < N; ++i) acc[i] = x[i];
        } else if (order == ORDER_DEVICE) {
#pragma unroll
          for (int i = 0; i < N; ++i) acc[i] = __fadd_rn(acc[i], x[i]);
        } else {   // ORDER_COMMCPU: in0 += ((in1+in2)+in3)+in4 per group of four (comm.h:359-393)
          const int pos = (k - 1) & 3;
#pragma unroll
          for (int i = 0; i < N; ++i) grp[i] = (pos == 0) ? x[i] : __fadd_rn(grp[i], x[i]);
          if (pos == 3 || k == n - 1) {
#pragma unroll
            for (int i = 0; i < N; ++i) acc[i] = __fadd_rn(acc[i], grp[i]);
          }
        }
      }
    }
  }
}

template <typename T, int N>
__device__ __forceinline__ void load_weight_t(const NormWork& tw, int64_t e, float (&w)[N]) {
  Packet<T, N> pw;
  pw.load(tw.w, e);
  pw.unpack(w);
}

// ---------------------------------------------------------------------------
// first: reduce (+ LAMB step 1 | park the gradient) + chunk partials
// ---------------------------------------------------------------------------
template <typename T, bool MP, bool GRAD_ONLY, int N>
__device__ __forceinline__ void first_elems(const NormWork& tw, int64_t e, const NormLaunch& L, float (&p)[3]) {
  float g[N], w[N];
  sum_sources<T, N>(tw, e, L.order, g);
  // the weight whose norm is taken: LAMB uses the fp32 master when there is one
  // (multi_lamb-inl.h:296-303); LARS and LANS always use the stored weight itself
  // (lars.py:119 `_l2norm(weight)`, multi_lans-inl.h:296-300)
  if (MP && !GRAD_ONLY) ldf<N>(tw.w32, e, w); else load_weight_t<T, N>(tw, e, w);
#pragma unroll
  for (int i = 0; i < N; ++i) p[2] += not_finite(g[i]) ? 1.0f : 0.0f;
  if (GRAD_ONLY) {
    stf<N>(tw.aux0, e, g);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      p[0] += w[i] * w[i];
      const float gs = (L.rescale != 1.0f) ? __fmul_rn(g[i], L.rescale) : g[i];   // multi_sum_sq.cc:52-56
      p[1] += gs * gs;
    }
  } else {
    float m[N], v[N], gh[N];
    ldf<N>(tw.s0, e, m);
    ldf<N>(tw.s1, e, v);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      gh[i] = lamb_step1(g[i], w[i], m[i], v[i], L, tw);
      p[0] += w[i] * w[i];
      p[1] += gh[i] * gh[i];
    }
    stf<N>(tw.s0, e, m);
    stf<N>(tw.s1, e, v);
    stf<N>(tw.aux0, e, gh);
  }
}

template <typename T, bool MP, bool GRAD_ONLY>
__global__ void __launch_bounds__(kNormThreads, 2)
kv_norm_first_kernel(NormLaunch L) {
  __shared__ NormWork tw;
  __shared__ float red[kNormWarps * 3];
  const bool sync = L.sync.mode != SYNC_NONE;
  if (sync) barrier_start(L.sync);
  int cur = -1;
  for (int64_t c = blockIdx.x; c < L.total_chunks; c += gridDim.x) {
    const int lo = find_entry(L.chunk_prefix, L.nworks, c);
    if (lo != cur) { load_work(&tw, L.works + lo); cur = lo; }
    const int64_t ci = c - L.chunk_prefix[lo];
    const int64_t cb = tw.begin + ci * L.chunk_elems;
    const int64_t ce = (cb + L.chunk_elems < tw.end) ? cb + L.chunk_elems : tw.end;
    float p[3] = {0.f, 0.f, 0.f};
    int64_t scalar_from = cb;
    if (tw.flags & 1) {
      const int64_t nvec = (ce - cb) / 4;
      for (int64_t v = threadIdx.x; v < nvec; v += blockDim.x)
        first_elems<T, MP, GRAD_ONLY, 4>(tw, cb + v * 4, L, p);
      scalar_from = cb + nvec * 4;
    }
    for (int64_t s = scalar_from + threadIdx.x; s < ce; s += blockDim.x)
      first_elems<T, MP, GRAD_ONLY, 1>(tw, s, L, p);
    block_sums<3>(p, red, tw.psum + ci * kPsumStride);
  }
  if (sync) barrier_end(L.sync, false);
}

// ---------------------------------------------------------------------------
// finalize: chunk partials -> this rank's per-key totals, one block per entry
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
kv_norm_finalize_kernel(const NormWork* works, const int64_t* prefix, int nslots, int slot0, int slot1, int slot2) {
  __shared__ float red[8 * 3];
  const NormWork* w = works + blockIdx.x;
  const int64_t nchunks = prefix[blockIdx.x + 1] - prefix[blockIdx.x];
  const float* psum = w->psum;
  float p[3] = {0.f, 0.f, 0.f};
  for (int64_t i = threadIdx.x; i < nchunks; i += blockDim.x) {
#pragma unroll
    for (int j = 0; j < 3; ++j)
      if (j < nslots) p[j] += psum[i * kPsumStride + j];
  }
  __shared__ float tot[3];
  block_sums<3>(p, red, tot);
  if (threadIdx.x == 0) {
    const int slots[3] = {slot0, slot1, slot2};
    for (int j = 0; j < nslots; ++j) w->nrm[slots[j]] = tot[j];
  }
}

// number of non-finite merged-gradient elements over every key of the push and every rank
__device__ __forceinline__ float launch_bad_total(const NormLaunch& L, float* red) {
  float p[1] = {0.f};
  for (int i = threadIdx.x; i < L.n_bad; i += blockDim.x) p[0] += *L.bad_list[i];
  __shared__ float tot[1];
  block_sums<1>(p, red, tot);
  return tot[0];
}

// ---------------------------------------------------------------------------
// mid: step 1 from the parked gradient (LANS; LAMB behind an overflow check)
// ---------------------------------------------------------------------------
template <typename T, bool MP, int KIND, int N>
__device__ __forceinline__ void mid_elems(const NormWork& tw, int64_t e, const NormLaunch& L, float g_norm,
                                          float (&p)[3]) {
  float g[N], w[N], m[N], v[N];
  ldf<N>(tw.aux0, e, g);
  if (MP) ldf<N>(tw.w32, e, w); else load_weight_t<T, N>(tw, e, w);
  ldf<N>(tw.s0, e, m);
  ldf<N>(tw.s1, e, v);
  if (KIND == NORM_LAMB) {
    float gh[N];
#pragma unroll
    for (int i = 0; i < N; ++i) {
      gh[i] = lamb_step1(g[i], w[i], m[i], v[i], L, tw);
      p[0] += w[i] * w[i];
      p[1] += gh[i] * gh[i];
    }
    stf<N>(tw.aux0, e, gh);
  } else {   // LANS step 1, multi_lans.cc:48-84
    float tm[N], tg[N];
#pragma unroll
    for (int i = 0; i < N; ++i) {
      lans_step1(g[i], w[i], m[i], v[i], g_norm, L, tw, tm[i], tg[i]);
      p[0] += tm[i] * tm[i];
      p[1] += tg[i] * tg[i];
    }
    stf<N>(tw.aux1, e, tm);
    stf<N>(tw.aux0, e, tg);
  }
  stf<N>(tw.s0, e, m);
  stf<N>(tw.s1, e, v);
}

template <typename T, bool MP, int KIND>
__global__ void __launch_bounds__(kNormThreads, 2)
kv_norm_mid_kernel(NormLaunch L) {
  __shared__ NormWork tw;
  __shared__ float red[kNormWarps * 3];
  __shared__ float sc[1];
  const bool sync = L.sync.mode != SYNC_NONE;
  if (sync) barrier_start(L.sync);   // the peers' totals of the first phase are complete
  bool skip = false;
  if (L.skip_nonfinite) skip = launch_bad_total(L, red) > 0.f;
  int cur = -1;
  for (int64_t c = blockIdx.x; c < L.total_chunks && !skip; c += gridDim.x) {
    const int lo = find_entry(L.chunk_prefix, L.nworks, c);
    if (lo != cur) {
      load_work(&tw, L.works + lo);
      cur = lo;
      if (KIND == NORM_LANS) {
        if (threadIdx.x == 0) sc[0] = __fsqrt_rn(rank_total(tw, kNrmG));   // multi_lans.cc:51
        __syncthreads();
      }
    }
    const float g_norm = (KIND == NORM_LANS) ? sc[0] : 1.0f;
    const int64_t ci = c - L.chunk_prefix[lo];
    const int64_t cb = tw.begin + ci * L.chunk_elems;
    const int64_t ce = (cb + L.chunk_elems < tw.end) ? cb + L.chunk_elems : tw.end;
    float p[3] = {0.f, 0.f, 0.f};
    int64_t scalar_from = cb;
    if (tw.flags & 1) {
      const int64_t nvec = (ce - cb) / 4;
      for (int64_t v = threadIdx.x; v < nvec; v += blockDim.x)
        mid_elems<T, MP, KIND, 4>(tw, cb + v * 4, L, g_norm, p);
      scalar_from = cb + nvec * 4;
    }
    for (int64_t s = scalar_from + threadIdx.x; s < ce; s += blockDim.x)
      mid_elems<T, MP, KIND, 1>(tw, s, L, g_norm, p);
    block_sums<3>(p, red, tw.psum + ci * kPsumStride);
  }
  if (sync) barrier_end(L.sync, false);
}

// ---------------------------------------------------------------------------
// apply: trust ratio from the totals, step 2, stores to every replica
// ---------------------------------------------------------------------------
template <typename T, bool MP, int FLAVOR, int N>
__device__ __forceinline__ void apply_elems(const NormWork& tw, int64_t e, const NormLaunch& L, const float* sc,
                                            bool skip) {
  float w[N], wn[N];
  if (MP) ldf<N>(tw.w32, e, w); else load_weight_t<T, N>(tw, e, w);
  if (skip) {
#pragma unroll
    for (int i = 0; i < N; ++i) wn[i] = w[i];
  } else if (FLAVOR == APPLY_LAMB) {
    float g[N];
    ldf<N>(tw.aux0, e, g);
#pragma unroll
    for (int i = 0; i < N; ++i) wn[i] = __fsub_rn(w[i], __fmul_rn(sc[0], g[i]));
  } else if (FLAVOR == APPLY_LANS) {
    float tm[N], tg[N];
    ldf<N>(tw.aux1, e, tm);
    ldf<N>(tw.aux0, e, tg);
#pragma unroll
    for (int i = 0; i < N; ++i)
      wn[i] = __fsub_rn(w[i], __fadd_rn(__fmul_rn(sc[0], tm[i]), __fmul_rn(sc[1], tg[i])));
  } else {
    float g[N], mom[N], unused = 0.f;
    ldf<N>(tw.aux0, e, g);
    Hyper h;
    h.lr = sc[0]; h.wd = tw.wd; h.eta = 1.f;
    h.rescale = L.rescale; h.clip = L.clip; h.momentum = L.momentum;
    h.beta1 = 0.f; h.beta2 = 0.f; h.eps = 0.f;
    if (FLAVOR == APPLY_LARS_MOM) {
      ldf<N>(tw.s0, e, mom);
#pragma unroll
      for (int i = 0; i < N; ++i) wn[i] = update_one<OPT_SGD_MOM>(g[i], w[i], mom[i], unused, h);
      stf<N>(tw.s0, e, mom);
    } else {
#pragma unroll
      for (int i = 0; i < N; ++i) wn[i] = update_one<OPT_SGD>(g[i], w[i], unused, unused, h);
    }
  }
  if (MP && !skip) stf<N>(tw.w32, e, wn);
  const int m = tw.n_out;
  for (int j = 0; j < m; ++j) Packet<T, N>::store(tw.out[j], e, wn);
}

template <typename T, bool MP, int FLAVOR>
__global__ void __launch_bounds__(kNormThreads, 2)
kv_norm_apply_kernel(NormLaunch L) {
  __shared__ NormWork tw;
  __shared__ float red[kNormWarps];
  __shared__ float sc[2];
  const bool sync = L.sync.mode != SYNC_NONE;
  if (sync) barrier_start(L.sync);   // every rank's totals are complete
  bool skip = false;
  if (L.skip_nonfinite) {
    skip = launch_bad_total(L, red) > 0.f;
    if (skip && L.overflow_flag != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *L.overflow_flag = 1;
  }
  int cur = -1;
  for (int64_t c = blockIdx.x; c < L.total_chunks; c += gridDim.x) {
    const int lo = find_entry(L.chunk_prefix, L.nworks, c);
    if (lo != cur) {
      load_work(&tw, L.works + lo);
      cur = lo;
      if (threadIdx.x == 0 && !skip) apply_scalars<FLAVOR>(tw, L, sc);
      __syncthreads();
    }
    const int64_t ci = c - L.chunk_prefix[lo];
    const int64_t cb = tw.begin + ci * L.chunk_elems;
    const int64_t ce = (cb + L.chunk_elems < tw.end) ? cb + L.chunk_elems : tw.end;
    int64_t scalar_from = cb;
    if (tw.flags & 1) {
      const int64_t nvec = (ce - cb) / 4;
      for (int64_t v = threadIdx.x; v < nvec; v += blockDim.x)
        apply_elems<T, MP, FLAVOR, 4>(tw, cb + v * 4, L, sc, skip);
      scalar_from = cb + nvec * 4;
    }
    for (int64_t s = scalar_from + threadIdx.x; s < ce; s += blockDim.x)
      apply_elems<T, MP, FLAVOR, 1>(tw, s, L, sc, skip);
  }
  if (sync) barrier_end(L.sync, L.sync.mode == SYNC_WRITE_PEERS);
}

// ---------------------------------------------------------------------------
// stand-alone multi_sum_sq / multi_all_finite
// ---------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kNormThreads, 2)
kv_sumsq_kernel(const SumSqItem* items, const int64_t* prefix, int nitems, int64_t total_chunks, float scale,
                float* psum, int chunk_elems) {
  __shared__ float red[kNormWarps * 2];
  for (int64_t c = blockIdx.x; c < total_chunks; c += gridDim.x) {
    const int lo = find_entry(prefix, nitems, c);
    const T* x = reinterpret_cast<const T*>(items[lo].ptr);
    const int64_t cb = (c - prefix[lo]) * chunk_elems;
    const int64_t ce = (cb + chunk_elems < items[lo].n) ? cb + chunk_elems : items[lo].n;
    float p[2] = {0.f, 0.f};
    for (int64_t i = cb + threadIdx.x; i < ce; i += blockDim.x) {
      float v = Cvt<T>::to(x[i]);
      p[1] += not_finite(v) ? 1.0f : 0.0f;
      if (scale != 1.0f) v = __fmul_rn(v, scale);
      p[0] += v * v;
    }
    block_sums<2>(p, red, psum + c * 2);
  }
}

__global__ void __launch_bounds__(256)
kv_sumsq_finalize_kernel(const int64_t* prefix, const float* psum, float* out_sumsq, float* out_bad) {
  __shared__ float red[8 * 2];
  __shared__ float tot[2];
  const int64_t b = prefix[blockIdx.x], e = prefix[blockIdx.x + 1];
  float p[2] = {0.f, 0.f};
  for (int64_t i = b + threadIdx.x; i < e; i += blockDim.x) { p[0] += psum[i * 2]; p[1] += psum[i * 2 + 1]; }
  block_sums<2>(p, red, tot);
  if (threadIdx.x == 0) {
    if (out_sumsq) out_sumsq[blockIdx.x] = tot[0];
    if (out_bad) out_bad[blockIdx.x] = tot[1];
  }
}

__global__ void kv_all_finite_flag_kernel(const float* bad, int n, float* out, int init) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    float v = init ? 1.0f : out[0];
    for (int i = 0; i < n; ++i) if (bad[i] > 0.f) v = 0.0f;
    out[0] = v;
  }
}

// ---------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------
#define NORM_DISPATCH_T(dtype, mp, CALL)                                                       \
  do {                                                                                         \
    if ((dtype) == kFloat32 && !(mp)) { CALL(float, false); }                                  \
    else if ((dtype) == kFloat32) { CALL(float, true); }                                       \
    else if ((dtype) == kFloat16 && (mp)) { CALL(__half, true); }                              \
    else if ((dtype) == kBfloat16 && (mp)) { CALL(__nv_bfloat16, true); }                      \
    else return static_cast<int>(cudaErrorInvalidValue);                                       \
  } while (0)

int NormMaxGrid(int device) {
  static int cache[64] = {0};
  if (device >= 0 && device < 64 && cache[device] > 0) return cache[device];
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = kNumSms;
  int occ = 2, o = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, kv_norm_first_kernel<__half, true, false>, kNormThreads, 0) ==
          cudaSuccess && o > 0) occ = o < occ ? o : occ;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, kv_norm_mid_kernel<__half, true, NORM_LANS>, kNormThreads, 0) ==
          cudaSuccess && o > 0) occ = o < occ ? o : occ;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, kv_norm_apply_kernel<__half, true, APPLY_LARS_MOM>,
                                                    kNormThreads, 0) == cudaSuccess && o > 0) occ = o < occ ? o : occ;
  cudaGetLastError();
  int g = sms * occ;
  if (g > kMaxBlocks) g = kMaxBlocks;
  if (device >= 0 && device < 64) cache[device] = g;
  return g;
}

int LaunchNormFirst(const NormLaunch& L, int grad_only, cudaStream_t stream) {
  if (L.total_chunks <= 0) return 0;
#define CALL_FIRST(T, MP)                                                                       \
  if (grad_only) kv_norm_first_kernel<T, MP, true><<<L.grid, kNormThreads, 0, stream>>>(L);     \
  else kv_norm_first_kernel<T, MP, false><<<L.grid, kNormThreads, 0, stream>>>(L)
  NORM_DISPATCH_T(L.dtype, L.multi_precision, CALL_FIRST);
#undef CALL_FIRST
  return static_cast<int>(cudaGetLastError());
}

int LaunchNormFinalize(const NormLaunch& L, int nslots, int slot0, int slot1, int slot2, cudaStream_t stream) {
  if (L.nworks <= 0) return 0;
  kv_norm_finalize_kernel<<<L.nworks, 256, 0, stream>>>(L.works, L.chunk_prefix, nslots, slot0, slot1, slot2);
  return static_cast<int>(cudaGetLastError());
}

int LaunchNormMid(const NormLaunch& L, cudaStream_t stream) {
  if (L.total_chunks <= 0) return 0;
#define CALL_MID(T, MP)                                                                         \
  if (L.kind == NORM_LANS) kv_norm_mid_kernel<T, MP, NORM_LANS><<<L.grid, kNormThreads, 0, stream>>>(L); \
  else kv_norm_mid_kernel<T, MP, NORM_LAMB><<<L.grid, kNormThreads, 0, stream>>>(L)
  NORM_DISPATCH_T(L.dtype, L.multi_precision, CALL_MID);
#undef CALL_MID
  return static_cast<int>(cudaGetLastError());
}

int LaunchNormApply(const NormLaunch& L, cudaStream_t stream) {
  if (L.total_chunks <= 0) return 0;
#define CALL_APPLY(T, MP)                                                                                    \
  if (L.kind == NORM_LAMB) kv_norm_apply_kernel<T, MP, APPLY_LAMB><<<L.grid, kNormThreads, 0, stream>>>(L);   \
  else if (L.kind == NORM_LANS) kv_norm_apply_kernel<T, MP, APPLY_LANS><<<L.grid, kNormThreads, 0, stream>>>(L); \
  else if (L.has_momentum) kv_norm_apply_kernel<T, MP, APPLY_LARS_MOM><<<L.grid, kNormThreads, 0, stream>>>(L);  \
  else kv_norm_apply_kernel<T, MP, APPLY_LARS><<<L.grid, kNormThreads, 0, stream>>>(L)
  NORM_DISPATCH_T(L.dtype, L.multi_precision, CALL_APPLY);
#undef CALL_APPLY
  return static_cast<int>(cudaGetLastError());
}

int LaunchMultiSumSq(const SumSqItem* d_items, const int64_t* d_chunk_prefix, int nitems, int64_t total_chunks,
                     int dtype, float scale, float* d_psum, float* d_out_sumsq, float* d_out_bad, int chunk_elems,
                     cudaStream_t stream) {
  if (nitems <= 0) return 0;
  if (total_chunks > 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    const int cap = NormMaxGrid(dev);
    const int grid = static_cast<int>(total_chunks < cap ? total_chunks : cap);
    if (dtype == kFloat32)
      kv_sumsq_kernel<float><<<grid, kNormThreads, 0, stream>>>(d_items, d_chunk_prefix, nitems, total_chunks, scale,
                                                                d_psum, chunk_elems);
    else if (dtype == kFloat16)
      kv_sumsq_kernel<__half><<<grid, kNormThreads, 0, stream>>>(d_items, d_chunk_prefix, nitems, total_chunks, scale,
                                                                 d_psum, chunk_elems);
    else if (dtype == kBfloat16)
      kv_sumsq_kernel<__nv_bfloat16><<<grid, kNormThreads, 0, stream>>>(d_items, d_chunk_prefix, nitems, total_chunks,
                                                                        scale, d_psum, chunk_elems);
    else if (dtype == kFloat64)
      kv_sumsq_kernel<double><<<grid, kNormThreads, 0, stream>>>(d_items, d_chunk_prefix, nitems, total_chunks, scale,
                                                                 d_psum, chunk_elems);
    else
      return static_cast<int>(cudaErrorInvalidValue);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  kv_sumsq_finalize_kernel<<<nitems, 256, 0, stream>>>(d_chunk_prefix, d_psum, d_out_sumsq, d_out_bad);
  return static_cast<int>(cudaGetLastError());
}

int LaunchAllFiniteFlag(const float* d_bad, int n, float* d_out, int init, cudaStream_t stream) {
  kv_all_finite_flag_kernel<<<1, 32, 0, stream>>>(d_bad, n, d_out, init);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace mxkv
