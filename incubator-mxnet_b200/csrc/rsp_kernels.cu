// rsp_kernels.cu -- row_sparse reduce (+ lazy optimizer) and row_sparse_pull kernels.
//
// Reference: ElementwiseSumRspImpl (src/ndarray/ndarray_function.cu:104-190) marks a flag per row
// of the FULL table (1 M flags for a 1 M-row embedding), prefix-sums all of them with cub, copies
// the count to the host and synchronises, then adds the inputs one kernel at a time; the update
// is a further op (SGDDnsRspKernel / AdamDnsRspDnsKernel, optimizer_op-inl.h:414-465,1305-1360);
// row_sparse_pull = cub sort + unique + D2H count + sync (src/kvstore/kvstore_utils.cu:44-97)
// followed by a zero-fill + gather (sparse_retain-inl.h:262-322).
//
// Here everything is proportional to the number of non-zero rows, nothing touches the host:
//   K1 first[s][r]  : is source s the first one that contains id idx_s[r]?   (binary searches)
//   K2 pf[s][*]     : per-source exclusive scan of `first`                    (one block per source)
//   K3 out_idx      : rank(id) = sum_s pf[s][lower_bound(idx_s, id)] -> sorted unique union
//   K4 rows         : one warp per union row: gather-sum the <= n contributions in source order
//                     (zero-initialised accumulator, like the reference), apply the lazy
//                     SGD / SGD-momentum / Adam update to that row of the dense table, and/or
//                     materialise the merged row_sparse value.
// The row counts stay on the device (every kernel reads nnz through a pointer).
#include "rsp_kernels.h"
#include "rsp_math.h"
#include "device_utils.cuh"

namespace mxkv {

namespace {

__device__ __forceinline__ int64_t lower_bound_i64(const int64_t* a, int64_t n, int64_t x) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void rsp_first_kernel(RspSources S, int32_t* first, int64_t cap) {
  const int s = blockIdx.y;
  const int64_t nnz = *S.nnz[s];
  const int64_t* idx = S.idx[s];
  for (int64_t r = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; r < nnz;
       r += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t id = idx[r];
    int f = 1;
    for (int t = 0; t < s && f; ++t) {
      const int64_t nt = *S.nnz[t];
      const int64_t p = lower_bound_i64(S.idx[t], nt, id);
      if (p < nt && S.idx[t][p] == id) f = 0;
    }
    first[s * cap + r] = f;
  }
}

// one block per source: exclusive scan of first[s][0..nnz) into pf[s][0..nnz], pf[s][nnz] = total
__global__ void rsp_scan_kernel(RspSources S, const int32_t* first, int32_t* pf, int64_t cap) {
  __shared__ int32_t warp_sums[32];
  __shared__ int32_t carry;
  const int s = blockIdx.x;
  const int64_t nnz = *S.nnz[s];
  const int32_t* f = first + s * cap;
  int32_t* out = pf + s * (cap + 1);
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  for (int64_t base = 0; base < nnz; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    const int32_t v = i < nnz ? f[i] : 0;
    int32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int32_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int32_t w = lane < nwarp ? warp_sums[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      warp_sums[lane] = w;   // inclusive over warps
    }
    __syncthreads();
    const int32_t before = carry + (warp > 0 ? warp_sums[warp - 1] : 0);
    if (i < nnz) out[i] = before + x - v;   // exclusive
    __syncthreads();
    if (threadIdx.x == 0) carry += warp_sums[nwarp - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[nnz] = carry;
}

__global__ void rsp_rank_kernel(RspSources S, const int32_t* first, const int32_t* pf, int64_t cap,
                                int64_t* out_idx, int64_t* d_nnz_out) {
  const int s = blockIdx.y;
  const int64_t nnz = *S.nnz[s];
  if (s == 0 && blockIdx.x == 0 && threadIdx.x == 0) {
    int64_t tot = 0;
    for (int t = 0; t < S.n; ++t) tot += pf[t * (cap + 1) + *S.nnz[t]];
    *d_nnz_out = tot;
  }
  for (int64_t r = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; r < nnz;
       r += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    if (!first[s * cap + r]) continue;
    const int64_t id = S.idx[s][r];
    int64_t rank = 0;
    for (int t = 0; t < S.n; ++t) {
      const int64_t p = (t == s) ? r : lower_bound_i64(S.idx[t], *S.nnz[t], id);
      rank += pf[t * (cap + 1) + p];
    }
    out_idx[rank] = id;
  }
}

// One warp per union row.  VEC = true: row_len % 4 == 0 and all pointers 16-byte aligned.
template <int OPT, bool VEC>
__global__ void __launch_bounds__(256)
rsp_rows_kernel(RspSources S, RspRowArgs A) {
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  const int64_t nrows = *A.d_nnz_out;
  const int64_t L = A.row_len;
  for (int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x >> 5) + (threadIdx.x >> 5); j < nrows;
       j += warps_total) {
    const int64_t id = A.out_idx[j];
    // positions of this row in every source (lane t searches source t; n <= 16 <= 32)
    int64_t mypos = -1;
    if (lane < S.n) {
      const int64_t nt = *S.nnz[lane];
      const int64_t p = lower_bound_i64(S.idx[lane], nt, id);
      if (p < nt && S.idx[lane][p] == id) mypos = p;
    }
    constexpr int W = VEC ? 4 : 1;
    // every lane runs every iteration (the shuffles below need the full warp); `act` masks the tail
    for (int64_t c0 = 0; c0 < L; c0 += 32 * W) {
      const int64_t c = c0 + static_cast<int64_t>(lane) * W;
      const bool act = c < L;
      float acc[W];
#pragma unroll
      for (int i = 0; i < W; ++i) acc[i] = 0.f;          // set_zero(out) then += inputs in order
      for (int t = 0; t < S.n; ++t) {
        const int64_t p = __shfl_sync(0xffffffffu, mypos, t);
        if (p < 0 || !act) continue;
        const float* src = S.val[t] + p * L + c;
        if (VEC) {
          const float4 v = *reinterpret_cast<const float4*>(src);
          acc[0] = __fadd_rn(acc[0], v.x); acc[1 % W] = __fadd_rn(acc[1 % W], v.y);
          acc[2 % W] = __fadd_rn(acc[2 % W], v.z); acc[3 % W] = __fadd_rn(acc[3 % W], v.w);
        } else {
          acc[0] = __fadd_rn(acc[0], src[0]);
        }
      }
      if (!act) continue;
      if (A.out_val != nullptr) {
        float* o = A.out_val + j * L + c;
#pragma unroll
        for (int i = 0; i < W; ++i) o[i] = acc[i];
      }
      if (OPT != OPT_NONE || A.assign) {
        float* w = A.table + id * L + c;
#pragma unroll
        for (int i = 0; i < W; ++i) {
          if (OPT == OPT_NONE) { w[i] = acc[i]; continue; }
          w[i] = rsp_lazy_update<OPT>(acc[i], w[i], id * L + c + i, A);
        }
      }
    }
  }
}

// ---- row_sparse_pull -----------------------------------------------------------------------
// single-block bitonic sort + unique of up to kUniqueMax int64 ids in shared memory
constexpr int kUniqueMax = 16384;

__device__ __forceinline__ void unique_block(const int64_t* in, int64_t n, int64_t* out, int64_t* d_count, int64_t* sm) {
  // fast path: ids that are already strictly increasing (e.g. the index array of a row_sparse
  // gradient) need neither the sort nor the compaction
  {
    int ok = 1;
    for (int64_t i = threadIdx.x; i + 1 < n; i += blockDim.x) ok &= (in[i] < in[i + 1]) ? 1 : 0;
    if (__syncthreads_and(ok)) {
      for (int64_t i = threadIdx.x; i < n; i += blockDim.x) out[i] = in[i];
      if (threadIdx.x == 0) *d_count = n;
      return;
    }
  }
  int64_t npad = 1;
  while (npad < n) npad <<= 1;
  for (int64_t i = threadIdx.x; i < npad; i += blockDim.x) sm[i] = i < n ? in[i] : INT64_MAX;
  __syncthreads();
  for (int64_t k = 2; k <= npad; k <<= 1) {
    for (int64_t j = k >> 1; j > 0; j >>= 1) {
      for (int64_t i = threadIdx.x; i < npad; i += blockDim.x) {
        const int64_t l = i ^ j;
        if (l > i) {
          const bool up = (i & k) == 0;
          const int64_t a = sm[i], b = sm[l];
          if ((a > b) == up) { sm[i] = b; sm[l] = a; }
        }
      }
      __syncthreads();
    }
  }
  // unique: flag + block-wide exclusive scan in chunks
  __shared__ int32_t warp_sums[32];
  __shared__ int32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  for (int64_t base = 0; base < n; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    const int32_t v = (i < n && (i == 0 || sm[i] != sm[i - 1])) ? 1 : 0;
    int32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int32_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int32_t w = lane < nwarp ? warp_sums[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      warp_sums[lane] = w;
    }
    __syncthreads();
    const int32_t before = carry + (warp > 0 ? warp_sums[warp - 1] : 0);
    if (v) out[before + x - 1] = sm[i];
    __syncthreads();
    if (threadIdx.x == 0) carry += warp_sums[nwarp - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) *d_count = carry;
}

__global__ void __launch_bounds__(1024)
rsp_unique_kernel(const int64_t* in, int64_t n, int64_t* out, int64_t* d_count) {
  extern __shared__ int64_t sm[];
  unique_block(in, n, out, d_count, sm);
}

// ---- large id lists (> kUniqueMax): bitonic sort in global memory, one launch per (k, j) step, then
// a single-block chunked compaction.  Rare path (the reference sorts with cub); correctness first.
__global__ void rsp_pad_kernel(const int64_t* in, int64_t n, int64_t* buf, int64_t npad) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < npad;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    buf[i] = i < n ? in[i] : INT64_MAX;
}

__global__ void rsp_bitonic_step_kernel(int64_t* buf, int64_t npad, int64_t k, int64_t j) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < npad;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t l = i ^ j;
    if (l > i) {
      const bool up = (i & k) == 0;
      const int64_t a = buf[i], b = buf[l];
      if ((a > b) == up) { buf[i] = b; buf[l] = a; }
    }
  }
}

__global__ void __launch_bounds__(1024)
rsp_compact_sorted_kernel(const int64_t* sorted, int64_t n, int64_t* out, int64_t* d_count) {
  __shared__ int32_t warp_sums[32];
  __shared__ int64_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  for (int64_t base = 0; base < n; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    const int32_t v = (i < n && (i == 0 || sorted[i] != sorted[i - 1])) ? 1 : 0;
    int32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int32_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int32_t w = lane < nwarp ? warp_sums[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      warp_sums[lane] = w;
    }
    __syncthreads();
    const int64_t before = carry + (warp > 0 ? warp_sums[warp - 1] : 0);
    if (v) out[before + x - 1] = sorted[i];
    __syncthreads();
    if (threadIdx.x == 0) carry += warp_sums[nwarp - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) *d_count = carry;
}

// out_val[j, :] = table[ids[j], :]  (the stored value is dense-backed: SparseRetain's "input rsp
// is dense" branch, sparse_retain-inl.h:286-311); one warp per row
__global__ void __launch_bounds__(256)
rsp_gather_kernel(const float* table, const int64_t* ids, const int64_t* d_count, int64_t L, float* out_val,
                  int64_t* out_idx, int vec) {
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  const int64_t n = *d_count;
  for (int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x >> 5) + (threadIdx.x >> 5); j < n; j += warps_total) {
    const int64_t id = ids[j];
    if (lane == 0 && out_idx != ids) out_idx[j] = id;
    const float* src = table + id * L;
    float* dst = out_val + j * L;
    if (vec) {
      for (int64_t c = lane * 4; c < L; c += 128)
        *reinterpret_cast<float4*>(dst + c) = *reinterpret_cast<const float4*>(src + c);
    } else {
      for (int64_t c = lane; c < L; c += 32) dst[c] = src[c];
    }
  }
}

// table[idx[r], :] = val[r, :]   (initialisation of the dense-backed store from a row_sparse value)
__global__ void __launch_bounds__(256)
rsp_scatter_kernel(float* table, const int64_t* idx, const int64_t* d_nnz, int64_t L, const float* val) {
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  const int64_t n = *d_nnz;
  for (int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x >> 5) + (threadIdx.x >> 5); j < n; j += warps_total) {
    float* dst = table + idx[j] * L;
    const float* src = val + j * L;
    for (int64_t c = lane; c < L; c += 32) dst[c] = src[c];
  }
}

// ---------------------------------------------------------------------------------------------------
// Fused row_sparse push: ONE launch for "publish my gradient to the peers, union of the ranks' row ids, gather-sum
// in source order, lazy optimizer update of the touched rows" (round 1: two rendezvous kernels + two staging
// copies + first / scan / rank / rows = up to nine launches, and every binary search of a peer's id list crossed
// NVLink one dependent load at a time).  Phases, separated by the grid-wide barrier of device_utils.cuh:
//   P0 (one process per GPU)  copy this rank's (ids, rows, count) into its peer-mapped staging area   | cross-GPU barrier
//   P1 (any remote source)    pull every source's id list into LOCAL memory with coalesced reads       | local barrier
//   P2                        one warp per candidate row (s, r): lane t searches source t's (local) id list; the
//                             candidate is processed iff no source before s holds the id (so every union row is
//                             summed exactly once, by its first holder's candidate) -- contributions added in
//                             source order onto a zero accumulator (ndarray_function.cu:176-187), then the lazy
//                             update of that row of the table (rsp_math.h).  No sorted union is materialised:
//                             nothing downstream of a fused update needs it.
//   P3 (one process per GPU)  cross-GPU barrier: no peer still reads this rank's staging area when it returns
// ---------------------------------------------------------------------------------------------------
template <int OPT, bool VEC>
__global__ void __launch_bounds__(256)
rsp_push_fused_kernel(RspSources S, RspRowArgs A, RspStage St, SyncArgs sync) {
  __shared__ int64_t s_nnz[kMaxSrc + 1];     // exclusive prefix of the sources' row counts
  const int lane = threadIdx.x & 31;
  const int64_t nthreads = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const int64_t gtid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t L = A.row_len;

  if (St.publish) {                                    // ---- P0
    const int64_t nnz = St.src_nnz;
    for (int64_t i = gtid; i < nnz; i += nthreads) St.dst_idx[i] = St.src_idx[i];
    if (VEC) {
      const int64_t nv = nnz * L / 4;
      const float4* sv = reinterpret_cast<const float4*>(St.src_val);
      float4* dv = reinterpret_cast<float4*>(St.dst_val);
      for (int64_t i = gtid; i < nv; i += nthreads) dv[i] = sv[i];
    } else {
      for (int64_t i = gtid; i < nnz * L; i += nthreads) St.dst_val[i] = St.src_val[i];
    }
    if (gtid == 0) *St.dst_nnz = nnz;
    grid_barrier(sync, true);
  }

  __shared__ int64_t s_cnt[kMaxSrc];
  if (threadIdx.x < S.n)                                                 // (peer memory: n round trips in parallel)
    s_cnt[threadIdx.x] = St.nnz_by_value ? St.nnz_val[threadIdx.x] : *S.nnz[threadIdx.x];
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t run = 0;
    for (int t = 0; t < S.n; ++t) { s_nnz[t] = run; run += s_cnt[t]; }
    s_nnz[S.n] = run;
  }
  __syncthreads();

  if (St.localize) {                                   // ---- P1
    for (int t = 0; t < S.n; ++t) {
      const int64_t nt = s_nnz[t + 1] - s_nnz[t];
      int64_t* dst = St.lidx + static_cast<int64_t>(t) * St.lcap;
      for (int64_t i = gtid; i < nt; i += nthreads) dst[i] = S.idx[t][i];
    }
    grid_barrier(sync, false);
  }

  // ---- P2
  const int64_t total = s_nnz[S.n];
  const int64_t warps_total = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  for (int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x >> 5) + (threadIdx.x >> 5); j < total; j += warps_total) {
    int s = 0;
    while (s + 1 < S.n && j >= s_nnz[s + 1]) ++s;
    const int64_t r = j - s_nnz[s];
    const int64_t* my_ids = St.localize ? St.lidx + static_cast<int64_t>(s) * St.lcap : S.idx[s];
    const int64_t id = my_ids[r];
    int64_t mypos = -1;
    if (lane < S.n) {
      if (lane == s) {
        mypos = r;
      } else {
        const int64_t nt = s_nnz[lane + 1] - s_nnz[lane];
        const int64_t* ids_t = St.localize ? St.lidx + static_cast<int64_t>(lane) * St.lcap : S.idx[lane];
        const int64_t p = lower_bound_i64(ids_t, nt, id);
        if (p < nt && ids_t[p] == id) mypos = p;
      }
    }
    const unsigned holders = __ballot_sync(0xffffffffu, mypos >= 0);
    if (holders & ((1u << s) - 1u)) continue;          // an earlier source holds this id: its candidate does the row
    constexpr int W = VEC ? 4 : 1;
    for (int64_t c0 = 0; c0 < L; c0 += 32 * W) {
      const int64_t c = c0 + static_cast<int64_t>(lane) * W;
      const bool act = c < L;
      float acc[W];
#pragma unroll
      for (int i = 0; i < W; ++i) acc[i] = 0.f;
      for (int t = s; t < S.n; ++t) {
        const int64_t p = __shfl_sync(0xffffffffu, mypos, t);
        if (p < 0 || !act) continue;
        const float* src = S.val[t] + p * L + c;
        if (VEC) {
          const float4 v = *reinterpret_cast<const float4*>(src);
          acc[0] = __fadd_rn(acc[0], v.x); acc[1 % W] = __fadd_rn(acc[1 % W], v.y);
          acc[2 % W] = __fadd_rn(acc[2 % W], v.z); acc[3 % W] = __fadd_rn(acc[3 % W], v.w);
        } else {
          acc[0] = __fadd_rn(acc[0], src[0]);
        }
      }
      if (!act) continue;
      float* w = A.table + id * L + c;
#pragma unroll
      for (int i = 0; i < W; ++i) w[i] = rsp_lazy_update<OPT>(acc[i], w[i], id * L + c + i, A);
    }
  }

  if (St.publish) grid_barrier(sync, true);            // ---- P3
}

// ---------------------------------------------------------------------------------------------------
// Fused row_sparse_pull: unique (block 0: already-increasing fast path, else bitonic sort + compaction in shared
// memory) | grid barrier | one warp per row gather -- one launch instead of two.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
rsp_pull_fused_kernel(const float* table, const int64_t* in, int64_t n, int64_t* out_idx, int64_t* d_count, int64_t L,
                      float* out_val, int vec, SyncArgs sync) {
  extern __shared__ int64_t sm[];
  if (blockIdx.x == 0) unique_block(in, n, out_idx, d_count, sm);
  grid_barrier(sync, false);
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  const int64_t cnt = *d_count;
  for (int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x >> 5) + (threadIdx.x >> 5); j < cnt; j += warps_total) {
    const int64_t id = out_idx[j];
    const float* src = table + id * L;
    float* dst = out_val + j * L;
    if (vec) {
      for (int64_t c = lane * 4; c < L; c += 128)
        *reinterpret_cast<float4*>(dst + c) = *reinterpret_cast<const float4*>(src + c);
    } else {
      for (int64_t c = lane; c < L; c += 32) dst[c] = src[c];
    }
  }
}

__global__ void rsp_set_i64_kernel(int64_t* p, int64_t v) { *p = v; }

}  // namespace

static int grid_for(int64_t items, int per_block) {
  int64_t g = (items + per_block - 1) / per_block;
  if (g < 1) g = 1;
  if (g > kMaxBlocks) g = kMaxBlocks;
  return static_cast<int>(g);
}

int LaunchRspSum(const RspSources& S, const RspRowArgs& A, int32_t* first, int32_t* pf, int64_t cap,
                 cudaStream_t stream) {
  if (S.n < 1 || S.n > kMaxSrc) return static_cast<int>(cudaErrorInvalidValue);
  dim3 g1(grid_for(cap, 256), S.n);
  rsp_first_kernel<<<g1, 256, 0, stream>>>(S, first, cap);
  rsp_scan_kernel<<<S.n, 1024, 0, stream>>>(S, first, pf, cap);
  rsp_rank_kernel<<<g1, 256, 0, stream>>>(S, first, pf, cap, A.out_idx, A.d_nnz_out);
  const int64_t maxrows = cap * S.n;
  const int grid = grid_for(maxrows, 8);
  const bool vec = A.vec != 0;
#define RSP_ROWS(OPT)                                                                   \
  if (vec) rsp_rows_kernel<OPT, true><<<grid, 256, 0, stream>>>(S, A);                  \
  else rsp_rows_kernel<OPT, false><<<grid, 256, 0, stream>>>(S, A)
  switch (A.opt) {
    case OPT_NONE: RSP_ROWS(OPT_NONE); break;
    case OPT_SGD: RSP_ROWS(OPT_SGD); break;
    case OPT_SGD_MOM: RSP_ROWS(OPT_SGD_MOM); break;
    case OPT_ADAM: RSP_ROWS(OPT_ADAM); break;
    default: return static_cast<int>(cudaErrorInvalidValue);
  }
#undef RSP_ROWS
  return static_cast<int>(cudaGetLastError());
}

static int resident_grid(int device, const void* fn, int threads, size_t smem) {
  int prev = -1;
  cudaGetDevice(&prev);
  if (prev != device) cudaSetDevice(device);
  int occ = 0, sms = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags(&occ, fn, threads, smem, cudaOccupancyDefault);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  if (prev >= 0 && prev != device) cudaSetDevice(prev);
  if (e != cudaSuccess || occ < 1 || sms < 1) { cudaGetLastError(); return 0; }
  const int64_t g = static_cast<int64_t>(occ) * sms;
  return static_cast<int>(g > kMaxBlocks ? kMaxBlocks : g);
}

int LaunchRspPushFused(int device, const RspSources& S, const RspRowArgs& A, const RspStage& St, const SyncArgs& sync,
                       int64_t est_rows, cudaStream_t stream) {
  if (S.n < 1 || S.n > kMaxSrc || A.out_val != nullptr || A.assign) return static_cast<int>(cudaErrorInvalidValue);
  typedef void (*Fn)(RspSources, RspRowArgs, RspStage, SyncArgs);
  Fn fn = nullptr;
  const bool vec = A.vec != 0;
  switch (A.opt) {
    case OPT_SGD: fn = vec ? rsp_push_fused_kernel<OPT_SGD, true> : rsp_push_fused_kernel<OPT_SGD, false>; break;
    case OPT_SGD_MOM: fn = vec ? rsp_push_fused_kernel<OPT_SGD_MOM, true> : rsp_push_fused_kernel<OPT_SGD_MOM, false>; break;
    case OPT_ADAM: fn = vec ? rsp_push_fused_kernel<OPT_ADAM, true> : rsp_push_fused_kernel<OPT_ADAM, false>; break;
    default: return static_cast<int>(cudaErrorInvalidValue);
  }
  // the grid barrier needs every block resident; more blocks than candidate rows / 8 warps would only spin
  static int cap[64][8] = {{0}};
  int& c = cap[device & 63][(A.opt & 3) * 2 + (vec ? 1 : 0)];
  if (c == 0) c = resident_grid(device, reinterpret_cast<const void*>(fn), 256, 0);
  if (c < 1) return static_cast<int>(cudaErrorLaunchOutOfResources);
  int64_t want = (est_rows + 7) / 8;
  if (St.publish) want = std::max<int64_t>(want, kNumSms);      // the staging copy wants the whole machine
  // two blocks per SM are plenty for a gather, and every block more makes the in-kernel barriers dearer
  const int grid = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(c, 2 * kNumSms), want)));
  fn<<<grid, 256, 0, stream>>>(S, A, St, sync);
  return static_cast<int>(cudaGetLastError());
}

int LaunchRspPullFused(int device, const float* table, const int64_t* ids, int64_t n, int64_t* out_idx, int64_t* d_count,
                       int64_t L, float* out_val, int vec, const SyncArgs& sync, cudaStream_t stream) {
  if (n < 1 || n > kUniqueMax) return static_cast<int>(cudaErrorInvalidValue);
  int64_t npad = 1;
  while (npad < n) npad <<= 1;
  const size_t smem = static_cast<size_t>(npad) * sizeof(int64_t);
  static bool attr_set[64] = {false};
  if (!attr_set[device & 63]) {
    int prev = -1;
    cudaGetDevice(&prev);
    if (prev != device) cudaSetDevice(device);
    cudaFuncSetAttribute(rsp_pull_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         kUniqueMax * static_cast<int>(sizeof(int64_t)));
    if (prev >= 0 && prev != device) cudaSetDevice(prev);
    attr_set[device & 63] = true;
  }
  const int c = resident_grid(device, reinterpret_cast<const void*>(rsp_pull_fused_kernel), 1024, smem);
  if (c < 1) return static_cast<int>(cudaErrorLaunchOutOfResources);
  const int grid = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(c, (n + 31) / 32)));
  rsp_pull_fused_kernel<<<grid, 1024, smem, stream>>>(table, ids, n, out_idx, d_count, L, out_val, vec, sync);
  return static_cast<int>(cudaGetLastError());
}

int RspUniqueMax() { return kUniqueMax; }

int LaunchRspUnique(const int64_t* ids, int64_t n, int64_t* out, int64_t* d_count, cudaStream_t stream) {
  if (n > kUniqueMax) {
    int64_t npad = 1;
    while (npad < n) npad <<= 1;
    int64_t* buf = nullptr;
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&buf), static_cast<size_t>(npad) * 8, stream);
    if (e != cudaSuccess) return static_cast<int>(e);
    const int grid = grid_for(npad, 256);
    rsp_pad_kernel<<<grid, 256, 0, stream>>>(ids, n, buf, npad);
    for (int64_t k = 2; k <= npad; k <<= 1)
      for (int64_t j = k >> 1; j > 0; j >>= 1) rsp_bitonic_step_kernel<<<grid, 256, 0, stream>>>(buf, npad, k, j);
    rsp_compact_sorted_kernel<<<1, 1024, 0, stream>>>(buf, n, out, d_count);
    cudaFreeAsync(buf, stream);
    return static_cast<int>(cudaGetLastError());
  }
  if (n == 0) {
    rsp_set_i64_kernel<<<1, 1, 0, stream>>>(d_count, 0);
    return static_cast<int>(cudaGetLastError());
  }
  int64_t npad = 1;
  while (npad < n) npad <<= 1;
  const size_t smem = static_cast<size_t>(npad) * sizeof(int64_t);
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(rsp_unique_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         kUniqueMax * static_cast<int>(sizeof(int64_t)));
    attr_set = true;
  }
  rsp_unique_kernel<<<1, 1024, smem, stream>>>(ids, n, out, d_count);
  return static_cast<int>(cudaGetLastError());
}

int LaunchRspGather(const float* table, const int64_t* ids, const int64_t* d_count, int64_t max_rows, int64_t L,
                    float* out_val, int64_t* out_idx, int vec, cudaStream_t stream) {
  rsp_gather_kernel<<<grid_for(max_rows, 8), 256, 0, stream>>>(table, ids, d_count, L, out_val, out_idx, vec);
  return static_cast<int>(cudaGetLastError());
}

int LaunchRspScatter(float* table, const int64_t* idx, const int64_t* d_nnz, int64_t max_rows, int64_t L,
                     const float* val, cudaStream_t stream) {
  rsp_scatter_kernel<<<grid_for(max_rows, 8), 256, 0, stream>>>(table, idx, d_nnz, L, val);
  return static_cast<int>(cudaGetLastError());
}

// row ids of any real dtype -> int64 (KVStoreLocal::Unique copies them with ndarray::Copy, which casts:
// src/kvstore/kvstore_local.h:507-512; the reference's tests pass float32 ids)
template <typename T>
__global__ void rsp_cast_ids_kernel(const T* src, int64_t* dst, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = static_cast<int64_t>(src[i]);
}

int LaunchCastIdsToI64(const void* src, int dtype, int64_t* dst, int64_t n, cudaStream_t stream) {
  if (n <= 0) return 0;
  const int threads = 256;
  const int grid = static_cast<int>(std::min<int64_t>((n + threads - 1) / threads, kMaxBlocks));
  switch (dtype) {
    case kFloat32: rsp_cast_ids_kernel<float><<<grid, threads, 0, stream>>>(static_cast<const float*>(src), dst, n); break;
    case kFloat64: rsp_cast_ids_kernel<double><<<grid, threads, 0, stream>>>(static_cast<const double*>(src), dst, n); break;
    case kInt32: rsp_cast_ids_kernel<int32_t><<<grid, threads, 0, stream>>>(static_cast<const int32_t*>(src), dst, n); break;
    case kInt64: rsp_cast_ids_kernel<int64_t><<<grid, threads, 0, stream>>>(static_cast<const int64_t*>(src), dst, n); break;
    default: return static_cast<int>(cudaErrorInvalidValue);
  }
  return static_cast<int>(cudaGetLastError());
}

int LaunchSetI64(int64_t* p, int64_t v, cudaStream_t stream) {
  rsp_set_i64_kernel<<<1, 1, 0, stream>>>(p, v);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace mxkv
