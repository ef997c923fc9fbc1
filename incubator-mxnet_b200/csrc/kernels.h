// kernels.h -- device work descriptors and launcher entry points shared between
// the host runtime (engine.cc) and the sm_90a kernels (kernels.cu).
//
// One launch of the dense kernel processes a *work list*: every entry is one key
// (or the shard of a key this rank owns) with up to kMaxSrc gradient sources and
// up to kMaxOut destinations.  Sources/destinations are plain global pointers:
// local HBM, or another GPU's HBM mapped over NVLink (cudaDeviceEnablePeerAccess
// in single-process mode, cudaIpcOpenMemHandle in one-process-per-GPU mode).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

namespace mxkv {

constexpr int kMaxSrc = 16;      // values per key in one push (reference tests use 4; 8 GPUs => 8)
constexpr int kMaxOut = 24;      // n store replicas + n user outputs + merge buffers
constexpr int kMaxRanks = 8;     // one NVSwitch domain
constexpr int kNumSms = 132;     // H100 SXM; launches query the device, this is the fallback
constexpr int kMaxBlocks = kNumSms * 8;
constexpr int kChunkElems = 8192;   // default elements per scheduling chunk (MXKV_B200_CHUNK)

// mshadow type flags, 3rdparty/mshadow/mshadow/base.h:352-366
enum DType : int {
  kFloat32 = 0, kFloat64 = 1, kFloat16 = 2, kUint8 = 3, kInt32 = 4, kInt8 = 5, kInt64 = 6,
  kBool = 7, kInt16 = 8, kUint16 = 9, kUint32 = 10, kUint64 = 11, kBfloat16 = 12
};

enum OptKind : int {
  OPT_NONE = 0,     // out = sum(src)                        (push without updater / allreduce)
  OPT_SGD = 1,      // SGDKernel / MP_SGDKernel              optimizer_op-inl.h:377-390,642-658
  OPT_SGD_MOM = 2,  // SGDMomKernel / MP_SGDMomKernel        optimizer_op-inl.h:590-606,681-701
  OPT_ADAM = 3,     // AdamUpdateKernel                      optimizer_op-inl.h:1246-1269
  OPT_ADAMW = 4,    // MPAdamWKernel                         contrib/adamw-inl.h:101-124
  OPT_TEST = 5,     // mx.optimizer.Test                     python/mxnet/optimizer/optimizer.py:570-577
  // standard (non-lazy) updates of a dense weight with a row_sparse gradient, applied to the
  // densified gradient (absent rows = 0); arithmetic of the reference's *Std* sparse kernels
  OPT_SGD_STD = 6,  // SGDUpdateDnsRspImpl, lazy_update=false: w*(1-lr*wd) then w - lr*g   optimizer_op-inl.h:471-515
  OPT_ADAM_STD = 7, // AdamStdDnsRspDnsKernel: (1-beta2)*square(g)                          optimizer_op.cu:125-152
  // layer-wise adaptive optimizers: need per-tensor norms, run as a launch sequence (norm_kernels.h)
  OPT_LAMB = 8,     // multi_lamb_update / multi_mp_lamb_update   contrib/multi_lamb.cc:36-120
  OPT_LANS = 9,     // multi_lans_update / multi_mp_lans_update   contrib/multi_lans.cc:36-130
  OPT_LARS = 10,    // LARS._get_lars + (mp_)sgd(_mom)_update     python/mxnet/optimizer/lars.py:117-133,244-275
  OPT_NAG = 11,     // NAGMomKernel / MP_NAGMomKernel        optimizer_op-inl.h:1029-1044,1066-1090
  OPT_ADABELIEF = 12, // MultiMPAdaBeliefKernel              contrib/adabelief-inl.h:354-384
  OPT_RMSPROP = 13,   // RMSPropUpdateKernel                 optimizer_op-inl.h:2005-2031
  OPT_RMSPROP_CENTERED = 14, // RMSPropAlexUpdateKernel      optimizer_op-inl.h:1905-1939
  OPT_SIGNSGD = 15,   // SignSGDKernel                       optimizer_op-inl.h:2293-2305
  OPT_SIGNUM = 16,    // SignumKernel                        optimizer_op-inl.h:2361-2379
  OPT_FTML = 17,      // FTMLKernel                          optimizer_op-inl.h:1159-1177
  // no reference operator: the optimizer class's own `step`, one NDArray operation per rounding
  OPT_ADAMAX = 18,    // Adamax.step                         python/mxnet/optimizer/adamax.py:74-111
  OPT_ADADELTA = 19,  // AdaDelta.step                       python/mxnet/optimizer/adadelta.py:72-111
  OPT_NADAM = 20      // Nadam.step                          python/mxnet/optimizer/nadam.py:74-124
};
constexpr int kNumOptKinds = OPT_NADAM + 1;   // one past the last kind: the size of tables indexed by kind
inline bool IsNormOpt(int kind) { return kind == OPT_LAMB || kind == OPT_LANS || kind == OPT_LARS; }

// The fp32 state arrays an element-wise kind streams through update_one: s0 (momentum / mean / RMSProp var;
// centered RMSProp: mean; Signum: the negated momentum; FTML: d; Adamax: mean; AdaDelta: acc_g; Nadam: mean), s1
// (variance; FTML: v; Adamax: the max-norm u; AdaDelta: acc_delta; Nadam: var), s2 (centered RMSProp: momentum; FTML: z) -- the tuple order of the
// reference's create_state.  Every dense kernel loads and stores exactly
// these, and the staged kernel counts them among its staged arrays.  The layer-wise adaptive kinds keep their state
// rules with their launch sequence (KVStore::EnsureState).
__host__ __device__ constexpr bool OptHasS0(int kind) {
  return kind == OPT_SGD_MOM || kind == OPT_ADAM || kind == OPT_ADAMW || kind == OPT_ADAM_STD || kind == OPT_NAG ||
         kind == OPT_ADABELIEF || kind == OPT_RMSPROP || kind == OPT_RMSPROP_CENTERED || kind == OPT_SIGNUM ||
         kind == OPT_FTML || kind == OPT_ADAMAX || kind == OPT_ADADELTA || kind == OPT_NADAM;
}
__host__ __device__ constexpr bool OptHasS1(int kind) {
  return kind == OPT_ADAM || kind == OPT_ADAMW || kind == OPT_ADAM_STD || kind == OPT_ADABELIEF ||
         kind == OPT_RMSPROP_CENTERED || kind == OPT_FTML || kind == OPT_ADAMAX || kind == OPT_ADADELTA ||
         kind == OPT_NADAM;
}
__host__ __device__ constexpr bool OptHasS2(int kind) { return kind == OPT_RMSPROP_CENTERED || kind == OPT_FTML; }
// The fp32 arrays a kind streams next to its gradients: the weight (every kind but OPT_NONE) and its state arrays.
// The staged kernel stages exactly these per tile.
__host__ __device__ constexpr int OptStreams(int kind) {
  return (kind != OPT_NONE ? 1 : 0) + (OptHasS0(kind) ? 1 : 0) + (OptHasS1(kind) ? 1 : 0) + (OptHasS2(kind) ? 1 : 0);
}
// The kinds whose per-thread kernel also has the two-packets-in-flight variant (DenseLaunch::small_n): only these
// stay inside the 64 registers that keep two blocks of 512 threads resident with it.
__host__ __device__ constexpr bool OptHasSmallN(int kind) {
  return kind == OPT_NONE || kind == OPT_SGD || kind == OPT_TEST;
}

// The element-wise kinds: every dense kernel (per-thread, staged, multicast, tree) is instantiated for each of them,
// with and without an fp32 master weight.  OPT_NONE and the float32 per-thread-only *_STD kinds are selected apart.
// Dispatch<R>(opt, f) returns f(std::integral_constant<int, opt>{}) when opt is in the list, R{} otherwise: the one
// runtime-to-template step of every kernel selection.
template <int... K>
struct OptKinds {
  template <typename R, typename F>
  static R Dispatch(int opt, F f) {
    R r{};
    (void)((opt == K && (r = f(std::integral_constant<int, K>{}), true)) || ...);
    return r;
  }
};
using ElementwiseOpts = OptKinds<OPT_SGD, OPT_SGD_MOM, OPT_ADAM, OPT_ADAMW, OPT_TEST, OPT_NAG, OPT_ADABELIEF,
                                 OPT_RMSPROP, OPT_RMSPROP_CENTERED, OPT_SIGNSGD, OPT_SIGNUM, OPT_FTML, OPT_ADAMAX,
                                 OPT_ADADELTA, OPT_NADAM>;

enum SumOrder : int {
  ORDER_DEVICE = 0,  // ((in0+in1)+in2)+...                  ndarray_function-inl.h:457-486
  ORDER_COMMCPU = 1, // in0 + (((in1+in2)+in3)+in4), groups of 4   comm.h:359-393
  ORDER_TREE = 2     // pairwise up a binary tree, per entry: TensorWork::tree_prog   comm_tree.h:91-177 (topology.h)
};
constexpr int kTreeStack = 3;   // partial sums pending at once in a reduction tree over <= kMaxRanks values (tree_math.h)

enum SyncMode : int {
  SYNC_NONE = 0,      // all pointers local to this launch's device
  SYNC_READ_PEERS = 1,  // one-shot: peers' sources are read, only own memory is written
  SYNC_WRITE_PEERS = 2  // two-shot: peers' sources are read AND peers' destinations are written
};

struct alignas(16) TensorWork {
  const void* src[kMaxSrc];
  void* out[kMaxOut];
  const void* w;     // current weight in the key dtype (non-MP optimizers); may alias an out[]
  float* w32;        // fp32 master weight (multi-precision); updated in place
  float* s0;         // momentum | adam mean
  float* s1;         // adam variance
  int64_t begin;     // element range [begin, end) of the key handled by this launch
  int64_t end;
  float lr;          // per-key learning rate (lr_mult, scheduler, Adam / Adamax bias correction folded in; FTML:
                     //   (1-beta1^t)/lr)
  float wd;          // per-key weight decay
  float eta;         // AdamW schedule multiplier (FTML: 1 - beta2^t; Adamax: 1 - beta1, AdaDelta: 1 - rho, in double;
                     //   Nadam: coef2 = 1 - beta2^t; its other per-key scalars: DenseLaunch::nadam)
  int n_src;
  int n_out;
  int flags;         // kWork* bits (WorkFlags)
  union {
    int n_mc;            // NVLS launches: the last n_mc entries of out[] are multicast addresses
    uint32_t tree_prog;  // ORDER_TREE launches (never NVLS): when to add which partial sums, src[] being in the
  };                     //   tree's leaf order (topology.h: ReduceProgram)
  int key;           // host side only: the key this entry belongs to
  float* s2;         // centered RMSProp momentum (appended: every field above keeps its offset)
};
static_assert(sizeof(TensorWork) == 416, "TensorWork layout");

constexpr int kWorkVec16 = 1;    // every pointer 16-byte aligned and begin % 8 == 0: 16-byte packet loads / stores
constexpr int kWorkStaged = 2;   // eligible for the shared-memory staged variant (implies kWorkVec16)

// The flags of a filled-in entry: kWorkVec16 from its own pointers and range, kWorkStaged where the caller
// allows it (that depends on dtype, key size and optimizer, which the entry does not carry).  An empty range
// touches no element, so where it begins does not count: the empty trailing shard of a two-shot key (begin = size)
// must not take its launch class off the staged kernel, a decision every rank has to make alike.
inline int WorkFlags(const TensorWork& t, bool staged) {
  uintptr_t low = t.begin < t.end ? static_cast<uintptr_t>(t.begin) & 7 : 0;
  for (int k = 0; k < t.n_src; ++k) low |= reinterpret_cast<uintptr_t>(t.src[k]) & 15;
  for (int k = 0; k < t.n_out; ++k) low |= reinterpret_cast<uintptr_t>(t.out[k]) & 15;
  low |= (reinterpret_cast<uintptr_t>(t.w) | reinterpret_cast<uintptr_t>(t.w32) | reinterpret_cast<uintptr_t>(t.s0) |
          reinterpret_cast<uintptr_t>(t.s1) | reinterpret_cast<uintptr_t>(t.s2)) & 15;
  if (low != 0) return 0;
  return kWorkVec16 | (staged ? kWorkStaged : 0);
}

struct SyncArgs {
  uint32_t* self;                // this rank's signal pad
  uint32_t* peers[kMaxRanks];    // every rank's signal pad as mapped into this device's address space
  int world;
  int rank;
  int mode;                      // SyncMode
  long long timeout;             // spin limit in SM clock cycles (0: wait for ever)
  // The value this launch's blocks exchange: the same on every participant of the launch, different from every
  // earlier launch that used these pads (Runtime::NextSyncEpoch).  Round 1 derived it from a per-device counter
  // in the pad, which only agrees across GPUs as long as every collective launch has the same participants --
  // a single-process store pushed from {0,1}, then {0,1,2} dead-locked (found on the first 8-GPU run of round 2).
  uint32_t epoch;
};

// signal pad layout in uint32 words
constexpr int kSigStartOff = 0;
constexpr int kSigEndOff = kMaxBlocks * kMaxRanks;
constexpr int kSigFlagOff = 2 * kMaxBlocks * kMaxRanks;
// grid-wide barrier words (device_utils.cuh: grid_barrier): arrival counter, generation, epoch of the cross-GPU
// exchange, one flag per rank
constexpr int kSigGridOff = 2 * kMaxBlocks * kMaxRanks + kMaxBlocks;
constexpr int kSigGridCount = 0, kSigGridGen = 1, kSigGridEpoch = 2, kSigGridFlags = 4;
constexpr int kSigGridWords = 4 + kMaxRanks;
constexpr size_t kSignalPadBytes = (2 * kMaxBlocks * kMaxRanks + kMaxBlocks + kSigGridWords) * sizeof(uint32_t);

struct DenseLaunch {
  const TensorWork* works;       // device pointer, nworks entries
  const int64_t* chunk_prefix;   // device pointer, nworks+1 entries (exclusive prefix of chunk counts)
  int nworks;
  int64_t total_chunks;
  int dtype;                     // DType of src/out/w
  int opt;                       // OptKind
  int multi_precision;           // 1: w32 is the master, out is a cast copy
  int order;                     // SumOrder
  int fp32_accum;                // fp16 only: 1 = accumulate in fp32, 0 = round every add (reference)
  float rescale, clip, momentum, beta1, beta2, eps;
  SyncArgs sync;
  int grid;                      // blocks to launch (identical on every rank of a collective)
  int chunk_elems;               // elements per scheduling chunk (multiple of 128)
  int threads;                   // block size: 128, 256 or 512
  int small_n;                   // every entry has n_src <= 2: use the two-packets-in-flight variant
  int nvls;                      // 1: src[0] is a multicast address (multimem.ld_reduce / multimem.st variant)
  int bulk;                      // 1: shared-memory staged variant (cp.async.bulk + mbarrier pipeline)
  int bulk_stages;               // pipeline depth
  int bulk_arrays;               // input arrays staged per tile (max over the work list)
  int bulk_group;                // consecutive tiles a block takes before it strides on by grid * bulk_group tiles
  int nvls_unroll;               // NVLS variant: multimem.ld_reduce requests in flight per thread (1, 2, 4 or 8)
  int nvls_pipe;                 // NVLS variant: 1 = next chunk's ld_reduce issued before this chunk's update/stores
  int mp_arith;                  // 1: a 16-bit key of an optimizer created with multi_precision -- update_one takes
                                 //   the mp_* operator's grouping where it differs from the plain one (Hyper::mp)
  float rho;                     // RMSProp: decay of the squared-gradient (and centered: gradient) averages
  float clip_weights;            // RMSProp: |new weight| <= clip_weights when >= 0 (< 0: off)
  float wd_lh;                   // Signum: decoupled weight decay, w *= 1 - lr*wd_lh before the sign step
  // Nadam: four more per-key scalars than TensorWork has room for, one float4 per entry (nworks of them), uploaded
  // with the work list right after the chunk prefix: (1 - m_schedule, 1 - m_schedule_next, momentum_t_1,
  // 1 - momentum_t), each computed in double and rounded once (KVStore::NadamAdvance).  Null for every other kind.
  const float4* nadam;
  float one_minus_beta1, one_minus_beta2;   // Nadam: 1 - beta1 / 1 - beta2 computed in double, rounded once
};

// returns cudaError_t as int; never throws
int LaunchDense(const DenseLaunch& L, cudaStream_t stream);
int DenseMaxGrid(int device, int threads);   // resident-block capacity of the dense kernel
// L.order == ORDER_TREE (tree_kernels.cu; LaunchDense forwards): per-thread transport, additions in the order of
// every entry's tree_prog.  Same residency as kv_dense_kernel (DenseMaxGrid), never the staged or multicast variant.
int LaunchDenseTree(const DenseLaunch& L, cudaStream_t stream);
int TreeKernelAvailable(int dtype, int opt, int multi_precision);
// Plan the shared-memory staged variant for a float32 launch with `arrays` staged input streams per
// tile: picks tile elements / stages and returns the resident grid capacity (0: not applicable).  `local`: the
// launch has no rendezvous (SYNC_NONE), every stream is in this GPU's HBM.
int BulkPlan(int device, int opt, int multi_precision, int arrays, bool local, int* tile_elems, int* stages);
// Plan the multicast (NVLS) variant: elements per scheduling chunk (= one block iteration) for the given
// requests-in-flight / pipelining / block size, and the resident grid capacity (0: not available).
int NvlsPlan(int device, int opt, int multi_precision, int unroll, int pipe, int threads, int* chunk_elems);

int LaunchFill(void* ptr, int value_byte, size_t bytes, cudaStream_t s);
// gradient compression codec (bits = 1 or 2); code stream = ceil(n / (32/bits)) 32-bit words
int LaunchQuantize(int bits, const float* grad, float* residual, uint32_t* out, int64_t n, float thr, cudaStream_t s);
int LaunchDequantize(int bits, const uint32_t* in, float* out, int64_t n, float thr, cudaStream_t s);
// dst[i] = float(src[i]) for float32/float16/bfloat16 sources (fp32 master-weight creation)
int LaunchCastToF32(const void* src, int dtype, float* dst, int64_t n, cudaStream_t s);

}  // namespace mxkv
