// optim_math.h -- the per-element arithmetic of the fused optimizers, in a header that compiles both for
// the device (nvcc: the kernels in kernels.cu / rsp_kernels.cu / norm_kernels.cu) and for the host (g++:
// tests/c/optim_host.cc, which the CPU test-suite checks bit-for-bit against the oracle -- the same source
// the GPU executes, verified without a GPU).
//
// On the device the __f*_rn intrinsics keep ptxas from contracting a*b+c into an FMA.  On the host they
// are plain IEEE single-precision operations; the host translation unit MUST be built with
// -ffp-contract=off for the same reason.
#pragma once
#include "kernels.h"

#if defined(__CUDACC__)
#define MXKV_HD __device__ __forceinline__
#else
#include <cmath>
#define MXKV_HD inline
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __fsqrt_rn(float a) { return std::sqrt(a); }
#endif

namespace mxkv {

struct Hyper {
  float lr, wd, eta, rescale, clip, momentum, beta1, beta2, eps;
  bool mp;    // OPT_NAG only: MP_NAGMomKernel's grouping of the weight step (DenseLaunch::mp_arith)
  float rho, clip_weights;   // OPT_RMSPROP / OPT_RMSPROP_CENTERED (DenseLaunch::rho / clip_weights)
  float wd_lh;               // OPT_SIGNUM (DenseLaunch::wd_lh)
  // OPT_NADAM only (make_hyper): 1 - beta1, 1 - beta2 per launch; per key 1 - m_schedule, 1 - m_schedule_next,
  // momentum_t_1, 1 - momentum_t (DenseLaunch::nadam).  h.eta carries coef2 = 1 - beta2^t
  float c1, c2, g_div, m_div, mom_t1, c_mom_t;
};

MXKV_HD float clipf(float x, float b) {   // mshadow_op::clip, mshadow_op.h:999-1009
  return x > b ? b : (x < -b ? -b : x);
}

// (x > 0) - (x < 0) as the reference's Signum kernels write it: NaN and +-0 give 0
MXKV_HD float signf(float x) {
  return static_cast<float>((x > 0.0f) - (x < 0.0f));
}

// mshadow_op::maximum (mshadow_op.h:1266-1275): a NaN in either operand gives NaN -- unlike fmaxf, which returns the
// other operand
MXKV_HD float maximumf(float a, float b) {
  return a != a ? a : (a > b ? a : b);
}

// one element of the fused update; returns the new weight.  Operation order is
// the reference source's, see the OptKind comments in kernels.h.
template <int OPT>
MXKV_HD float update_one(float g, float w, float& s0, float& s1, const Hyper& h) {
  if (OPT == OPT_SGD) {
    float r = __fmul_rn(h.rescale, g);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(h.wd, w));
    return __fsub_rn(w, __fmul_rn(h.lr, r));
  } else if (OPT == OPT_SGD_MOM) {
    float r = __fmul_rn(h.rescale, g);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(h.wd, w));
    float m = __fmul_rn(s0, h.momentum);
    m = __fsub_rn(m, __fmul_rn(h.lr, r));
    s0 = m;
    return __fadd_rn(w, m);
  } else if (OPT == OPT_ADAM) {
    float r = __fmul_rn(g, h.rescale);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(w, h.wd));
    const float m = __fadd_rn(__fmul_rn(h.beta1, s0), __fmul_rn(__fsub_rn(1.f, h.beta1), r));
    const float v = __fadd_rn(__fmul_rn(h.beta2, s1),
                              __fmul_rn(__fmul_rn(__fsub_rn(1.f, h.beta2), r), r));
    s0 = m; s1 = v;
    return __fsub_rn(w, __fdiv_rn(__fmul_rn(h.lr, m), __fadd_rn(__fsqrt_rn(v), h.eps)));
  } else if (OPT == OPT_ADAMW) {
    float sg = __fmul_rn(h.rescale, g);
    if (h.clip >= 0.0f) sg = clipf(sg, h.clip);
    const float m = __fadd_rn(__fmul_rn(h.beta1, s0), __fmul_rn(__fsub_rn(1.0f, h.beta1), sg));
    const float v = __fadd_rn(__fmul_rn(h.beta2, s1),
                              __fmul_rn(__fsub_rn(1.0f, h.beta2), __fmul_rn(sg, sg)));
    s0 = m; s1 = v;
    const float step = __fadd_rn(__fdiv_rn(__fmul_rn(h.lr, m), __fadd_rn(__fsqrt_rn(v), h.eps)),
                                 __fmul_rn(h.wd, w));
    return __fsub_rn(w, __fmul_rn(h.eta, step));
  } else if (OPT == OPT_TEST) {
    const float gr = __fmul_rn(h.rescale, g);
    const float s = __fadd_rn(gr, __fmul_rn(h.wd, w));
    return __fsub_rn(w, __fmul_rn(h.lr, s));
  } else if (OPT == OPT_SGD_STD) {
    // every row: w *= (1 - lr*wd); rows of the gradient: w -= lr * clip(rescale*g) (wd already applied)
    const float ws = __fmul_rn(w, __fsub_rn(1.0f, __fmul_rn(h.lr, h.wd)));
    float r = __fmul_rn(h.rescale, g);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(0.0f, ws));
    return __fsub_rn(ws, __fmul_rn(h.lr, r));
  } else if (OPT == OPT_ADAM_STD) {
    float r = __fmul_rn(g, h.rescale);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(w, h.wd));
    const float m = __fadd_rn(__fmul_rn(h.beta1, s0), __fmul_rn(__fsub_rn(1.f, h.beta1), r));
    const float v = __fadd_rn(__fmul_rn(h.beta2, s1), __fmul_rn(__fsub_rn(1.f, h.beta2), __fmul_rn(r, r)));
    s0 = m; s1 = v;
    return __fsub_rn(w, __fdiv_rn(__fmul_rn(h.lr, m), __fadd_rn(__fsqrt_rn(v), h.eps)));
  } else if (OPT == OPT_NAG) {
    float r = __fmul_rn(h.rescale, g);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(h.wd, w));
    float m = __fmul_rn(s0, h.momentum);
    m = __fsub_rn(m, __fmul_rn(h.lr, r));
    s0 = m;
    // NAGMomKernel: (w + momentum*mom) - lr*r;  MP_NAGMomKernel: w + (momentum*mom - lr*r)
    if (h.mp) return __fadd_rn(w, __fsub_rn(__fmul_rn(h.momentum, m), __fmul_rn(h.lr, r)));
    return __fsub_rn(__fadd_rn(w, __fmul_rn(h.momentum, m)), __fmul_rn(h.lr, r));
  } else if (OPT == OPT_ADABELIEF) {
    // MultiMPAdaBeliefKernel: wd is added BEFORE the clip; eps is added to the variance state every step
    float r = __fmul_rn(h.rescale, g);
    r = __fadd_rn(r, __fmul_rn(h.wd, w));
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    const float m = __fadd_rn(__fmul_rn(h.beta1, __fsub_rn(s0, r)), r);
    const float d = __fsub_rn(m, r);
    const float adj = __fmul_rn(d, d);
    const float v = __fadd_rn(__fadd_rn(__fmul_rn(h.beta2, __fsub_rn(s1, adj)), adj), h.eps);
    s0 = m; s1 = v;
    return __fsub_rn(w, __fmul_rn(h.eta, __fdiv_rn(__fmul_rn(h.lr, m), __fadd_rn(__fsqrt_rn(v), h.eps))));
  } else if (OPT == OPT_RMSPROP) {
    // RMSPropUpdateKernel (s0 = var): wd is added AFTER the clip; the weight clip is applied to the new weight
    float r = __fmul_rn(h.rescale, g);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(h.wd, w));
    const float n = __fadd_rn(__fmul_rn(__fsub_rn(1.f, h.rho), __fmul_rn(r, r)), __fmul_rn(h.rho, s0));
    s0 = n;
    const float wn = __fsub_rn(w, __fdiv_rn(__fmul_rn(h.lr, r), __fadd_rn(__fsqrt_rn(n), h.eps)));
    return h.clip_weights >= 0.0f ? clipf(wn, h.clip_weights) : wn;
  } else if (OPT == OPT_SIGNSGD) {
    // SignSGDKernel: the sign of the summed gradient as it arrives -- rescale_grad and clip_gradient do not enter;
    // wd is wd + wd_lh (KVStore::KeyScalars).  lr * sign is exact.
    return __fsub_rn(__fmul_rn(__fsub_rn(1.f, __fmul_rn(h.lr, h.wd)), w), __fmul_rn(h.lr, signf(g)));
  } else if (OPT == OPT_SIGNUM) {
    // SignumKernel (s0 = mom, the NEGATED average: the weight step is + lr * sign(mom))
    float r = __fmul_rn(h.rescale, g);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(h.wd, w));
    float m = __fmul_rn(s0, h.momentum);
    m = __fsub_rn(m, __fmul_rn(__fsub_rn(1.f, h.momentum), r));
    s0 = m;
    return __fadd_rn(__fmul_rn(__fsub_rn(1.f, __fmul_rn(h.lr, h.wd_lh)), w), __fmul_rn(h.lr, signf(m)));
  } else if (OPT == OPT_ADAMAX) {
    // Adamax.step (s0 = mean, s1 = var, the max-norm u), one NDArray operation per rounding.  Per key
    // (KVStore::KeyScalars): h.lr = lr / (1 - beta1^t) and h.eta = 1 - beta1, each computed in double and rounded once,
    // as Python hands a scalar to an NDArray operation
    float r = __fmul_rn(g, h.rescale);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(h.wd, w));
    const float m = __fadd_rn(__fmul_rn(s0, h.beta1), __fmul_rn(h.eta, r));
    const float u = maximumf(__fmul_rn(h.beta2, s1), fabsf(r));
    s0 = m; s1 = u;
    return __fsub_rn(w, __fmul_rn(h.lr, __fdiv_rn(m, __fadd_rn(u, h.eps))));
  } else if (OPT == OPT_ADADELTA) {
    // AdaDelta.step (s0 = acc_g, s1 = acc_delta), one NDArray operation per rounding; h.eta = 1 - rho computed in
    // double and rounded once (KVStore::KeyScalars).  The step size is taken from the OLD acc_delta
    float r = __fmul_rn(g, h.rescale);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(h.wd, w));
    const float ag = __fadd_rn(__fmul_rn(s0, h.rho), __fmul_rn(h.eta, __fmul_rn(r, r)));
    float cd = __fsqrt_rn(__fadd_rn(s1, h.eps));
    cd = __fdiv_rn(cd, __fsqrt_rn(__fadd_rn(ag, h.eps)));
    cd = __fmul_rn(cd, r);
    const float ad = __fadd_rn(__fmul_rn(s1, h.rho), __fmul_rn(h.eta, __fmul_rn(cd, cd)));
    s0 = ag; s1 = ad;
    return __fsub_rn(w, __fmul_rn(h.lr, cd));
  } else if (OPT == OPT_NADAM) {
    // Nadam.step (s0 = mean, s1 = var), one NDArray operation per rounding, in step's order.  square(grad) and
    // (1 - beta2) * square(grad) round separately.  The momentum schedule's scalars arrive per key, each computed in
    // double and rounded once (KVStore::KeyScalars): h.g_div = 1 - m_schedule, h.m_div = 1 - m_schedule_next,
    // h.mom_t1 = momentum_t_1, h.c_mom_t = 1 - momentum_t, h.eta = coef2 = 1 - beta2^t
    float r = __fmul_rn(g, h.rescale);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(h.wd, w));
    const float m = __fadd_rn(__fmul_rn(s0, h.beta1), __fmul_rn(h.c1, r));
    const float v = __fadd_rn(__fmul_rn(s1, h.beta2), __fmul_rn(h.c2, __fmul_rn(r, r)));
    s0 = m; s1 = v;
    const float gp = __fdiv_rn(r, h.g_div);
    const float mp = __fdiv_rn(m, h.m_div);
    const float vp = __fdiv_rn(v, h.eta);
    const float mb = __fadd_rn(__fmul_rn(h.mom_t1, mp), __fmul_rn(h.c_mom_t, gp));
    return __fsub_rn(w, __fmul_rn(h.lr, __fdiv_rn(mb, __fadd_rn(__fsqrt_rn(vp), h.eps))));
  }
  return g;  // OPT_NONE
}

// The kinds with a third state array (OptHasS2) are computed here; every other kind is the five-argument form
// above, and s2 is not touched.
template <int OPT>
MXKV_HD float update_one(float g, float w, float& s0, float& s1, float& s2, const Hyper& h) {
  if constexpr (OPT == OPT_RMSPROP_CENTERED) {
    // RMSPropAlexUpdateKernel (s0 = mean, s1 = var, s2 = mom):
    //   n = (1-rho)*r*r + rho*n;  gbar = (1-rho)*r + rho*gbar;  mom = momentum*mom - (lr*r) / sqrt((n - gbar*gbar) + eps)
    float r = __fmul_rn(h.rescale, g);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(h.wd, w));
    const float c = __fsub_rn(1.f, h.rho);
    const float n = __fadd_rn(__fmul_rn(c, __fmul_rn(r, r)), __fmul_rn(h.rho, s1));
    const float m = __fadd_rn(__fmul_rn(c, r), __fmul_rn(h.rho, s0));
    const float d = __fsub_rn(__fmul_rn(h.momentum, s2),
                              __fdiv_rn(__fmul_rn(h.lr, r), __fsqrt_rn(__fadd_rn(__fsub_rn(n, __fmul_rn(m, m)), h.eps))));
    s0 = m; s1 = n; s2 = d;
    const float wn = __fadd_rn(w, d);
    return h.clip_weights >= 0.0f ? clipf(wn, h.clip_weights) : wn;
  } else if constexpr (OPT == OPT_FTML) {
    // FTMLKernel (s0 = d, s1 = v, s2 = z).  The two powers of t arrive per key (KVStore::KeyScalars):
    // h.lr = (1 - beta1^t) / lr and h.eta = 1 - beta2^t, so that
    //   v = beta2*v + (1-beta2)*r*r;  d_t = h.lr * (sqrt(v / h.eta) + eps)
    //   z = (beta1*z + (1-beta1)*r) - (d_t - beta1*d)*w;  d = d_t;  w = -z / d_t
    float r = __fmul_rn(h.rescale, g);
    if (h.clip >= 0.0f) r = clipf(r, h.clip);
    r = __fadd_rn(r, __fmul_rn(h.wd, w));
    const float v = __fadd_rn(__fmul_rn(h.beta2, s1), __fmul_rn(__fsub_rn(1.f, h.beta2), __fmul_rn(r, r)));
    const float dt = __fmul_rn(h.lr, __fadd_rn(__fsqrt_rn(__fdiv_rn(v, h.eta)), h.eps));
    const float z = __fsub_rn(__fadd_rn(__fmul_rn(h.beta1, s2), __fmul_rn(__fsub_rn(1.f, h.beta1), r)),
                              __fmul_rn(__fsub_rn(dt, __fmul_rn(h.beta1, s0)), w));
    s0 = dt; s1 = v; s2 = z;
    return __fdiv_rn(-z, dt);
  } else {
    return update_one<OPT>(g, w, s0, s1, h);
  }
}

// ---------------------------------------------------------------------------
// 1-bit / 2-bit gradient compression with error feedback (src/kvstore/gradient_compression-inl.h:44-227).
// Bit layout is the reference's: byte j of the stream holds values 4j..4j+3 (2-bit) or 8j..8j+7 (1-bit),
// first value in the most significant bits.
// ---------------------------------------------------------------------------
// code word w of the stream: residual += grad for its values, emit the codes, keep the quantisation error
template <int BITS>
MXKV_HD uint32_t quantize_word(const float* grad, float* residual, int64_t n, float thr, int64_t w) {
  constexpr int PER_WORD = 32 / BITS;
  uint32_t word = 0;
  const int64_t base = w * PER_WORD;
#pragma unroll
  for (int j = 0; j < PER_WORD; ++j) {
    const int64_t i = base + j;
    if (i >= n) break;
    float r = __fadd_rn(residual[i], grad[i]);
    const int byte = j / (8 / BITS);           // byte within the word (little endian in memory)
    const int slot = j % (8 / BITS);           // value within the byte, MSB first
    if (BITS == 2) {
      if (r >= thr) { word |= (0x3u << (6 - 2 * slot)) << (8 * byte); r = __fsub_rn(r, thr); }
      else if (r <= -thr) { word |= (0x2u << (6 - 2 * slot)) << (8 * byte); r = __fsub_rn(r, -thr); }
    } else {
      if (r > thr) { word |= (0x1u << (7 - slot)) << (8 * byte); r = __fsub_rn(r, 1.0f); }
      else r = __fadd_rn(r, 1.0f);
    }
    residual[i] = r;
  }
  return word;
}

// value i of a code stream
template <int BITS>
MXKV_HD float dequantize_value(const uint32_t* in, float thr, int64_t i) {
  constexpr int PER_WORD = 32 / BITS;
  const uint32_t word = in[i / PER_WORD];
  const int j = static_cast<int>(i % PER_WORD);
  const int byte = j / (8 / BITS), slot = j % (8 / BITS);
  const uint32_t b = (word >> (8 * byte)) & 0xffu;
  if (BITS == 2) {
    const uint32_t code = (b >> (6 - 2 * slot)) & 0x3u;
    return code == 0x3u ? thr : (code == 0x2u ? -thr : 0.0f);
  }
  return ((b >> (7 - slot)) & 0x1u) ? 1.0f : -1.0f;
}

}  // namespace mxkv
