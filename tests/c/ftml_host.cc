// ftml_host.cc -- the FTML branch of csrc/optim_math.h compiled for the HOST (like optim_host.cc, with
// -ffp-contract=off): tests/test_ftml.py checks it bit for bit against the oracle's FTMLKernel restatement, for
// float32 keys and for the fp32 master of 16-bit keys.
#include <cstdint>
#include "optim_math.h"

using namespace mxkv;

// s0 = d, s1 = v, s2 = z; lr_op = (1 - beta1^t) / lr and eta_op = 1 - beta2^t, the per-key scalars of
// KVStore::KeyScalars
extern "C" int host_ftml(int64_t n, const float* g, float* w, float* s0, float* s1, float* s2, float lr_op, float wd,
                         float eta_op, float beta1, float beta2, float eps, float rescale, float clip) {
  Hyper h;
  h.lr = lr_op; h.wd = wd; h.eta = eta_op; h.rescale = rescale; h.clip = clip; h.momentum = 0.f;
  h.beta1 = beta1; h.beta2 = beta2; h.eps = eps;
  h.mp = false;
  h.rho = 0.f; h.clip_weights = -1.f;
  h.wd_lh = 0.f;
  for (int64_t i = 0; i < n; ++i) w[i] = update_one<OPT_FTML>(g[i], w[i], s0[i], s1[i], s2[i], h);
  return 0;
}
