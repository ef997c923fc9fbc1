// adamax_host.cc -- the Adamax branch of csrc/optim_math.h compiled for the HOST (like optim_host.cc, with
// -ffp-contract=off): tests/test_adamax.py checks it bit for bit against the oracle's restatement of Adamax.step, for
// float32 keys and for the fp32 master of 16-bit keys.
#include <cstdint>
#include "optim_math.h"

using namespace mxkv;

// s0 = mean, s1 = var; lr_op = lr / (1 - beta1^t) and eta_op = 1 - beta1, the per-key scalars of KVStore::KeyLR /
// KeyEta
extern "C" int host_adamax(int64_t n, const float* g, float* w, float* s0, float* s1, float lr_op, float wd,
                           float eta_op, float beta1, float beta2, float eps, float rescale, float clip) {
  Hyper h;
  h.lr = lr_op; h.wd = wd; h.eta = eta_op; h.rescale = rescale; h.clip = clip; h.momentum = 0.f;
  h.beta1 = beta1; h.beta2 = beta2; h.eps = eps;
  h.mp = false;
  h.rho = 0.f; h.clip_weights = -1.f;
  h.wd_lh = 0.f;
  for (int64_t i = 0; i < n; ++i) w[i] = update_one<OPT_ADAMAX>(g[i], w[i], s0[i], s1[i], h);
  return 0;
}
