// adadelta_host.cc -- the AdaDelta branch of csrc/optim_math.h compiled for the HOST (like optim_host.cc, with
// -ffp-contract=off): tests/test_adadelta.py checks it bit for bit against the oracle's restatement of AdaDelta.step,
// for float32 keys and for the fp32 master of 16-bit keys.
#include <cstdint>
#include "optim_math.h"

using namespace mxkv;

// s0 = acc_g, s1 = acc_delta; lr_op = lr and eta_op = 1 - rho, the per-key scalars of KVStore::KeyLR / KeyEta
extern "C" int host_adadelta(int64_t n, const float* g, float* w, float* s0, float* s1, float lr_op, float wd,
                             float eta_op, float rho, float eps, float rescale, float clip) {
  Hyper h;
  h.lr = lr_op; h.wd = wd; h.eta = eta_op; h.rescale = rescale; h.clip = clip; h.momentum = 0.f;
  h.beta1 = 0.f; h.beta2 = 0.f; h.eps = eps;
  h.mp = false;
  h.rho = rho; h.clip_weights = -1.f;
  h.wd_lh = 0.f;
  for (int64_t i = 0; i < n; ++i) w[i] = update_one<OPT_ADADELTA>(g[i], w[i], s0[i], s1[i], h);
  return 0;
}
