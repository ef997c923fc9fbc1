// adabelief_host.cc -- the AdaBelief branch of csrc/optim_math.h compiled for the HOST (like optim_host.cc, with
// -ffp-contract=off): tests/test_adabelief.py checks it bit for bit against the oracle's MultiMPAdaBeliefKernel
// restatement, for float32 keys and for the fp32 master of 16-bit keys.
#include <cstdint>
#include "optim_math.h"

using namespace mxkv;

extern "C" int host_adabelief(int64_t n, const float* g, float* w, float* mean, float* var, float lr, float eta,
                              float wd, float beta1, float beta2, float eps, float rescale, float clip) {
  Hyper h;
  h.lr = lr; h.wd = wd; h.eta = eta; h.rescale = rescale; h.clip = clip; h.momentum = 0.f;
  h.beta1 = beta1; h.beta2 = beta2; h.eps = eps;
  h.mp = false;
  for (int64_t i = 0; i < n; ++i) w[i] = update_one<OPT_ADABELIEF>(g[i], w[i], mean[i], var[i], h);
  return 0;
}
