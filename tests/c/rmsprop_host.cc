// rmsprop_host.cc -- the two RMSProp branches of csrc/optim_math.h compiled for the HOST (like optim_host.cc, with
// -ffp-contract=off): tests/test_rmsprop.py checks them bit for bit against the oracle's RMSPropUpdateKernel and
// RMSPropAlexUpdateKernel restatements, for float32 keys and for the fp32 master of 16-bit keys.
#include <cstdint>
#include "optim_math.h"

using namespace mxkv;

static Hyper make_hyper(float lr, float wd, float rho, float momentum, float eps, float rescale, float clip,
                        float clip_weights) {
  Hyper h;
  h.lr = lr; h.wd = wd; h.eta = 1.f; h.rescale = rescale; h.clip = clip; h.momentum = momentum;
  h.beta1 = 0.f; h.beta2 = 0.f; h.eps = eps;
  h.mp = false;
  h.rho = rho; h.clip_weights = clip_weights;
  return h;
}

// centered == 0: rmsprop_update (s0 = var); centered != 0: rmspropalex_update (s0 = mean, s1 = var, s2 = mom)
extern "C" int host_rmsprop(int centered, int64_t n, const float* g, float* w, float* s0, float* s1, float* s2,
                            float lr, float wd, float rho, float momentum, float eps, float rescale, float clip,
                            float clip_weights) {
  const Hyper h = make_hyper(lr, wd, rho, momentum, eps, rescale, clip, clip_weights);
  for (int64_t i = 0; i < n; ++i) {
    if (centered) {
      w[i] = update_one<OPT_RMSPROP_CENTERED>(g[i], w[i], s0[i], s1[i], s2[i], h);
    } else {
      float unused = 0.f;
      w[i] = update_one<OPT_RMSPROP>(g[i], w[i], s0[i], unused, h);
    }
  }
  return 0;
}
