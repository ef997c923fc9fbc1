// signum_host.cc -- the two Signum branches of csrc/optim_math.h compiled for the HOST (like optim_host.cc, with
// -ffp-contract=off): tests/test_signum.py checks them bit for bit against the oracle's SignSGDKernel and SignumKernel
// restatements, for float32 keys and for the fp32 master of 16-bit keys.
#include <cstdint>
#include "optim_math.h"

using namespace mxkv;

// momentum_kind == 0: signsgd_update (no state); != 0: signum_update (s0 = mom).  The arguments are the operator's:
// momentum and clip as the store hands them to the kernel.
extern "C" int host_signum(int momentum_kind, int64_t n, const float* g, float* w, float* s0, float lr, float wd,
                           float momentum, float wd_lh, float rescale, float clip) {
  Hyper h;
  h.lr = lr; h.wd = wd; h.eta = 1.f; h.rescale = rescale; h.clip = clip; h.momentum = momentum;
  h.beta1 = 0.f; h.beta2 = 0.f; h.eps = 0.f;
  h.mp = false;
  h.rho = 0.f; h.clip_weights = -1.f;
  h.wd_lh = wd_lh;
  for (int64_t i = 0; i < n; ++i) {
    float unused = 0.f;
    if (momentum_kind) {
      w[i] = update_one<OPT_SIGNUM>(g[i], w[i], s0[i], unused, h);
    } else {
      float none = 0.f;
      w[i] = update_one<OPT_SIGNSGD>(g[i], w[i], none, unused, h);
    }
  }
  return 0;
}
