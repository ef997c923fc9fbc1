// nag_host.cc -- the NAG branch of csrc/optim_math.h compiled for the HOST (like optim_host.cc, with
// -ffp-contract=off): tests/test_nag.py checks it bit for bit against the oracle's NAGMomKernel /
// MP_NAGMomKernel restatements, for float32 keys and for the fp32 master of 16-bit keys with and without
// multi_precision (Hyper::mp).
#include <cstdint>
#include "optim_math.h"

using namespace mxkv;

extern "C" int host_nag(int64_t n, const float* g, float* w, float* mom, float lr, float wd, float rescale,
                        float clip, float momentum, int mp) {
  Hyper h;
  h.lr = lr; h.wd = wd; h.eta = 1.f; h.rescale = rescale; h.clip = clip; h.momentum = momentum;
  h.beta1 = h.beta2 = h.eps = 0.f;
  h.mp = mp != 0;
  float unused = 0.f;
  for (int64_t i = 0; i < n; ++i) w[i] = update_one<OPT_NAG>(g[i], w[i], mom[i], unused, h);
  return 0;
}
