// nadam_host.cc -- the Nadam branch of csrc/optim_math.h compiled for the HOST (like optim_host.cc, with
// -ffp-contract=off): tests/test_nadam.py checks it bit for bit against the oracle's restatement of Nadam.step, for
// float32 keys and for the fp32 master of 16-bit keys.
#include <cstdint>
#include "optim_math.h"

using namespace mxkv;

// s0 = mean, s1 = var.  Per launch c1 = 1 - beta1, c2 = 1 - beta2; per key lr, coef2 (the entry's eta) and the side
// array's 1 - m_schedule, 1 - m_schedule_next, momentum_t_1, 1 - momentum_t (KVStore::KeyScalars)
extern "C" int host_nadam(int64_t n, const float* g, float* w, float* s0, float* s1, float lr, float wd, float coef2,
                          float g_div, float m_div, float mom_t1, float c_mom_t, float beta1, float beta2, float c1,
                          float c2, float eps, float rescale, float clip) {
  Hyper h;
  h.lr = lr; h.wd = wd; h.eta = coef2; h.rescale = rescale; h.clip = clip; h.momentum = 0.f;
  h.beta1 = beta1; h.beta2 = beta2; h.eps = eps;
  h.mp = false;
  h.rho = 0.f; h.clip_weights = -1.f;
  h.wd_lh = 0.f;
  h.c1 = c1; h.c2 = c2; h.g_div = g_div; h.m_div = m_div; h.mom_t1 = mom_t1; h.c_mom_t = c_mom_t;
  for (int64_t i = 0; i < n; ++i) w[i] = update_one<OPT_NADAM>(g[i], w[i], s0[i], s1[i], h);
  return 0;
}
