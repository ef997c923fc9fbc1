"""AdaBelief for the CPU oracle (test infrastructure): the reference's fused kernel restated operation by operation on
float32 numpy arrays, and the optimizer bookkeeping that drives it.

* ``adabelief_update``    -- MultiMPAdaBeliefKernel (src/operator/contrib/adabelief-inl.h:354-384) on a float32 weight,
  the grouping of every aggregated AdaBelief operator::

      r    = clip(rescale*g + wd*w)                  (weight decay BEFORE the clip)
      mean = beta1*(mean - r) + r
      adj  = (mean - r)*(mean - r)
      var  = (beta2*(var - adj) + adj) + eps
      w    = w - eta*((lr*mean) / (sqrt(var) + eps))

* ``lp_adabelief_update`` -- the same on the fp32 master of a 16-bit key, the stored weight its one rounding to the key
  type (for float16 with multi_precision that is ``_multi_mp_adabelief_update``; bfloat16 keys, and float16 keys without
  multi_precision, follow the engine's convention of an fp32 master for every 16-bit key)
* ``OracleAdaBelief``     -- AdaBelief.fused_step (python/mxnet/optimizer/adabelief.py:141-231) with the bookkeeping of
  ``oracle.OracleOptimizer``: per-index update counts from ``begin_num_update``, lr / wd multipliers, operator lr = 1 and
  operator eta = the bias-corrected learning rate (in double, rounded once), and no change at all -- after the count
  has advanced -- when ``rescale_grad`` is 0, inf or nan (adabelief-inl.h:454-466)

Every operation is one IEEE single-precision operation (numpy float32 element-wise arithmetic, no contraction into
FMAs), with the hyper-parameters rounded to float32 first, as the reference's float kernel parameters are; results
are bit-identical to the kernels' arithmetic (tests/test_adabelief.py checks that against the kernels' own source
compiled for the host), and pinned to the reference's own ``AdaBelief.step`` by tests/golden/adabelief_steps.npz.
"""
import numpy as np

from oracle import oracle as O

_F = np.float32


def adabelief_update(w, g, mean, var, eta, wd=0.0, beta1=0.9, beta2=0.999, eps=1e-6, rescale=1.0, clip=None,
                     lr=1.0):
    """MultiMPAdaBeliefKernel on float32 arrays; w, mean and var updated in place"""
    w0 = w.copy()
    r = _F(rescale) * np.asarray(g, np.float32)
    r = r + _F(wd) * w0
    c = -1.0 if clip is None else clip
    if c >= 0.0:                                   # mshadow_op::clip, mshadow_op.h:999-1009
        b = _F(c)
        r = np.where(r > b, b, np.where(r < -b, -b, r)).astype(np.float32)
    m = _F(beta1) * (mean - r) + r
    d = m - r
    adj = d * d
    v = (_F(beta2) * (var - adj) + adj) + _F(eps)
    mean[...] = m
    var[...] = v
    w[...] = w0 - _F(eta) * ((_F(lr) * m) / (np.sqrt(v) + _F(eps)))


def lp_adabelief_update(w_lp, lp_kind, w32, mean, var, g32, eta, wd=0.0, beta1=0.9, beta2=0.999, eps=1e-6,
                        rescale=1.0, clip=None):
    """a 16-bit key: the update on the fp32 master w32 (in place); w_lp (uint16 bits; lp_kind 1 fp16, 2 bf16) = its
    rounding to the key type"""
    adabelief_update(w32, g32, mean, var, eta, wd, beta1, beta2, eps, rescale, clip)
    if w_lp is None or lp_kind == 0:
        return
    flat = w_lp.reshape(-1)
    if lp_kind == 1:
        flat[...] = w32.reshape(-1).astype(np.float16).view(np.uint16)
    else:
        flat[...] = O.f32_to_bf16(w32.reshape(-1))


def bias_corrected_lr(lr, beta1, beta2, t):
    """lr * sqrt(1 - beta2^t) / (1 - beta1^t) in double (adabelief.py:174-181), grouped as the engine groups it
    (oracle.adam_lr)"""
    return O.adam_lr(lr, beta1, beta2, t)


class OracleAdaBelief(object):
    """AdaBelief.fused_step over float32 weights, updated in place; usable as ``OracleKVStore.set_optimizer(...)``."""

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-6, correct_bias=True, wd=0.0,
                 rescale_grad=1.0, clip_gradient=None, lr_mult=None, wd_mult=None, begin_num_update=0):
        self.lr, self.beta1, self.beta2, self.epsilon = learning_rate, beta1, beta2, epsilon   # adabelief.py:79
        self.correct_bias, self.wd = correct_bias, wd
        self.rescale_grad, self.clip_gradient = rescale_grad, clip_gradient
        self.lr_mult, self.wd_mult = dict(lr_mult or {}), dict(wd_mult or {})
        self.begin_num_update = begin_num_update
        self.count, self.states = {}, {}

    def eta(self, index):
        """the operator's eta for the CURRENT count of ``index``"""
        lr = self.lr * self.lr_mult.get(index, 1.0)
        if self.correct_bias:
            lr = bias_corrected_lr(lr, self.beta1, self.beta2, self.count[index])
        return float(np.float32(lr))

    def state(self, index, like):
        if index not in self.states:
            self.states[index] = (np.zeros_like(like, np.float32), np.zeros_like(like, np.float32))
        return self.states[index]

    def skips(self):
        rg = self.rescale_grad
        return not np.isfinite(rg) or rg == 0

    def update(self, index, weight, grad):
        self.count[index] = self.count.get(index, self.begin_num_update) + 1
        mean, var = self.state(index, weight)
        if self.skips():
            return
        adabelief_update(weight, grad, mean, var, self.eta(index), self.wd * self.wd_mult.get(index, 1.0),
                         self.beta1, self.beta2, self.epsilon, self.rescale_grad, self.clip_gradient)

    def update_lp(self, index, w_lp, lp_kind, w32, grad32):
        """a 16-bit key: ``w32`` is the fp32 master (updated in place), ``w_lp`` receives the stored bits"""
        self.count[index] = self.count.get(index, self.begin_num_update) + 1
        mean, var = self.state(index, w32)
        if self.skips():
            return
        lp_adabelief_update(w_lp, lp_kind, w32, mean, var, grad32, self.eta(index),
                            self.wd * self.wd_mult.get(index, 1.0), self.beta1, self.beta2, self.epsilon,
                            self.rescale_grad, self.clip_gradient)
