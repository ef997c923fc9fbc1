"""RMSProp for the CPU oracle (test infrastructure): the reference's two fused kernels restated operation by operation
on float32 numpy arrays, and the optimizer bookkeeping that drives them.

* ``rmsprop_update``          -- RMSPropUpdateKernel (src/operator/optimizer_op-inl.h:2005-2031), state ``var``::

      r   = clip(rescale*g) + wd*w                   (weight decay AFTER the clip)
      var = (1-rho)*(r*r) + rho*var
      w   = clip_w(w - (lr*r) / (sqrt(var) + eps))

* ``rmspropalex_update``      -- RMSPropAlexUpdateKernel (:1905-1939), states ``mean``, ``var``, ``mom``::

      var  = (1-rho)*(r*r) + rho*var
      mean = (1-rho)*r + rho*mean
      mom  = momentum*mom - (lr*r) / sqrt((var - mean*mean) + eps)
      w    = clip_w(w + mom)

* ``OracleRMSProp``           -- RMSProp.fused_step (python/mxnet/optimizer/rmsprop.py:143-181) with the bookkeeping of
  ``oracle.OracleOptimizer``: per-index update counts from ``begin_num_update``, lr / wd multipliers, no bias correction,
  and the operator's clips switched on only where ``clip_gradient`` / ``clip_weights`` is truthy (rmsprop.py:169-172):
  0, a negative value or None is off.  A 16-bit key is updated on its fp32 master and stored as its one rounding.

Every operation is one IEEE single-precision operation (numpy float32 element-wise arithmetic, no contraction into
FMAs), with the hyper-parameters rounded to float32 first, as the reference's float kernel parameters are; results
are bit-identical to the kernels' arithmetic (tests/test_rmsprop.py checks that against the kernels' own source
compiled for the host), and pinned to the reference's own ``RMSProp.step`` by tests/golden/rmsprop_steps.npz.
"""
import numpy as np

from oracle import oracle as O

_F = np.float32


def _clip(x, b):
    """mshadow_op::clip (mshadow_op.h:999-1009) where the bound is >= 0; a negative bound is off"""
    if b is None or b < 0.0:
        return x
    b = _F(b)
    return np.where(x > b, b, np.where(x < -b, -b, x)).astype(np.float32)


def _grad(w, g, wd, rescale, clip):
    r = _clip(_F(rescale) * np.asarray(g, np.float32), clip)
    return r + _F(wd) * w


def rmsprop_update(w, g, var, lr, wd=0.0, rho=0.9, eps=1e-8, rescale=1.0, clip=None, clip_weights=None):
    """RMSPropUpdateKernel on float32 arrays; w and var updated in place.  ``clip`` / ``clip_weights``: the operator's
    parameters (< 0 or None: off)"""
    w0 = w.copy()
    r = _grad(w0, g, wd, rescale, clip)
    n = (_F(1.0) - _F(rho)) * (r * r) + _F(rho) * var
    var[...] = n
    w[...] = _clip(w0 - (_F(lr) * r) / (np.sqrt(n) + _F(eps)), clip_weights)


def rmspropalex_update(w, g, mean, var, mom, lr, wd=0.0, rho=0.9, momentum=0.9, eps=1e-8, rescale=1.0, clip=None,
                       clip_weights=None):
    """RMSPropAlexUpdateKernel on float32 arrays; w, mean, var and mom updated in place"""
    w0 = w.copy()
    r = _grad(w0, g, wd, rescale, clip)
    c = _F(1.0) - _F(rho)
    n = c * (r * r) + _F(rho) * var
    m = c * r + _F(rho) * mean
    d = _F(momentum) * mom - (_F(lr) * r) / np.sqrt((n - m * m) + _F(eps))
    mean[...] = m
    var[...] = n
    mom[...] = d
    w[...] = _clip(w0 + d, clip_weights)


def fused_switch(v):
    """rmsprop.py:169-172: the value the operator receives -- the option where it is truthy, else off"""
    return v if v else None


class OracleRMSProp(object):
    """RMSProp.fused_step over float32 weights, updated in place; usable as ``OracleKVStore.set_optimizer(...)``."""

    def __init__(self, learning_rate=0.001, rho=0.9, momentum=0.9, epsilon=1e-8, centered=False, clip_weights=None,
                 wd=0.0, rescale_grad=1.0, clip_gradient=None, lr_mult=None, wd_mult=None, begin_num_update=0,
                 multi_precision=False):
        self.lr, self.rho, self.momentum, self.epsilon = learning_rate, rho, momentum, epsilon   # rmsprop.py:70-71
        self.centered, self.clip_weights, self.wd = centered, clip_weights, wd
        self.rescale_grad, self.clip_gradient = rescale_grad, clip_gradient
        self.lr_mult, self.wd_mult = dict(lr_mult or {}), dict(wd_mult or {})
        self.begin_num_update = begin_num_update
        self.count, self.states = {}, {}

    def state(self, index, like):
        if index not in self.states:
            n = 3 if self.centered else 1
            self.states[index] = tuple(np.zeros_like(like, np.float32) for _ in range(n))
        return self.states[index]

    def _run(self, index, w, g):
        self.count[index] = self.count.get(index, self.begin_num_update) + 1
        st = self.state(index, w)
        lr = float(np.float32(self.lr * self.lr_mult.get(index, 1.0)))
        wd = float(np.float32(self.wd * self.wd_mult.get(index, 1.0)))
        clip, cw = fused_switch(self.clip_gradient), fused_switch(self.clip_weights)
        if self.centered:
            rmspropalex_update(w, g, st[0], st[1], st[2], lr, wd, self.rho, self.momentum, self.epsilon,
                               self.rescale_grad, clip, cw)
        else:
            rmsprop_update(w, g, st[0], lr, wd, self.rho, self.epsilon, self.rescale_grad, clip, cw)

    def update(self, index, weight, grad):
        self._run(index, weight, grad)

    def update_lp(self, index, w_lp, lp_kind, w32, grad32):
        """a 16-bit key: ``w32`` is the fp32 master (updated in place), ``w_lp`` (uint16 bits; 1 fp16, 2 bf16)
        receives its rounding to the key type"""
        self._run(index, w32, grad32)
        if w_lp is None or lp_kind == 0:
            return
        flat = w_lp.reshape(-1)
        if lp_kind == 1:
            flat[...] = w32.reshape(-1).astype(np.float16).view(np.uint16)
        else:
            flat[...] = O.f32_to_bf16(w32.reshape(-1))
