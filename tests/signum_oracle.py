"""Signum for the CPU oracle (test infrastructure): the reference's two fused kernels restated operation by operation on
float32 numpy arrays, and the optimizer bookkeeping that drives them.

* ``signsgd_update``          -- SignSGDKernel (src/operator/optimizer_op-inl.h:2293-2305), no state::

      w = (1 - lr*wd)*w - lr*sign(g)               (rescale_grad and clip_gradient do not enter)

* ``signum_update``           -- SignumKernel (:2361-2379), state ``mom`` (the NEGATED average)::

      r   = clip(rescale*g) + wd*w                 (weight decay AFTER the clip)
      mom = mom*momentum - (1-momentum)*r
      w   = (1 - lr*wd_lh)*w + lr*sign(mom)

  ``sign(x) = (x > 0) - (x < 0)``: NaN and +-0 give 0.

* ``OracleSignum``            -- Signum.fused_step (python/mxnet/optimizer/signum.py:121-158) with the bookkeeping of
  ``oracle.OracleOptimizer``: per-index update counts from ``begin_num_update``, lr / wd multipliers, no bias
  correction.  State exists where momentum != 0 (``create_state``); signsgd_update runs where it does not, with
  ``wd + wd_lh`` (a double sum, ``wd_lh`` not multiplied by wd_mult) as its weight decay.  signum_update is handed the
  momentum only where it is > 0 and clip_gradient only where it is truthy (signum.py:144-147): a negative momentum runs
  at 0, a clip of 0, below 0 or None is off.  A 16-bit key is updated on its fp32 master and stored as its one rounding.

Every operation is one IEEE single-precision operation (numpy float32 element-wise arithmetic, no contraction into
FMAs), with the hyper-parameters rounded to float32 first, as the reference's float kernel parameters are; results
are bit-identical to the kernels' arithmetic (tests/test_signum.py checks that against the kernels' own source
compiled for the host), and pinned to the reference's own ``Signum.step`` by tests/golden/signum_steps.npz.
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


def sign(x):
    """(x > 0) - (x < 0) as float32: NaN and +-0 give 0"""
    x = np.asarray(x, np.float32)
    return (x > 0).astype(np.float32) - (x < 0).astype(np.float32)


def signsgd_update(w, g, lr, wd=0.0):
    """SignSGDKernel on float32 arrays; w updated in place"""
    w[...] = (_F(1.0) - _F(lr) * _F(wd)) * w - _F(lr) * sign(g)


def signum_update(w, g, mom, lr, wd=0.0, momentum=0.0, wd_lh=0.0, rescale=1.0, clip=None):
    """SignumKernel on float32 arrays; w and mom updated in place.  ``momentum`` / ``clip``: the operator's parameters
    (clip < 0 or None: off)"""
    w0 = w.copy()
    with np.errstate(invalid="ignore"):       # inf / NaN gradients propagate into mom as they do in the kernel
        r = _clip(_F(rescale) * np.asarray(g, np.float32), clip)
        r = r + _F(wd) * w0
        m = mom * _F(momentum)
        m = m - (_F(1.0) - _F(momentum)) * r
    mom[...] = m
    w[...] = (_F(1.0) - _F(lr) * _F(wd_lh)) * w0 + _F(lr) * sign(m)


def fused_clip(v):
    """signum.py:146-147: the clip the operator receives -- the option where it is truthy, else off"""
    return v if v else None


def fused_momentum(v):
    """signum.py:144-145: the momentum the operator receives -- the option where it is > 0, else the default 0"""
    return v if v > 0 else 0.0


class OracleSignum(object):
    """Signum.fused_step over float32 weights, updated in place; usable as ``OracleKVStore.set_optimizer(...)``.
    ``states[index]`` is ``(mom,)`` where momentum != 0 and ``()`` otherwise."""

    def __init__(self, learning_rate=0.01, momentum=0.9, wd_lh=0.0, wd=0.0, rescale_grad=1.0, clip_gradient=None,
                 lr_mult=None, wd_mult=None, begin_num_update=0, multi_precision=False):
        self.lr, self.momentum, self.wd_lh = learning_rate, momentum, wd_lh       # signum.py:67
        self.wd, self.rescale_grad, self.clip_gradient = wd, rescale_grad, clip_gradient
        self.lr_mult, self.wd_mult = dict(lr_mult or {}), dict(wd_mult or {})
        self.begin_num_update = begin_num_update
        self.count, self.states = {}, {}

    def state(self, index, like):
        if index not in self.states:
            self.states[index] = (np.zeros_like(like, np.float32),) if self.momentum != 0.0 else ()
        return self.states[index]

    def key_scalars(self, index):
        """(lr, wd) as the operator receives them, each rounded to float32 once"""
        lr = self.lr * self.lr_mult.get(index, 1.0)
        wd = self.wd * self.wd_mult.get(index, 1.0)
        if self.momentum == 0.0:
            wd += self.wd_lh                       # signum.py:156
        return float(np.float32(lr)), float(np.float32(wd))

    def _run(self, index, w, g):
        self.count[index] = self.count.get(index, self.begin_num_update) + 1
        st = self.state(index, w)
        lr, wd = self.key_scalars(index)
        if st:
            signum_update(w, g, st[0], lr, wd, fused_momentum(self.momentum), self.wd_lh, self.rescale_grad,
                          fused_clip(self.clip_gradient))
        else:
            signsgd_update(w, g, lr, wd)

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
