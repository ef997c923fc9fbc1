"""Adamax for the CPU oracle (test infrastructure): the reference's ``Adamax.step`` restated operation by operation on
float32 numpy arrays, and the optimizer bookkeeping that drives it.  The reference has no operator for Adamax (its
``use_fused_step`` defaults to False and there is no ``fused_step``), so ``step`` itself is the definition.

* ``adamax_scalars``          -- the two per-key scalars the engine hands the kernel for update count t
  (KVStore::KeyScalars): ``lr_op = float32(lr / (1 - beta1**t))`` with ``lr`` the double learning rate x lr_mult
  (adamax.py:91-93), and ``eta_op = float32(1 - beta1)``, the complement ``step`` writes as ``(1. - self.beta1) *
  grad`` -- both computed in double and rounded once.

* ``adamax_update``           -- adamax.py:95-111, states ``mean``, ``var`` (the max-norm u)::

      r    = clip(g*rescale) + wd*w
      mean = mean*beta1 + eta_op*r
      var  = maximum(beta2*var, |r|)            (mshadow_op::maximum: NaN in either operand gives NaN)
      w    = w - lr_op*(mean / (var + eps))

* ``OracleAdamax``            -- the bookkeeping of ``oracle.OracleOptimizer``: per-index update counts from
  ``begin_num_update``, lr / wd multipliers, and the clip on wherever ``clip_gradient`` is not None and >= 0 (``step``
  clips at 0 too).  A 16-bit key is updated on its fp32 master and stored as its one rounding.

Every operation is one IEEE single-precision operation (numpy float32 element-wise arithmetic, no contraction into
FMAs), and every Python scalar is rounded to float32 from its double, as an NDArray operation receives it; results are
bit-identical to the kernel's arithmetic (tests/test_adamax.py checks that against the kernel's own source compiled
for the host) and to the reference's own ``Adamax.step`` (tests/golden/adamax_steps.npz).
"""
import numpy as np

from oracle import oracle as O

_F = np.float32


def clip_on(c):
    """the clip the kernel applies: ``step`` clips whenever clip_gradient is not None; a negative bound is off"""
    return c is not None and c >= 0.0


def prep_grad(g, w, wd, rescale, clip):
    """``grad *= rescale_grad; grad = clip(grad, -c, c); grad += wd * weight`` -- mshadow_op::clip where the bound is
    on (NaN passes through)"""
    r = np.asarray(g, np.float32) * _F(rescale)
    if clip_on(clip):
        b = _F(clip)
        r = np.where(r > b, b, np.where(r < -b, -b, r)).astype(np.float32)
    return r + _F(wd) * w


def maximum(a, b):
    """mshadow_op::maximum (mshadow_op.h:1266-1275): ``isnan(a) ? a : (a > b ? a : b)``"""
    return np.where(np.isnan(a), a, np.where(a > b, a, b)).astype(np.float32)


def adamax_scalars(lr, beta1, t):
    """(lr_op, eta_op) for update count ``t`` and the double learning rate ``lr`` (lr x lr_mult)"""
    return _F(lr / (1. - beta1 ** t)), _F(1. - beta1)


def adamax_update(w, g, mean, var, lr_op, eta_op, wd=0.0, beta1=0.9, beta2=0.999, eps=1e-8, rescale=1.0, clip=None):
    """Adamax.step on float32 arrays; w, mean and var updated in place"""
    with np.errstate(all="ignore"):
        r = prep_grad(g, w, wd, rescale, clip)
        m = mean * _F(beta1) + _F(eta_op) * r
        u = maximum(_F(beta2) * var, np.abs(r))
        mean[...] = m
        var[...] = u
        w[...] = w - _F(lr_op) * (m / (u + _F(eps)))


class OracleTwoState(object):
    """The bookkeeping both step-defined kinds share (this file and tests/adadelta_oracle.py): update counts, lr / wd
    multipliers, two float32 states per index in the tuple order of the reference's create_state; usable as
    ``OracleKVStore.set_optimizer(...)``."""

    def __init__(self, learning_rate, wd=0.0, rescale_grad=1.0, clip_gradient=None, lr_mult=None, wd_mult=None,
                 begin_num_update=0, multi_precision=False):
        self.lr, self.wd, self.rescale_grad, self.clip_gradient = learning_rate, wd, rescale_grad, clip_gradient
        self.lr_mult, self.wd_mult = dict(lr_mult or {}), dict(wd_mult or {})
        self.begin_num_update = begin_num_update
        self.count, self.states = {}, {}

    def state(self, index, like):
        if index not in self.states:
            self.states[index] = tuple(np.zeros_like(like, np.float32) for _ in range(2))
        return self.states[index]

    def _lr_wd(self, index):
        """Optimizer._get_lr / _get_wd: the multipliers applied in double"""
        return self.lr * self.lr_mult.get(index, 1.0), self.wd * self.wd_mult.get(index, 1.0)

    def _run(self, index, w, g):
        self.count[index] = self.count.get(index, self.begin_num_update) + 1
        self._apply(index, w, g, self.state(index, w))

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


class OracleAdamax(OracleTwoState):
    """Adamax.step over float32 weights, updated in place.  ``states[index]`` is ``(mean, var)``."""

    def __init__(self, learning_rate=0.002, beta1=0.9, beta2=0.999, epsilon=1e-8, **kw):     # adamax.py:61
        super(OracleAdamax, self).__init__(learning_rate, **kw)
        self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon

    def key_scalars(self, index, t=None):
        """(lr_op, wd, eta_op) as the kernel receives them for update count ``t`` (default: the index's current one)"""
        t = self.count.get(index, self.begin_num_update) if t is None else t
        lr, wd = self._lr_wd(index)
        lr_op, eta_op = adamax_scalars(lr, self.beta1, t)
        return lr_op, _F(wd), eta_op

    def _apply(self, index, w, g, st):
        lr_op, wd, eta_op = self.key_scalars(index)
        adamax_update(w, g, st[0], st[1], lr_op, eta_op, wd, self.beta1, self.beta2, self.epsilon, self.rescale_grad,
                      self.clip_gradient)
