"""FTML for the CPU oracle (test infrastructure): the reference's fused kernel restated operation by operation on float32
numpy arrays, and the optimizer bookkeeping that drives it.

* ``ftml_scalars``            -- the two per-key scalars the engine hands the kernel for update count t
  (KVStore::KeyScalars): ``t`` cast to float as the operator casts it, ``p = float(pow(float(beta), t))`` computed
  in double and rounded once, then ``lr_op = (1 - p1) / lr`` and ``eta_op = 1 - p2`` in float -- the operator's
  ``(1 - pow(beta1, t)) / lr`` and ``1 - pow(beta2, t)``, evaluated once per key.

* ``ftml_update``             -- FTMLKernel (src/operator/optimizer_op-inl.h:1159-1177), states ``d``, ``v``, ``z``::

      r   = clip(rescale*g) + wd*w                   (weight decay AFTER the clip)
      v   = beta2*v + (1-beta2)*(r*r)
      d_t = lr_op * (sqrt(v / eta_op) + eps)
      z   = (beta1*z + (1-beta1)*r) - (d_t - beta1*d)*w
      d   = d_t
      w   = -z / d_t

* ``OracleFTML``              -- FTML.fused_step (python/mxnet/optimizer/ftml.py:127-158) with the bookkeeping of
  ``oracle.OracleOptimizer``: per-index update counts from ``begin_num_update``, lr / wd multipliers, and the operator's
  clip switched on only where ``clip_gradient`` is truthy (ftml.py:152-153): 0, a negative value or None is off.  A
  16-bit key is updated on its fp32 master and stored as its one rounding.

Every operation is one IEEE single-precision operation (numpy float32 element-wise arithmetic, no contraction into
FMAs), with the hyper-parameters rounded to float32 first, as the reference's float kernel parameters are; results
are bit-identical to the kernel's arithmetic (tests/test_ftml.py checks that against the kernel's own source compiled
for the host), and pinned to the reference's own ``FTML.step`` by tests/golden/ftml_steps.npz.
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


def ftml_scalars(lr, beta1, beta2, t):
    """(lr_op, eta_op) for update count ``t`` and the float32 learning rate ``lr`` (lr x lr_mult, rounded once)"""
    tf = float(_F(t))
    p1 = _F(float(_F(beta1)) ** tf)
    p2 = _F(float(_F(beta2)) ** tf)
    return _F(_F(1.0) - p1) / _F(lr), _F(1.0) - p2


def ftml_update(w, g, d, v, z, lr_op, eta_op, wd=0.0, beta1=0.6, beta2=0.999, eps=1e-8, rescale=1.0, clip=None):
    """FTMLKernel on float32 arrays; w, d, v and z updated in place.  ``clip``: the operator's clip_grad (< 0 or
    None: off)"""
    with np.errstate(all="ignore"):
        w0 = w.copy()
        r = _clip(_F(rescale) * np.asarray(g, np.float32), clip) + _F(wd) * w0
        b1, b2 = _F(beta1), _F(beta2)
        nv = b2 * v + (_F(1.0) - b2) * (r * r)
        dt = _F(lr_op) * (np.sqrt(nv / _F(eta_op)) + _F(eps))
        nz = (b1 * z + (_F(1.0) - b1) * r) - (dt - b1 * d) * w0
        v[...] = nv
        z[...] = nz
        d[...] = dt
        w[...] = -nz / dt


def fused_clip(v):
    """ftml.py:152-153: the clip the operator receives -- the option where it is truthy, else off"""
    return v if v else None


class OracleFTML(object):
    """FTML.fused_step over float32 weights, updated in place; usable as ``OracleKVStore.set_optimizer(...)``.
    ``states[index]`` is ``(d, v, z)``, the tuple order of the reference's create_state."""

    def __init__(self, learning_rate=0.0025, beta1=0.6, beta2=0.999, epsilon=1e-8, wd=0.0, rescale_grad=1.0,
                 clip_gradient=None, lr_mult=None, wd_mult=None, begin_num_update=0, multi_precision=False):
        self.lr, self.beta1, self.beta2, self.epsilon = learning_rate, beta1, beta2, epsilon     # ftml.py:66
        self.wd, self.rescale_grad, self.clip_gradient = wd, rescale_grad, clip_gradient
        self.lr_mult, self.wd_mult = dict(lr_mult or {}), dict(wd_mult or {})
        self.begin_num_update = begin_num_update
        self.count, self.states = {}, {}

    def state(self, index, like):
        if index not in self.states:
            self.states[index] = tuple(np.zeros_like(like, np.float32) for _ in range(3))
        return self.states[index]

    def key_scalars(self, index, t=None):
        """(lr_op, wd, eta_op) as the kernel receives them for update count ``t`` (default: the index's current one)"""
        t = self.count.get(index, self.begin_num_update) if t is None else t
        lr = float(_F(self.lr * self.lr_mult.get(index, 1.0)))
        wd = float(_F(self.wd * self.wd_mult.get(index, 1.0)))
        lr_op, eta_op = ftml_scalars(lr, self.beta1, self.beta2, t)
        return lr_op, _F(wd), eta_op

    def _run(self, index, w, g):
        self.count[index] = self.count.get(index, self.begin_num_update) + 1
        d, v, z = self.state(index, w)
        lr_op, wd, eta_op = self.key_scalars(index)
        ftml_update(w, g, d, v, z, lr_op, eta_op, wd, self.beta1, self.beta2, self.epsilon, self.rescale_grad,
                    fused_clip(self.clip_gradient))

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
