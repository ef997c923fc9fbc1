"""AdaDelta for the CPU oracle (test infrastructure): the reference's ``AdaDelta.step`` restated operation by operation
on float32 numpy arrays.  The reference has no operator for AdaDelta (its ``use_fused_step`` defaults to False and
there is no ``fused_step``), so ``step`` itself is the definition.

* ``adadelta_scalars``        -- the per-key scalars the engine hands the kernel (KVStore::KeyScalars):
  ``lr_op = float32(lr)`` with ``lr`` the double learning rate x lr_mult, and ``eta_op = float32(1 - rho)``, the
  complement ``step`` writes as ``(1. - self.rho) * square(...)``, computed in double and rounded once.

* ``adadelta_update``         -- adadelta.py:90-111, states ``acc_g``, ``acc_delta``::

      r         = clip(g*rescale) + wd*w
      acc_g     = acc_g*rho + eta_op*(r*r)
      delta     = sqrt(acc_delta + eps);  delta = delta / sqrt(acc_g + eps);  delta = delta*r   (the OLD acc_delta)
      acc_delta = acc_delta*rho + eta_op*(delta*delta)
      w         = w - lr_op*delta

* ``OracleAdaDelta``          -- the bookkeeping of tests/adamax_oracle.py's ``OracleTwoState``.

Every operation is one IEEE single-precision operation and every Python scalar is rounded to float32 from its double,
as an NDArray operation receives it; bit-identical to the kernel's arithmetic (tests/test_adadelta.py) and to the
reference's own ``AdaDelta.step`` (tests/golden/adadelta_steps.npz).
"""
import numpy as np

from adamax_oracle import OracleTwoState, prep_grad

_F = np.float32


def adadelta_scalars(lr, rho):
    """(lr_op, eta_op) for the double learning rate ``lr`` (lr x lr_mult)"""
    return _F(lr), _F(1. - rho)


def adadelta_update(w, g, acc_g, acc_delta, lr_op, eta_op, wd=0.0, rho=0.9, eps=1e-6, rescale=1.0, clip=None):
    """AdaDelta.step on float32 arrays; w, acc_g and acc_delta updated in place"""
    with np.errstate(all="ignore"):
        r = prep_grad(g, w, wd, rescale, clip)
        ag = acc_g * _F(rho) + _F(eta_op) * (r * r)
        cd = np.sqrt(acc_delta + _F(eps))
        cd = cd / np.sqrt(ag + _F(eps))
        cd = cd * r
        ad = acc_delta * _F(rho) + _F(eta_op) * (cd * cd)
        acc_g[...] = ag
        acc_delta[...] = ad
        w[...] = w - _F(lr_op) * cd


class OracleAdaDelta(OracleTwoState):
    """AdaDelta.step over float32 weights, updated in place.  ``states[index]`` is ``(acc_g, acc_delta)``."""

    def __init__(self, learning_rate=1.0, rho=0.9, epsilon=1e-6, **kw):      # adadelta.py:62
        super(OracleAdaDelta, self).__init__(learning_rate, **kw)
        self.rho, self.epsilon = rho, epsilon

    def key_scalars(self, index, t=None):
        """(lr_op, wd, eta_op) as the kernel receives them; none depends on the update count ``t``"""
        lr, wd = self._lr_wd(index)
        lr_op, eta_op = adadelta_scalars(lr, self.rho)
        return lr_op, _F(wd), eta_op

    def _apply(self, index, w, g, st):
        lr_op, wd, eta_op = self.key_scalars(index)
        adadelta_update(w, g, st[0], st[1], lr_op, eta_op, wd, self.rho, self.epsilon, self.rescale_grad,
                        self.clip_gradient)
