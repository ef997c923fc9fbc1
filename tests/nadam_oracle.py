"""Nadam for the CPU oracle (test infrastructure): the reference's ``Nadam.step`` restated operation by operation on
float32 numpy arrays, and the optimizer bookkeeping that drives it.  The reference has no operator for Nadam (its
``use_fused_step`` defaults to False and there is no ``fused_step``), so ``step`` itself is the definition.

* ``nadam_scalars``           -- nadam.py:95-101 in double for update count t and the optimizer's momentum-schedule
  product ``m_schedule`` as it stands before this update: returns the advanced product (a double, the caller's state)
  and the per-key scalars the engine hands the kernel, each rounded once to float32 (KVStore::KeyEta /
  KVStore::NadamAdvance)::

      coef2 = 1 - beta2**t
      momentum_t   = beta1 * (1 - 0.5 * 0.96**(t * schedule_decay))
      momentum_t_1 = beta1 * (1 - 0.5 * 0.96**((t + 1) * schedule_decay))
      m_schedule = m_schedule * momentum_t;  m_schedule_next = m_schedule * momentum_t_1
      -> (1 - m_schedule, 1 - m_schedule_next, momentum_t_1, 1 - momentum_t, coef2)

* ``nadam_update``            -- nadam.py:86-124, states ``mean``, ``var``::

      r    = clip(g*rescale) + wd*w
      mean = mean*beta1 + (1 - beta1)*r
      var  = var*beta2 + (1 - beta2)*square(r)
      w    = w - lr*((momentum_t_1*(mean / (1 - m_next)) + (1 - momentum_t)*(r / (1 - m_schedule)))
                     / (sqrt(var / coef2) + eps))

* ``OracleNadam``             -- the bookkeeping of ``oracle.OracleOptimizer`` plus the ONE ``m_schedule`` of the
  optimizer, advanced by every update in the order the caller makes them (an ``OracleKVStore`` push: sorted keys).

Every operation is one IEEE single-precision operation (numpy float32 element-wise arithmetic, no contraction into
FMAs), and every Python scalar is rounded to float32 from its double, as an NDArray operation receives it; results are
bit-identical to the kernel's arithmetic (tests/test_nadam.py checks that against the kernel's own source compiled
for the host) and to the reference's own ``Nadam.step`` (tests/golden/nadam_steps.npz).
"""
import numpy as np

from adamax_oracle import OracleTwoState, prep_grad

_F = np.float32


def nadam_scalars(beta1, beta2, schedule_decay, t, m_schedule):
    """(m_schedule after this update, (g_div, m_div, mom_t1, c_mom_t, coef2) as float32) for update count ``t``"""
    coef2 = 1. - beta2 ** t
    momentum_t = beta1 * (1. - 0.5 * (pow(0.96, t * schedule_decay)))
    momentum_t_1 = beta1 * (1. - 0.5 * (pow(0.96, (t + 1) * schedule_decay)))
    m_schedule = m_schedule * momentum_t
    m_next = m_schedule * momentum_t_1
    return m_schedule, (_F(1. - m_schedule), _F(1. - m_next), _F(momentum_t_1), _F(1. - momentum_t), _F(coef2))


def nadam_update(w, g, mean, var, lr_op, sc, wd=0.0, beta1=0.9, beta2=0.999, eps=1e-8, rescale=1.0, clip=None):
    """Nadam.step on float32 arrays with the per-key scalars ``sc`` of ``nadam_scalars``; w, mean, var in place"""
    g_div, m_div, mom_t1, c_mom_t, coef2 = sc
    with np.errstate(all="ignore"):
        r = prep_grad(g, w, wd, rescale, clip)
        m = mean * _F(beta1) + _F(1. - beta1) * r
        v = var * _F(beta2) + _F(1. - beta2) * np.square(r)
        mean[...] = m
        var[...] = v
        gp = r / g_div
        mp = m / m_div
        vp = v / coef2
        mb = mom_t1 * mp + c_mom_t * gp
        w[...] = w - _F(lr_op) * (mb / (np.sqrt(vp) + _F(eps)))


class OracleNadam(OracleTwoState):
    """Nadam.step over float32 weights, updated in place.  ``states[index]`` is ``(mean, var)``; ``m_schedule`` is
    the optimizer's one momentum-schedule product, advanced by every update."""

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, schedule_decay=0.004,
                 m_schedule=1., **kw):     # nadam.py:58-67
        super(OracleNadam, self).__init__(learning_rate, **kw)
        self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon
        self.schedule_decay, self.m_schedule = schedule_decay, m_schedule

    def key_scalars(self, index, t=None):
        """(lr_op, wd, coef2) as the kernel receives them in its work entry for update count ``t`` (default: the
        index's current one) -- what MXKVB200GetKeyHyper reports"""
        t = self.count.get(index, self.begin_num_update) if t is None else t
        lr, wd = self._lr_wd(index)
        return _F(lr), _F(wd), _F(1. - self.beta2 ** t)

    def _apply(self, index, w, g, st):
        t = self.count[index]
        lr, wd = self._lr_wd(index)
        self.m_schedule, sc = nadam_scalars(self.beta1, self.beta2, self.schedule_decay, t, self.m_schedule)
        nadam_update(w, g, st[0], st[1], _F(lr), sc, wd, self.beta1, self.beta2, self.epsilon, self.rescale_grad,
                     self.clip_gradient)
