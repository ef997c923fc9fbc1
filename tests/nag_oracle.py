"""NAG for the CPU oracle (test infrastructure): the reference's fused kernels restated operation by operation on
float32 numpy arrays, and the optimizer bookkeeping that drives them.

* ``nag_mom_update``    -- NAGMomKernel (src/operator/optimizer_op-inl.h:1029-1044):
  ``r = clip(rescale*g) + wd*w;  mom = mom*momentum - lr*r;  out = (w + momentum*mom) - lr*r``
* ``mp_nag_mom_update`` -- MP_NAGMomKernel (:1066-1090), on the fp32 master of a 16-bit weight:
  the weight step is grouped ``w32 + (momentum*mom - lr*r)``, the 16-bit weight is its cast
* ``lp_nag_mom_update`` -- the fused engine on a 16-bit key without multi_precision: NAGMomKernel's grouping on the
  fp32 master, one rounding to the key type (the convention of every fused optimizer of the engine)
* ``OracleNAG``         -- NAG.fused_step (python/mxnet/optimizer/nag.py:111-154) with the bookkeeping of
  ``oracle.OracleOptimizer``: per-index update counts, lr / wd multipliers; momentum 0 is ``sgd_update`` without state

Every operation is one IEEE single-precision operation (numpy float32 element-wise arithmetic, no contraction into
FMAs), with the hyper-parameters rounded to float32 first, as the reference's float kernel parameters are; results
are bit-identical to the kernels' arithmetic (tests/test_nag.py checks that against the kernels' own source
compiled for the host), and pinned to the reference's own ``NAG.step`` by tests/golden/nag_steps.npz.
"""
import numpy as np

from oracle import oracle as O

_F = np.float32


def _grad(g, w, wd, rescale, clip):
    r = _F(rescale) * np.asarray(g, np.float32)
    c = -1.0 if clip is None else clip
    if c >= 0.0:                                   # mshadow_op::clip, mshadow_op.h:999-1009
        b = _F(c)
        r = np.where(r > b, b, np.where(r < -b, -b, r)).astype(np.float32)
    return r + _F(wd) * w


def _mom(mom, r, lr, momentum):
    m = mom * _F(momentum)
    m = m - _F(lr) * r
    mom[...] = m
    return m


def _store_lp(w_lp, lp_kind, w32):
    if w_lp is None or lp_kind == 0:
        return
    flat = w_lp.reshape(-1)
    if lp_kind == 1:
        flat[...] = w32.reshape(-1).astype(np.float16).view(np.uint16)
    else:
        flat[...] = O.f32_to_bf16(w32.reshape(-1))


def nag_mom_update(w, g, mom, lr, wd=0.0, momentum=0.0, rescale=1.0, clip=None):
    """NAGMomKernel on float32 arrays; w and mom updated in place"""
    w0 = w.copy()
    r = _grad(g, w0, wd, rescale, clip)
    m = _mom(mom, r, lr, momentum)
    w[...] = (w0 + _F(momentum) * m) - _F(lr) * r


def mp_nag_mom_update(w_lp, lp_kind, w32, mom, g32, lr, wd=0.0, momentum=0.0, rescale=1.0, clip=None):
    """MP_NAGMomKernel: fp32 master w32 and momentum in place; w_lp (uint16 bits; lp_kind 1 fp16, 2 bf16) = its cast"""
    w = w32.copy()
    r = _grad(g32, w, wd, rescale, clip)
    m = _mom(mom, r, lr, momentum)
    w32[...] = w + (_F(momentum) * m - _F(lr) * r)
    _store_lp(w_lp, lp_kind, w32)


def lp_nag_mom_update(w_lp, lp_kind, w32, mom, g32, lr, wd=0.0, momentum=0.0, rescale=1.0, clip=None):
    """the engine's NAG on a 16-bit key without multi_precision: NAGMomKernel's grouping on the fp32 master"""
    nag_mom_update(w32, g32, mom, lr, wd, momentum, rescale, clip)
    _store_lp(w_lp, lp_kind, w32)


class OracleNAG(object):
    """NAG.fused_step over float32 weights, updated in place; usable as ``OracleKVStore.set_optimizer(...)``."""

    def __init__(self, learning_rate=0.1, momentum=0.9, wd=0.0, rescale_grad=1.0, clip_gradient=None,
                 lr_mult=None, wd_mult=None, begin_num_update=0):
        self.lr, self.momentum, self.wd = learning_rate, momentum, wd     # nag.py:58
        self.rescale_grad, self.clip_gradient = rescale_grad, clip_gradient
        self.lr_mult, self.wd_mult = dict(lr_mult or {}), dict(wd_mult or {})
        self.begin_num_update = begin_num_update
        self.count, self.states = {}, {}

    def update(self, index, weight, grad):
        self.count[index] = self.count.get(index, self.begin_num_update) + 1
        lr = self.lr * self.lr_mult.get(index, 1.0)
        wd = self.wd * self.wd_mult.get(index, 1.0)
        if self.momentum == 0.0:                   # create_state -> None, fused_step -> sgd_update
            O.sgd_update(weight, grad, lr, wd, self.rescale_grad, self.clip_gradient)
            return
        if index not in self.states:
            self.states[index] = np.zeros_like(weight)
        nag_mom_update(weight, grad, self.states[index], lr, wd, self.momentum, self.rescale_grad, self.clip_gradient)
