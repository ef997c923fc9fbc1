"""tests/lp_oracle.py, the expected values of tests/test_gpu_lowp_optimizers.py, checked without a GPU: on float32
keys it is the existing oracle bit for bit, and one step of every optimizer on float32 / float16 / bfloat16 keys
agrees with the float64 restatement of the operator within the stated bound."""
import os
import sys

import numpy as np
import pytest

from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import lp_oracle as L  # noqa: E402
import nag_oracle as N  # noqa: E402

E = 20011
KW = {
    "sgd": dict(learning_rate=0.1, wd=1e-3, rescale_grad=0.5, clip_gradient=0.6),
    "sgd_mom": dict(learning_rate=0.05, momentum=0.9, wd=1e-3, rescale_grad=0.5, clip_gradient=0.6),
    "nag": dict(learning_rate=0.05, momentum=0.9, wd=1e-3, rescale_grad=0.5, clip_gradient=0.6),
    "adam": dict(learning_rate=0.01, wd=1e-3, rescale_grad=0.5, clip_gradient=0.6),
    "adamw": dict(learning_rate=0.01, wd=1e-2, rescale_grad=0.5, clip_gradient=0.6, eta=0.7),
    "test": dict(learning_rate=0.1, wd=1e-3, rescale_grad=0.5),
}
NAME = {"sgd_mom": "sgd"}


def _data(seed, steps=4):
    rng = np.random.default_rng(seed)
    w0 = rng.uniform(-1, 1, E).astype(np.float32)
    grads = [(2 * rng.uniform(-1, 1, E)).astype(np.float32) for _ in range(steps)]
    return w0, grads


@pytest.mark.parametrize("optkey", list(KW))
def test_float32_keys_are_the_existing_oracle(optkey):
    """kind 0: O.sgd_update / sgd_mom_update / adam_update / test_update, OracleNAG and OracleOptimizer('adamw')
    bit for bit, with lr_mult / wd_mult on one index"""
    name, kw = NAME.get(optkey, optkey), KW[optkey]
    w0, grads = _data(1)
    mults = ({0: 0.5}, {0: 2.0})
    lo = L.LpOracle(name, 0, lr_mult=mults[0], wd_mult=mults[1], **kw)
    lo.init(0, w0)
    w, s0, s1 = w0.copy(), np.zeros(E, np.float32), np.zeros(E, np.float32)
    ref = None
    if name == "nag":
        ref = N.OracleNAG(lr_mult=mults[0], wd_mult=mults[1], **kw)
    elif name == "adamw":
        ref = O.OracleOptimizer("adamw", lr_mult=mults[0], wd_mult=mults[1], **kw)
    clip = kw.get("clip_gradient")
    for t, g in enumerate(grads, 1):
        lr, wd = kw["learning_rate"] * 0.5, kw["wd"] * 2.0
        if ref is not None:
            ref.update(0, w, g)
        elif optkey == "sgd":
            O.sgd_update(w, g, lr, wd, kw["rescale_grad"], clip)
        elif optkey == "sgd_mom":
            O.sgd_mom_update(w, g, s0, lr, wd, kw["momentum"], kw["rescale_grad"], clip)
        elif optkey == "adam":
            O.adam_update(w, g, s0, s1, O.adam_lr(lr, 0.9, 0.999, t), wd, 0.9, 0.999, 1e-8, kw["rescale_grad"], clip)
        else:
            O.test_update(w, g, lr, wd, kw["rescale_grad"])
        got = lo.update(0, g)
        assert np.array_equal(got.view(np.uint32), w.view(np.uint32)), "%s step %d" % (optkey, t)


def test_sixteen_bit_keys_round_the_master_once():
    """the 16-bit result is the persistent master rounded once; the master is what the float32 oracle computes
    from the widened initial value"""
    w0, grads = _data(2)
    for kind in (1, 2):
        init = L.to_lp(w0, kind)
        lo = L.LpOracle("adam", kind, **KW["adam"])
        lo.init(0, init)
        w = L.widen(init, kind)
        s0, s1 = np.zeros(E, np.float32), np.zeros(E, np.float32)
        for t, g in enumerate(grads, 1):
            got = lo.update(0, g)
            O.adam_update(w, g, s0, s1, O.adam_lr(0.01, 0.9, 0.999, t), 1e-3, 0.9, 0.999, 1e-8, 0.5, 0.6)
            assert np.array_equal(lo.w32[0].view(np.uint32), w.view(np.uint32))
            assert np.array_equal(got, L.to_lp(w, kind))


def test_adamw_skip_keeps_everything():
    w0, grads = _data(3, 2)
    lo = L.LpOracle("adamw", 2, **dict(KW["adamw"], rescale_grad=0.0))
    lo.init(0, L.to_lp(w0, 2))
    before = lo.w32[0].copy()
    out = lo.update(0, grads[0])
    assert np.array_equal(out, L.to_lp(w0, 2)) and np.array_equal(lo.w32[0], before) and lo.count[0] == 1


@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("optkey", list(KW))
def test_one_step_against_float64(optkey, kind):
    """after two steps (non-zero state), the third step of the oracle's master against step_f64 within
    f64_bound; the largest error / bound ratio seen here is well under 1 (the bound is not loose by orders of
    magnitude either: see test_float64_bound_is_not_vacuous)"""
    name, kw = NAME.get(optkey, optkey), KW[optkey]
    w0, grads = _data(4 + kind, 3)
    for mp in (False, True):
        lo = L.LpOracle(name, kind, multi_precision=mp, **kw)
        lo.init(0, L.to_lp(w0, kind))
        for g in grads[:2]:
            lo.update(0, g)
        h = lo.hyper(0)
        w, s0, s1 = lo.w32[0].copy(), lo.s0[0].copy(), lo.s1[0].copy()
        lo.update(0, grads[2])
        want, _, _, mag = L.step_f64(h, w, grads[2], s0, s1)
        ratio = L.assert_close_f64(lo.w32[0], want, mag, "%s kind %d mp %s" % (optkey, kind, mp))
        assert ratio < 0.5, ratio


def test_float64_bound_is_not_vacuous():
    """the bound is tight enough to catch a wrong formula: AdamW with Adam's coupled weight decay, or a step with
    another epsilon, falls outside it"""
    w0, grads = _data(9, 2)
    lo = L.LpOracle("adamw", 0, **KW["adamw"])
    lo.init(0, w0)
    lo.update(0, grads[0])
    h = lo.hyper(0)
    w, s0, s1 = lo.w32[0].copy(), lo.s0[0].copy(), lo.s1[0].copy()
    lo.update(0, grads[1])
    wrong = L.LpOracle("adam", 0, **dict(KW["adamw"], eta=1.0))   # Adam's coupled weight decay
    wrong.init(0, w)
    wrong.s0[0][...], wrong.s1[0][...] = s0, s1
    wrong.count[0] = 1
    wrong.lr = KW["adamw"]["learning_rate"] * 0.7
    wrong.update(0, grads[1])
    want, _, _, mag = L.step_f64(h, w, grads[1], s0, s1)
    with pytest.raises(AssertionError):
        L.assert_close_f64(wrong.w32[0], want, mag)
    h2 = dict(h, eps=1e-3)
    want2, _, _, mag2 = L.step_f64(h2, w, grads[1], s0, s1)
    with pytest.raises(AssertionError):
        L.assert_close_f64(lo.w32[0], want2, mag2)
