"""The fused optimizers on float16 / bfloat16 keys, for the CPU oracle (test infrastructure).

``LpOracle`` drives the oracle's update kernels the way the engine drives its fused kernels on a 16-bit key: one
fp32 master per key (initialised from the 16-bit initial value), fp32 optimizer state, and the new weight rounded
once to the key type.  The master is persistent: it is kept whether or not the optimizer asked for
``multi_precision``, and the stored 16-bit weight is never widened again.  ``multi_precision`` only selects NAG's
operator grouping (MP_NAGMomKernel instead of NAGMomKernel).  ``kind = 0`` is a float32 key: the master is the
weight itself.

The bookkeeping is ``oracle.OracleOptimizer``'s: per-index update counts, lr / wd multipliers, Adam's host-side bias
correction (adam.py:166-175), AdamW's operator ``lr = 1`` / ``eta = bias-corrected lr`` (adamW.py:176-200) and its
skip on a 0 / inf / nan ``rescale_grad`` (contrib/adamw-inl.h:455).

``step_f64`` is an independent float64 restatement of the same operators (optimizer_op-inl.h SGDKernel,
SGDMomKernel, NAGMomKernel / MP_NAGMomKernel, AdamUpdateKernel; contrib/adamw-inl.h MPAdamWKernel; the Test
optimizer of optimizer.py:570-577).  It shares no code with the oracle and is meant for one step at a time: it
catches a formula error that the oracle and the kernels share, which a bit-exact comparison cannot.
"""
import numpy as np

from oracle import oracle as O

import nag_oracle as N

_F = np.float32

DEFAULT_LR = {"sgd": 0.1, "nag": 0.1, "adam": 0.001, "adamw": 0.001, "test": 0.01}


def to_lp(x, kind):
    """float32 values -> uint16 bit patterns of the key type (kind 1 fp16, 2 bf16); kind 0 returns float32"""
    x = np.ascontiguousarray(x, np.float32)
    if kind == 0:
        return x.copy()
    return x.astype(np.float16).view(np.uint16) if kind == 1 else O.f32_to_bf16(x)


def widen(bits, kind):
    """uint16 bit patterns (or float32 for kind 0) -> float32"""
    if kind == 0:
        return np.array(bits, np.float32, copy=True)
    bits = np.ascontiguousarray(bits).view(np.uint16)
    return bits.view(np.float16).astype(np.float32) if kind == 1 else O.bf16_to_f32(bits)


class LpOracle(object):
    """one optimizer over keys of one kind (0 float32, 1 float16, 2 bfloat16); ``update`` returns the expected
    weight: uint16 bit patterns for a 16-bit key, float32 values for a float32 one.  ``rewiden=True`` models the rule
    the engine does NOT follow (the master re-widened from the stored 16-bit weight before every step); tests use it
    to show that their data tells the two rules apart."""

    def __init__(self, name, kind, learning_rate=None, wd=0.0, rescale_grad=1.0, clip_gradient=None, momentum=None,
                 beta1=0.9, beta2=0.999, epsilon=None, eta=1.0, correct_bias=True, multi_precision=False,
                 lr_mult=None, wd_mult=None, rewiden=False):
        self.name, self.kind = name.lower(), kind
        self.lr = DEFAULT_LR[self.name] if learning_rate is None else learning_rate
        self.wd, self.rescale_grad, self.clip_gradient = wd, rescale_grad, clip_gradient
        self.momentum = (0.9 if self.name == "nag" else 0.0) if momentum is None else momentum
        self.beta1, self.beta2, self.eta, self.correct_bias = beta1, beta2, eta, correct_bias
        self.epsilon = (1e-6 if self.name == "adamw" else 1e-8) if epsilon is None else epsilon
        self.multi_precision, self.rewiden = multi_precision, rewiden
        self.lr_mult, self.wd_mult = dict(lr_mult or {}), dict(wd_mult or {})
        self.w32, self.s0, self.s1, self.count, self.out = {}, {}, {}, {}, {}

    def init(self, index, w0):
        """w0: the key's initial value (uint16 bits for a 16-bit key, float32 for a float32 one)"""
        self.w32[index] = widen(w0, self.kind).reshape(-1)
        self.out[index] = np.array(w0, copy=True).reshape(-1)
        n = self.w32[index].size
        self.s0[index] = np.zeros(n, np.float32)
        self.s1[index] = np.zeros(n, np.float32)
        self.count[index] = 0

    def scalars(self, index):
        """the per-key scalars the kernel receives for the NEXT update of ``index``: (lr, wd, eta) as Python
        floats, before their rounding to float32"""
        t = self.count[index] + 1
        lr = self.lr * self.lr_mult.get(index, 1.0)
        wd = self.wd * self.wd_mult.get(index, 1.0)
        eta = 1.0
        if self.name == "adam":
            lr = O.adam_lr(lr, self.beta1, self.beta2, t)
        elif self.name == "adamw":
            lr_c = O.adam_lr(lr, self.beta1, self.beta2, t) if self.correct_bias else lr
            lr, eta = 1.0, float(np.float32(lr_c * self.eta))
        return lr, wd, eta

    def update(self, index, grad32):
        lr, wd, eta = self.scalars(index)
        self.count[index] += 1
        g = np.ascontiguousarray(grad32, np.float32).reshape(-1)
        w32, s0, s1 = self.w32[index], self.s0[index], self.s1[index]
        if self.rewiden and self.kind != 0:
            w32[...] = widen(self.out[index], self.kind)
        lp = None if self.kind == 0 else np.zeros(w32.size, np.uint16)
        rs, clip, n = self.rescale_grad, self.clip_gradient, self.name
        if n == "adamw" and (not np.isfinite(rs) or rs == 0):
            return self.out[index].copy()
        if n == "sgd" or (n == "nag" and self.momentum == 0.0):
            if self.momentum == 0.0:
                O.mp_sgd_update(lp, self.kind, w32, g, lr, wd, rs, clip)
            else:
                O.mp_sgd_mom_update(lp, self.kind, w32, s0, g, lr, wd, self.momentum, rs, clip)
        elif n == "nag":
            upd = N.mp_nag_mom_update if (self.multi_precision and self.kind != 0) else N.lp_nag_mom_update
            upd(lp, self.kind, w32, s0, g, lr, wd, self.momentum, rs, clip)
        elif n == "adam":
            O.mp_adam_update(lp, self.kind, w32, s0, s1, g, lr, wd, self.beta1, self.beta2, self.epsilon, rs, clip)
        elif n == "adamw":
            O.mp_adamw_update(lp, self.kind, w32, s0, s1, g, lr, eta, wd, self.beta1, self.beta2, self.epsilon,
                              rs, clip)
        elif n == "test":
            # optimizer.py:570-577 as NDArray ops: every operation a separate float32 element-wise op
            gr = _F(rs) * g
            t = _F(wd) * w32
            s = gr + t
            u = _F(lr) * s
            w32[...] = w32 - u
        else:
            raise ValueError("unknown optimizer " + n)
        self.out[index] = w32.copy() if self.kind == 0 else to_lp(w32, self.kind)
        return self.out[index].copy()

    def hyper(self, index):
        """everything ``step_f64`` needs for the next update of ``index``, as the kernel receives it (float32)"""
        lr, wd, eta = self.scalars(index)
        f = lambda x: float(np.float32(x))                       # noqa: E731
        return dict(name=self.name, lr=f(lr), wd=f(wd), eta=f(eta), rescale=f(self.rescale_grad),
                    clip=None if self.clip_gradient is None else f(self.clip_gradient), momentum=f(self.momentum),
                    beta1=f(self.beta1), beta2=f(self.beta2), eps=f(self.epsilon),
                    mp=bool(self.multi_precision and self.kind != 0))


# ---------------------------------------------------------------------------
# float64 restatement of one step, with a rounding-error bound
# ---------------------------------------------------------------------------
def step_f64(h, w, g, s0, s1):
    """One step of optimizer ``h`` (``LpOracle.hyper``) in float64 on the fp32 master ``w``, state ``s0`` / ``s1``
    and gradient sum ``g`` (all widened to float64).  Returns (w_new, s0_new, s1_new, mag): ``mag`` is the same
    expression evaluated on absolute values, the scale the float32 rounding errors of the step are proportional to
    (a running error bound: each of the k roundings contributes at most 2^-24 of it)."""
    w, g = np.asarray(w, np.float64), np.asarray(g, np.float64)
    s0, s1 = np.asarray(s0, np.float64), np.asarray(s1, np.float64)
    n = h["name"]
    r = h["rescale"] * g
    if h["clip"] is not None and n != "test":
        r = np.clip(r, -h["clip"], h["clip"])
    ar = np.abs(r)
    with_momentum = n in ("sgd", "nag") and h["momentum"] != 0.0
    if n in ("sgd", "nag", "test") and not with_momentum:
        # SGDKernel / the Test optimizer: w - lr * (r + wd * w)
        d = h["lr"] * (r + h["wd"] * w)
        return w - d, s0, s1, np.abs(w) + h["lr"] * (ar + abs(h["wd"]) * np.abs(w))
    if n in ("sgd", "nag"):
        rr = r + h["wd"] * w
        arr = ar + abs(h["wd"]) * np.abs(w)
        m = h["momentum"] * s0 - h["lr"] * rr                   # SGDMomKernel / NAGMomKernel: the momentum
        am = h["momentum"] * np.abs(s0) + h["lr"] * arr
        if n == "sgd":
            return w + m, m, s1, np.abs(w) + am
        # NAGMomKernel (w + momentum*m) - lr*r; MP_NAGMomKernel w + (momentum*m - lr*r): the same real number
        return w + h["momentum"] * m - h["lr"] * rr, m, s1, np.abs(w) + h["momentum"] * am + h["lr"] * arr
    if n == "adam":
        # AdamUpdateKernel: r = rescale*g (clipped) + wd*w; m, v; w - lr * m / (sqrt(v) + eps)
        rr = r + h["wd"] * w
        arr = ar + abs(h["wd"]) * np.abs(w)
        m = h["beta1"] * s0 + (1.0 - h["beta1"]) * rr
        v = h["beta2"] * s1 + (1.0 - h["beta2"]) * rr * rr
        am = h["beta1"] * np.abs(s0) + (1.0 - h["beta1"]) * arr
        av = h["beta2"] * np.abs(s1) + (1.0 - h["beta2"]) * arr * arr
        den = np.sqrt(v) + h["eps"]
        return (w - h["lr"] * m / den, m, v,
                np.abs(w) + h["lr"] * am / den * (1.0 + np.where(v > 0, av / np.where(v > 0, v, 1.0), 0.0)))
    if n == "adamw":
        # MPAdamWKernel: no wd in the gradient; w - eta * (lr * m / (sqrt(v) + eps) + wd * w)
        m = h["beta1"] * s0 + (1.0 - h["beta1"]) * r
        v = h["beta2"] * s1 + (1.0 - h["beta2"]) * r * r
        am = h["beta1"] * np.abs(s0) + (1.0 - h["beta1"]) * ar
        av = h["beta2"] * np.abs(s1) + (1.0 - h["beta2"]) * ar * ar
        den = np.sqrt(v) + h["eps"]
        step = h["lr"] * m / den + h["wd"] * w
        astep = h["lr"] * am / den * (1.0 + np.where(v > 0, av / np.where(v > 0, v, 1.0), 0.0)) + \
            abs(h["wd"]) * np.abs(w)
        return w - h["eta"] * step, m, v, np.abs(w) + h["eta"] * astep
    raise ValueError("unknown optimizer " + n)


# 2^-24-roundings of the step's magnitude allowed beyond the result's own half ulp.  The longest chain of any
# operator above (Adam's weight step) has 12 roundings, but their errors do not line up: one step on uniform data
# needs at most 1.6 of them for every optimizer and key type (tests/test_lp_oracle.py).  8 leaves a factor of 5.
ROUNDINGS = 8


def f64_bound(w_new64, mag):
    """|float32 result - float64 result| allowed: half an ulp of the result (its own rounding) plus ROUNDINGS
    roundings of 2^-24 relative to the magnitude of the step's terms"""
    ulp_half = np.spacing(np.abs(w_new64).astype(np.float32)).astype(np.float64) / 2
    return ulp_half + ROUNDINGS * 2.0 ** -24 * mag


def assert_close_f64(got32, want64, mag, msg=""):
    got = np.asarray(got32, np.float32).astype(np.float64).reshape(-1)
    want64, mag = np.asarray(want64).reshape(-1), np.asarray(mag).reshape(-1)
    err = np.abs(got - want64)
    bound = f64_bound(want64, mag)
    bad = err > bound
    assert not bad.any(), "%s: %d / %d elements beyond the float64 bound, worst err / bound %.3g" % (
        msg, bad.sum(), bad.size, (err / np.maximum(bound, 1e-300)).max())
    return float((err / np.maximum(bound, 1e-300)).max())
