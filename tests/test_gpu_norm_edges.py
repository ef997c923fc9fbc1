"""LAMB, LANS and LARS (csrc/norm_kernels.cu, csrc/kvstore_norm.cc::LaunchNormWorks) and the stand-alone
multi_sum_sq / multi_all_finite reductions at the edges of their kernels: blocks that walk many chunks and many
keys (a small chunk and a small grid), trust ratios recovered from the update itself, zero norms, float32 keys
on the multi-precision instantiations, several launch classes in one push, the whole-key scalar path, non-finite
bit patterns at chunk boundaries, and arrays above 2^31 elements.

Reference.  Every step is recomputed from the kernel's own weight and state before that step with the CPU oracle's
element arithmetic (``oracle.py``: the reference's step 1 / step 2 kernels) and its sums of squares taken in float64
and rounded once (``norm_mode='f64'``).  What does not depend on a norm is compared bit for bit: LAMB / LANS mean
and var, the copy-out of a multi-precision master, skipped steps, keys whose trust ratio is 1.  LANS gradients are
+-1/4 or +-1/2 with one sign per element across the sources, so every partial sum of their squares is exact in
float32 (6 sources over 65 539 elements stay below 2^24 sixteenths) and g_norm -- and with it LANS' mean, var and
directions -- is the same in any summation order.

The bound.  A sum of squares of non-negative terms computed as a tree of float32 additions has a relative error of
at most D * 2^-24, D the longest chain of roundings from a term to the total (``_depth``): the square itself (1),
a thread's sequential partial over its elements of one chunk (ceil(min(chunk, n) / 512) + 4: vector iterations of
four, the scalar tail), 5 warp-shuffle levels, the 16 warp totals in order, the finalize kernel's ceil(chunks / 256)
strided terms per thread, its own 5 shuffle levels and 8 warp totals, and one addition per contributing rank.  A
ratio of two square roots of such sums is then off by at most D * 2^-24 relative, plus a few roundings of its own
(square roots, quotient, product with lr) on the kernel's side and the oracle's: ``_ratio_eps`` = (D + 6) * 2^-24.
Weights (and LARS momenta) may differ from the oracle by that relative error times the size of the step, plus two
ulps of the result for the final roundings.  ``WORST`` records the largest error / bound of each kind of check; it
is printed at the end of the module (``-s``).
"""
import math
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import mxnet_b200 as mx
from oracle import oracle as O

SIM = bool(os.environ.get("MXKV_SIM"))
U = 2.0 ** -24
G = mx.gpu(0)
WORST = {}


def _note(what, frac):
    WORST[what] = max(WORST.get(what, 0.0), float(frac))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print("norm-edges worst fraction of bound  %-28s %.3g" % (k, WORST[k]))


def _default_chunk():
    """the chunk the runtime starts with (runtime.cc: MXKV_B200_CHUNK, at least 128, rounded up to 128)"""
    c = int(os.environ.get("MXKV_B200_CHUNK", "8192"))
    return (max(c, 128) + 127) // 128 * 128


@pytest.fixture
def tuning():
    """set_tuning for one test; the chunk and grid every later test expects are restored whatever happens"""
    try:
        yield mx.kv.set_tuning
    finally:
        mx.kv.set_tuning(chunk_elems=_default_chunk(), max_blocks=int(os.environ.get("MXKV_B200_MAX_BLOCKS", "0")))


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def _bits_equal(a, b):
    return np.array_equal(_bits(np.asarray(a)), _bits(np.asarray(b)))


def _state(kv, key, which):
    h = kv._state_handle(key, which)
    return None if h is None else h.asnumpy()


def _ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


def _ss64(x):
    x = np.asarray(x, np.float64).ravel()
    return float(np.dot(x, x))


def _depth(n, chunk, ranks=1):
    nch = -(-n // chunk)
    return 1 + (-(-min(chunk, n) // 512) + 4) + 5 + 16 + (-(-nch // 256)) + 5 + 8 + ranks


def _ratio_eps(n, chunk, ranks=1):
    return (_depth(n, chunk, ranks) + 6) * U


def _to_lp(x, kind):
    return O.f32_to_bf16(x) if kind == 2 else np.asarray(x, np.float32).astype(np.float16).view(np.uint16)


def _lp_f32(h, kind):
    return O.bf16_to_f32(h) if kind == 2 else np.asarray(h, np.uint16).view(np.float16).astype(np.float32)


def _nd_lp(h, kind, ctx=G):
    """a 16-bit device array from uint16 bit patterns"""
    if kind == 2:
        return mx.nd.array(h, ctx, dtype="bfloat16")
    return mx.nd.array(np.asarray(h, np.uint16).view(np.float16), ctx, dtype=np.float16)


def _raw(nd, kind):
    return nd.asnumpy(raw=True) if kind == 2 else nd.asnumpy().view(np.uint16)


# ---- the reference step -------------------------------------------------------------------------------------------
VARIANTS = {
    "lamb": ("lamb", dict(learning_rate=0.01, wd=0.01)),
    "lamb_skip": ("lamb", dict(learning_rate=0.01, wd=0.01, skip_nonfinite=True)),
    "lans": ("lans", dict(learning_rate=0.01, wd=0.01)),
    "lars": ("lars", dict(learning_rate=0.1, wd=0.05, eta=0.01)),
    "lars_mom": ("lars", dict(learning_rate=0.1, wd=0.05, eta=0.01, momentum=0.9)),
}
LAUNCHES = {"lamb": 3, "lamb_skip": 5, "lans": 5, "lars": 3, "lars_mom": 3}


class Track(object):
    """one key as the kernel left it: the float32 weight (the master under multi precision), the stored 16-bit
    weight, the optimizer state and the update count; ``step`` checks the kernel's next step against the reference
    computed from exactly these values and then takes over the kernel's results"""

    def __init__(self, name, kw, w32, kind=0, no_trust=False):
        self.name, self.kind, self.no_trust = name, kind, no_trust
        self.lr = kw.get("learning_rate")
        self.wd = kw.get("wd", 0.0)
        self.b1, self.b2 = kw.get("beta1", 0.9), kw.get("beta2", 0.999)
        self.eps = kw.get("epsilon", 1e-8 if name == "lars" else 1e-6)
        self.lower, self.upper = kw.get("lower_bound"), kw.get("upper_bound")
        self.momentum = kw.get("momentum", 0.0)
        self.eta = kw.get("eta", 0.001)
        self.w32 = np.array(w32, np.float32).ravel()
        self.stored = _to_lp(self.w32, kind) if kind else None
        z = np.zeros_like(self.w32)
        self.mean, self.var, self.mom = z.copy(), z.copy(), z.copy()
        self.t = 0

    def _norm_src(self):
        """LAMB takes r1 from the master, LANS and LARS from the stored weight (multi_lans-inl.h:296-300, lars.py:119)"""
        if self.kind and self.name != "lamb":
            return _lp_f32(self.stored, self.kind)
        return self.w32

    def reference(self, g):
        """one step from the tracked values: new weight, state, the step's magnitude, the float64 ratio(s) and the
        update direction(s)"""
        t = self.t + 1
        w = self.w32.copy()
        mean, var, mom = self.mean.copy(), self.var.copy(), self.mom.copy()
        wsrc = self._norm_src()
        n = w.size
        lib, F, P = O.lib(), O._F, O.c_f32p
        g = np.ascontiguousarray(g, np.float32).ravel()
        r = {}
        if self.name == "lamb":
            gh = np.empty_like(w)
            lib.kvo_lamb_step1_f32(O._I64(n), O._ptr(w, P), O._ptr(g, P), O._ptr(mean, P), O._ptr(var, P),
                                   O._ptr(gh, P), F(self.b1), F(self.b2), F(self.eps), F(self.wd), F(1.0), F(-1.0),
                                   1, t)
            ssw, ssg = O.sum_sq(w, 1.0, "f64"), O.sum_sq(gh, 1.0, "f64")
            lib.kvo_lamb_step2_f32(O._I64(n), O._ptr(w, P), O._ptr(gh, P), F(self.lr), F(ssw), F(ssg),
                                   F(self.lower if self.lower else -1.0), F(self.upper if self.upper else -1.0))
            r1 = self._bounded(math.sqrt(_ss64(self.w32)))
            r2 = math.sqrt(_ss64(gh))
            ratio = 1.0 if r1 == 0 or r2 == 0 else r1 / r2
            r.update(dir=gh, ratio=ratio, mag=self.lr * ratio * np.abs(gh.astype(np.float64)))
        elif self.name == "lans":
            tm, tg = np.empty_like(w), np.empty_like(w)
            gsq = O.sum_sq(g, 1.0, "f64")
            lib.kvo_lans_step1_f32(O._I64(n), O._ptr(w, P), O._ptr(g, P), O._ptr(mean, P), O._ptr(var, P),
                                   O._ptr(tm, P), O._ptr(tg, P), F(self.b1), F(self.b2), F(self.eps), F(self.wd),
                                   F(1.0), F(-1.0), t, F(gsq))
            ssw = O.sum_sq(wsrc, 1.0, "f64")
            ssm, ssg = O.sum_sq(tm, 1.0, "f64"), O.sum_sq(tg, 1.0, "f64")
            lib.kvo_lans_step2_f32(O._I64(n), O._ptr(w, P), O._ptr(tm, P), O._ptr(tg, P), F(self.lr), F(self.b1),
                                   F(ssw), F(ssm), F(ssg), F(self.lower if self.lower else -1.0),
                                   F(self.upper if self.upper else -1.0))
            r1 = self._bounded(math.sqrt(_ss64(wsrc)))
            rm, rg = math.sqrt(_ss64(tm)), math.sqrt(_ss64(tg))
            rm = 1.0 if r1 == 0 or rm == 0 else r1 / rm
            rg = 1.0 if r1 == 0 or rg == 0 else r1 / rg
            lr32, b1 = float(np.float32(self.lr)), float(np.float32(self.b1))     # the kernel's float32 arguments
            a, b = lr32 * rm * b1, lr32 * rg * (1.0 - b1)
            r.update(dir=(tm, tg), ratio=(a, b), mag=a * np.abs(tm.astype(np.float64)) + b * np.abs(tg.astype(np.float64)))
        else:
            lr = self.lr
            lars = 1.0
            if not self.no_trust:
                lr = O.lars_lr(self.lr, wsrc, g, self.wd, self.eta, self.eps, 1.0, "f64")
                wn, gn = math.sqrt(_ss64(wsrc)), math.sqrt(_ss64(g))
                if wn != 0 and gn != 0:
                    lars = self.eta * wn / (gn + self.wd * wn + self.eps)
            if self.momentum:
                O.sgd_mom_update(w, g, mom, lr, self.wd, self.momentum)
            else:
                O.sgd_update(w, g, lr, self.wd)
            d = g.astype(np.float64) + np.float64(np.float32(self.wd)) * self.w32.astype(np.float64)
            r.update(dir=d, ratio=lars, mag=self.lr * lars * np.abs(d))
        r.update(w=w, mean=mean, var=var, mom=mom)
        return r

    def _bounded(self, r1):
        if self.lower is not None:
            r1 = max(r1, self.lower)
        if self.upper is not None:
            r1 = min(r1, self.upper)
        return r1

    def check(self, kv, key, g, out, eps, what=""):
        """the kernel's step (already run) against the reference; then follow the kernel"""
        ref = self.reference(g)
        self.t += 1
        if self.kind:
            got = _state(kv, key, 1).ravel()
            raw = _raw(out, self.kind).ravel()
            assert _bits_equal(raw, _to_lp(got, self.kind)), "%s: copy-out is not the rounded master" % what
        else:
            got = out.asnumpy().ravel()
        self._within(got, ref["w"], ref["mag"], eps, what + " weight")
        if self.name in ("lamb", "lans"):
            mean, var = _state(kv, key, 2).ravel(), _state(kv, key, 3).ravel()
            assert _bits_equal(mean, ref["mean"]), "%s: mean" % what
            assert _bits_equal(var, ref["var"]), "%s: var" % what
            self.mean, self.var = mean, var
        elif self.momentum:
            mom = _state(kv, key, 2).ravel()
            self._within(mom, ref["mom"], ref["mag"], eps, what + " momentum")
            self.mom = mom
        self.w32 = got.copy()
        if self.kind:
            self.stored = raw.copy()
        return ref

    def _within(self, got, want, mag, eps, what):
        got64, want64 = got.astype(np.float64), want.astype(np.float64)
        both_nan = np.isnan(got64) & np.isnan(want64)
        err = np.where(both_nan, 0.0, np.abs(got64 - want64))
        bound = 2 * _ulp(want) + mag * (eps + 4 * U)
        bad = ~(err <= bound) & ~both_nan
        assert not bad.any(), "%s: %d elements beyond the bound, first at %d: got %r want %r bound %r" % (
            what, int(bad.sum()), int(np.argmax(bad)), got[bad][0], want[bad][0], bound[bad][0])
        nz = bound > 0
        if nz.any():
            _note("weights/state", float(np.max(err[nz] / bound[nz])))


def _grads(rng, name, shape, n, kind):
    """n gradient replicas; LANS' are dyadic (exact sums of squares, see the module docstring)"""
    out = []
    sign = rng.choice(np.array([-1.0, 1.0], np.float32), shape)
    for _ in range(n):
        if name == "lans":     # one sign per element across the sources: the sum is never zero (g_norm > 0)
            x = sign * rng.choice(np.array([0.25, 0.5], np.float32), shape)
        else:
            x = rng.uniform(-1, 1, shape).astype(np.float32)
        out.append(_to_lp(x, kind) if kind else x)
    return out


def _gsum(gs, kind):
    return O.sum_device_lp_f32out(gs, kind) if kind else O.sum_device(gs)


def _nd(x, kind, ctx=G):
    return _nd_lp(x, kind, ctx) if kind else mx.nd.array(x, ctx)


class Store(object):
    """a device store with keys of the given shapes and kinds (0 float32, 1 float16, 2 bfloat16) and its tracks"""

    def __init__(self, variant, shapes, kinds, seed, mp=None, kw_extra=None, w_init=None):
        self.name, kw = VARIANTS[variant]
        kw = dict(kw, **(kw_extra or {}))
        self.variant, self.shapes, self.kinds = variant, shapes, kinds
        self.rng = np.random.default_rng(seed)
        self.keys = list(range(len(shapes)))
        mp = any(kinds) if mp is None else mp
        self.mp = mp
        self.kv = mx.kv.create("device")
        self.tracks, init = [], []
        for k, (s, kind) in enumerate(zip(shapes, kinds)):
            w = w_init(k, s) if w_init else self.rng.uniform(-1, 1, s).astype(np.float32)
            if kind:
                h = _to_lp(w, kind)
                init.append(_nd_lp(h, kind))
                w = _lp_f32(h, kind)
            else:
                init.append(mx.nd.array(w, G))
            self.tracks.append(Track(self.name, {k2: v for k2, v in kw.items() if k2 != "skip_nonfinite"}, w, kind))
        self.kv.init(self.keys, init)
        self.kv.set_optimizer(mx.optimizer.create(self.name, multi_precision=mp, **kw))
        self.outs = [mx.nd.empty(s, G, dtype={0: np.float32, 1: np.float16, 2: "bfloat16"}[kind])
                     for s, kind in zip(shapes, kinds)]

    def push(self, grads):
        before = mx.kv.launch_count()
        self.kv.pushpull(self.keys, [[_nd(g, kind) for g in gs] for gs, kind in zip(grads, self.kinds)],
                         out=self.outs)
        return mx.kv.launch_count() - before

    def step(self, n, chunk, what=""):
        grads = [_grads(self.rng, self.name, s, n, kind) for s, kind in zip(self.shapes, self.kinds)]
        first = self.tracks[0].t == 0
        launches = self.push(grads)
        # each phase once per launch class; the first push also casts every key to its fp32 master
        want = LAUNCHES[self.variant] * len(set(self.kinds)) + (len(self.keys) if self.mp and first else 0)
        assert launches == want, "%s: %d launches, not %d" % (what, launches, want)
        refs = []
        for k, tr in enumerate(self.tracks):
            n_el = int(np.prod(self.shapes[k]))
            refs.append(tr.check(self.kv, k, _gsum(grads[k], self.kinds[k]), self.outs[k],
                                 _ratio_eps(n_el, chunk), "%s key %d step %d" % (what, k, tr.t + 1)))
        return grads, refs


# ---- 1. blocks that walk many chunks and many keys ----------------------------------------------------------------
SHAPES = [(1,), (3,), (127,), (128,), (129,), (4099,), (65539,), (257, 33)]


@pytest.mark.parametrize("max_blocks", [1, 2, 3, 7])
@pytest.mark.parametrize("chunk", [128, 256])
@pytest.mark.parametrize("prec", ["f32", "lp"])
@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_blocks_walk_many_chunks_and_keys(tuning, variant, prec, chunk, max_blocks):
    """a grid of 1 ... 7 blocks over ~570 (chunk 128) or ~290 (256) chunks of eight keys: every block crosses many
    key boundaries (the work reload, LANS' g_norm, apply's per-key scalars) and the finalize kernel sums more than
    256 partials of the largest key.  1, 3 and 6 sources over the three steps; the 16-bit run takes bfloat16 keys at
    chunk 128 and float16 keys at chunk 256, with fp32 masters."""
    tuning(chunk_elems=chunk, max_blocks=max_blocks)
    kind = 0 if prec == "f32" else (2 if chunk == 128 else 1)
    st = Store(variant, SHAPES, [kind] * len(SHAPES), seed=chunk + max_blocks)
    for s, n in enumerate((1, 3, 6)):
        st.step(n, chunk, "%s %s chunk %d grid %d" % (variant, prec, chunk, max_blocks))


@pytest.mark.skipif(SIM, reason="31 M elements: minutes on the simulated runtime")
@pytest.mark.parametrize("variant", ["lamb", "lars"])
def test_bert_large_embedding(variant):
    """one 30522 x 1024 float32 key at the default chunk (3 815 chunks: every block of the grid walks ~15 of them,
    the finalize threads add 15 partials each); the trust ratio is also recovered from the update (see item 2)"""
    shape = (30522, 1024)
    st = Store(variant, [shape], [0], seed=5, kw_extra=RATIO_KW[variant], w_init=_small)
    w_prev = st.tracks[0].w32.copy()
    _, refs = st.step(2, _default_chunk(), variant + " bert")
    _check_ratio(variant, w_prev, st.tracks[0].w32, refs[0], st.tracks[0], _default_chunk(), "bert " + variant)


# ---- 2. the trust ratio itself --------------------------------------------------------------------------------------
def _check_ratio(variant, w_prev, w_new, ref, tr, chunk, what):
    """recover the ratio the kernel applied from w - w' and compare it with the float64 ratio"""
    n = w_prev.size
    eps = _ratio_eps(n, chunk)
    dw = w_prev.astype(np.float64) - w_new.astype(np.float64)
    noise_abs = _ulp(w_new) / 2        # w' is rounded once; w - w' is exact in float64
    if variant.startswith("lans"):
        tm, tg = (x.astype(np.float64) for x in ref["dir"])
        X = np.stack([tm, tg], 1)
        coef, *_ = np.linalg.lstsq(X, dw, rcond=None)
        pinv = np.linalg.pinv(X)
        # |coefficient error| <= sum_i |pinv_ji| * |e_i|, e_i: the roundings of the product terms and of w'
        e = noise_abs + U * (ref["mag"] * 2)
        noise = np.abs(pinv) @ e
        for j, (got, want) in enumerate(zip(coef, ref["ratio"])):
            bound = eps * abs(want) + noise[j]
            _note("ratio " + variant, abs(got - want) / bound)
            assert abs(got - want) <= bound, "%s: lans coefficient %d %r vs %r (bound %r)" % (what, j, got, want, bound)
        return
    d = ref["dir"].astype(np.float64) * tr.lr
    a = np.abs(d)
    # the kernel rounds lr * direction (LAMB), or wd * w, + g and lr * (...) (LARS): relative to |direction|
    noise_rel = np.full(d.shape, U)
    if variant.startswith("lars"):
        noise_rel = U * (1.5 + np.abs(np.float32(tr.wd) * w_prev.astype(np.float64)) * tr.lr / np.maximum(a, 1e-300))
    sel = a >= np.median(a)
    sel &= a > 0
    x = dw[sel] / d[sel]
    got = float(np.median(x))
    want = ref["ratio"]
    # the median lies within the largest per-element deviation from the true value
    noise = float(np.max(noise_abs[sel] / a[sel] + noise_rel[sel] * np.abs(want)))
    bound = eps * want + noise
    _note("ratio " + variant, abs(got - want) / bound)
    assert abs(got - want) <= bound, "%s: ratio %r vs float64 %r (bound %r)" % (what, got, want, bound)


RATIO_SHAPES = [(4099,), (65539,), (257, 33), (300007,)]
# lr = 0.5 with |w| ~ 1e-3 moves a weight by a good fraction of itself; LARS' ratio eta * |w| / |g| needs eta = 2 for that
RATIO_KW = {"lamb": dict(learning_rate=0.5), "lans": dict(learning_rate=0.5), "lars": dict(learning_rate=0.5, eta=2.0)}


def _small(k, s):
    return np.random.default_rng(k).uniform(-1e-3, 1e-3, s).astype(np.float32)


@pytest.mark.parametrize("tune", [None, (128, 3)])
@pytest.mark.parametrize("variant", ["lamb", "lans", "lars"])
def test_trust_ratio_recovered_from_the_update(tuning, variant, tune):
    """lr = 0.5 and weights of order 1e-3: a step moves each weight by a good fraction of itself, so w - w' carries
    the ratio to many digits.  LAMB: median of (w - w') / (lr * ghat) over the larger half of |ghat|; LARS (no
    momentum): the same with g + wd * w; LANS: a two-column least-squares fit of w - w' on (temp_m, temp_g) gives
    lr * r_m * beta1 and lr * r_g * (1 - beta1).  Each is compared with the float64 ratio within (D + 6) * 2^-24
    relative plus the rounding noise of the recovery itself."""
    chunk = _default_chunk()
    if tune:
        tuning(chunk_elems=tune[0], max_blocks=tune[1])
        chunk = tune[0]
    st = Store(variant, RATIO_SHAPES, [0] * len(RATIO_SHAPES), seed=77, kw_extra=RATIO_KW[variant], w_init=_small)
    for s in range(2):
        prev = [tr.w32.copy() for tr in st.tracks]
        _, refs = st.step(2, chunk, variant + " ratio")
        if variant == "lans" and s == 0:
            continue        # at step 1 temp_m and temp_g are nearly parallel (mean_hat ~ g): the fit needs step 2
        for k, tr in enumerate(st.tracks):
            _check_ratio(variant, prev[k], tr.w32, refs[k], tr, chunk, "%s key %d step %d" % (variant, k, s + 1))


# ---- 3. zero norms ----------------------------------------------------------------------------------------------------
def test_lamb_zero_weight_takes_ratio_one():
    """r1 = 0 (a zero-initialised key): the ratio is 1 and w' = -lr * ghat exactly; with lower_bound = 1e-3 r1 is the
    bound instead"""
    E = 4099
    st = Store("lamb", [(E,)], [0], seed=3, w_init=lambda k, s: np.zeros(s, np.float32))
    _, refs = st.step(2, _default_chunk(), "lamb zero weight")
    want = -(np.float32(0.01) * refs[0]["dir"])
    assert _bits_equal(st.tracks[0].w32, want), "r1 = 0 must give w' = -lr * ghat"
    st = Store("lamb", [(E,)], [0], seed=3, kw_extra=dict(lower_bound=1e-3, learning_rate=0.5),
               w_init=lambda k, s: np.zeros(s, np.float32))
    _, refs = st.step(2, _default_chunk(), "lamb zero weight, lower bound")
    assert abs(refs[0]["ratio"] - 1e-3 / math.sqrt(_ss64(refs[0]["dir"]))) < 1e-12
    _check_ratio("lamb", np.zeros(E, np.float32), st.tracks[0].w32, refs[0], st.tracks[0], _default_chunk(),
                 "lamb lower bound")


def test_lamb_zero_gradient_leaves_the_weight():
    """g = 0 and wd = 0: ghat = 0, r2 = 0, ratio 1, and w' = w - lr * 0 = w; mean and var stay zero"""
    E = 4099
    kv = mx.kv.create("device")
    w = np.random.default_rng(1).uniform(-1, 1, E).astype(np.float32)
    kv.init(0, mx.nd.array(w, G))
    kv.set_optimizer(mx.optimizer.create("lamb", learning_rate=0.01, wd=0.0))
    out = mx.nd.empty((E,), G)
    kv.pushpull(0, [mx.nd.zeros((E,), G), mx.nd.zeros((E,), G)], out=out)
    assert _bits_equal(out.asnumpy(), w)
    assert not _state(kv, 0, 2).any() and not _state(kv, 0, 3).any()


@pytest.mark.parametrize("normal_first", [True, False])
def test_lars_zero_norms_fall_back_to_the_plain_rate(tuning, normal_first):
    """LARS' nan_or_zero rule: a zero weight (ratio 0), a zero gradient (ratio inf) and both (NaN) give lars = 1,
    i.e. exactly SGD-momentum at the plain learning rate, in the same push as a normal key that must keep its own
    ratio.  One block walks all four keys (a stale per-key scalar would carry one key's rate into the next)."""
    tuning(chunk_elems=128, max_blocks=1)
    E = 1031
    rng = np.random.default_rng(11)
    kw = dict(learning_rate=0.1, momentum=0.9, wd=0.05, eta=0.01)
    w = {"normal": rng.uniform(-1, 1, E), "zero_w": np.zeros(E), "zero_g": rng.uniform(-1, 1, E),
         "both": np.zeros(E)}
    names = ["normal", "zero_w", "zero_g", "both"] if normal_first else ["zero_w", "zero_g", "both", "normal"]
    w0 = [w[n].astype(np.float32) for n in names]
    kv = mx.kv.create("device")
    kv.init(list(range(4)), [mx.nd.array(x, G) for x in w0])
    kv.set_optimizer(mx.optimizer.create("lars", **kw))
    outs = [mx.nd.empty((E,), G) for _ in range(4)]
    tracks = [Track("lars", kw, x) for x in w0]
    for s in range(2):
        g = [np.zeros(E, np.float32) if n in ("zero_g", "both") else rng.uniform(-1, 1, E).astype(np.float32)
             for n in names]
        kv.pushpull(list(range(4)), [mx.nd.array(x, G) for x in g], out=outs)
        for k, n in enumerate(names):
            if tracks[k].w32.any() and g[k].any():      # (the zero weight has moved after its first step)
                ref = tracks[k].check(kv, k, g[k], outs[k], _ratio_eps(E, 128), "lars %s step %d" % (n, s))
                assert abs(ref["ratio"] - 1.0) > 0.5, "a key with both norms non-zero keeps its own ratio"
            else:
                plain_w, plain_m = tracks[k].w32.copy(), tracks[k].mom.copy()
                O.sgd_mom_update(plain_w, g[k], plain_m, 0.1, 0.05, 0.9)
                assert _bits_equal(outs[k].asnumpy(), plain_w), "%s step %d: not sgd at the plain rate" % (n, s)
                assert _bits_equal(_state(kv, k, 2), plain_m), "%s step %d: momentum" % (n, s)
                tracks[k].w32, tracks[k].mom = plain_w, plain_m


def test_lans_zero_weight_both_ratios_one():
    """r1 = 0: both trust ratios are 1, so w' = 0 - (lr * beta1 * temp_m + lr * (1 - beta1) * temp_g) exactly"""
    E = 4099
    st = Store("lans", [(E,)], [0], seed=9, w_init=lambda k, s: np.zeros(s, np.float32))
    g = _grads(st.rng, "lans", (E,), 2, 0)
    st.push([g])
    ref = st.tracks[0].reference(_gsum(g, 0))
    assert _bits_equal(st.outs[0].asnumpy(), ref["w"])
    assert _bits_equal(_state(st.kv, 0, 2), ref["mean"]) and _bits_equal(_state(st.kv, 0, 3), ref["var"])


@pytest.mark.parametrize("skip", [False, True])
def test_lans_zero_gradient_is_the_reference_nan(skip):
    """an all-zero merged gradient: the reference divides by g_norm = 0 (multi_lans.cc:48-51) and every weight
    becomes NaN.  The merged gradient itself is finite, so skip_nonfinite does not skip the step.  This pins the
    reference's behaviour; it is not a recommendation."""
    E = 1000
    w = np.random.default_rng(2).uniform(-1, 1, E).astype(np.float32)
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w, G))
    kv.set_optimizer(mx.optimizer.create("lans", learning_rate=0.01, wd=0.01, skip_nonfinite=skip))
    out = mx.nd.empty((E,), G)
    kv.pushpull(0, [mx.nd.zeros((E,), G)], out=out)
    if skip:
        assert kv.overflow() is False
    tr = Track("lans", dict(learning_rate=0.01, wd=0.01), w)
    ref = tr.reference(np.zeros(E, np.float32))
    assert np.isnan(ref["w"]).all()
    assert np.isnan(out.asnumpy()).all()


# ---- 4. float32 keys with multi_precision=True --------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["lamb", "lamb_skip", "lans", "lars_mom"])
def test_float32_keys_on_the_multi_precision_kernels(variant):
    """a float32 key under multi_precision=True runs the (float, true) instantiations with an fp32 master: after
    every one of 4 steps weights, outputs and state equal the run without multi precision bit for bit, and the
    master equals the weight"""
    name, kw = VARIANTS[variant]
    shapes = [(5,), (4099,), (65539,)]
    rng = np.random.default_rng(21)
    w0 = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
    keys = list(range(len(shapes)))
    kvs, outs = [], []
    for mp in (False, True):
        kv = mx.kv.create("device")
        kv.init(keys, [mx.nd.array(w, G) for w in w0])
        kv.set_optimizer(mx.optimizer.create(name, multi_precision=mp, **kw))
        kvs.append(kv)
        outs.append([mx.nd.empty(s, G) for s in shapes])
    which = [2, 3] if name != "lars" else [2]
    for s in range(4):
        g = [_grads(rng, name, sh, 2, 0) for sh in shapes]
        for kv, o in zip(kvs, outs):
            kv.pushpull(keys, [[mx.nd.array(x, G) for x in gs] for gs in g], out=o)
        for k in keys:
            a, b = outs[0][k].asnumpy(), outs[1][k].asnumpy()
            assert _bits_equal(a, b), "%s key %d step %d: weight" % (variant, k, s)
            assert _bits_equal(_state(kvs[1], k, 1), b), "%s key %d step %d: master" % (variant, k, s)
            for w in which:
                assert _bits_equal(_state(kvs[0], k, w), _state(kvs[1], k, w)), "%s key %d state %d" % (variant, k, w)


# ---- 5. several launch classes in one push ------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["lamb", "lans", "lars_mom"])
def test_launch_classes_in_one_push(variant):
    """float32, float16 and bfloat16 keys under one multi-precision optimizer, 2 sources each: three launch classes,
    phase-major; every key matches its own single-key reference"""
    shapes = [(4099,), (20011,), (1031,)]
    st = Store(variant, shapes, [0, 1, 2], seed=31, mp=True)
    for _ in range(2):
        st.step(2, _default_chunk(), variant + " classes")


@pytest.mark.parametrize("variant", ["lamb_skip", "lans", "lars_mom"])
def test_overflow_in_one_class_skips_every_class(variant):
    """skip_nonfinite over three launch classes: an inf in the bfloat16 key only, then a NaN in the float32 key only,
    leaves every key's weight, master, state and update count unchanged; overflow() reports it once; the next good
    step is step 2 of the bias correction for every key"""
    name, kw = VARIANTS[variant]
    kw = dict(kw, skip_nonfinite=True)
    shapes = [(4099,), (20011,), (1031,)]
    kinds = [0, 1, 2]
    st = Store(variant, shapes, kinds, seed=41, mp=True, kw_extra=dict(skip_nonfinite=True))
    st.variant = "lamb_skip" if name == "lamb" else variant
    st.step(2, _default_chunk(), variant + " good")

    def snapshot():
        snap = []
        for k in st.keys:
            snap.append([_bits(_raw(st.outs[k], kinds[k]) if kinds[k] else st.outs[k].asnumpy()).copy()] +
                        [_state(st.kv, k, w) for w in (1, 2, 3)])
        return snap

    before = snapshot()
    for bad_key, val in ((2, np.inf), (0, np.nan)):
        grads = [_grads(st.rng, name, s, 2, kind) for s, kind in zip(shapes, kinds)]
        if kinds[bad_key] == 2:
            grads[bad_key][1][7] = 0x7f80
        else:
            grads[bad_key][0][-1] = val
        st.push(grads)
        assert st.kv.overflow() is True
        assert st.kv.overflow() is False
        after = snapshot()
        for k in st.keys:
            for a, b in zip(before[k], after[k]):
                assert (a is None and b is None) or _bits_equal(a, b), "%s key %d changed on a skipped step" % (variant, k)
    st.step(2, _default_chunk(), variant + " after two skipped steps")
    assert all(tr.t == 2 for tr in st.tracks)


# ---- 6. the scalar path over a whole key ----------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["lamb", "lans", "lars_mom"])
def test_unaligned_gradients_take_the_scalar_path(tuning, variant):
    """float32 gradients that are views at element offsets 1 ... 3 of larger buffers (4-byte aligned only): the whole
    key goes through the scalar loops of first, mid and apply, at chunk 128 on 3 blocks"""
    import torch
    tuning(chunk_elems=128, max_blocks=3)
    name, kw = VARIANTS[variant]
    E = 65539
    st = Store(variant, [(E,)], [0], seed=51)
    for s in range(3):
        gs = _grads(st.rng, name, (E,), 3, 0)
        bases = [torch.zeros(E + 4, dtype=torch.float32, device="cuda") for _ in gs]
        views = []
        for j, (b, x) in enumerate(zip(bases, gs)):
            b[j + 1:j + 1 + E].copy_(torch.from_numpy(x))
            views.append(b[j + 1:j + 1 + E])
        torch.cuda.synchronize()
        before = mx.kv.launch_count()
        st.kv.pushpull(0, [mx.nd.from_torch(v) for v in views], out=st.outs[0])
        assert mx.kv.launch_count() - before == LAUNCHES[variant]
        st.tracks[0].check(st.kv, 0, O.sum_device(gs), st.outs[0], _ratio_eps(E, 128), "%s unaligned step %d" % (variant, s))


# ---- 7. multi_sum_sq / multi_all_finite ---------------------------------------------------------------------------------
NP = {"float16": np.float16, "bfloat16": np.uint16, "float32": np.float32, "float64": np.float64}


def _sumsq_nd(x, dt):
    if dt == "bfloat16":
        return mx.nd.array(x, G, dtype="bfloat16")
    return mx.nd.array(x, G, dtype=NP[dt])


def _as_f32(x, dt):
    if dt == "bfloat16":
        return O.bf16_to_f32(x)
    return np.asarray(x).astype(np.float32)       # float64 above FLT_MAX becomes inf, like the kernel's cast


def _check_sumsq(got, xs, dt, scale=1.0, chunk=None):
    chunk = chunk or _default_chunk()
    for i, x in enumerate(xs):
        v = _as_f32(x, dt).astype(np.float64)
        if scale != 1.0:
            v = (v.astype(np.float32) * np.float32(scale)).astype(np.float64)
        want = float(np.dot(v, v))
        bound = _depth(v.size, chunk) * U * want
        err = abs(float(got[i]) - want)
        if bound > 0:
            _note("multi_sum_sq", err / bound)
        assert err <= bound, "array %d (%d elements, %s): %r vs %r (bound %r)" % (i, v.size, dt, got[i], want, bound)


@pytest.mark.parametrize("dt", ["float32", "float16", "bfloat16", "float64"])
def test_multi_sum_sq_sizes_and_many_arrays(dt):
    """one call over the chunk-boundary sizes, one over 1 000 arrays of random sizes, each against a float64 sum"""
    rng = np.random.default_rng(61)
    C = _default_chunk()
    sizes = [1, 127, 128, C - 1, C, C + 1, 2 * C, 2 * C + 1, 3 * C + 1]
    for szs in (sizes, list(rng.integers(1, 3000, 1000))):
        xs = []
        for n in szs:
            x = rng.uniform(-2, 2, int(n))
            xs.append(O.f32_to_bf16(x.astype(np.float32)) if dt == "bfloat16" else x.astype(NP[dt]))
        arrs = [_sumsq_nd(x, dt) for x in xs]
        for scale in (1.0, 0.37):
            _check_sumsq(mx.nd.multi_sum_sq(*arrs, scale=scale).asnumpy(), xs, dt, scale)
        assert mx.nd.multi_all_finite(*arrs).asnumpy()[0] == 1.0


def test_multi_sum_sq_squares_in_float32():
    """float16 values 256 ... 65504 square beyond float16's range but not float32's: the sum must be finite and
    right.  bfloat16 values near 1e20 square beyond float32's range: the sum is inf while every element is finite.
    float64 values above FLT_MAX are cast to float first (all_finite.cu:70) and count as non-finite."""
    rng = np.random.default_rng(62)
    h = rng.uniform(256, 65504, 20000).astype(np.float16)
    got = mx.nd.multi_sum_sq(_sumsq_nd(h, "float16")).asnumpy()
    assert np.isfinite(got).all()
    _check_sumsq(got, [h], "float16")
    b = O.f32_to_bf16(rng.uniform(0.9e20, 1.1e20, 9000).astype(np.float32))
    a = _sumsq_nd(b, "bfloat16")
    assert np.isinf(mx.nd.multi_sum_sq(a).asnumpy()[0])
    assert mx.nd.multi_all_finite(a).asnumpy()[0] == 1.0
    d = rng.uniform(-1, 1, 9000)
    d[4321] = 1e39
    a = _sumsq_nd(d, "float64")
    assert mx.nd.multi_all_finite(a).asnumpy()[0] == 0.0
    assert np.isinf(mx.nd.multi_sum_sq(a).asnumpy()[0])
    d[4321] = 3.0e38                                 # below FLT_MAX: finite
    assert mx.nd.multi_all_finite(_sumsq_nd(d, "float64")).asnumpy()[0] == 1.0


BAD_BITS = {
    "float16": [0x7c00, 0xfc00, 0x7e00, 0x7c01],
    "bfloat16": [0x7f80, 0xff80, 0x7fc0, 0x7f81],
    "float32": [0x7f800000, 0xff800000, 0x7fc00000, 0x7f800001],
    "float64": [0x7ff0000000000000, 0xfff0000000000000, 0x7ff8000000000000, 0x7ff0000000000001],
}


@pytest.mark.parametrize("dt", sorted(BAD_BITS))
def test_multi_all_finite_bit_patterns_at_chunk_edges(dt):
    """+inf, -inf, a quiet NaN and a signalling NaN at element 0, the last element of a chunk, the first element of
    the next chunk and the last element of the last array: the flag drops to 0, the array's sum is inf / NaN and
    every other array's sum is untouched; init_output=False keeps a preset 0.0 and keeps a preset 1.0 only when
    every element is finite"""
    rng = np.random.default_rng(63)
    C = _default_chunk()
    sizes = [3 * C + 1, 100, C + 5]
    ui = {2: np.uint16, 4: np.uint32, 8: np.uint64}
    xs = []
    for n in sizes:
        x = rng.uniform(-1, 1, n)
        xs.append(O.f32_to_bf16(x.astype(np.float32)) if dt == "bfloat16" else x.astype(NP[dt]))
    good = mx.nd.multi_sum_sq(*[_sumsq_nd(x, dt) for x in xs]).asnumpy()
    _check_sumsq(good, xs, dt)
    for where in ((0, 0), (0, C - 1), (0, C), (2, sizes[2] - 1)):
        for pat in BAD_BITS[dt]:
            ys = [x.copy() for x in xs]
            y = ys[where[0]]
            y.view(ui[y.dtype.itemsize])[where[1]] = pat
            arrs = [_sumsq_nd(x, dt) for x in ys]
            assert mx.nd.multi_all_finite(*arrs).asnumpy()[0] == 0.0, (where, hex(pat))
            got = mx.nd.multi_sum_sq(*arrs).asnumpy()
            is_nan = (pat & {2: 0x03ff if dt == "float16" else 0x007f, 4: 0x7fffff, 8: (1 << 52) - 1}[y.dtype.itemsize]) != 0
            assert (np.isnan(got[where[0]]) if is_nan else got[where[0]] == np.inf), (where, hex(pat), got)
            others = [i for i in range(len(xs)) if i != where[0]]
            assert _bits_equal(got[others], good[others])
            for preset in (0.0, 1.0):
                out = mx.nd.array(np.array([preset], np.float32), G)
                mx.nd.multi_all_finite(*arrs, init_output=False, out=out)
                assert out.asnumpy()[0] == 0.0
    arrs = [_sumsq_nd(x, dt) for x in xs]
    for preset in (0.0, 1.0):
        out = mx.nd.array(np.array([preset], np.float32), G)
        mx.nd.multi_all_finite(*arrs, init_output=False, out=out)
        assert out.asnumpy()[0] == preset


# ---- 8. 2^31 elements ---------------------------------------------------------------------------------------------------
def _free_bytes():
    import torch
    return torch.cuda.mem_get_info(0)[0]


def _periodic(period, lo, hi, seed, kind=None):
    """a seeded pattern of `period` values that an array repeats (its float64 sums follow from the counts per value)"""
    p = np.random.default_rng(seed).uniform(lo, hi, period).astype(np.float32)
    if kind is not None:
        p = _lp_f32(_to_lp(p, kind), kind)
    return p


def _ss_periodic(p, n):
    q, r = divmod(n, p.size)
    p64 = p.astype(np.float64)
    return q * float(np.dot(p64, p64)) + float(np.dot(p64[:r], p64[:r]))


@pytest.mark.skipif(SIM, reason="4.3 GB: not on the simulated runtime")
def test_multi_sum_sq_above_2_31_elements():
    """one float16 array of 2^31 + 8193 elements (4.3 GB; skipped below 12 GB free): the sum against float64, then a
    NaN past element 2^31 found by multi_all_finite"""
    if _free_bytes() < 12 << 30:
        pytest.skip("needs 12 GB of free device memory")
    n = (1 << 31) + 8193
    p = _periodic(1021, -4, 4, 71).astype(np.float16)
    x = np.resize(p, n)
    a = mx.nd.array(x, G, dtype=np.float16)
    got = mx.nd.multi_sum_sq(a).asnumpy()[0]
    want = _ss_periodic(p.astype(np.float32), n)
    bound = _depth(n, _default_chunk()) * U * want
    _note("multi_sum_sq 2^31", abs(float(got) - want) / bound)
    assert abs(float(got) - want) <= bound, (got, want, bound)
    assert mx.nd.multi_all_finite(a).asnumpy()[0] == 1.0
    x[(1 << 31) + 4097] = np.nan
    a = mx.nd.array(x, G, dtype=np.float16)
    del x
    assert mx.nd.multi_all_finite(a).asnumpy()[0] == 0.0
    assert np.isnan(mx.nd.multi_sum_sq(a).asnumpy()[0])


@pytest.mark.skipif(SIM, reason="30 GB: not on the simulated runtime")
def test_lars_step_above_2_31_elements():
    """one LARS step (no momentum) on a bfloat16 key of 2^31 + 4101 elements with an fp32 master (about 30 GB on the
    device; skipped below 40 GB free).  The norms come from float64 sums over the periodic data; the update is
    checked on windows at the start, around 2^31 and at the end."""
    import torch
    if _free_bytes() < 40 << 30:
        pytest.skip("needs 40 GB of free device memory")
    n = (1 << 31) + 4101
    pw = _periodic(4093, -1, 1, 81, kind=2)
    pg = _periodic(3001, -1, 1, 82, kind=2)
    lr, wd, eta = 0.1, 0.05, 0.01
    kv = mx.kv.create("device")
    w_t = torch.from_numpy(np.resize(_to_lp(pw, 2), n).view(np.int16)).view(torch.bfloat16).cuda()
    kv.init(0, mx.nd.from_torch(w_t))
    del w_t
    kv.set_optimizer(mx.optimizer.create("lars", learning_rate=lr, wd=wd, eta=eta, multi_precision=True))
    g_t = torch.from_numpy(np.resize(_to_lp(pg, 2), n).view(np.int16)).view(torch.bfloat16).cuda()
    out_t = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    kv.pushpull(0, [mx.nd.from_torch(g_t)], out=mx.nd.from_torch(out_t))
    mx.nd.waitall()
    del g_t
    ssw, ssg = _ss_periodic(pw, n), _ss_periodic(pg, n)
    wn, gn = math.sqrt(ssw), math.sqrt(ssg)
    lars = eta * wn / (gn + wd * wn + 1e-8)
    eps = _ratio_eps(n, _default_chunk())
    master = kv._state_handle(0, 1).as_torch()
    for lo in (0, (1 << 31) - 4096, n - 8192):
        idx = np.arange(lo, lo + 8192)
        w = pw[idx % pw.size].astype(np.float64)
        g = pg[idx % pg.size].astype(np.float64)
        d = g + np.float64(np.float32(wd)) * w
        want = w - lr * lars * d
        got = master[lo:lo + 8192].cpu().numpy().astype(np.float64)
        bound = 2 * _ulp(want) + lr * lars * np.abs(d) * (eps + 4 * U)
        err = np.abs(got - want)
        _note("lars 2^31", float(np.max(err / bound)))
        assert (err <= bound).all(), "window at %d: worst %r" % (lo, float(np.max(err / bound)))
        got_lp = out_t[lo:lo + 8192].view(torch.int16).cpu().numpy().view(np.uint16)
        assert _bits_equal(got_lp, _to_lp(got.astype(np.float32), 2)), "window at %d: copy-out" % lo


# ---- 9. sharded keys on several GPUs ------------------------------------------------------------------------------------
@pytest.mark.multigpu
@pytest.mark.parametrize("ndev", [2, 3])
@pytest.mark.parametrize("variant", ["lamb", "lans", "lars_mom"])
def test_sharded_key_with_small_chunks(tuning, variant, ndev):
    """a key of 2^20 + 3 elements sharded over 2 or 3 GPUs (shard boundaries not multiples of 4), chunk 128 and 3
    blocks on every device: the norms are added across the shards in rank order and every replica is identical"""
    if mx.num_gpus() < ndev:
        pytest.skip("needs %d GPUs" % ndev)
    tuning(chunk_elems=128, max_blocks=3)
    name, kw = VARIANTS[variant]
    E = (1 << 20) + 3
    rng = np.random.default_rng(91)
    w0 = rng.uniform(-1, 1, E).astype(np.float32)
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w0, G))
    kv.set_optimizer(mx.optimizer.create(name, **kw))
    tr = Track(name, kw, w0)
    outs = [mx.nd.empty((E,), mx.gpu(d)) for d in range(ndev)]
    for s in range(2):
        g = _grads(rng, name, (E,), ndev, 0)
        kv.pushpull(0, [mx.nd.array(x, mx.gpu(d)) for d, x in enumerate(g)], out=outs)
        first = outs[0].asnumpy()
        for o in outs[1:]:
            assert _bits_equal(o.asnumpy(), first), "%s: replicas differ" % variant
        ref = tr.reference(O.sum_device(g))
        tr.t += 1
        tr._within(first, ref["w"], ref["mag"], _ratio_eps(E, 128, ranks=ndev), "%s sharded step %d" % (variant, s))
        tr.w32 = first.copy()
        if name != "lars":
            assert _bits_equal(_state(kv, 0, 2), ref["mean"]) and _bits_equal(_state(kv, 0, 3), ref["var"])
            tr.mean, tr.var = ref["mean"], ref["var"]
        else:
            tr.mom = _state(kv, 0, 2)
