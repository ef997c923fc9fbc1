"""1-bit / 2-bit gradient compression (csrc/kernels.cu kv_quantize_kernel / kv_dequantize_kernel, the arithmetic of
csrc/optim_math.h, csrc/kvstore.cc ReduceUpdateCompressed) at its edges: sizes whose code streams end in a partial
word, keys large enough that both codec kernels walk their grid-stride loops more than once, residuals that land
exactly on a threshold, signed zeros, subnormals and non-finite gradients, every fused optimizer fed by dequantised
streams, the per-slot residual bookkeeping, and the steps AdamW / AdaBelief skip on a bad ``rescale_grad``.

Expected values come from two sides.  The oracle codec (``oracle.quantize_*`` / ``dequantize_*``, pinned to the
reference's bit-level simulator by tests/golden/compression.npz) feeds ``oracle.OracleKVStore`` or the optimizer
oracles of the per-optimizer suites: weights and states bit for bit (LAMB, LANS and LARS within
tests/test_gpu_norm_edges.py's bound).  The numpy model of tests/gc_model.py, which shares no code with the oracle,
gives the integer code of every element: with a power-of-two threshold every dequantised sum of a few sources is
exact in float32 in any order, so the pulled sum must also equal the code counts times the threshold."""
import os
import re
import shutil
import sys
import tempfile
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import mxnet_b200 as mx
from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gc_model as M  # noqa: E402
import adabelief_oracle as AB  # noqa: E402
import adadelta_oracle as AD  # noqa: E402
import adamax_oracle as AX  # noqa: E402
import ftml_oracle as FT  # noqa: E402
import nadam_oracle as NA  # noqa: E402
import nag_oracle as NG  # noqa: E402
import rmsprop_oracle as RM  # noqa: E402
import signum_oracle as SG  # noqa: E402
from test_gpu_norm_edges import Track, _ratio_eps, _default_chunk  # noqa: E402

SIM = bool(os.environ.get("MXKV_SIM"))
G = mx.gpu(0)


def _max_blocks():
    """the codec's compile-time grid cap, kMaxBlocks = kNumSms * k, as csrc/kernels.h defines it"""
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "incubator-mxnet_b200",
                           "csrc", "kernels.h")) as f:
        src = f.read()
    sms = int(re.search(r"constexpr int kNumSms = (\d+);", src).group(1))
    return sms * int(re.search(r"constexpr int kMaxBlocks = kNumSms \* (\d+);", src).group(1))


KMAX = _max_blocks()
GRID_THREADS = KMAX * 256          # one quantize thread per 32-bit code word, one dequantize thread per element


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_bits_equal(got, want, msg=""):
    got, want = np.asarray(got, np.float32).reshape(-1), np.asarray(want, np.float32).reshape(-1)
    ne = _u32(got) != _u32(want)
    if ne.any():
        i = int(np.argmax(ne))
        raise AssertionError("%s: %d / %d elements differ, first at %d: %r vs %r" % (msg, ne.sum(), ne.size, i,
                                                                                     got[i], want[i]))


class Codec(object):
    """the oracle codec with one residual per pushed-value slot of a key, checked against the numpy model as it goes"""

    def __init__(self, bits, thr, size, model=True):
        self.bits, self.thr, self.size = bits, thr, size
        self.res = []
        self.model = M.Model(bits, thr, size) if model else None
        self.codes = None

    def push(self, grads):
        while len(self.res) < len(grads):
            self.res.append(np.zeros(self.size, np.float32))
        q = O.quantize_2bit if self.bits == 2 else O.quantize_1bit
        d = O.dequantize_2bit if self.bits == 2 else O.dequantize_1bit
        deq = [d(q(np.ascontiguousarray(g, np.float32), self.res[k], self.thr), self.size, self.thr)
               for k, g in enumerate(grads)]
        if self.model is not None:
            self.codes = self.model.push(grads)
            for k, (a, b) in enumerate(zip(self.model.deq(self.codes), deq)):
                assert_bits_equal(a, b, "the numpy model and the oracle codec disagree on slot %d" % k)
        return deq

    def exact_sum(self):
        """the sum of the last push from integer code counts (exact for a power-of-two threshold)"""
        count = np.sum(np.stack(self.codes).astype(np.int64), axis=0)
        unit = self.thr if self.bits == 2 else 1.0
        return (count * unit).astype(np.float32)


def _store(bits, thr, keys, w0, opt=None):
    kv = mx.kv.create("device")
    kv.set_gradient_compression({"type": "%dbit" % bits, "threshold": thr})
    kv.init(keys, [mx.nd.array(w, G) for w in w0])
    if opt is not None:
        kv.set_optimizer(opt)
    return kv


def _want(deq):
    return O.sum_device(deq) if len(deq) > 1 else deq[0]


def _count(kv, key):
    import ctypes
    from mxnet_b200.base import _LIB, check_call
    n = ctypes.c_int64()
    check_call(_LIB.MXKVB200GetUpdateCount(kv.handle, int(key), None, ctypes.byref(n)))
    return n.value


def _state(kv, key, which):
    h = kv._state_handle(key, which)
    return None if h is None else h.asnumpy().reshape(-1)


def _states_of(opt, key):
    st = opt.states.get(key)
    if st is None:
        return ()
    return (st,) if isinstance(st, np.ndarray) else tuple(st)


# ---- 1. sizes: partial last words and the grid-stride loops -------------------------------------------------------
SMALL = [1, 15, 16, 17, 31, 32, 33, 4097]
# three quantize passes and a partial last word (2-bit: 16 elements a word, 1-bit: 32), and a dequantize-only
# multi-pass size (one quantize pass, four dequantize passes)
BIG = {2: 3 * GRID_THREADS * 16 + 7, 1: 3 * GRID_THREADS * 32 + 13}
DEQ_ONLY = 4 * GRID_THREADS - 3


@pytest.mark.parametrize("bits,thr", [(2, 0.5), (1, 0.0)])
@pytest.mark.parametrize("size", SMALL + ["big", "deq_only"])
def test_sizes_against_the_oracle_and_the_code_counts(bits, thr, size):
    E = BIG[bits] if size == "big" else (DEQ_ONLY if size == "deq_only" else size)
    if SIM and E > 100000:
        pytest.skip("the codec's grid cap is the compile-time kMaxBlocks: the loops need sizes the simulator is too "
                    "slow for")
    n = 2 if E > 100000 else 3
    rng = np.random.default_rng(E + bits)
    kv = _store(bits, thr, [0], [np.zeros(E, np.float32)])
    codec = Codec(bits, thr, E)
    out = mx.nd.empty((E,), G)
    gdev = [mx.nd.empty((E,), G) for _ in range(n)]
    for step in range(3):
        grads = [rng.uniform(-1.2, 1.2, E).astype(np.float32) for _ in range(n)]
        for d, g in zip(gdev, grads):
            d[:] = g
        mx.nd.waitall()
        before = mx.kv.launch_count()
        kv.pushpull(0, gdev, out=out)
        mx.nd.waitall()
        assert mx.kv.launch_count() - before == 2 * n + 1, "one quantize and one dequantize per source, one sum"
        deq = codec.push(grads)
        got = out.asnumpy()
        assert_bits_equal(got, _want(deq), "%d-bit E %d step %d vs the oracle" % (bits, E, step))
        assert_bits_equal(got, codec.exact_sum(), "%d-bit E %d step %d vs the code counts" % (bits, E, step))


# ---- 2. above 2^31 elements ------------------------------------------------------------------------------------------
@pytest.mark.skipif(SIM, reason="8.6 GB arrays: not on the simulated runtime")
def test_2bit_key_above_2_31_elements():
    """one 2-bit key of 2^31 + 37 elements, one source, no optimizer, two steps (about 45 GB on the device; skipped
    below 50 GB free).  The gradient repeats a seeded pattern whose period is not a multiple of a code word, so every
    window differs; windows aligned to code words at the head, around element 2^31 (word 2^27) and at the tail are
    checked against the oracle codec run on the same windows (the codec is element-wise: a window's codes and
    residuals depend on its own elements only)"""
    import torch
    if torch.cuda.mem_get_info(0)[0] < 50 << 30:
        pytest.skip("needs 50 GB of free device memory")
    n = (1 << 31) + 37
    thr = 0.5
    period = 4093
    p = np.random.default_rng(231).uniform(-1.2, 1.2, period).astype(np.float32)
    pt = torch.from_numpy(p).cuda()
    g_t = pt.repeat(n // period + 1)[:n].contiguous()
    del pt
    kv = mx.kv.create("device")
    kv.set_gradient_compression({"type": "2bit", "threshold": thr})
    kv.init(0, mx.nd.from_torch(torch.zeros(n, device="cuda")))
    out_t = torch.empty(n, device="cuda")
    W = 16 * 1024
    # [start, end): the head; across element 2^31 to the end (the key is only 37 elements longer); the last W words'
    # worth of elements, ending in the partial last word
    windows = [(0, W), ((1 << 31) - W // 2, n), ((n // 16) * 16 - W, n)]
    assert all(lo % 16 == 0 for lo, _ in windows)
    codecs = {lo: Codec(2, thr, hi - lo) for lo, hi in windows}
    for step in range(2):
        kv.pushpull(0, mx.nd.from_torch(g_t), out=mx.nd.from_torch(out_t))
        mx.nd.waitall()
        for lo, codec in codecs.items():
            hi = lo + codec.size
            g = p[np.arange(lo, hi) % period]
            got = out_t[lo:hi].cpu().numpy()
            assert_bits_equal(got, _want(codec.push([g])), "window at %d step %d" % (lo, step))
            assert_bits_equal(got, codec.exact_sum(), "window at %d step %d vs the code counts" % (lo, step))


# ---- 3. ties, signed zeros, subnormals, non-finite gradients ------------------------------------------------------
TIE_CASES = [(2, 0.5), (2, 0.3), (2, 1.0), (1, 0.0), (1, 0.5), (1, -0.25)]


@pytest.mark.parametrize("bits,thr", TIE_CASES)
@pytest.mark.parametrize("nonfinite", [False, True])
def test_ties_zeros_subnormals_and_sticky_non_finite_codes(bits, thr, nonfinite):
    """residuals on +-thr, thr +- 1 ulp, +-0 and subnormals over five steps; with ``nonfinite``, NaN / +inf / -inf at
    the first and last element of a word and in the partial last word at step 1, and the codes they leave behind
    at every later step: NaN never fires in 2-bit and is -1 in 1-bit, an infinity fires in its direction forever"""
    n, steps = 2, 5
    per_word = 32 // bits
    E = 3 * per_word + 5
    slots = [M.special_steps(bits, thr, E, steps, seed=7 + k, nonfinite=nonfinite) for k in range(n)]
    kv = _store(bits, thr, [0], [np.zeros(E, np.float32)])
    codec = Codec(bits, thr, E)
    out = mx.nd.empty((E,), G)
    exact = float(np.log2(abs(thr))).is_integer() if thr else True
    for s in range(steps):
        grads = [slots[k][s] for k in range(n)]
        kv.pushpull(0, [mx.nd.array(g, G) for g in grads], out=out)
        deq = codec.push(grads)
        got = out.asnumpy()
        assert_bits_equal(got, _want(deq), "%d-bit thr %r step %d" % (bits, thr, s))
        if exact or bits == 1:
            assert_bits_equal(got, codec.exact_sum(), "%d-bit thr %r step %d vs the code counts" % (bits, thr, s))
        if nonfinite:
            unit = np.float32(thr if bits == 2 else 1.0)
            g0 = slots[0][0]
            for i in np.flatnonzero(~np.isfinite(g0)):
                if np.isnan(g0[i]):
                    want = 0.0 if bits == 2 else -n * unit
                else:
                    want = np.sign(g0[i]) * n * unit
                assert got[i] == np.float32(want), "element %d (%r at step 1) at step %d: %r" % (i, g0[i], s, got[i])


def test_skip_nonfinite_sees_a_finite_dequantised_sum():
    """the reference's behaviour, pinned: a non-finite gradient never reaches the optimizer under compression (its
    residual is sticky, its codes are finite), so a store with ``skip_nonfinite`` does not skip the step"""
    E = 4099
    rng = np.random.default_rng(3)
    w0 = rng.uniform(-1, 1, E).astype(np.float32)
    kv = _store(2, 0.5, [0], [w0], mx.optimizer.LAMB(learning_rate=0.01, wd=0.01, skip_nonfinite=True))
    out = mx.nd.empty((E,), G)
    for s in range(3):
        grads = [rng.uniform(-1, 1, E).astype(np.float32) for _ in range(2)]
        if s == 0:
            grads[0][[0, 15, E - 1]] = [np.nan, np.inf, -np.inf]
        kv.pushpull(0, [mx.nd.array(g, G) for g in grads], out=out)
        assert not kv.overflow(), "step %d was skipped" % s
        assert np.isfinite(out.asnumpy()).all()
    assert _count(kv, 0) == 3


# ---- 4. every fused optimizer on the compressed path --------------------------------------------------------------
def _ew(cls, oracle, **kw):
    return ("ew", lambda mp: cls(multi_precision=mp, **kw), lambda: oracle(**kw))


OPTS = {
    "sgd": _ew(mx.optimizer.SGD, lambda **k: O.OracleOptimizer("sgd", **k), learning_rate=0.1, wd=1e-3, rescale_grad=0.5),
    "sgd_mom": _ew(mx.optimizer.SGD, lambda **k: O.OracleOptimizer("sgd", **k), learning_rate=0.05, momentum=0.9,
                   wd=1e-3, rescale_grad=0.5),
    "nag": _ew(mx.optimizer.NAG, NG.OracleNAG, learning_rate=0.05, momentum=0.9, wd=1e-4, rescale_grad=0.5,
               clip_gradient=0.7),
    "adam": _ew(mx.optimizer.Adam, lambda **k: O.OracleOptimizer("adam", **k), learning_rate=0.01, wd=1e-3,
                rescale_grad=0.5),
    "adamw": _ew(mx.optimizer.AdamW, lambda **k: O.OracleOptimizer("adamw", **k), learning_rate=0.01, wd=1e-2,
                 epsilon=1e-6, rescale_grad=0.5),
    "rmsprop": _ew(mx.optimizer.RMSProp, RM.OracleRMSProp, learning_rate=0.01, rho=0.8, wd=1e-4, rescale_grad=0.5,
                   clip_gradient=0.7, clip_weights=0.95, centered=False),
    "rmsprop_centered": _ew(mx.optimizer.RMSProp, RM.OracleRMSProp, learning_rate=0.01, rho=0.8, wd=1e-4,
                            rescale_grad=0.5, clip_gradient=0.7, clip_weights=0.95, centered=True),
    "signum": _ew(mx.optimizer.Signum, SG.OracleSignum, learning_rate=0.01, momentum=0.9, wd=1e-4, wd_lh=1e-3,
                  rescale_grad=0.5, clip_gradient=0.7),
    "ftml": _ew(mx.optimizer.FTML, FT.OracleFTML, learning_rate=0.0025, beta1=0.5, beta2=0.9, wd=1e-4,
                rescale_grad=0.5, clip_gradient=0.7),
    "adabelief": _ew(mx.optimizer.AdaBelief, AB.OracleAdaBelief, learning_rate=0.01, beta1=0.8, wd=1e-4,
                     rescale_grad=0.5, clip_gradient=0.7),
    "adamax": _ew(mx.optimizer.Adamax, AX.OracleAdamax, learning_rate=0.002, beta1=0.5, beta2=0.9, wd=1e-4,
                  rescale_grad=0.5, clip_gradient=0.7),
    "adadelta": _ew(mx.optimizer.AdaDelta, AD.OracleAdaDelta, learning_rate=1.0, rho=0.95, wd=1e-4, rescale_grad=0.5,
                    clip_gradient=0.7),
    "nadam": _ew(mx.optimizer.Nadam, NA.OracleNadam, learning_rate=0.002, beta1=0.5, beta2=0.9, schedule_decay=0.008,
                 wd=1e-4, rescale_grad=0.5, clip_gradient=0.7),
    "test": _ew(mx.optimizer.Test, lambda **k: O.OracleOptimizer("test", **k), learning_rate=0.1, wd=1e-3,
                rescale_grad=0.5),
    "lamb": ("norm", "lamb", dict(learning_rate=0.01, wd=0.01)),
    "lans": ("norm", "lans", dict(learning_rate=0.01, wd=0.01)),
    "lars": ("norm", "lars", dict(learning_rate=0.1, wd=0.05, eta=0.01, momentum=0.9)),
}


class _tuned(object):
    """the staged-kernel setting for one test ('on' 2: wherever eligible, 'off' 0: never, 'auto' 1: the default
    policy), restored to auto whatever happens; counts the dense launches of each variant"""
    MODE = {"on": 2, "off": 0, "auto": 1}

    def __init__(self, bulk):
        self.bulk = bulk

    def __enter__(self):
        mx.kv.set_tuning(bulk=self.MODE[self.bulk])
        self.before = {v: mx.kv.launch_count(v) for v in ("per_thread", "bulk")}
        return self

    def launched(self, v):
        return mx.kv.launch_count(v) - self.before[v]

    def __exit__(self, *a):
        mx.kv.set_tuning(bulk=1)


# launches of one compressed LAMB / LANS / LARS update (test_gpu_norm_edges.py LAUNCHES: the norm phases)
NORM_LAUNCHES = {"lamb": 3, "lans": 5, "lars": 3}


@pytest.mark.parametrize("mp", [False, True])
@pytest.mark.parametrize("E,bulk", [(4100, "on"), (4100, "off"), (4097, "on"), (4100, "auto")])
@pytest.mark.parametrize("n", [1, 2, 5])
@pytest.mark.parametrize("name", list(OPTS))
def test_every_fused_optimizer_under_compression(name, n, E, bulk, mp):
    """three steps of each fused optimizer on the sum of n dequantised 2-bit streams: the staged kernel (<= 2
    sources, E a multiple of 4, forced on), the per-thread kernel (forced, or 5 sources under the default policy),
    the scalar path (E odd), and the multi-precision instantiation on a float32 key; weights, states, the update
    count and the launches of every step"""
    spec = OPTS[name]
    bits, thr = 2, 0.5
    rng = np.random.default_rng(zlib.crc32(repr((name, n, E, bulk, mp)).encode()))
    w0 = rng.uniform(-1, 1, E).astype(np.float32)
    if spec[0] == "ew":
        opt = spec[1](mp)
        oracle = spec[2]()
    else:
        opt = mx.optimizer.create(spec[1], multi_precision=mp, **spec[2])
        track = Track(spec[1], spec[2], w0)
    with _tuned(bulk) as f:
        kv = _store(bits, thr, [0], [w0], opt)
        okv = O.OracleKVStore("device")
        okv.init(0, w0.copy())
        if spec[0] == "ew":
            okv.set_optimizer(oracle)
        codec = Codec(bits, thr, E, model=False)
        out = mx.nd.empty((E,), G)
        update = 1 if spec[0] == "ew" else NORM_LAUNCHES[spec[1]]
        for s in range(3):
            grads = [rng.uniform(-1.5, 1.5, E).astype(np.float32) for _ in range(n)]
            vals = [mx.nd.array(g, G) for g in grads]
            mx.nd.waitall()
            before = mx.kv.launch_count()
            kv.pushpull(0, vals, out=out)
            mx.nd.waitall()
            what = "%s n=%d E=%d bulk=%s mp=%s step %d" % (name, n, E, bulk, mp, s)
            # a quantize and a dequantize per source, the update; the first step also casts the fp32 master
            want_launches = 2 * n + update + (1 if mp and s == 0 else 0)
            assert mx.kv.launch_count() - before == want_launches, what + ": launches"
            deq = codec.push(grads)
            if spec[0] == "ew":
                okv.push(0, deq)
                want = np.empty(E, np.float32)
                okv.pull(0, want)
                assert_bits_equal(out.asnumpy(), want, what)
            else:
                track.check(kv, 0, _want(deq), out, _ratio_eps(E, _default_chunk()), what)
        mx.nd.waitall()
        if spec[0] == "ew":
            for i, st in enumerate(_states_of(oracle, 0)):
                assert_bits_equal(_state(kv, 0, 2 + i), st, "%s state %d" % (name, i))
            if len(_states_of(oracle, 0)) < 3:
                assert _state(kv, 0, 2 + len(_states_of(oracle, 0))) is None, "%s: a state too many" % name
            assert f.launched("bulk") + f.launched("per_thread") == 3
            if bulk == "off" or E % 4:    # never the staged kernel, or a size that keeps the scalar path
                assert f.launched("bulk") == 0, "bulk launches %d" % f.launched("bulk")
            elif bulk == "on" and n <= 2:
                assert f.launched("bulk") == 3, "bulk launches %d" % f.launched("bulk")
            elif bulk == "auto" and n >= 3:   # enough sources keep loads in flight: the per-thread kernel
                assert f.launched("per_thread") == 3, "per-thread launches %d" % f.launched("per_thread")
        if mp:
            assert_bits_equal(_state(kv, 0, 1), out.asnumpy(), "the float32 master is the weight")
        else:
            assert _state(kv, 0, 1) is None
    assert _count(kv, 0) == 3


# ---- 5. the steps AdamW and AdaBelief skip --------------------------------------------------------------------------
SKIPPERS = {
    "adamw": (mx.optimizer.AdamW, lambda **k: O.OracleOptimizer("adamw", **k),
              dict(learning_rate=0.01, wd=1e-2, epsilon=1e-6, rescale_grad=0.5)),
    "adabelief": (mx.optimizer.AdaBelief, AB.OracleAdaBelief,
                  dict(learning_rate=0.01, beta1=0.8, wd=1e-4, rescale_grad=0.5)),
}


@pytest.mark.parametrize("how", ["pushpull", "push_pull"])
@pytest.mark.parametrize("bad", [float("inf"), 0.0])
@pytest.mark.parametrize("name", list(SKIPPERS))
def test_a_skipped_step_still_advances_the_residuals(name, bad, how):
    """AdamW / AdaBelief leave weight and state alone when rescale_grad is 0, inf or nan -- but the reference has
    reduced the push first (kvstore_local.h:240-280), and under compression that quantises every pushed value and
    moves its residual on.  Step 2 is skipped; steps 3 and 4 must continue from the advanced residuals.  The
    skipped step launches the quantisations only, and counts the update once"""
    cls, ocls, kw = SKIPPERS[name]
    sizes = [4099, 64]
    keys = [0, 1]
    n = 2
    rng = np.random.default_rng(5)
    w0 = [rng.uniform(-1, 1, e).astype(np.float32) for e in sizes]
    opt, oopt = cls(**kw), ocls(**kw)
    kv = _store(2, 0.5, keys, w0, opt)
    okv = O.OracleKVStore("device")
    okv.init(keys, [w.copy() for w in w0])
    okv.set_optimizer(oopt)
    codecs = [Codec(2, 0.5, e) for e in sizes]
    outs = [mx.nd.empty((e,), G) for e in sizes]
    for step in (1, 2, 3, 4):
        rg = bad if step == 2 else 0.5
        opt.rescale_grad = oopt.rescale_grad = rg
        kv.set_optimizer(opt)
        grads = [[rng.uniform(-1, 1, e).astype(np.float32) for _ in range(n)] for e in sizes]
        vals = [[mx.nd.array(g, G) for g in gs] for gs in grads]
        held = [(o.asnumpy(), _state(kv, k, 2), _state(kv, k, 3)) for k, o in zip(keys, outs)] if step == 2 else None
        mx.nd.waitall()
        before = mx.kv.launch_count()
        if how == "pushpull":
            kv.pushpull(keys, vals, out=outs)
        else:
            kv.push(keys, vals)
            kv.pull(keys, out=outs)
        mx.nd.waitall()
        if step == 2:
            assert mx.kv.launch_count() - before == n * len(keys), "a skipped step quantises and launches nothing else"
        okv.push(keys, [c.push(gs) for c, gs in zip(codecs, grads)])
        for k in keys:
            want = np.empty(sizes[k], np.float32)
            okv.pull(k, want)
            assert_bits_equal(outs[k].asnumpy(), want, "%s rescale %r step %d key %d" % (name, bad, step, k))
            for i, st in enumerate(_states_of(oopt, k)):
                assert_bits_equal(_state(kv, k, 2 + i), st, "%s step %d key %d state %d" % (name, step, k, i))
            assert _count(kv, k) == step
        if step == 2:
            for k, (w, s0, s1) in zip(keys, held):
                assert_bits_equal(outs[k].asnumpy(), w, "the skipped step changed key %d" % k)
                assert_bits_equal(_state(kv, k, 2), s0)
                assert_bits_equal(_state(kv, k, 3), s1)


@pytest.mark.parametrize("name", list(SKIPPERS))
def test_a_skipped_trainer_step_still_advances_the_residuals(name):
    """the same through the Trainer with ``compression_params``, the loss scale making step 2's rescale_grad inf
    (as a dynamic loss scale that met an overflow does)"""
    import torch
    cls, ocls, kw = SKIPPERS[name]
    kw = {k: v for k, v in kw.items() if k != "rescale_grad"}
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(33, 17), torch.nn.ReLU(), torch.nn.Linear(17, 5)).cuda()
    params = list(model.parameters())
    trainer = mx.Trainer(params, cls(**kw), kvstore="device", compression_params={"type": "2bit", "threshold": 0.5})
    oopt = ocls(**kw)
    ref_w = [p.detach().cpu().numpy().copy().reshape(-1) for p in params]
    codecs = [Codec(2, 0.5, w.size) for w in ref_w]
    x = torch.randn(8, 33, device="cuda")
    for step in (1, 2, 3, 4):
        model.zero_grad()
        (model(x).square().sum() * 40).backward()
        grads = [p.grad.detach().cpu().numpy().copy().reshape(-1) for p in params]
        kv = trainer._kvstore
        held = [(_state(kv, i, 2), _state(kv, i, 3)) for i in range(len(params))] if step == 2 else None
        trainer._scale = float("inf") if step == 2 else 1.0        # what AMP's loss scaler writes
        trainer.step(8)
        torch.cuda.synchronize()
        kv = trainer._kvstore
        oopt.rescale_grad = trainer._scale / 8
        for i, (w, g) in enumerate(zip(ref_w, grads)):
            oopt.update(i, w, codecs[i].push([g])[0])
        for i, (p, w) in enumerate(zip(params, ref_w)):
            what = "%s step %d param %d" % (name, step, i)
            assert_bits_equal(p.detach().cpu().numpy(), w, what)
            for j, st in enumerate(_states_of(oopt, i)):
                assert_bits_equal(_state(kv, i, 2 + j), st, what + " state %d" % j)
            assert _count(kv, i) == step, what + ": update count"
            if step == 2:
                assert_bits_equal(_state(kv, i, 2), held[i][0], what + ": the skipped step changed state 0")
                assert_bits_equal(_state(kv, i, 3), held[i][1], what + ": the skipped step changed state 1")


# ---- 6. residual bookkeeping ----------------------------------------------------------------------------------------
def test_several_keys_and_a_changing_number_of_sources():
    """keys of different sizes in one call, 2 -> 4 -> 2 -> 4 values per key: slots 2 and 3 resume from their own
    residuals; host-resident values mixed with device values stage through the same slots"""
    sizes = [17, 4099, 1000]
    keys = [0, 1, 2]
    rng = np.random.default_rng(11)
    kv = _store(2, 0.5, keys, [np.zeros(e, np.float32) for e in sizes])
    codecs = [Codec(2, 0.5, e) for e in sizes]
    outs = [mx.nd.empty((e,), G) for e in sizes]
    for step, n in enumerate([2, 4, 2, 4, 3]):
        grads = [[rng.uniform(-1, 1, e).astype(np.float32) for _ in range(n)] for e in sizes]
        ctx = [[mx.cpu() if (step >= 3 and j % 2) else G for j in range(n)] for _ in sizes]
        kv.pushpull(keys, [[mx.nd.array(g, c) for g, c in zip(gs, cs)] for gs, cs in zip(grads, ctx)], out=outs)
        for k in keys:
            deq = codecs[k].push(grads[k])
            assert_bits_equal(outs[k].asnumpy(), _want(deq), "step %d n %d key %d" % (step, n, k))
            assert_bits_equal(outs[k].asnumpy(), codecs[k].exact_sum())


def test_outputs_that_alias_the_pushed_values():
    """pushpull(key, vals, out=vals): the kernel reads the dequantised scratch, so the outputs may be the inputs"""
    E, n = 4099, 3
    rng = np.random.default_rng(12)
    kv = _store(1, 0.0, [0], [np.zeros(E, np.float32)])
    codec = Codec(1, 0.0, E)
    for step in range(3):
        grads = [rng.uniform(-1, 1, E).astype(np.float32) for _ in range(n)]
        vals = [mx.nd.array(g, G) for g in grads]
        kv.pushpull(0, vals, out=vals)
        want = _want(codec.push(grads))
        for v in vals:
            assert_bits_equal(v.asnumpy(), want, "step %d" % step)


def test_deferred_prioritised_calls():
    """a deferred store issues compressed calls one by one (compression is not merged): two calls of different
    priority, each on its own key, both reach the right residuals"""
    sizes = [100, 33]
    rng = np.random.default_rng(13)
    kv = _store(2, 0.5, [0, 1], [np.zeros(e, np.float32) for e in sizes])
    codecs = [Codec(2, 0.5, e) for e in sizes]
    outs = [mx.nd.empty((e,), G) for e in sizes]
    kv.set_deferred(True)
    try:
        for step in range(3):
            grads = [[rng.uniform(-1, 1, e).astype(np.float32) for _ in range(2)] for e in sizes]
            kv.pushpull(1, [mx.nd.array(g, G) for g in grads[1]], out=outs[1], priority=-1)
            kv.pushpull(0, [mx.nd.array(g, G) for g in grads[0]], out=outs[0], priority=0)
            kv.flush()
            for k in (0, 1):
                assert_bits_equal(outs[k].asnumpy(), _want(codecs[k].push(grads[k])), "step %d key %d" % (step, k))
    finally:
        kv.set_deferred(False)


def test_checkpoint_reload_starts_from_zero_residuals():
    """save_optimizer_states after step 2 and a reload into a fresh store: weights, Adam state and count continue,
    and the fresh store's residuals start at zero -- as the reference's do, which keeps them in the store's
    gradient-compression object and never writes them to a state file"""
    E, n = 4099, 2
    kw = dict(learning_rate=0.01, wd=1e-3, rescale_grad=0.5)
    rng = np.random.default_rng(14)
    w0 = rng.uniform(-1, 1, E).astype(np.float32)
    kv = _store(2, 0.5, [0], [w0], mx.optimizer.Adam(**kw))
    oopt = O.OracleOptimizer("adam", **kw)
    okv = O.OracleKVStore("device")
    okv.init(0, w0.copy())
    okv.set_optimizer(oopt)
    codec = Codec(2, 0.5, E)
    out = mx.nd.empty((E,), G)
    for step in range(4):
        if step == 2:
            tmp = tempfile.mkdtemp(prefix="mxkv_gc_states_")
            try:
                fname = os.path.join(tmp, "states")
                kv.save_optimizer_states(fname, dump_optimizer=True)      # with its update counts
                w = out.asnumpy()
                kv = _store(2, 0.5, [0], [w], mx.optimizer.Adam(**kw))
                kv.load_optimizer_states(fname)
            finally:
                shutil.rmtree(tmp)
            assert _count(kv, 0) == 2 and kv._optimizer._index_update_count[0] == 2, "the count was not restored"
            codec = Codec(2, 0.5, E)                         # the reloaded store's residuals are zero
        grads = [rng.uniform(-1, 1, E).astype(np.float32) for _ in range(n)]
        kv.pushpull(0, [mx.nd.array(g, G) for g in grads], out=out)
        okv.push(0, codec.push(grads))
        want = np.empty(E, np.float32)
        okv.pull(0, want)
        assert_bits_equal(out.asnumpy(), want, "step %d" % step)
    assert _count(kv, 0) == 4


def test_refusals_leave_everything_untouched():
    """a float16 key and a Python updater callback are refused with the existing messages; the weights, the counts
    and another key's residuals are as before"""
    E = 100
    rng = np.random.default_rng(15)
    kv = mx.kv.create("device")
    kv.set_gradient_compression({"type": "2bit", "threshold": 0.5})
    kv.init(0, mx.nd.zeros((E,), G))
    kv.init(1, mx.nd.zeros((E,), G, dtype=np.float16))
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9))
    codec = Codec(2, 0.5, E)
    okv = O.OracleKVStore("device")
    okv.init(0, np.zeros(E, np.float32))
    okv.set_optimizer(O.OracleOptimizer("sgd", learning_rate=0.1, momentum=0.9))
    out = mx.nd.empty((E,), G)

    def good_step():
        grads = [rng.uniform(-1, 1, E).astype(np.float32) for _ in range(2)]
        kv.pushpull(0, [mx.nd.array(g, G) for g in grads], out=out)
        okv.push(0, codec.push(grads))
        want = np.empty(E, np.float32)
        okv.pull(0, want)
        assert_bits_equal(out.asnumpy(), want)

    good_step()
    w16 = mx.nd.empty((E,), G, dtype=np.float16)
    kv.pull(1, out=w16)
    before16 = w16.asnumpy().copy()
    with pytest.raises(Exception, match="Gradient compression is only supported for float32"):
        kv.pushpull(1, [mx.nd.ones((E,), G, dtype=np.float16)] * 2, out=w16)
    kv.pull(1, out=w16)
    assert np.array_equal(w16.asnumpy().view(np.uint16), before16.view(np.uint16))
    assert _count(kv, 0) == 1
    good_step()

    w2 = rng.uniform(-1, 1, E).astype(np.float32)
    kv2 = _store(2, 0.5, [0], [w2])
    kv2._set_updater(lambda key, recv, local: local.__iadd__(recv))
    out2 = mx.nd.array(np.full(E, 7.0, np.float32), G)
    with pytest.raises(Exception, match="gradient compression together with a Python updater callback"):
        kv2.pushpull(0, [mx.nd.ones((E,), G)], out=out2)
    assert np.all(out2.asnumpy() == 7.0), "the refused call wrote its output"
    kv2.pull(0, out=out2)
    assert_bits_equal(out2.asnumpy(), w2, "the refused call changed the weight")
    good_step()
    assert _count(kv, 0) == 3 and _count(kv, 1) == 0


# ---- 7. several GPUs ---------------------------------------------------------------------------------------------------
@pytest.mark.multigpu
@pytest.mark.parametrize("name", ["adam", "nadam"])
def test_several_consumers_and_a_moving_slot(name):
    """2 to 4 GPUs, outputs on every GPU and on one that pushed nothing, the device set changing between calls so that
    a residual slot moves to another GPU; the update count advances once per call, not once per consumer"""
    ndev = min(mx.num_gpus(), 4)
    if ndev < 2:
        pytest.skip("needs 2 GPUs")
    spec = OPTS[name]
    E = 4099
    rng = np.random.default_rng(16)
    w0 = rng.uniform(-1, 1, E).astype(np.float32)
    kv = _store(2, 0.5, [0], [w0], spec[1](False))
    oracle = spec[2]()
    okv = O.OracleKVStore("device")
    okv.init(0, w0.copy())
    okv.set_optimizer(oracle)
    codec = Codec(2, 0.5, E)
    plans = [list(range(ndev)), list(range(ndev))[::-1], [ndev - 1], list(range(ndev))]
    for step, devs in enumerate(plans):
        grads = [rng.uniform(-1, 1, E).astype(np.float32) for _ in devs]
        outs = [mx.nd.empty((E,), mx.gpu(d)) for d in range(ndev)]
        kv.pushpull(0, [mx.nd.array(g, mx.gpu(d)) for g, d in zip(grads, devs)], out=outs)
        okv.push(0, codec.push(grads))
        want = np.empty(E, np.float32)
        okv.pull(0, want)
        for d, o in enumerate(outs):
            assert_bits_equal(o.asnumpy(), want, "%s step %d GPU %d" % (name, step, d))
        assert _count(kv, 0) == step + 1
