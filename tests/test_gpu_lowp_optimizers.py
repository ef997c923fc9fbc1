"""The fused optimizers on float16 / bfloat16 keys -- the path of the BERT-base bf16 multi-precision Adam workload:
4-element packets of the per-thread kernel, an fp32 master and fp32 state, one rounding to the key type on the way
out -- against ``lp_oracle.LpOracle`` (the oracle's mp_sgd / mp_sgd_mom / mp_adam / mp_adamw / NAG kernels), bit for
bit on the 16-bit output, the master and the state.  Also: the copy-out rounding against numpy / an integer
round-to-nearest-even, the fp32-accumulate flag of float16 sums, the cached-plan / checkpoint / native-updater /
Trainer lifecycle, sharded state over several GPUs, and one step of every optimizer against a float64
restatement of the operator."""
import os
import sys
import tempfile

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import mxnet_b200 as mx
from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import lp_oracle as L  # noqa: E402

_SIM = bool(os.environ.get("MXKV_SIM"))
# the simulator runs the kernels on one CPU core: the same boundaries, a smaller largest key
SIZES = [1, 3, 7, 8, 4099, 8192 + 4] + ([20011] if _SIM else [100003, (1 << 20) + 8])
DT = {1: np.float16, 2: "bfloat16"}
KIND = {"float16": 1, "bfloat16": 2}
# option sets of the matrix; rescale_grad != 1 everywhere so that its place in each formula matters
OPTS = {
    "sgd": ("sgd", dict(learning_rate=0.1, wd=1e-3, rescale_grad=0.5)),
    "sgd_mom": ("sgd", dict(learning_rate=0.05, momentum=0.9, wd=1e-3, rescale_grad=0.5)),
    "nag": ("nag", dict(learning_rate=0.05, momentum=0.9, wd=1e-3, rescale_grad=0.5)),
    "adam": ("adam", dict(learning_rate=0.01, wd=1e-3, rescale_grad=0.5)),
    "adamw": ("adamw", dict(learning_rate=0.01, wd=1e-2, rescale_grad=0.5)),
    "test": ("test", dict(learning_rate=0.1, wd=1e-3, rescale_grad=0.5)),
}
HAS = {"sgd": (), "test": (), "sgd_mom": (2,), "nag": (2,), "adam": (2, 3), "adamw": (2, 3)}


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32}[a.dtype.itemsize])


def assert_bits_equal(a, b, msg=""):
    a, b = np.asarray(a).reshape(-1), np.asarray(b).reshape(-1)
    assert a.shape == b.shape, (a.shape, b.shape, msg)
    ne = _bits(a) != _bits(b)
    if ne.any():
        i = int(np.argwhere(ne)[0][0])
        raise AssertionError("%s: %d / %d elements differ, first at %d: %r vs %r" % (msg, ne.sum(), ne.size, i,
                                                                                     a[i], b[i]))


def _nd(bits, kind, ctx=None):
    ctx = ctx or mx.gpu(0)
    if kind == 0:
        return mx.nd.array(bits, ctx)
    return mx.nd.array(bits.view(np.float16) if kind == 1 else bits, ctx, dtype=DT[kind])


def _get(nd, kind):
    """an engine array as uint16 bit patterns (16-bit) or float32"""
    if kind == 0:
        return nd.asnumpy().reshape(-1)
    return (nd.asnumpy(raw=True) if kind == 2 else nd.asnumpy().view(np.uint16)).reshape(-1)


def _state(kv, key, which):
    h = kv._state_handle(key, which)
    return None if h is None else h.asnumpy().reshape(-1)


def _gsum(g, kind, kvtype="device"):
    """the fp32 gradient sum the engine hands a fused optimizer: CommDevice / CommCPU order, fp32 accumulation"""
    if kvtype == "local":
        return O.sum_cpu([L.widen(x, kind) for x in g])
    return O.sum_device_lp_f32out(g, kind) if kind else O.sum_device(g)


def _check_state(kv, lo, key, optkey, msg):
    if lo.kind == 0 and not lo.multi_precision:
        assert _state(kv, key, 1) is None, "%s: a float32 key without multi_precision has a master" % msg
    else:
        assert_bits_equal(_state(kv, key, 1), lo.w32[key], "%s master" % msg)
    for which in (2, 3):
        got = _state(kv, key, which)
        if which in HAS[optkey]:
            assert_bits_equal(got, (lo.s0, lo.s1)[which - 2][key], "%s state %d" % (msg, which - 1))
        else:
            assert got is None, "%s: unexpected state %d" % (msg, which - 1)


def _store(name, kw, kind, keys, w0, kvtype="device", mults=None, ctx=None):
    kv = mx.kv.create(kvtype)
    kv.init(keys, [_nd(w, kind, ctx) for w in w0])
    opt = mx.optimizer.create(name, **kw)
    if mults:
        opt.set_lr_mult(mults[0])
        opt.set_wd_mult(mults[1])
    kv.set_optimizer(opt)
    lo = L.LpOracle(name, kind, lr_mult=mults and mults[0], wd_mult=mults and mults[1], **kw)
    for k, w in zip(keys, w0):
        lo.init(k, w)
    return kv, lo


def _run(optkey, kind, mp, sizes=SIZES, n=3, steps=4, kvtype="device", kw_extra=None, mults=None, seed=0,
         gscale=1.0, rewiden_check=False):
    """``steps`` multi-key pushpulls of n 16-bit gradients per key, each output bit-exact against LpOracle;
    the master and the state at the end.  Returns (kv, oracle, the fp32 gradient sums of the last step, the
    outputs)."""
    name, kw = OPTS[optkey]
    kw = dict(kw, multi_precision=mp, **(kw_extra or {}))
    rng = np.random.default_rng(seed + 97 * kind + len(sizes) + n)
    keys = list(range(len(sizes)))
    w0 = [L.to_lp(rng.uniform(-1, 1, e).astype(np.float32), kind) for e in sizes]
    kv, lo = _store(name, kw, kind, keys, w0, kvtype, mults)
    other = L.LpOracle(name, kind, rewiden=True, lr_mult=mults and mults[0], wd_mult=mults and mults[1], **kw)
    for k, w in zip(keys, w0):
        other.init(k, w)
    differs = False
    outs = [mx.nd.empty((e,), mx.gpu(0), dtype=DT.get(kind, np.float32)) for e in sizes]
    sums = []
    for s in range(steps):
        g = [[L.to_lp(gscale * rng.uniform(-1, 1, e).astype(np.float32), kind) for _ in range(n)] for e in sizes]
        kv.pushpull(keys, [[_nd(x, kind) for x in gs] for gs in g], out=outs)
        sums = [_gsum(gs, kind, kvtype) for gs in g]
        for k in keys:
            want = lo.update(k, sums[k])
            assert_bits_equal(_get(outs[k], kind), want, "%s kind=%d mp=%s %s n=%d E=%d step %d" % (
                optkey, kind, mp, kvtype, n, sizes[k], s))
            if rewiden_check:
                differs = differs or not np.array_equal(other.update(k, sums[k]), want)
    for k in keys:
        _check_state(kv, lo, k, optkey, "%s kind=%d mp=%s E=%d" % (optkey, kind, mp, sizes[k]))
    if rewiden_check:
        assert differs, "a master re-widened from the 16-bit weight gives the same results on this data: the " \
                        "test cannot tell it from the persistent master"
    return kv, lo, sums, outs


# ---------------------------------------------------------------------------
# the matrix: optimizers x dtype x multi_precision
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("mp", [False, True])
@pytest.mark.parametrize("lp", ["float16", "bfloat16"])
@pytest.mark.parametrize("optkey", list(OPTS))
def test_optimizer_matrix(optkey, lp, mp):
    """every 16-bit key with a fused optimizer keeps a persistent fp32 master, with or without multi_precision;
    the 16-bit weight is the master rounded once.  Without multi_precision the results must differ from a master
    re-widened from the stored weight every step (which is what the test would see if the engine did that)"""
    _run(optkey, KIND[lp], mp, rewiden_check=not mp)


@pytest.mark.parametrize("n", [1, 2, 5])
@pytest.mark.parametrize("lp", ["float16", "bfloat16"])
def test_source_counts(lp, n):
    """1 and 2 sources (the small-n kernel), 5 (crosses the per-thread kernel's 4-source load batch)"""
    for optkey in ("adam", "sgd_mom"):
        _run(optkey, KIND[lp], True, n=n, steps=3, seed=n)


@pytest.mark.parametrize("lp", ["float16", "bfloat16"])
def test_local_store_commcpu_order(lp):
    """kv.create('local'): six sources are summed in CommCPU's groups of four, in fp32, before the update"""
    for optkey in ("adamw", "nag"):
        _run(optkey, KIND[lp], lp == "bfloat16", n=6, steps=3, kvtype="local", seed=6)


def test_unaligned_view_takes_the_scalar_path():
    """16-bit torch views offset by one element (2-byte aligned only): the scalar path of the per-thread kernel"""
    import torch
    E, n, kind = 10001, 3, 2
    rng = np.random.default_rng(12)
    w0 = L.to_lp(rng.uniform(-1, 1, E).astype(np.float32), kind)
    kv, lo = _store("adam", dict(OPTS["adam"][1], multi_precision=True), kind, [0], [w0])
    wbase = torch.zeros(E + 3, dtype=torch.bfloat16, device="cuda")
    wview = wbase[1:E + 1]
    for s in range(3):
        g = [L.to_lp(rng.uniform(-1, 1, E).astype(np.float32), kind) for _ in range(n)]
        gbase = [torch.zeros(E + 3, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
        for b, x in zip(gbase, g):
            b[1:E + 1].copy_(torch.from_numpy(x.view(np.int16)).view(torch.bfloat16))
        torch.cuda.synchronize()
        kv.pushpull(0, [mx.nd.from_torch(b[1:E + 1]) for b in gbase], out=mx.nd.from_torch(wview))
        mx.nd.waitall()
        got = wview.view(torch.int16).cpu().numpy().view(np.uint16)
        assert_bits_equal(got, lo.update(0, _gsum(g, kind)), "unaligned view step %d" % s)


# ---------------------------------------------------------------------------
# option grid
# ---------------------------------------------------------------------------
GRID = {
    # Trainer.step's rescale_grad = 1 / (batch * world) and a clip that binds after it
    "clip_rescale": (dict(rescale_grad=1.0 / 32, clip_gradient=0.03), None),
    "wd0": (dict(wd=0.0), None),
    "mults": (dict(), ({1: 0.5, 4: 2.0}, {2: 0.0, 4: 3.0})),
    "eps": (dict(epsilon=1e-3), None),
}


@pytest.mark.parametrize("optkey,grid", [(o, g) for o in ("adam", "adamw") for g in GRID] +
                         [("adamw", "no_bias_correction_eta"), ("sgd_mom", "clip_rescale"), ("sgd_mom", "mults")])
def test_option_grid(optkey, grid):
    extra, mults = (dict(correct_bias=False, eta=0.7), None) if grid == "no_bias_correction_eta" else GRID[grid]
    sizes = SIZES[:6] + [20011]
    for kind in (1, 2):
        _, lo, sums, _ = _run(optkey, kind, kind == 2, sizes=sizes, steps=3, kw_extra=extra, mults=mults,
                              seed=len(grid))
        if "clip_gradient" in extra:
            big = max(float(np.abs(np.float32(lo.rescale_grad) * s).max()) for s in sums)
            assert big > extra["clip_gradient"], "the clip never binds on this data"


def test_option_grid_takes_effect():
    """each option of the grid changes the result (a run that ignored it would not match the oracle either, but
    this keeps the grid from silently degenerating)"""
    base = _run("adamw", 2, True, sizes=[4099], steps=3, seed=3)[1].w32[0]
    for extra in (dict(rescale_grad=1.0 / 32, clip_gradient=0.03), dict(wd=0.0), dict(epsilon=1e-3),
                  dict(correct_bias=False), dict(eta=0.7)):
        got = _run("adamw", 2, True, sizes=[4099], steps=3, seed=3, kw_extra=extra)[1].w32[0]   # (the master)
        assert not np.array_equal(got, base), extra


@pytest.mark.parametrize("bad", [0.0, float("inf"), float("nan")])
def test_adamw_skips_on_a_bad_rescale(bad):
    """contrib/adamw-inl.h:455: a rescale_grad of 0 / inf / nan leaves the 16-bit weight, the master and the state
    untouched (the update count still moves on, as Optimizer._update_count has run)"""
    kind, sizes = 2, [7, 4099]
    keys = [0, 1]
    rng = np.random.default_rng(21)
    w0 = [L.to_lp(rng.uniform(-1, 1, e).astype(np.float32), kind) for e in sizes]
    kv, lo = _store("adamw", dict(OPTS["adamw"][1], multi_precision=False), kind, keys, w0)
    outs = [mx.nd.empty((e,), mx.gpu(0), dtype="bfloat16") for e in sizes]

    def step(tag):
        g = [[L.to_lp(rng.uniform(-1, 1, e).astype(np.float32), kind) for _ in range(2)] for e in sizes]
        kv.pushpull(keys, [[_nd(x, kind) for x in gs] for gs in g], out=outs)
        for k in keys:
            assert_bits_equal(_get(outs[k], kind), lo.update(k, _gsum(g[k], kind)), "%s key %d" % (tag, k))

    step("before")
    held = [(_get(outs[k], kind), _state(kv, k, 1), _state(kv, k, 2), _state(kv, k, 3)) for k in keys]
    opt = kv._optimizer
    opt.rescale_grad = lo.rescale_grad = bad
    kv.set_optimizer(opt)
    step("skipped")
    for k in keys:
        for a, b in zip(held[k], (_get(outs[k], kind), _state(kv, k, 1), _state(kv, k, 2), _state(kv, k, 3))):
            assert_bits_equal(b, a, "rescale %r changed key %d" % (bad, k))
    opt.rescale_grad = lo.rescale_grad = 0.5
    kv.set_optimizer(opt)
    step("after")


# ---------------------------------------------------------------------------
# the fp32-accumulate flag of float16 sums without an optimizer
# ---------------------------------------------------------------------------
def test_fp16_fp32_accumulate_flag(monkeypatch):
    """MXKV_B200_FP16_FP32_ACCUM=1: float16 pushes without an optimizer are summed in fp32 and rounded once"""
    monkeypatch.setenv("MXKV_B200_FP16_FP32_ACCUM", "1")
    differs = False
    for n in (2, 3, 5):
        for E in (3, 4099, 70001):
            rng = np.random.default_rng(E + n)
            vals = [rng.uniform(-1, 1, E).astype(np.float16) for _ in range(n)]
            kv = mx.kv.create("device")
            kv.init(0, mx.nd.zeros((E,), mx.gpu(0), dtype=np.float16))
            out = mx.nd.empty((E,), mx.gpu(0), dtype=np.float16)
            kv.pushpull(0, [mx.nd.array(v, mx.gpu(0), dtype=np.float16) for v in vals], out=out)
            want = O.sum_device_lp_f32out([v.view(np.uint16) for v in vals], 1).astype(np.float16)
            assert_bits_equal(out.asnumpy(), want, "fp32-accumulated fp16 n=%d E=%d" % (n, E))
            differs = differs or not np.array_equal(want.view(np.uint16), O.sum_device(vals).view(np.uint16))
    assert differs, "per-add rounding gives the same sums on this data: the flag is not tested"


# ---------------------------------------------------------------------------
# the copy-out rounding at the format edges, against references that share no code with the kernel or the oracle
# ---------------------------------------------------------------------------
def _rne_bf16(x32):
    """round-to-nearest-even of float32 values to bfloat16, on the integer bits"""
    u = np.ascontiguousarray(x32, np.float32).view(np.uint32)
    hi, lo = (u >> 16).astype(np.uint32), u & 0xFFFF
    up = (lo > 0x8000) | ((lo == 0x8000) & ((hi & 1) == 1))
    return (hi + up.astype(np.uint32)).astype(np.uint16)


def _edge_cases(kind):
    """(g1, g2, rescale) with 16-bit g1, g2 and g1 + g2, rescale * (g1 + g2) exact in float32"""
    if kind == 2:
        p = lambda e: 2.0 ** e                                                     # noqa: E731
        ties = [(1.0, p(-8)), (1.0 + p(-7), p(-8)), (1.0, p(-8) + p(-9)), (-1.0, -p(-8)), (4.0, p(-6)),
                ((2 - p(-7)) * p(126), p(118)),          # odd neighbour at the top of the range: rounds up to 2^127
                ((2 - p(-7)) * p(127), p(119))]          # halfway past the largest bf16: +inf
        sub = [(3 * p(-133), 0.0), (5 * p(-133), 0.0), (p(-126), -p(-133)), (7 * p(-133), p(-133))]
    else:
        p = lambda e: 2.0 ** e                                                     # noqa: E731
        ties = [(1.0, p(-11)), (1.0 + p(-10), p(-11)), (1.0, p(-11) + p(-12)), (-1.0, -p(-11)), (1024.0, 0.5),
                (65504.0, 15.0),                         # 65519: rounds to 65504
                (65504.0, 16.0)]                         # 65520: halfway past the largest float16, +inf
        sub = [(3 * p(-24), 0.0), (5 * p(-24), 0.0), (p(-14), -p(-24)), (p(-14), p(-24) * 3), (7 * p(-24), p(-24))]
    return ties, sub


@pytest.mark.parametrize("lp", ["float16", "bfloat16"])
def test_copy_out_rounding_at_the_format_edges(lp):
    """SGD with lr = 1, wd = 0 and a zero initial weight stores w32 = -rescale * (g1 + g2), exactly; the 16-bit
    weight must be that value rounded to nearest-even: ties both ways, the largest finite value and +inf (the
    master stays finite), and values that land in the 16-bit subnormal range (rescale 0.5 moves them below the
    16-bit grid)"""
    kind = KIND[lp]
    ties, sub = _edge_cases(kind)
    for cases, rescale in ((ties, 1.0), (sub, 0.5)):
        g1 = np.array([-a for a, _ in cases], np.float64)
        g2 = np.array([-b for _, b in cases], np.float64)
        exact = -rescale * (g1 + g2)
        assert np.array_equal(exact.astype(np.float32).astype(np.float64), exact), "a case is not exact in fp32"
        b1, b2 = L.to_lp(g1.astype(np.float32), kind), L.to_lp(g2.astype(np.float32), kind)
        assert np.array_equal(L.widen(b1, kind), g1.astype(np.float32)) and \
            np.array_equal(L.widen(b2, kind), g2.astype(np.float32)), "a gradient is not a %s value" % lp
        E = len(cases)
        kv = mx.kv.create("device")
        kv.init(0, _nd(np.zeros(E, np.uint16), kind))
        kv.set_optimizer(mx.optimizer.SGD(learning_rate=1.0, wd=0.0, rescale_grad=rescale))
        out = mx.nd.empty((E,), mx.gpu(0), dtype=DT[kind])
        kv.pushpull(0, [_nd(b1, kind), _nd(b2, kind)], out=out)
        x32 = exact.astype(np.float32)
        with np.errstate(over="ignore"):
            want = x32.astype(np.float16).view(np.uint16) if kind == 1 else _rne_bf16(x32)
        assert_bits_equal(_get(out, kind), want, "%s copy-out rescale %g" % (lp, rescale))
        assert_bits_equal(_state(kv, 0, 1), x32, "%s master" % lp)
        assert np.isfinite(_state(kv, 0, 1)).all()
        if rescale == 1.0:
            assert np.isinf(L.widen(want, kind)).sum() == 1, "the +inf case is missing"
        else:
            assert (L.widen(want, kind) != 0).all() and (np.abs(L.widen(want, kind)) < (6.2e-5 if kind == 1 else
                                                                                        1.2e-38)).any()


# ---------------------------------------------------------------------------
# lifecycle on 16-bit Adam / AdamW keys
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("optkey", ["adam", "adamw"])
def test_cached_plan_replays(optkey):
    kind = 2
    sizes = [8, 1000, 4096 + 4, 20011]
    rng = np.random.default_rng(31)
    keys = list(range(len(sizes)))
    w0 = [L.to_lp(rng.uniform(-1, 1, e).astype(np.float32), kind) for e in sizes]
    kv, lo = _store(OPTS[optkey][0], dict(OPTS[optkey][1], multi_precision=True), kind, keys, w0)
    gdev = [[mx.nd.empty((e,), mx.gpu(0), dtype="bfloat16") for _ in range(2)] for e in sizes]
    outs = [mx.nd.empty((e,), mx.gpu(0), dtype="bfloat16") for e in sizes]

    def step():
        g = [[L.to_lp(rng.uniform(-1, 1, e).astype(np.float32), kind) for _ in range(2)] for e in sizes]
        for gd, gs in zip(gdev, g):
            for d, x in zip(gd, gs):
                d[:] = _nd(x, kind)
        kv.pushpull(keys, gdev, out=outs)
        for k in keys:
            assert_bits_equal(_get(outs[k], kind), lo.update(k, _gsum(g[k], kind)), "%s replay key %d" % (optkey, k))

    h0 = kv.plan_hits()
    for _ in range(6):
        step()
    assert kv.plan_hits() - h0 == 4, kv.plan_hits() - h0
    h1 = kv.plan_hits()
    kv._optimizer.set_learning_rate(kv._optimizer.learning_rate * 0.5)
    lo.lr *= 0.5
    step()
    assert kv.plan_hits() == h1 + 1
    for k in keys:
        _check_state(kv, lo, k, optkey, "after replays key %d" % k)


@pytest.mark.parametrize("lp", ["float16", "bfloat16"])
@pytest.mark.parametrize("optkey", ["adam", "adamw"])
def test_save_load_continues_bit_exact(optkey, lp):
    kind = KIND[lp]
    sizes = [7, 4099, 20011]
    keys = list(range(len(sizes)))
    rng = np.random.default_rng(8)
    w0 = [L.to_lp(rng.uniform(-1, 1, e).astype(np.float32), kind) for e in sizes]
    kw = dict(OPTS[optkey][1], multi_precision=optkey == "adam")
    kv, lo = _store(OPTS[optkey][0], kw, kind, keys, w0)
    outs = [mx.nd.empty((e,), mx.gpu(0), dtype=DT[kind]) for e in sizes]

    def step(store, tag):
        g = [[L.to_lp(rng.uniform(-1, 1, e).astype(np.float32), kind) for _ in range(2)] for e in sizes]
        store.pushpull(keys, [[_nd(x, kind) for x in gs] for gs in g], out=outs)
        for k in keys:
            assert_bits_equal(_get(outs[k], kind), lo.update(k, _gsum(g[k], kind)), "%s key %d" % (tag, k))

    for _ in range(2):
        step(kv, "before")
    d = tempfile.mkdtemp(prefix="mxkv_lp_")
    f = os.path.join(d, "states")
    kv.save_optimizer_states(f, dump_optimizer=True)
    kv2 = mx.kv.create("device")
    kv2.init(keys, [_nd(_get(o, kind), kind) for o in outs])
    kv2.set_optimizer(mx.optimizer.create(OPTS[optkey][0], **kw))
    kv2.load_optimizer_states(f)
    os.remove(f)
    os.rmdir(d)
    for k in keys:
        _check_state(kv2, lo, k, optkey, "reloaded key %d" % k)      # the master round-trips
    for _ in range(2):
        step(kv2, "after reload")


@pytest.mark.parametrize("lp", ["float16", "bfloat16"])
@pytest.mark.parametrize("optkey", ["adam", "adamw"])
def test_native_updater(optkey, lp):
    """mx.optimizer.get_updater on 16-bit weights: in place, one launch for the whole list"""
    kind = KIND[lp]
    shapes = [(64,), (3, 5), (1000,), (257, 33), (7,)]
    rng = np.random.default_rng(5)
    w0 = [L.to_lp(rng.uniform(-1, 1, s).astype(np.float32).reshape(-1), kind) for s in shapes]
    weights = [_nd(w, kind).reshape(s) for w, s in zip(w0, shapes)]
    kw = dict(OPTS[optkey][1], clip_gradient=0.3, multi_precision=optkey == "adam")
    upd = mx.optimizer.get_updater(mx.optimizer.create(OPTS[optkey][0], **kw))
    assert isinstance(upd, mx.optimizer.NativeUpdater)
    lo = L.LpOracle(OPTS[optkey][0], kind, **kw)
    idx = list(range(len(shapes)))
    for i in idx:
        lo.init(i, w0[i])
    for step in range(3):
        g = [L.to_lp(rng.uniform(-1, 1, s).astype(np.float32).reshape(-1), kind) for s in shapes]
        gnd = [_nd(x, kind).reshape(s) for x, s in zip(g, shapes)]
        mx.nd.waitall()
        before = mx.kv.launch_count()
        upd(idx, gnd, weights)
        # (the first call also widens every 16-bit weight into its new fp32 master: one launch per tensor)
        assert mx.kv.launch_count() - before == (1 + len(shapes) if step == 0 else 1), \
            "one launch for the whole parameter list"
        for i in idx:
            assert_bits_equal(_get(weights[i], kind), lo.update(i, L.widen(g[i], kind)),
                              "updater step %d index %d" % (step, i))


def test_trainer_bf16_multi_precision_adam():
    """the benchmark's shape: Trainer(params, 'adam', {'multi_precision': True, 'wd': 0.01}) over a bf16 model,
    rescale_grad = 1 / batch"""
    import torch
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(64, 256), torch.nn.GELU(), torch.nn.Linear(256, 10)).cuda()
    model = model.to(torch.bfloat16)
    params = list(model.parameters())
    trainer = mx.Trainer(params, "adam", {"multi_precision": True, "wd": 0.01}, kvstore="device")
    B = 32
    lo = L.LpOracle("adam", 2, wd=0.01, rescale_grad=1.0 / B, multi_precision=True)
    bits = lambda t: t.detach().contiguous().view(torch.int16).cpu().numpy().view(np.uint16).reshape(-1)  # noqa
    for i, p in enumerate(params):
        lo.init(i, bits(p))
    for step in range(3):
        x = torch.randn(B, 64, device="cuda", dtype=torch.bfloat16)
        model.zero_grad(set_to_none=False)
        model(x).float().square().mean().backward()
        grads = [bits(p.grad) for p in params]
        trainer.step(B)
        torch.cuda.synchronize()
        for i, p in enumerate(params):
            assert_bits_equal(bits(p), lo.update(i, L.widen(grads[i], 2)), "trainer step %d param %d" % (step, i))


# ---------------------------------------------------------------------------
# one step against float64
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("lp", ["float32", "float16", "bfloat16"])
@pytest.mark.parametrize("optkey", list(OPTS))
def test_one_step_against_float64(optkey, lp):
    """the device's fp32 master after one step, from the master / state / gradient sum read back before it,
    within half an ulp plus L.ROUNDINGS roundings of the step's terms of the float64 operator"""
    kind = KIND.get(lp, 0)
    sizes = [4099, 20011]
    kw_extra = dict(clip_gradient=0.4) if optkey in ("adam", "adamw", "sgd_mom") else None
    kv, lo, _, _ = _run(optkey, kind, True, sizes=sizes, steps=2, kw_extra=kw_extra, seed=44)
    rng = np.random.default_rng(45)
    keys = [0, 1]
    # (multi_precision=True: a float32 key keeps a master too, equal to its weight)
    before = {k: (_state(kv, k, 1), _state(kv, k, 2), _state(kv, k, 3)) for k in keys}
    g = [[L.to_lp(rng.uniform(-1, 1, e).astype(np.float32), kind) for _ in range(3)] for e in sizes]
    outs = [mx.nd.empty((e,), mx.gpu(0), dtype=DT.get(kind, np.float32)) for e in sizes]
    hyper = {k: lo.hyper(k) for k in keys}
    kv.pushpull(keys, [[_nd(x, kind) for x in gs] for gs in g], out=outs)
    for k in keys:
        w, s0, s1 = before[k]
        zero = np.zeros_like(w)
        want, m, v, mag = L.step_f64(hyper[k], w, _gsum(g[k], kind), zero if s0 is None else s0,
                                     zero if s1 is None else s1)
        got = _state(kv, k, 1)
        L.assert_close_f64(got, want, mag, "%s %s key %d" % (optkey, lp, k))
        assert not np.array_equal(got, w), "the step changed nothing"


# ---------------------------------------------------------------------------
# float32 keys of an optimizer created with multi_precision: the MP instantiations of both dense kernels
# ---------------------------------------------------------------------------
class _forced(object):
    """force one dense kernel variant; restores the automatic choice"""

    def __init__(self, variant):
        self.variant = variant

    def __enter__(self):
        mx.kv.set_tuning(bulk={"bulk": 2, "per_thread": 0}[self.variant])
        self.before = {v: mx.kv.launch_count(v) for v in ("per_thread", "bulk")}
        return self

    def launched(self, v):
        return mx.kv.launch_count(v) - self.before[v]

    def __exit__(self, *a):
        mx.kv.set_tuning(bulk=1)


@pytest.mark.parametrize("optkey", ["sgd_mom", "adam", "adamw", "nag"])
@pytest.mark.parametrize("variant", ["bulk", "per_thread"])
def test_float32_multi_precision_keys(variant, optkey):
    """a float32 key with multi_precision keeps an fp32 master next to its weight (kv_dense_bulk_kernel<..., true>,
    kv_dense_kernel<float, ..., true>): every step is bit-exact against the oracle and bit-identical to
    multi_precision=False, and the stored master equals the weight"""
    sizes = [4, 2052, 8196, 3 * 2048 + 12, 100004]
    got = {}
    for mp in (False, True):
        with _forced(variant) as f:
            kv, lo, _, outs = _run(optkey, 0, mp, sizes=sizes, n=2, steps=3, seed=7)
            mx.nd.waitall()
            other = "per_thread" if variant == "bulk" else "bulk"
            assert f.launched(variant) >= 3, "the %s kernel did not run" % variant
            assert f.launched(other) == 0, "the %s kernel ran under a forced %s" % (other, variant)
        got[mp] = [_get(o, 0) for o in outs]
        if mp:
            for k, o in enumerate(got[mp]):
                assert_bits_equal(_state(kv, k, 1), o, "%s master of key %d" % (variant, k))
    for k in range(len(sizes)):
        assert_bits_equal(got[True][k], got[False][k], "%s %s key %d: multi_precision changed a float32 key" % (
            variant, optkey, k))


# ---------------------------------------------------------------------------
# several GPUs: two-shot keys with sharded master and state, and a checkpoint in between
# ---------------------------------------------------------------------------
@pytest.mark.multigpu
@pytest.mark.parametrize("optkey,lp", [("adamw", "bfloat16"), ("adam", "float16")])
def test_multi_gpu_sharded_master_and_state_with_a_checkpoint(optkey, lp):
    n = min(mx.num_gpus(), 8)
    kind = KIND[lp]
    sizes = [1001, 70001, (1 << 20) + 12, (1 << 21) + 6]
    keys = list(range(len(sizes)))
    rng = np.random.default_rng(40 + n)
    w0 = [L.to_lp(rng.uniform(-1, 1, e).astype(np.float32), kind) for e in sizes]
    kw = dict(OPTS[optkey][1], rescale_grad=0.25, clip_gradient=0.3, multi_precision=True)
    kv, lo = _store(OPTS[optkey][0], kw, kind, keys, w0)
    outs = [[mx.nd.empty((e,), mx.gpu(d), dtype=DT[kind]) for d in range(n)] for e in sizes]

    def step(store, tag):
        g = [[L.to_lp(rng.uniform(-1, 1, e).astype(np.float32), kind) for _ in range(n)] for e in sizes]
        store.pushpull(keys, [[_nd(x, kind, mx.gpu(d)) for d, x in enumerate(gs)] for gs in g], out=outs)
        for k in keys:
            want = lo.update(k, _gsum(g[k], kind))
            for d in range(n):
                assert_bits_equal(_get(outs[k][d], kind), want, "%s n=%d key %d gpu %d" % (tag, n, k, d))

    for _ in range(2):
        step(kv, "before")
    d = tempfile.mkdtemp(prefix="mxkv_lp_")
    f = os.path.join(d, "states")
    kv.save_optimizer_states(f, dump_optimizer=True)
    kv2 = mx.kv.create("device")
    kv2.init(keys, [_nd(_get(outs[k][0], kind), kind) for k in keys])
    kv2.set_optimizer(mx.optimizer.create(OPTS[optkey][0], **kw))
    kv2.load_optimizer_states(f)
    os.remove(f)
    os.rmdir(d)
    for _ in range(2):
        step(kv2, "after reload")
    for k in keys:
        _check_state(kv2, lo, k, optkey, "gathered key %d" % k)
