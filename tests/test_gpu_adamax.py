"""The Adamax optimizer (python/mxnet/optimizer/adamax.py) fused into the gradient exchange and the native updater:
``Adamax.step`` restated in the kernel, against the CPU oracle, bit for bit unless stated, on every dense kernel variant
that serves it.  Its learning rate carries 1 / (1 - beta1^t), so every comparison runs over several steps.

The suite is written once for both kinds that restate a Python ``step`` (Adamax here, AdaDelta in
tests/test_gpu_adadelta.py, which imports these tests and overrides the ``spec`` fixture)."""
import ctypes
import os
import pickle
import sys
import tempfile

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import mxnet_b200 as mx
from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import adamax_oracle as A  # noqa: E402

_SIM = bool(os.environ.get("MXKV_SIM"))
# the bench sweep: 9 float32 keys 2^10 ... 2^26 (the simulator runs on one CPU core: up to 2^18)
SWEEP = [1 << p for p in (range(10, 19, 2) if _SIM else range(10, 27, 2))]


class Spec(object):
    """one optimizer kind under test: its class, oracle, and the options each test runs"""

    def __init__(self, name, cls, oracle, kw, base, variants, lp_kw, updater_kw, python_kw, multi_kw):
        self.name, self.cls, self.oracle = name, cls, oracle
        self.kw, self.base, self.variants = kw, base, variants
        self.lp_kw, self.updater_kw, self.python_kw, self.multi_kw = lp_kw, updater_kw, python_kw, multi_kw


ADAMAX = Spec(
    "adamax", mx.optimizer.Adamax, A.OracleAdamax,
    kw=dict(learning_rate=0.002, wd=1e-4),
    base=dict(learning_rate=0.002, wd=0.05),
    # clip_gradient 0 is on (step clips at 0): with wd > 0 the weight decay alone drives the update
    variants=[dict(rescale_grad=0.14), dict(clip_gradient=0.3), dict(clip_gradient=0.0), dict(learning_rate=0.01),
              dict(beta1=0.5), dict(beta2=0.8), dict(epsilon=1e-2), dict(wd=0.0)],
    lp_kw=dict(learning_rate=0.002, wd=1e-3, rescale_grad=0.5, clip_gradient=0.6, beta1=0.5),
    updater_kw=dict(learning_rate=0.002, wd=1e-2, clip_gradient=0.3, beta1=0.5, beta2=0.9),
    python_kw=dict(learning_rate=0.002, wd=1e-3, clip_gradient=0.01, beta1=0.5),
    multi_kw=dict(learning_rate=0.002, wd=1e-4, rescale_grad=0.5, clip_gradient=0.7, beta1=0.5))


@pytest.fixture
def spec():
    return ADAMAX


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32}[a.dtype.itemsize])


def assert_bits_equal(a, b, msg=""):
    assert a.shape == b.shape, (a.shape, b.shape, msg)
    ne = _bits(a) != _bits(b)
    assert not ne.any(), "%s: %d / %d elements differ" % (msg, ne.sum(), ne.size)


def _fill(rng, lo, hi, e):
    if e <= (1 << 20):
        return rng.uniform(lo, hi, e).astype(np.float32)
    return np.resize(rng.uniform(lo, hi, 1000003).astype(np.float32), e)


class _forced(object):
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


def _stores(spec, keys, w0, opt_kw, kvtype="device"):
    kv = mx.kv.create(kvtype)
    kv.init(keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
    kv.set_optimizer(spec.cls(**opt_kw))
    okv = O.OracleKVStore(kvtype)
    okv.init(keys, [w.copy() for w in w0])
    okv.set_optimizer(spec.oracle(**opt_kw))
    return kv, okv


def _check(okv, keys, outs, msg):
    for k, o in zip(keys, outs):
        want = np.empty(o.shape, np.float32)
        okv.pull(k, want)
        assert_bits_equal(o.asnumpy(), want, "%s key %s" % (msg, k))


def _state(kv, key, which):
    h = kv._state_handle(key, which)
    return None if h is None else h.asnumpy().reshape(-1)


def _check_states(kv, okv, keys, msg):
    """GetState(2 / 3) is state0 / state1; there is no state2"""
    for k in keys:
        for i, want in enumerate(okv.optimizer.states[k]):
            assert_bits_equal(_state(kv, k, 2 + i), want.reshape(-1), "%s key %s state%d" % (msg, k, i))
        assert _state(kv, k, 4) is None, "%s key %s has a third state" % (msg, k)


def _count(kv, key):
    from mxnet_b200.base import _LIB, check_call
    n = ctypes.c_int64()
    check_call(_LIB.MXKVB200GetUpdateCount(kv.handle, int(key), None, ctypes.byref(n)))
    return n.value


@pytest.mark.parametrize("n", [1, 2, 4])
@pytest.mark.parametrize("variant", ["bulk", "per_thread"])
def test_forced_variant_whole_sweep_key_set(spec, variant, n):
    """the sweep key set in one pushpull, several steps (t = 1, 2, 3), with each dense kernel variant forced and the
    launch counters proving which one ran"""
    rng = np.random.default_rng(20 + n)
    keys = list(range(len(SWEEP)))
    w0 = [_fill(rng, 0, 1, e) for e in SWEEP]
    with _forced(variant) as f:
        kv, okv = _stores(spec, keys, w0, spec.kw)
        outs = [mx.nd.empty((e,), mx.gpu(0)) for e in SWEEP]
        gdev = [[mx.nd.empty((e,), mx.gpu(0)) for _ in range(n)] for e in SWEEP]
        for s in range(3):
            if s < 2:     # the third step pushes the same gradients again (t and the states have moved on)
                grads = [[_fill(rng, -1, 1, e) for _ in range(n)] for e in SWEEP]
                for gd, gs in zip(gdev, grads):
                    for d, g in zip(gd, gs):
                        d[:] = g
            kv.pushpull(keys, gdev, out=outs)
            okv.push(keys, grads)
            _check(okv, keys, outs, "%s n=%d step %d" % (variant, n, s))
        _check_states(kv, okv, keys, "%s n=%d" % (variant, n))
        mx.nd.waitall()
        other = "per_thread" if variant == "bulk" else "bulk"
        assert f.launched(variant) >= 3, "the %s kernel did not run" % variant
        assert f.launched(other) == 0, "the %s kernel ran under a forced %s" % (other, variant)


def test_ragged_sizes_and_hyper_parameters_take_effect(spec):
    """sizes off every vector / tile boundary; lr_mult / wd_mult per key and every option: the result matches the
    oracle bit for bit AND differs from the run without the option.  clip_gradient 0 is on, as `step` clips at 0; a
    negative clip_gradient is off and leaves the result of the run without it"""
    sizes = [1, 7, 1000, 4099, 8196, 100003]
    keys = list(range(len(sizes)))
    same = [dict(clip_gradient=-1.0)]
    finals = []
    for extra in [dict()] + spec.variants + same + ["mult"]:
        rng = np.random.default_rng(3)
        w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in sizes]
        kw = dict(spec.base, **(extra if extra != "mult" else {}))
        kv = mx.kv.create("device")
        kv.init(keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
        opt = spec.cls(**kw)
        oopt = spec.oracle(**kw)
        if extra == "mult":
            opt.set_lr_mult({1: 0.5, 3: 2.0})
            opt.set_wd_mult({2: 0.0, 3: 3.0})
            oopt.lr_mult, oopt.wd_mult = {1: 0.5, 3: 2.0}, {2: 0.0, 3: 3.0}
        kv.set_optimizer(opt)
        okv = O.OracleKVStore("device")
        okv.init(keys, [w.copy() for w in w0])
        okv.set_optimizer(oopt)
        outs = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]
        for s in range(3):
            grads = [[rng.uniform(-0.5, 0.5, e).astype(np.float32) for _ in range(3)] for e in sizes]
            kv.pushpull(keys, [[mx.nd.array(g, mx.gpu(0)) for g in gs] for gs in grads], out=outs)
            okv.push(keys, grads)
            _check(okv, keys, outs, "%r step %d" % (extra, s))
        _check_states(kv, okv, keys, repr(extra))
        finals.append([o.asnumpy() for o in outs])
    nv = 1 + len(spec.variants)
    for i, extra in enumerate(spec.variants, 1):
        for k in range(2, len(sizes)):
            assert not np.array_equal(finals[i][k], finals[0][k]), ("option had no effect", extra, k)
    for i, extra in enumerate(same, nv):
        for k in range(len(sizes)):
            assert_bits_equal(finals[i][k], finals[0][k], "%r is not off" % (extra,))
    for k in (1, 3):
        assert not np.array_equal(finals[-1][k], finals[0][k]), ("multiplier had no effect", k)


def test_engine_defaults_for_a_c_caller(spec):
    """A C caller naming the optimizer alone gets the class defaults (Adamax: learning_rate 0.002, beta1 0.9, beta2
    0.999, epsilon 1e-8; AdaDelta: learning_rate 1.0, rho 0.9, epsilon 1e-6), no clip"""
    from mxnet_b200.base import _LIB, check_call
    E = 5003
    rng = np.random.default_rng(4)
    w0 = rng.uniform(0, 1, E).astype(np.float32)
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w0, mx.gpu(0)))
    check_call(_LIB.MXKVB200SetOptimizer(kv.handle, spec.name.encode(), 0, None, None))
    oopt = spec.oracle()
    ow = w0.copy()
    out = mx.nd.empty((E,), mx.gpu(0))
    for s in range(3):
        grads = [rng.uniform(-1, 1, E).astype(np.float32) for _ in range(2)]
        kv.pushpull(0, [mx.nd.array(g, mx.gpu(0)) for g in grads], out=out)
        oopt.update(0, ow, O.sum_device(grads))
        assert_bits_equal(out.asnumpy(), ow, "C defaults step %d" % s)


@pytest.mark.parametrize("mp", [False, True])
@pytest.mark.parametrize("lp", ["bfloat16", np.float16])
def test_low_precision_keys(spec, lp, mp):
    """float16 / bfloat16 weights and gradients: the update on the fp32 master, the stored weight its one rounding --
    for float16 with multi_precision that is update_multi_precision's float32 step on the master; the other keys
    follow the engine's rule of an fp32 master for every 16-bit key, so multi_precision does not change the result"""
    kind = 2 if lp == "bfloat16" else 1
    E, n = 50003, 3
    rng = np.random.default_rng(99 + mp)
    w0 = rng.uniform(0, 1, E).astype(np.float32)
    w0_lp = O.f32_to_bf16(w0) if kind == 2 else w0.astype(np.float16)
    w32 = O.bf16_to_f32(w0_lp) if kind == 2 else w0_lp.astype(np.float32)
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w0_lp, mx.gpu(0), dtype=lp))
    kv.set_optimizer(spec.cls(multi_precision=mp, **spec.lp_kw))
    oopt = spec.oracle(**spec.lp_kw)
    out = mx.nd.empty((E,), mx.gpu(0), dtype=lp)
    want_lp = np.zeros(E, np.uint16)
    for s in range(3):
        g = [rng.uniform(-1, 1, E).astype(np.float32) for _ in range(n)]
        g_lp = [O.f32_to_bf16(x) if kind == 2 else x.astype(np.float16) for x in g]
        kv.pushpull(0, [mx.nd.array(x, mx.gpu(0), dtype=lp) for x in g_lp], out=out)
        oopt.update_lp(0, want_lp, kind, w32, O.sum_device_lp_f32out(g_lp, kind))
        got = out.asnumpy(raw=True) if kind == 2 else out.asnumpy().view(np.uint16)
        assert_bits_equal(got, want_lp, "%s mp=%s step %d" % (lp, mp, s))
        assert_bits_equal(_state(kv, 0, 1), w32, "%s mp=%s master step %d" % (lp, mp, s))
        for i, st in enumerate(oopt.states[0]):
            assert_bits_equal(_state(kv, 0, 2 + i), st, "%s mp=%s state%d step %d" % (lp, mp, i, s))


def test_unaligned_view_takes_the_scalar_path(spec):
    """bfloat16 torch views offset by one element (2-byte aligned only): the scalar path of the per-thread kernel with
    both state arrays"""
    import torch
    E, n, kind = 10001, 3, 2
    rng = np.random.default_rng(12)
    w0 = O.f32_to_bf16(rng.uniform(-1, 1, E).astype(np.float32))
    w32 = O.bf16_to_f32(w0)
    wbase = torch.zeros(E + 3, dtype=torch.bfloat16, device="cuda")
    wview = wbase[1:E + 1]
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w0, mx.gpu(0), dtype="bfloat16"))
    kv.set_optimizer(spec.cls(**spec.kw))
    oopt = spec.oracle(**spec.kw)
    want = np.zeros(E, np.uint16)
    for s in range(3):
        g = [O.f32_to_bf16(rng.uniform(-1, 1, E).astype(np.float32)) for _ in range(n)]
        gbase = [torch.zeros(E + 3, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
        for b, x in zip(gbase, g):
            b[1:E + 1].copy_(torch.from_numpy(x.view(np.int16)).view(torch.bfloat16))
        torch.cuda.synchronize()
        kv.pushpull(0, [mx.nd.from_torch(b[1:E + 1]) for b in gbase], out=mx.nd.from_torch(wview))
        mx.nd.waitall()
        oopt.update_lp(0, want, kind, w32, O.sum_device_lp_f32out(g, kind))
        got = wview.view(torch.int16).cpu().numpy().view(np.uint16)
        assert_bits_equal(got, want, "unaligned view step %d" % s)


def test_cached_launch_plan_replays_with_the_update_count_of_each_step(spec):
    """identical calls replay a recorded launch plan; Adamax's learning rate depends on t, so every replayed step must
    carry that step's lr / (1 - beta1^t).  A learning-rate change is patched in"""
    sizes = [8, 1000, 4096 + 4, 70001, 1 << 18]
    rng = np.random.default_rng(31)
    keys = list(range(len(sizes)))
    w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in sizes]
    kv, okv = _stores(spec, keys, w0, spec.kw)
    gdev = [[mx.nd.empty((e,), mx.gpu(0)) for _ in range(2)] for e in sizes]
    outs = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]

    def step():
        grads = [[rng.uniform(-1, 1, e).astype(np.float32) for _ in range(2)] for e in sizes]
        for gd, gs in zip(gdev, grads):
            for d, g in zip(gd, gs):
                d[:] = g
        kv.pushpull(keys, gdev, out=outs)
        okv.push(keys, grads)
        _check(okv, keys, outs, "replay t=%d" % okv.optimizer.count[0])

    h0 = kv.plan_hits()
    for _ in range(6):
        step()
    assert kv.plan_hits() - h0 == 4, kv.plan_hits() - h0
    h1 = kv.plan_hits()
    kv._optimizer.set_learning_rate(kv._optimizer.learning_rate * 0.5)
    okv.optimizer.lr = okv.optimizer.lr * 0.5
    step()
    assert kv.plan_hits() == h1 + 1
    _check_states(kv, okv, keys, "after replays")
    assert all(_count(kv, k) == 7 for k in keys)


def test_deferred_queue_merges_per_key_calls_into_one_launch(spec):
    """MXKVB200SetDeferred: per-key pushpulls with priorities are issued at the flush point as one launch; every key
    carries its own update count's scalars, bit for bit against the oracle over three steps"""
    sizes = [5, 1000, 4099, 1 << 14, 33, 70001]
    keys = list(range(len(sizes)))
    rng = np.random.default_rng(77)
    w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in sizes]
    kv, okv = _stores(spec, keys, w0, spec.kw)
    kv.set_deferred(True)
    outs = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]
    for s in range(3):
        grads = [rng.uniform(-1, 1, e).astype(np.float32) for e in sizes]
        gdev = [mx.nd.array(g, mx.gpu(0)) for g in grads]
        l0 = mx.kv.launch_count()
        for i in keys:
            kv.pushpull(i, gdev[i], out=outs[i], priority=-i)
        assert mx.kv.launch_count() == l0, "deferred calls must not launch before the flush point"
        okv.push(keys, [[g] for g in grads])
        _check(okv, keys, outs, "deferred step %d" % s)        # reading an array is a flush point
        assert mx.kv.launch_count() - l0 == 1
    assert kv.deferred_batches() == 3
    _check_states(kv, okv, keys, "deferred")


def test_save_load_round_trip_continues_bit_exact(spec):
    """save / load of the fused states (state0 / state1) and of the update counts: the reloaded store continues bit
    for bit at t = 3, 4"""
    sizes = [1000, 70001, (1 << 20) + 4]
    rng = np.random.default_rng(8)
    keys = list(range(len(sizes)))
    w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in sizes]
    kv, okv = _stores(spec, keys, w0, spec.kw)
    outs = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]
    for _ in range(2):
        grads = [[rng.uniform(-1, 1, e).astype(np.float32) for _ in range(2)] for e in sizes]
        kv.pushpull(keys, [[mx.nd.array(g, mx.gpu(0)) for g in gs] for gs in grads], out=outs)
        okv.push(keys, grads)
    d = tempfile.mkdtemp(prefix="mxkv_%s_" % spec.name)
    f = os.path.join(d, "states")
    kv.save_optimizer_states(f, dump_optimizer=True)
    with open(f, "rb") as fin:
        payload = pickle.load(fin)
    assert payload["format"] == "mxkv_b200_fused_v1"
    for k in keys:
        ent = payload["states"][k]
        assert ent["count"] == 2
        for i, name in enumerate(["state0", "state1"]):
            assert_bits_equal(ent[name].reshape(-1), okv.optimizer.states[k][i].reshape(-1), name)
        assert "state2" not in ent or ent["state2"] is None
    kv2 = mx.kv.create("device")
    kv2.init(keys, [mx.nd.array(o.asnumpy(), mx.gpu(0)) for o in outs])
    kv2.set_optimizer(spec.cls(**spec.kw))
    kv2.load_optimizer_states(f)
    os.remove(f)
    os.rmdir(d)
    assert all(_count(kv2, k) == 2 for k in keys)
    outs2 = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]
    for s in range(2):
        grads = [[rng.uniform(-1, 1, e).astype(np.float32) for _ in range(2)] for e in sizes]
        kv2.pushpull(keys, [[mx.nd.array(g, mx.gpu(0)) for g in gs] for gs in grads], out=outs2)
        okv.push(keys, grads)
        _check(okv, keys, outs2, "after reload step %d" % s)
    assert all(_count(kv2, k) == 4 for k in keys)
    _check_states(kv2, okv, keys, "after reload")


def test_get_state_and_set_state(spec):
    """MXKVB200SetState(2 / 3) replaces state0 / state1; the next step starts from them"""
    from mxnet_b200.base import _LIB, check_call
    E = 4099
    rng = np.random.default_rng(21)
    w0 = rng.uniform(0, 1, E).astype(np.float32)
    kv, okv = _stores(spec, [0], [w0], spec.kw)
    out = mx.nd.empty((E,), mx.gpu(0))
    g = rng.uniform(-1, 1, E).astype(np.float32)
    kv.pushpull(0, mx.nd.array(g, mx.gpu(0)), out=out)
    okv.push([0], [[g]])
    new = tuple(rng.uniform(0.1, 0.5, E).astype(np.float32) for _ in range(2))
    for which, s in zip((2, 3), new):
        v = mx.nd.array(s, mx.gpu(0))          # held: the handle is freed with the array
        check_call(_LIB.MXKVB200SetState(kv.handle, 0, None, which, v.handle))
    okv.optimizer.states[0] = tuple(s.copy() for s in new)
    for which, s in zip((2, 3), new):
        assert_bits_equal(_state(kv, 0, which), s, "state %d" % which)
    g = rng.uniform(-1, 1, E).astype(np.float32)
    kv.pushpull(0, mx.nd.array(g, mx.gpu(0)), out=out)
    okv.push([0], [[g]])
    _check(okv, [0], [out], "after SetState")
    _check_states(kv, okv, [0], "after SetState")


def test_native_updater(spec):
    shapes = [(64,), (3, 5), (1000,), (257, 33), (7,)]
    rng = np.random.default_rng(5)
    w0 = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
    weights = [mx.nd.array(w, mx.gpu(0)) for w in w0]
    upd = mx.optimizer.get_updater(mx.optimizer.create(spec.name, **spec.updater_kw))
    assert isinstance(upd, mx.optimizer.NativeUpdater)
    oopt = spec.oracle(**spec.updater_kw)
    ow = [w.copy() for w in w0]
    idx = list(range(len(shapes)))
    for step in range(3):
        g = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
        before = mx.kv.launch_count()
        upd(idx, [mx.nd.array(x, mx.gpu(0)) for x in g], weights)
        assert mx.kv.launch_count() - before == 1, "one launch for the whole parameter list"
        for k in idx:
            oopt.update(k, ow[k], g[k].copy())
            assert_bits_equal(weights[k].asnumpy(), ow[k], "updater step %d index %d" % (step, k))


def test_row_sparse_gradient_is_refused(spec):
    rows, L = 100, 8
    kv = mx.kv.create("device")
    kv.init("w", mx.nd.array(np.zeros((rows, L), np.float32), mx.gpu(0)))
    kv.set_optimizer(spec.cls(learning_rate=0.1))
    idx = np.array([1, 5, 7], np.int64)
    vals = np.ones((3, L), np.float32)
    with pytest.raises(mx.MXNetError, match="only the lazy SGD / SGD-momentum / Adam updates are fused"):
        kv.push("w", mx.nd.row_sparse_array((vals, idx), shape=(rows, L), ctx=mx.gpu(0)))
        mx.nd.waitall()


# ---------------------------------------------------------------------------
# Trainer over torch parameters
# ---------------------------------------------------------------------------
def _net(seed=0):
    import torch
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(64, 256), torch.nn.ReLU(), torch.nn.Linear(256, 256),
                               torch.nn.ReLU(), torch.nn.Linear(256, 10)).cuda()


def _bits_equal32(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32),
                          np.ascontiguousarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("mode", ["update_on_kvstore", "local_update", "no_kvstore", "overlap"])
def test_trainer_modes_match_the_oracle(spec, mode):
    import torch
    model = _net()
    params = list(model.parameters())
    kw = dict(spec.kw)
    targs = {"update_on_kvstore": dict(kvstore="device", update_on_kvstore=True),
             "local_update": dict(kvstore="device", update_on_kvstore=False),
             "no_kvstore": dict(kvstore=None),
             "overlap": dict(kvstore="device", overlap=True, bucket_bytes=64 << 10)}[mode]
    trainer = mx.Trainer(params, spec.name, dict(kw), **targs)
    ref_w = [p.detach().cpu().numpy().copy().reshape(-1) for p in params]
    opt = spec.oracle(**kw)
    torch.manual_seed(9)
    for step in range(3):
        x = torch.randn(32, 64, device="cuda")
        model.zero_grad(set_to_none=False)
        if mode == "overlap" and step > 0:
            trainer.arm(32)
        model(x).square().mean().backward()
        grads = [p.grad.detach().cpu().numpy().copy().reshape(-1) for p in params]
        trainer.step(32)
        torch.cuda.synchronize()
        opt.rescale_grad = 1.0 / 32
        for i, (w, g) in enumerate(zip(ref_w, grads)):
            opt.update(i, w, g)
        for i, (p, w) in enumerate(zip(params, ref_w)):
            assert _bits_equal32(p.detach().cpu().numpy().reshape(-1), w), (mode, step, i)


def test_fused_and_python_step_agree(spec):
    """use_fused_step=False runs the torch restatement of the reference's step through the Python updater; it agrees
    with the fused kernel within float32 tolerance"""
    import torch
    ma, mb = _net(1), _net(1)
    kw = spec.python_kw
    ta = mx.Trainer(list(ma.parameters()), spec.name, dict(kw), kvstore="device")
    tb = mx.Trainer(list(mb.parameters()), spec.name, dict(kw, use_fused_step=False), kvstore="device")
    assert mx.optimizer.fused_name_of(tb._optimizer) is None
    torch.manual_seed(2)
    for step in range(5):
        x = torch.randn(16, 64, device="cuda")
        for m, t in ((ma, ta), (mb, tb)):
            m.zero_grad(set_to_none=False)
            m(x).square().mean().backward()
            t.step(16)
        torch.cuda.synchronize()
        for pa, pb in zip(ma.parameters(), mb.parameters()):
            np.testing.assert_allclose(pb.detach().cpu().numpy(), pa.detach().cpu().numpy(), rtol=1e-5, atol=1e-6)


# ---------------------------------------------------------------------------
# several GPUs in one process
# ---------------------------------------------------------------------------
@pytest.mark.multigpu
def test_multi_gpu_one_and_two_shot_keys_with_a_checkpoint(spec):
    """one value per GPU, outputs on every GPU; the large keys are split into shards (two-shot) and so are their two
    states; a save / load round trip in between gathers and redistributes them and restores the update counts"""
    n = min(mx.num_gpus(), 8)
    shapes = [(1000,), (37, 13), (70001,), ((1 << 20) + 12,), (1 << 21,)]
    keys = list(range(len(shapes)))
    rng = np.random.default_rng(40 + n)
    w0 = [rng.uniform(0, 1, s).astype(np.float32) for s in shapes]
    kw = spec.multi_kw
    kv, okv = _stores(spec, keys, w0, kw)
    outs = [[mx.nd.empty(s, mx.gpu(d)) for d in range(n)] for s in shapes]

    def step(store):
        grads = [[rng.uniform(-1, 1, s).astype(np.float32) for _ in range(n)] for s in shapes]
        store.pushpull(keys, [[mx.nd.array(g, mx.gpu(d)) for d, g in enumerate(gs)] for gs in grads], out=outs)
        okv.push(keys, grads)
        for k, s in enumerate(shapes):
            want = np.empty(s, np.float32)
            okv.pull(k, want)
            for d in range(n):
                assert_bits_equal(outs[k][d].asnumpy(), want, "n=%d key %d gpu %d" % (n, k, d))
    for _ in range(2):
        step(kv)
    _check_states(kv, okv, keys, "gathered n=%d" % n)
    d = tempfile.mkdtemp(prefix="mxkv_%s_" % spec.name)
    f = os.path.join(d, "states")
    kv.save_optimizer_states(f, dump_optimizer=True)
    kv2 = mx.kv.create("device")
    kv2.init(keys, [mx.nd.array(outs[k][0].asnumpy(), mx.gpu(0)) for k in keys])
    kv2.set_optimizer(spec.cls(**kw))
    kv2.load_optimizer_states(f)
    os.remove(f)
    os.rmdir(d)
    for _ in range(2):
        step(kv2)


@pytest.mark.multigpu
@pytest.mark.parametrize("n", [3, 8])
def test_tree_sum_feeds_the_update(spec, monkeypatch, n):
    """MXNET_KVSTORE_USETREE=1: the update consumes the sum of the reference's tree order, bit for bit against
    oracle.tree_reduce followed by the oracle's step"""
    if mx.num_gpus() < n:
        pytest.skip("needs %d GPUs" % n)
    bound = 5000
    W = mx.topology.query_links(list(range(n)))
    topo, scan, depth = mx.topology.compute_trees(W, 0.7, False)
    tree = dict(topo=topo, scan=scan, depth=depth, bound=bound)
    monkeypatch.setenv("MXNET_KVSTORE_USETREE", "1")
    monkeypatch.setenv("MXNET_KVSTORE_TREE_ARRAY_BOUND", str(bound))
    shapes = [(1000,), (64, 33), (70001,), (300, 257)]
    keys = list(range(len(shapes)))
    rng = np.random.default_rng(n)
    w0 = [rng.uniform(0, 1, s).astype(np.float32) for s in shapes]
    kv = mx.kv.create("device")
    kv.init(keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
    kv.set_optimizer(spec.cls(**spec.kw))
    okv = O.OracleKVStore("device", tree=tree)
    okv.init(keys, [w.copy() for w in w0])
    okv.set_optimizer(spec.oracle(**spec.kw))
    outs = [[mx.nd.empty(s, mx.gpu(d)) for d in range(n)] for s in shapes]
    t0 = mx.kv.launch_count("tree")
    for _ in range(3):
        grads = [[rng.uniform(-1, 1, s).astype(np.float32) for _ in range(n)] for s in shapes]
        kv.pushpull(keys, [[mx.nd.array(g, mx.gpu(d)) for d, g in enumerate(gs)] for gs in grads], out=outs)
        okv.push(keys, grads)
    assert mx.kv.launch_count("tree") > t0, "the tree kernel did not run"
    for k, s in enumerate(shapes):
        want = np.empty(s, np.float32)
        okv.pull(k, want)
        for o in outs[k]:
            assert_bits_equal(o.asnumpy(), want, "tree n=%d key %d" % (n, k))
