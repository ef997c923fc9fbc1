"""The RMSProp optimizer (python/mxnet/optimizer/rmsprop.py), plain and centered, fused into the gradient exchange and the
native updater: rmsprop_update / rmspropalex_update (src/operator/optimizer_op-inl.h:1905-2031) against the CPU oracle,
bit for bit unless stated, on every dense kernel variant that serves it."""
import ctypes
import os
import sys
import tempfile

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import mxnet_b200 as mx
from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rmsprop_oracle as R  # noqa: E402

_SIM = bool(os.environ.get("MXKV_SIM"))
# the bench sweep: 9 float32 keys 2^10 ... 2^26 (the simulator runs on one CPU core: up to 2^18)
SWEEP = [1 << p for p in (range(10, 19, 2) if _SIM else range(10, 27, 2))]
KW = dict(learning_rate=0.01, wd=1e-4)
CENTERED = [False, True]


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


def _stores(keys, w0, opt_kw, kvtype="device"):
    kv = mx.kv.create(kvtype)
    kv.init(keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
    kv.set_optimizer(mx.optimizer.RMSProp(**opt_kw))
    okv = O.OracleKVStore(kvtype)
    okv.init(keys, [w.copy() for w in w0])
    okv.set_optimizer(R.OracleRMSProp(**opt_kw))
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
    for k in keys:
        for i, want in enumerate(okv.optimizer.states[k]):
            assert_bits_equal(_state(kv, k, 2 + i), want.reshape(-1), "%s key %s state%d" % (msg, k, i))


@pytest.mark.parametrize("centered", CENTERED)
@pytest.mark.parametrize("n", [1, 2, 4])
@pytest.mark.parametrize("variant", ["bulk", "per_thread"])
def test_forced_variant_whole_sweep_key_set(variant, n, centered):
    """the sweep key set in one pushpull, several steps, with each dense kernel variant forced and the launch counters
    proving which one ran"""
    rng = np.random.default_rng(20 + n)
    keys = list(range(len(SWEEP)))
    w0 = [_fill(rng, 0, 1, e) for e in SWEEP]
    with _forced(variant) as f:
        kv, okv = _stores(keys, w0, dict(KW, centered=centered))
        outs = [mx.nd.empty((e,), mx.gpu(0)) for e in SWEEP]
        gdev = [[mx.nd.empty((e,), mx.gpu(0)) for _ in range(n)] for e in SWEEP]
        for s in range(3):
            if s < 2:     # the third step pushes the same gradients again (the states have moved on)
                grads = [[_fill(rng, -1, 1, e) for _ in range(n)] for e in SWEEP]
                for gd, gs in zip(gdev, grads):
                    for d, g in zip(gd, gs):
                        d[:] = g
            kv.pushpull(keys, gdev, out=outs)
            okv.push(keys, grads)
            _check(okv, keys, outs, "%s n=%d centered=%s step %d" % (variant, n, centered, s))
        mx.nd.waitall()
        other = "per_thread" if variant == "bulk" else "bulk"
        assert f.launched(variant) >= 3, "the %s kernel did not run" % variant
        assert f.launched(other) == 0, "the %s kernel ran under a forced %s" % (other, variant)


@pytest.mark.parametrize("centered", CENTERED)
def test_ragged_sizes_and_hyper_parameters_take_effect(centered):
    """sizes off every vector / tile boundary; lr_mult / wd_mult per key, rescale_grad, a binding clip_gradient, a
    binding clip_weights, rho, momentum and epsilon: the result matches the oracle bit for bit AND differs from the
    run without the option.  clip_gradient = 0 and clip_weights = 0 are off (RMSProp.fused_step passes falsy clips
    to the operator as absent) and leave the result of the run without them"""
    sizes = [1, 7, 1000, 4099, 8196, 100003]
    keys = list(range(len(sizes)))
    base = dict(learning_rate=0.01, wd=0.05, centered=centered)
    variants = [dict(), dict(rescale_grad=0.14), dict(clip_gradient=0.3), dict(clip_weights=0.5), dict(rho=0.5),
                dict(epsilon=1e-3), dict(momentum=0.5) if centered else dict(rho=0.99)]
    same = [dict(clip_gradient=0.0), dict(clip_weights=0.0), dict(clip_gradient=-1.0, clip_weights=-2.0)]
    finals = []
    for extra in variants + same + ["mult"]:
        rng = np.random.default_rng(3)
        w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in sizes]
        kw = dict(base, **(extra if extra != "mult" else {}))
        kv = mx.kv.create("device")
        kv.init(keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
        opt = mx.optimizer.RMSProp(**kw)
        oopt = R.OracleRMSProp(**kw)
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
    nv = len(variants)
    for i, extra in enumerate(variants[1:], 1):
        for k in range(2, len(sizes)):
            assert not np.array_equal(finals[i][k], finals[0][k]), ("option had no effect", extra, k)
    for i, extra in enumerate(same, nv):
        for k in range(len(sizes)):
            assert_bits_equal(finals[i][k], finals[0][k], "%r is not off" % (extra,))
    for k in (1, 2, 3):
        assert not np.array_equal(finals[-1][k], finals[0][k]), ("multiplier had no effect", k)


@pytest.mark.parametrize("centered", CENTERED)
def test_engine_defaults_for_a_c_caller(centered):
    """A C caller naming "rmsprop" (with centered alone, or nothing) gets the class defaults (rmsprop.py:70-71):
    learning_rate 0.001, rho 0.9, momentum 0.9, epsilon 1e-8, both clips off"""
    from mxnet_b200.base import _LIB, check_call, c_str_array
    E = 5003
    rng = np.random.default_rng(4)
    w0 = rng.uniform(0, 1, E).astype(np.float32)
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w0, mx.gpu(0)))
    if centered:
        check_call(_LIB.MXKVB200SetOptimizer(kv.handle, b"rmsprop", 1, c_str_array(["centered"]),
                                             c_str_array(["True"])))
    else:
        check_call(_LIB.MXKVB200SetOptimizer(kv.handle, b"rmsprop", 0, None, None))
    oopt = R.OracleRMSProp(centered=centered)
    ow = w0.copy()
    out = mx.nd.empty((E,), mx.gpu(0))
    for s in range(3):
        grads = [rng.uniform(-1, 1, E).astype(np.float32) for _ in range(2)]
        kv.pushpull(0, [mx.nd.array(g, mx.gpu(0)) for g in grads], out=out)
        oopt.update(0, ow, O.sum_device(grads))
        assert_bits_equal(out.asnumpy(), ow, "C defaults step %d" % s)


@pytest.mark.parametrize("centered", CENTERED)
@pytest.mark.parametrize("mp", [False, True])
@pytest.mark.parametrize("lp", ["bfloat16", np.float16])
def test_low_precision_keys(lp, mp, centered):
    """float16 / bfloat16 weights and gradients: the update on the fp32 master, the stored weight its one rounding --
    for float16 with multi_precision that is update_multi_precision's float32 operator on the master; the other keys
    follow the engine's rule of an fp32 master for every 16-bit key, so multi_precision does not change the result"""
    kind = 2 if lp == "bfloat16" else 1
    E, n = 50003, 3
    rng = np.random.default_rng(99 + mp)
    w0 = rng.uniform(0, 1, E).astype(np.float32)
    w0_lp = O.f32_to_bf16(w0) if kind == 2 else w0.astype(np.float16)
    w32 = O.bf16_to_f32(w0_lp) if kind == 2 else w0_lp.astype(np.float32)
    kw = dict(learning_rate=0.01, wd=1e-3, rescale_grad=0.5, clip_gradient=0.6, clip_weights=0.9, centered=centered)
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w0_lp, mx.gpu(0), dtype=lp))
    kv.set_optimizer(mx.optimizer.RMSProp(multi_precision=mp, **kw))
    oopt = R.OracleRMSProp(**kw)
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


def test_unaligned_view_takes_the_scalar_path():
    """bfloat16 torch views offset by one element (2-byte aligned only): the scalar path of the per-thread kernel,
    centered (all three state arrays)"""
    import torch
    E, n, kind = 10001, 3, 2
    kw = dict(KW, centered=True)
    rng = np.random.default_rng(12)
    w0 = O.f32_to_bf16(rng.uniform(-1, 1, E).astype(np.float32))
    w32 = O.bf16_to_f32(w0)
    wbase = torch.zeros(E + 3, dtype=torch.bfloat16, device="cuda")
    wview = wbase[1:E + 1]
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w0, mx.gpu(0), dtype="bfloat16"))
    kv.set_optimizer(mx.optimizer.RMSProp(**kw))
    oopt = R.OracleRMSProp(**kw)
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


@pytest.mark.parametrize("centered", CENTERED)
def test_cached_launch_plan_replays(centered):
    """identical calls replay a recorded launch plan (the centered momentum travels in the recorded entries); a
    learning-rate change is patched in"""
    sizes = [8, 1000, 4096 + 4, 70001, 1 << 18]
    rng = np.random.default_rng(31)
    keys = list(range(len(sizes)))
    w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in sizes]
    kv, okv = _stores(keys, w0, dict(KW, centered=centered))
    gdev = [[mx.nd.empty((e,), mx.gpu(0)) for _ in range(2)] for e in sizes]
    outs = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]

    def step():
        grads = [[rng.uniform(-1, 1, e).astype(np.float32) for _ in range(2)] for e in sizes]
        for gd, gs in zip(gdev, grads):
            for d, g in zip(gd, gs):
                d[:] = g
        kv.pushpull(keys, gdev, out=outs)
        okv.push(keys, grads)
        _check(okv, keys, outs, "replay")

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


def _set_state_4(kv, key, value):
    from mxnet_b200.base import _LIB, check_call
    v = mx.nd.array(value, mx.gpu(0))
    check_call(_LIB.MXKVB200SetState(kv.handle, int(key), None, 4, v.handle))
    mx.nd.waitall()


@pytest.mark.parametrize("centered", CENTERED)
def test_save_load_round_trip_continues_bit_exact(centered):
    """save / load of the fused states: the reloaded store continues bit for bit; the file holds state2 (the centered
    momentum) for the centered kind only"""
    import pickle
    sizes = [1000, 70001, (1 << 20) + 4]
    rng = np.random.default_rng(8)
    keys = list(range(len(sizes)))
    w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in sizes]
    kw = dict(KW, centered=centered)
    kv, okv = _stores(keys, w0, kw)
    outs = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]
    for _ in range(2):
        grads = [[rng.uniform(-1, 1, e).astype(np.float32) for _ in range(2)] for e in sizes]
        kv.pushpull(keys, [[mx.nd.array(g, mx.gpu(0)) for g in gs] for gs in grads], out=outs)
        okv.push(keys, grads)
    d = tempfile.mkdtemp(prefix="mxkv_rmsprop_")
    f = os.path.join(d, "states")
    kv.save_optimizer_states(f, dump_optimizer=True)
    with open(f, "rb") as fin:
        payload = pickle.load(fin)
    assert payload["format"] == "mxkv_b200_fused_v1"
    for k in keys:
        ent = payload["states"][k]
        assert ("state1" in ent) == ("state2" in ent) == centered, sorted(ent)
        for i, name in enumerate(["state0", "state1", "state2"][:3 if centered else 1]):
            assert_bits_equal(ent[name].reshape(-1), okv.optimizer.states[k][i].reshape(-1), name)
    kv2 = mx.kv.create("device")
    kv2.init(keys, [mx.nd.array(o.asnumpy(), mx.gpu(0)) for o in outs])
    kv2.set_optimizer(mx.optimizer.RMSProp(**kw))
    kv2.load_optimizer_states(f)
    os.remove(f)
    os.rmdir(d)
    outs2 = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]
    for s in range(2):
        grads = [[rng.uniform(-1, 1, e).astype(np.float32) for _ in range(2)] for e in sizes]
        kv2.pushpull(keys, [[mx.nd.array(g, mx.gpu(0)) for g in gs] for gs in grads], out=outs2)
        okv.push(keys, grads)
        _check(okv, keys, outs2, "after reload step %d" % s)
    _check_states(kv2, okv, keys, "after reload")


@pytest.mark.parametrize("opt", ["rmsprop", "sgd_momentum"])
def test_no_third_state_where_the_optimizer_has_none(opt):
    """GetState(4) is NULL for plain RMSProp and for an optimizer of before (SGD-momentum); SetState(4) is refused with
    the "no such state" message"""
    rng = np.random.default_rng(6)
    w0 = rng.uniform(0, 1, 4099).astype(np.float32)
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w0, mx.gpu(0)))
    kv.set_optimizer(mx.optimizer.RMSProp(**KW) if opt == "rmsprop" else mx.optimizer.SGD(momentum=0.9, **KW))
    out = mx.nd.empty((4099,), mx.gpu(0))
    kv.pushpull(0, [mx.nd.array(rng.uniform(-1, 1, 4099).astype(np.float32), mx.gpu(0))], out=out)
    assert _state(kv, 0, 2) is not None and _state(kv, 0, 3) is None
    assert _state(kv, 0, 4) is None
    with pytest.raises(mx.MXNetError, match="the active optimizer has no such state"):
        _set_state_4(kv, 0, np.zeros(4099, np.float32))


def test_centered_to_plain_switch_drops_the_third_state():
    """set_optimizer with a NEW RMSProp(centered=False) after centered steps starts from fresh state like the
    reference's new Updater: mean and momentum are gone, var starts from zero, and the results are plain RMSProp's"""
    sizes = [1000, 70001]
    keys = list(range(len(sizes)))
    rng = np.random.default_rng(17)
    w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in sizes]
    kv, okv = _stores(keys, w0, dict(KW, centered=True))
    outs = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]
    for _ in range(2):
        grads = [[rng.uniform(-1, 1, e).astype(np.float32) for _ in range(2)] for e in sizes]
        kv.pushpull(keys, [[mx.nd.array(g, mx.gpu(0)) for g in gs] for gs in grads], out=outs)
        okv.push(keys, grads)
    assert all(_state(kv, k, 4) is not None for k in keys)
    kv.set_optimizer(mx.optimizer.RMSProp(**KW))
    okv2 = O.OracleKVStore("device")
    okv2.init(keys, [o.asnumpy() for o in outs])
    okv2.set_optimizer(R.OracleRMSProp(**KW))
    for s in range(2):
        grads = [[rng.uniform(-1, 1, e).astype(np.float32) for _ in range(2)] for e in sizes]
        kv.pushpull(keys, [[mx.nd.array(g, mx.gpu(0)) for g in gs] for gs in grads], out=outs)
        okv2.push(keys, grads)
        _check(okv2, keys, outs, "plain after centered step %d" % s)
    for k in keys:
        assert _state(kv, k, 3) is None and _state(kv, k, 4) is None
    _check_states(kv, okv2, keys, "plain after centered")
    with pytest.raises(mx.MXNetError, match="the active optimizer has no such state"):
        _set_state_4(kv, 0, np.zeros(sizes[0], np.float32))


@pytest.mark.parametrize("centered", CENTERED)
def test_native_updater(centered):
    shapes = [(64,), (3, 5), (1000,), (257, 33), (7,)]
    rng = np.random.default_rng(5)
    w0 = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
    weights = [mx.nd.array(w, mx.gpu(0)) for w in w0]
    kw = dict(learning_rate=0.01, wd=1e-2, clip_gradient=0.3, rho=0.8, clip_weights=0.9, centered=centered)
    upd = mx.optimizer.get_updater(mx.optimizer.create("rmsprop", **kw))
    assert isinstance(upd, mx.optimizer.NativeUpdater)
    oopt = R.OracleRMSProp(**kw)
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


@pytest.mark.parametrize("centered", CENTERED)
def test_row_sparse_gradient_is_refused(centered):
    rows, L = 100, 8
    kv = mx.kv.create("device")
    kv.init("w", mx.nd.array(np.zeros((rows, L), np.float32), mx.gpu(0)))
    kv.set_optimizer(mx.optimizer.RMSProp(learning_rate=0.1, centered=centered))
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
def test_trainer_modes_match_the_oracle(mode):
    import torch
    model = _net()
    params = list(model.parameters())
    kw = dict(learning_rate=0.01, wd=1e-4, centered=True)
    targs = {"update_on_kvstore": dict(kvstore="device", update_on_kvstore=True),
             "local_update": dict(kvstore="device", update_on_kvstore=False),
             "no_kvstore": dict(kvstore=None),
             "overlap": dict(kvstore="device", overlap=True, bucket_bytes=64 << 10)}[mode]
    trainer = mx.Trainer(params, "rmsprop", dict(kw), **targs)
    ref_w = [p.detach().cpu().numpy().copy().reshape(-1) for p in params]
    opt = R.OracleRMSProp(**kw)
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


@pytest.mark.parametrize("centered", CENTERED)
def test_fused_and_python_step_agree(centered):
    """use_fused_step=False runs RMSProp.step (rmsprop.py:90-141 restated in torch) through the Python updater; it
    agrees with the fused kernel within the reference's test_rms float32 tolerance (rtol 1e-2, atol 1e-2)"""
    import torch
    ma, mb = _net(1), _net(1)
    kw = dict(learning_rate=0.001, wd=1e-3, clip_gradient=0.01, clip_weights=0.2, rho=0.8, centered=centered)
    ta = mx.Trainer(list(ma.parameters()), "rmsprop", dict(kw), kvstore="device")
    tb = mx.Trainer(list(mb.parameters()), "rmsprop", dict(kw, use_fused_step=False), kvstore="device")
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
            np.testing.assert_allclose(pb.detach().cpu().numpy(), pa.detach().cpu().numpy(), rtol=1e-2, atol=1e-2)


# ---------------------------------------------------------------------------
# several GPUs in one process
# ---------------------------------------------------------------------------
@pytest.mark.multigpu
@pytest.mark.parametrize("centered", CENTERED)
def test_multi_gpu_one_and_two_shot_keys_with_a_checkpoint(centered):
    """one value per GPU, outputs on every GPU; the large keys are split into shards (two-shot) and so are their
    states, the centered momentum included; a save / load round trip in between gathers and redistributes them"""
    n = min(mx.num_gpus(), 8)
    shapes = [(1000,), (37, 13), (70001,), ((1 << 20) + 12,), (1 << 21,)]
    keys = list(range(len(shapes)))
    rng = np.random.default_rng(40 + n)
    w0 = [rng.uniform(0, 1, s).astype(np.float32) for s in shapes]
    kw = dict(KW, rescale_grad=0.5, clip_gradient=0.7, clip_weights=0.95, centered=centered)
    kv, okv = _stores(keys, w0, kw)
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
    d = tempfile.mkdtemp(prefix="mxkv_rmsprop_")
    f = os.path.join(d, "states")
    kv.save_optimizer_states(f, dump_optimizer=True)
    kv2 = mx.kv.create("device")
    kv2.init(keys, [mx.nd.array(outs[k][0].asnumpy(), mx.gpu(0)) for k in keys])
    kv2.set_optimizer(mx.optimizer.RMSProp(**kw))
    kv2.load_optimizer_states(f)
    os.remove(f)
    os.rmdir(d)
    for _ in range(2):
        step(kv2)


@pytest.mark.multigpu
@pytest.mark.parametrize("centered", CENTERED)
@pytest.mark.parametrize("n", [3, 8])
def test_tree_sum_feeds_rmsprop(monkeypatch, n, centered):
    """MXNET_KVSTORE_USETREE=1: RMSProp consumes the sum of the reference's tree order, bit for bit against
    oracle.tree_reduce followed by RMSProp"""
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
    kw = dict(KW, centered=centered)
    rng = np.random.default_rng(n)
    w0 = [rng.uniform(0, 1, s).astype(np.float32) for s in shapes]
    kv = mx.kv.create("device")
    kv.init(keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
    kv.set_optimizer(mx.optimizer.RMSProp(**kw))
    okv = O.OracleKVStore("device", tree=tree)
    okv.init(keys, [w.copy() for w in w0])
    okv.set_optimizer(R.OracleRMSProp(**kw))
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
