"""Semantics added late in round 1 (DESIGN.md §10 item 0): update counts that follow the Python optimizer, a new optimizer starting from fresh
state, row_sparse gradients for dense keys, user-defined Python optimizers on the store, the reference's
`test_sparse_aggregator` / bandwidth-tool / many-array `multi_sum_sq` cases.  They pass on the simulated runtime
(tests/sim); the file name keeps them behind the hardware-validated tests in a `pytest -x` run."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import mxnet_b200 as mx
from oracle import oracle as O
import test_gpu_dense as _dense_tests          # its fused-case driver

shape = (4, 4)
keys = [5, 7, 11]
str_keys = ["b", "c", "d"]


def ctx_of(dev, i=0):
    return mx.gpu(0) if dev == "gpu" else mx.Context("cpu", i)


def _rng(seed):
    return np.random.default_rng(4321 + seed)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32, 8: np.uint64, 1: np.uint8}[a.dtype.itemsize])


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def assert_bits_equal(a, b, msg=""):
    assert a.shape == b.shape, (a.shape, b.shape)
    ne = _bits(a) != _bits(b)
    assert not ne.any(), "%s: %d / %d elements differ" % (msg, ne.sum(), ne.size)


def _rand_rsp(rng, rows, L, nnz):
    idx = np.sort(rng.choice(rows, nnz, replace=False)).astype(np.int64)
    val = rng.uniform(-1, 1, (nnz, L)).astype(np.float32)
    return idx, val


def _mk(idx, val, shape, ctx):
    return mx.nd.row_sparse_array((val, idx), shape=shape, ctx=ctx)


def test_update_count_follows_the_python_optimizer(tmp_path):
    """The t of Adam's bias correction is the optimizer's per-index update count (adam.py:166-175 via
    optimizer.py:445-462): it starts at begin_num_update, carries over when an optimizer that has already been
    stepping is handed to another store, and is NOT restored by states saved without their optimizer
    (updater.py:118-127)."""
    rng = np.random.default_rng(31)
    E = 1000
    w0 = rng.uniform(-1, 1, E).astype(np.float32)
    gs = [rng.uniform(-1, 1, E).astype(np.float32) for _ in range(6)]
    kw = dict(learning_rate=0.01, begin_num_update=7)

    def push(kv, g):
        kv.push(3, mx.nd.array(g, mx.gpu(0)))
        o = mx.nd.empty((E,), mx.gpu(0))
        kv.pull(3, out=o)
        return o.asnumpy()

    kv = mx.kv.create("device")
    kv.init(3, mx.nd.array(w0, mx.gpu(0)))
    opt = mx.optimizer.Adam(**kw)
    kv.set_optimizer(opt)
    oopt = O.OracleOptimizer("adam", **kw)
    ow = w0.copy()
    for g in gs[:2]:
        oopt.update(3, ow, g)
        assert_bits_equal(push(kv, g), ow, "t = 8, 9")
    assert opt._index_update_count[3] == 9
    # the same optimizer object on a fresh store: t goes on at 10 while the moments restart from zero
    kv2 = mx.kv.create("device")
    kv2.init(3, mx.nd.array(ow, mx.gpu(0)))
    kv2.set_optimizer(opt)
    oopt.states.pop(3, None)
    for g in gs[2:4]:
        oopt.update(3, ow, g)
        assert_bits_equal(push(kv2, g), ow, "t = 10, 11 on a fresh store")
    # states saved WITHOUT the optimizer, loaded into a store whose optimizer starts from scratch: the moments come
    # back, t restarts at 1
    f = str(tmp_path / "adam.states")
    kv2.save_optimizer_states(f)
    kv3 = mx.kv.create("device")
    kv3.init(3, mx.nd.array(ow, mx.gpu(0)))
    kv3.set_optimizer(mx.optimizer.Adam(learning_rate=0.01))
    kv3.load_optimizer_states(f)
    o3 = O.OracleOptimizer("adam", learning_rate=0.01)
    o3.states[3] = oopt.states[3]
    for g in gs[4:]:
        o3.update(3, ow, g)
        assert_bits_equal(push(kv3, g), ow, "loaded moments, t from 1")


def test_a_new_optimizer_starts_from_fresh_state():
    """kvstore.py:559-606: set_optimizer installs a NEW updater, so the momentum of the previous optimizer is gone
    (and never reinterpreted as another optimizer's state); handing the SAME optimizer object again (what the
    Trainer does when rescale_grad changes with the batch size) keeps the state."""
    rng = np.random.default_rng(77)
    E = 4099
    w0 = rng.uniform(-1, 1, E).astype(np.float32)
    gs = [rng.uniform(-1, 1, E).astype(np.float32) for _ in range(6)]

    def push(kv, g):
        kv.push(0, mx.nd.array(g, mx.gpu(0)))
        o = mx.nd.empty((E,), mx.gpu(0))
        kv.pull(0, out=o)
        return o.asnumpy()

    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w0, mx.gpu(0)))
    sgd = mx.optimizer.SGD(learning_rate=0.1, momentum=0.9)
    kv.set_optimizer(sgd)
    o1 = O.OracleOptimizer("sgd", learning_rate=0.1, momentum=0.9)
    ow = w0.copy()
    for g in gs[:2]:
        o1.update(0, ow, g)
        assert_bits_equal(push(kv, g), ow, "sgd momentum")
    sgd.rescale_grad = 0.5                                  # same object, new hyper-parameter: momentum carries on
    kv.set_optimizer(sgd)
    o1.rescale_grad = 0.5
    o1.update(0, ow, gs[2])
    assert_bits_equal(push(kv, gs[2]), ow, "same optimizer again keeps its state")
    kv.set_optimizer(mx.optimizer.Adam(learning_rate=0.01))   # a new optimizer: fresh mean / variance, t = 1
    o2 = O.OracleOptimizer("adam", learning_rate=0.01)
    for g in gs[3:5]:
        o2.update(0, ow, g)
        assert_bits_equal(push(kv, g), ow, "adam after sgd starts from zero moments")
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9))   # and back: the old momentum is not revived
    o3 = O.OracleOptimizer("sgd", learning_rate=0.1, momentum=0.9)
    o3.update(0, ow, gs[5])
    assert_bits_equal(push(kv, gs[5]), ow, "a second sgd starts with zero momentum")


def test_update_count_is_the_optimizers():
    """begin_num_update and an optimizer that has already been stepping: the native updater's t follows the
    optimizer's table (optimizer.py:445-462), like the reference's Updater"""
    rng = np.random.default_rng(12)
    w0 = rng.uniform(-1, 1, 500).astype(np.float32)
    gs = [rng.uniform(-1, 1, 500).astype(np.float32) for _ in range(4)]
    kw = dict(learning_rate=0.01, begin_num_update=5)
    opt = mx.optimizer.Adam(**kw)
    oopt = O.OracleOptimizer("adam", **kw)
    ow = w0.copy()
    w = mx.nd.array(w0, mx.gpu(0))
    upd = mx.optimizer.get_updater(opt)
    for g in gs[:2]:
        upd(0, mx.nd.array(g, mx.gpu(0)), w)
        oopt.update(0, ow, g)
        assert _bits_equal(w.asnumpy(), ow)
    assert opt._index_update_count[0] == 7
    upd2 = mx.optimizer.get_updater(opt)            # a second updater, same optimizer: t goes on, moments restart
    oopt.states.pop(0)
    for g in gs[2:]:
        upd2(0, mx.nd.array(g, mx.gpu(0)), w)
        oopt.update(0, ow, g)
        assert _bits_equal(w.asnumpy(), ow)


@pytest.mark.parametrize("lazy", [True, False])
@pytest.mark.parametrize("optname,kw", [
    ("sgd", dict(learning_rate=0.1, wd=1e-3, momentum=0.9)),
    ("adam", dict(learning_rate=0.01, wd=1e-3)),
])
def test_dense_key_takes_row_sparse_and_dense_gradients(optname, kw, lazy):
    """A DENSE weight updated on the store with row_sparse gradients (gluon Parameter(grad_stype='row_sparse')
    with update_on_kvstore=True, trainer.py:204-236; SGDUpdateDnsRspImpl / SGDMomLazy... / AdamLazy... on a dense
    weight): the key stays dense -- plain pull and pushpull keep working --, dense and row_sparse pushes may
    alternate, the optimizer state is shared between the two kinds of update, and with several GPUs the sharded
    state of a large dense push is gathered before the rows are updated."""
    kw = dict(kw, lazy_update=lazy)
    devs = list(range(min(mx.num_gpus(), 4)))
    rng = np.random.default_rng(21)
    rows, L, nnz = 3000, 64, 200                       # 768 KB: a dense push from several GPUs is sharded
    shape = (rows, L)
    w0 = rng.uniform(0, 1, shape).astype(np.float32)
    kv = mx.kv.create("device")
    kv.init(7, mx.nd.array(w0, mx.gpu(0)))
    kv.set_optimizer(mx.optimizer.create(optname, **kw))
    okv = O.OracleKVStore("device")
    okv.init(7, w0.copy())
    okv.set_optimizer(O.OracleOptimizer(optname, **kw))
    for step, kind in enumerate(["rsp", "dense", "rsp", "rsp", "dense", "rsp"]):
        if kind == "rsp":
            srcs = [_rand_rsp(rng, rows, L, nnz) for _ in devs]
            kv.push(7, [_mk(i, v, shape, mx.gpu(d)) for (i, v), d in zip(srcs, devs)])
            okv.push(7, [O.RowSparse(i, v, shape) for i, v in srcs])
        else:
            gs = [rng.uniform(-1, 1, shape).astype(np.float32) for _ in devs]
            kv.push(7, [mx.nd.array(g, mx.gpu(d)) for g, d in zip(gs, devs)])
            okv.push(7, gs)
        for d in devs:
            out = mx.nd.empty(shape, mx.gpu(d))
            kv.pull(7, out=out)
            assert _bits_equal(out.asnumpy(), okv.local[7]), (optname, lazy, step, kind, d)


@pytest.mark.parametrize("sparse_pull", [False, True])
@pytest.mark.parametrize("dev", ["cpu", "gpu"])
def test_sparse_aggregator(sparse_pull, dev):
    # tests/python/unittest/test_kvstore.py:174-220: row_sparse keys, random row_sparse values on four contexts,
    # pushed and then read back INTO THE SAME ARRAYS, either with row_sparse_pull of every row or with
    # pull(ignore_sparse=False); single key, then the key list with one shared list of values
    rng = np.random.default_rng(11 + int(sparse_pull))

    def rand_rsp(ctx):
        dense = rng.normal(size=shape).astype(np.float32)
        dense[rng.random(shape[0]) < 0.5] = 0                     # rand_ndarray: random density
        return mx.nd.array(dense, ctx).tostype("row_sparse")

    kv = mx.kv.create("device")
    kv.init("a", mx.nd.zeros(shape, stype="row_sparse"))
    kv.init(str_keys, [mx.nd.zeros(shape, stype="row_sparse")] * len(keys))
    num_devs = 4
    devs = [ctx_of(dev, i) for i in range(num_devs)]
    all_rows = mx.nd.array(np.arange(shape[0]), dtype=np.float32)

    vals = [rand_rsp(d) for d in devs]
    expected_sum = np.zeros(shape)
    for v in vals:
        expected_sum += v.todense_numpy()
    kv.push("a", vals)
    if sparse_pull:
        kv.row_sparse_pull("a", out=vals, row_ids=[all_rows] * len(vals))
    else:
        kv.pull("a", out=vals, ignore_sparse=False)
    result_sum = np.zeros(shape)
    for v in vals:
        result_sum += v.todense_numpy()
    np.testing.assert_allclose(result_sum, expected_sum * num_devs, rtol=1e-5, atol=1e-6)

    vals = [[rand_rsp(d) for d in devs]] * len(keys)
    expected_sum = np.zeros(shape)
    for v in vals[0]:
        expected_sum += v.todense_numpy()
    kv.push(str_keys, vals)
    if sparse_pull:
        kv.row_sparse_pull(str_keys, out=vals, row_ids=[[all_rows] * num_devs] * len(vals))
    else:
        kv.pull(str_keys, out=vals, ignore_sparse=False)
    for vv in vals:
        result_sum = np.zeros(shape)
        for v in vv:
            result_sum += v.todense_numpy()
        np.testing.assert_allclose(result_sum, expected_sum * num_devs, rtol=1e-5, atol=1e-6)


def test_user_defined_python_optimizer_on_the_store():
    # kvstore.py:559-606: an optimizer without a fused kernel runs through the updater callback, on the merged
    # value, once per pushed key; written against the reference's Optimizer protocol (list-valued step that
    # counts the update itself)
    @mx.optimizer.register
    class HalfStep(mx.optimizer.Optimizer):
        def create_state(self, index, weight):
            return mx.nd.zeros(weight.shape, weight.context)

        def step(self, indices, weights, grads, states):
            self._update_count(indices)
            for i, w, g, s, lr in zip(indices, weights, grads, states, self._get_lrs(indices)):
                s[:] = s.asnumpy() + 1
                w[:] = w.asnumpy() - lr * self.rescale_grad * g.asnumpy() / s.asnumpy()

    kv = mx.kv.create("device")
    kv.init(keys, [mx.nd.ones(shape, mx.gpu(0))] * len(keys))
    opt = mx.optimizer.create("halfstep", learning_rate=0.5, rescale_grad=0.25)
    kv.set_optimizer(opt)
    want = np.ones(shape, np.float32)
    for step in (1, 2, 3):
        kv.push(keys, [[mx.nd.ones(shape, mx.gpu(0)) * 2.0 for _ in range(4)]] * len(keys))
        want = want - np.float32(0.5 * 0.25) * np.float32(8.0) / np.float32(step)
        outs = [mx.nd.empty(shape, mx.gpu(0)) for _ in keys]
        kv.pull(keys, out=outs)
        for o in outs:
            np.testing.assert_allclose(o.asnumpy(), want, rtol=1e-6)
    assert opt._index_update_count == {k: 3 for k in keys} and opt.num_update == 3


@pytest.mark.parametrize("kv_store,optimizer", [("device", None), ("device", "sgd"), ("local", None), ("local", "sgd")])
def test_bandwidth_tool_results(kv_store, optimizer):
    # tools/bandwidth/test_measure.py:30-44 over tools/bandwidth/measure.py:76-152: the ResNet-50 key set, one
    # gradient per GPU, per-key push(i, g, priority=i) then pull(i, w, priority=i) for two batches; the relative L1
    # error against numpy-summed gradients (and a host-side SGD updater when an optimizer is set) stays below 1e-4
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("bench", os.path.join(os.path.dirname(__file__), "..", "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    shapes = bench.keyset("resnet50")
    devs = [mx.gpu(i) for i in range(max(1, min(mx.num_gpus(), 8)))]
    rng = np.random.default_rng(50)
    kv = mx.kv.create(kv_store)
    oopt = None
    if optimizer is not None:
        kv.set_optimizer(mx.optimizer.create(optimizer))
        oopt = O.OracleOptimizer(optimizer)
    for i, s in enumerate(shapes):
        kv.init(i, mx.nd.zeros(s))
    grads_val = [[rng.uniform(-1, 1, s).astype(np.float32) for _ in devs] for s in shapes]
    grads = [[mx.nd.array(g, d) for g, d in zip(gs, devs)] for gs in grads_val]
    weights = [[mx.nd.zeros(s, d) for d in devs] for s in shapes]
    cpu_grads = [np.sum(np.stack(gs).astype(np.float64), axis=0).astype(np.float32) for gs in grads_val]
    cpu_weights = [np.zeros(s, np.float32) for s in shapes]
    for _ in range(2):
        for i, g in enumerate(grads):
            kv.push(i, g, i)
        for i, w in enumerate(weights):
            kv.pull(i, w, i)
        if oopt is None:
            want = cpu_grads
        else:
            for i in range(len(shapes)):
                oopt.update(i, cpu_weights[i], cpu_grads[i])
            want = cpu_weights
        num = sum(np.sum(np.abs(a.asnumpy() - b)) for w, b in zip(weights, want) for a in w)
        den = sum(np.sum(np.abs(b)) for b in want)
        assert num / den < 1e-4, (kv_store, optimizer, num / den)


@pytest.mark.parametrize("dtype", [np.float16, np.float32, np.float64])
def test_multi_sum_sq_reference_case(dtype):
    # tests/python/gpu/test_operator_gpu.py:192-220: more than a hundred arrays of 50 000 ... 100 000 elements in one
    # call (float16 / float32 / float64 inputs, float32 sums), deterministic, within 1e-5 of numpy's float32 sum
    rng = _rng(40 + np.dtype(dtype).itemsize)
    nparam = int(rng.integers(101, 121))
    xs = [(rng.random(int(rng.integers(50000, 100001))) * 10.).astype(dtype) for _ in range(nparam)]
    arrs = [mx.nd.array(x, mx.gpu(0), dtype=dtype) for x in xs]
    a = mx.nd.multi_sum_sq(*arrs).asnumpy()
    b = mx.nd.multi_sum_sq(*arrs).asnumpy()
    assert _bits_equal(a, b)
    ref = np.array([(x.astype(np.float32) ** 2).sum() for x in xs], np.float32)
    np.testing.assert_allclose(a, ref, rtol=1e-5, atol=1e-5)
    # all-finite over the same arrays, and with one bad element somewhere (test_operator.py:4379-4403)
    assert mx.nd.multi_all_finite(*arrs).asnumpy()[0] == 1.0
    y = xs[nparam // 2].copy(); y[1234] = np.inf
    arrs[nparam // 2] = mx.nd.array(y, mx.gpu(0), dtype=dtype)
    assert mx.nd.multi_all_finite(*arrs).asnumpy()[0] == 0.0


def test_fused_adamw():
    # AdamW as the reference's optimizer class drives the operator: lr = 1, eta = bias-corrected learning
    # rate (adamW.py:176-200), i.e. w -= lr_t * (m / (sqrt(v) + eps) + wd * w); `eta` is this engine's extra
    # schedule multiplier
    kw = dict(learning_rate=0.01, wd=1e-2, beta1=0.9, beta2=0.98, epsilon=1e-6, clip_gradient=0.5)
    for extra in (dict(correct_bias=True), dict(correct_bias=False, eta=0.7)):
        k2 = dict(kw, **extra)
        _dense_tests._fused_case("adamw", k2, k2, 2, 4099, 3)
    # rescale_grad of 0 / inf / nan: the operator leaves weight and state untouched (adamw-inl.h:455)
    for bad in (0.0, float("inf"), float("nan")):
        E = 1003
        w0 = _rng(3).uniform(0, 1, E).astype(np.float32)
        kv = mx.kv.create("device")
        kv.init(0, mx.nd.array(w0, mx.gpu(0)))
        kv.set_optimizer(mx.optimizer.AdamW(learning_rate=0.01, wd=0.1, rescale_grad=bad))
        out = mx.nd.empty((E,), mx.gpu(0))
        kv.pushpull(0, [mx.nd.ones((E,), mx.gpu(0))] * 2, out=out)
        assert_bits_equal(out.asnumpy(), w0, "adamw rescale %r" % bad)
        kv.push(0, mx.nd.ones((E,), mx.gpu(0)))
        kv.pull(0, out=out)
        assert_bits_equal(out.asnumpy(), w0, "adamw rescale %r (push/pull)" % bad)


def _halfstep_cls(name):
    @mx.optimizer.register
    class _HS(mx.optimizer.Optimizer):
        def create_state(self, index, weight):
            return mx.nd.zeros(weight.shape, weight.context)

        def step(self, indices, weights, grads, states):
            self._update_count(indices)
            for i, w, g, s, lr in zip(indices, weights, grads, states, self._get_lrs(indices)):
                s[:] = s.asnumpy() + 1          # "momentum": a state that must survive between steps
                w[:] = w.asnumpy() - lr * self.rescale_grad * g.asnumpy() * s.asnumpy()
    _HS.__name__ = name
    return _HS


def test_switch_from_custom_to_fused_optimizer_replaces_the_updater():
    # ADVICE r1: kvstore.py:559-606 always replaces the updater; a callback left over from an earlier
    # set_optimizer(custom) must not keep running once a fused optimizer is set
    HS = _halfstep_cls("HalfStepA")
    kv = mx.kv.create("device")
    kv.init(3, mx.nd.ones(shape, mx.gpu(0)))
    kv.set_optimizer(HS(learning_rate=0.5))
    kv.push(3, mx.nd.ones(shape, mx.gpu(0)))
    out = mx.nd.empty(shape, mx.gpu(0))
    kv.pull(3, out=out)
    np.testing.assert_allclose(out.asnumpy(), 0.5, rtol=1e-6)
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.5))          # plain SGD: w -= 0.5 * g
    kv.push(3, mx.nd.ones(shape, mx.gpu(0)) * 4.0)
    kv.pull(3, out=out)
    np.testing.assert_allclose(out.asnumpy(), 0.5 - 0.5 * 4.0, rtol=1e-6)
    assert kv._updater is None and kv._fused
    # ... and back again
    kv.set_optimizer(HS(learning_rate=1.0))
    kv.push(3, mx.nd.ones(shape, mx.gpu(0)))
    kv.pull(3, out=out)
    np.testing.assert_allclose(out.asnumpy(), -1.5 - 1.0, rtol=1e-6)


def test_subclass_overriding_step_is_not_sent_to_the_fused_kernel():
    # ADVICE r1: fused_name is inherited; a subclass with its own step() (or use_fused_step=False) must run in Python
    class MySGD(mx.optimizer.SGD):
        def create_state(self, index, weight):
            return None

        def step(self, indices, weights, grads, states):
            self._update_count(indices)
            for w in weights:
                w[:] = 42.0

    assert mx.optimizer.fused_name_of(mx.optimizer.SGD(learning_rate=0.1)) == "sgd"
    assert mx.optimizer.fused_name_of(MySGD(learning_rate=0.1)) is None
    assert mx.optimizer.fused_name_of(mx.optimizer.SGD(learning_rate=0.1, use_fused_step=False)) is None

    class Renamed(mx.optimizer.SGD):          # nothing overridden: still fused
        pass
    assert mx.optimizer.fused_name_of(Renamed(learning_rate=0.1)) == "sgd"

    kv = mx.kv.create("device")
    kv.init(3, mx.nd.ones(shape, mx.gpu(0)))
    kv.set_optimizer(MySGD(learning_rate=0.1))
    assert not kv._fused
    kv.push(3, mx.nd.ones(shape, mx.gpu(0)))
    out = mx.nd.empty(shape, mx.gpu(0))
    kv.pull(3, out=out)
    np.testing.assert_allclose(out.asnumpy(), 42.0)


def test_deferred_issue_orders_by_priority_and_merges():
    """`priority` on this engine (MXKVB200SetDeferred): queued calls are issued highest priority first, never ahead
    of an earlier call on the same key, neighbours on disjoint keys merged into one launch -- the reference's
    per-parameter loop `for i: kv.pushpull(i, g_i, out=w_i, priority=-i)` (gluon/trainer.py:386-409) becomes ONE
    launch, with the results of the immediate form."""
    n = 12
    ks = list(range(n))
    sizes = [5, 64, 1000, 4099, 1 << 14, 7, 300, 2052, 9, 1 << 12, 33, 70001]
    rng = _rng(77)
    w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in sizes]
    kw = dict(learning_rate=0.05, momentum=0.9, wd=1e-3)

    def run(deferred):
        kv = mx.kv.create("device")
        kv.init(ks, [mx.nd.array(w, mx.gpu(0)) for w in w0])
        kv.set_optimizer(mx.optimizer.SGD(**kw))
        if deferred:
            kv.set_deferred(True)
        r = _rng(78)
        outs = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]
        launches = []
        for step in range(3):
            grads = [mx.nd.array(r.uniform(-1, 1, e).astype(np.float32), mx.gpu(0)) for e in sizes]
            l0 = mx.kv.launch_count()
            for i in ks:
                kv.pushpull(i, grads[i], out=outs[i], priority=-i)
            if deferred:
                assert mx.kv.launch_count() == l0, "deferred calls must not launch before the flush point"
            got = [o.asnumpy() for o in outs]          # reading an array is a flush point
            launches.append(mx.kv.launch_count() - l0)
        return got, launches, kv

    want, imm_launches, _ = run(False)
    got, def_launches, kv = run(True)
    for a, b in zip(got, want):
        assert_bits_equal(a, b, "deferred vs immediate")
    assert imm_launches == [n, n, n] and def_launches == [1, 1, 1], (imm_launches, def_launches)
    assert kv.deferred_batches() == 3

    # two pushes of the SAME key keep their program order whatever their priorities (the engine's write-after-write
    # dependency); an independent key with a higher priority goes first but changes nothing else
    kv2 = mx.kv.create("device")
    kv2.init([0, 1], [mx.nd.zeros((8,), mx.gpu(0)), mx.nd.zeros((8,), mx.gpu(0))])
    kv2.set_deferred(True)
    a, b, c = (mx.nd.ones((8,), mx.gpu(0)) * v for v in (1.0, 2.0, 3.0))
    kv2.push(0, a, priority=-5)
    kv2.push(0, b, priority=0)          # later call on key 0: must stay after the first
    kv2.push(1, c, priority=9)
    out0, out1 = mx.nd.empty((8,), mx.gpu(0)), mx.nd.empty((8,), mx.gpu(0))
    kv2.pull([0, 1], out=[out0, out1])  # a pull is a flush point
    assert (out0.asnumpy() == 2.0).all() and (out1.asnumpy() == 3.0).all()
