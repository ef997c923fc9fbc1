"""The plug-in side of the boundary: `KVStoreBase.register` + `create(name)` (python/mxnet/kvstore/base.py:74-243,
406-461), driven the way tests/python/unittest/test_kvstore_custom.py:148-184 drives the reference's own sample
plug-in.  The sample store here is written by the *test*, as a third party would write one, against this package's
base class; host arrays only, so no GPU is needed."""
import numpy as np
import pytest

import mxnet_b200 as mx
from mxnet_b200.kvstore import KVStoreBase


@KVStoreBase.register
class SampleStore(KVStoreBase):
    """broadcast copies, pushpull sums on the first value's context -- what the reference's sample plug-in does"""

    def broadcast(self, key, value, out, priority=0):
        for o in (out if isinstance(out, list) else [out]):
            o[:] = value

    def pushpull(self, key, value, out=None, priority=0):
        if isinstance(value, mx.nd.NDArray):
            if out is not None:
                for o in (out if isinstance(out, list) else [out]):
                    o[:] = value
            return
        ctx = value[0].context
        reduced = sum([v.as_in_context(ctx) for v in value])
        for o in (value if out is None else (out if isinstance(out, list) else [out])):
            o[:] = reduced

    @staticmethod
    def is_capable(capability):
        if capability.lower() == KVStoreBase.OPTIMIZER:
            return False
        raise ValueError("Unknown capability: {}".format(capability))

    @property
    def type(self):
        return "samplestore"

    @property
    def rank(self):
        return 0

    @property
    def num_workers(self):
        return 1


def check_diff_to_scalar(A, x):
    assert np.sum(np.abs(A.asnumpy() - x)) == 0, (A.asnumpy(), x)


def test_custom_store():
    # test_kvstore_custom.py:148-163
    kv = mx.kv.create("samplestore")
    assert isinstance(kv, SampleStore)
    out = mx.nd.empty((1,))
    kv.broadcast(1, mx.nd.ones((1,)), out=out)
    check_diff_to_scalar(out, 1)
    assert type(kv).is_capable("optimizer") is False
    kv.broadcast(1, mx.nd.ones((1,)), out=out)
    check_diff_to_scalar(out, 1)
    arr_list = [mx.nd.empty((1,))] * 2
    kv.pushpull(1, [mx.nd.ones((1,))] * 2, out=arr_list)
    for arr in arr_list:
        check_diff_to_scalar(arr, 2)
    kv.pushpull(1, arr_list)
    for arr in arr_list:
        check_diff_to_scalar(arr, 4)


def test_get_type_of_a_registered_store():
    # test_kvstore_custom.py:165-168; the name is the lower-cased class name, matched case-insensitively
    assert mx.kv.create("samplestore").type == "samplestore"
    assert isinstance(mx.kv.create("SampleStore"), SampleStore)


def test_set_optimizer_unsupported_by_a_plug_in():
    # test_kvstore_custom.py:170-180: what a plug-in does not override raises NotImplementedError
    kv = mx.kv.create("samplestore")
    assert not kv.is_capable("optimizer")
    with pytest.raises(NotImplementedError):
        kv.set_optimizer(mx.optimizer.create("sgd"))
    with pytest.raises(NotImplementedError):
        kv.save_optimizer_states("test")
    with pytest.raises(NotImplementedError):
        kv.load_optimizer_states("test")


def test_registry_rules():
    # base.py:225-243 (register takes classes), :432-435 (create takes a string); names that are not registered
    # fall through to the native factory, which knows the reference's built-in types and rejects the rest
    with pytest.raises(AssertionError):
        KVStoreBase.register(SampleStore())
    with pytest.raises(TypeError):
        mx.kv.create(3)
    # src/kvstore/kvstore.cc:42-84: any other name is a local store that reports the name it was given
    assert mx.kv.create("no_such_store").type == "no_such_store"
    with pytest.raises(mx.MXNetError):
        mx.kv.create("dist_sync")                            # out of scope of this library, said loudly
    assert "b200device" in KVStoreBase.kv_registry          # the engine's own entry
    assert mx.kv.KVStore.is_capable("optimizer") is True
    with pytest.raises(mx.MXNetError):
        mx.kv.KVStore.is_capable("no_such_capability")


def test_trainer_refuses_update_on_kvstore_for_a_plug_in_without_optimizer_support():
    # gluon/trainer.py:225-229: a store that is not capable of 'optimizer' cannot own the update;
    # with update_on_kvstore left to the trainer it falls back to local updates
    # (tests/nightly/dist_device_sync_kvstore.py:107-125 checks the same table for its store)
    class Param(object):
        def __init__(self, ctx):
            self.data = mx.nd.zeros((10, 1), ctx)
            self.grad = mx.nd.ones((10, 1), ctx)

    params = [[Param(mx.Context("cpu", 0)), Param(mx.Context("cpu", 1))]]
    kv = mx.kv.create("samplestore")
    tr = mx.Trainer(params, "sgd", {"learning_rate": 0.1}, kvstore=kv, update_on_kvstore=True)
    with pytest.raises(ValueError):
        tr._init_kvstore()
    for uok in (False, None):
        tr = mx.Trainer(params, "sgd", {"learning_rate": 0.1}, kvstore=kv, update_on_kvstore=uok)
        tr._init_kvstore()
        assert tr._kv_initialized and tr._update_on_kvstore is False
        # the plug-in is driven one key per call, as the reference's Trainer drives it
        tr.allreduce_grads()
        for p in params[0]:
            check_diff_to_scalar(p.grad, 2)
        for p in params[0]:
            p.grad[:] = 1


# ---- the other plug-in point: optimizers written in Python against the reference's protocol ----------------------
@mx.optimizer.register
class SignSGD(mx.optimizer.Optimizer):
    """a user-defined optimizer exactly as one is written for the reference (optimizer.py:214-352): list-valued
    ``step`` that counts the update itself, a state per index, learning rates through ``_get_lrs``"""

    def create_state(self, index, weight):
        return mx.nd.zeros(weight.shape, weight.context)           # number of sign flips seen, say

    def step(self, indices, weights, grads, states):
        self._update_count(indices)
        lrs = self._get_lrs(indices)
        wds = self._get_wds(indices)
        for w, g, s, lr, wd in zip(weights, grads, states, lrs, wds):
            step = np.sign(g.asnumpy() * self.rescale_grad + wd * w.asnumpy())
            w[:] = w.asnumpy() - lr * step
            s[:] = s.asnumpy() + np.abs(step)


def test_user_defined_optimizer_through_the_updater():
    """updater.py:39-93 + optimizer.py:287-352 with host arrays: single and list calls, per-index states, update
    counts taken by the optimizer's own ``step`` (once per call, not twice), lr multipliers by index."""
    opt = mx.optimizer.create("signsgd", learning_rate=0.5, wd=0.0)
    opt.set_lr_mult({1: 0.5})
    upd = mx.optimizer.get_updater(opt)
    assert type(upd).__name__ == "Updater"                      # no fused kernel of that name
    w = [mx.nd.zeros((4,)), mx.nd.ones((3,))]
    g = [mx.nd.array(np.array([1, -1, 2, -2], np.float32)), mx.nd.array(np.array([1, 1, -1], np.float32))]
    upd(0, g[0], w[0])
    assert np.array_equal(w[0].asnumpy(), [-0.5, 0.5, -0.5, 0.5])
    upd([0, 1], g, w)
    assert np.array_equal(w[0].asnumpy(), [-1, 1, -1, 1])
    assert np.array_equal(w[1].asnumpy(), [0.75, 0.75, 1.25])
    assert opt._index_update_count == {0: 2, 1: 1} and opt.num_update == 2
    assert np.array_equal(upd.states[0].asnumpy(), [2, 2, 2, 2])
    # states survive get_states / set_states, with and without the optimizer
    blob = upd.get_states(dump_optimizer=True)
    upd2 = mx.optimizer.get_updater(mx.optimizer.create("signsgd", learning_rate=0.5))
    upd2.set_states(blob)
    assert upd2.optimizer._index_update_count == {0: 2, 1: 1}
    assert np.array_equal(upd2.states[1].asnumpy(), [1, 1, 1])
    upd2(1, g[1], w[1])
    assert np.array_equal(w[1].asnumpy(), [0.5, 0.5, 1.5])
    assert np.array_equal(upd2.states[1].asnumpy(), [2, 2, 2])


def test_multi_precision_protocol_of_python_optimizers():
    """optimizer.py:214-243,320-352: float16 weights get a float32 master copy in front of the state; the update
    runs on the master and is cast back"""
    opt = mx.optimizer.create("signsgd", learning_rate=2.0 ** -12, multi_precision=True)
    upd = mx.optimizer.get_updater(opt)
    w = mx.nd.array(np.ones((4,), np.float16), dtype=np.float16)
    g = mx.nd.array(np.ones((4,), np.float16), dtype=np.float16)
    for _ in range(3):
        upd(7, g, w)
    master, state = upd.states[7]
    assert master.dtype == np.float32 and np.all(master.asnumpy() == np.float32(1 - 3 * 2.0 ** -12))
    assert w.dtype == np.float16 and np.all(w.asnumpy() == np.float16(1 - 3 * 2.0 ** -12))   # 1 - 2^-12 alone would round to 1
    assert np.all(state.asnumpy() == 3)


# ---- tests/python/unittest/test_optimizer.py: the learning-rate plumbing and the schedulers' closed-form points ---------
def test_learning_rate():
    # test_optimizer.py:30-43
    o1 = mx.optimizer.Optimizer(learning_rate=0.01)
    o1.set_learning_rate(0.2)
    assert o1.learning_rate == 0.2
    lr_s = mx.lr_scheduler.FactorScheduler(step=1)
    o2 = mx.optimizer.Optimizer(lr_scheduler=lr_s, learning_rate=0.3)
    assert o2.learning_rate == 0.3
    o2.lr_scheduler.base_lr = 0.4
    assert o2.learning_rate == 0.4
    lr_s = mx.lr_scheduler.FactorScheduler(step=1, base_lr=1024)
    o3 = mx.optimizer.Optimizer(lr_scheduler=lr_s)
    assert o3.learning_rate == 1024


def test_learning_rate_expect_user_warning():
    # test_optimizer.py:46-51
    o = mx.optimizer.Optimizer(lr_scheduler=mx.lr_scheduler.FactorScheduler(step=1), learning_rate=0.3)
    with pytest.raises(UserWarning):
        o.set_learning_rate(0.5)


def test_scheduler_known_points():
    # test_optimizer.py:951-1005
    sched = mx.lr_scheduler.FactorScheduler(100, 0.1, stop_factor_lr=1e-4, base_lr=1, warmup_steps=20,
                                            warmup_begin_lr=0.1, warmup_mode="constant")
    assert sched(0) == 0.1
    np.testing.assert_almost_equal(sched(10), 0.1)
    assert sched(21) == 1
    np.testing.assert_almost_equal(sched(101), 0.1)
    np.testing.assert_almost_equal(sched(201), 0.01)
    np.testing.assert_almost_equal(sched(1000), 1e-4)
    sched = mx.lr_scheduler.MultiFactorScheduler([15, 25], 0.1, base_lr=0.1, warmup_steps=10, warmup_begin_lr=0.05,
                                                 warmup_mode="linear")
    assert sched(0) == 0.05
    np.testing.assert_almost_equal(sched(5), 0.05 + (0.1 - 0.05) / 2)
    np.testing.assert_almost_equal(sched(15), 0.1)
    np.testing.assert_almost_equal(sched(16), 0.01)
    np.testing.assert_almost_equal(sched(20), 0.01)
    np.testing.assert_almost_equal(sched(26), 0.001)
    np.testing.assert_almost_equal(sched(100), 0.001)
    poly = mx.lr_scheduler.PolyScheduler(1000, base_lr=3, pwr=2, final_lr=0, warmup_steps=100, warmup_begin_lr=0,
                                         warmup_mode="linear")
    np.testing.assert_almost_equal(poly(0), 0)
    np.testing.assert_almost_equal(poly(50), 1.5)
    np.testing.assert_almost_equal(poly(100), 3)
    assert poly(101) < poly(100) and poly(500) < 1.6
    np.testing.assert_almost_equal(poly(1000), 0)
    cos = mx.lr_scheduler.CosineScheduler(1000, base_lr=3, final_lr=0.1)
    np.testing.assert_almost_equal(cos(0), 3)
    np.testing.assert_almost_equal(cos(1000), 0.1)
    assert cos(500) > 1.5


def test_bench_helpers_without_a_gpu():
    """bench.py's host-side pieces: deterministic synthetic data (what lets rank 0 regenerate every rank's gradients for
    the parity check), the workload key sets, and the in-process NVML clock sampler driven by a stand-in module."""
    import importlib
    import os
    import sys
    import time
    import types
    import numpy as np
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    bench = importlib.import_module("bench")
    sweep = bench.keyset("sweep")
    assert [bench.nelem(s) for s in sweep] == [1 << p for p in range(10, 27, 2)]
    assert len(bench.keyset("resnet50")) == 193 and sum(bench.nelem(s) for s in bench.keyset("resnet50")) == 25575912
    assert len(bench.keyset("bert")) == 199
    small = [(1000,), (1 << 21,)]
    a, b = bench.rank_grads(3, small), bench.rank_grads(3, small)
    assert all(np.array_equal(x, y) for x, y in zip(a, b)) and not np.array_equal(a[1], bench.rank_grads(4, small)[1])
    big = a[1]                                         # above 2^20 elements: a random block of 1 000 003 elements, repeated
    assert np.array_equal(big[:1000003][:1000], big[1000003:1000003 + 1000]) and big.dtype == np.float32
    # --dump-outputs: the same positions every run, within the budget; small key sets are dumped whole
    for wl in ("sweep", "resnet50", "bert"):
        shapes = bench.keyset(wl)
        pos, again = bench.dump_positions(shapes), bench.dump_positions(shapes)
        assert sum(bench.nelem(s) if p is None else p.size for s, p in zip(shapes, pos)) <= bench.DUMP_ELEMS
        assert all((p is None and q is None) or np.array_equal(p, q) for p, q in zip(pos, again))
        assert all(p is None or (np.all(np.diff(p) > 0) and p[-1] < bench.nelem(s)) for s, p in zip(shapes, pos))
    assert bench.dump_positions(small) == [None, None]
    # clock sampler on a stand-in pynvml
    fake = types.ModuleType("pynvml")
    fake.NVML_CLOCK_SM = 1
    fake.nvmlInit = lambda: None
    fake.nvmlDeviceGetHandleByIndex = lambda i: i
    fake.nvmlDeviceGetMaxClockInfo = lambda h, c: 1965
    fake.nvmlDeviceGetClockInfo = lambda h, c: 1950
    fake.nvmlDeviceGetCurrentClocksEventReasons = lambda h: 0x4 | 0x40
    saved = sys.modules.get("pynvml")
    sys.modules["pynvml"] = fake
    try:
        s = bench.ClockSampler(0)
        s.start()
        s.wait_first()
        t0 = time.time(); time.sleep(0.35); t1 = time.time()
        rec = s.stop(t0, t1)
    finally:
        if saved is not None:
            sys.modules["pynvml"] = saved
        else:
            del sys.modules["pynvml"]
    assert rec["samples"] >= 2 and rec["sm_mhz"] == 1950.0 and rec["sm_max_mhz"] == 1965.0
    assert rec["reasons"] == ["hw_thermal_slowdown", "sw_power_cap"] and "NVML" in rec["how"]
    info = bench.bind_to_gpu_numa(0)                   # no driver here: a description, never an exception
    assert info["gpu"] == 0
