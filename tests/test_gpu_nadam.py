"""The Nadam optimizer (python/mxnet/optimizer/nadam.py) fused into the gradient exchange and the native updater:
``Nadam.step`` restated in the kernel, against the CPU oracle, bit for bit unless stated, on every dense kernel variant
that serves it.

Most tests are tests/test_gpu_adamax.py's, imported here and run with the ``spec`` fixture below.  The ones after them
are Nadam's own: its ``m_schedule`` is ONE product for the optimizer, multiplied by every key update in the reference's
call order (the sorted keys of a push, the pair order of an updater call, device after device for the per-device
updaters of a Trainer), so key k's update depends on every update before it.  Because ``1 - m_schedule`` rounds to
1.0f after about 22 updates, these tests compare the first steps of a few keys, where the coupling shows."""
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
import nadam_oracle as N  # noqa: E402
from test_gpu_adamax import Spec, assert_bits_equal, _check, _check_states, _count, _net, _bits_equal32  # noqa: E402
from test_gpu_adamax import (  # noqa: E402,F401  (the suite, collected here once more with this file's spec)
    test_forced_variant_whole_sweep_key_set, test_ragged_sizes_and_hyper_parameters_take_effect,
    test_engine_defaults_for_a_c_caller, test_low_precision_keys, test_unaligned_view_takes_the_scalar_path,
    test_cached_launch_plan_replays_with_the_update_count_of_each_step, test_save_load_round_trip_continues_bit_exact,
    test_get_state_and_set_state, test_native_updater, test_row_sparse_gradient_is_refused,
    test_fused_and_python_step_agree, test_multi_gpu_one_and_two_shot_keys_with_a_checkpoint,
    test_tree_sum_feeds_the_update)

NADAM = Spec(
    "nadam", mx.optimizer.Nadam, N.OracleNadam,
    kw=dict(learning_rate=0.001, wd=1e-4),
    base=dict(learning_rate=0.001, wd=0.05),
    # clip_gradient 0 is on (step clips at 0): with wd > 0 the weight decay alone drives the update
    variants=[dict(rescale_grad=0.14), dict(clip_gradient=0.3), dict(clip_gradient=0.0), dict(learning_rate=0.01),
              dict(beta1=0.5), dict(beta2=0.8), dict(epsilon=1e-2), dict(schedule_decay=0.5), dict(wd=0.0)],
    lp_kw=dict(learning_rate=0.001, wd=1e-3, rescale_grad=0.5, clip_gradient=0.6, beta1=0.5),
    updater_kw=dict(learning_rate=0.002, wd=1e-2, clip_gradient=0.3, beta1=0.5, beta2=0.9, schedule_decay=0.008),
    python_kw=dict(learning_rate=0.001, wd=1e-3, clip_gradient=0.01, beta1=0.5),
    multi_kw=dict(learning_rate=0.001, wd=1e-4, rescale_grad=0.5, clip_gradient=0.7, beta1=0.5))


@pytest.fixture
def spec():
    return NADAM


SIZES = [5, 1000, 4099, 1 << 14, 33, 70001]


def _grads(rng, sizes):
    return [rng.uniform(-1, 1, e).astype(np.float32) for e in sizes]


def test_unsorted_keys_advance_the_product_in_sorted_order():
    """a multi-key pushpull whose keys arrive unsorted is updated in sorted key order (GroupKVPairs), and so is the
    schedule product: bit for bit against the oracle store, which sorts the same way, and different from the updates
    in the order of the call.  The store's m_schedule equals the oracle's after every step, and so does the Python
    optimizer's, which is read back after each push.  String keys sort by their order of first use (init)."""
    for str_keys in (False, True):
        rng = np.random.default_rng(5 + str_keys)
        ids = list(range(len(SIZES)))
        keys = ["k%d" % i for i in ids] if str_keys else ids       # "k0" < "k1" < ...: sorted = init order
        w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in SIZES]
        kv = mx.kv.create("device")
        kv.init(keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
        kv.set_optimizer(mx.optimizer.Nadam(**NADAM.kw))
        okv = O.OracleKVStore("device")
        okv.init(keys, [w.copy() for w in w0])
        okv.set_optimizer(N.OracleNadam(**NADAM.kw))
        in_call = N.OracleNadam(**NADAM.kw)            # the same updates in the order the call lists the keys
        cw = [w.copy() for w in w0]
        order = [3, 0, 5, 1, 4, 2]
        outs = [mx.nd.empty((e,), mx.gpu(0)) for e in SIZES]
        for s in range(3):
            grads = _grads(rng, SIZES)
            kv.pushpull([keys[i] for i in order], [mx.nd.array(grads[i], mx.gpu(0)) for i in order],
                        out=[outs[i] for i in order])
            okv.push(keys, [[g] for g in grads])
            for i in order:
                in_call.update(i, cw[i], grads[i])
            _check(okv, keys, outs, "str=%s step %d" % (str_keys, s))
            assert kv._get_scalar("m_schedule") == okv.optimizer.m_schedule
            assert kv._optimizer.m_schedule == okv.optimizer.m_schedule
        assert any(not np.array_equal(outs[i].asnumpy(), cw[i]) for i in ids), "the call order made no difference"


def test_plan_replay_and_deferred_queue_keep_the_call_order():
    """a replayed launch plan gives the bits of a fresh store at every step; with the deferred queue on, per-key calls
    with reversed priorities are issued at once, in call order -- the same bits as with the queue off, and no call
    was deferred (reordering by priority would reorder the schedule product)"""
    rng = np.random.default_rng(77)
    keys = list(range(len(SIZES)))
    w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in SIZES]
    steps = [_grads(rng, SIZES) for _ in range(4)]

    def run(mode):
        kv = mx.kv.create("device")
        kv.init(keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
        kv.set_optimizer(mx.optimizer.Nadam(**NADAM.kw))
        outs = [mx.nd.empty((e,), mx.gpu(0)) for e in SIZES]
        gdev = [mx.nd.empty((e,), mx.gpu(0)) for e in SIZES]
        if mode == "deferred":
            kv.set_deferred(True)
        res = []
        for grads in steps:
            for d, g in zip(gdev, grads):
                d[:] = g
            if mode == "fresh":                       # new arrays every step: nothing to replay
                kv.pushpull(keys, [mx.nd.array(g, mx.gpu(0)) for g in grads], out=outs)
            elif mode == "replay":
                kv.pushpull(keys, gdev, out=outs)
            else:
                for i in keys:
                    kv.pushpull(i, gdev[i], out=outs[i], priority=i)     # the queue would issue the last key first
            res.append([o.asnumpy() for o in outs])
        return kv, res

    kv_f, fresh = run("fresh")
    kv_r, replay = run("replay")
    assert kv_r.plan_hits() >= 2
    kv_d, deferred = run("deferred")
    assert kv_d.deferred_batches() == 0, "a Nadam call was deferred"
    okv = O.OracleKVStore("device")
    okv.init(keys, [w.copy() for w in w0])
    okv.set_optimizer(N.OracleNadam(**NADAM.kw))
    for s, grads in enumerate(steps):
        okv.push(keys, [[g] for g in grads])
        for k in keys:
            want = np.empty(SIZES[k], np.float32)
            okv.pull(k, want)
            assert_bits_equal(fresh[s][k], want, "fresh step %d key %d" % (s, k))
            assert_bits_equal(replay[s][k], want, "replay step %d key %d" % (s, k))
            assert_bits_equal(deferred[s][k], want, "deferred step %d key %d" % (s, k))
    for kv in (kv_f, kv_r, kv_d):
        assert kv._get_scalar("m_schedule") == okv.optimizer.m_schedule


def test_checkpoint_and_re_sent_optimizer_keep_the_product():
    """save_optimizer_states(dump_optimizer=True) pickles the product where the store's updates took it and a store
    that loads the file continues bit for bit; re-sending the current optimizer (rescale_grad per batch) keeps the
    product, a new optimizer object starts from its own"""
    rng = np.random.default_rng(8)
    keys = [0, 1, 2]
    sizes = [1000, 33, 70001]
    w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in sizes]
    kv = mx.kv.create("device")
    kv.init(keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
    opt = mx.optimizer.Nadam(**NADAM.kw)
    kv.set_optimizer(opt)
    okv = O.OracleKVStore("device")
    okv.init(keys, [w.copy() for w in w0])
    okv.set_optimizer(N.OracleNadam(**NADAM.kw))
    outs = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]

    def step(store, outs, rescale=None):
        grads = _grads(rng, sizes)
        if rescale is not None:
            store._optimizer.rescale_grad = okv.optimizer.rescale_grad = rescale
            store.set_optimizer(store._optimizer)
        store.pushpull(keys, [mx.nd.array(g, mx.gpu(0)) for g in grads], out=outs)
        okv.push(keys, [[g] for g in grads])
        _check(okv, keys, outs, "step")

    step(kv, outs)
    step(kv, outs, rescale=0.5)                      # re-sent: the product continues
    assert opt.m_schedule == okv.optimizer.m_schedule < 0.1
    d = tempfile.mkdtemp(prefix="mxkv_nadam_")
    f = os.path.join(d, "states")
    kv.save_optimizer_states(f, dump_optimizer=True)
    with open(f, "rb") as fin:
        assert pickle.load(fin)["optimizer"].m_schedule == okv.optimizer.m_schedule
    kv2 = mx.kv.create("device")
    kv2.init(keys, [mx.nd.array(o.asnumpy(), mx.gpu(0)) for o in outs])
    kv2.set_optimizer(mx.optimizer.Nadam(**NADAM.kw))
    assert kv2._get_scalar("m_schedule") == 1.0
    kv2.load_optimizer_states(f)
    os.remove(f)
    os.rmdir(d)
    assert kv2._get_scalar("m_schedule") == okv.optimizer.m_schedule
    outs2 = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]
    for _ in range(2):
        step(kv2, outs2)
    _check_states(kv2, okv, keys, "after reload")
    assert all(_count(kv2, k) == 4 for k in keys)
    fresh = mx.optimizer.Nadam(**NADAM.kw)
    fresh.m_schedule = 0.25
    kv2.set_optimizer(fresh)
    assert kv2._get_scalar("m_schedule") == 0.25


@pytest.mark.multigpu
def test_native_updaters_of_two_devices_share_the_product():
    """Trainer(update_on_kvstore=False) keeps one updater per device over ONE optimizer: the reference's per-device
    update counts (Optimizer._set_current_context) and one m_schedule, advanced by device 0's pairs in pair order,
    then device 1's.  Each device's weights against an oracle per device that hands the product on"""
    if mx.num_gpus() < 2:
        pytest.skip("needs 2 GPUs")
    shapes = [(64,), (3, 5), (1000,), (7,)]
    rng = np.random.default_rng(6)
    w0 = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
    opt = mx.optimizer.create("nadam", **NADAM.updater_kw)
    upd = [mx.optimizer.get_updater(opt) for _ in range(2)]
    assert all(isinstance(u, mx.optimizer.NativeUpdater) for u in upd)
    weights = [[mx.nd.array(w, mx.gpu(d)) for w in w0] for d in range(2)]
    oracles = [N.OracleNadam(**NADAM.updater_kw) for _ in range(2)]
    ow = [[w.copy() for w in w0] for _ in range(2)]
    idx = [2, 0, 3, 1]                                # pair order, not sorted
    m = 1.0
    for step in range(3):
        for d in range(2):
            g = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
            upd[d](idx, [mx.nd.array(g[k], mx.gpu(d)) for k in idx], [weights[d][k] for k in idx])
            oracles[d].m_schedule = m
            for k in idx:
                oracles[d].update(k, ow[d][k], g[k])
            m = oracles[d].m_schedule
            assert opt.m_schedule == m, (step, d)
            for k in idx:
                assert_bits_equal(weights[d][k].asnumpy(), ow[d][k], "device %d step %d index %d" % (d, step, k))
    assert opt._all_index_update_counts[0][0] == opt._all_index_update_counts[1][0] == 3


@pytest.mark.parametrize("mode", ["update_on_kvstore", "local_update", "no_kvstore"])
def test_trainer_modes_match_the_oracle_and_the_python_step(mode):
    """Trainer(params, 'nadam') with update_on_kvstore True and False (and without a store): bit for bit against the
    oracle stepping the parameters in order, and the optimizer's m_schedule equal to the oracle's and to the one a
    use_fused_step=False Trainer's Python step reaches"""
    import torch
    model, pmodel = _net(), _net()
    params = list(model.parameters())
    targs = {"update_on_kvstore": dict(kvstore="device", update_on_kvstore=True),
             "local_update": dict(kvstore="device", update_on_kvstore=False),
             "no_kvstore": dict(kvstore=None)}[mode]
    trainer = mx.Trainer(params, "nadam", dict(NADAM.kw), **targs)
    ptrainer = mx.Trainer(list(pmodel.parameters()), "nadam", dict(NADAM.kw, use_fused_step=False), kvstore="device")
    ref_w = [p.detach().cpu().numpy().copy().reshape(-1) for p in params]
    opt = N.OracleNadam(**NADAM.kw)
    torch.manual_seed(9)
    for step in range(3):
        x = torch.randn(32, 64, device="cuda")
        for m, t in ((model, trainer), (pmodel, ptrainer)):
            m.zero_grad(set_to_none=False)
            m(x).square().mean().backward()
        grads = [p.grad.detach().cpu().numpy().copy().reshape(-1) for p in params]
        trainer.step(32)
        ptrainer.step(32)
        torch.cuda.synchronize()
        opt.rescale_grad = 1.0 / 32
        for i, (w, g) in enumerate(zip(ref_w, grads)):
            opt.update(i, w, g)
        for i, (p, w) in enumerate(zip(params, ref_w)):
            assert _bits_equal32(p.detach().cpu().numpy().reshape(-1), w), (mode, step, i)
        assert trainer._optimizer.m_schedule == opt.m_schedule == ptrainer._optimizer.m_schedule, (mode, step)
        for pa, pb in zip(model.parameters(), pmodel.parameters()):
            np.testing.assert_allclose(pb.detach().cpu().numpy(), pa.detach().cpu().numpy(), rtol=1e-5, atol=1e-6)


def test_aggregating_updater_steps_the_pairs_dtype_by_dtype():
    """an optimizer with aggregate_num > 1: the reference's updater groups the pairs by dtype, in the order the dtypes
    first appear, before it steps them (updater.py:65-80), and the schedule product follows that order -- float16
    pairs (multi_precision: step on the fp32 master) first here, then the float32 ones"""
    shapes = [(64,), (3, 5), (1000,), (7,)]
    dtypes = [np.float16, np.float32, np.float16, np.float32]
    rng = np.random.default_rng(11)
    w32 = [rng.uniform(-1, 1, s).astype(dt).astype(np.float32) for s, dt in zip(shapes, dtypes)]
    weights = [mx.nd.array(w.astype(dt), mx.gpu(0), dtype=dt) for w, dt in zip(w32, dtypes)]
    opt = mx.optimizer.Nadam(aggregate_num=4, multi_precision=True, **NADAM.updater_kw)
    upd = mx.optimizer.get_updater(opt)
    oopt = N.OracleNadam(**NADAM.updater_kw)
    ow = [w.copy() for w in w32]
    for step in range(2):
        g = [rng.uniform(-1, 1, s).astype(dt) for s, dt in zip(shapes, dtypes)]
        upd(list(range(4)), [mx.nd.array(x, mx.gpu(0), dtype=dt) for x, dt in zip(g, dtypes)], weights)
        for k in (0, 2, 1, 3):
            oopt.update(k, ow[k], g[k].astype(np.float32))
        assert opt.m_schedule == oopt.m_schedule, step
        for k, dt in enumerate(dtypes):
            assert_bits_equal(weights[k].asnumpy(), ow[k].astype(dt), "step %d index %d" % (step, k))
