"""Placement edge cases of the single-process multi-GPU shape: which GPUs take part, where the stored value
and the optimizer state live, what happens when the set of devices changes between calls, outputs on GPUs
that did not push, host and device values mixed, more destinations than one launch can address, in-place
forms.  Everything is compared bit-for-bit with the oracle.  On hardware these need several GPUs (skipped
otherwise); the CPU suite runs them on 8 simulated GPUs (tests/test_sim_host_logic.py)."""
import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

import mxnet_b200 as mx
from oracle import oracle as O


import os as _os
_EXTRA = int(_os.environ.get("MXKV_FUZZ_SEEDS", "0"))     # more random walks on demand (soak runs on the simulator)


def _need(n):
    if mx.num_gpus() < n:
        pytest.skip("needs %d GPUs" % n)


def _bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _rng(seed):
    return np.random.default_rng(777 + seed)


@pytest.mark.parametrize("E", [1000, 300007])          # one-shot and two-shot sizes
def test_subset_of_gpus_and_outputs_elsewhere(E):
    """values pushed from GPUs 1 and 3 only; outputs on 0, 2 (not participants) and on the host"""
    _need(4)
    rng = _rng(E)
    w0 = rng.uniform(0, 1, E).astype(np.float32)
    kw = dict(learning_rate=0.1, momentum=0.9, wd=1e-4)
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w0, mx.gpu(2)))
    kv.set_optimizer(mx.optimizer.SGD(**kw))
    okv = O.OracleKVStore("device"); okv.init(0, w0.copy()); okv.set_optimizer(O.OracleOptimizer("sgd", **kw))
    outs = [mx.nd.empty((E,), mx.gpu(0)), mx.nd.empty((E,), mx.gpu(2)), mx.nd.empty((E,), mx.cpu()),
            mx.nd.empty((E,), mx.gpu(3))]
    want = np.empty(E, np.float32)
    for step in range(3):
        g = [rng.uniform(-1, 1, E).astype(np.float32) for _ in range(2)]
        kv.pushpull(0, [mx.nd.array(g[0], mx.gpu(1)), mx.nd.array(g[1], mx.gpu(3))], out=outs)
        okv.push(0, g); okv.pull(0, want)
        for o in outs:
            assert _bits_equal(o.asnumpy(), want), (step, o.context)


def test_device_set_changes_between_calls():
    """2 GPUs, then 4, then 1, then 3 different ones: the stored value and the (sharded or replicated) Adam
    state follow -- the reference keeps them on one root and does not care; here they are re-gathered."""
    _need(4)
    E = 300007
    rng = _rng(1)
    w0 = rng.uniform(0, 1, E).astype(np.float32)
    kw = dict(learning_rate=0.01, wd=1e-3)
    kv = mx.kv.create("device")
    kv.init("w", mx.nd.array(w0, mx.gpu(0)))
    kv.set_optimizer(mx.optimizer.Adam(**kw))
    okv = O.OracleKVStore("device"); okv.init("w", w0.copy()); okv.set_optimizer(O.OracleOptimizer("adam", **kw))
    want = np.empty(E, np.float32)
    for devs in ([0, 1], [0, 1, 2, 3], [2], [3, 1, 0], [0, 1]):
        g = [rng.uniform(-1, 1, E).astype(np.float32) for _ in devs]
        outs = [mx.nd.empty((E,), mx.gpu(d)) for d in devs]
        kv.pushpull("w", [mx.nd.array(x, mx.gpu(d)) for x, d in zip(g, devs)], out=outs)
        okv.push("w", g); okv.pull("w", want)
        for o in outs:
            assert _bits_equal(o.asnumpy(), want), devs
    pulled = mx.nd.empty((E,), mx.gpu(3))
    kv.pull("w", out=pulled)
    assert _bits_equal(pulled.asnumpy(), want)


def test_host_and_device_values_mixed():
    """one value in host memory, the others on two GPUs: staged onto the root, summed in push order"""
    _need(2)
    E = 50003
    rng = _rng(2)
    kv = mx.kv.create("device")
    kv.init(5, mx.nd.zeros((E,), mx.gpu(0)))
    g = [rng.uniform(-1, 1, E).astype(np.float32) for _ in range(3)]
    vals = [mx.nd.array(g[0], mx.gpu(1)), mx.nd.array(g[1], mx.cpu()), mx.nd.array(g[2], mx.gpu(0))]
    out = mx.nd.empty((E,), mx.gpu(1))
    kv.pushpull(5, vals, out=out)
    assert _bits_equal(out.asnumpy(), O.sum_device(g))
    host_out = mx.nd.empty((E,), mx.cpu())
    kv.pull(5, out=host_out)
    assert _bits_equal(host_out.asnumpy(), O.sum_device(g))


def test_more_outputs_than_one_launch_addresses():
    """40 outputs of one key (kMaxOut is 24): the surplus is served by copies after the launch"""
    _need(2)
    E = 4099
    rng = _rng(3)
    devs = list(range(min(mx.num_gpus(), 4)))
    kv = mx.kv.create("device")
    kv.init(1, mx.nd.zeros((E,), mx.gpu(0)))
    g = [rng.uniform(-1, 1, E).astype(np.float32) for _ in devs]
    outs = [mx.nd.empty((E,), mx.gpu(devs[i % len(devs)])) for i in range(40)]
    kv.pushpull(1, [mx.nd.array(x, mx.gpu(d)) for x, d in zip(g, devs)], out=outs)
    want = O.sum_device(g)
    for i, o in enumerate(outs):
        assert _bits_equal(o.asnumpy(), want), i


@pytest.mark.parametrize("E", [1000, 300007])
def test_in_place_forms(E):
    """pushpull(key, values) overwrites the values with the result: one-shot keys must not be written while
    a peer still reads them (served by a copy afterwards), two-shot keys write disjoint shards directly"""
    _need(2)
    rng = _rng(4 + E)
    devs = list(range(min(mx.num_gpus(), 4)))
    kv = mx.kv.create("device")
    kv.init(["a", "b"], [mx.nd.zeros((E,), mx.gpu(0))] * 2)
    ga = [rng.uniform(-1, 1, E).astype(np.float32) for _ in devs]
    gb = [rng.uniform(-1, 1, E).astype(np.float32) for _ in devs]
    va = [mx.nd.array(x, mx.gpu(d)) for x, d in zip(ga, devs)]
    vb = [mx.nd.array(x, mx.gpu(d)) for x, d in zip(gb, devs)]
    kv.pushpull(["a", "b"], [va, vb])
    for v in va:
        assert _bits_equal(v.asnumpy(), O.sum_device(ga))
    for v in vb:
        assert _bits_equal(v.asnumpy(), O.sum_device(gb))
    # the same arrays pushed for BOTH keys and pulled in place (the reference's tests do this): every reduce of
    # the call happens before any pull (kvstore_local.h:358-365)
    shared = [mx.nd.array(x, mx.gpu(d)) for x, d in zip(ga, devs)]
    kv.pushpull(["a", "b"], [shared, shared])
    for v in shared:
        assert _bits_equal(v.asnumpy(), O.sum_device(ga))


def test_many_keys_many_gpus_layerwise_and_plain_mixed_dtypes():
    """fp32 and bf16 keys in one call (two launch classes), 8 GPUs if there are that many, LAMB with the
    device-side overflow skip spanning both classes"""
    _need(2)
    devs = list(range(min(mx.num_gpus(), 8)))
    rng = _rng(5)
    shapes = [(64,), (513, 9), (1 << 18,), (300, 1000)]
    kw = dict(learning_rate=0.01, wd=0.01)
    kv = mx.kv.create("device")
    w32 = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
    wbf = [O.f32_to_bf16(rng.uniform(-1, 1, s).astype(np.float32)) for s in shapes]
    keys32 = ["f%d" % i for i in range(len(shapes))]
    keysbf = ["h%d" % i for i in range(len(shapes))]
    kv.init(keys32, [mx.nd.array(w, mx.gpu(0)) for w in w32])
    kv.init(keysbf, [mx.nd.array(w, mx.gpu(0), dtype="bfloat16") for w in wbf])
    kv.set_optimizer(mx.optimizer.LAMB(skip_nonfinite=True, multi_precision=True, **kw))
    o32 = [[mx.nd.empty(s, mx.gpu(d)) for d in devs] for s in shapes]
    obf = [[mx.nd.empty(s, mx.gpu(d), dtype="bfloat16") for d in devs] for s in shapes]
    oopt = O.OracleOptimizer("lamb", norm_mode="f64", **kw)
    ref32 = [w.copy() for w in w32]
    for step in range(3):
        g32 = [[rng.uniform(-1, 1, s).astype(np.float32) for _ in devs] for s in shapes]
        gbf = [[O.f32_to_bf16(rng.uniform(-1, 1, s).astype(np.float32)) for _ in devs] for s in shapes]
        overflow = step == 1
        if overflow:
            gbf[0][-1][3] = O.f32_to_bf16(np.array([np.inf], np.float32))[0]     # a bf16 key poisons the push
        kv.pushpull(keys32 + keysbf,
                    [[mx.nd.array(g, mx.gpu(d)) for g, d in zip(gs, devs)] for gs in g32] +
                    [[mx.nd.array(g, mx.gpu(d), dtype="bfloat16") for g, d in zip(gs, devs)] for gs in gbf],
                    out=o32 + obf)
        assert kv.overflow() == overflow
        for k in range(len(shapes)):
            if not overflow:
                oopt.update(k, ref32[k], O.sum_device(g32[k]).reshape(shapes[k]))
            first = o32[k][0].asnumpy()
            np.testing.assert_allclose(first, ref32[k], rtol=2e-6, atol=2e-7, err_msg=str((step, k)))
            for o in o32[k][1:]:
                assert _bits_equal(o.asnumpy(), first)
            hb = obf[k][0].asnumpy(raw=True)
            for o in obf[k][1:]:
                assert np.array_equal(o.asnumpy(raw=True), hb)


def test_row_sparse_device_set_changes():
    """row_sparse push from GPUs 0 and 1, then from GPU 2 alone, then from the host; pulls to every device"""
    _need(3)
    rows, L, nnz = 500, 8, 60
    rng = _rng(6)
    shape = (rows, L)
    w0 = rng.uniform(0, 1, shape).astype(np.float32)
    kw = dict(learning_rate=0.1, momentum=0.9, wd=1e-3, lazy_update=True)
    kv = mx.kv.create("device")
    kv.init("e", mx.nd.row_sparse_array(w0, ctx=mx.gpu(0)))
    kv.set_optimizer(mx.optimizer.SGD(**kw))
    okv = O.OracleKVStore("device"); okv.init("e", O.RowSparse.from_dense(w0))
    okv.set_optimizer(O.OracleOptimizer("sgd", **kw))

    def rsp():
        idx = np.sort(rng.choice(rows, nnz, replace=False)).astype(np.int64)
        return idx, rng.uniform(-1, 1, (nnz, L)).astype(np.float32)

    for ctxs in ([mx.gpu(0), mx.gpu(1)], [mx.gpu(2)], [mx.cpu()], [mx.gpu(1), mx.gpu(2), mx.gpu(0)]):
        parts = [rsp() for _ in ctxs]
        kv.push("e", [mx.nd.row_sparse_array((v, i), shape=shape, ctx=c) for (i, v), c in zip(parts, ctxs)])
        okv.push("e", [O.RowSparse(i, v, shape) for i, v in parts])
        ids = rng.integers(0, rows, 100).astype(np.int64)
        want = O.sparse_retain(okv.local["e"], O.unique(ids))
        for c in (mx.gpu(0), mx.gpu(2), mx.cpu()):
            out = mx.nd.zeros(shape, c, stype="row_sparse")
            kv.row_sparse_pull("e", out=out, row_ids=mx.nd.array(ids, c, dtype=np.int64))
            assert np.array_equal(out.indices.asnumpy(), want.indices), (ctxs, c)
            assert _bits_equal(out.data.asnumpy(), want.data.reshape(-1, L)), (ctxs, c)
        dense = mx.nd.empty(shape, mx.gpu(1))
        kv.pull("e", out=dense, ignore_sparse=False)
        assert _bits_equal(dense.asnumpy(), okv.local["e"].todense())


def test_updater_callback_with_changing_devices():
    """test_kvstore.py:222-274 generalised: the Python updater sees the merged value on whatever GPU reduced"""
    _need(3)
    shape = (6, 5)
    kv = mx.kv.create("device")
    kv.init(9, mx.nd.zeros(shape, mx.gpu(1)))
    calls = []

    def updater(key, recv, local):
        calls.append((key, recv.context.device_id, local.context.device_id))
        local += recv
    kv._set_updater(updater)
    total = 0
    for devs in ([0, 1, 2], [2], [1, 0]):
        kv.push(9, [mx.nd.ones(shape, mx.gpu(d)) * (d + 1) for d in devs])
        total += sum(d + 1 for d in devs)
        for d in (0, 1, 2):
            o = mx.nd.empty(shape, mx.gpu(d))
            kv.pull(9, out=o)
            assert np.all(o.asnumpy() == total), (devs, d)
    assert len(calls) == 3 and all(c[0] == 9 for c in calls)


def test_compression_with_changing_devices():
    _need(3)
    E, thr = 9000, 0.5
    rng = _rng(8)
    kv = mx.kv.create("device")
    kv.set_gradient_compression({"type": "2bit", "threshold": thr})
    kv.init(0, mx.nd.zeros((E,), mx.gpu(0)))
    residual = {}
    for devs in ([0, 1], [0, 1, 2], [1]):
        g = [rng.uniform(-1, 1, E).astype(np.float32) for _ in devs]
        outs = [mx.nd.empty((E,), mx.gpu(d)) for d in (0, 1, 2)]
        kv.pushpull(0, [mx.nd.array(x, mx.gpu(d)) for x, d in zip(g, devs)], out=outs)
        # residuals are kept per pushed-value slot (comm.h:575-580), not per device
        deq = []
        for slot, x in enumerate(g):
            r = residual.setdefault(slot, np.zeros(E, np.float32))
            deq.append(O.dequantize_2bit(O.quantize_2bit(x, r, thr), E, thr))
        want = O.sum_device(deq)
        for o in outs:
            assert _bits_equal(o.asnumpy(), want), devs


def test_checkpoint_after_device_set_change(tmp_path):
    """optimizer states saved while sharded over 4 GPUs, loaded into a store that then runs on 2"""
    _need(4)
    E = 300007
    rng = _rng(9)
    w0 = rng.uniform(0, 1, E).astype(np.float32)
    kw = dict(learning_rate=0.01, wd=1e-3)
    grads = [[rng.uniform(-1, 1, E).astype(np.float32) for _ in range(4)] for _ in range(4)]
    okv = O.OracleKVStore("device"); okv.init(0, w0.copy()); okv.set_optimizer(O.OracleOptimizer("adam", **kw))
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w0, mx.gpu(0)))
    kv.set_optimizer(mx.optimizer.Adam(**kw))
    for g in grads[:2]:
        kv.push(0, [mx.nd.array(x, mx.gpu(d)) for d, x in enumerate(g)])
        okv.push(0, g)
    f = str(tmp_path / "adam.states")
    kv.save_optimizer_states(f, dump_optimizer=True)      # the optimizer carries the update counts
    mid = mx.nd.empty((E,), mx.gpu(0)); kv.pull(0, out=mid)
    kv2 = mx.kv.create("device")
    kv2.init(0, mx.nd.array(mid.asnumpy(), mx.gpu(1)))
    kv2.set_optimizer(mx.optimizer.Adam(**kw))
    kv2.load_optimizer_states(f)
    for g in grads[2:]:
        kv2.push(0, [mx.nd.array(g[0] + g[1], mx.gpu(1)), mx.nd.array(g[2] + g[3], mx.gpu(3))])
        okv.push(0, [g[0] + g[1], g[2] + g[3]])
    out = mx.nd.empty((E,), mx.gpu(2)); kv2.pull(0, out=out)
    want = np.empty(E, np.float32); okv.pull(0, want)
    assert _bits_equal(out.asnumpy(), want)


def test_call_level_rules():
    """rules of one call: different device sets for different keys, too many values, duplicate keys"""
    _need(2)
    kv = mx.kv.create("device")
    kv.init([0, 1], [mx.nd.zeros((8,), mx.gpu(0))] * 2)
    # key 0 from GPUs {0,1}, key 1 from GPU {0}: different reduction sites in one call are served one group
    # after the other (every key has its own merge buffer in the reference, so it accepts this too)
    outs = [mx.nd.empty((8,), mx.gpu(1)), mx.nd.empty((8,), mx.gpu(0))]
    kv.pushpull([0, 1], [[mx.nd.ones((8,), mx.gpu(0)), mx.nd.ones((8,), mx.gpu(1)) * 2], [mx.nd.ones((8,), mx.gpu(0)) * 5]],
                out=outs)
    assert np.all(outs[0].asnumpy() == 3) and np.all(outs[1].asnumpy() == 5)
    with pytest.raises(mx.MXNetError):       # more values than one launch addresses
        kv.push(0, [mx.nd.ones((8,), mx.gpu(0))] * 17)
    # the same key twice in one list: the values are summed (GroupKVPairs, kvstore_local.h:440-469)
    kv2 = mx.kv.create("device")
    kv2.init(3, mx.nd.zeros((8,), mx.gpu(0)))
    kv2.push([3, 3, 3], [mx.nd.ones((8,), mx.gpu(0)) * 2, mx.nd.ones((8,), mx.gpu(1)), mx.nd.ones((8,), mx.gpu(0))])
    o = mx.nd.empty((8,), mx.gpu(1)); kv2.pull(3, out=o)
    assert np.all(o.asnumpy() == 4)


@pytest.mark.parametrize("dtype", [np.float64, np.int32, np.int64, np.uint8, np.float16])
def test_other_dtypes_across_gpus(dtype):
    """ElementwiseSum accepts every MSHADOW_TYPE_SWITCH type (ndarray_function-inl.h:443-489); fp16 rounds every
    add to half like mshadow's half_t"""
    _need(2)
    devs = list(range(min(mx.num_gpus(), 4)))
    E = 70001
    rng = _rng(10)
    if np.issubdtype(dtype, np.floating):
        vals = [rng.uniform(-1, 1, E).astype(dtype) for _ in devs]
    else:
        vals = [rng.integers(0, 50, E).astype(dtype) for _ in devs]
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(np.zeros(E, dtype), mx.gpu(0), dtype=dtype))
    outs = [mx.nd.empty((E,), mx.gpu(d), dtype=dtype) for d in devs]
    kv.pushpull(0, [mx.nd.array(v, mx.gpu(d), dtype=dtype) for v, d in zip(vals, devs)], out=outs)
    if dtype == np.float16:
        acc = vals[0].copy()
        for v in vals[1:]:
            acc = (acc.astype(np.float32) + v.astype(np.float32)).astype(np.float16)
        want = acc
    else:
        want = vals[0].copy()
        for v in vals[1:]:
            want = (want + v).astype(dtype)
    for o in outs:
        assert np.array_equal(o.asnumpy(), want)


@pytest.mark.parametrize("optname,kw", [
    (None, {}),
    ("sgd", dict(learning_rate=0.1, momentum=0.9, wd=1e-4)),
    ("adam", dict(learning_rate=0.01, wd=1e-3)),
    ("lamb", dict(learning_rate=0.01, wd=0.01)),
])
def test_host_resident_key_lists(optname, kw, monkeypatch):
    """kv.create('local')-style use with whole key lists in host memory: small and large keys mixed (the large
    ones go through the segmented H2D / kernel / D2H pipeline), in place and out of place, several steps"""
    monkeypatch.setenv("MXKV_B200_HOST_SEG_ELEMS", str(1 << 16))
    shapes = [(7,), (300, 1000), (64,), ((1 << 18) + 37,), (5, 5)]
    keys = ["k%d" % i for i in range(len(shapes))]
    n = 3
    rng = _rng(11)
    w0 = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]
    kv = mx.kv.create("local")
    kv.init(keys, [mx.nd.array(w) for w in w0])
    okv = O.OracleKVStore("local"); okv.init(keys, [w.copy() for w in w0])
    oopt = None
    if optname:
        kv.set_optimizer(mx.optimizer.create(optname, **kw))
        oopt = O.OracleOptimizer(optname, **(dict(kw, norm_mode="f64") if optname == "lamb" else kw))
        okv.set_optimizer(oopt)
    outs = [mx.nd.empty(s, mx.cpu_pinned()) for s in shapes]
    for step in range(3):
        grads = [[rng.uniform(-1, 1, s).astype(np.float32) for _ in range(n)] for s in shapes]
        vals = [[mx.nd.array(g, mx.cpu_pinned() if (step + j) % 2 else mx.cpu()) for j, g in enumerate(gs)]
                for gs in grads]
        if step == 1 and optname is None:
            kv.pushpull(keys, vals)                      # in place: every value array receives the sum
            okv.push(keys, grads)
            for k, vs in enumerate(vals):
                want = np.empty(shapes[k], np.float32); okv.pull(keys[k], want)
                for v in vs:
                    assert _bits_equal(v.asnumpy(), want), (step, k)
            continue
        kv.pushpull(keys, vals, out=outs)
        okv.push(keys, grads)
        for k in range(len(shapes)):
            want = np.empty(shapes[k], np.float32); okv.pull(keys[k], want)
            if optname == "lamb":
                np.testing.assert_allclose(outs[k].asnumpy(), want, rtol=2e-6, atol=2e-7)
            else:
                assert _bits_equal(outs[k].asnumpy(), want), (optname, step, k)


@pytest.mark.parametrize("seed", list(range(12 + _EXTRA)))
def test_randomized_call_sequences(seed):
    """A random walk over the store's states: keys of one-shot and two-shot size, values pushed from random
    subsets of the GPUs (or the host), pushes and fused pushpulls interleaved with pulls to random devices, a
    fused optimizer that is switched on part-way -- compared with the oracle after every call."""
    _need(2)
    ngpu = min(mx.num_gpus(), 8)
    rng = _rng(1000 + seed)
    sizes = [int(x) for x in rng.choice([5, 640, 4099, 70001, 300007], size=3, replace=False)]
    keys = list(range(len(sizes)))
    w0 = [rng.uniform(-1, 1, e).astype(np.float32) for e in sizes]
    kv = mx.kv.create("device")
    okv = O.OracleKVStore("device")
    kv.init(keys, [mx.nd.array(w, mx.gpu(int(rng.integers(ngpu)))) for w in w0])
    okv.init(keys, [w.copy() for w in w0])
    optname = [None, "sgd", "adam"][seed % 3]
    kw = {"sgd": dict(learning_rate=0.05, momentum=0.9, wd=1e-3), "adam": dict(learning_rate=0.01, wd=1e-3)}.get(optname)
    switch_at = int(rng.integers(0, 4))

    def ctx_of(d):
        return mx.cpu() if d < 0 else mx.gpu(d)

    def check(ks):
        for k in ks:
            d = int(rng.integers(-1, ngpu))
            o = mx.nd.empty((sizes[k],), ctx_of(d))
            kv.pull(k, out=o)
            want = np.empty(sizes[k], np.float32)
            okv.pull(k, want)
            assert _bits_equal(o.asnumpy(), want), ("pull", seed, k, d)

    for step in range(10):
        if optname and step == switch_at:
            kv.set_optimizer(mx.optimizer.create(optname, **kw))
            okv.set_optimizer(O.OracleOptimizer(optname, **kw))
        nk = int(rng.integers(1, len(keys) + 1))
        ks = sorted(int(x) for x in rng.choice(keys, size=nk, replace=False))
        ndev = int(rng.integers(1, ngpu + 1))
        devs = [int(x) for x in rng.choice(ngpu, size=ndev, replace=False)]
        if rng.random() < 0.2:
            devs = [-1] + devs[: max(0, len(devs) - 1)]          # one value from the host
        grads = [[rng.uniform(-1, 1, sizes[k]).astype(np.float32) for _ in devs] for k in ks]
        vals = [[mx.nd.array(g, ctx_of(d)) for g, d in zip(gs, devs)] for gs in grads]
        mode = rng.choice(["push", "pushpull", "inplace"]) if optname is None or step < switch_at else \
            rng.choice(["push", "pushpull"])
        if mode == "push":
            kv.push(ks, vals)
            okv.push(ks, grads)
        elif mode == "pushpull":
            odevs = [int(x) for x in rng.choice(ngpu, size=int(rng.integers(1, ngpu + 1)), replace=False)]
            outs = [[mx.nd.empty((sizes[k],), mx.gpu(d)) for d in odevs] for k in ks]
            kv.pushpull(ks, vals, out=outs)
            okv.push(ks, grads)
            for k, oo in zip(ks, outs):
                want = np.empty(sizes[k], np.float32)
                okv.pull(k, want)
                for o in oo:
                    assert _bits_equal(o.asnumpy(), want), ("pushpull", seed, step, k)
        else:
            kv.pushpull(ks, vals)
            okv.push(ks, grads)
            for k, vs in zip(ks, vals):
                want = np.empty(sizes[k], np.float32)
                okv.pull(k, want)
                for v in vs:
                    assert _bits_equal(v.asnumpy(), want), ("inplace", seed, step, k)
        check(ks)


_FUZZ_OPTS = [
    (None, {}),
    ("sgd", dict(learning_rate=0.05, wd=1e-3, rescale_grad=0.5)),
    ("sgd", dict(learning_rate=0.05, momentum=0.9, wd=1e-3, clip_gradient=0.7)),
    ("adam", dict(learning_rate=0.01, wd=1e-3)),
    ("adamw", dict(learning_rate=0.01, wd=0.05)),
    ("test", dict(learning_rate=0.1, wd=0.01, rescale_grad=0.5)),
    ("lamb", dict(learning_rate=0.01, wd=0.01)),
    ("lans", dict(learning_rate=0.01, wd=0.01)),
    ("lars", dict(learning_rate=0.1, momentum=0.9, wd=1e-3, eta=0.01)),
]


@pytest.mark.parametrize("seed", list(range(27 + _EXTRA)))
def test_randomized_optimizers_store_types_and_checkpoints(seed, tmp_path):
    """Every fused optimizer x {'device', 'local'} association order, random device subsets per call, and a
    save / load of the optimizer states into a fresh store in the middle of the run."""
    _need(2)
    ngpu = min(mx.num_gpus(), 8)
    rng = _rng(5000 + seed)
    optname, kw = _FUZZ_OPTS[seed % len(_FUZZ_OPTS)]
    kvtype = ["device", "local", "device"][seed % 3]
    layerwise = optname in ("lamb", "lans", "lars")
    sizes = [int(x) for x in rng.choice([7, 640, 4099, 70001, 300007], size=3, replace=False)]
    keys = ["p%d" % i for i in range(len(sizes))]
    w0 = [rng.uniform(-1, 1, e).astype(np.float32) for e in sizes]

    def make_store(weights):
        s = mx.kv.create(kvtype)
        s.init(keys, [mx.nd.array(w, mx.gpu(int(rng.integers(ngpu)))) for w in weights])
        if optname:
            s.set_optimizer(mx.optimizer.create(optname, **kw))
        return s

    kv = make_store(w0)
    okv = O.OracleKVStore(kvtype)
    okv.init(keys, [w.copy() for w in w0])
    if optname:
        okv.set_optimizer(O.OracleOptimizer(optname, **(dict(kw, norm_mode="f64") if layerwise else kw)))
    reload_at = int(rng.integers(2, 6)) if optname else -1

    def compare(got, want, what):
        if layerwise:
            np.testing.assert_allclose(got, want, rtol=5e-6, atol=5e-7, err_msg=str(what))
        else:
            assert _bits_equal(got, want), what

    for step in range(8):
        if step == reload_at:
            f = str(tmp_path / ("states_%d" % seed))
            kv.save_optimizer_states(f, dump_optimizer=True)      # with its update counts
            cur = []
            for k, e in zip(keys, sizes):
                o = mx.nd.empty((e,), mx.cpu())
                kv.pull(k, out=o)
                cur.append(o.asnumpy().copy())
            kv = make_store(cur)
            kv.load_optimizer_states(f)
        nk = int(rng.integers(1, len(keys) + 1))
        ks = sorted(rng.choice(len(keys), size=nk, replace=False).tolist())
        devs = [int(x) for x in rng.choice(ngpu, size=int(rng.integers(1, ngpu + 1)), replace=False)]
        grads = [[rng.uniform(-1, 1, sizes[k]).astype(np.float32) for _ in devs] for k in ks]
        vals = [[mx.nd.array(g, mx.gpu(d)) for g, d in zip(gs, devs)] for gs in grads]
        names = [keys[k] for k in ks]
        if rng.random() < 0.5:
            kv.push(names, vals)
        else:
            odevs = [int(x) for x in rng.choice(ngpu, size=int(rng.integers(1, min(4, ngpu + 1))), replace=False)]
            outs = [[mx.nd.empty((sizes[k],), mx.gpu(d)) for d in odevs] for k in ks]
            kv.pushpull(names, vals, out=outs)
        okv.push(names, grads)
        for k in ks:
            d = int(rng.integers(ngpu))
            o = mx.nd.empty((sizes[k],), mx.gpu(d))
            kv.pull(keys[k], out=o)
            want = np.empty(sizes[k], np.float32)
            okv.pull(keys[k], want)
            compare(o.asnumpy(), want, (optname, kvtype, seed, step, k, devs))
            if layerwise:
                okv.local[keys[k]][...] = o.asnumpy().reshape(okv.local[keys[k]].shape)   # follow the device trajectory


@pytest.mark.parametrize("seed", list(range(16 + _EXTRA)))
def test_randomized_row_sparse_compression_callback(seed):
    """Random walks over the other three kinds of keys: row_sparse (lazy / standard SGD, Adam, or plain
    assignment), 2-bit compressed dense keys, and keys updated through the Python updater callback."""
    _need(2)
    ngpu = min(mx.num_gpus(), 8)
    rng = _rng(9000 + seed)
    flavour = ["rsp", "gc", "callback", "rsp"][seed % 4]

    def ctx_of(d):
        return mx.cpu() if d < 0 else mx.gpu(d)

    if flavour == "rsp":
        rows, L = int(rng.choice([40, 300])), int(rng.choice([4, 6, 16]))
        shape = (rows, L)
        w0 = rng.uniform(-1, 1, shape).astype(np.float32)
        optname, kw = [(None, {}), ("sgd", dict(learning_rate=0.1, momentum=0.9, wd=1e-3, lazy_update=True)),
                       ("sgd", dict(learning_rate=0.1, wd=1e-3, lazy_update=False)),
                       ("adam", dict(learning_rate=0.01, wd=1e-3, lazy_update=bool(seed & 8)))][(seed // 4) % 4]
        kv = mx.kv.create("device")
        kv.init("e", mx.nd.row_sparse_array(w0, ctx=ctx_of(int(rng.integers(-1, ngpu)))))
        okv = O.OracleKVStore("device")
        okv.init("e", O.RowSparse.from_dense(w0))
        if optname:
            kv.set_optimizer(mx.optimizer.create(optname, **kw))
            okv.set_optimizer(O.OracleOptimizer(optname, **kw))
        for step in range(6):
            devs = [int(x) for x in rng.choice(np.arange(-1, ngpu), size=int(rng.integers(1, min(5, ngpu + 2))), replace=False)]
            parts = []
            for _ in devs:
                nnz = int(rng.integers(0, rows // 2 + 1))
                idx = np.sort(rng.choice(rows, nnz, replace=False)).astype(np.int64)
                parts.append((idx, rng.uniform(-1, 1, (nnz, L)).astype(np.float32)))
            kv.push("e", [mx.nd.row_sparse_array((v, i), shape=shape, ctx=ctx_of(d)) for (i, v), d in zip(parts, devs)])
            okv.push("e", [O.RowSparse(i, v, shape) for i, v in parts])
            ids = rng.integers(0, rows, int(rng.integers(1, 2 * rows))).astype(np.int64)
            d = int(rng.integers(-1, ngpu))
            out = mx.nd.zeros(shape, ctx_of(d), stype="row_sparse")
            kv.row_sparse_pull("e", out=out, row_ids=mx.nd.array(ids, ctx_of(int(rng.integers(-1, ngpu))), dtype=np.int64))
            want = O.sparse_retain(okv.local["e"], O.unique(ids))
            assert np.array_equal(out.indices.asnumpy(), want.indices), (seed, step)
            assert _bits_equal(out.data.asnumpy(), want.data.reshape(-1, L)), (seed, step, devs, d)
    elif flavour == "gc":
        E, thr = int(rng.choice([33, 4099, 70001])), 0.5
        bits = "2bit" if seed & 4 else "1bit"
        thr = 0.5 if bits == "2bit" else 0.0
        kv = mx.kv.create("device")
        kv.set_gradient_compression({"type": bits, "threshold": thr})
        kv.init(0, mx.nd.zeros((E,), mx.gpu(int(rng.integers(ngpu)))))
        n_slots = int(rng.integers(1, min(5, ngpu + 1)))
        residual = [np.zeros(E, np.float32) for _ in range(n_slots)]
        q, dq = (O.quantize_2bit, O.dequantize_2bit) if bits == "2bit" else (O.quantize_1bit, O.dequantize_1bit)
        for step in range(5):
            devs = [int(x) for x in rng.choice(ngpu, size=n_slots, replace=False)]
            g = [rng.uniform(-1, 1, E).astype(np.float32) for _ in devs]
            outs = [mx.nd.empty((E,), mx.gpu(int(d))) for d in rng.choice(ngpu, size=min(2, ngpu), replace=False)]
            kv.pushpull(0, [mx.nd.array(x, mx.gpu(d)) for x, d in zip(g, devs)], out=outs)
            deq = [dq(q(x, r, thr), E, thr) for x, r in zip(g, residual)]
            want = O.sum_device(deq) if len(deq) > 1 else deq[0]
            for o in outs:
                assert _bits_equal(o.asnumpy(), want), (seed, step, devs)
    else:
        shape = (int(rng.integers(1, 9)), int(rng.integers(1, 9)))
        kv = mx.kv.create("device")
        kv.init("c", mx.nd.zeros(shape, ctx_of(int(rng.integers(-1, ngpu)))))
        kv._set_updater(lambda key, recv, local: local.__iadd__(recv * 2))
        total = np.zeros(shape, np.float32)
        for step in range(6):
            devs = [int(x) for x in rng.choice(np.arange(-1, ngpu), size=int(rng.integers(1, min(5, ngpu + 2))), replace=False)]
            g = [rng.integers(-3, 4, shape).astype(np.float32) for _ in devs]
            kv.push("c", [mx.nd.array(x, ctx_of(d)) for x, d in zip(g, devs)])
            total += 2 * sum(g)
            o = mx.nd.empty(shape, ctx_of(int(rng.integers(-1, ngpu))))
            kv.pull("c", out=o)
            assert np.array_equal(o.asnumpy(), total), (seed, step, devs)


@pytest.mark.parametrize("seed", list(range(6 + _EXTRA)))
def test_randomized_low_precision_master_weights(seed):
    """bf16 / fp16 keys with an fp32 master and momentum (multi_precision SGD): the master and the momentum
    must follow the key when the set of GPUs changes from call to call."""
    _need(2)
    ngpu = min(mx.num_gpus(), 8)
    rng = _rng(12000 + seed)
    lp = "bfloat16" if seed % 2 == 0 else np.float16
    kind = 2 if lp == "bfloat16" else 1
    to_lp = (lambda x: O.f32_to_bf16(x)) if kind == 2 else (lambda x: x.astype(np.float16))
    to_f32 = (lambda x: O.bf16_to_f32(x)) if kind == 2 else (lambda x: x.astype(np.float32))
    E = int(rng.choice([4099, 70001, 300007]))
    w_lp = to_lp(rng.uniform(-1, 1, E).astype(np.float32))
    w32, mom = to_f32(w_lp), np.zeros(E, np.float32)
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.array(w_lp, mx.gpu(int(rng.integers(ngpu))), dtype=lp))
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, wd=1e-4, multi_precision=True))
    want = np.zeros(E, np.uint16)
    for step in range(6):
        devs = [int(x) for x in rng.choice(ngpu, size=int(rng.integers(1, ngpu + 1)), replace=False)]
        g_lp = [to_lp(rng.uniform(-1, 1, E).astype(np.float32)) for _ in devs]
        kv.push(0, [mx.nd.array(x, mx.gpu(d), dtype=lp) for x, d in zip(g_lp, devs)])
        gsum = O.sum_device_lp_f32out(g_lp, kind) if len(g_lp) > 1 else to_f32(g_lp[0])
        O.mp_sgd_mom_update(want, kind, w32, mom, gsum, 0.1, 1e-4, 0.9)
        out = mx.nd.empty((E,), mx.gpu(int(rng.integers(ngpu))), dtype=lp)
        kv.pull(0, out=out)
        got = out.asnumpy(raw=True) if kind == 2 else out.asnumpy().view(np.uint16)
        assert np.array_equal(got, want), (seed, step, devs)


def test_sharding_threshold_and_chunking_change_between_calls():
    """MXKVB200SetTwoShotBytes / MXKVB200SetTuning between steps: the same key goes from redundant (one-shot) to
    sharded (two-shot) updates and back, with Adam state and with the LAMB sequence, and the scheduling chunk
    changes under it -- results do not depend on any of that."""
    _need(2)
    import ctypes
    from mxnet_b200.base import _LIB, check_call
    devs = list(range(min(mx.num_gpus(), 4)))
    E = 70001
    try:
        for optname, kw, exact in (("adam", dict(learning_rate=0.01, wd=1e-3), True),
                                   ("lamb", dict(learning_rate=0.01, wd=0.01), False)):
            rng = _rng(13)
            w0 = rng.uniform(-1, 1, E).astype(np.float32)
            kv = mx.kv.create("device")
            kv.init(0, mx.nd.array(w0, mx.gpu(0)))
            kv.set_optimizer(mx.optimizer.create(optname, **kw))
            oopt = O.OracleOptimizer(optname, **(kw if exact else dict(kw, norm_mode="f64")))
            ow = w0.copy()
            outs = [mx.nd.empty((E,), mx.gpu(d)) for d in devs]
            for step, (thr, chunk) in enumerate([(1 << 30, 8192), (1024, 8192), (1024, 2048), (1 << 30, 4096), (4096, 8192)]):
                check_call(_LIB.MXKVB200SetTwoShotBytes(ctypes.c_int64(thr)))
                check_call(_LIB.MXKVB200SetTuning(ctypes.c_int64(chunk), 512, 0, -1))
                g = [rng.uniform(-1, 1, E).astype(np.float32) for _ in devs]
                kv.pushpull(0, [mx.nd.array(x, mx.gpu(d)) for x, d in zip(g, devs)], out=outs)
                oopt.update(0, ow, O.sum_device(g))
                for o in outs:
                    if exact:
                        assert _bits_equal(o.asnumpy(), ow), (optname, step)
                    else:
                        np.testing.assert_allclose(o.asnumpy(), ow, rtol=5e-6, atol=5e-7, err_msg=str((optname, step)))
                if not exact:
                    ow = outs[0].asnumpy().copy()
    finally:
        check_call(_LIB.MXKVB200SetTwoShotBytes(ctypes.c_int64(262144)))
        check_call(_LIB.MXKVB200SetTuning(ctypes.c_int64(8192), 512, 0, -1))


def test_empty_trailing_shard_keeps_the_staged_kernel():
    """A two-shot float32 key of 516 elements over 4 GPUs: shards of 256, so the last rank's range is empty and
    starts at 516, which is not on a packet boundary.  An empty range reads and writes nothing, so it must not take
    the launch class (here with a larger key) off the staged kernel -- in one-process-per-GPU mode every rank
    decides the variant from its own entries, and the ranks would disagree on the grid."""
    _need(4)
    import ctypes
    from mxnet_b200.base import _LIB, check_call
    devs = list(range(4))
    sizes = [516, 70000]
    rng = _rng(21)
    try:
        check_call(_LIB.MXKVB200SetTwoShotBytes(ctypes.c_int64(1024)))
        kv = mx.kv.create("device")
        kv.init([0, 1], [mx.nd.zeros((E,), mx.gpu(0)) for E in sizes])
        vals = [[rng.uniform(-1, 1, E).astype(np.float32) for _ in devs] for E in sizes]
        outs = [[mx.nd.empty((E,), mx.gpu(d)) for d in devs] for E in sizes]
        bulk0, thread0 = mx.kv.launch_count("bulk"), mx.kv.launch_count("per_thread")
        kv.pushpull([0, 1], [[mx.nd.array(v, mx.gpu(d)) for v, d in zip(vs, devs)] for vs in vals], out=outs)
        assert mx.kv.launch_count("per_thread") == thread0
        assert mx.kv.launch_count("bulk") - bulk0 == len(devs)
        for vs, os_ in zip(vals, outs):
            want = O.sum_device(vs)
            for o in os_:
                assert _bits_equal(o.asnumpy(), want)
    finally:
        check_call(_LIB.MXKVB200SetTwoShotBytes(ctypes.c_int64(262144)))


@pytest.mark.parametrize("seed", list(range(12 + _EXTRA)))
def test_randomized_dense_keys_with_row_sparse_gradients(seed):
    """Dense weights updated on the store by a random mix of dense and row_sparse gradients (Parameter(grad_stype=
    'row_sparse') next to dense parameters): random device subsets and host values for both kinds, keys on either
    side of the sharding threshold, one optimizer state serving both kinds of update."""
    _need(2)
    ngpu = min(mx.num_gpus(), 8)
    rng = _rng(12000 + seed)
    optname, kw = [("sgd", dict(learning_rate=0.1, momentum=0.9, wd=1e-3, lazy_update=True)),
                   ("sgd", dict(learning_rate=0.1, wd=1e-3, lazy_update=False)),
                   ("adam", dict(learning_rate=0.01, wd=1e-3, lazy_update=True)),
                   ("adam", dict(learning_rate=0.01, wd=1e-3, lazy_update=False)),
                   ("sgd", dict(learning_rate=0.05, momentum=0.5, lazy_update=False, rescale_grad=0.25,
                                clip_gradient=0.4))][seed % 5]
    shapes = [(int(rng.choice([30, 200])), int(rng.choice([4, 6]))), (1100, 64), (int(rng.choice([17, 500])),)]
    keys = ["k%d" % i for i in range(len(shapes))]
    w0 = [rng.uniform(-1, 1, s).astype(np.float32) for s in shapes]

    def ctx_of(d):
        return mx.cpu() if d < 0 else mx.gpu(d)

    kv = mx.kv.create(["device", "local"][seed % 2])
    kv.init(keys, [mx.nd.array(w, ctx_of(int(rng.integers(-1, ngpu)))) for w in w0])
    kv.set_optimizer(mx.optimizer.create(optname, **kw))
    okv = O.OracleKVStore(["device", "local"][seed % 2])
    okv.init(keys, [w.copy() for w in w0])
    okv.set_optimizer(O.OracleOptimizer(optname, **kw))
    for step in range(8):
        k = int(rng.integers(len(keys)))
        shape, rows = shapes[k], shapes[k][0]
        if rng.random() < 0.55:
            devs = [int(x) for x in rng.choice(np.arange(-1, ngpu), size=int(rng.integers(1, min(5, ngpu + 2))),
                                               replace=False)]
            parts = []
            for _ in devs:
                nnz = int(rng.integers(0, rows // 2 + 1))
                idx = np.sort(rng.choice(rows, nnz, replace=False)).astype(np.int64)
                parts.append((idx, rng.uniform(-1, 1, (nnz,) + shape[1:]).astype(np.float32)))
            kv.push(keys[k], [mx.nd.row_sparse_array((v, i), shape=shape, ctx=ctx_of(d))
                              for (i, v), d in zip(parts, devs)])
            okv.push(keys[k], [O.RowSparse(i, v, shape) for i, v in parts])
            what = ("rsp", devs)
        else:
            devs = [int(x) for x in rng.choice(ngpu, size=int(rng.integers(1, ngpu + 1)), replace=False)]
            gs = [rng.uniform(-1, 1, shape).astype(np.float32) for _ in devs]
            vals = [mx.nd.array(g, mx.gpu(d)) for g, d in zip(gs, devs)]
            if rng.random() < 0.5:
                kv.push(keys[k], vals)
            else:
                kv.pushpull(keys[k], vals, out=[mx.nd.empty(shape, mx.gpu(d)) for d in devs[:3]])
            okv.push(keys[k], gs)
            what = ("dense", devs)
        d = int(rng.integers(-1, ngpu))
        o = mx.nd.empty(shape, ctx_of(d))
        kv.pull(keys[k], out=o)
        assert _bits_equal(o.asnumpy(), okv.local[keys[k]]), (optname, kw, seed, step, k, what, d)
