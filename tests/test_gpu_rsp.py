"""row_sparse push / row_sparse_pull on the GPU vs the CPU oracle (bit-exact)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import mxnet_b200 as mx
from oracle import oracle as O


def _bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32),
                          np.ascontiguousarray(b, np.float32).view(np.uint32))


def _rand_rsp(rng, rows, L, nnz):
    idx = np.sort(rng.choice(rows, nnz, replace=False)).astype(np.int64)
    val = rng.uniform(-1, 1, (nnz, L)).astype(np.float32)
    return idx, val


def _mk(idx, val, shape, ctx):
    return mx.nd.row_sparse_array((val, idx), shape=shape, ctx=ctx)


@pytest.mark.parametrize("rows,L,nnz,n", [(50, 8, 12, 4), (1000, 256, 100, 4), (5000, 33, 700, 3),
                                          (20000, 64, 3000, 8), (100, 4, 100, 2), (64, 16, 0, 2)])
def test_push_no_updater_is_rsp_sum(rows, L, nnz, n):
    """push of n row_sparse values: stored value = sorted-union row sums, inputs added in order
    onto zero (ndarray_function.cu:176-187)."""
    rng = np.random.default_rng(rows + L + n)
    shape = (rows, L)
    srcs = [_rand_rsp(rng, rows, L, nnz) for _ in range(n)]
    kv = mx.kv.create("device")
    kv.init("e", mx.nd.row_sparse_array(np.ones(shape, np.float32), ctx=mx.gpu(0)))
    kv.push("e", [_mk(i, v, shape, mx.gpu(0)) for i, v in srcs])
    out = mx.nd.empty(shape, mx.gpu(0))
    kv.pull("e", out=out, ignore_sparse=False)
    want = O.rsp_sum([O.RowSparse(i, v, shape) for i, v in srcs]).todense()
    assert _bits_equal(out.asnumpy(), want)


def test_row_sparse_pull_retain():
    """tests/python/unittest/test_kvstore.py:68-94 with random (unsorted, repeated) ids."""
    rng = np.random.default_rng(3)
    rows, L = 300, 20
    shape = (rows, L)
    table = rng.uniform(-1, 1, shape).astype(np.float32)
    kv = mx.kv.create("device")
    kv.init("e", mx.nd.row_sparse_array(table, ctx=mx.gpu(0)))
    for count in (1, 7, 300, 1000, 40000):      # 40000 > 16384: global-memory sort path
        ids = rng.integers(0, rows, count).astype(np.int64)
        out = mx.nd.empty(shape, mx.gpu(0), stype="row_sparse", capacity=max(count, 1))
        kv.row_sparse_pull("e", out=out, row_ids=mx.nd.array(ids, mx.gpu(0), dtype=np.int64))
        want = O.sparse_retain(O.RowSparse(np.arange(rows), table, shape), O.unique(ids))
        assert np.array_equal(out.indices.asnumpy(), want.indices)
        assert _bits_equal(out.data.asnumpy(), want.data.reshape(-1, L))
    # host-resident ids and output (the reference unit test's placement)
    ids = rng.integers(0, rows, 40).astype(np.int64)
    out = mx.nd.zeros(shape, stype="row_sparse")
    kv.row_sparse_pull("e", out=out, row_ids=mx.nd.array(ids.reshape(2, 20), dtype=np.int64))
    dense = out.asnumpy()
    for r in range(rows):
        assert _bits_equal(dense[r], table[r] if r in ids else np.zeros(L, np.float32))


@pytest.mark.parametrize("lazy", [True, False, "four-kernel"])
@pytest.mark.parametrize("optname,kw", [
    ("sgd", dict(learning_rate=0.1, wd=1e-3, rescale_grad=0.5, clip_gradient=0.6)),
    ("sgd", dict(learning_rate=0.1, wd=1e-3, momentum=0.9)),
    ("adam", dict(learning_rate=0.01, wd=1e-3)),
])
def test_fused_sparse_update(optname, kw, lazy, monkeypatch):
    """lazy_update=True: only the rows present in the summed gradient are touched (SGDDnsRspKernel /
    SGDMomDnsRspDnsKernel / AdamDnsRspDnsKernel); lazy_update=False (the reference default): the
    standard update over every row (SGDUpdateDnsRspImpl non-lazy branch, SGDMomStdDnsRspDnsKernel,
    AdamStdDnsRspDnsKernel).  "four-kernel": the lazy update with MXKV_B200_RSP_FUSED=0, run by the union +
    gather-sum kernels (the code of the multi-node push's final merge) instead of rsp_push_fused_kernel."""
    if lazy == "four-kernel":
        monkeypatch.setenv("MXKV_B200_RSP_FUSED", "0")
        lazy = True
    kw = dict(kw, lazy_update=lazy)
    rng = np.random.default_rng(11)
    rows, L, nnz, n = 2000, 64, 150, 4
    shape = (rows, L)
    w0 = rng.uniform(0, 1, shape).astype(np.float32)
    kv = mx.kv.create("device")
    kv.init(5, mx.nd.row_sparse_array(w0, ctx=mx.gpu(0)))
    kv.set_optimizer(mx.optimizer.create(optname, **kw))
    okv = O.OracleKVStore("device")
    okv.init(5, O.RowSparse.from_dense(w0))
    okv.set_optimizer(O.OracleOptimizer(optname, **kw))
    for step in range(3):
        srcs = [_rand_rsp(rng, rows, L, nnz) for _ in range(n)]
        kv.push(5, [_mk(i, v, shape, mx.gpu(0)) for i, v in srcs])
        okv.push(5, [O.RowSparse(i, v, shape) for i, v in srcs])
        out = mx.nd.empty(shape, mx.gpu(0))
        kv.pull(5, out=out, ignore_sparse=False)
        assert _bits_equal(out.asnumpy(), okv.local[5].todense()), (optname, step)


def test_reference_kats_row_sparse():
    """test_kvstore.py:55-66 (single pair), :123-136 (list), :222-274 (updater), :281-339 (invalid)."""
    shape = (4, 4)
    kv = mx.kv.create("device")
    kv.init(3, mx.nd.zeros(shape, stype="row_sparse"))
    kv.push(3, mx.nd.ones(shape).tostype("row_sparse"))
    val = mx.nd.empty(shape)
    kv.pull(3, out=val)
    assert np.all(val.asnumpy() == 1)
    keys = [5, 7, 11]
    kv.init(keys, [mx.nd.zeros(shape, stype="row_sparse")] * 3)
    kv.push(keys, [(mx.nd.ones(shape) * 4).tostype("row_sparse")] * 3)
    vals = [mx.nd.empty(shape) for _ in keys]
    kv.pull(keys, out=vals)
    assert all(np.all(v.asnumpy() == 4) for v in vals)
    # updater with 4 "devices"
    kv2 = mx.kv.create("device")
    kv2.init("a", mx.nd.zeros(shape, mx.gpu(0), stype="row_sparse"))

    def upd(key, recv, local):
        assert isinstance(key, str)
        local += recv
    kv2._set_updater(upd)
    for it in range(1, 3):
        kv2.push("a", [mx.nd.ones(shape, mx.gpu(0)).tostype("row_sparse") for _ in range(4)])
        o = mx.nd.empty(shape, mx.gpu(0))
        kv2.pull("a", out=o, ignore_sparse=False)
        assert np.all(o.asnumpy() == 4 * it)
    # ignored / invalid pulls
    rsp_out = (mx.nd.ones(shape) * 2).tostype("row_sparse")
    kv.pull(3, out=rsp_out)                       # ignored: values untouched
    assert np.all(rsp_out.asnumpy() == 2)
    with pytest.raises(mx.MXNetError):
        kv.row_sparse_pull(3, out=mx.nd.ones(shape) * 2, row_ids=mx.nd.array([1], dtype=np.int64))


@pytest.mark.multigpu
def test_sp_multi_gpu_sources():
    devs = list(range(min(mx.num_gpus(), 4)))
    rng = np.random.default_rng(8)
    rows, L, nnz = 5000, 128, 400
    shape = (rows, L)
    w0 = rng.uniform(0, 1, shape).astype(np.float32)
    kw = dict(learning_rate=0.1, momentum=0.9, wd=1e-4, lazy_update=True)
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.row_sparse_array(w0, ctx=mx.gpu(0)))
    kv.set_optimizer(mx.optimizer.SGD(**kw))
    okv = O.OracleKVStore("device")
    okv.init(0, O.RowSparse.from_dense(w0))
    okv.set_optimizer(O.OracleOptimizer("sgd", **kw))
    for step in range(3):
        srcs = [_rand_rsp(rng, rows, L, nnz) for _ in devs]
        kv.push(0, [_mk(i, v, shape, mx.gpu(d)) for (i, v), d in zip(srcs, devs)])
        okv.push(0, [O.RowSparse(i, v, shape) for i, v in srcs])
        ids = rng.integers(0, rows, 500).astype(np.int64)
        for d in devs:
            out = mx.nd.empty(shape, mx.gpu(d), stype="row_sparse", capacity=500)
            kv.row_sparse_pull(0, out=out, row_ids=mx.nd.array(ids, mx.gpu(d), dtype=np.int64))
            want = O.sparse_retain(okv.local[0], O.unique(ids))
            assert np.array_equal(out.indices.asnumpy(), want.indices)
            assert _bits_equal(out.data.asnumpy(), want.data.reshape(-1, L)), (step, d)


@pytest.mark.multigpu
def test_sp_multi_gpu_sources_four_kernel_path(monkeypatch):
    """The same with MXKV_B200_RSP_FUSED=0 (peer sources read by the union + gather-sum kernels)."""
    monkeypatch.setenv("MXKV_B200_RSP_FUSED", "0")
    test_sp_multi_gpu_sources()


@pytest.mark.parametrize("n", [1, 4])
def test_c5_shape_fused_push_and_pull(n):
    """BASELINE.json configs[4] at its exact shape -- one row_sparse key of 1 M x 256 float32, 10 000 distinct rows
    per value, lazy SGD-momentum -- through the fused kernels (rsp_push_fused_kernel, rsp_pull_fused_kernel): n
    values per push on one GPU (the cross-GPU form of the same kernels: tests/mp_worker.py scenario 5), three
    pushes, row_sparse_pull of the touched rows after each; only the touched rows are compared (the oracle keeps
    the table sparse; untouched rows are checked once by sampling)."""
    import os
    sim = bool(os.environ.get("MXKV_SIM"))
    R, L, nnz = (20000, 64, 500) if sim else (1_000_000, 256, 10_000)
    shape = (R, L)
    rng = np.random.default_rng(55 + n)
    kw = dict(learning_rate=0.01, momentum=0.9, wd=0.0, lazy_update=True)
    kv = mx.kv.create("device")
    kv.init("emb", mx.nd.row_sparse_array((np.zeros((1, L), np.float32), np.zeros(1, np.int64)), shape=shape, ctx=mx.gpu(0)))
    kv.set_optimizer(mx.optimizer.SGD(**kw))
    # host model of the touched rows only: weight and momentum per row id
    w, m = {}, {}
    before = mx.kv.launch_count()
    for step in range(3):
        srcs = [_rand_rsp(rng, R, L, nnz) for _ in range(n)]
        kv.push("emb", [_mk(i, v, shape, mx.gpu(0)) for i, v in srcs])
        merged = O.rsp_sum([O.RowSparse(i, v, shape) for i, v in srcs])
        for j, rid in enumerate(merged.indices):
            rid = int(rid)
            g = merged.data.reshape(-1, L)[j]
            wr = w.get(rid, np.zeros(L, np.float32))
            mr = m.get(rid, np.zeros(L, np.float32))
            O.sgd_mom_update(wr, g.copy(), mr, kw["learning_rate"], kw["wd"], kw["momentum"])
            w[rid], m[rid] = wr, mr
        ids = merged.indices.astype(np.int64)
        if step == 1:                       # unsorted ids with repeats: the sort + compaction path of the pull kernel
            ids = np.concatenate([ids[::-1][: min(len(ids), 16000)], ids[:100]])
        out = mx.nd.empty(shape, mx.gpu(0), stype="row_sparse", capacity=len(ids))
        kv.row_sparse_pull("emb", out=out, row_ids=mx.nd.array(ids, mx.gpu(0), dtype=np.int64))
        got_idx, got = out.indices.asnumpy(), out.data.asnumpy().reshape(-1, L)
        want_idx = np.unique(ids)
        assert np.array_equal(got_idx, want_idx), (n, step)
        want = np.stack([w[int(r)] for r in want_idx])
        assert _bits_equal(got, want), (n, step)
    assert mx.kv.launch_count() - before <= 3 * 2 + 2, "push and row_sparse_pull are one launch each"
    # rows nobody pushed are still zero
    probe = np.setdiff1d(rng.choice(R, 200, replace=False), np.fromiter(w.keys(), dtype=np.int64))
    out = mx.nd.empty(shape, mx.gpu(0), stype="row_sparse", capacity=len(probe))
    kv.row_sparse_pull("emb", out=out, row_ids=mx.nd.array(probe.astype(np.int64), mx.gpu(0), dtype=np.int64))
    assert not out.data.asnumpy().any()
