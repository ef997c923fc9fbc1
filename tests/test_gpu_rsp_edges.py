"""The row_sparse push, its lazy and standard updates and row_sparse_pull at the edges of their kernels
(csrc/rsp_kernels.cu): row widths that take the scalar loop over several 32-column passes or the float4 loop with a
partial last pass, 9 ... 16 sources (the fused kernel's lane-per-source search and its "first holder" ballot),
overlap patterns that decide which candidate sums a row, the update options, id lists at the unique kernels' size
boundaries, and tables above 2^31 elements.

Every result is compared bit for bit with the CPU oracle (``oracle.OracleKVStore`` / ``O.rsp_sum`` /
``O.sparse_retain``: sums added in source order onto zero).  The updates are also compared with a float64 numpy model
that shares no code with the oracle -- the union sum with ``np.add.at`` and one step of ``lp_oracle.step_f64`` per
push, from the kernel's own float32 weight and state before that push -- so that a source dropped or counted twice by
the oracle and the kernel alike still fails.  The allowed error is ``_f64_bound``: half an ulp of the result, plus
``lp_oracle.ROUNDINGS`` (8) roundings of 2^-24 of the step's magnitude, plus the float32 sum's own error (one rounding
of the sum of absolute contributions per source after the first) carried through the step.  The worst ratio of error
to that bound over the push tests is 0.30 (standard SGD): under three of the eight roundings are used.

Row_sparse values are always engine-allocated (16-byte aligned), so the scalar instantiations are reached through
row widths that are not multiples of 4 (1, 3, 6, 33, 129).  Launch counters show which path ran: one launch per
fused push, the union / scan / rank / rows kernels (and the per-source row-count copies) for the four-kernel path.
"""
import gc
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import mxnet_b200 as mx
from oracle import oracle as O
from lp_oracle import ROUNDINGS, step_f64

SIM = bool(os.environ.get("MXKV_SIM"))
U = 2.0 ** -24
G = mx.gpu(0)


def _bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32),
                          np.ascontiguousarray(b, np.float32).view(np.uint32))


def _mk(idx, val, shape, ctx):
    return mx.nd.row_sparse_array((val, idx), shape=shape, ctx=ctx)


def _path(monkeypatch, fused):
    monkeypatch.setenv("MXKV_B200_RSP_FUSED", "1" if fused else "0")


# ---- the float64 model -------------------------------------------------------------------------------------------
def _union_f64(srcs, shape):
    """float64 union sum of the sources, the sum of their absolute values, and the number of holders per row"""
    g = np.zeros(shape, np.float64)
    gabs = np.zeros(shape, np.float64)
    cnt = np.zeros(shape[0], np.int64)
    for idx, val in srcs:
        np.add.at(g, idx, val.astype(np.float64))
        np.add.at(gabs, idx, np.abs(val.astype(np.float64)))
        np.add.at(cnt, idx, 1)
    return g, gabs, cnt


def _sum_err(gabs, cnt):
    """bound on |float32 sum in source order onto zero - exact sum|: the first addition is exact, every later one
    rounds once, by at most 2^-24 of the running sum's magnitude"""
    return np.maximum(cnt - 1, 0)[:, None] * U * gabs


def _f64_bound(w64, mag):
    return np.spacing(np.abs(w64).astype(np.float32)).astype(np.float64) / 2 + ROUNDINGS * U * mag


class Model(object):
    """hyper-parameters of one store key, in the form ``lp_oracle.step_f64`` takes"""

    def __init__(self, name, kw, lr_mult=1.0, wd_mult=1.0):
        self.name, self.kw = name, kw
        self.lazy = kw.get("lazy_update", False)
        self.lr = kw.get("learning_rate", 0.1 if name == "sgd" else 0.001) * lr_mult
        self.wd = kw.get("wd", 0.0) * wd_mult
        self.momentum = kw.get("momentum", 0.0)
        self.b1, self.b2 = kw.get("beta1", 0.9), kw.get("beta2", 0.999)
        self.eps = kw.get("epsilon", 1e-8)
        self.rescale = kw.get("rescale_grad", 1.0)
        self.clip = kw.get("clip_gradient")
        self.t = 0

    def states(self):
        return {"sgd": 1 if self.momentum else 0, "adam": 2}[self.name]

    def check(self, w_prev, s_prev, srcs, got):
        """one push: the kernel's new weight `got` against one float64 step from its previous weight / state; returns
        the largest error / bound"""
        self.t += 1
        shape = w_prev.shape
        g, gabs, cnt = _union_f64(srcs, shape)
        lr = self.lr
        if self.name == "adam":             # adam.py:166-175, in double like the host
            lr = lr * np.sqrt(1.0 - self.b2 ** self.t) / (1.0 - self.b1 ** self.t)
        f = lambda x: None if x is None else float(np.float32(x))     # noqa: E731  (the kernel's float32 arguments)
        h = dict(name=self.name, lr=f(lr), wd=f(self.wd), momentum=f(self.momentum), beta1=f(self.b1),
                 beta2=f(self.b2), eps=f(self.eps), rescale=f(self.rescale), clip=f(self.clip))
        lr, b1, b2 = h["lr"], h["beta1"], h["beta2"]
        s0 = s_prev[0] if len(s_prev) > 0 else np.zeros(shape, np.float32)
        s1 = s_prev[1] if len(s_prev) > 1 else np.zeros(shape, np.float32)
        w64, s0n, s1n, mag = step_f64(h, w_prev, g, s0, s1)
        # the float32 sum's error, carried through the step (clip is 1-Lipschitz): SGD moves w by lr * rescale * dg;
        # Adam by lr * rescale * dg * ((1 - b1) / den + |m| * sqrt(1 - b2) / den^2), as (1 - b2) * |r| <= sqrt((1 - b2) * v)
        dg = h["rescale"] * _sum_err(gabs, cnt)
        if self.name == "adam":
            den = np.sqrt(s1n) + h["eps"]
            m = np.abs(s0n)
            sens = lr * ((1.0 - b1) / den + m * np.sqrt(1.0 - b2) / den ** 2)
        else:
            sens = lr
        bound = _f64_bound(w64, mag) + sens * dg
        rows = cnt > 0 if self.lazy else np.ones(shape[0], bool)
        err = np.abs(got.astype(np.float64) - w64)
        bad = (err > bound) & rows[:, None]
        assert not bad.any(), "%d elements beyond the float64 bound (t=%d), worst err/bound %.3g" % (
            bad.sum(), self.t, (err / bound)[rows].max())
        if self.lazy:                       # untouched rows keep their weight exactly
            assert _bits_equal(got[~rows], w_prev[~rows])
        return float((err / np.maximum(bound, 1e-300))[rows].max()) if rows.any() else 0.0


# ---- a store and its oracle, side by side ------------------------------------------------------------------------
class Pair(object):
    def __init__(self, key, w0, optname=None, kw=None, lr_mult=None, wd_mult=None):
        self.key, self.shape = key, w0.shape
        self.kv = mx.kv.create("device")
        self.kv.init(key, mx.nd.row_sparse_array(w0, ctx=G))
        self.okv = O.OracleKVStore("device")
        self.okv.init(key, O.RowSparse.from_dense(w0))
        self.model = None
        if optname:
            opt = mx.optimizer.create(optname, **kw)
            if lr_mult is not None:
                opt.set_lr_mult({key: lr_mult})
            if wd_mult is not None:
                opt.set_wd_mult({key: wd_mult})
            self.kv.set_optimizer(opt)
            self.okv.set_optimizer(O.OracleOptimizer(
                optname, lr_mult={key: lr_mult} if lr_mult is not None else None,
                wd_mult={key: wd_mult} if wd_mult is not None else None, **kw))
            self.model = Model(optname, kw, lr_mult or 1.0, wd_mult or 1.0)
        self.w = w0.copy()

    def weight(self):
        out = mx.nd.empty(self.shape, G)
        self.kv.pull(self.key, out=out, ignore_sparse=False)
        return out.asnumpy()

    def state(self):
        if self.model is None or self.model.states() == 0:
            return []
        hs = [self.kv._state_handle(self.key, which) for which in (2, 3)[:self.model.states()]]
        return [h.asnumpy().reshape(self.shape) if h is not None else np.zeros(self.shape, np.float32) for h in hs]

    def oracle_state(self):
        st = self.okv.optimizer.states.get(self.key) if self.okv.optimizer else None
        if st is None:
            return []
        return list(st) if isinstance(st, tuple) else [st]

    def push(self, srcs):
        """push, then: weight and state bit for bit against the oracle, the weight against the float64 model (or,
        without an optimizer, the stored value against the float64 union sum); returns the push's launch count"""
        s_prev = self.state()
        vals = [_mk(i, v, self.shape, G) for i, v in srcs]
        before = mx.kv.launch_count()
        self.kv.push(self.key, vals)
        launches = mx.kv.launch_count() - before
        self.okv.push(self.key, [O.RowSparse(i, v, self.shape) for i, v in srcs])
        got = self.weight()
        assert _bits_equal(got, self.okv.local[self.key].todense()), "weight differs from the oracle"
        st, ost = self.state(), self.oracle_state()
        assert len(st) == len(ost)
        for a, b in zip(st, ost):
            assert _bits_equal(a, b), "optimizer state differs from the oracle"
        if self.model is not None:
            self.model.check(self.w, s_prev, srcs, got)
        else:                               # assign: the union sum, rows outside it zero
            g, gabs, cnt = _union_f64(srcs, self.shape)
            bound = _f64_bound(g, 0.0) + _sum_err(gabs, cnt)
            assert (np.abs(got - g) <= bound).all(), "stored value is not the union sum"
        self.w = got
        return launches


# ---- source patterns ---------------------------------------------------------------------------------------------
def _rand_ids(rng, pool, k):
    return np.sort(rng.choice(pool, min(k, len(pool)), replace=False)).astype(np.int64)


def _pattern(name, rng, rows, n):
    """row ids of n sources (each sorted and unique)"""
    k = max(rows // 3, 1)
    allrows = np.arange(rows)
    if name == "random":
        return [_rand_ids(rng, allrows, k) for _ in range(n)]
    if name == "identical":
        ids = _rand_ids(rng, allrows, k)
        return [ids.copy() for _ in range(n)]
    if name == "disjoint":
        perm = rng.permutation(rows)
        return [np.sort(c).astype(np.int64) for c in np.array_split(perm[: (rows // n) * n], n)]
    if name == "first_empty":
        return [np.zeros(0, np.int64)] + [_rand_ids(rng, allrows, k) for _ in range(n - 1)]
    if name == "middle_empty":
        return [_rand_ids(rng, allrows, k) if s in (0, n - 1) else np.zeros(0, np.int64) for s in range(n)]
    if name == "all_empty":
        return [np.zeros(0, np.int64) for _ in range(n)]
    if name == "single_row":
        r = int(rng.integers(1, rows - 1))
        return [np.array([r], np.int64) for _ in range(n)]
    if name == "edges":
        return [np.array([0, rows - 1], np.int64) for _ in range(n)]
    if name == "late":
        # sources 0 ... 7 stay off the last 24 rows; every one of those is held by two or more of the sources 8 and
        # up, so its first holder is source 8 or later and a later source holds it as well
        assert n >= 10
        late = np.arange(rows - 24, rows)
        ids = [_rand_ids(rng, allrows[: rows - 24], k) for _ in range(8)]
        extra = [set() for _ in range(n - 8)]
        for r in late:
            for s in rng.choice(n - 8, int(rng.integers(2, n - 7)), replace=False):
                extra[s].add(int(r))
        for s in range(n - 8):
            ids.append(np.union1d(_rand_ids(rng, allrows, k), np.array(sorted(extra[s]), np.int64)).astype(np.int64))
        return ids
    raise ValueError(name)


def _values(rng, ids, L):
    return [(i, rng.uniform(-1, 1, (len(i), L)).astype(np.float32)) for i in ids]


_OPTS = {
    "sgd": ("sgd", dict(learning_rate=0.1, wd=1e-3, rescale_grad=0.5, clip_gradient=0.6)),
    "sgd_mom": ("sgd", dict(learning_rate=0.1, wd=1e-3, momentum=0.9)),
    "adam": ("adam", dict(learning_rate=0.01, wd=1e-3)),
}
# lazy-fused: rsp_push_fused_kernel; lazy-four: MXKV_B200_RSP_FUSED=0, union + rows kernels with the update in them;
# std: the standard update (union + rows kernels, then the dense "Std" kernel over the whole table)
_MODES = ["lazy-fused", "lazy-four", "std"]


def _check_launches(mode, launches):
    if mode == "lazy-fused":
        assert launches == 1, "a fused push is one launch (%d)" % launches
    else:
        assert launches >= 4 + (mode == "std"), "the four-kernel path did not run (%d launches)" % launches


@pytest.mark.parametrize("mode", _MODES)
@pytest.mark.parametrize("opt", sorted(_OPTS))
@pytest.mark.parametrize("L", [1, 3, 6, 33, 129, 132, 260])
def test_row_widths(L, opt, mode, monkeypatch):
    """Scalar rows over one partial pass (1, 3, 6), several passes with a ragged tail (33, 129), float4 rows over two
    and three passes with a partial last one (132, 260); 101 rows, so every table but the float4 ones has a size
    that is not a multiple of 4 (the standard update's dense kernel then takes its scalar path)."""
    _path(monkeypatch, mode != "lazy-four")
    optname, kw = _OPTS[opt]
    kw = dict(kw, lazy_update=mode != "std")
    rng = np.random.default_rng(L * 31 + len(opt))
    rows = 101
    p = Pair(3, rng.uniform(-1, 1, (rows, L)).astype(np.float32), optname, kw)
    for step in range(3):
        launches = p.push(_values(rng, _pattern("random", rng, rows, 4), L))
        if step > 0:
            _check_launches(mode, launches)


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "four-kernel"])
@pytest.mark.parametrize("n", [1, 2, 8, 9, 10, 15, 16])
def test_source_counts(n, fused, monkeypatch):
    """n values in one push on one GPU, lazy SGD-momentum on 129-wide rows.  From 10 sources on, the last 24 rows
    are held only by sources 8 and up, each by two or more of them: the rows whose first holder the fused kernel
    finds in the upper half of its ballot."""
    _path(monkeypatch, fused)
    rng = np.random.default_rng(100 + n)
    rows, L = 203, 129
    kw = dict(learning_rate=0.1, momentum=0.9, wd=1e-3, lazy_update=True)
    p = Pair("k", rng.uniform(-1, 1, (rows, L)).astype(np.float32), "sgd", kw)
    for step in range(3):
        pattern = "late" if n >= 10 and step != 1 else "random"
        launches = p.push(_values(rng, _pattern(pattern, rng, rows, n), L))
        if step > 0:
            _check_launches("lazy-fused" if fused else "lazy-four", launches)


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "four-kernel"])
def test_seventeen_values_are_refused(fused, monkeypatch):
    """kMaxSrc = 16: a push of 17 values raises MXNetError and changes nothing -- not the weight, not the Adam state,
    not the update count (the next push's bias correction would show a counted refusal)."""
    _path(monkeypatch, fused)
    rng = np.random.default_rng(17)
    rows, L = 64, 12
    p = Pair(9, rng.uniform(-1, 1, (rows, L)).astype(np.float32), "adam", dict(learning_rate=0.01, lazy_update=True))
    p.push(_values(rng, _pattern("random", rng, rows, 16), L))
    w, st = p.weight(), p.state()
    srcs = _values(rng, _pattern("random", rng, rows, 17), L)
    with pytest.raises(mx.MXNetError):
        p.kv.push(9, [_mk(i, v, (rows, L), G) for i, v in srcs])
    assert _bits_equal(p.weight(), w)
    for a, b in zip(p.state(), st):
        assert _bits_equal(a, b)
    p.push(_values(rng, _pattern("random", rng, rows, 16), L))


_PATTERNS = ["identical", "disjoint", "first_empty", "middle_empty", "all_empty", "single_row", "edges"]


@pytest.mark.parametrize("mode", ["assign"] + _MODES)
@pytest.mark.parametrize("pattern", _PATTERNS)
def test_overlap_patterns(pattern, mode, monkeypatch):
    """Which candidate sums a row: every source holding the same ids, no two sharing one, an empty first source,
    empty sources in the middle, all empty, one row held by all, only rows 0 and rows - 1.  `assign` is the push
    without an updater (rows outside the union become zero); the others update with Adam."""
    _path(monkeypatch, mode != "lazy-four")
    rng = np.random.default_rng(_PATTERNS.index(pattern) * 7 + len(mode))
    rows, L, n = 257, 132, 5
    w0 = rng.uniform(-1, 1, (rows, L)).astype(np.float32)
    if mode == "assign":
        p = Pair(2, w0)
    else:
        p = Pair(2, w0, "adam", dict(learning_rate=0.01, wd=1e-3, lazy_update=mode != "std"))
    for step in range(3):
        launches = p.push(_values(rng, _pattern(pattern, rng, rows, n), L))
        if step > 0 and mode != "assign":
            _check_launches(mode, launches)


_OPTION_CASES = {
    # binding clip after rescale_grad, betas and epsilon off their defaults, weight decay, lr / wd multipliers
    "adam": ("adam", dict(learning_rate=0.02, rescale_grad=0.7, clip_gradient=0.4, beta1=0.5, beta2=0.8, epsilon=1e-3,
                          wd=0.03), 0.5, 2.0),
    # binding clip, no weight decay, lr / wd multipliers
    "sgd_mom": ("sgd", dict(learning_rate=0.05, momentum=0.8, rescale_grad=1.5, clip_gradient=0.5, wd=0.0), 3.0, 0.25),
}


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "four-kernel"])
@pytest.mark.parametrize("case", sorted(_OPTION_CASES))
def test_lazy_update_options(case, fused, monkeypatch):
    """The lazy updates' options on the kernels, over four pushes so that the state feeds back."""
    _path(monkeypatch, fused)
    optname, kw, lr_mult, wd_mult = _OPTION_CASES[case]
    kw = dict(kw, lazy_update=True)
    rng = np.random.default_rng(7 + len(case))
    rows, L = 151, 36
    p = Pair("opt", rng.uniform(-1, 1, (rows, L)).astype(np.float32), optname, kw, lr_mult=lr_mult, wd_mult=wd_mult)
    clipped = 0
    for step in range(4):
        srcs = _values(rng, _pattern("random", rng, rows, 4), L)
        g, _, _ = _union_f64(srcs, (rows, L))
        clipped += int((np.abs(kw["rescale_grad"] * g) > kw["clip_gradient"]).sum())
        launches = p.push(srcs)
        if step > 0:
            _check_launches("lazy-fused" if fused else "lazy-four", launches)
    assert clipped > 0, "the clip never bound"


# ---- row_sparse_pull ---------------------------------------------------------------------------------------------
_PULL_ROWS, _PULL_L = 20000, 33


def _pull_ids(kind, rng, n):
    if kind == "random":
        return rng.integers(0, _PULL_ROWS, n)
    ids = np.sort(rng.choice(_PULL_ROWS, n, replace=False))
    if kind == "last_pair" and n > 1:
        ids[-2], ids[-1] = ids[-1], ids[-2]
    if kind == "equal":
        ids = np.full(n, int(rng.integers(0, _PULL_ROWS)))
    return ids


@pytest.fixture(scope="module")
def pull_table():
    rng = np.random.default_rng(5)
    table = rng.uniform(-1, 1, (_PULL_ROWS, _PULL_L)).astype(np.float32)
    kv = mx.kv.create("device")
    kv.init("e", mx.nd.row_sparse_array(table, ctx=G))
    return kv, table


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unique+gather"])
@pytest.mark.parametrize("kind", ["random", "last_pair", "equal", "increasing"])
@pytest.mark.parametrize("n", [1, 1024, 1025, 8193, 16383, 16384, 16385])
def test_row_sparse_pull_sizes(n, kind, fused, pull_table, monkeypatch):
    """n ids around the unique kernels' edges: 1024 / 1025 (the scan's chunk), 8193 (npad doubles), 16384
    (kUniqueMax: 128 KB of shared memory, npad = n), 16385 (the global bitonic sort); random with repeats, strictly
    increasing but for the last pair (the fast path fails at its very end), all equal, strictly increasing (the fast
    path); ids as int64, int32, float32 and float64; 33-wide rows (the gather's scalar branch); an output that holds
    exactly the unique rows and one that holds more."""
    _path(monkeypatch, fused)
    kv, table = pull_table
    rng = np.random.default_rng(n * 4 + len(kind))
    ids = _pull_ids(kind, rng, n)
    want = O.sparse_retain(O.RowSparse(np.arange(_PULL_ROWS), table, table.shape), O.unique(ids.astype(np.int64)))
    nu = len(want.indices)
    assert np.array_equal(want.indices, np.unique(ids))
    for dt in (np.int64, np.int32, np.float32, np.float64):
        for cap in (nu, n + 5):
            out = mx.nd.empty(table.shape, G, stype="row_sparse", capacity=cap)
            before = mx.kv.launch_count()
            kv.row_sparse_pull("e", out=out, row_ids=mx.nd.array(ids.astype(dt), G, dtype=dt))
            launches = mx.kv.launch_count() - before - (dt != np.int64)
            got_idx = out.indices.asnumpy()
            assert len(got_idx) == nu, (dt, cap)
            assert np.array_equal(got_idx, want.indices), (dt, cap)
            got = out.data.asnumpy().reshape(-1, _PULL_L)
            assert _bits_equal(got, want.data.reshape(-1, _PULL_L)), (dt, cap)
            assert _bits_equal(got, table[np.unique(ids)]), (dt, cap)
            if fused and n <= 16384:
                assert launches == 1, "the fused pull is one launch (%d)" % launches
            else:
                assert launches >= 2, launches


# ---- 64-bit offsets ----------------------------------------------------------------------------------------------
def test_tables_above_2_31_elements(monkeypatch):
    """One row_sparse key of 8 388 617 x 260 float32 (2.18e9 elements, 8.7 GB): lazy SGD on rows whose offset
    id * 260 is above 2^31, through the fused push and the four-kernel push, read back with the fused pull and with
    the unique + gather kernels; then, on a second table of that size, one standard SGD step (the dense kernel over
    all 2.18e9 elements), sampled at rows with and without a gradient, including the last.  The oracle and the float64
    model run on a compact table of the sampled rows (every update here is row by row)."""
    if SIM:
        pytest.skip("an 8.7 GB table does not fit the simulated runtime's host memory")
    import torch
    if torch.cuda.mem_get_info(0)[0] < 24 * 2 ** 30:
        pytest.skip("needs 24 GB of free GPU memory (two 8.7 GB tables one after the other, and a dense gradient)")
    rows, L = 8_388_617, 260
    shape = (rows, L)
    assert rows * L > 2 ** 31
    rng = np.random.default_rng(31)
    edge = 2 ** 31 // L
    pool = np.unique(np.concatenate([[0, 1, edge - 1, edge, edge + 1, rows // 2], np.arange(rows - 40, rows)]))
    pool = pool.astype(np.int64)

    def compact(srcs):
        return [(np.searchsorted(pool, i).astype(np.int64), v) for i, v in srcs]

    def pull(kv, key, ids):
        out = mx.nd.empty(shape, G, stype="row_sparse", capacity=len(ids))
        kv.row_sparse_pull(key, out=out, row_ids=mx.nd.array(ids, G, dtype=np.int64))
        assert np.array_equal(out.indices.asnumpy(), np.unique(ids))
        return out.data.asnumpy().reshape(-1, L)

    # lazy SGD on a table that starts at zero
    kw = dict(learning_rate=0.1, wd=0.01, rescale_grad=0.5, lazy_update=True)
    kv = mx.kv.create("device")
    kv.init("big", mx.nd.row_sparse_array((np.zeros((1, L), np.float32), np.zeros(1, np.int64)), shape=shape, ctx=G))
    kv.set_optimizer(mx.optimizer.SGD(**kw))
    cshape = (len(pool), L)
    okv = O.OracleKVStore("device")
    okv.init(0, np.zeros(cshape, np.float32))
    okv.set_optimizer(O.OracleOptimizer("sgd", **kw))
    model = Model("sgd", kw)
    w = np.zeros(cshape, np.float32)
    for step, fused in enumerate((True, False)):
        _path(monkeypatch, fused)
        srcs = _values(rng, [np.sort(rng.choice(pool, 30, replace=False)) for _ in range(2)], L)
        before = mx.kv.launch_count()
        kv.push("big", [_mk(i, v, shape, G) for i, v in srcs])
        assert (mx.kv.launch_count() - before == 1) == fused
        okv.push(0, [O.RowSparse(i, v, cshape) for i, v in compact(srcs)])
        for pull_fused in (True, False):
            _path(monkeypatch, pull_fused)
            got = pull(kv, "big", pool[::-1].copy())
            assert _bits_equal(got, okv.local[0]), (step, pull_fused)
        model.check(w, [], compact(srcs), got)
        w = got
    del kv
    gc.collect()
    mx.nd.waitall()

    # one standard SGD step over the whole second table
    kw = dict(learning_rate=0.1, wd=0.25, rescale_grad=1.0, lazy_update=False)
    init_ids = pool[1::2]                       # (rows - 1 among them)
    assert init_ids[-1] == rows - 1
    init_val = rng.uniform(-1, 1, (len(init_ids), L)).astype(np.float32)
    kv = mx.kv.create("device")
    kv.init("big2", _mk(init_ids, init_val, shape, G))
    kv.set_optimizer(mx.optimizer.SGD(**kw))
    gids = np.sort(rng.choice(pool, 20, replace=False))
    gval = rng.uniform(-1, 1, (len(gids), L)).astype(np.float32)
    kv.push("big2", [_mk(gids, gval, shape, G)])
    w0 = np.zeros(cshape, np.float32)
    w0[np.searchsorted(pool, init_ids)] = init_val
    want = w0.copy()
    (ci, cv), = compact([(gids, gval)])
    O.sgd_std_rsp(want, O.RowSparse(ci, cv, cshape), kw["learning_rate"], kw["wd"], kw["rescale_grad"])
    got = pull(kv, "big2", pool)
    assert _bits_equal(got, want)
    Model("sgd", kw).check(w0, [], [(ci, cv)], got)
    assert not _bits_equal(got[-1], w0[-1]), "the last row was not updated"
    del kv
    gc.collect()
    mx.nd.waitall()


# ---- peers -------------------------------------------------------------------------------------------------------
@pytest.mark.multigpu
@pytest.mark.parametrize("L", [33, 132])
def test_multi_gpu_localise_phase(L, monkeypatch):
    """The fused kernel's P1 (every source's id list copied into local memory) on each replica: one value per GPU
    (2 ... 4) read in place from its peer, one more from the host; lazy SGD-momentum, row_sparse_pull from every
    device after every push."""
    _path(monkeypatch, True)
    devs = list(range(min(mx.num_gpus(), 4)))
    rng = np.random.default_rng(L)
    rows = 1001
    shape = (rows, L)
    kw = dict(learning_rate=0.1, momentum=0.9, wd=1e-4, lazy_update=True)
    w0 = rng.uniform(-1, 1, shape).astype(np.float32)
    kv = mx.kv.create("device")
    kv.init(0, mx.nd.row_sparse_array(w0, ctx=G))
    kv.set_optimizer(mx.optimizer.SGD(**kw))
    okv = O.OracleKVStore("device")
    okv.init(0, O.RowSparse.from_dense(w0))
    okv.set_optimizer(O.OracleOptimizer("sgd", **kw))
    ctxs = [mx.gpu(d) for d in devs] + [mx.cpu()]
    for step in range(3):
        srcs = _values(rng, _pattern("random", rng, rows, len(ctxs)), L)
        kv.push(0, [_mk(i, v, shape, c) for (i, v), c in zip(srcs, ctxs)])
        okv.push(0, [O.RowSparse(i, v, shape) for i, v in srcs])
        ids = rng.integers(0, rows, 700).astype(np.int64)
        want = O.sparse_retain(okv.local[0], O.unique(ids))
        for d in devs:
            out = mx.nd.empty(shape, mx.gpu(d), stype="row_sparse", capacity=700)
            kv.row_sparse_pull(0, out=out, row_ids=mx.nd.array(ids, mx.gpu(d), dtype=np.int64))
            assert np.array_equal(out.indices.asnumpy(), want.indices)
            assert _bits_equal(out.data.asnumpy(), want.data.reshape(-1, L)), (step, d)
