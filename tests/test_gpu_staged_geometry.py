"""The staged dense kernel at the ring geometries its plan picks for a launch without a rendezvous: 4096-element tiles
for kinds with at most one state array (no optimizer, SGD-momentum, NAG, RMSProp, Signum), 2048 for the wider ones
(Adam, centered RMSProp, FTML), 1024 when many sources leave no room for more.  Every thread takes its columns of a
tile into registers and the block releases the stage before anyone stores, so these sizes put partial last tiles,
tiles of a few elements and keys smaller than one tile on each side of every tile width, against the oracle bit for
bit."""
import pytest

from test_gpu_dense import _run_keyset

pytestmark = pytest.mark.gpu

# multiples of 4 elements around 1024, 2048 and 4096: ragged last tiles of every width the plan picks
RAGGED = [4, 1020, 2052, 4092, 4100, 2 * 4096 + 12, 3 * 4096 - 4, (1 << 20) + 4, 12]


@pytest.mark.parametrize("n", [1, 2])
@pytest.mark.parametrize("optkey", ["none", "sgd_mom"])
def test_staged_wide_tiles_ragged(optkey, n):
    """4096-element tiles (three staged arrays at n = 1), and the 2048-element fallback of a fourth array (n = 2)"""
    _run_keyset("bulk", optkey, n, RAGGED, steps=2, seed=41 + n)


@pytest.mark.parametrize("n", [1, 3])
def test_staged_state_kinds_ragged(n):
    """Adam: two state arrays, 2048-element tiles of two register columns per thread"""
    _run_keyset("bulk", "adam", n, RAGGED, steps=2, seed=51 + n)


def test_staged_many_sources_narrow_tiles():
    """ten sources of SGD-momentum: twelve staged arrays, 1024-element tiles"""
    _run_keyset("bulk", "sgd_mom", 10, [4, 1028, 4096 + 8, 100004], steps=2, seed=61)


def test_resident_work_list_follows_every_change():
    """a pushpull whose work list is byte-for-byte the last one reads the device's resident copy without an upload;
    every other list replaces it.  Key sets alternate (A, A, B, A, B, B), one list is too long to be resident and the
    learning rate changes between two identical key sets: every step bit-exact against the oracle"""
    import numpy as np
    import mxnet_b200 as mx
    from oracle import oracle as O
    from test_gpu_dense import _rng, assert_bits_equal

    kw = dict(learning_rate=0.01, momentum=0.9, wd=1e-4)
    sizes = [4, 4100, 70004, 12] + [8] * 320           # the last 320 keys: a list past the resident capacity
    rng = _rng(71)
    keys = list(range(len(sizes)))
    w0 = [rng.uniform(0, 1, e).astype(np.float32) for e in sizes]
    kv = mx.kv.create("device")
    kv.init(keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
    opt = mx.optimizer.SGD(**kw)
    kv.set_optimizer(opt)
    okv = O.OracleKVStore("device")
    okv.init(keys, [w.copy() for w in w0])
    oopt = O.OracleOptimizer("sgd", **kw)
    okv.set_optimizer(oopt)
    grads = [rng.uniform(-1, 1, e).astype(np.float32) for e in sizes]
    gdev = [mx.nd.array(g, mx.gpu(0)) for g in grads]
    outs = [mx.nd.empty((e,), mx.gpu(0)) for e in sizes]
    sets = {"A": [0, 1], "B": [1, 2, 3], "all": keys}
    for step, name in enumerate(["A", "A", "B", "A", "all", "B", "B", "lr", "lr"]):
        ks = sets["A" if name == "lr" else name]
        if name == "lr" and step == 7:
            opt.set_learning_rate(0.005)
            oopt.lr = 0.005
        kv.pushpull(ks, [gdev[k] for k in ks], out=[outs[k] for k in ks])
        okv.push(ks, [[grads[k]] for k in ks])
        for k in ks:
            want = np.empty(sizes[k], np.float32)
            okv.pull(k, want)
            assert_bits_equal(outs[k].asnumpy(), want, "step %d (%s) key %d" % (step, name, k))
