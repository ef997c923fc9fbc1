"""One-process-per-GPU worker for Adamax on the store (tests/test_adamax.py, simulated runtime): fused Adamax over a key
list with one-shot and two-shot (sharded) keys, its two sharded states (mean, var) gathered, saved with the update counts
on every rank and loaded into a fresh store that continues at the next count, the multicast kernel forced where the
arena has a multicast alias, and -- with MXKV_STEP_OPT_TREE=1 -- the sum of the reference's tree order feeding the
update.  Every rank regenerates every rank's data from seeds and checks itself.  tests/adadelta_mp_worker.py runs the
same ``main`` for AdaDelta."""
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "sim"))
import mxnet_b200 as mx          # noqa: E402
from oracle import oracle as O   # noqa: E402
from file_comm import FileComm   # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import adamax_oracle as A         # noqa: E402

KW = dict(learning_rate=0.002, beta1=0.5, beta2=0.9, wd=1e-4, rescale_grad=0.5, clip_gradient=0.7)


def bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def data(seed, shape, r):
    return np.random.default_rng(seed * 1000 + r).uniform(-1, 1, shape).astype(np.float32)


def main(cls=mx.optimizer.Adamax, oracle_cls=A.OracleAdamax, kw=KW, marker="ADAMAX"):
    def stores(ks, shapes, ctx, tree=None):
        w0 = [data(7 + k, s, 0) for k, s in zip(ks, shapes)]
        kv = mx.kv.create("device")
        kv.init(ks, [mx.nd.array(w, ctx) for w in w0])
        kv.set_optimizer(cls(**kw))
        okv = O.OracleKVStore("device", tree=tree)
        okv.init(ks, [w.copy() for w in w0])
        okv.set_optimizer(oracle_cls(**kw))
        return kv, okv

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    comm = FileComm(rank, world, os.environ["MXKV_SIM_RDV"])
    mx.dist.init_with_allgather(rank, world, rank, comm.allgather)
    ctx = mx.gpu(rank)
    mx.kv.set_nvls(0)

    if os.environ.get("MXKV_STEP_OPT_TREE"):
        os.environ["MXNET_KVSTORE_USETREE"] = "1"
        os.environ["MXNET_KVSTORE_TREE_ARRAY_BOUND"] = "4000"
        devs = comm.allgather_int(rank)
        topo, scan, depth = mx.topology.compute_trees(mx.topology.query_links(devs), 0.7, False)
        tree = dict(topo=topo, scan=scan, depth=depth, bound=4000)
        shapes = [(1000,), (64, 33), (70001,), (300, 257)]
        ks = list(range(len(shapes)))
        kv, okv = stores(ks, shapes, ctx, tree)
        outs = [mx.nd.empty(s, ctx) for s in shapes]
        t0 = mx.kv.launch_count("tree")
        for step in range(3):
            vals = [mx.nd.array(data(500 + 10 * step + k, s, rank), ctx) for k, s in zip(ks, shapes)]
            mx.nd.waitall(); comm.barrier()
            kv.pushpull(ks, vals, out=outs)
            okv.push(ks, [[data(500 + 10 * step + k, s, r) for r in range(world)] for k, s in zip(ks, shapes)])
            for k, s in zip(ks, shapes):
                want = np.empty(s, np.float32)
                okv.pull(k, want)
                assert bits_equal(outs[k].asnumpy(), want), ("tree", step, k)
        assert mx.kv.launch_count("tree") > t0, "the tree kernel did not run"
        mx.nd.waitall(); comm.barrier()
        print(marker + "_WORKER_OK rank", rank, "tree", flush=True)
        return

    # the fused update over one-shot and two-shot keys, then the two sharded states and the counts through a checkpoint
    shapes = [(64,), (513, 9), (1 << 19,), ((1 << 20) + 12,)]
    ks = list(range(len(shapes)))
    kv, okv = stores(ks, shapes, ctx)
    outs = [mx.nd.empty_symmetric(s) for s in shapes]
    gsym = [mx.nd.empty_symmetric(s) for s in shapes]

    def step(store, seed, check=True):
        for k, s in zip(ks, shapes):
            gsym[k][:] = data(seed + k, s, rank)
        mx.nd.waitall(); comm.barrier()
        store.pushpull(ks, gsym, out=outs)
        okv.push(ks, [[data(seed + k, s, r) for r in range(world)] for k, s in zip(ks, shapes)])
        for k, s in zip(ks, shapes):
            want = np.empty(s, np.float32)
            okv.pull(k, want)
            assert bits_equal(outs[k].asnumpy(), want), (marker, seed, k)
    for i in range(3):
        step(kv, 100 * i)
    for k in ks:      # GetState gathers the shards of every state array onto this rank
        for which, want in zip((2, 3), okv.optimizer.states[k]):
            assert bits_equal(kv._state_handle(k, which).asnumpy().reshape(-1), want.reshape(-1)), ("state", which, k)
    d = tempfile.mkdtemp(prefix="mxkv_%s_states_" % marker.lower())
    f = os.path.join(d, "states_%d_%d" % (world, rank))
    kv.save_optimizer_states(f, dump_optimizer=True)
    kv2 = mx.kv.create("device")
    kv2.init(ks, [mx.nd.array(o.asnumpy(), ctx) for o in outs])
    kv2.set_optimizer(cls(**kw))
    kv2.load_optimizer_states(f)
    shutil.rmtree(d)
    assert [kv2._optimizer._index_update_count[k] for k in ks] == [3] * len(ks)
    for i in range(3, 5):
        step(kv2, 100 * i)

    # the multicast kernel (in-switch sum: 1e-6 relative to the oracle, identical replicas on every rank)
    if mx.nd.has_multicast(mx.nd.empty_symmetric((1024,))):
        mx.kv.set_nvls(2)
        nv0 = mx.kv.launch_count("nvls")
        shapes = [(1 << 10,), (3 * (1 << 16),), (1 << 18,)]
        ks = list(range(len(shapes)))
        gm = [mx.nd.empty_symmetric(s) for s in shapes]
        om = [mx.nd.empty_symmetric(s) for s in shapes]
        for i in range(6):
            if i == 0:
                kv7, okv7 = stores(ks, shapes, ctx)
            for k, s in zip(ks, shapes):
                gm[k][:] = data(300 + 10 * i + k, s, rank)
            mx.nd.waitall(); comm.barrier()
            kv7.pushpull(ks, gm, out=om)
            okv7.push(ks, [[data(300 + 10 * i + k, s, r) for r in range(world)] for k, s in zip(ks, shapes)])
            for k, s in zip(ks, shapes):
                want = np.empty(s, np.float32)
                okv7.pull(k, want)
                got = om[k].asnumpy()
                err = np.abs(got.astype(np.float64) - want).sum() / max(np.abs(want).sum(), 1e-30)
                assert err < 1e-6, ("nvls", i, k, err)
                chk = int(got.view(np.int32).astype(np.int64).sum())
                assert all(c == chk for c in comm.allgather_int(chk)), ("nvls replicas differ", i, k)
        assert mx.kv.launch_count("nvls") - nv0 == 6, "the multimem kernel did not serve every pushpull"
        mx.kv.set_nvls(0)
        print(marker + "_NVLS_OK rank", rank, flush=True)
    mx.nd.waitall(); comm.barrier()
    print(marker + "_WORKER_OK rank", rank, flush=True)


if __name__ == "__main__":
    main()
