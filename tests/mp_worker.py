"""Worker of tests/test_gpu_multi.py::test_mp_one_process_per_gpu (launched by torchrun).
Every rank regenerates every rank's data from seeds, so each can check itself against the oracle."""
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SIM = bool(os.environ.get("MXKV_SIM"))      # tests/sim: stand-in CUDA runtime, no torch, files as the process group
if not SIM:
    import torch
    import torch.distributed as dist
import mxnet_b200 as mx          # noqa: E402
from oracle import oracle as O   # noqa: E402


def bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def tree_scenario(rank, world, local, ctx, data, device_sync, allgather_int):
    # 10. MXNET_KVSTORE_USETREE=1 (CommDeviceTree): with three ranks or more the sums go pairwise up the trees the
    #     reference's solver builds from the ranks' link matrix -- whole keys up tree 0, keys above the bound by row
    #     slices, slice i up the tree rooted at rank i -- whatever the engine's own sharding of the key is; with an
    #     optimizer on the store the update consumes that sum.  Oracle: comm_tree.h restated level by level.
    if world >= 3:
        os.environ["MXNET_KVSTORE_USETREE"] = "1"
        os.environ["MXNET_KVSTORE_TREE_ARRAY_BOUND"] = "4000"
        try:
            devs = allgather_int(local)
            topo, scan, depth = mx.topology.compute_trees(mx.topology.query_links(devs), 0.7, False)
            tree = dict(topo=topo, scan=scan, depth=depth, bound=4000)
            shapes = [(1000,), (37, 13), (64, 33), (70001,), (300, 257), ((1 << 20) + 77,)]
            ks = list(range(len(shapes)))
            kvt = mx.kv.create("device")
            kvt.init(ks, [mx.nd.zeros(s, ctx) for s in shapes])
            n0 = mx.kv.launch_count("tree")
            differs = 0
            for kind in ("plain", "symmetric"):
                vals, outs = [], []
                for k, s in zip(ks, shapes):
                    v = mx.nd.empty_symmetric(s) if kind == "symmetric" else mx.nd.empty(s, ctx)
                    v[:] = data(900 + k, s, rank)
                    vals.append(v)
                    outs.append(mx.nd.empty_symmetric(s) if kind == "symmetric" else mx.nd.empty(s, ctx))
                device_sync()
                kvt.pushpull(ks, vals, out=outs)
                for k, s, o in zip(ks, shapes, outs):
                    srcs = [data(900 + k, s, r) for r in range(world)]
                    want = O.sum_tree(srcs, topo, scan, depth, 4000)
                    differs += int(not bits_equal(want, O.sum_device(srcs)))
                    assert bits_equal(o.asnumpy(), want), ("tree allreduce", kind, s)
            assert mx.kv.launch_count("tree") > n0, "the tree kernel did not run"
            assert differs > 0, "tree order indistinguishable from the plain order on this data"
            for optname, kw in (("sgd", dict(learning_rate=0.1, momentum=0.9, wd=1e-4)), ("adam", dict(learning_rate=0.01))):
                kvo = mx.kv.create("device")
                w0 = [data(950 + k, s, 0) for k, s in zip(ks, shapes)]
                kvo.init(ks, [mx.nd.array(w, ctx) for w in w0])
                kvo.set_optimizer(mx.optimizer.create(optname, **kw))
                okv = O.OracleKVStore("device", tree=tree)
                okv.init(ks, [w.copy() for w in w0])
                okv.set_optimizer(O.OracleOptimizer(optname, **kw))
                outs = [mx.nd.empty_symmetric(s) for s in shapes]
                gsym = [mx.nd.empty_symmetric(s) for s in shapes]
                for step in range(3):
                    for k, s in zip(ks, shapes):
                        gsym[k][:] = data(960 + 10 * step + k, s, rank)
                    device_sync()
                    kvo.pushpull(ks, gsym, out=outs)
                    okv.push(ks, [[data(960 + 10 * step + k, s, r) for r in range(world)] for k, s in zip(ks, shapes)])
                for k, s in zip(ks, shapes):
                    want = np.empty(s, np.float32)
                    okv.pull(k, want)
                    assert bits_equal(outs[k].asnumpy(), want), ("tree " + optname, s)
        finally:
            del os.environ["MXNET_KVSTORE_USETREE"], os.environ["MXNET_KVSTORE_TREE_ARRAY_BOUND"]


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    if SIM:
        sys.path.insert(0, os.path.join(ROOT, "tests", "sim"))
        from file_comm import FileComm
        comm = FileComm(rank, world, os.environ["MXKV_SIM_RDV"])
        mx.dist.init_with_allgather(rank, world, local, comm.allgather)
        device_sync, barrier, allgather_int = mx.nd.waitall, comm.barrier, comm.allgather_int
    else:
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        mx.dist.init_process_group(device=local)
        device_sync, barrier = torch.cuda.synchronize, dist.barrier

        def allgather_int(x):
            chk = torch.tensor([int(x)], dtype=torch.int64).cuda()
            allc = [torch.empty_like(chk) for _ in range(world)]
            dist.all_gather(allc, chk)
            return [int(c) for c in allc]
    ctx = mx.gpu(local)
    # The arena's arrays may carry an NVSwitch multicast alias (engine-owned VMM arena): above 4 ranks the engine
    # would then pick the multimem kernel on its own, whose in-switch sum is not bit-identical to the reference's
    # left-to-right order.  Everything below except scenario 7 asserts bits: keep to the peer-memory kernels.
    mx.kv.set_nvls(0)

    def data(seed, shape, r):
        return np.random.default_rng(seed * 1000 + r).uniform(-1, 1, shape).astype(np.float32)

    if os.environ.get("MXKV_MP_ARENA_ONLY"):
        # tests/test_sim_host_logic.py::test_engine_owned_arena_and_its_fallbacks: which arena came up (every rank must
        # agree), and that it works: symmetric arrays of several segments' worth, a sharded and an unsharded key
        have = [bool(mx.nd.has_multicast(mx.nd.empty_symmetric((1024,)))) for _ in range(2)]
        assert all(h == have[0] for h in have)
        assert len(set(allgather_int(int(have[0])))) == 1, "the ranks disagree on the kind of arena"
        want_mc = os.environ["MXKV_MP_ARENA_ONLY"] == "multicast"
        assert have[0] == want_mc, ("arena kind", have[0], want_mc)
        kva = mx.kv.create("device")
        shapes = [(3000,), (1 << 20,), ((1 << 22) + 12,)]
        kva.init(list(range(len(shapes))), [mx.nd.zeros(s, ctx) for s in shapes])
        for rep in range(3):                      # (more arena than one 16 MB segment: a later segment is created)
            vals = [mx.nd.empty_symmetric(s) for s in shapes]
            outs = [mx.nd.empty_symmetric(s) for s in shapes]
            for k, s in enumerate(shapes):
                vals[k][:] = data(1200 + 10 * rep + k, s, rank)
            device_sync(); barrier()
            kva.pushpull(list(range(len(shapes))), vals, out=outs)
            for k, s in enumerate(shapes):
                want = O.sum_device([data(1200 + 10 * rep + k, s, r) for r in range(world)])
                assert bits_equal(outs[k].asnumpy(), want), ("arena", rep, k)
        mx.nd.waitall()
        barrier()
        print("MP_WORKER_OK rank", rank, "multicast" if have[0] else "ipc", flush=True)
        return

    if os.environ.get("MXKV_MP_TREE_ONLY"):
        # tests/test_gpu_zzz_tree.py::test_one_process_per_gpu_under_the_tree: scenario 10 alone (it has not met
        # hardware yet; the scenarios below have, and stay as they ran)
        tree_scenario(rank, world, local, ctx, data, device_sync, allgather_int)
        mx.nd.waitall()
        barrier()
        print("MP_WORKER_OK rank", rank, flush=True)
        if not SIM:
            dist.destroy_process_group()
        return

    # 1. init/broadcast: rank 0's value wins
    kv = mx.kv.create("device")
    assert kv.rank == rank and kv.num_workers == world
    shape = (300, 7)
    out = mx.nd.empty(shape, ctx)
    kv.broadcast("w", mx.nd.array(data(1, shape, rank), ctx), out=out)
    assert bits_equal(out.asnumpy(), data(1, shape, 0)), "broadcast"

    # 2. allreduce (no optimizer): one-shot and two-shot sizes; plain, symmetric and torch arrays
    sizes = [5, 1000, 65536, 70001, (1 << 20) + 3, 3_000_001]
    keys = list(range(len(sizes)))
    kv.init([str(k) for k in keys], [mx.nd.zeros((e,), ctx) for e in sizes])
    for mode in ("plain", "symmetric", "host") if SIM else ("plain", "symmetric", "torch", "host"):
        vals, outs, keep = [], [], []
        for k, e in zip(keys, sizes):
            src = data(2 + k, (e,), rank)
            if mode == "symmetric":
                v = mx.nd.empty_symmetric((e,)); v[:] = src
                o = mx.nd.empty_symmetric((e,))
            elif mode == "torch":
                t = torch.from_numpy(src).cuda(); keep.append(t)
                v = mx.nd.from_torch(t)
                to = torch.empty(e, device="cuda"); keep.append(to)
                o = mx.nd.from_torch(to)
            elif mode == "host":
                v = mx.nd.array(src, mx.cpu_pinned())
                o = mx.nd.empty((e,), mx.cpu_pinned())
            else:
                v = mx.nd.array(src, ctx)
                o = mx.nd.empty((e,), ctx)
            vals.append(v); outs.append(o)
        device_sync()
        kv.pushpull([str(k) for k in keys], vals, out=outs)
        for k, e, o in zip(keys, sizes, outs):
            want = O.sum_device([data(2 + k, (e,), r) for r in range(world)])
            assert bits_equal(o.asnumpy(), want), ("allreduce", mode, e)
    # in-place
    for e, k in zip(sizes, keys):
        v = mx.nd.array(data(50 + k, (e,), rank), ctx)
        kv.pushpull(str(k), v)
        want = O.sum_device([data(50 + k, (e,), r) for r in range(world)])
        assert bits_equal(v.asnumpy(), want), ("inplace", e)

    # 3. fused optimizers over a key list, several steps
    for optname, kw in (("sgd", dict(learning_rate=0.1, momentum=0.9, wd=1e-4, rescale_grad=0.5)),
                        ("adam", dict(learning_rate=0.01, wd=1e-3))):
        shapes = [(64,), (513, 9), (1 << 19,), (1 << 21,)]
        ks = list(range(len(shapes)))
        kv2 = mx.kv.create("device")
        w0 = [data(7 + k, s, 0) for k, s in zip(ks, shapes)]
        kv2.init(ks, [mx.nd.array(w, ctx) for w in w0])
        kv2.set_optimizer(mx.optimizer.create(optname, **kw))
        okv = O.OracleKVStore("device")
        okv.init(ks, [w.copy() for w in w0])
        okv.set_optimizer(O.OracleOptimizer(optname, **kw))
        outs = [mx.nd.empty_symmetric(s) for s in shapes]
        gsym = [mx.nd.empty_symmetric(s) for s in shapes]
        for step in range(3):
            for k, s in zip(ks, shapes):
                gsym[k][:] = data(100 * step + k, s, rank)
            kv2.pushpull(ks, gsym, out=outs)
            okv.push(ks, [[data(100 * step + k, s, r) for r in range(world)] for k, s in zip(ks, shapes)])
            for k, s in zip(ks, shapes):
                want = np.empty(s, np.float32)
                okv.pull(k, want)
                assert bits_equal(outs[k].asnumpy(), want), (optname, step, k)
        if optname == "adam":
            # sharded state: save on every rank (gathers), reload into a fresh store, continue
            # a private directory: a fixed name under /tmp may be held by another user's earlier run
            f = os.path.join(tempfile.mkdtemp(prefix="mxkv_states_"), "states_%d_%d" % (world, rank))
            kv2.save_optimizer_states(f, dump_optimizer=True)     # with its update counts
            mids = [o.asnumpy() for o in outs]
            kv3 = mx.kv.create("device")
            kv3.init(ks, [mx.nd.array(m, ctx) for m in mids])
            kv3.set_optimizer(mx.optimizer.create(optname, **kw))
            kv3.load_optimizer_states(f)
            shutil.rmtree(os.path.dirname(f))
            outs3 = [mx.nd.empty(s, ctx) for s in shapes]
            for k, s in zip(ks, shapes):
                gsym[k][:] = data(900 + k, s, rank)
            kv2.pushpull(ks, gsym, out=outs)
            kv3.pushpull(ks, gsym, out=outs3)
            for k in ks:
                assert bits_equal(outs[k].asnumpy(), outs3[k].asnumpy()), ("reload", k)

    # 4. python updater callback (every rank applies it to its own replica)
    kv4 = mx.kv.create("device")
    kv4.init(3, mx.nd.zeros((4, 4), ctx))
    kv4._set_updater(lambda key, recv, local: local.__iadd__(recv))
    for it in range(1, 3):
        kv4.push(3, mx.nd.ones((4, 4), ctx))
        o = mx.nd.empty((4, 4), ctx)
        kv4.pull(3, out=o)
        assert np.all(o.asnumpy() == it * world), "callback"

    # 5. row_sparse: lazy SGD-momentum over the ranks' sparse gradients + row_sparse_pull
    rows, L, nnz = 3000, 64, 200
    shape = (rows, L)
    w0 = data(31, shape, 0)
    kw = dict(learning_rate=0.1, momentum=0.9, wd=1e-4, lazy_update=True)
    kv5 = mx.kv.create("device")
    kv5.init("emb", mx.nd.row_sparse_array(w0, ctx=ctx))
    kv5.set_optimizer(mx.optimizer.SGD(**kw))
    okv = O.OracleKVStore("device")
    okv.init("emb", O.RowSparse.from_dense(w0))
    okv.set_optimizer(O.OracleOptimizer("sgd", **kw))

    def rsp(seed, r):
        g = np.random.default_rng(seed * 100 + r)
        idx = np.sort(g.choice(rows, nnz, replace=False)).astype(np.int64)
        return idx, g.uniform(-1, 1, (nnz, L)).astype(np.float32)
    for step in range(3):
        i, v = rsp(step, rank)
        kv5.push("emb", mx.nd.row_sparse_array((v, i), shape=shape, ctx=ctx))
        okv.push("emb", [O.RowSparse(*rsp(step, r), shape) for r in range(world)])
        ids = np.random.default_rng(step).integers(0, rows, 300).astype(np.int64)
        out = mx.nd.empty(shape, ctx, stype="row_sparse", capacity=300)
        kv5.row_sparse_pull("emb", out=out, row_ids=mx.nd.array(ids, ctx, dtype=np.int64))
        want = O.sparse_retain(okv.local["emb"], O.unique(ids))
        assert np.array_equal(out.indices.asnumpy(), want.indices), "rsp idx"
        assert bits_equal(out.data.asnumpy(), want.data.reshape(-1, L)), ("rsp", step)

    # 5b. a DENSE weight updated on the store by alternating dense (sharded) and row_sparse gradients
    kw = dict(learning_rate=0.01, wd=1e-3, lazy_update=False)
    kv5b = mx.kv.create("device")
    kv5b.init("w", mx.nd.array(w0, ctx))
    kv5b.set_optimizer(mx.optimizer.Adam(**kw))
    okv = O.OracleKVStore("device")
    okv.init("w", w0.copy())
    okv.set_optimizer(O.OracleOptimizer("adam", **kw))
    for step, kind in enumerate(["dense", "rsp", "dense", "rsp", "rsp"]):
        if kind == "rsp":
            i, v = rsp(10 + step, rank)
            kv5b.push("w", mx.nd.row_sparse_array((v, i), shape=shape, ctx=ctx))
            okv.push("w", [O.RowSparse(*rsp(10 + step, r), shape) for r in range(world)])
        else:
            kv5b.push("w", mx.nd.array(data(40 + step, shape, rank), ctx))
            okv.push("w", [data(40 + step, shape, r) for r in range(world)])
        o = mx.nd.empty(shape, ctx)
        kv5b.pull("w", out=o)
        assert bits_equal(o.asnumpy(), okv.local["w"]), ("dense key, rsp grads", step, kind)

    # 6. 2-bit gradient compression with error feedback, one code stream per rank
    E, thr = 30000, 0.5
    kv6 = mx.kv.create("device")
    kv6.set_gradient_compression({"type": "2bit", "threshold": thr})
    kv6.init("c", mx.nd.zeros((E,), ctx))
    residual = [np.zeros(E, np.float32) for _ in range(world)]
    for step in range(3):
        out = mx.nd.empty((E,), ctx)
        kv6.pushpull("c", mx.nd.array(data(70 + step, (E,), rank), ctx), out=out)
        deq = [O.dequantize_2bit(O.quantize_2bit(data(70 + step, (E,), r), residual[r], thr), E, thr)
               for r in range(world)]
        assert bits_equal(out.asnumpy(), O.sum_device(deq)), ("compression", step)

    # 7. NVLS: arrays bound to an NVSwitch multicast object -> multimem.ld_reduce / multimem.st kernel.
    #    The switch's summation order is not left-to-right: tolerance 1e-6 relative (the reference's
    #    own bound) against the oracle, and bit-identical replicas across ranks.
    allocs = []
    if mx.nd.has_multicast(mx.nd.empty_symmetric((1024,))):          # engine-owned multicast arena (vmm_arena.cc)
        allocs.append(("engine", mx.nd.empty_symmetric))
    if not SIM:
        try:
            if mx.nd.has_multicast(mx.nd.empty_multicast((1024,))):  # memory of torch's symmetric-memory allocator
                allocs.append(("torch", mx.nd.empty_multicast))
        except Exception as e:          # torch symmetric memory unavailable
            print("torch multicast unavailable:", repr(e), flush=True)
    print("NVLS allocators:", [a for a, _ in allocs], flush=True)
    for alloc_name, empty_mc in allocs:
        mx.kv.set_nvls(2)            # FORCE the multimem kernel at every world size (auto: above 4 ranks only)
        nv0 = mx.kv.launch_count("nvls")
        # the bench sweep's sizes in one call (every rank regenerates every rank's data: bounded for large worlds)
        big = [(1 << p,) for p in range(10, (25 if world <= 2 else 23) if not SIM else 19, 2)]   # (CPU: up to 2^18)
        small = [(1 << 10,), (3 * (1 << 16),), (1 << 21,)]
        sgd = dict(learning_rate=0.1, momentum=0.9, wd=1e-4)
        expected = 0
        # (requests in flight per thread, pipelined, grid cap, block size): the default and the corners of the
        # tuning space (tools/tune_nvls.py) -- every instantiation that may become the default is compared
        cfgs = [(2, 0, 48, 512), (4, 1, 0, 512), (1, 0, 32, 256), (8, 1, 64, 512), (2, 1, 148, 512)]
        if SIM:
            cfgs = cfgs[:4]
        for ci, cfg in enumerate(cfgs if alloc_name == allocs[0][0] else cfgs[:1]):
            mx.kv.set_nvls_tuning(*cfg)
            cases = [(None, {}, small), ("sgd", sgd, small), ("sgd", dict(sgd, learning_rate=0.01), big),
                     ("adam", dict(learning_rate=0.001, wd=1e-3), big), (None, {}, big)] if ci == 0 else \
                    [("sgd", sgd, small), ("adam", dict(learning_rate=0.001, wd=1e-3), small), (None, {}, small)]
            for optname, kw, shapes in cases:
                ks = list(range(len(shapes)))
                kv7 = mx.kv.create("device")
                w0 = [data(41 + k, s, 0) for k, s in zip(ks, shapes)]
                kv7.init(ks, [mx.nd.array(w, ctx) for w in w0])
                okv = O.OracleKVStore("device")
                okv.init(ks, [w.copy() for w in w0])
                if optname:
                    kv7.set_optimizer(mx.optimizer.create(optname, **kw))
                    okv.set_optimizer(O.OracleOptimizer(optname, **kw))
                gm = [empty_mc(s) for s in shapes]
                om = [empty_mc(s) for s in shapes]
                before = mx.kv.launch_count()
                for step in range(3):
                    for k, s in zip(ks, shapes):
                        gm[k][:] = data(300 + 10 * step + k, s, rank)
                    device_sync(); barrier()
                    kv7.pushpull(ks, gm, out=om)
                    okv.push(ks, [[data(300 + 10 * step + k, s, r) for r in range(world)] for k, s in zip(ks, shapes)])
                    for k, s in zip(ks, shapes):
                        want = np.empty(s, np.float32)
                        okv.pull(k, want)
                        got = om[k].asnumpy()
                        err = np.abs(got.astype(np.float64) - want).sum() / max(np.abs(want).sum(), 1e-30)
                        assert err < 1e-6, ("nvls", cfg, optname, step, k, err)
                        chk = int(got.view(np.int32).astype(np.int64).sum())
                        assert all(c == chk for c in allgather_int(chk)), ("nvls replicas differ", cfg, optname, step, k)
                assert mx.kv.launch_count() - before == 3, "one launch per pushpull expected"
                expected += 3
        assert mx.kv.launch_count("nvls") - nv0 == expected, "the multimem kernel did not serve every pushpull"
        mx.kv.set_nvls_tuning(2, 0, 48, 512)
        mx.kv.set_nvls(0)
        print("NVLS_OK", alloc_name, "rank", rank, flush=True)

    # 7b. the peer-memory kernels, each variant FORCED (VERDICT r1 weak #1): the shared-memory staged kernel
    #     (cp.async.bulk from peer HBM) and the per-thread kernel over the bench sweep's sizes in one call and
    #     one key per call, two-shot and one-shot, SGD momentum / Adam / plain sum, bit-exact
    big = [1 << p for p in (range(10, 19, 2) if SIM else range(10, 25 if world <= 2 else 23, 2))]
    for variant, bulk in (("bulk", 2), ("per_thread", 0)):
        mx.kv.set_tuning(bulk=bulk)
        c0 = {v: mx.kv.launch_count(v) for v in ("bulk", "per_thread")}
        for optname, kw in ((None, {}), ("sgd", dict(learning_rate=0.01, momentum=0.9, wd=1e-4)),
                            ("adam", dict(learning_rate=0.001, wd=1e-3))):
            for group in ([big] + [[e] for e in big[::2]]):
                ks = list(range(len(group)))
                kvb = mx.kv.create("device")
                w0 = [data(51 + k, (e,), 0) for k, e in zip(ks, group)]
                kvb.init(ks, [mx.nd.array(w, ctx) for w in w0])
                okv = O.OracleKVStore("device")
                okv.init(ks, [w.copy() for w in w0])
                if optname:
                    kvb.set_optimizer(mx.optimizer.create(optname, **kw))
                    okv.set_optimizer(O.OracleOptimizer(optname, **kw))
                gs = [mx.nd.empty_symmetric((e,)) for e in group]
                outs = [mx.nd.empty_symmetric((e,)) for e in group]
                for step in range(2):
                    for k, e in zip(ks, group):
                        gs[k][:] = data(400 + 10 * step + k, (e,), rank)
                    device_sync(); barrier()
                    kvb.pushpull(ks, gs, out=outs)
                    okv.push(ks, [[data(400 + 10 * step + k, (e,), r) for r in range(world)] for k, e in zip(ks, group)])
                    for k, e in zip(ks, group):
                        want = np.empty(e, np.float32)
                        okv.pull(k, want)
                        assert bits_equal(outs[k].asnumpy(), want), ("forced", variant, optname, step, e)
        other = "per_thread" if variant == "bulk" else "bulk"
        assert mx.kv.launch_count(variant) > c0[variant] and mx.kv.launch_count(other) == c0[other], \
            ("forced variant did not hold", variant)
    mx.kv.set_tuning(bulk=1)

    # 8. layer-wise adaptive optimizers: sharded keys take the norms across the ranks' shards, small
    #    keys are updated redundantly; replicas must stay bit-identical across ranks
    for optname, kw in (("lamb", dict(learning_rate=0.01, wd=0.01)),
                        ("lans", dict(learning_rate=0.01, wd=0.01)),
                        ("lars", dict(learning_rate=0.1, momentum=0.9, wd=1e-3, eta=0.01)),
                        ("lamb", dict(learning_rate=0.01, wd=0.01, skip_nonfinite=True))):
        shapes = [(64,), (513, 9), (1 << 19,), (1 << 21,)]
        ks = list(range(len(shapes)))
        kv8 = mx.kv.create("device")
        w0 = [data(61 + k, s, 0) for k, s in zip(ks, shapes)]
        kv8.init(ks, [mx.nd.array(w, ctx) for w in w0])
        kv8.set_optimizer(mx.optimizer.create(optname, **kw))
        okw = {k: v for k, v in kw.items() if k != "skip_nonfinite"}
        oopt = O.OracleOptimizer(optname, norm_mode="f64", **okw)
        ow = [w.copy() for w in w0]
        outs = [mx.nd.empty(s, ctx) for s in shapes]
        for step in range(3):
            overflow = kw.get("skip_nonfinite") and step == 1

            def grad(k, s, r):
                g = data(500 + 10 * step + k, s, r)
                if overflow and k == 0 and r == world - 1:
                    g.flat[3] = np.inf
                return g
            kv8.pushpull(ks, [mx.nd.array(grad(k, s, rank), ctx) for k, s in zip(ks, shapes)], out=outs)
            if kw.get("skip_nonfinite"):
                assert kv8.overflow() == bool(overflow), ("overflow flag", step)
            for k, s in zip(ks, shapes):
                if not overflow:
                    oopt.update(k, ow[k], O.sum_device([grad(k, s, r) for r in range(world)]).reshape(s))
                got = outs[k].asnumpy()
                np.testing.assert_allclose(got, ow[k], rtol=2e-6, atol=2e-7, err_msg=str((optname, step, k)))
                chk = int(got.view(np.int32).astype(np.int64).sum())
                assert all(c == chk for c in allgather_int(chk)), ("replicas differ", optname, step, k)

    # 9. random walks (every rank draws the same walk from a shared seed): key subsets, plain / symmetric /
    #    host-resident gradients and outputs, pushes and fused pushpulls, pulls, every optimizer family
    opts = [(None, {}), ("sgd", dict(learning_rate=0.05, momentum=0.9, wd=1e-3)), ("adam", dict(learning_rate=0.01, wd=1e-3)),
            ("adamw", dict(learning_rate=0.01, wd=0.05)), ("lars", dict(learning_rate=0.1, momentum=0.9, wd=1e-3, eta=0.01))]
    for walk in range(5 * (1 + int(os.environ.get("MXKV_FUZZ_SEEDS", "0")))):      # soak runs: more walks
        wr = np.random.default_rng(31337 + walk)               # the walk itself: identical on every rank
        optname, kw = opts[walk % len(opts)]
        layerwise = optname == "lars"
        sizes = [int(x) for x in wr.choice([5, 640, 4099, 70001, 300007], size=3, replace=False)]
        ks = ["r%d" % i for i in range(len(sizes))]
        kv9 = mx.kv.create("device")
        w0 = [data(700 + 10 * walk + i, (e,), 0) for i, e in enumerate(sizes)]
        kv9.init(ks, [mx.nd.array(w, ctx) for w in w0])
        okv = O.OracleKVStore("device")
        okv.init(ks, [w.copy() for w in w0])
        if optname:
            kv9.set_optimizer(mx.optimizer.create(optname, **kw))
            okv.set_optimizer(O.OracleOptimizer(optname, **(dict(kw, norm_mode="f64") if layerwise else kw)))

        def same(got, want, what):
            if layerwise:
                np.testing.assert_allclose(got, want, rtol=5e-6, atol=5e-7, err_msg=str(what))
            else:
                assert bits_equal(got, want), what

        for step in range(6):
            sub = sorted(wr.choice(len(ks), size=int(wr.integers(1, len(ks) + 1)), replace=False).tolist())
            kind = str(wr.choice(["plain", "symmetric", "host"]))
            fused_pull = bool(wr.integers(0, 2))
            seed0 = 800 + 100 * walk + 10 * step

            def make(e):
                if kind == "symmetric":
                    return mx.nd.empty_symmetric((e,))
                return mx.nd.empty((e,), mx.cpu_pinned() if kind == "host" else ctx)
            vals = []
            for k in sub:
                v = make(sizes[k]); v[:] = data(seed0 + k, (sizes[k],), rank); vals.append(v)
            names = [ks[k] for k in sub]
            device_sync()
            if fused_pull:
                outs = [make(sizes[k]) for k in sub]
                kv9.pushpull(names, vals, out=outs)
            else:
                kv9.push(names, vals)
                outs = [mx.nd.empty((sizes[k],), ctx) for k in sub]
                kv9.pull(names, out=outs)
            okv.push(names, [[data(seed0 + k, (sizes[k],), r) for r in range(world)] for k in sub])
            for k, o in zip(sub, outs):
                want = np.empty(sizes[k], np.float32)
                okv.pull(ks[k], want)
                got = o.asnumpy()
                same(got, want, ("walk", walk, optname, step, k, kind, fused_pull))
                chk = int(got.view(np.int32).astype(np.int64).sum())
                assert all(c == chk for c in allgather_int(chk)), ("walk replicas differ", walk, step, k)
                if layerwise:
                    okv.local[ks[k]][...] = got

    mx.nd.waitall()
    barrier()
    print("MP_WORKER_OK rank", rank, flush=True)
    if not SIM:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
