"""Sweep the scheduling of the multicast (NVLS) kernel -- requests in flight per thread, software pipelining,
grid, block size -- and, beside it, the peer-load kernels and NCCL's own all-reduce on the same box, on the
bench workload (BASELINE.json configs[1] key set).  Run under torchrun with N >= 2:

  python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29571 tools/tune_nvls.py

One line per configuration: ms per pushpull (CUDA events, max over ranks), busbw 2S(n-1)/n/t and the link
bytes per direction S(1+1/n)/t of the multicast path.  Every configuration's plain all-reduce result is
checked against the known sum (rank r pushes (r+1) * base)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mxnet_b200 as mx                      # noqa: E402
from bench import keyset, nelem              # noqa: E402


def timed(fn, steps, world, warm=4):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize(); dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / steps], device="cuda", dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    mx.dist.init_process_group(device=local)
    shapes = keyset(os.environ.get("TUNE_WORKLOAD", "sweep"))
    S = 4 * sum(nelem(s) for s in shapes)
    keys = list(range(len(shapes)))
    steps = int(os.environ.get("TUNE_STEPS", 30))
    base = [np.random.default_rng(7 + k).uniform(-1, 1, s).astype(np.float32) for k, s in enumerate(shapes)]
    have_mc = False
    engine_mc = mx.nd.has_multicast(mx.nd.empty_symmetric((1024,)))      # engine-owned multicast arena
    try:
        have_mc = engine_mc or mx.nd.has_multicast(mx.nd.empty_multicast((1024,)))
    except Exception as e:      # noqa: BLE001
        if rank == 0:
            print("multicast unavailable:", repr(e), flush=True)
    if rank == 0:
        print("multicast memory:", "engine-owned (VMM arena)" if engine_mc else ("torch" if have_mc else "none"), flush=True)

    def say(tag, ms):
        if rank == 0:
            print("%-46s %.4f ms  busbw %6.1f GB/s  nvls-link %6.1f GB/s/dir" % (
                tag, ms, 2.0 * S * (world - 1) / world / (ms * 1e-3) / 1e9, S * (1 + 1.0 / world) / (ms * 1e-3) / 1e9),
                flush=True)

    # ---- NCCL all-reduce of the same bytes (one flat buffer and key by key), same process, same box
    flat = torch.empty(S // 4, device="cuda", dtype=torch.float32).uniform_(-1, 1)
    say("nccl all_reduce flat %d MB" % (S >> 20), timed(lambda: dist.all_reduce(flat), steps, world))
    per_key = [torch.empty(nelem(s), device="cuda", dtype=torch.float32).uniform_(-1, 1) for s in shapes]

    def nccl_keys():
        for t in per_key:
            dist.all_reduce(t)
    say("nccl all_reduce key by key (%d calls)" % len(shapes), timed(nccl_keys, steps, world))
    del flat, per_key

    for optname in os.environ.get("TUNE_OPTS", "none,sgd").split(","):
        for alloc_name in (("multicast", "symmetric") if have_mc else ("symmetric",)):
            alloc = mx.nd.empty_multicast if (alloc_name == "multicast" and not engine_mc) else mx.nd.empty_symmetric
            grads = [alloc(s) for s in shapes]
            weights = [alloc(s) for s in shapes]
            for g, b in zip(grads, base):
                g[:] = b * np.float32(rank + 1)
            kv = mx.kv.create("device")
            kv.init(keys, [mx.nd.zeros(s, mx.gpu(local)) for s in shapes])
            if optname == "sgd":
                kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.01, momentum=0.9, wd=1e-4))
            elif optname == "adam":
                kv.set_optimizer(mx.optimizer.Adam(learning_rate=0.001))

            def step():
                kv.pushpull(keys, grads, out=weights)

            def check(tag):
                if optname != "none":
                    return
                k = len(shapes) - 2                      # the 64 MB key (two-shot) and the smallest (one-shot)
                for kk in (0, k):
                    got = weights[kk].asnumpy().astype(np.float64)
                    want = base[kk].astype(np.float64) * (world * (world + 1) / 2.0)
                    err = np.abs(got - want).sum() / np.abs(want).sum()
                    assert err < 1e-6, (tag, kk, err)

            if alloc_name == "symmetric":
                mx.kv.set_nvls(0)
                for bulk in (2, 0):
                    mx.kv.set_tuning(bulk=bulk)
                    ms = timed(step, steps, world)
                    check("p2p")
                    say("%s p2p %s" % (optname, "bulk" if bulk else "per-thread"), ms)
                mx.kv.set_tuning(bulk=1)
                mx.kv.set_nvls(1)
            else:
                mx.kv.set_nvls(2)
                grids = [int(x) for x in os.environ.get("TUNE_GRIDS", "0,132,96,64,48,32,24,16").split(",")]
                quick = bool(os.environ.get("TUNE_QUICK"))      # the default configuration only
                for threads in ((512,) if quick else (512, 256)):
                    for pipe in ((0,) if quick else (0, 1)):
                        for unroll in ((2,) if quick else (1, 2, 4, 8)):
                            for grid in grids:
                                if threads == 256 and grid not in (0, 132, 32):
                                    continue
                                mx.kv.set_nvls_tuning(unroll=unroll, pipe=pipe, grid=grid, threads=threads)
                                n0 = mx.kv.launch_count("nvls")
                                ms = timed(step, steps, world, warm=3)
                                assert mx.kv.launch_count("nvls") > n0
                                tag = "%s nvls U=%d pipe=%d grid=%d thr=%d" % (optname, unroll, pipe, grid, threads)
                                check(tag)
                                say(tag, ms)
                mx.kv.set_nvls_tuning(unroll=2, pipe=0, grid=0, threads=512)
                mx.kv.set_nvls(1)
            mx.nd.waitall()
            del kv, grads, weights
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
