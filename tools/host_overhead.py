"""Host-side cost of one pushpull call (Python marshalling + the engine's C++ bookkeeping), measured on the
simulated CUDA runtime with kernel launches turned into no-ops -- no GPU needed:

    python tests/sim/build_sim.py
    MXKV_SIM=1 MXKV_SIM_NOEXEC=1 MXKV_SIM_DEVICES=4 \\
    MXKV_B200_LIBRARY_PATH=$PWD/tests/sim/_build/libmxkv_b200_sim.so python tools/host_overhead.py

Launches are asynchronous on a real GPU, so this cost is hidden as long as it stays below the kernel time of
the same call; when it does not (hundreds of small keys, several GPUs driven by one process) the step becomes
host-bound."""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mxnet_b200 as mx                                            # noqa: E402
from mxnet_b200.kvstore import _ctype_key_value, _c_keys, _c_vals  # noqa: E402


def bench(nkeys, opt, ndev=1, elems=4, steps=300):
    kv = mx.kv.create("device")
    keys = list(range(nkeys))
    kv.init(keys, [mx.nd.zeros((elems,), mx.gpu(0)) for _ in keys])
    if opt:
        kv.set_optimizer(mx.optimizer.create(opt))
    if ndev == 1:
        grads = [mx.nd.ones((elems,), mx.gpu(0)) for _ in keys]
        outs = [mx.nd.empty((elems,), mx.gpu(0)) for _ in keys]
    else:
        grads = [[mx.nd.ones((elems,), mx.gpu(d)) for d in range(ndev)] for _ in keys]
        outs = [[mx.nd.empty((elems,), mx.gpu(d)) for d in range(ndev)] for _ in keys]
    for _ in range(5):
        kv.pushpull(keys, grads, out=outs)

    def call():
        kv.pushpull(keys, grads, out=outs)

    def marshal():                      # the Python share of a call: (cached) marshalling + update counts
        packed = kv._marshalled(1, keys, grads, outs)
        kv._advance_counts(packed[0])

    def best(fn):                       # the machine is shared: best of five batches
        out = []
        for _ in range(5):
            t = time.perf_counter()
            for _ in range(steps // 5):
                fn()
            out.append((time.perf_counter() - t) / (steps // 5))
        return min(out)
    total, py = best(call), best(marshal)
    print("%4d keys  %-5s  %d GPU(s): %7.1f us per pushpull = python %6.1f + native %7.1f  (%.2f us per key per GPU native)"
          % (nkeys, opt, ndev, total * 1e6, py * 1e6, (total - py) * 1e6, (total - py) * 1e6 / nkeys / ndev))


if __name__ == "__main__":
    assert os.environ.get("MXKV_SIM") and os.environ.get("MXKV_SIM_NOEXEC"), __doc__
    for nk in (1, 9, 199):
        bench(nk, "sgd")
    for opt in ("adam", "lamb", None):
        bench(199, opt)
    for nd in (2, 4):
        bench(199, "sgd", ndev=nd)
    bench(199, "lamb", ndev=4)
