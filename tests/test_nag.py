"""NAG on the store without a GPU: the oracle against the reference's own `NAG.step` (golden/nag_steps.npz), the
kernels' NAG arithmetic compiled for the host against the oracle bit for bit, the per-key scalars the fused kernel
receives, and tests/test_gpu_nag.py plus a one-process-per-GPU worker (tests/nag_mp_worker.py) on the simulated CUDA
runtime (tests/sim).

Counterpart of the reference's tests/python/unittest/test_optimizer.py::test_nag (NAG.step against nag_mom_update /
mp_nag_mom_update, rtol 1e-3, atol 1e-4): the reference's step pins the oracle (tests/nag_oracle.py) through the
fixture tests/golden/make_nag_golden.py writes, and the oracle pins the kernels -- here their arithmetic compiled for
the host, in tests/test_gpu_nag.py their launches on the GPU."""
import ast
import ctypes
import glob
import importlib.util
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import mxnet_b200 as mx
from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import nag_oracle as N  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "sim")
F32P = ctypes.POINTER(ctypes.c_float)


def _bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def test_oracle_matches_the_reference_step_golden():
    """nag_steps.npz: the reference's NAG.step (nag.py:72-109) over 8 option sets x 4 shapes x 5 steps; the oracle's
    restatement of the fused kernels (nag_mom_update, sgd_update at momentum 0) within the reference's own
    fused-vs-step tolerance of test_nag (rtol 1e-3, atol 1e-4)"""
    d = np.load(os.path.join(ROOT, "tests", "golden", "nag_steps.npz"))
    worst = 0.0
    for ci, meta in enumerate(d["cases"]):
        name, lr, wd, kw = ast.literal_eval(str(meta))
        for si in range(4):
            tag = "c%d_s%d" % (ci, si)
            opt = N.OracleNAG(learning_rate=lr, wd=wd, **kw)
            w = d["w0_" + tag].reshape(-1).copy()
            for t in range(5):
                opt.update(0, w, d["g%d_%s" % (t, tag)].reshape(-1).copy())
                want = d["w%d_%s" % (t + 1, tag)].reshape(-1)
                np.testing.assert_allclose(w, want, rtol=1e-3, atol=1e-4, err_msg="%s step %d" % (tag, t))
                worst = max(worst, float(np.max(np.abs(w.astype(np.float64) - want))))
    print("largest |oracle - reference step|: %.3g" % worst)
    assert worst < 1e-5


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no C++ compiler")
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("CUDA headers not installed")
    so = str(tmp_path_factory.mktemp("nag_host") / "libnag_host.so")
    subprocess.run([gxx, "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-Werror",
                    "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "incubator-mxnet_b200", "csrc"), "-I", cuda_inc,
                    os.path.join(ROOT, "tests", "c", "nag_host.cc"), "-o", so], check=True, capture_output=True)
    return ctypes.CDLL(so)


def _host_nag(host, g, w, mom, lr, wd, rescale, clip, momentum, mp):
    f = ctypes.c_float
    p = lambda a: a.ctypes.data_as(F32P)       # noqa: E731
    assert host.host_nag(ctypes.c_int64(w.size), p(g), p(w), p(mom), f(lr), f(wd), f(rescale),
                         f(-1.0 if clip is None else clip), f(momentum), ctypes.c_int(mp)) == 0


@pytest.mark.parametrize("clip", [None, 0.4])
@pytest.mark.parametrize("flavour", ["f32", "lp", "mp"])
def test_kernel_arithmetic_on_the_host_is_the_oracle_bit_for_bit(host, flavour, clip):
    """float32 keys and 16-bit keys without multi_precision: NAGMomKernel's (w + momentum*mom) - lr*r; 16-bit keys
    with multi_precision: MP_NAGMomKernel's w + (momentum*mom - lr*r) on the fp32 master"""
    rng = np.random.default_rng(11)
    n = 20011
    w1 = rng.uniform(-1, 1, n).astype(np.float32)
    w2, m1, m2 = w1.copy(), np.zeros(n, np.float32), np.zeros(n, np.float32)
    for t in range(4):
        g = rng.uniform(-2, 2, n).astype(np.float32)
        args = (0.1, 1e-3, 0.9)
        _host_nag(host, g, w1, m1, 0.1, 1e-3, 0.5, clip, 0.9, flavour == "mp")
        if flavour == "f32":
            N.nag_mom_update(w2, g, m2, 0.1, 1e-3, 0.9, 0.5, clip)
        else:
            for kind in (1, 2):       # the rounding to the key type is the store's, after the update
                fn = N.mp_nag_mom_update if flavour == "mp" else N.lp_nag_mom_update
                ww, mm = w2.copy(), m2.copy()
                fn(np.zeros(n, np.uint16), kind, ww, mm, g, *args, 0.5, clip)
            fn(None, 0, w2, m2, g, *args, 0.5, clip)
        assert _bits_equal(w1, w2) and _bits_equal(m1, m2), (flavour, t)


def _key_hyper(kv, key):
    from mxnet_b200.base import _LIB, check_call
    lr, wd, eta = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
    check_call(_LIB.MXKVB200GetKeyHyper(kv.handle, int(key), None, ctypes.byref(lr), ctypes.byref(wd), ctypes.byref(eta)))
    return np.float32(lr.value), np.float32(wd.value), np.float32(eta.value)


def test_per_key_scalars_defaults_and_multipliers():
    """what the fused kernel receives per key: the reference class's defaults (learning_rate 0.1, nag.py:58) for a
    C caller that names "nag" alone, lr_mult / wd_mult, and no bias correction at any update count"""
    from mxnet_b200.base import _LIB, check_call
    kv = mx.kv.create("device")
    kv.init([0, 1], [mx.nd.zeros((4,)), mx.nd.zeros((4,))])
    check_call(_LIB.MXKVB200SetOptimizer(kv.handle, b"nag", 0, None, None))
    for t in (0, 1, 7, 1000):
        check_call(_LIB.MXKVB200SetUpdateCount(kv.handle, 0, None, ctypes.c_int64(t)))
        assert _key_hyper(kv, 0) == (np.float32(0.1), np.float32(0.0), np.float32(1.0))
    assert mx.optimizer.create("nag").learning_rate == 0.1 and mx.optimizer.create("nag").momentum == 0.9
    opt = mx.optimizer.NAG(learning_rate=0.03, momentum=0.5, wd=0.02)
    opt.set_lr_mult({1: 0.5})
    opt.set_wd_mult({1: 3.0})
    kv.set_optimizer(opt)
    assert opt.fused_kwargs()["momentum"] == 0.5
    assert _key_hyper(kv, 0) == (np.float32(0.03), np.float32(0.02), np.float32(1.0))
    assert _key_hyper(kv, 1) == (np.float32(0.015), np.float32(0.06), np.float32(1.0))
    # momentum 0 is the plain SGD update (checked numerically on the simulated runtime below): same scalars
    kv.set_optimizer(mx.optimizer.NAG(learning_rate=0.2, momentum=0.0))
    assert _key_hyper(kv, 0)[0] == np.float32(0.2)
    assert mx.optimizer.NAG(momentum=0.0).create_state(0, None) is None


# ---------------------------------------------------------------------------
# the simulated CUDA runtime
# ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sim_lib():
    if shutil.which("g++") is None or not os.path.exists("/usr/local/cuda/bin/nvcc"):
        pytest.skip("needs g++ and nvcc to build the simulated runtime")
    spec = importlib.util.spec_from_file_location("build_sim", os.path.join(SIM, "build_sim.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    lib, _ = b.build()
    return lib


@pytest.mark.parametrize("devices", [1, 2, 4, 8])
def test_gpu_nag_on_the_simulator(sim_lib, devices):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_B200_LIBRARY_PATH=sim_lib, MXKV_SIM_DEVICES=str(devices))
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_gpu_nag.py")],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    import re
    m = re.search(r"(\d+) passed", r.stdout)
    # torch-based tests skip next to the stand-in runtime; the multi-GPU ones need two simulated GPUs or more
    assert m and int(m.group(1)) >= (12 if devices == 1 else 13), r.stdout[-1000:]


def _run_workers(sim_lib, world, tmp_path, extra):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_SIM_MP="1", MXKV_SIM_RDV=str(tmp_path), MXKV_B200_LIBRARY_PATH=sim_lib,
               MXKV_SIM_DEVICES=str(world), MXKV_B200_ARENA_MB="256", WORLD_SIZE=str(world), **extra)
    procs = []
    for r in range(world):
        e = dict(env, RANK=str(r), LOCAL_RANK=str(r))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "nag_mp_worker.py")], env=e,
                                      cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            out, _ = p.communicate(timeout=900)
            outs.append(out)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for p in procs:
            for f in glob.glob("/dev/shm/mxkvsim_%d_*" % p.pid):
                os.unlink(f)
    for r, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d:\n%s" % (r, out[-3000:])
        assert "NAG_WORKER_OK rank %d" % r in out, out[-2000:]
    return outs


@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_process_per_gpu_on_the_simulator(sim_lib, world, tmp_path):
    """two-shot keys with sharded momentum, a checkpoint of it on every rank, and the multicast kernel forced
    (the engine-owned multicast arena of tests/sim/fake_driver.cc): within 1e-6 of the oracle"""
    outs = _run_workers(sim_lib, world, tmp_path, {})
    assert all("NAG_NVLS_OK" in o for o in outs), outs[0][-2000:]


@pytest.mark.parametrize("world", [3, 8])
def test_one_process_per_gpu_under_the_tree_on_the_simulator(sim_lib, world, tmp_path):
    _run_workers(sim_lib, world, tmp_path, {"MXKV_NAG_TREE": "1"})
