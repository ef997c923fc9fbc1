"""AdaBelief on the store without a GPU: the oracle against the reference's own `AdaBelief.step`
(golden/adabelief_steps.npz), the kernels' AdaBelief arithmetic compiled for the host against the oracle bit for bit,
the per-key scalars the fused kernel receives, and tests/test_gpu_adabelief.py plus a one-process-per-GPU worker
(tests/adabelief_mp_worker.py) on the simulated CUDA runtime (tests/sim).

Counterpart of the reference's tests/python/unittest/test_optimizer.py::test_adabelief (AdaBelief.step against the fused
operators, rtol 1e-3, atol 2e-3): the reference's step pins the oracle (tests/adabelief_oracle.py) through the fixture
tests/golden/make_adabelief_golden.py writes, and the oracle pins the kernels -- here their arithmetic compiled for the
host, in tests/test_gpu_adabelief.py their launches on the GPU."""
import ast
import ctypes
import glob
import importlib.util
import math
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

import mxnet_b200 as mx
from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import adabelief_oracle as A  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "sim")
F32P = ctypes.POINTER(ctypes.c_float)


def _bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def test_oracle_matches_the_reference_step_golden():
    """adabelief_steps.npz: the reference's AdaBelief.step (adabelief.py:96-139) over 8 option sets x 4 shapes x 5
    steps; the oracle's restatement of MultiMPAdaBeliefKernel within the reference's own fused-vs-step tolerance of
    test_adabelief (rtol 1e-3, atol 2e-3)"""
    d = np.load(os.path.join(ROOT, "tests", "golden", "adabelief_steps.npz"))
    worst = 0.0
    for ci, meta in enumerate(d["cases"]):
        name, lr, wd, kw = ast.literal_eval(str(meta))
        assert name == "adabelief"
        for si in range(4):
            tag = "c%d_s%d" % (ci, si)
            opt = A.OracleAdaBelief(learning_rate=lr, wd=wd, **kw)
            w = d["w0_" + tag].reshape(-1).copy()
            for t in range(5):
                opt.update(0, w, d["g%d_%s" % (t, tag)].reshape(-1).copy())
                want = d["w%d_%s" % (t + 1, tag)].reshape(-1)
                np.testing.assert_allclose(w, want, rtol=1e-3, atol=2e-3, err_msg="%s step %d" % (tag, t))
                worst = max(worst, float(np.max(np.abs(w.astype(np.float64) - want))))
    # The fused grouping beta2*(var - adj) + adj cancels where beta2 is close to 1 (the first step computes
    # adj - 0.999*adj), so the fused operators sit further from exact arithmetic than `step` does: 6.6e-5 on this
    # data (beta1 0.5, beta2 0.999), while `step` stays within 4e-7 of a float64 evaluation.
    print("largest |oracle - reference step|: %.3g" % worst)
    assert worst < 2e-4


def test_golden_option_grid_exercises_every_option():
    """both values of correct_bias occur, and the clip binds on the gradient with the wd term added in a set with
    wd > 0 (with rescale_grad 0.14 it cannot bind: that set only pairs the two values)"""
    d = np.load(os.path.join(ROOT, "tests", "golden", "adabelief_steps.npz"))
    cases = [ast.literal_eval(str(m)) for m in d["cases"]]
    assert {c[3]["correct_bias"] for c in cases} == {True, False}
    binds = []
    for ci, (_, lr, wd, kw) in enumerate(cases):
        if kw["clip_gradient"] is None:
            continue
        g = d["g0_c%d_s3" % ci] * np.float32(kw["rescale_grad"]) + np.float32(wd) * d["w0_c%d_s3" % ci]
        if np.abs(g).max() > kw["clip_gradient"]:
            binds.append(wd)
    assert any(wd > 0 for wd in binds), binds


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no C++ compiler")
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("CUDA headers not installed")
    so = str(tmp_path_factory.mktemp("adabelief_host") / "libadabelief_host.so")
    subprocess.run([gxx, "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-Werror",
                    "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "incubator-mxnet_b200", "csrc"), "-I", cuda_inc,
                    os.path.join(ROOT, "tests", "c", "adabelief_host.cc"), "-o", so], check=True, capture_output=True)
    return ctypes.CDLL(so)


def _host_adabelief(host, g, w, mean, var, eta, wd, beta1, beta2, eps, rescale, clip):
    f = ctypes.c_float
    p = lambda a: a.ctypes.data_as(F32P)       # noqa: E731
    assert host.host_adabelief(ctypes.c_int64(w.size), p(g), p(w), p(mean), p(var), f(1.0), f(eta), f(wd), f(beta1),
                               f(beta2), f(eps), f(rescale), f(-1.0 if clip is None else clip)) == 0


@pytest.mark.parametrize("wd", [0.0, 0.03])
@pytest.mark.parametrize("clip", [None, 0.4])
@pytest.mark.parametrize("flavour", ["f32", "lp"])
def test_kernel_arithmetic_on_the_host_is_the_oracle_bit_for_bit(host, flavour, clip, wd):
    """update_one<OPT_ADABELIEF> against MultiMPAdaBeliefKernel's restatement: float32 keys, and the fp32 master of
    16-bit keys with the stored weight its one rounding to float16 / bfloat16"""
    rng = np.random.default_rng(12)
    n = 20011
    w1 = rng.uniform(-1, 1, n).astype(np.float32)
    w2 = w1.copy()
    s1 = [np.zeros(n, np.float32), np.zeros(n, np.float32)]
    s2 = [np.zeros(n, np.float32), np.zeros(n, np.float32)]
    bound = False
    for t in range(1, 5):
        g = rng.uniform(-2, 2, n).astype(np.float32)
        eta = float(np.float32(A.bias_corrected_lr(0.01, 0.9, 0.999, t)))
        args = (eta, wd, 0.9, 0.999, 1e-6, 0.5)
        _host_adabelief(host, g, w1, s1[0], s1[1], *args, clip)
        if flavour == "f32":
            A.adabelief_update(w2, g, s2[0], s2[1], *args, clip)
        else:
            for kind in (1, 2):       # the rounding to the key type is the store's, after the update
                ww, mm, vv, lp = w2.copy(), s2[0].copy(), s2[1].copy(), np.zeros(n, np.uint16)
                A.lp_adabelief_update(lp, kind, ww, mm, vv, g, *args, clip)
                want = ww.astype(np.float16).view(np.uint16) if kind == 1 else O.f32_to_bf16(ww)
                assert np.array_equal(lp, want)
            A.lp_adabelief_update(None, 0, w2, s2[0], s2[1], g, *args, clip)
        assert _bits_equal(w1, w2) and _bits_equal(s1[0], s2[0]) and _bits_equal(s1[1], s2[1]), (flavour, t)
        if clip is not None:
            bound = bound or bool(np.any(np.abs(np.float32(0.5) * g + np.float32(wd) * w2) > clip))
    assert clip is None or bound


def _key_hyper(kv, key):
    from mxnet_b200.base import _LIB, check_call
    lr, wd, eta = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
    check_call(_LIB.MXKVB200GetKeyHyper(kv.handle, int(key), None, ctypes.byref(lr), ctypes.byref(wd), ctypes.byref(eta)))
    return np.float32(lr.value), np.float32(wd.value), np.float32(eta.value)


def _bc(lr, b1, b2, t):
    """the reference class's lr_t in double (adabelief.py:174-181)"""
    return lr * math.sqrt(1. - b2 ** t) / (1. - b1 ** t)


def test_per_key_scalars_defaults_and_multipliers():
    """what the fused kernel receives per key: operator lr = 1 and operator eta = the bias-corrected learning rate at
    the key's update count (the plain learning rate with correct_bias=False), the multipliers, and the reference
    class's defaults (learning_rate 0.001, beta1 0.9, beta2 0.999, adabelief.py:79) for a C caller that names
    "adabelief" alone"""
    from mxnet_b200.base import _LIB, check_call
    kv = mx.kv.create("device")
    kv.init([0, 1], [mx.nd.zeros((4,)), mx.nd.zeros((4,))])
    check_call(_LIB.MXKVB200SetOptimizer(kv.handle, b"adabelief", 0, None, None))
    for t in (1, 2, 7, 1000):
        check_call(_LIB.MXKVB200SetUpdateCount(kv.handle, 0, None, ctypes.c_int64(t)))
        lr, wd, eta = _key_hyper(kv, 0)
        assert (lr, wd) == (np.float32(1.0), np.float32(0.0))
        assert eta == np.float32(A.bias_corrected_lr(0.001, 0.9, 0.999, t))
        assert abs(eta - _bc(0.001, 0.9, 0.999, t)) <= 1e-7 * _bc(0.001, 0.9, 0.999, t)
    opt = mx.optimizer.create("adabelief")
    assert isinstance(opt, mx.optimizer.AdaBelief)
    assert (opt.learning_rate, opt.beta1, opt.beta2, opt.epsilon, opt.correct_bias) == (0.001, 0.9, 0.999, 1e-6, True)
    assert mx.optimizer.fused_name_of(opt) == "adabelief"
    opt = mx.optimizer.AdaBelief(learning_rate=0.03, beta1=0.5, beta2=0.8, epsilon=1e-4, wd=0.02)
    opt.set_lr_mult({1: 0.5})
    opt.set_wd_mult({1: 3.0})
    kv.set_optimizer(opt)
    kw = opt.fused_kwargs()
    assert (kw["beta1"], kw["beta2"], kw["epsilon"], kw["correct_bias"]) == (0.5, 0.8, 1e-4, True)
    for k, lr, wd in ((0, 0.03, 0.02), (1, 0.015, 0.06)):
        check_call(_LIB.MXKVB200SetUpdateCount(kv.handle, k, None, ctypes.c_int64(3)))
        assert _key_hyper(kv, k) == (np.float32(1.0), np.float32(wd), np.float32(A.bias_corrected_lr(lr, 0.5, 0.8, 3)))
    kv.set_optimizer(mx.optimizer.AdaBelief(learning_rate=0.2, correct_bias=False))
    for t in (1, 5):
        check_call(_LIB.MXKVB200SetUpdateCount(kv.handle, 0, None, ctypes.c_int64(t)))
        assert _key_hyper(kv, 0) == (np.float32(1.0), np.float32(0.0), np.float32(0.2))


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
def test_gpu_adabelief_on_the_simulator(sim_lib, devices):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_B200_LIBRARY_PATH=sim_lib, MXKV_SIM_DEVICES=str(devices))
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_gpu_adabelief.py")],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    m = re.search(r"(\d+) passed", r.stdout)
    # torch-based tests skip next to the stand-in runtime; the multi-GPU ones need two simulated GPUs or more
    assert m and int(m.group(1)) >= (19 if devices == 1 else 20), r.stdout[-1000:]


def _run_workers(sim_lib, world, tmp_path, extra):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_SIM_MP="1", MXKV_SIM_RDV=str(tmp_path), MXKV_B200_LIBRARY_PATH=sim_lib,
               MXKV_SIM_DEVICES=str(world), MXKV_B200_ARENA_MB="256", WORLD_SIZE=str(world), **extra)
    procs = []
    for r in range(world):
        e = dict(env, RANK=str(r), LOCAL_RANK=str(r))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "adabelief_mp_worker.py")], env=e,
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
        assert "ADABELIEF_WORKER_OK rank %d" % r in out, out[-2000:]
    return outs


@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_process_per_gpu_on_the_simulator(sim_lib, world, tmp_path):
    """two-shot keys with sharded mean / variance, a checkpoint of them on every rank, and the multicast kernel forced
    (the engine-owned multicast arena of tests/sim/fake_driver.cc): within 1e-6 of the oracle"""
    outs = _run_workers(sim_lib, world, tmp_path, {})
    assert all("ADABELIEF_NVLS_OK" in o for o in outs), outs[0][-2000:]


@pytest.mark.parametrize("world", [3, 8])
def test_one_process_per_gpu_under_the_tree_on_the_simulator(sim_lib, world, tmp_path):
    _run_workers(sim_lib, world, tmp_path, {"MXKV_ADABELIEF_TREE": "1"})
