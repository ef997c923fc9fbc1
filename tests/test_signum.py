"""Signum on the store without a GPU: the oracle against the reference's own `Signum.step` (golden/signum_steps.npz),
the kernels' signSGD and Signum arithmetic compiled for the host against the oracle bit for bit, the per-key scalars
the fused kernel receives, and tests/test_gpu_signum.py plus a one-process-per-GPU worker (tests/signum_mp_worker.py)
on the simulated CUDA runtime (tests/sim).

Counterpart of the reference's tests/python/unittest/test_optimizer.py::test_signum (Signum.step against the fused
operators, float32 rtol 1e-4, atol 1e-5): the reference's step pins the oracle (tests/signum_oracle.py) through the
fixture tests/golden/make_signum_golden.py writes, and the oracle pins the kernels -- here their arithmetic compiled
for the host, in tests/test_gpu_signum.py their launches on the GPU."""
import ast
import ctypes
import glob
import importlib.util
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
import signum_oracle as S  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "sim")
F32P = ctypes.POINTER(ctypes.c_float)


def _bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _golden():
    d = np.load(os.path.join(ROOT, "tests", "golden", "signum_steps.npz"))
    return d, [ast.literal_eval(str(m)) for m in d["cases"]]


def test_oracle_matches_the_reference_step_golden():
    """signum_steps.npz: the reference's Signum.step (signum.py:80-119) over 8 option sets x 4 shapes x 5 steps; the
    oracle's restatement of the fused operators within the float32 tolerance of the reference's test_signum
    (rtol 1e-4, atol 1e-5)"""
    d, cases = _golden()
    worst = 0.0
    for ci, (name, lr, wd, kw) in enumerate(cases):
        assert name == "signum"
        for si in range(4):
            tag = "c%d_s%d" % (ci, si)
            opt = S.OracleSignum(learning_rate=lr, wd=wd, **kw)
            w = d["w0_" + tag].reshape(-1).copy()
            for t in range(5):
                opt.update(0, w, d["g%d_%s" % (t, tag)].reshape(-1).copy())
                want = d["w%d_%s" % (t + 1, tag)].reshape(-1)
                np.testing.assert_allclose(w, want, rtol=1e-4, atol=1e-5, err_msg="%s step %d" % (tag, t))
                worst = max(worst, float(np.max(np.abs(w.astype(np.float64) - want))))
    # `step` rounds 1 - lr * wd_lh (and signSGD's wd + wd_lh) in double, the operators in float: last bits apart
    print("largest |oracle - reference step|: %.3g" % worst)
    assert worst < 1e-6


def test_golden_option_grid_exercises_every_option():
    """both kinds occur; exact zero gradients occur; in some set with momentum the gradient clip binds"""
    d, cases = _golden()
    assert {c[3]["momentum"] for c in cases} == {0.9, 0.0}
    assert all(np.any(d["g0_c%d_s3" % ci] == 0) for ci in range(len(cases)))
    clip_binds = False
    for ci, (_, lr, wd, kw) in enumerate(cases):
        g = d["g0_c%d_s3" % ci] * np.float32(kw["rescale_grad"])
        if kw["momentum"] and kw["clip_gradient"] is not None and np.abs(g).max() > kw["clip_gradient"]:
            clip_binds = True
    assert clip_binds


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no C++ compiler")
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("CUDA headers not installed")
    so = str(tmp_path_factory.mktemp("signum_host") / "libsignum_host.so")
    subprocess.run([gxx, "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-Werror",
                    "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "incubator-mxnet_b200", "csrc"), "-I", cuda_inc,
                    os.path.join(ROOT, "tests", "c", "signum_host.cc"), "-o", so], check=True, capture_output=True)
    return ctypes.CDLL(so)


def _host_step(host, opt, index, g, w, mom):
    """one update_one pass with the operator parameters the store hands the kernel for ``opt`` (an OracleSignum)"""
    f = ctypes.c_float
    p = lambda a: a.ctypes.data_as(F32P)       # noqa: E731
    lr, wd = opt.key_scalars(index)
    clip = S.fused_clip(opt.clip_gradient)
    stateful = opt.momentum != 0.0
    assert host.host_signum(int(stateful), ctypes.c_int64(w.size), p(g), p(w), p(mom if stateful else w), f(lr),
                            f(wd), f(S.fused_momentum(opt.momentum)), f(opt.wd_lh), f(opt.rescale_grad),
                            f(-1.0 if clip is None else clip)) == 0


@pytest.mark.parametrize("momentum", [0.9, 0.0, -0.5])
@pytest.mark.parametrize("clip", [None, 0.4, 0.0, -0.3])
@pytest.mark.parametrize("wd", [0.0, 0.03])
@pytest.mark.parametrize("flavour", ["f32", "lp"])
def test_kernel_arithmetic_on_the_host_is_the_oracle_bit_for_bit(host, flavour, wd, clip, momentum):
    """update_one<OPT_SIGNUM> / <OPT_SIGNSGD> against the oracle's SignumKernel / SignSGDKernel, with NaN, +-inf and
    +-0 gradient elements: float32 keys, and the fp32 master of 16-bit keys with the stored weight its one rounding to
    float16 / bfloat16.  A negative momentum creates the state and runs at momentum 0; a clip of 0, below 0 or None
    is off"""
    rng = np.random.default_rng(12)
    n = 20011
    w1 = rng.uniform(-1, 1, n).astype(np.float32)
    w2 = w1.copy()
    m1 = np.zeros(n, np.float32)
    kw = dict(learning_rate=0.01, momentum=momentum, wd_lh=0.02, wd=wd, rescale_grad=0.5, clip_gradient=clip)
    oopt = S.OracleSignum(**kw)
    special = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0], np.float32)
    bound = False
    for t in range(1, 5):
        g = rng.uniform(-2, 2, n).astype(np.float32)
        g[rng.integers(0, n, 50)] = special[rng.integers(0, len(special), 50)]
        _host_step(host, oopt, 0, g, w1, m1)
        if clip:
            bound = bound or bool(np.any(np.abs(np.float32(0.5) * g) > clip))
        if flavour == "f32":
            oopt.update(0, w2, g)
        else:
            for kind in (1, 2):       # the rounding to the key type is the store's, after the update
                o2 = S.OracleSignum(**kw)
                o2.states[0] = tuple(x.copy() for x in oopt.state(0, w2))
                ww, lp = w2.copy(), np.zeros(n, np.uint16)
                o2.update_lp(0, lp, kind, ww, g)
                want = ww.astype(np.float16).view(np.uint16) if kind == 1 else O.f32_to_bf16(ww)
                assert np.array_equal(lp, want)
            oopt.update_lp(0, None, 0, w2, g)
        assert _bits_equal(w1, w2), (flavour, t)
        if momentum != 0.0:
            assert _bits_equal(m1, oopt.states[0][0]), (flavour, t)
        else:
            assert oopt.states[0] == ()
    assert (not clip or momentum == 0.0) or bound


def test_sign_of_nan_and_signed_zero_is_zero(host):
    """sign(x) = (x > 0) - (x < 0): a NaN, +0 or -0 gradient leaves signSGD's weight at (1 - lr*wd)*w"""
    g = np.array([np.nan, 0.0, -0.0, 1e-30, -1e-30, np.inf, -np.inf], np.float32)
    w = np.full(g.size, 0.5, np.float32)
    opt = S.OracleSignum(learning_rate=0.25, momentum=0.0)
    _host_step(host, opt, 0, g, w, None)
    assert w.tolist() == [0.5, 0.5, 0.5, 0.25, 0.75, 0.25, 0.75]


def _key_hyper(kv, key):
    from mxnet_b200.base import _LIB, check_call
    lr, wd, eta = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
    check_call(_LIB.MXKVB200GetKeyHyper(kv.handle, int(key), None, ctypes.byref(lr), ctypes.byref(wd), ctypes.byref(eta)))
    return np.float32(lr.value), np.float32(wd.value), np.float32(eta.value)


def test_per_key_scalars_defaults_and_multipliers():
    """what the fused kernel receives per key: the learning rate times lr_mult -- no bias correction, at any update
    count; Signum: wd times wd_mult; signSGD: wd times wd_mult plus wd_lh, summed in double and rounded once (wd_lh is
    not multiplied by wd_mult); the reference class's defaults (learning_rate 0.01, momentum 0.9, wd_lh 0,
    signum.py:67) for a C caller that names "signum" alone"""
    from mxnet_b200.base import _LIB, check_call
    kv = mx.kv.create("device")
    kv.init([0, 1], [mx.nd.zeros((4,)), mx.nd.zeros((4,))])
    check_call(_LIB.MXKVB200SetOptimizer(kv.handle, b"signum", 0, None, None))
    for t in (1, 2, 7, 1000):
        check_call(_LIB.MXKVB200SetUpdateCount(kv.handle, 0, None, ctypes.c_int64(t)))
        assert _key_hyper(kv, 0)[:2] == (np.float32(0.01), np.float32(0.0))
    opt = mx.optimizer.create("signum")
    assert isinstance(opt, mx.optimizer.Signum)
    assert (opt.learning_rate, opt.momentum, opt.wd_lh) == (0.01, 0.9, 0.0)
    assert mx.optimizer.fused_name_of(opt) == "signum"
    assert mx.optimizer.fused_name_of(mx.optimizer.Signum(use_fused_step=False)) is None
    # 0.02 * 3 + 0.015 = 0.075 in double; float32 sums of the rounded terms give 0.074999996
    assert np.float32(0.02 * 3.0 + 0.015) != np.float32(np.float32(0.02 * 3.0) + np.float32(0.015))
    for momentum in (0.9, 0.0):
        opt = mx.optimizer.Signum(learning_rate=0.03, momentum=momentum, wd_lh=0.015, wd=0.02)
        opt.set_lr_mult({1: 0.5})
        opt.set_wd_mult({1: 3.0})
        kv.set_optimizer(opt)
        kw = opt.fused_kwargs()
        assert (kw["momentum"], kw["wd_lh"]) == (momentum, 0.015)
        oopt = S.OracleSignum(learning_rate=0.03, momentum=momentum, wd_lh=0.015, wd=0.02, lr_mult={1: 0.5},
                              wd_mult={1: 3.0})
        for k, lr, wd in ((0, 0.03, 0.02), (1, 0.015, 0.06)):
            check_call(_LIB.MXKVB200SetUpdateCount(kv.handle, k, None, ctypes.c_int64(3)))
            want_wd = np.float32(wd + 0.015) if momentum == 0.0 else np.float32(wd)
            assert _key_hyper(kv, k)[:2] == (np.float32(lr), want_wd), (momentum, k)
            assert tuple(map(np.float32, oopt.key_scalars(k))) == (np.float32(lr), want_wd)


def test_create_state_follows_the_reference():
    """create_state: a zeroed ``mom`` where momentum != 0 (a negative momentum too), None at momentum 0"""
    w = mx.nd.zeros((5,))
    try:
        import torch  # noqa: F401
    except ImportError:
        pytest.skip("create_state allocates torch tensors")
    s = mx.optimizer.Signum().create_state(0, w)
    assert tuple(s.shape) == (5,) and not s.any()
    assert tuple(mx.optimizer.Signum(momentum=-0.5).create_state(0, w).shape) == (5,)
    assert mx.optimizer.Signum(momentum=0.0).create_state(0, w) is None


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
def test_gpu_signum_on_the_simulator(sim_lib, devices):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_B200_LIBRARY_PATH=sim_lib, MXKV_SIM_DEVICES=str(devices))
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_gpu_signum.py")],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    m = re.search(r"(\d+) passed", r.stdout)
    # torch-based tests skip next to the stand-in runtime; the multi-GPU ones need two simulated GPUs or more
    assert m and int(m.group(1)) >= (35 if devices == 1 else 37), r.stdout[-1000:]


def _run_workers(sim_lib, world, tmp_path, extra):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_SIM_MP="1", MXKV_SIM_RDV=str(tmp_path), MXKV_B200_LIBRARY_PATH=sim_lib,
               MXKV_SIM_DEVICES=str(world), MXKV_B200_ARENA_MB="256", WORLD_SIZE=str(world), **extra)
    procs = []
    for r in range(world):
        e = dict(env, RANK=str(r), LOCAL_RANK=str(r))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "signum_mp_worker.py")], env=e,
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
        assert "SIGNUM_WORKER_OK rank %d" % r in out, out[-2000:]
    return outs


@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_process_per_gpu_on_the_simulator(sim_lib, world, tmp_path):
    """two-shot keys with the sharded momentum, a checkpoint of it on every rank, signSGD next to Signum, and the
    multicast kernel forced (the engine-owned multicast arena of tests/sim/fake_driver.cc): bit for bit against the
    oracle on gradients of a dyadic grid"""
    outs = _run_workers(sim_lib, world, tmp_path, {})
    assert all("SIGNUM_NVLS_OK" in o for o in outs), outs[0][-2000:]


@pytest.mark.parametrize("world", [3, 8])
def test_one_process_per_gpu_under_the_tree_on_the_simulator(sim_lib, world, tmp_path):
    _run_workers(sim_lib, world, tmp_path, {"MXKV_SIGNUM_TREE": "1"})
