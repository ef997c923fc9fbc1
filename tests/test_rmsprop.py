"""RMSProp on the store without a GPU: the oracle against the reference's own `RMSProp.step` (golden/rmsprop_steps.npz),
the kernels' RMSProp arithmetic (plain and centered) compiled for the host against the oracle bit for bit, the per-key
scalars the fused kernel receives, and tests/test_gpu_rmsprop.py plus a one-process-per-GPU worker
(tests/rmsprop_mp_worker.py) on the simulated CUDA runtime (tests/sim).

Counterpart of the reference's tests/python/unittest/test_optimizer.py::test_rms (RMSProp.step against the fused
operators, float32 rtol 1e-2, atol 1e-2): the reference's step pins the oracle (tests/rmsprop_oracle.py) through the
fixture tests/golden/make_rmsprop_golden.py writes, and the oracle pins the kernels -- here their arithmetic compiled
for the host, in tests/test_gpu_rmsprop.py their launches on the GPU."""
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
import rmsprop_oracle as R  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "sim")
F32P = ctypes.POINTER(ctypes.c_float)


def _bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _golden():
    d = np.load(os.path.join(ROOT, "tests", "golden", "rmsprop_steps.npz"))
    return d, [ast.literal_eval(str(m)) for m in d["cases"]]


def test_oracle_matches_the_reference_step_golden():
    """rmsprop_steps.npz: the reference's RMSProp.step (rmsprop.py:90-141) over 8 option sets x 4 shapes x 5 steps;
    the oracle's restatement of the fused operators within the float32 tolerance of the reference's test_rms
    (rtol 1e-2, atol 1e-2)"""
    d, cases = _golden()
    worst = 0.0
    for ci, (name, lr, wd, kw) in enumerate(cases):
        assert name == "rmsprop"
        for si in range(4):
            tag = "c%d_s%d" % (ci, si)
            opt = R.OracleRMSProp(learning_rate=lr, wd=wd, **kw)
            w = d["w0_" + tag].reshape(-1).copy()
            for t in range(5):
                opt.update(0, w, d["g%d_%s" % (t, tag)].reshape(-1).copy())
                want = d["w%d_%s" % (t + 1, tag)].reshape(-1)
                np.testing.assert_allclose(w, want, rtol=1e-2, atol=1e-2, err_msg="%s step %d" % (tag, t))
                worst = max(worst, float(np.max(np.abs(w.astype(np.float64) - want))))
    # `step` computes lr * (g / (sqrt(var) + eps)), the operators (lr * g) / (sqrt(var) + eps): one rounding apart
    print("largest |oracle - reference step|: %.3g" % worst)
    assert worst < 1e-6


def test_golden_option_grid_exercises_every_option():
    """both kinds occur, and in some set with wd > 0 the gradient clip binds and in another the weight clip binds"""
    d, cases = _golden()
    assert {c[3]["centered"] for c in cases} == {True, False}
    clip_binds, wclip_binds = False, False
    for ci, (_, lr, wd, kw) in enumerate(cases):
        g = d["g0_c%d_s3" % ci] * np.float32(kw["rescale_grad"])
        if kw["clip_gradient"] is not None and np.abs(g).max() > kw["clip_gradient"]:
            clip_binds = True
        if kw["clip_weights"] is not None and np.abs(d["w0_c%d_s3" % ci]).max() > kw["clip_weights"]:
            wclip_binds = True
    assert clip_binds and wclip_binds


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no C++ compiler")
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("CUDA headers not installed")
    so = str(tmp_path_factory.mktemp("rmsprop_host") / "librmsprop_host.so")
    subprocess.run([gxx, "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-Werror",
                    "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "incubator-mxnet_b200", "csrc"), "-I", cuda_inc,
                    os.path.join(ROOT, "tests", "c", "rmsprop_host.cc"), "-o", so], check=True, capture_output=True)
    return ctypes.CDLL(so)


def _host_rmsprop(host, centered, g, w, st, lr, wd, rho, momentum, eps, rescale, clip, clip_weights):
    f = ctypes.c_float
    p = lambda a: a.ctypes.data_as(F32P)       # noqa: E731
    s = list(st) + [st[0]] * (3 - len(st))
    off = lambda v: f(-1.0 if v is None else v)   # noqa: E731
    assert host.host_rmsprop(int(centered), ctypes.c_int64(w.size), p(g), p(w), p(s[0]), p(s[1]), p(s[2]), f(lr),
                             f(wd), f(rho), f(momentum), f(eps), f(rescale), off(clip), off(clip_weights)) == 0


@pytest.mark.parametrize("centered", [False, True])
@pytest.mark.parametrize("clips", [(None, None), (0.4, None), (None, 0.3), (0.4, 0.3)])
@pytest.mark.parametrize("wd", [0.0, 0.03])
@pytest.mark.parametrize("flavour", ["f32", "lp"])
def test_kernel_arithmetic_on_the_host_is_the_oracle_bit_for_bit(host, flavour, wd, clips, centered):
    """update_one<OPT_RMSPROP> and the six-argument update_one<OPT_RMSPROP_CENTERED> against the oracle's
    RMSPropUpdateKernel / RMSPropAlexUpdateKernel: float32 keys, and the fp32 master of 16-bit keys with the stored
    weight its one rounding to float16 / bfloat16"""
    clip, clip_w = clips
    rng = np.random.default_rng(12)
    n = 20011
    w1 = rng.uniform(-1, 1, n).astype(np.float32)
    w2 = w1.copy()
    ns = 3 if centered else 1
    s1 = [np.zeros(n, np.float32) for _ in range(ns)]
    s2 = [np.zeros(n, np.float32) for _ in range(ns)]
    oopt = R.OracleRMSProp(learning_rate=0.01, rho=0.8, momentum=0.7, epsilon=1e-6, centered=centered,
                           clip_weights=clip_w, wd=wd, rescale_grad=0.5, clip_gradient=clip)
    oopt.states[0] = tuple(s2)
    bound = [False, False]
    for t in range(1, 5):
        g = rng.uniform(-2, 2, n).astype(np.float32)
        _host_rmsprop(host, centered, g, w1, s1, 0.01, wd, 0.8, 0.7, 1e-6, 0.5, clip, clip_w)
        if clip is not None:
            bound[0] = bound[0] or bool(np.any(np.abs(np.float32(0.5) * g) > clip))
        if flavour == "f32":
            oopt.update(0, w2, g)
        else:
            for kind in (1, 2):       # the rounding to the key type is the store's, after the update
                o2 = R.OracleRMSProp(**{k: getattr(oopt, a) for k, a in (
                    ("learning_rate", "lr"), ("rho", "rho"), ("momentum", "momentum"), ("epsilon", "epsilon"),
                    ("centered", "centered"), ("clip_weights", "clip_weights"), ("wd", "wd"),
                    ("rescale_grad", "rescale_grad"), ("clip_gradient", "clip_gradient"))})
                o2.states[0] = tuple(x.copy() for x in s2)
                ww, lp = w2.copy(), np.zeros(n, np.uint16)
                o2.update_lp(0, lp, kind, ww, g)
                want = ww.astype(np.float16).view(np.uint16) if kind == 1 else O.f32_to_bf16(ww)
                assert np.array_equal(lp, want)
            oopt.update_lp(0, None, 0, w2, g)
        assert _bits_equal(w1, w2), (flavour, t)
        for a, b in zip(s1, s2):
            assert _bits_equal(a, b), (flavour, t)
        if clip_w is not None:
            bound[1] = bound[1] or bool(np.any(np.abs(w2) >= clip_w))
    assert (clip is None or bound[0]) and (clip_w is None or bound[1])


def _key_hyper(kv, key):
    from mxnet_b200.base import _LIB, check_call
    lr, wd, eta = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
    check_call(_LIB.MXKVB200GetKeyHyper(kv.handle, int(key), None, ctypes.byref(lr), ctypes.byref(wd), ctypes.byref(eta)))
    return np.float32(lr.value), np.float32(wd.value), np.float32(eta.value)


def test_per_key_scalars_defaults_and_multipliers():
    """what the fused kernel receives per key: the learning rate times lr_mult -- no bias correction, at any update
    count -- and wd times wd_mult; the reference class's defaults (learning_rate 0.001, rho 0.9, momentum 0.9, epsilon
    1e-8, rmsprop.py:70-71) for a C caller that names "rmsprop" alone"""
    from mxnet_b200.base import _LIB, check_call
    kv = mx.kv.create("device")
    kv.init([0, 1], [mx.nd.zeros((4,)), mx.nd.zeros((4,))])
    check_call(_LIB.MXKVB200SetOptimizer(kv.handle, b"rmsprop", 0, None, None))
    for t in (1, 2, 7, 1000):
        check_call(_LIB.MXKVB200SetUpdateCount(kv.handle, 0, None, ctypes.c_int64(t)))
        assert _key_hyper(kv, 0)[:2] == (np.float32(0.001), np.float32(0.0))
    opt = mx.optimizer.create("rmsprop")
    assert isinstance(opt, mx.optimizer.RMSProp)
    assert (opt.learning_rate, opt.rho, opt.momentum, opt.epsilon, opt.centered, opt.clip_weights) == \
        (0.001, 0.9, 0.9, 1e-8, False, None)
    assert mx.optimizer.fused_name_of(opt) == "rmsprop"
    assert mx.optimizer.fused_name_of(mx.optimizer.RMSProp(use_fused_step=False)) is None
    opt = mx.optimizer.RMSProp(learning_rate=0.03, rho=0.5, momentum=0.8, epsilon=1e-4, centered=True,
                               clip_weights=0.2, wd=0.02)
    opt.set_lr_mult({1: 0.5})
    opt.set_wd_mult({1: 3.0})
    kv.set_optimizer(opt)
    kw = opt.fused_kwargs()
    assert (kw["rho"], kw["momentum"], kw["epsilon"], kw["centered"], kw["clip_weights"]) == (0.5, 0.8, 1e-4, True, 0.2)
    for k, lr, wd in ((0, 0.03, 0.02), (1, 0.015, 0.06)):
        check_call(_LIB.MXKVB200SetUpdateCount(kv.handle, k, None, ctypes.c_int64(3)))
        assert _key_hyper(kv, k)[:2] == (np.float32(lr), np.float32(wd))


def test_create_state_follows_the_reference_tuple_order():
    """create_state: ``var`` alone, or ``(mean, var, mom)`` for the centered kind -- the order of the engine's state0,
    state1, state2"""
    w = mx.nd.zeros((5,))
    try:
        import torch  # noqa: F401
    except ImportError:
        pytest.skip("create_state allocates torch tensors")
    s = mx.optimizer.RMSProp().create_state(0, w)
    assert tuple(s.shape) == (5,)
    s = mx.optimizer.RMSProp(centered=True).create_state(0, w)
    assert len(s) == 3 and all(tuple(x.shape) == (5,) for x in s)


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
def test_gpu_rmsprop_on_the_simulator(sim_lib, devices):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_B200_LIBRARY_PATH=sim_lib, MXKV_SIM_DEVICES=str(devices))
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_gpu_rmsprop.py")],
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
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "rmsprop_mp_worker.py")], env=e,
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
        assert "RMSPROP_WORKER_OK rank %d" % r in out, out[-2000:]
    return outs


@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_process_per_gpu_on_the_simulator(sim_lib, world, tmp_path):
    """two-shot keys with three sharded states, a checkpoint of them on every rank, and the multicast kernel forced
    (the engine-owned multicast arena of tests/sim/fake_driver.cc): within 1e-6 of the oracle"""
    outs = _run_workers(sim_lib, world, tmp_path, {})
    assert all("RMSPROP_NVLS_OK" in o for o in outs), outs[0][-2000:]


@pytest.mark.parametrize("world", [3, 8])
def test_one_process_per_gpu_under_the_tree_on_the_simulator(sim_lib, world, tmp_path):
    _run_workers(sim_lib, world, tmp_path, {"MXKV_RMSPROP_TREE": "1"})
