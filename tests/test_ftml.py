"""FTML on the store without a GPU: the oracle against the reference's own `FTML.step` (golden/ftml_steps.npz), the
kernel's FTML arithmetic compiled for the host against the oracle bit for bit, the per-key scalars the fused kernel
receives, and tests/test_gpu_ftml.py plus a one-process-per-GPU worker (tests/ftml_mp_worker.py) on the simulated CUDA
runtime (tests/sim).

Counterpart of the reference's tests/python/unittest/test_optimizer.py::test_ftml (FTML.step against the fused
operator, rtol 1e-3, atol 1e-4): the reference's step pins the oracle (tests/ftml_oracle.py) through the fixture
tests/golden/make_ftml_golden.py writes, and the oracle pins the kernel -- here its arithmetic compiled for the host,
in tests/test_gpu_ftml.py its launches on the GPU."""
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
import ftml_oracle as F  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "sim")
F32P = ctypes.POINTER(ctypes.c_float)


def _same(a, b):
    """bit for bit, except that any NaN equals any NaN: IEEE 754 leaves the sign and payload of a NaN result open, and
    the host compiler may order the operands of a commutative operation either way"""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def _golden():
    d = np.load(os.path.join(ROOT, "tests", "golden", "ftml_steps.npz"))
    return d, [ast.literal_eval(str(m)) for m in d["cases"]]


def _load_generator():
    spec = importlib.util.spec_from_file_location("make_ftml_golden",
                                                  os.path.join(ROOT, "tests", "golden", "make_ftml_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_oracle_matches_the_reference_step_golden():
    """ftml_steps.npz: the reference's FTML.step (ftml.py:80-125) over 8 option sets x 4 shapes x 6 steps; the
    oracle's restatement of the fused operator within the tolerance of the reference's test_ftml (rtol 1e-3,
    atol 1e-4)"""
    d, cases = _golden()
    steps = int(d["steps"][0])
    assert steps >= 5
    worst = 0.0
    for ci, (name, lr, wd, kw) in enumerate(cases):
        assert name == "ftml"
        for si in range(4):
            tag = "c%d_s%d" % (ci, si)
            opt = F.OracleFTML(learning_rate=lr, wd=wd, **kw)
            w = d["w0_" + tag].reshape(-1).copy()
            for t in range(steps):
                opt.update(0, w, d["g%d_%s" % (t, tag)].reshape(-1).copy())
                want = d["w%d_%s" % (t + 1, tag)].reshape(-1)
                np.testing.assert_allclose(w, want, rtol=1e-3, atol=1e-4, err_msg="%s step %d" % (tag, t))
                worst = max(worst, float(np.max(np.abs(w.astype(np.float64) - want))))
    # `step` evaluates sqrt(v / coef2) + eps and coef1 / lr with coef1, coef2 and 1 - beta in double and multiplies
    # d by coef1 / lr afterwards; the operator rounds every scalar to float first: last bits apart
    print("largest |oracle - reference step|: %.3g" % worst)
    assert worst < 1e-6


def test_golden_option_grid_covers_every_pair():
    """the 8 option sets: every pair of levels of two options meets, and in some set the gradient clip binds"""
    gen = _load_generator()
    assert gen._covers_every_pair(gen.GRID)
    d, cases = _golden()
    opts = [(kw["beta1"], kw["beta2"], kw["clip_gradient"], kw["rescale_grad"], wd) for _, _, wd, kw in cases]
    assert opts == gen.GRID
    clip_binds = False
    for ci, (_, lr, wd, kw) in enumerate(cases):
        g = d["g0_c%d_s3" % ci] * np.float32(kw["rescale_grad"])
        if kw["clip_gradient"] is not None and np.abs(g).max() > kw["clip_gradient"]:
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
    so = str(tmp_path_factory.mktemp("ftml_host") / "libftml_host.so")
    subprocess.run([gxx, "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-Werror",
                    "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "incubator-mxnet_b200", "csrc"), "-I", cuda_inc,
                    os.path.join(ROOT, "tests", "c", "ftml_host.cc"), "-o", so], check=True, capture_output=True)
    return ctypes.CDLL(so)


def _host_step(host, opt, index, t, g, w, st):
    """one update_one pass with the operator parameters the store hands the kernel for ``opt`` (an OracleFTML) at
    update count ``t``"""
    f = ctypes.c_float
    p = lambda a: a.ctypes.data_as(F32P)       # noqa: E731
    lr_op, wd, eta_op = opt.key_scalars(index, t)
    clip = F.fused_clip(opt.clip_gradient)
    assert host.host_ftml(ctypes.c_int64(w.size), p(g), p(w), p(st[0]), p(st[1]), p(st[2]), f(lr_op), f(wd),
                          f(eta_op), f(opt.beta1), f(opt.beta2), f(opt.epsilon), f(opt.rescale_grad),
                          f(-1.0 if clip is None else clip)) == 0


@pytest.mark.parametrize("clip", [None, 0.4, 0.0, -0.3])
@pytest.mark.parametrize("wd", [0.0, 0.03])
@pytest.mark.parametrize("flavour", ["f32", "lp"])
def test_kernel_arithmetic_on_the_host_is_the_oracle_bit_for_bit(host, flavour, wd, clip):
    """update_one<OPT_FTML> against the oracle's FTMLKernel at update counts 1, 2, 7 and 10^6 (where beta2^t
    underflows to 0), with NaN, +-inf and +-0 gradient elements: float32 keys, and the fp32 master of 16-bit keys with
    the stored weight its one rounding to float16 / bfloat16.  A clip of 0, below 0 or None is off"""
    rng = np.random.default_rng(12)
    n = 20011
    w1 = rng.uniform(-1, 1, n).astype(np.float32)
    w2 = w1.copy()
    s1 = [np.zeros(n, np.float32) for _ in range(3)]
    kw = dict(learning_rate=0.01, beta1=0.5, beta2=0.8, epsilon=1e-6, wd=wd, rescale_grad=0.5, clip_gradient=clip)
    oopt = F.OracleFTML(**kw)
    special = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0], np.float32)
    bound = False
    counts = (1, 2, 7, 10 ** 6)
    assert F.ftml_scalars(0.01, 0.8, 0.8, 10 ** 6)[1] == np.float32(1.0)      # 0.8^(10^6) is 0 in double
    for t in counts:
        oopt.count[0] = t - 1                   # the oracle's next update runs at update count t
        g = rng.uniform(-2, 2, n).astype(np.float32)
        g[rng.integers(0, n, 50)] = special[rng.integers(0, len(special), 50)]
        _host_step(host, oopt, 0, t, g, w1, s1)
        if clip:
            bound = bound or bool(np.any(np.abs(np.float32(0.5) * g) > clip))
        if flavour == "f32":
            oopt.update(0, w2, g)
        else:
            for kind in (1, 2):       # the rounding to the key type is the store's, after the update
                o2 = F.OracleFTML(**kw)
                o2.states[0] = tuple(x.copy() for x in oopt.state(0, w2))
                o2.count[0] = t - 1
                ww, lp = w2.copy(), np.zeros(n, np.uint16)
                o2.update_lp(0, lp, kind, ww, g)
                want = ww.astype(np.float16).view(np.uint16) if kind == 1 else O.f32_to_bf16(ww)
                assert np.array_equal(lp, want)
            oopt.update_lp(0, None, 0, w2, g)
        assert oopt.count[0] == t
        assert _same(w1, w2), (flavour, t)
        for a, b in zip(s1, oopt.states[0]):
            assert _same(a, b), (flavour, t)
        assert np.any(np.isnan(w1)) and np.any(np.isfinite(w1))
    assert not clip or bound


def _key_hyper(kv, key):
    from mxnet_b200.base import _LIB, check_call
    lr, wd, eta = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
    check_call(_LIB.MXKVB200GetKeyHyper(kv.handle, int(key), None, ctypes.byref(lr), ctypes.byref(wd), ctypes.byref(eta)))
    return np.float32(lr.value), np.float32(wd.value), np.float32(eta.value)


def test_per_key_scalars_defaults_and_multipliers():
    """what the fused kernel receives per key for update count t: lr = (1 - beta1^t) / (learning rate x lr_mult) and
    eta = 1 - beta2^t, in float as the operator computes them (the powers correctly rounded), wd = wd x wd_mult; the
    reference class's defaults (learning_rate 0.0025, beta1 0.6, beta2 0.999, epsilon 1e-8, ftml.py:66) for a C caller
    that names "ftml" alone"""
    from mxnet_b200.base import _LIB, check_call
    kv = mx.kv.create("device")
    kv.init([0, 1], [mx.nd.zeros((4,)), mx.nd.zeros((4,))])
    check_call(_LIB.MXKVB200SetOptimizer(kv.handle, b"ftml", 0, None, None))
    dflt = F.OracleFTML()
    for t in (1, 2, 7, 1000, 10 ** 6):
        check_call(_LIB.MXKVB200SetUpdateCount(kv.handle, 0, None, ctypes.c_int64(t)))
        got = _key_hyper(kv, 0)
        assert got == dflt.key_scalars(0, t), (t, got)
    # t = 1: (1 - 0.6f) / 0.0025f and 1 - 0.999f, every operation in float
    assert dflt.key_scalars(0, 1) == (np.float32(np.float32(1) - np.float32(0.6)) / np.float32(0.0025), np.float32(0),
                                      np.float32(1) - np.float32(0.999))
    # 10^6 updates: beta2^t underflows, both scalars lose their power
    assert dflt.key_scalars(0, 10 ** 6) == (np.float32(1) / np.float32(0.0025), np.float32(0), np.float32(1))
    opt = mx.optimizer.create("ftml")
    assert isinstance(opt, mx.optimizer.FTML)
    assert (opt.learning_rate, opt.beta1, opt.beta2, opt.epsilon) == (0.0025, 0.6, 0.999, 1e-8)
    assert mx.optimizer.fused_name_of(opt) == "ftml"
    assert mx.optimizer.fused_name_of(mx.optimizer.FTML(use_fused_step=False)) is None
    opt = mx.optimizer.FTML(learning_rate=0.03, beta1=0.5, beta2=0.8, epsilon=1e-4, wd=0.02, clip_gradient=0.3)
    opt.set_lr_mult({1: 0.5})
    opt.set_wd_mult({1: 3.0})
    kv.set_optimizer(opt)
    kw = opt.fused_kwargs()
    assert (kw["beta1"], kw["beta2"], kw["epsilon"], kw["clip_gradient"]) == (0.5, 0.8, 1e-4, 0.3)
    oopt = F.OracleFTML(learning_rate=0.03, beta1=0.5, beta2=0.8, epsilon=1e-4, wd=0.02, lr_mult={1: 0.5},
                        wd_mult={1: 3.0})
    for k, lr, wd in ((0, 0.03, 0.02), (1, 0.015, 0.06)):
        for t in (1, 2, 3, 7, 200):
            check_call(_LIB.MXKVB200SetUpdateCount(kv.handle, k, None, ctypes.c_int64(t)))
            got = _key_hyper(kv, k)
            assert got == oopt.key_scalars(k, t), (k, t, got)
            assert got[1] == np.float32(wd)
            lr_op, eta_op = F.ftml_scalars(np.float32(lr), 0.5, 0.8, t)
            assert (got[0], got[2]) == (lr_op, eta_op)


def test_create_state_follows_the_reference_tuple_order():
    """create_state: ``(d, v, z)``, three float32 zeros -- the order of the engine's state0, state1, state2; one
    torch `step` (ftml.py:80-125) leaves d_1, v_1 and z_1 in those places"""
    try:
        import torch
    except ImportError:
        pytest.skip("create_state allocates torch tensors")
    w0 = np.array([0.5, -0.25, 1.0, 0.0, 2.0], np.float32)
    g = np.array([0.3, -0.7, 0.0, 1.5, -0.1], np.float32)
    w = mx.nd.array(w0)
    opt = mx.optimizer.FTML(learning_rate=0.01, beta1=0.5, beta2=0.8, use_fused_step=False)
    s = opt.create_state(0, w)
    assert len(s) == 3 and all(tuple(x.shape) == (5,) and x.dtype == torch.float32 and not x.any() for x in s)
    opt.update([0], [w], [mx.nd.array(g)], [s])
    d, v, z = (x.cpu().numpy().astype(np.float64) for x in s)
    g64, w64 = g.astype(np.float64), w0.astype(np.float64)
    np.testing.assert_allclose(v, 0.2 * g64 * g64, rtol=1e-6)
    np.testing.assert_allclose(d, 0.5 / 0.01 * (np.sqrt(v / 0.2) + 1e-8), rtol=1e-6)
    np.testing.assert_allclose(z, 0.5 * g64 - d * w64, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(w.asnumpy(), -z / d, rtol=1e-6, atol=1e-6)


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
def test_gpu_ftml_on_the_simulator(sim_lib, devices):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_B200_LIBRARY_PATH=sim_lib, MXKV_SIM_DEVICES=str(devices))
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_gpu_ftml.py")],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    m = re.search(r"(\d+) passed", r.stdout)
    # torch-based tests skip next to the stand-in runtime; the multi-GPU ones need two simulated GPUs or more
    assert m and int(m.group(1)) >= (16 if devices == 1 else 17), r.stdout[-1000:]


def _run_workers(sim_lib, world, tmp_path, extra):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_SIM_MP="1", MXKV_SIM_RDV=str(tmp_path), MXKV_B200_LIBRARY_PATH=sim_lib,
               MXKV_SIM_DEVICES=str(world), MXKV_B200_ARENA_MB="256", WORLD_SIZE=str(world), **extra)
    procs = []
    for r in range(world):
        e = dict(env, RANK=str(r), LOCAL_RANK=str(r))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "ftml_mp_worker.py")], env=e,
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
        assert "FTML_WORKER_OK rank %d" % r in out, out[-2000:]
    return outs


@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_process_per_gpu_on_the_simulator(sim_lib, world, tmp_path):
    """two-shot keys with three sharded states, a checkpoint of them on every rank, and the multicast kernel forced
    (the engine-owned multicast arena of tests/sim/fake_driver.cc): within 1e-6 of the oracle"""
    outs = _run_workers(sim_lib, world, tmp_path, {})
    assert all("FTML_NVLS_OK" in o for o in outs), outs[0][-2000:]


@pytest.mark.parametrize("world", [3, 8])
def test_one_process_per_gpu_under_the_tree_on_the_simulator(sim_lib, world, tmp_path):
    _run_workers(sim_lib, world, tmp_path, {"MXKV_FTML_TREE": "1"})
