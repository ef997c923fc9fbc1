"""Adamax on the store without a GPU: the oracle against the reference's own `Adamax.step` (golden/adamax_steps.npz) bit
for bit, the kernel's Adamax arithmetic compiled for the host against the oracle bit for bit, the per-key scalars the
fused kernel receives, and tests/test_gpu_adamax.py plus a one-process-per-GPU worker (tests/adamax_mp_worker.py) on the
simulated CUDA runtime (tests/sim).

Counterpart of the reference's tests/python/unittest/test_optimizer.py::test_adamax.  The reference has no operator for
Adamax: its `step` is the definition, so the fixture tests/golden/make_adamax_golden.py writes from it pins the oracle
(tests/adamax_oracle.py) bit for bit, and the oracle pins the kernel -- here its arithmetic compiled for the host, in
tests/test_gpu_adamax.py its launches on the GPU.  The helpers here serve tests/test_adadelta.py too."""
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
import adamax_oracle as A  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "sim")
F32P = ctypes.POINTER(ctypes.c_float)
_F = np.float32


def same(a, b):
    """bit for bit, except that any NaN equals any NaN: IEEE 754 leaves the sign and payload of a NaN result open, and
    the host compiler may order the operands of a commutative operation either way"""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def golden(name):
    d = np.load(os.path.join(ROOT, "tests", "golden", "%s_steps.npz" % name))
    return d, [ast.literal_eval(str(m)) for m in d["cases"]]


def load_generator(name):
    spec = importlib.util.spec_from_file_location("make_%s_golden" % name,
                                                  os.path.join(ROOT, "tests", "golden", "make_%s_golden.py" % name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def check_golden(name, oracle_cls):
    """the oracle replays every fixture case from its initial weight; weights after every step and both states after
    the last one are the reference step's, bit for bit"""
    d, cases = golden(name)
    steps = int(d["steps"][0])
    assert steps >= 5 and len(cases) == 9
    for ci, (tag_name, lr, wd, kw) in enumerate(cases):
        assert tag_name == name
        for si in range(4):
            tag = "c%d_s%d" % (ci, si)
            opt = oracle_cls(learning_rate=lr, wd=wd, **kw)
            w = d["w0_" + tag].reshape(-1).copy()
            for t in range(steps):
                opt.update(0, w, d["g%d_%s" % (t, tag)].reshape(-1).copy())
                assert same(w, d["w%d_%s" % (t + 1, tag)].reshape(-1)), (tag, t, kw)
            for i in range(2):
                assert same(opt.states[0][i], d["s%d_%s" % (i, tag)].reshape(-1)), (tag, i, kw)


def check_grid(name, names):
    """the 8 option sets meet every pair of levels; the clip binds in some set; one more set clips at 0"""
    gen = load_generator(name)
    assert gen.covers_every_pair(gen.GRID)
    d, cases = golden(name)
    opts = [tuple(wd if n == "wd" else kw[n] for n in names) for _, _, wd, kw in cases]
    assert opts == gen.GRID + gen.EXTRA
    assert [o[names.index("clip_gradient")] for o in gen.EXTRA] == [0.0]
    clip_binds = False
    for ci, (_, lr, wd, kw) in enumerate(cases[:8]):
        g = d["g0_c%d_s3" % ci] * np.float32(kw["rescale_grad"])
        if kw["clip_gradient"] is not None and np.abs(g).max() > kw["clip_gradient"]:
            clip_binds = True
    assert clip_binds


def build_host(tmp_path_factory, name):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no C++ compiler")
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("CUDA headers not installed")
    so = str(tmp_path_factory.mktemp("%s_host" % name) / ("lib%s_host.so" % name))
    subprocess.run([gxx, "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-Werror",
                    "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "incubator-mxnet_b200", "csrc"), "-I", cuda_inc,
                    os.path.join(ROOT, "tests", "c", "%s_host.cc" % name), "-o", so], check=True, capture_output=True)
    return ctypes.CDLL(so)


def check_host_against_oracle(host_step, oracle_cls, kw, flavour, clip, counts=(1, 2, 7, 10 ** 6)):
    """``host_step(opt, t, g, w, states)`` runs update_one over the arrays with the scalars of update count ``t``; the
    oracle runs the same step.  NaN, +-inf and +-0 gradient elements; a clip of 0 is on, one below 0 off"""
    rng = np.random.default_rng(12)
    n = 20011
    w1 = rng.uniform(-1, 1, n).astype(np.float32)
    w2 = w1.copy()
    s1 = [np.zeros(n, np.float32) for _ in range(2)]
    oopt = oracle_cls(**dict(kw, clip_gradient=clip))
    special = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0], np.float32)
    bound = False
    for t in counts:
        oopt.count[0] = t - 1                   # the oracle's next update runs at update count t
        g = rng.uniform(-2, 2, n).astype(np.float32)
        g[rng.integers(0, n, 50)] = special[rng.integers(0, len(special), 50)]
        host_step(oopt, t, g, w1, s1)
        if clip is not None and clip >= 0:
            bound = bound or bool(np.any(np.abs(np.float32(oopt.rescale_grad) * g) > clip))
        if flavour == "f32":
            oopt.update(0, w2, g)
        else:
            for kind in (1, 2):       # the rounding to the key type is the store's, after the update
                o2 = oracle_cls(**dict(kw, clip_gradient=clip))
                o2.states[0] = tuple(x.copy() for x in oopt.state(0, w2))
                o2.count[0] = t - 1
                ww, lp = w2.copy(), np.zeros(n, np.uint16)
                o2.update_lp(0, lp, kind, ww, g)
                want = ww.astype(np.float16).view(np.uint16) if kind == 1 else O.f32_to_bf16(ww)
                assert np.array_equal(lp, want)
            oopt.update_lp(0, None, 0, w2, g)
        assert oopt.count[0] == t
        assert same(w1, w2), (flavour, t)
        for a, b in zip(s1, oopt.states[0]):
            assert same(a, b), (flavour, t)
        assert np.any(np.isnan(w1)) and np.any(np.isfinite(w1))
    assert clip is None or clip < 0 or bound


def key_hyper(kv, key):
    from mxnet_b200.base import _LIB, check_call
    lr, wd, eta = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
    check_call(_LIB.MXKVB200GetKeyHyper(kv.handle, int(key), None, ctypes.byref(lr), ctypes.byref(wd), ctypes.byref(eta)))
    return np.float32(lr.value), np.float32(wd.value), np.float32(eta.value)


def set_count(kv, key, t):
    from mxnet_b200.base import _LIB, check_call
    check_call(_LIB.MXKVB200SetUpdateCount(kv.handle, int(key), None, ctypes.c_int64(t)))


def c_caller_store(name):
    from mxnet_b200.base import _LIB, check_call
    kv = mx.kv.create("device")
    kv.init([0, 1], [mx.nd.zeros((4,)), mx.nd.zeros((4,))])
    check_call(_LIB.MXKVB200SetOptimizer(kv.handle, name.encode(), 0, None, None))
    return kv


# ---------------------------------------------------------------------------
# Adamax
# ---------------------------------------------------------------------------
def test_oracle_matches_the_reference_step_golden():
    """adamax_steps.npz: the reference's Adamax.step (adamax.py:74-111) over 9 option sets x 4 shapes x 6 steps; the
    oracle reproduces every weight and both states bit for bit -- the same correctly rounded float32 operations in the
    same order, every scalar rounded once from its double"""
    check_golden("adamax", A.OracleAdamax)


def test_golden_option_grid_covers_every_pair():
    check_grid("adamax", ("beta1", "beta2", "clip_gradient", "rescale_grad", "wd"))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return build_host(tmp_path_factory, "adamax")


@pytest.mark.parametrize("clip", [None, 0.4, 0.0, -0.3])
@pytest.mark.parametrize("wd", [0.0, 0.03])
@pytest.mark.parametrize("flavour", ["f32", "lp"])
def test_kernel_arithmetic_on_the_host_is_the_oracle_bit_for_bit(host, flavour, wd, clip):
    """update_one<OPT_ADAMAX> against the oracle at update counts 1, 2, 7 and 10^6 (where beta1^t underflows to 0):
    float32 keys, and the fp32 master of 16-bit keys with the stored weight its one rounding to float16 / bfloat16"""
    f = ctypes.c_float
    p = lambda a: a.ctypes.data_as(F32P)       # noqa: E731

    def step(opt, t, g, w, st):
        lr_op, wd_op, eta_op = opt.key_scalars(0, t)
        clip_op = opt.clip_gradient if A.clip_on(opt.clip_gradient) else -1.0
        assert host.host_adamax(ctypes.c_int64(w.size), p(g), p(w), p(st[0]), p(st[1]), f(lr_op), f(wd_op),
                                f(eta_op), f(opt.beta1), f(opt.beta2), f(opt.epsilon), f(opt.rescale_grad),
                                f(clip_op)) == 0
    kw = dict(learning_rate=0.01, beta1=0.9, beta2=0.8, epsilon=1e-6, wd=wd, rescale_grad=0.5)     # 1 - 0.9 is not 1.f - 0.9f
    check_host_against_oracle(step, A.OracleAdamax, kw, flavour, clip)


def test_maximum_propagates_nan_from_either_operand(host):
    """mshadow_op::maximum: a NaN state (beta2*var) or a NaN gradient both give a NaN var -- fmaxf would return the
    other operand"""
    f = ctypes.c_float
    p = lambda a: a.ctypes.data_as(F32P)       # noqa: E731
    g = np.array([np.nan, 0.5, 0.25, np.nan], np.float32)
    w = np.zeros(4, np.float32)
    mean = np.zeros(4, np.float32)
    var = np.array([1.0, np.nan, 0.0, np.nan], np.float32)
    host.host_adamax(ctypes.c_int64(4), p(g), p(w), p(mean), p(var), f(0.01), f(0.0), f(0.1), f(0.9), f(0.999),
                     f(1e-8), f(1.0), f(-1.0))
    assert np.array_equal(np.isnan(var), [True, True, False, True])
    assert var[2] == np.float32(0.25)


def test_per_key_scalars_defaults_and_multipliers():
    """what the fused kernel receives per key for update count t: lr = learning rate x lr_mult / (1 - beta1^t) in
    double, rounded once; eta = 1 - beta1 in double, rounded once (not 1 - float(beta1)); wd = wd x wd_mult.  The
    reference class's defaults (learning_rate 0.002, beta1 0.9, beta2 0.999, epsilon 1e-8, adamax.py:61) for a C
    caller that names "adamax" alone"""
    kv = c_caller_store("adamax")
    dflt = A.OracleAdamax()
    for t in (1, 2, 7, 1000, 10 ** 6):
        set_count(kv, 0, t)
        got = key_hyper(kv, 0)
        assert got == dflt.key_scalars(0, t), (t, got)
    assert dflt.key_scalars(0, 1) == (_F(0.002 / (1. - 0.9)), _F(0), _F(1. - 0.9))
    # the double-rounded complement is not the float one at the default beta1
    assert _F(1. - 0.9) == _F(0.1) and _F(1. - 0.9) != _F(1) - _F(0.9)
    opt = mx.optimizer.create("adamax")
    assert isinstance(opt, mx.optimizer.Adamax)
    assert (opt.learning_rate, opt.beta1, opt.beta2, opt.epsilon) == (0.002, 0.9, 0.999, 1e-8)
    assert mx.optimizer.fused_name_of(opt) == "adamax"
    assert mx.optimizer.fused_name_of(mx.optimizer.Adamax(use_fused_step=False)) is None
    opt = mx.optimizer.Adamax(learning_rate=0.03, beta1=0.8, beta2=0.95, epsilon=1e-4, wd=0.02, clip_gradient=0.0)
    opt.set_lr_mult({1: 0.5})
    opt.set_wd_mult({1: 3.0})
    kv.set_optimizer(opt)
    kw = opt.fused_kwargs()
    assert (kw["beta1"], kw["beta2"], kw["epsilon"], kw["clip_gradient"]) == (0.8, 0.95, 1e-4, 0.0)
    oopt = A.OracleAdamax(learning_rate=0.03, beta1=0.8, beta2=0.95, epsilon=1e-4, wd=0.02, lr_mult={1: 0.5},
                          wd_mult={1: 3.0})
    for k, lr, wd in ((0, 0.03, 0.02), (1, 0.015, 0.06)):
        for t in (1, 2, 3, 7, 200):
            set_count(kv, k, t)
            got = key_hyper(kv, k)
            assert got == oopt.key_scalars(k, t), (k, t, got)
            assert got == (_F(lr / (1. - 0.8 ** t)), _F(wd), _F(1. - 0.8))
    assert _F(1. - 0.8) != _F(1) - _F(0.8)


def test_create_state_follows_the_reference_tuple_order():
    """create_state: ``(mean, var)``, two float32 zeros -- the engine's state0, state1; one torch `step` leaves the
    oracle's mean, var and weight there"""
    try:
        import torch
    except ImportError:
        pytest.skip("create_state allocates torch tensors")
    w0 = np.array([0.5, -0.25, 1.0, 0.0, 2.0], np.float32)
    g = np.array([0.3, -0.7, 0.0, 1.5, -0.1], np.float32)
    w = mx.nd.array(w0)
    opt = mx.optimizer.Adamax(learning_rate=0.01, beta1=0.5, beta2=0.8, use_fused_step=False)
    s = opt.create_state(0, w)
    assert len(s) == 2 and all(tuple(x.shape) == (5,) and x.dtype == torch.float32 and not x.any() for x in s)
    opt.update([0], [w], [mx.nd.array(g)], [s])
    oopt = A.OracleAdamax(learning_rate=0.01, beta1=0.5, beta2=0.8)
    ow = w0.copy()
    oopt.update(0, ow, g)
    for x, want in zip(s, oopt.states[0]):
        np.testing.assert_allclose(x.cpu().numpy(), want, rtol=1e-6)
    np.testing.assert_allclose(w.asnumpy(), ow, rtol=1e-6)


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


def run_gpu_file_on_sim(sim_lib, devices, fname, min_passed):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_B200_LIBRARY_PATH=sim_lib, MXKV_SIM_DEVICES=str(devices))
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", fname)],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= min_passed, r.stdout[-1000:]


def run_workers(sim_lib, world, tmp_path, worker, marker, extra):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_SIM_MP="1", MXKV_SIM_RDV=str(tmp_path), MXKV_B200_LIBRARY_PATH=sim_lib,
               MXKV_SIM_DEVICES=str(world), MXKV_B200_ARENA_MB="256", WORLD_SIZE=str(world), **extra)
    procs = []
    for r in range(world):
        e = dict(env, RANK=str(r), LOCAL_RANK=str(r))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", worker)], env=e,
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
        assert "%s_WORKER_OK rank %d" % (marker, r) in out, out[-2000:]
    return outs


@pytest.mark.parametrize("devices", [1, 2, 4, 8])
def test_gpu_adamax_on_the_simulator(sim_lib, devices):
    # torch-based tests skip next to the stand-in runtime; the multi-GPU ones need two simulated GPUs or more
    run_gpu_file_on_sim(sim_lib, devices, "test_gpu_adamax.py", 16 if devices == 1 else 17)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_process_per_gpu_on_the_simulator(sim_lib, world, tmp_path):
    """two-shot keys with two sharded states, a checkpoint of them on every rank, and the multicast kernel forced
    (the engine-owned multicast arena of tests/sim/fake_driver.cc): within 1e-6 of the oracle"""
    outs = run_workers(sim_lib, world, tmp_path, "adamax_mp_worker.py", "ADAMAX", {})
    assert all("ADAMAX_NVLS_OK" in o for o in outs), outs[0][-2000:]


@pytest.mark.parametrize("world", [3, 8])
def test_one_process_per_gpu_under_the_tree_on_the_simulator(sim_lib, world, tmp_path):
    run_workers(sim_lib, world, tmp_path, "adamax_mp_worker.py", "ADAMAX", {"MXKV_STEP_OPT_TREE": "1"})
