"""AdaDelta on the store without a GPU: the oracle against the reference's own `AdaDelta.step`
(golden/adadelta_steps.npz) bit for bit, the kernel's AdaDelta arithmetic compiled for the host against the oracle bit
for bit, the per-key scalars the fused kernel receives, and tests/test_gpu_adadelta.py plus a one-process-per-GPU worker
(tests/adadelta_mp_worker.py) on the simulated CUDA runtime (tests/sim).

Counterpart of the reference's tests/python/unittest/test_optimizer.py::test_adadelta.  The reference has no operator
for AdaDelta: its `step` is the definition, so the fixture tests/golden/make_adadelta_golden.py writes from it pins the
oracle (tests/adadelta_oracle.py) bit for bit, and the oracle pins the kernel.  The helpers are tests/test_adamax.py's."""
import ctypes
import os
import sys

import numpy as np
import pytest

import mxnet_b200 as mx

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import adadelta_oracle as D  # noqa: E402
import test_adamax as T      # noqa: E402

F32P = ctypes.POINTER(ctypes.c_float)
_F = np.float32
sim_lib = T.sim_lib


def test_oracle_matches_the_reference_step_golden():
    """adadelta_steps.npz: the reference's AdaDelta.step (adadelta.py:72-111) over 9 option sets x 4 shapes x 6 steps;
    the oracle reproduces every weight and both states bit for bit"""
    T.check_golden("adadelta", D.OracleAdaDelta)


def test_golden_option_grid_covers_every_pair():
    T.check_grid("adadelta", ("rho", "epsilon", "clip_gradient", "rescale_grad", "wd"))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return T.build_host(tmp_path_factory, "adadelta")


@pytest.mark.parametrize("clip", [None, 0.4, 0.0, -0.3])
@pytest.mark.parametrize("wd", [0.0, 0.03])
@pytest.mark.parametrize("flavour", ["f32", "lp"])
def test_kernel_arithmetic_on_the_host_is_the_oracle_bit_for_bit(host, flavour, wd, clip):
    """update_one<OPT_ADADELTA> against the oracle at update counts 1, 2, 7 and 10^6: float32 keys, and the fp32 master
    of 16-bit keys with the stored weight its one rounding to float16 / bfloat16"""
    f = ctypes.c_float
    p = lambda a: a.ctypes.data_as(F32P)       # noqa: E731

    def step(opt, t, g, w, st):
        lr_op, wd_op, eta_op = opt.key_scalars(0, t)
        clip_op = opt.clip_gradient if T.A.clip_on(opt.clip_gradient) else -1.0
        assert host.host_adadelta(ctypes.c_int64(w.size), p(g), p(w), p(st[0]), p(st[1]), f(lr_op), f(wd_op),
                                  f(eta_op), f(opt.rho), f(opt.epsilon), f(opt.rescale_grad), f(clip_op)) == 0
    kw = dict(learning_rate=0.5, rho=0.95, epsilon=1e-5, wd=wd, rescale_grad=0.5)
    T.check_host_against_oracle(step, D.OracleAdaDelta, kw, flavour, clip)


def test_step_size_comes_from_the_old_acc_delta(host):
    """delta = sqrt(acc_delta + eps) / sqrt(acc_g + eps) * grad reads acc_delta BEFORE this step updates it: from zero
    states the first step is sqrt(eps) / sqrt((1 - rho) g^2 + eps) * g"""
    f = ctypes.c_float
    p = lambda a: a.ctypes.data_as(F32P)       # noqa: E731
    g = np.array([1.0, -2.0, 0.5], np.float32)
    w = np.zeros(3, np.float32)
    s = [np.zeros(3, np.float32) for _ in range(2)]
    eta = _F(1. - 0.9)
    host.host_adadelta(ctypes.c_int64(3), p(g), p(w), p(s[0]), p(s[1]), f(1.0), f(0.0), f(eta), f(0.9), f(1e-6),
                       f(1.0), f(-1.0))
    ag = eta * (g * g)
    delta = np.sqrt(_F(1e-6)) / np.sqrt(ag + _F(1e-6)) * g
    assert np.array_equal(w, -delta)
    assert np.array_equal(s[1], eta * (delta * delta))


def test_per_key_scalars_defaults_and_multipliers():
    """what the fused kernel receives per key: lr = learning rate x lr_mult (double, rounded once), eta = 1 - rho in
    double, rounded once (not 1 - float(rho)), wd = wd x wd_mult; none depends on t.  The reference class's defaults
    (learning_rate 1.0, rho 0.9, epsilon 1e-6, adadelta.py:62) for a C caller that names "adadelta" alone"""
    kv = T.c_caller_store("adadelta")
    dflt = D.OracleAdaDelta()
    for t in (1, 2, 7, 10 ** 6):
        T.set_count(kv, 0, t)
        got = T.key_hyper(kv, 0)
        assert got == dflt.key_scalars(0, t) == (_F(1.0), _F(0), _F(1. - 0.9)), (t, got)
    assert _F(1. - 0.9) != _F(1) - _F(0.9)
    opt = mx.optimizer.create("adadelta")
    assert isinstance(opt, mx.optimizer.AdaDelta)
    assert (opt.learning_rate, opt.rho, opt.epsilon) == (1.0, 0.9, 1e-6)
    assert mx.optimizer.fused_name_of(opt) == "adadelta"
    assert mx.optimizer.fused_name_of(mx.optimizer.AdaDelta(use_fused_step=False)) is None
    for rho in (0.95, 0.99, 0.8):
        opt = mx.optimizer.AdaDelta(learning_rate=0.3, rho=rho, epsilon=1e-4, wd=0.02, clip_gradient=0.0)
        opt.set_lr_mult({1: 0.5})
        opt.set_wd_mult({1: 3.0})
        kv.set_optimizer(opt)
        kw = opt.fused_kwargs()
        assert (kw["rho"], kw["epsilon"], kw["clip_gradient"]) == (rho, 1e-4, 0.0)
        oopt = D.OracleAdaDelta(learning_rate=0.3, rho=rho, epsilon=1e-4, wd=0.02, lr_mult={1: 0.5}, wd_mult={1: 3.0})
        for k, lr, wd in ((0, 0.3, 0.02), (1, 0.15, 0.06)):
            got = T.key_hyper(kv, k)
            assert got == oopt.key_scalars(k) == (_F(lr), _F(wd), _F(1. - rho)), (rho, k, got)
        # each of these complements differs from the float subtraction
        assert _F(1. - rho) != _F(1) - _F(rho), rho


def test_create_state_follows_the_reference_tuple_order():
    """create_state: ``(acc_g, acc_delta)``, two float32 zeros -- the engine's state0, state1; one torch `step` leaves
    the oracle's states and weight there"""
    try:
        import torch
    except ImportError:
        pytest.skip("create_state allocates torch tensors")
    w0 = np.array([0.5, -0.25, 1.0, 0.0, 2.0], np.float32)
    g = np.array([0.3, -0.7, 0.0, 1.5, -0.1], np.float32)
    w = mx.nd.array(w0)
    opt = mx.optimizer.AdaDelta(learning_rate=0.5, rho=0.95, use_fused_step=False)
    s = opt.create_state(0, w)
    assert len(s) == 2 and all(tuple(x.shape) == (5,) and x.dtype == torch.float32 and not x.any() for x in s)
    opt.update([0], [w], [mx.nd.array(g)], [s])
    oopt = D.OracleAdaDelta(learning_rate=0.5, rho=0.95)
    ow = w0.copy()
    oopt.update(0, ow, g)
    for x, want in zip(s, oopt.states[0]):
        np.testing.assert_allclose(x.cpu().numpy(), want, rtol=1e-6)
    np.testing.assert_allclose(w.asnumpy(), ow, rtol=1e-6)


@pytest.mark.parametrize("devices", [1, 2, 4, 8])
def test_gpu_adadelta_on_the_simulator(sim_lib, devices):
    T.run_gpu_file_on_sim(sim_lib, devices, "test_gpu_adadelta.py", 16 if devices == 1 else 17)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_process_per_gpu_on_the_simulator(sim_lib, world, tmp_path):
    """two-shot keys with two sharded states, a checkpoint of them on every rank, and the multicast kernel forced:
    within 1e-6 of the oracle"""
    outs = T.run_workers(sim_lib, world, tmp_path, "adadelta_mp_worker.py", "ADADELTA", {})
    assert all("ADADELTA_NVLS_OK" in o for o in outs), outs[0][-2000:]


@pytest.mark.parametrize("world", [3, 8])
def test_one_process_per_gpu_under_the_tree_on_the_simulator(sim_lib, world, tmp_path):
    T.run_workers(sim_lib, world, tmp_path, "adadelta_mp_worker.py", "ADADELTA", {"MXKV_STEP_OPT_TREE": "1"})
