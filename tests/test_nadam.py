"""Nadam on the store without a GPU: the oracle against the reference's own `Nadam.step` (golden/nadam_steps.npz) bit
for bit, the kernel's Nadam arithmetic compiled for the host against the oracle bit for bit, the per-key scalars and the
momentum-schedule product the store keeps, and tests/test_gpu_nadam.py plus a one-process-per-GPU worker
(tests/nadam_mp_worker.py) on the simulated CUDA runtime (tests/sim).

Counterpart of the reference's tests/python/unittest/test_optimizer.py::test_nadam.  The reference has no operator for
Nadam: its `step` is the definition, so the fixture tests/golden/make_nadam_golden.py writes from it pins the oracle
(tests/nadam_oracle.py) bit for bit, and the oracle pins the kernel.  Nadam's `m_schedule` is one product for the whole
optimizer, multiplied by every key update in call order; the fixture updates four keys with one optimizer so that the
coupling shows while `1 - m_schedule` is still below 1.0f."""
import ctypes
import os
import sys

import numpy as np
import pytest

import mxnet_b200 as mx

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import nadam_oracle as N  # noqa: E402
from adamax_oracle import clip_on  # noqa: E402
from test_adamax import (F32P, _F, build_host, c_caller_store, check_host_against_oracle, golden,  # noqa: E402
                         key_hyper, load_generator, run_gpu_file_on_sim, run_workers, same, set_count, sim_lib)

NKEYS = 4


def m_schedule(kv):
    return kv._get_scalar("m_schedule")


def replay_golden(ci, lr, wd, kw, d):
    """the fixture's run ``ci`` through the oracle; yields (step, oracle, weights) after every step"""
    opt = N.OracleNadam(learning_rate=lr, wd=wd, **kw)
    ws = [d["w0_c%d_k%d" % (ci, k)].copy() for k in range(NKEYS)]
    active = d["active_c%d" % ci]
    for t in range(int(d["steps"][0])):
        for k in range(NKEYS):
            if active[t, k]:
                opt.update(k, ws[k], d["g%d_c%d_k%d" % (t, ci, k)])
        yield t, opt, ws


def test_oracle_matches_the_reference_step_golden():
    """nadam_steps.npz: the reference's Nadam.step (nadam.py:74-124) over 9 option sets, four keys sharing one
    optimizer, 6 steps; the oracle reproduces every weight, both states and m_schedule after every step bit for bit"""
    d, cases = golden("nadam")
    assert len(cases) == 9 and int(d["steps"][0]) == 6
    for ci, (tag_name, lr, wd, kw) in enumerate(cases):
        assert tag_name == "nadam"
        for t, opt, ws in replay_golden(ci, lr, wd, kw, d):
            for k in range(NKEYS):
                tag = "%d_c%d_k%d" % (t + 1, ci, k)
                assert same(ws[k], d["w" + tag]), (ci, t, k, kw)
                for i in range(2):
                    assert same(opt.states[k][i], d["s%d_%s" % (i, tag)]), (ci, t, k, i, kw)
            assert opt.m_schedule == d["msched_c%d" % ci][t], (ci, t)


def test_golden_covers_the_option_pairs_and_the_coupled_window():
    """the 8 option sets meet every pair of levels, one more clips at 0, the clip binds somewhere; 1 - m_schedule is
    below 1.0f through the first steps of every run (the product couples the keys) and reaches 1.0f in some; one run
    leaves a key behind, so that keys update at different counts"""
    gen = load_generator("nadam")
    assert gen.covers_every_pair(gen.GRID)
    d, cases = golden("nadam")
    names = gen.NAMES
    assert [tuple(wd if n == "wd" else kw[n] for n in names) for _, _, wd, kw in cases] == gen.GRID + gen.EXTRA
    assert [o[names.index("clip_gradient")] for o in gen.EXTRA] == [0.0]
    binds, reaches_one, uneven = False, False, False
    for ci, (_, lr, wd, kw) in enumerate(cases):
        ms = d["msched_c%d" % ci]
        assert _F(1. - ms[1]) < 1.0, (ci, ms)          # two steps of four keys: still coupled
        reaches_one = reaches_one or _F(1. - ms[-1]) == 1.0
        g = d["g0_c%d_k3" % ci] * _F(kw["rescale_grad"])
        binds = binds or (kw["clip_gradient"] is not None and np.abs(g).max() > kw["clip_gradient"])
        uneven = uneven or len(set(d["active_c%d" % ci].sum(axis=0))) > 1
    assert binds and reaches_one and uneven


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return build_host(tmp_path_factory, "nadam")


def host_step_fn(host):
    f = ctypes.c_float
    p = lambda a: a.ctypes.data_as(F32P)       # noqa: E731

    def step(opt, t, g, w, st):
        lr, wd = opt._lr_wd(0)
        _, sc = N.nadam_scalars(opt.beta1, opt.beta2, opt.schedule_decay, t, opt.m_schedule)
        g_div, m_div, mom_t1, c_mom_t, coef2 = sc
        step.g_divs.append(g_div)
        clip_op = opt.clip_gradient if clip_on(opt.clip_gradient) else -1.0
        assert host.host_nadam(ctypes.c_int64(w.size), p(g), p(w), p(st[0]), p(st[1]), f(lr), f(wd), f(coef2),
                               f(g_div), f(m_div), f(mom_t1), f(c_mom_t), f(opt.beta1), f(opt.beta2),
                               f(_F(1. - opt.beta1)), f(_F(1. - opt.beta2)), f(opt.epsilon), f(opt.rescale_grad),
                               f(clip_op)) == 0
    step.g_divs = []
    return step


@pytest.mark.parametrize("start", [1.0, 1e-9])
@pytest.mark.parametrize("clip", [None, 0.4, 0.0, -0.3])
@pytest.mark.parametrize("wd", [0.0, 0.03])
@pytest.mark.parametrize("flavour", ["f32", "lp"])
def test_kernel_arithmetic_on_the_host_is_the_oracle_bit_for_bit(host, flavour, wd, clip, start):
    """update_one<OPT_NADAM> against the oracle at update counts 1, 2, 7 and 10^6, the schedule product carried from
    one to the next: from a fresh optimizer's 1 (1 - m_schedule below 1.0f) and from one far into training (1.0f):
    float32 keys, and the fp32 master of 16-bit keys with the stored weight its one rounding to float16 / bfloat16"""
    kw = dict(learning_rate=0.01, beta1=0.9, beta2=0.8, epsilon=1e-6, schedule_decay=0.008, wd=wd, rescale_grad=0.5,
              m_schedule=start)
    step = host_step_fn(host)
    check_host_against_oracle(step, N.OracleNadam, kw, flavour, clip)
    assert all((g < 1.0) == (start == 1.0) for g in step.g_divs), step.g_divs


def test_per_key_scalars_and_the_schedule_product():
    """what the fused kernel receives per key for update count t: lr = learning rate x lr_mult rounded once, wd =
    wd x wd_mult, eta = coef2 = 1 - beta2^t in double rounded once.  The reference class's defaults (learning_rate
    0.001, beta1 0.9, beta2 0.999, epsilon 1e-8, schedule_decay 0.004, nadam.py:58-67) for a C caller that names
    "nadam" alone; m_schedule starts at 1, an explicit one sets it, re-sent hyper-parameters keep it and a new
    optimizer (reset_states) starts from its own"""
    from mxnet_b200.base import _LIB, check_call, c_str, c_str_array
    kv = c_caller_store("nadam")
    dflt = N.OracleNadam()
    for t in (1, 2, 7, 1000, 10 ** 6):
        set_count(kv, 0, t)
        assert key_hyper(kv, 0) == dflt.key_scalars(0, t), t
    assert dflt.key_scalars(0, 1) == (_F(0.001), _F(0), _F(1. - 0.999))
    assert m_schedule(kv) == 1.0

    def send(**kw):
        keys = list(kw)
        check_call(_LIB.MXKVB200SetOptimizer(kv.handle, c_str("nadam"), len(keys), c_str_array(keys),
                                             c_str_array([str(kw[k]) for k in keys])))
    send(m_schedule=0.123456789012345678)
    assert m_schedule(kv) == 0.123456789012345678     # parsed as a double, not rounded to float
    kv._set_scalar("m_schedule", 0.0625)
    send(rescale_grad=0.5)                            # re-sent: the product stays
    assert m_schedule(kv) == 0.0625
    send(rescale_grad=0.5, reset_states=True)         # a new optimizer without a product of its own starts at 1
    assert m_schedule(kv) == 1.0
    with pytest.raises(mx.base.MXNetError):
        kv._get_scalar("momentum")

    opt = mx.optimizer.create("nadam")
    assert isinstance(opt, mx.optimizer.Nadam)
    assert (opt.learning_rate, opt.beta1, opt.beta2, opt.epsilon, opt.schedule_decay, opt.m_schedule) == \
        (0.001, 0.9, 0.999, 1e-8, 0.004, 1.0)
    assert mx.optimizer.fused_name_of(opt) == "nadam"
    assert mx.optimizer.fused_name_of(mx.optimizer.Nadam(use_fused_step=False)) is None
    opt = mx.optimizer.Nadam(learning_rate=0.03, beta1=0.8, beta2=0.95, epsilon=1e-4, schedule_decay=0.01, wd=0.02,
                             clip_gradient=0.0)
    opt.m_schedule = 0.3
    opt.set_lr_mult({1: 0.5})
    opt.set_wd_mult({1: 3.0})
    kv.set_optimizer(opt)
    kw = opt.fused_kwargs()
    assert (kw["beta1"], kw["beta2"], kw["epsilon"], kw["clip_gradient"], kw["schedule_decay"], kw["m_schedule"]) == \
        (0.8, 0.95, 1e-4, 0.0, 0.01, 0.3)
    assert m_schedule(kv) == 0.3
    oopt = N.OracleNadam(learning_rate=0.03, beta2=0.95, wd=0.02, lr_mult={1: 0.5}, wd_mult={1: 3.0})
    for k, lr, wd in ((0, 0.03, 0.02), (1, 0.015, 0.06)):
        for t in (1, 2, 3, 7, 200):
            set_count(kv, k, t)
            got = key_hyper(kv, k)
            assert got == oopt.key_scalars(k, t) == (_F(lr), _F(wd), _F(1. - 0.95 ** t)), (k, t, got)


def test_create_state_and_the_python_step_follow_the_reference():
    """create_state: ``(mean, var)``, two float32 zeros -- the engine's state0, state1; the torch `step` over two
    indices advances m_schedule exactly as the oracle does and leaves its weights and states there"""
    try:
        import torch
    except ImportError:
        pytest.skip("create_state allocates torch tensors")
    rng = np.random.default_rng(3)
    w0 = [rng.uniform(-1, 1, 5).astype(np.float32), rng.uniform(-1, 1, 3).astype(np.float32)]
    ws = [mx.nd.array(w) for w in w0]
    opt = mx.optimizer.Nadam(learning_rate=0.01, beta1=0.5, beta2=0.8, use_fused_step=False)
    st = [opt.create_state(i, w) for i, w in enumerate(ws)]
    assert all(len(s) == 2 and all(x.dtype == torch.float32 and not x.any() for x in s) for s in st)
    oopt = N.OracleNadam(learning_rate=0.01, beta1=0.5, beta2=0.8)
    ow = [w.copy() for w in w0]
    for _ in range(3):
        gs = [rng.uniform(-1, 1, w.shape).astype(np.float32) for w in w0]
        opt.update([0, 1], ws, [mx.nd.array(g) for g in gs], st)
        for k in (0, 1):
            oopt.update(k, ow[k], gs[k])
        assert opt.m_schedule == oopt.m_schedule
    for k in (0, 1):
        np.testing.assert_allclose(ws[k].asnumpy(), ow[k], rtol=1e-6)
        for x, want in zip(st[k], oopt.states[k]):
            np.testing.assert_allclose(x.cpu().numpy(), want, rtol=1e-6)


# ---------------------------------------------------------------------------
# the simulated CUDA runtime
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("devices", [1, 2, 8])
def test_gpu_nadam_on_the_simulator(sim_lib, devices):
    run_gpu_file_on_sim(sim_lib, devices, "test_gpu_nadam.py", 8 if devices == 1 else 10)


@pytest.mark.parametrize("world", [2, 8])
def test_one_process_per_gpu_on_the_simulator(sim_lib, world, tmp_path):
    """two-shot keys with two sharded states and the schedule product advanced alike on every rank, a checkpoint on
    every rank, and the multicast kernel forced: within 1e-6 of the oracle"""
    outs = run_workers(sim_lib, world, tmp_path, "nadam_mp_worker.py", "NADAM", {})
    assert all("NADAM_NVLS_OK" in o for o in outs), outs[0][-2000:]
