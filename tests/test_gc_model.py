"""The numpy model of gradient compression (tests/gc_model.py) against the oracle codec, which is pinned to the
reference's bit-level simulator (tests/golden/compression.npz): codes, packed bytes, residuals and dequantised values
bit for bit on every tie, signed-zero, subnormal and non-finite vector the GPU edge tests push
(tests/test_gpu_compression_edges.py).  The two share no code, so an error that the oracle and the kernel had in
common would show here as a disagreement with the model."""
import os
import sys

import numpy as np
import pytest

from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gc_model as M  # noqa: E402

CASES = [(2, 0.5), (2, 0.3), (2, 1.0), (1, 0.0), (1, 0.5), (1, -0.25)]
SIZES = [1, 15, 16, 17, 31, 32, 33, 4097]


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _oracle(bits, g, res, thr):
    """one push through the oracle codec: (packed bytes, dequantised values); ``res`` is updated in place"""
    q = O.quantize_2bit if bits == 2 else O.quantize_1bit
    d = O.dequantize_2bit if bits == 2 else O.dequantize_1bit
    packed = q(g, res, thr)
    return packed, d(packed, g.size, thr)


@pytest.mark.parametrize("bits,thr", CASES)
@pytest.mark.parametrize("nonfinite", [False, True])
def test_model_matches_the_oracle_codec(bits, thr, nonfinite):
    for E in SIZES:
        grads = M.special_steps(bits, thr, E, 5, seed=E + bits, nonfinite=nonfinite)
        res_o = np.zeros(E, np.float32)
        model = M.Model(bits, thr, E)
        for s, g in enumerate(grads):
            packed, deq = _oracle(bits, g, res_o, thr)
            codes = model.push([g])
            what = "%d-bit thr %r E %d step %d" % (bits, thr, E, s)
            assert np.array_equal(M.pack(bits, codes[0]), packed), what + ": packed codes"
            assert np.array_equal(_u32(model.res[0]), _u32(res_o)), what + ": residual"
            assert np.array_equal(_u32(model.deq(codes)[0]), _u32(deq)), what + ": dequantised"


@pytest.mark.parametrize("bits,thr", CASES)
def test_the_threshold_decides_as_the_reference(bits, thr):
    """2-bit fires at r >= thr and r <= -thr; 1-bit only at r > thr (a tie goes to -1)"""
    t = np.float32(thr)
    r = np.array([t, -t, np.nextafter(t, np.float32(np.inf)), np.nextafter(t, np.float32(-np.inf))], np.float32)
    code, _ = M.quantize(bits, r, np.zeros_like(r), thr)
    if bits == 2:
        assert code.tolist() == [1, -1, 1, 0]
    else:
        assert code.tolist() == [-1, 1 if -t > t else -1, 1, -1]
    packed, _ = _oracle(bits, r.copy(), np.zeros_like(r), thr)
    assert np.array_equal(M.pack(bits, code), packed)


@pytest.mark.parametrize("bits,thr", CASES)
def test_non_finite_residuals_are_sticky(bits, thr):
    """the reference's behaviour, pinned: a NaN residual never fires in 2-bit and is -1 in 1-bit; an infinite one
    fires in its own direction at every later step, whatever the gradient"""
    g0 = np.array([np.nan, np.inf, -np.inf], np.float32)
    model = M.Model(bits, thr, 3)
    res_o = np.zeros(3, np.float32)
    rng = np.random.default_rng(bits)
    for s in range(6):
        g = g0 if s == 0 else rng.uniform(-5, 5, 3).astype(np.float32)
        packed, _ = _oracle(bits, g, res_o, thr)
        code = model.push([g])[0]
        assert np.array_equal(M.pack(bits, code), packed)
        assert code.tolist() == ([0, 1, -1] if bits == 2 else [-1, 1, -1]), (s, code)
        assert np.isnan(res_o[0]) and res_o[1] == np.inf and res_o[2] == -np.inf
