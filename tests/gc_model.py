"""An independent model of 1-bit / 2-bit gradient compression (src/kvstore/gradient_compression-inl.h), for tests.

It shares no code with the oracle codec (``oracle.quantize_*`` / ``dequantize_*``): whole arrays in numpy float32,
one IEEE single-precision operation per step of the reference's per-element loop, and codes kept as one small
integer per element (+1, 0, -1) instead of packed bits.  ``pack`` restates the reference's bit layout (byte j holds
elements 4j..4j+3 for 2-bit or 8j..8j+7 for 1-bit, the first in the most significant bits) so that a packed stream can
be compared with the oracle's.

Per element, with r = residual + grad:
  2-bit: r >= thr -> code +1, r -= thr;  r <= -thr -> code -1, r -= -thr;  else code 0.   Dequantised: code * thr.
  1-bit: r >  thr -> code +1, r -= 1;    else code -1, r += 1.                          Dequantised: +1 / -1.
A NaN residual compares false everywhere: it never fires in 2-bit and is always -1 in 1-bit.  An infinite residual
stays infinite, so it fires (in its sign's direction) at every later step.
"""
import numpy as np

_F = np.float32


def quantize(bits, grad, residual, thr):
    """one quantisation: (codes as int8, the new residual); ``residual`` is not modified"""
    r = np.asarray(residual, _F) + np.asarray(grad, _F)
    t = _F(thr)
    with np.errstate(invalid="ignore", over="ignore"):
        if bits == 2:
            pos = r >= t
            neg = ~pos & (r <= -t)
            code = pos.astype(np.int8) - neg.astype(np.int8)
            r = np.where(pos, r - t, np.where(neg, r - (-t), r))
        elif bits == 1:
            pos = r > t
            code = np.where(pos, 1, -1).astype(np.int8)
            r = np.where(pos, r - _F(1.0), r + _F(1.0))
        else:
            raise ValueError(bits)
    return code, r.astype(_F)


def dequantize(bits, code, thr):
    code = np.asarray(code)
    if bits == 2:
        t = _F(thr)
        return np.where(code > 0, t, np.where(code < 0, -t, _F(0.0))).astype(_F)
    return np.where(code > 0, _F(1.0), _F(-1.0)).astype(_F)


def pack(bits, code):
    """codes -> the reference's byte stream (whole 32-bit words, unused trailing positions 0)"""
    code = np.asarray(code).astype(np.int64)
    per_byte = 8 // bits
    nwords = -(-code.size // (32 // bits))
    field = np.zeros(nwords * 4 * per_byte, np.uint8)
    if bits == 2:
        field[:code.size] = np.where(code > 0, 3, np.where(code < 0, 2, 0))
    else:
        field[:code.size] = code > 0
    shifts = (np.arange(per_byte)[::-1] * bits).astype(np.uint8)
    return (field.reshape(-1, per_byte).astype(np.uint16) << shifts).sum(axis=1).astype(np.uint8)


def tie_values(thr):
    """residual values where a threshold decides: +-thr, one ulp either side of each, +-0, subnormals, and the
    1-bit boundary's neighbours +-1 (the residual moves by 1 there)"""
    t = _F(thr)
    sub = np.array([1e-45, 1e-40, np.finfo(_F).tiny / 2], _F)        # the smallest subnormal, two more
    v = [t, -t, np.nextafter(t, _F(np.inf)), np.nextafter(t, _F(-np.inf)),
         -np.nextafter(t, _F(np.inf)), -np.nextafter(t, _F(-np.inf)), _F(0.0), _F(-0.0), _F(1.0), _F(-1.0)]
    return np.concatenate([np.array(v, _F), sub, -sub, t + sub, t - sub])


def special_steps(bits, thr, size, steps, seed, nonfinite):
    """gradients for ``steps`` pushes of one slot: the first lands every residual exactly on a tie value (residuals
    start at 0); each later one lands the residual the model predicts on a tie value again where a float32
    difference reaches it exactly, and is a tie value itself elsewhere.  With ``nonfinite``, NaN / +inf / -inf at
    the first and last element of word 0 and word 1 and in the partial last word, at the first step only."""
    rng = np.random.default_rng(seed)
    ties = tie_values(thr)
    per_word = 32 // bits
    out, res = [], np.zeros(size, _F)
    for s in range(steps):
        target = ties[rng.integers(0, ties.size, size)]
        with np.errstate(invalid="ignore", over="ignore"):
            g = (target - res).astype(_F)
            hit = np.isfinite(g) & ((res + g) == target) & (np.signbit(res + g) == np.signbit(target))
            g = np.where(hit, g, target).astype(_F)
        if nonfinite and s == 0:
            where = [0, per_word - 1, per_word, 2 * per_word - 1, size - 1, size - 2, size - 3]
            vals = [np.nan, np.inf, -np.inf, np.nan, np.inf, -np.inf, np.nan]
            for i, x in zip(where, vals):
                if 0 <= i < size:
                    g[i] = x
        out.append(g)
        _, res = quantize(bits, g, res, thr)
    return out


class Model(object):
    """n pushed-value slots of one key, each with its own residual; ``push`` returns the codes of every slot.  Slots
    that a push does not reach keep their residual (comm.h:575-580)"""

    def __init__(self, bits, thr, size):
        self.bits, self.thr, self.size = bits, thr, size
        self.res = []

    def push(self, grads):
        while len(self.res) < len(grads):
            self.res.append(np.zeros(self.size, _F))
        codes = []
        for k, g in enumerate(grads):
            c, self.res[k] = quantize(self.bits, g, self.res[k], self.thr)
            codes.append(c)
        return codes

    def deq(self, codes):
        return [dequantize(self.bits, c, self.thr) for c in codes]
