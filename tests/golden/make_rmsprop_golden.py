"""Regenerates tests/golden/rmsprop_steps.npz.  Needs the reference source tree (make_golden.REF).

rmsprop_steps.npz -- weights produced by the reference's own non-fused ``RMSProp.step``
(python/mxnet/optimizer/rmsprop.py:90-141), executed from the reference file on the float32 numpy stand-in for NDArray
of make_golden.py (``_step_functions``, ``_FakeOptimizer``; nothing is copied into this repository).  The options of
the reference's test_rms -- rho 0.9 / 0.5, momentum 0.9 / 0, centered False / True, clip_gradient none / 0.4,
clip_weights none / 0.01, rescale_grad 1 / 0.14, wd 0 / 0.03 -- in 8 sets in which every pair of values of two options
meets (the two-level orthogonal array of 8 runs, checked below) x 4 shapes ((3, 4, 5), (10, 4), (7,), (1001,)) x 5
steps, learning rate 0.01, epsilon 1e-8 (the class default).  It pins tests/rmsprop_oracle.py (tests/test_rmsprop.py,
within the float32 tolerance of the reference's own test_rms: rtol 1e-2, atol 1e-2).  The other fixtures stay
make_golden.py's.
"""
import importlib.util
import itertools
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

LEVELS = [(0.9, 0.5), (0.9, 0.0), (False, True), (None, 0.4), (None, 0.01), (1.0, 0.14), (0.0, 0.03)]
# (rho, momentum, centered, clip_gradient, clip_weights, rescale_grad, wd): run i takes level parity(i & j) of
# column j = 1..7
GRID = [tuple(LEVELS[j - 1][bin(i & j).count("1") & 1] for j in range(1, 8)) for i in range(8)]


def _covers_every_pair(grid):
    values = [sorted(set(map(repr, col))) for col in zip(*grid)]
    seen = {(i, repr(r[i]), j, repr(r[j])) for r in grid for i, j in itertools.combinations(range(len(r)), 2)}
    return all((i, a, j, b) in seen for i, j in itertools.combinations(range(len(values)), 2)
               for a in values[i] for b in values[j])


def _make_golden():
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def rmsprop_steps():
    """`step` scales the gradient in place (`grad *= self.rescale_grad`), so every step gets a fresh gradient array.
    Its weight clip writes in place (`clip(weight, ..., out=weight)`), which the stand-in's `clip` does not take: the
    compiled function gets one that does."""
    assert _covers_every_pair(GRID)
    mg = _make_golden()
    out = {}
    fns = mg._step_functions("rmsprop.py", "RMSProp", ["step"])
    F32 = type(mg._nd(np.zeros(1)))

    def clip(x, lo, hi, out=None):
        r = np.clip(np.asarray(x), np.float32(lo), np.float32(hi))
        if out is not None:
            out[...] = r
            return out
        return r.view(F32)

    fns["step"].__globals__["clip"] = clip
    rng = np.random.default_rng(20261016)
    meta = []
    for ci, (rho, momentum, centered, clip_g, clip_w, rescale, wd) in enumerate(GRID):
        lr = 0.01
        kw = dict(rho=rho, momentum=momentum, epsilon=1e-8, centered=centered, clip_weights=clip_w,
                  clip_gradient=clip_g, rescale_grad=rescale)
        for si, shape in enumerate([(3, 4, 5), (10, 4), (7,), (1001,)]):
            opt = mg._FakeOptimizer(fns, lr, wd, **kw)
            w = mg._nd(rng.uniform(0, 1, shape))
            state = tuple(mg._nd(np.zeros(shape)) for _ in range(3)) if centered else mg._nd(np.zeros(shape))
            tag = "c%d_s%d" % (ci, si)
            out["w0_" + tag] = np.asarray(w).copy()
            for t in range(5):
                g = rng.uniform(-1, 1, shape).astype(np.float32)
                out["g%d_%s" % (t, tag)] = g
                opt.step([0], [w], [mg._nd(g.copy())], [state])
                out["w%d_%s" % (t + 1, tag)] = np.asarray(w).copy()
        meta.append(repr(("rmsprop", lr, wd, kw)))
    out["cases"] = np.array(meta)
    np.savez_compressed(os.path.join(HERE, "rmsprop_steps.npz"), **out)


if __name__ == "__main__":
    rmsprop_steps()
    print("wrote", os.path.join(HERE, "rmsprop_steps.npz"))
