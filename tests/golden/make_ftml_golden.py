"""Regenerates tests/golden/ftml_steps.npz.  Needs the reference source tree (make_golden.REF).

ftml_steps.npz -- weights produced by the reference's own non-fused ``FTML.step`` (python/mxnet/optimizer/ftml.py:80-125),
executed from the reference file on the float32 numpy stand-in for NDArray of make_golden.py (``_step_functions``,
``_FakeOptimizer``; nothing is copied into this repository).  The option levels of the reference's test_ftml -- beta1
0.6 / 0.5, beta2 0.999 / 0.8, clip_gradient none / 0.4, rescale_grad 1 / 0.14, wd 0 / 0.03 -- in 8 sets in which every
pair of values of two options meets (the two-level orthogonal array of 8 runs, checked below) x 4 shapes ((3, 4, 5),
(10, 4), (7,), (1001,)) x 6 steps, learning rate 0.0025 and epsilon 1e-8 (the class defaults).  It pins
tests/ftml_oracle.py (tests/test_ftml.py, within the float32 tolerance of the reference's test_ftml: rtol 1e-3,
atol 1e-4).  The other fixtures stay make_golden.py's.
"""
import importlib.util
import itertools
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

LEVELS = [(0.6, 0.5), (0.999, 0.8), (None, 0.4), (1.0, 0.14), (0.0, 0.03)]
# (beta1, beta2, clip_gradient, rescale_grad, wd): run i takes level parity(i & j) of column j, for five of the seven
# columns j = 1..7 of the array
COLUMNS = (1, 2, 4, 3, 5)
GRID = [tuple(LEVELS[c][bin(i & j).count("1") & 1] for c, j in enumerate(COLUMNS)) for i in range(8)]
STEPS = 6
SHAPES = [(3, 4, 5), (10, 4), (7,), (1001,)]


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


def ftml_steps():
    """`step` scales the gradient in place (`grad *= self.rescale_grad`), so every step gets a fresh gradient array."""
    assert _covers_every_pair(GRID)
    mg = _make_golden()
    out = {}
    fns = mg._step_functions("ftml.py", "FTML", ["step"])
    rng = np.random.default_rng(20261018)
    meta = []
    for ci, (beta1, beta2, clip_g, rescale, wd) in enumerate(GRID):
        lr = 0.0025
        kw = dict(beta1=beta1, beta2=beta2, epsilon=1e-8, clip_gradient=clip_g, rescale_grad=rescale)
        for si, shape in enumerate(SHAPES):
            opt = mg._FakeOptimizer(fns, lr, wd, **kw)
            w = mg._nd(rng.uniform(0, 1, shape))
            state = tuple(mg._nd(np.zeros(shape)) for _ in range(3))       # d, v, z
            tag = "c%d_s%d" % (ci, si)
            out["w0_" + tag] = np.asarray(w).copy()
            for t in range(STEPS):
                g = rng.uniform(-1, 1, shape).astype(np.float32)
                out["g%d_%s" % (t, tag)] = g
                opt.step([0], [w], [mg._nd(g.copy())], [state])
                out["w%d_%s" % (t + 1, tag)] = np.asarray(w).copy()
        meta.append(repr(("ftml", lr, wd, kw)))
    out["cases"] = np.array(meta)
    out["steps"] = np.array([STEPS])
    np.savez_compressed(os.path.join(HERE, "ftml_steps.npz"), **out)


if __name__ == "__main__":
    ftml_steps()
    print("wrote", os.path.join(HERE, "ftml_steps.npz"))
