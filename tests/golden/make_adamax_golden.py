"""Regenerates tests/golden/adamax_steps.npz.  Needs the reference source tree (make_golden.REF).

adamax_steps.npz -- weights produced by the reference's own ``Adamax.step`` (python/mxnet/optimizer/adamax.py:74-111),
executed from the reference file on the float32 numpy stand-in for NDArray of make_golden.py (``_step_functions``,
``_FakeOptimizer``; nothing is copied into this repository), with ``NDabs`` added here as ``np.abs``.  The option levels
of the reference's test_adamax -- beta1 0.9 / 0.5, beta2 0.999 / 0.8, clip_gradient none / 0.4, rescale_grad 1 / 0.14,
wd 0 / 0.03 -- in 8 sets in which every pair of values of two options meets (the two-level orthogonal array of 8 runs,
checked below), plus one set with clip_gradient 0 (which ``step`` applies), x 4 shapes ((3, 4, 5), (10, 4), (7,),
(1001,)) x 6 steps, learning rate 0.002 and epsilon 1e-8 (the class defaults).  It pins tests/adamax_oracle.py bit for
bit (tests/test_adamax.py).  tests/golden/make_adadelta_golden.py runs the same machinery over AdaDelta.
"""
import importlib.util
import itertools
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

LEVELS = [(0.9, 0.5), (0.999, 0.8), (None, 0.4), (1.0, 0.14), (0.0, 0.03)]
NAMES = ("beta1", "beta2", "clip_gradient", "rescale_grad", "wd")
# run i takes level parity(i & j) of column j, for five of the seven columns j = 1..7 of the array
COLUMNS = (1, 2, 4, 3, 5)
STEPS = 6
SHAPES = [(3, 4, 5), (10, 4), (7,), (1001,)]


def orthogonal_grid(levels):
    return [tuple(levels[c][bin(i & j).count("1") & 1] for c, j in enumerate(COLUMNS)) for i in range(8)]


GRID = orthogonal_grid(LEVELS)
# the gradient clip at 0: every gradient element clipped to +-0, so the weight decay alone drives the update
EXTRA = [(LEVELS[0][0], LEVELS[1][0], 0.0, LEVELS[3][1], LEVELS[4][1])]


def covers_every_pair(grid):
    values = [sorted(set(map(repr, col))) for col in zip(*grid)]
    seen = {(i, repr(r[i]), j, repr(r[j])) for r in grid for i, j in itertools.combinations(range(len(r)), 2)}
    return all((i, a, j, b) in seen for i, j in itertools.combinations(range(len(values)), 2)
               for a in values[i] for b in values[j])


def _make_golden():
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_steps(fname, cls, names, sets, lr, fixed, seed, out_name, tag_name):
    """``step`` of class ``cls`` in the reference file ``fname`` over the option ``sets`` (values in the order of
    ``names``; ``wd`` goes to the stand-in optimizer, the rest are attributes) and ``fixed`` attributes.  ``step``
    scales the gradient in place (``grad *= self.rescale_grad``), so every step gets a fresh gradient array."""
    mg = _make_golden()
    fns = mg._step_functions(fname, cls, ["step"])
    fns["step"].__globals__["NDabs"] = lambda x: np.abs(x).view(mg._F32)
    out = {}
    rng = np.random.default_rng(seed)
    meta = []
    for ci, values in enumerate(sets):
        kw = dict(fixed, **dict(zip(names, values)))
        wd = kw.pop("wd")
        for si, shape in enumerate(SHAPES):
            opt = mg._FakeOptimizer(fns, lr, wd, **kw)
            w = mg._nd(rng.uniform(0, 1, shape))
            state = tuple(mg._nd(np.zeros(shape)) for _ in range(2))
            tag = "c%d_s%d" % (ci, si)
            out["w0_" + tag] = np.asarray(w).copy()
            for t in range(STEPS):
                g = rng.uniform(-1, 1, shape).astype(np.float32)
                out["g%d_%s" % (t, tag)] = g
                opt.step([0], [w], [mg._nd(g.copy())], [state])
                out["w%d_%s" % (t + 1, tag)] = np.asarray(w).copy()
            for i, s in enumerate(state):
                out["s%d_%s" % (i, tag)] = np.asarray(s).copy()
        meta.append(repr((tag_name, lr, wd, kw)))
    out["cases"] = np.array(meta)
    out["steps"] = np.array([STEPS])
    np.savez_compressed(os.path.join(HERE, out_name), **out)


def adamax_steps():
    assert covers_every_pair(GRID)
    run_steps("adamax.py", "Adamax", NAMES, GRID + EXTRA, 0.002, dict(epsilon=1e-8), 20261019, "adamax_steps.npz",
              "adamax")


if __name__ == "__main__":
    adamax_steps()
    print("wrote", os.path.join(HERE, "adamax_steps.npz"))
