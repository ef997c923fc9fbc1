"""Regenerates tests/golden/adabelief_steps.npz.  Needs the reference source tree (make_golden.REF).

adabelief_steps.npz -- weights produced by the reference's own non-fused ``AdaBelief.step``
(python/mxnet/optimizer/adabelief.py:96-139), executed from the reference file on the float32 numpy stand-in for NDArray
of make_golden.py (``_step_functions``, ``_FakeOptimizer``; nothing is copied into this repository).  8 option sets
(beta1 0.9 / 0.5, beta2 0.999 / 0.8, clip_gradient none / 0.4, rescale_grad 1 / 0.14 / 0.8, wd 0 / 0.03, correct_bias
True / False; every pair of values of two options meets in some set, checked below) x 4 shapes ((3, 4, 5), (10, 4),
(7,), (1001,)) x 5 steps, epsilon 1e-6 (the class default).  It pins tests/adabelief_oracle.py (tests/test_adabelief.py,
within the tolerance of the reference's own test_adabelief: rtol 1e-3, atol 2e-3).  The other fixtures stay
make_golden.py's.
"""
import importlib.util
import itertools
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# (beta1, beta2, clip_gradient, rescale_grad, wd, correct_bias)
GRID = [(0.9, 0.999, None, 1.0, 0.0, True), (0.5, 0.999, None, 1.0, 0.03, False),
        (0.9, 0.8, None, 0.14, 0.03, True), (0.5, 0.8, 0.4, 0.8, 0.03, True),
        (0.9, 0.999, None, 0.8, 0.0, False), (0.5, 0.999, 0.4, 0.14, 0.0, False),
        (0.9, 0.8, 0.4, 1.0, 0.0, False), (0.9, 0.999, 0.4, 1.0, 0.0, True)]


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


def adabelief_steps():
    """`step` scales the gradient in place (`grad *= self.rescale_grad`), so every step gets a fresh gradient array."""
    assert _covers_every_pair(GRID)
    mg = _make_golden()
    out = {}
    fns = mg._step_functions("adabelief.py", "AdaBelief", ["step"])
    rng = np.random.default_rng(20261017)
    meta = []
    for ci, (beta1, beta2, clip, rescale, wd, correct_bias) in enumerate(GRID):
        lr = 0.01
        kw = dict(beta1=beta1, beta2=beta2, epsilon=1e-6, correct_bias=correct_bias, clip_gradient=clip,
                  rescale_grad=rescale)
        for si, shape in enumerate([(3, 4, 5), (10, 4), (7,), (1001,)]):
            opt = mg._FakeOptimizer(fns, lr, wd, **kw)
            w = mg._nd(rng.uniform(0, 1, shape))
            state = (mg._nd(np.zeros(shape)), mg._nd(np.zeros(shape)))
            tag = "c%d_s%d" % (ci, si)
            out["w0_" + tag] = np.asarray(w).copy()
            for t in range(5):
                g = rng.uniform(-1, 1, shape).astype(np.float32)
                out["g%d_%s" % (t, tag)] = g
                opt.step([0], [w], [mg._nd(g.copy())], [state])
                out["w%d_%s" % (t + 1, tag)] = np.asarray(w).copy()
        meta.append(repr(("adabelief", lr, wd, kw)))
    out["cases"] = np.array(meta)
    np.savez_compressed(os.path.join(HERE, "adabelief_steps.npz"), **out)


if __name__ == "__main__":
    adabelief_steps()
    print("wrote", os.path.join(HERE, "adabelief_steps.npz"))
