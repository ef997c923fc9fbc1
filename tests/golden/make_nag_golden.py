"""Regenerates tests/golden/nag_steps.npz.  Needs the reference source tree (make_golden.REF).

nag_steps.npz -- weights produced by the reference's own non-fused ``NAG.step`` (python/mxnet/optimizer/nag.py:72-109),
executed from the reference file on the float32 numpy stand-in for NDArray of make_golden.py (``_step_functions``,
``_FakeOptimizer``; nothing is copied into this repository).  8 option sets (momentum 0 / 0.9, clip_gradient none / 0.4,
rescale_grad 1 / 0.14 / 0.8, wd 0 / 0.03; every pair of values of two options meets in some set) x 4 shapes
((3, 4, 5), (10, 4), (7,), (1001,)) x 5 steps.  It pins tests/nag_oracle.py (tests/test_nag.py, within the tolerance of
the reference's own test_nag: rtol 1e-3, atol 1e-4).  The other fixtures stay make_golden.py's.
"""
import importlib.util
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def _make_golden():
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def nag_steps():
    """`step` scales the gradient in place (`grad *= self.rescale_grad`), so every step gets a fresh gradient array."""
    mg = _make_golden()
    out = {}
    nag = mg._step_functions("nag.py", "NAG", ["step"])
    rng = np.random.default_rng(20261016)
    meta = []
    # (momentum, clip_gradient, rescale_grad, wd)
    grid = [(0.9, None, 1.0, 0.0), (0.9, 0.4, 0.14, 0.03), (0.9, None, 0.8, 0.03), (0.9, 0.4, 1.0, 0.0),
            (0.9, 0.4, 0.8, 0.0), (0.0, None, 0.14, 0.0), (0.0, 0.4, 0.8, 0.03), (0.0, None, 1.0, 0.03)]
    for ci, (momentum, clip, rescale, wd) in enumerate(grid):
        lr = 0.1
        kw = dict(momentum=momentum, clip_gradient=clip, rescale_grad=rescale)
        for si, shape in enumerate([(3, 4, 5), (10, 4), (7,), (1001,)]):
            opt = mg._FakeOptimizer(nag, lr, wd, **kw)
            w = mg._nd(rng.uniform(0, 1, shape))
            state = mg._nd(np.zeros(shape)) if momentum != 0.0 else None
            tag = "c%d_s%d" % (ci, si)
            out["w0_" + tag] = np.asarray(w).copy()
            for t in range(5):
                g = rng.uniform(-1, 1, shape).astype(np.float32)
                out["g%d_%s" % (t, tag)] = g
                opt.step([0], [w], [mg._nd(g.copy())], [state])
                out["w%d_%s" % (t + 1, tag)] = np.asarray(w).copy()
        meta.append(repr(("nag", lr, wd, kw)))
    out["cases"] = np.array(meta)
    np.savez_compressed(os.path.join(HERE, "nag_steps.npz"), **out)


if __name__ == "__main__":
    nag_steps()
    print("wrote", os.path.join(HERE, "nag_steps.npz"))
