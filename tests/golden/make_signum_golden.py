"""Regenerates tests/golden/signum_steps.npz.  Needs the reference source tree (make_golden.REF).

signum_steps.npz -- weights produced by the reference's own non-fused ``Signum.step``
(python/mxnet/optimizer/signum.py:80-119), executed from the reference file on the float32 numpy stand-in for NDArray
of make_golden.py (``_step_functions``, ``_FakeOptimizer``; nothing is copied into this repository).  Options: momentum
0.9 / 0, clip_gradient none / 0.4, rescale_grad 1 / 0.14, wd 0 / 0.03, wd_lh 0 / 0.015 and learning rate 0.05 / 0.01,
in 8 sets in which every pair of values of two options meets (the two-level orthogonal array of 8 runs, checked
below) x 4 shapes ((3, 4, 5), (10, 4), (7,), (1001,)) x 5 steps; about one gradient element in eight is an exact 0.
Momentum 0 is there on purpose: both momentum options of the reference's own test_signum are 0.9, so it never reaches
signsgd_update.  The fixture pins tests/signum_oracle.py (tests/test_signum.py, within the float32 tolerance of the
reference's test_signum: rtol 1e-4, atol 1e-5).  The other fixtures stay make_golden.py's.
"""
import importlib.util
import itertools
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

LEVELS = [(0.9, 0.0), (None, 0.4), (1.0, 0.14), (0.0, 0.03), (0.0, 0.015), (0.05, 0.01)]
# (momentum, clip_gradient, rescale_grad, wd, wd_lh, learning_rate): run i takes level parity(i & j) of column j, for
# six of the seven columns j = 1..7 of the array
COLUMNS = (1, 2, 4, 3, 5, 6)
GRID = [tuple(LEVELS[c][bin(i & j).count("1") & 1] for c, j in enumerate(COLUMNS)) for i in range(8)]
# `step` rounds 1 - momentum and 1 - lr * wd_lh in double, the operators in float: the momentum whose sign is taken
# may differ in its last bits.  No non-zero momentum may lie this close to 0, so that no sign can flip between them.
NEAR_ZERO = 1e-5


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


def signum_steps():
    """`step` computes `(mom > 0) - (mom < 0)`; on the stand-in those comparisons are numpy bool arrays, whose
    difference raises.  NDArray's comparisons return 0 / 1 in the array's dtype: the arrays handed to `step` are of a
    stand-in subclass whose comparisons do that.  `step` scales the gradient in place, so every step gets a fresh
    gradient array."""
    assert _covers_every_pair(GRID)
    mg = _make_golden()
    F32 = type(mg._nd(np.zeros(1)))

    class Cmp(F32):
        def __gt__(self, other):
            return (np.asarray(self) > other).astype(np.float32).view(Cmp)

        def __lt__(self, other):
            return (np.asarray(self) < other).astype(np.float32).view(Cmp)

    def nd(a):
        return np.array(a, dtype=np.float32).view(Cmp)

    fns = mg._step_functions("signum.py", "Signum", ["step"])
    clip = fns["step"].__globals__["clip"]
    fns["step"].__globals__["clip"] = lambda x, lo, hi: np.asarray(clip(x, lo, hi)).view(Cmp)
    def run(fns_kw, lr, wd, momentum, shape, rng):
        """one (option set, shape) block: w0, the 5 gradients and the weight after each step, and the smallest
        non-zero |momentum| met (signsgd_update takes the sign of the gradient as given: inf)"""
        opt = mg._FakeOptimizer(fns, lr, wd, **fns_kw)
        w = nd(rng.uniform(0, 1, shape))
        state = nd(np.zeros(shape)) if momentum != 0.0 else None
        blk = {"w0": np.asarray(w).copy()}
        closest = np.inf
        for t in range(5):
            g = rng.uniform(-1, 1, shape).astype(np.float32)
            g[rng.uniform(0, 1, shape) < 0.125] = 0.0
            blk["g%d" % t] = g
            opt.step([0], [w], [nd(g.copy())], [state])
            if state is not None:
                pre = np.abs(np.asarray(state))
                closest = min(closest, float(pre[pre > 0].min()))
            blk["w%d" % (t + 1)] = np.asarray(w).copy()
        return blk, closest

    out = {}
    rng = np.random.default_rng(20261017)
    meta = []
    for ci, (momentum, clip_g, rescale, wd, wd_lh, lr) in enumerate(GRID):
        kw = dict(momentum=momentum, wd_lh=wd_lh, clip_gradient=clip_g, rescale_grad=rescale)
        for si, shape in enumerate([(3, 4, 5), (10, 4), (7,), (1001,)]):
            # a block whose momentum comes within NEAR_ZERO of 0 (a few in a thousand elements over 5 steps) is drawn
            # again from the same generator
            blk, closest = run(kw, lr, wd, momentum, shape, rng)
            while closest <= NEAR_ZERO:
                blk, closest = run(kw, lr, wd, momentum, shape, rng)
            for name, v in blk.items():
                out["%s_c%d_s%d" % (name, ci, si)] = v
        meta.append(repr(("signum", lr, wd, kw)))
    out["cases"] = np.array(meta)
    np.savez_compressed(os.path.join(HERE, "signum_steps.npz"), **out)


if __name__ == "__main__":
    signum_steps()
    print("wrote", os.path.join(HERE, "signum_steps.npz"))
