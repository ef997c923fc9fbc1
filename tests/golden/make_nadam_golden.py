"""Regenerates tests/golden/nadam_steps.npz.  Needs the reference source tree (make_golden.REF).

nadam_steps.npz -- weights, states and the momentum-schedule product produced by the reference's own ``Nadam.step``
(python/mxnet/optimizer/nadam.py:74-124), executed from the reference file on the float32 numpy stand-in for NDArray
of make_golden.py (``_step_functions``, ``_FakeOptimizer``; nothing is copied into this repository).  The option levels
of the reference's test_nadam -- beta1 0.9 / 0.5, beta2 0.999 / 0.8, schedule_decay 0.004 / 0.008, clip_gradient
none / 0.4, rescale_grad 1 / 0.14, wd 0 / 0.03 -- in 8 sets in which every pair of values of two options meets (the
two-level orthogonal array of 8 runs, checked below), plus one set with clip_gradient 0 (which ``step`` applies).

Nadam's ``m_schedule`` is ONE attribute of the optimizer, multiplied by every update of every index, so each run
updates four keys of different shapes with one optimizer object, in key order, for 6 steps: at most 24 updates, so
that ``1 - m_schedule`` is still below 1.0f and the coupling between the keys shows in the weights.  Run 3 skips key 2
on steps 1 and 3, so its keys reach different update counts.  Recorded after every step: every weight, both states
and ``m_schedule``.  Learning rate 0.001 and epsilon 1e-8 (the class defaults).  It pins tests/nadam_oracle.py bit for
bit (tests/test_nadam.py).
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_adamax_golden import HERE, covers_every_pair, _make_golden   # noqa: E402

LEVELS = [(0.9, 0.5), (0.999, 0.8), (0.004, 0.008), (None, 0.4), (1.0, 0.14), (0.0, 0.03)]
NAMES = ("beta1", "beta2", "schedule_decay", "clip_gradient", "rescale_grad", "wd")
# run i takes level parity(i & j) of column j, for six of the seven columns j = 1..7 of the array
COLUMNS = (1, 2, 4, 3, 5, 6)
STEPS = 6
SHAPES = [(3, 4, 5), (10, 4), (7,), (257,)]
SKIP = {3: {(1, 2), (3, 2)}}        # run -> {(step, key)} not updated


def orthogonal_grid(levels):
    return [tuple(levels[c][bin(i & j).count("1") & 1] for c, j in enumerate(COLUMNS)) for i in range(8)]


GRID = orthogonal_grid(LEVELS)
EXTRA = [(LEVELS[0][0], LEVELS[1][0], LEVELS[2][0], 0.0, LEVELS[4][1], LEVELS[5][1])]


def nadam_steps():
    assert covers_every_pair(GRID)
    mg = _make_golden()
    fns = mg._step_functions("nadam.py", "Nadam", ["step"])
    out = {}
    rng = np.random.default_rng(20261020)
    meta = []
    lr = 0.001
    for ci, values in enumerate(GRID + EXTRA):
        kw = dict(epsilon=1e-8, **dict(zip(NAMES, values)))
        wd = kw.pop("wd")
        opt = mg._FakeOptimizer(fns, lr, wd, m_schedule=1., **kw)
        ws = [mg._nd(rng.uniform(0, 1, s)) for s in SHAPES]
        states = [tuple(mg._nd(np.zeros(s)) for _ in range(2)) for s in SHAPES]
        active = np.ones((STEPS, len(SHAPES)), np.int8)
        for k, w in enumerate(ws):
            out["w0_c%d_k%d" % (ci, k)] = np.asarray(w).copy()
        msched = []
        for t in range(STEPS):
            for k, (shape, w, st) in enumerate(zip(SHAPES, ws, states)):
                if (t, k) in SKIP.get(ci, ()):
                    active[t, k] = 0
                    continue
                g = rng.uniform(-1, 1, shape).astype(np.float32)
                out["g%d_c%d_k%d" % (t, ci, k)] = g
                # step scales the gradient in place (grad *= self.rescale_grad): a fresh array every time
                opt.step([k], [w], [mg._nd(g.copy())], [st])
            for k, (w, st) in enumerate(zip(ws, states)):
                out["w%d_c%d_k%d" % (t + 1, ci, k)] = np.asarray(w).copy()
                for i, s in enumerate(st):
                    out["s%d_%d_c%d_k%d" % (i, t + 1, ci, k)] = np.asarray(s).copy()
            msched.append(opt.m_schedule)
        out["msched_c%d" % ci] = np.array(msched, np.float64)
        out["active_c%d" % ci] = active
        meta.append(repr(("nadam", lr, wd, kw)))
    out["cases"] = np.array(meta)
    out["steps"] = np.array([STEPS])
    np.savez_compressed(os.path.join(HERE, "nadam_steps.npz"), **out)


if __name__ == "__main__":
    nadam_steps()
    print("wrote", os.path.join(HERE, "nadam_steps.npz"))
