"""Regenerates tests/golden/adadelta_steps.npz.  Needs the reference source tree (make_golden.REF).

adadelta_steps.npz -- weights and states produced by the reference's own ``AdaDelta.step``
(python/mxnet/optimizer/adadelta.py:72-111), executed from the reference file on the float32 numpy stand-in for NDArray
of make_golden.py by the machinery of make_adamax_golden.py.  Options: rho 0.9 / 0.95 (so that the double-rounded
complement 1 - rho is exercised at two values), epsilon 1e-6 / 1e-8, clip_gradient none / 0.4, rescale_grad 1 / 0.14,
wd 0 / 0.03, in the 8-run two-level array in which every pair of values of two options meets, plus one set with
clip_gradient 0, x 4 shapes ((3, 4, 5), (10, 4), (7,), (1001,)) x 6 steps at learning rate 1.0 (the class default).
It pins tests/adadelta_oracle.py bit for bit (tests/test_adadelta.py).
"""
import importlib.util
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def _machinery():
    spec = importlib.util.spec_from_file_location("make_adamax_golden", os.path.join(HERE, "make_adamax_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


M = _machinery()
covers_every_pair = M.covers_every_pair
LEVELS = [(0.9, 0.95), (1e-6, 1e-8), (None, 0.4), (1.0, 0.14), (0.0, 0.03)]
NAMES = ("rho", "epsilon", "clip_gradient", "rescale_grad", "wd")
GRID = M.orthogonal_grid(LEVELS)
EXTRA = [(LEVELS[0][0], LEVELS[1][0], 0.0, LEVELS[3][1], LEVELS[4][1])]


def adadelta_steps():
    assert M.covers_every_pair(GRID)
    M.run_steps("adadelta.py", "AdaDelta", NAMES, GRID + EXTRA, 1.0, {}, 20261020, "adadelta_steps.npz", "adadelta")


if __name__ == "__main__":
    adadelta_steps()
    print("wrote", os.path.join(HERE, "adadelta_steps.npz"))
