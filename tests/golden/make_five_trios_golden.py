"""Generates tests/golden/five_trios.npz: five-trio problems (T = 1024) and the outputs of the UNMODIFIED reference C++
PedigreeDPTable (oracle/_ref/libwhref.so) on them.  Run where the reference is built:  python tests/golden/make_five_trios_golden.py

At most 7 reads are active per column (the reference takes about 1.4e8 steps per such column).  Shapes:
  nuclear5   father, mother and five children (P = 4)
  three_gen  two grandparent couples, their two children, and five grandchildren of those (P = 8)
Cases: trusted and distrusted genotypes, tie-heavy weights (phred 0-2, recombination costs 0-2), gaps, one chain or several, and
distrusted genotype likelihoods so large that 32-bit sums of a path can wrap (the device then skips the transition transform).
"""
import os
import sys
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from whatshap_b200 import synth  # noqa: E402

SHAPES = {
    "nuclear5": (7, [0, 1, 2, 0, 1, 3, 0, 1, 4, 0, 1, 5, 0, 1, 6]),
    "three_gen": (9, [0, 1, 2, 3, 4, 5, 2, 5, 6, 2, 5, 7, 2, 5, 8]),
}


def five_trio_problem(seed, shape, n_cols, max_cov=6, distrust=False, rc_max=3, max_phred=2, gap=0.15, burst=3, huge_gl=False):
    """synth.random_problem on a five-trio shape, recombination costs in [0, rc_max)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    with mock.patch.dict(synth.PEDIGREES, {shape: SHAPES[shape]}):
        prob = synth.random_problem(rng, n_cols, max_cov, shape, distrust=distrust, max_phred=max_phred, gap=gap, burst=burst)
    prob.recombcost = rng.integers(0, rc_max, n_cols).astype(np.uint32)
    if huge_gl:  # a path's cost exceeds 2^32 - 1 in total while every single cost fits (the reference's unsigned sums wrap)
        prob.gl = (rng.integers(0, 3, prob.gl.shape) * 1.5e8 + rng.integers(0, 4, prob.gl.shape)).astype(np.float64)
    return prob


def cases():
    out = []
    for i, (shape, distrust, rc_max, burst, gap) in enumerate([
        ("nuclear5", False, 3, 3, 0.15),
        ("nuclear5", False, 1, 3, 0.0),    # rc = 0 everywhere: every j ties
        ("nuclear5", True, 3, 2, 0.15),
        ("nuclear5", False, 3, 2, 0.3),    # sparse: several chains
        ("three_gen", False, 3, 3, 0.15),
        ("three_gen", True, 2, 3, 0.0),
        ("three_gen", False, 3, 4, 0.15),  # dense: one chain
    ]):
        out.append((f"{shape}/distrust={distrust}/rc<{rc_max}/burst={burst}", five_trio_problem(100 + i, shape, 24, distrust=distrust,
                                                                                               rc_max=rc_max, burst=burst, gap=gap)))
    out.append(("nuclear5/wrapping GLs", five_trio_problem(200, "nuclear5", 20, distrust=True, huge_gl=True)))
    return out


if __name__ == "__main__":
    from make_golden import pack

    np.savez_compressed(os.path.join(HERE, "five_trios.npz"), **pack(cases()))
