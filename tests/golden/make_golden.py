"""Generates tests/golden/*.npz: inputs (flat problems) and the outputs of the UNMODIFIED
reference C++ PedigreeDPTable (oracle/_ref/libwhref.so, compiled in place from $WHATSHAP_REF by
oracle/Makefile) on them.  Run in the machine with the reference:  python tests/golden/make_golden.py

Groups
  reference_cases   the read matrices / pedigrees of the reference's own tests
                    (tests/test_phasing.py, tests/test_pedigreephasing.py, tests/test.matrix)
  fuzz              seeded irregular instances over six pedigree shapes, trusted and distrusted
                    genotypes, Mendelian conflicts included (the error text is stored)
  synthetic         small instances of the BASELINE.json generators (sliding window, trio)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import checker  # noqa: E402
from whatshap_b200 import synth  # noqa: E402
from whatshap_b200._abi import FlatProblem  # noqa: E402

PROBLEM_FIELDS = ("positions", "read_off", "ent_col", "ent_allele", "ent_phred", "read_ind", "recombcost", "trios", "gt", "gl")
SOLUTION_FIELDS = ("path_index", "path_tv", "partition", "sr_allele", "sr_quality")


def pack(cases):
    ref = checker.reference()
    assert ref is not None, "the compiled reference (oracle/_ref) is required to make golden vectors"
    out = {"n": np.array(len(cases))}
    for i, (label, prob) in enumerate(cases):
        out[f"{i}.label"] = np.array(label)
        out[f"{i}.n_ind"] = np.array(prob.n_ind)
        out[f"{i}.distrust"] = np.array(int(prob.distrust))
        for f in PROBLEM_FIELDS:
            v = getattr(prob, f)
            if v is not None:
                out[f"{i}.{f}"] = v
        try:
            sol = ref.solve(prob)
            out[f"{i}.error"] = np.array("")
            out[f"{i}.cost"] = np.array(sol.cost, np.uint32)
            for f in SOLUTION_FIELDS:
                out[f"{i}.{f}"] = getattr(sol, f)
        except RuntimeError as e:
            out[f"{i}.error"] = np.array(str(e))
    return out


def reference_cases():
    import test_pedigreephasing as tp
    import test_phasing as ts
    import test_verification as tv
    from whatshap_b200 import ReadSet
    from whatshap_b200.core import _flatten
    from whatshap_b200.testhelpers import matrix_to_readset, string_to_readset, string_to_readset_pedigree

    cases = []
    for name in sorted(ts.MATRICES):
        reads, weights = ts.MATRICES[name]
        rs = string_to_readset(reads, weights)
        positions = rs.get_positions()
        for het in (True, False):
            for trio in (False, True):
                ped = ts.build_pedigree_for(positions, het, trio)
                cases.append((f"phasing/{name}/het={het}/trio={trio}", _flatten(rs, [1] * len(positions), ped, not het, None)))
    for name, rs in (("test.matrix", matrix_to_readset(tv.TEST_MATRIX)), ("string", string_to_readset(tv.STRING_MATRIX))):
        positions = rs.get_positions()
        for het in (True, False):
            ped = ts.build_pedigree_for(positions, het, False)
            cases.append((f"verification/{name}/het={het}", _flatten(rs, [1] * len(positions), ped, not het, None)))
    for name in sorted(tp.CASES):
        case = tp.CASES[name]
        ped = tp.build_pedigree(case)
        rs = string_to_readset_pedigree(case["reads"]) if case["reads"].strip() else ReadSet()
        cases.append((f"pedigree/{name}", _flatten(rs, case["recomb"], ped, case.get("distrust", False), case.get("positions"))))
    return cases


def fuzz_cases():
    rng = np.random.default_rng(20250923)
    peds = list(synth.PEDIGREES)
    cases = []
    for it in range(180):
        ped = peds[it % len(peds)]
        maxcov = 6 if ped in ("quartet", "three_generations") else 9
        prob = synth.random_problem(rng, int(rng.integers(1, 16)), int(rng.integers(1, maxcov)), ped,
                                    distrust=bool(rng.integers(0, 2)), conflict_free=bool(rng.integers(0, 4)),
                                    max_phred=int(rng.integers(1, 8)), mean_len=float(rng.choice([2, 4, 8])))
        cases.append((f"fuzz/{it}/{ped}", prob))
    return cases


def synthetic_cases():
    return [
        ("sliding/n=120/c=10", synth.sliding_window(120, 10, block_len=50, seed=3)),
        ("sliding/n=90/c=8/stride=2/gap", synth.sliding_window(90, 8, stride=2, block_len=45, seed=4, gap=0.1)),
        ("sliding/n=64/c=12", synth.sliding_window(64, 12, block_len=32, seed=12)),
        ("sliding/n=40/c=16", synth.sliding_window(40, 16, block_len=20, seed=16)),
        ("sliding/n=36/c=17", synth.sliding_window(36, 17, block_len=36, seed=17)),
        ("trio/n=60/c=3", synth.trio(60, 3, block_len=30, seed=5)),
        ("trio/n=40/c=4", synth.trio(40, 4, block_len=40, seed=6)),
    ]


if __name__ == "__main__":
    for group, fn in (("reference_cases", reference_cases), ("fuzz", fuzz_cases), ("synthetic", synthetic_cases)):
        data = pack(fn())
        path = os.path.join(HERE, group + ".npz")
        np.savez_compressed(path, **data)
        print(group, int(data["n"]), "cases ->", path, os.path.getsize(path), "bytes")
