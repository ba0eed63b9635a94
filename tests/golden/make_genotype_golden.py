"""Generates tests/golden/genotype.npz: flat problems and the genotype likelihoods the UNMODIFIED reference
GenotypeDPTable (oracle/_ref/libwhref.so: whref_genotype, compiled in place from $WHATSHAP_REF by oracle/Makefile)
computes for them, rounded from long double to double.  Run in the machine with the reference:
    python tests/golden/make_genotype_golden.py

Cases
  kat.*    the read matrices of the reference's own known-answer tests (tests/test_genotyping.py:113-190 of the
           reference: uniform and non-uniform priors, phred 10), built through this package's containers; the
           likelihoods the reference's test file states are stored beside the ones the compiled reference returns
  prior.*  24 seeded single-sample read sets with the per-column priors of the reference's compute_genotypes
           (src/genotyper.cpp:12-54; whref_compute_genotypes), doubles stored exactly
  fuzz.*   seeded irregular instances over six pedigree shapes (gaps, blanks, phred 0..60, uniform / random / sparse
           priors, recombination costs 0..30)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import checker  # noqa: E402
from whatshap_b200 import NumericSampleIds, Pedigree, PhredGenotypeLikelihoods, synth  # noqa: E402
from whatshap_b200.core import _flatten  # noqa: E402
from whatshap_b200.testhelpers import canonic_index_to_biallelic_gt, string_to_readset  # noqa: E402

FIELDS = ("positions", "read_off", "ent_col", "ent_allele", "ent_phred", "read_ind", "recombcost", "trios", "gl")

# (reads, weights, priors or None, likelihoods stated by the reference's tests)
KATS = {
    "exact1": ("  11\n   01", None, None,
               [[0.06666666666666667, 0.3333333333333333, 0.6], [0.20930232558139536, 0.5813953488372093, 0.20930232558139536],
                [0.06666666666666667, 0.3333333333333333, 0.6]]),
    "exact2": ("11\n11", "11\n11", None,
               [[0.00914139256727894, 0.25040580948312685, 0.7404527979495942]] * 2),
    "exact3": ("01\n11", None, None,
               [[0.22163406214039125, 0.5567318757192175, 0.22163406214039125], [0.009896432681242807, 0.18849252013808976, 0.8016110471806674]]),
    "priors1": ("01\n11", None, [[0.1, 0.8, 0.1], [0.1, 0.2, 0.7]],
                [[0.04257892641700095, 0.9148421471659981, 0.04257892641700095], [0.0016688611936185199, 0.05208684202468078, 0.9462442967817007]]),
    "priors2": (" 11\n  01", None, [[0, 0.5, 0.5], [0.25, 0.5, 0.25], [0.1, 0.4, 0.5]],
                [[0.0, 0.35714285714285715, 0.6428571428571429], [0.1323529411764706, 0.7352941176470589, 0.1323529411764706],
                 [0.015151515151515152, 0.30303030303030304, 0.6818181818181818]]),
}


def kat_problem(reads, weights, priors):
    rs = string_to_readset(s=reads, w=weights, scale_quality=10)
    positions = rs.get_positions()
    ids = NumericSampleIds()
    ped = Pedigree(ids)
    gls = [PhredGenotypeLikelihoods(p) for p in priors] if priors else [PhredGenotypeLikelihoods([1 / 3.0] * 3)] * len(positions)
    ped.add_individual("individual0", [canonic_index_to_biallelic_gt(1)] * len(positions), gls)
    return _flatten(rs, [1] * len(positions), ped, True, None)


def main():
    ref = checker.reference()
    assert ref is not None, "the compiled reference (oracle/_ref) is required"
    cases = []
    for name, (reads, weights, priors, stated) in KATS.items():
        cases.append(("kat." + name, kat_problem(reads, weights, priors), np.array(stated)))
    rng = np.random.default_rng(20260923)
    peds = ("single", "two_unrelated", "trio", "trio_child_first", "quartet", "three_generations")
    for i in range(60):
        ped = peds[i % len(peds)]
        cov = int(rng.integers(2, 9 if ped == "single" else (6 if ped == "two_unrelated" else 5)))
        prob = synth.genotyping_problem(rng, int(rng.integers(2, 40)), cov, ped, prior=("uniform", "random", "sparse")[i % 3],
                                        max_phred=int(rng.choice([5, 40, 60])), gap=float(rng.random() * 0.3))
        cases.append((f"fuzz.{i}.{ped}", prob, None))
    out = {"n": np.array(len(cases))}
    for i, (label, prob, stated) in enumerate(cases):
        out[f"{i}.label"] = np.array(label)
        out[f"{i}.n_ind"] = np.array(prob.n_ind)
        for f in FIELDS:
            out[f"{i}.{f}"] = getattr(prob, f)
        out[f"{i}.likelihoods"] = ref.genotype(prob)
        if stated is not None:
            out[f"{i}.stated"] = stated
            assert np.allclose(out[f"{i}.likelihoods"][0], stated, rtol=0, atol=1e-9), label
    # compute_genotypes (src/genotyper.cpp:12-54): per-column priors of one sample's reads, bit-exact doubles
    import ctypes as C

    from whatshap_b200._abi import CProblem

    lib = ref.lib
    lib.whref_compute_genotypes.argtypes = [C.POINTER(CProblem), C.POINTER(C.c_double), C.POINTER(C.c_int8), C.c_char_p, C.c_size_t]
    n_prior = 24
    out["n_prior"] = np.array(n_prior)
    for i in range(n_prior):
        prob = synth.random_problem(rng, int(rng.integers(1, 80)), int(rng.integers(1, 25)), "single", max_phred=int(rng.choice([3, 20, 60])), gap=0.2)
        gl, gt = np.zeros((prob.n_cols, 3)), np.zeros(prob.n_cols, np.int8)
        cp, err = prob.as_c(), C.create_string_buffer(256)
        rc = lib.whref_compute_genotypes(C.byref(cp), gl.ctypes.data_as(C.POINTER(C.c_double)), gt.ctypes.data_as(C.POINTER(C.c_int8)), err, 256)
        assert rc == 0, err.value
        for f in ("positions", "read_off", "ent_col", "ent_allele", "ent_phred", "read_ind", "recombcost"):
            out[f"prior.{i}.{f}"] = getattr(prob, f)
        out[f"prior.{i}.gl"] = gl
        out[f"prior.{i}.gt"] = gt
    np.savez_compressed(os.path.join(HERE, "genotype.npz"), **out)
    print("wrote", len(cases), "cases")


if __name__ == "__main__":
    main()
