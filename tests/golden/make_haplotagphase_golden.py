"""Regenerates tests/golden/haplotagphase.npz: the reference's own run_haplotagphase (whatshap/cli/haplotagphase.py, with pysam,
pyfaidx and xopen stubbed as make_haplotag_golden.py stubs them, and whatshap.core compiled by oracle/build_pyref.build()) on
the seeded cases of tests/haplotagphase_cases.py, with stand-ins for VcfReader, PhasedInputReader, PhasedVcfWriter and
IndexedFasta assigned into the module.  The writer's stand-in captures write(chromosome, sample_to_super_reads,
sample_to_components), and compute_votes is wrapped to capture the votes.  Needs the WhatsHap source tree at $WHATSHAP_REF.

    python tests/golden/make_haplotagphase_golden.py

Each case stores its inputs and the reference's result (per sample its votes, super-reads and components) or the name of the
exception it raised.  The reference's test_compute_votes and the best_candidate doctests are restated as cases of their own."""
import json
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import haplotagphase_cases as hc  # noqa: E402
from make_haplotag_golden import _StubFinder  # noqa: E402


def reference_module():
    """The reference's whatshap.cli.haplotagphase, imported with the stubs (None without the source tree)."""
    from oracle import build_pyref

    path = build_pyref.build()
    if not path:
        return None
    sys.meta_path.insert(0, _StubFinder())
    sys.path.insert(0, path)
    import whatshap.cli.haplotagphase as h

    return h


def build_cases():
    rng = random.Random(20261018)
    cases = [hc.tie_case(), hc.boundary_case(29), hc.boundary_case(28)]
    for _ in range(60):
        cases.append(hc.make_case(rng))
    for n in (2, 3):
        for _ in range(4):
            cases.append(hc.make_case(rng, n_samples=n, included=["S1"] if n == 3 else None))
    for cut in (-1, 0, 1, 2, 10):
        for _ in range(2):
            cases.append(hc.make_case(rng, cut_poly=cut))
    for _ in range(4):
        cases.append(hc.make_case(rng, only_indels=True))
    for error in ("position", "allele", "haplotype", "zero"):
        for _ in range(3):
            cases.append(hc.make_case(rng, error=error))
    for _ in range(3):
        cases.append(hc.make_case(rng, big=True, n_samples=2))
    return cases


# The reference's test_compute_votes (tests/test_run_haplotagphase.py): reads (HP_tag, PS_tag, entries) and the expected votes,
# keys in insertion order.
COMPUTE_VOTES = {
    "homozygous": [[1, False], [2, False], [3, True]],
    "reads": [[1, 1, [[1, 0, 30], [2, 0, 10], [3, 0, 50]]], [2, 1, [[1, 1, 20], [2, 0, 30], [3, 0, 90]]], [1, 2, [[1, 1, 20], [3, 0, 10]]]],
    "allele_to_id": [[1, [[0, 0], [1, 1]]], [2, [[0, 0], [1, 1]]], [3, [[0, 0], [1, 1]]]],
    "want": [[1, [[0, 0, 50], [0, 1, 0], [1, 0, 0], [1, 1, 20]]], [2, [[0, 0, 10], [0, 1, 30]]]],
}
# The best_candidate doctests: (vote as [[ps, h, score]], (h, ps, q, score)).
BEST_CANDIDATE = [
    ([[1, 2, 50], [2, 3, 100], [3, 4, 75]], [3, 2, 0.4444444444444444, 100]),
    ([[1, 1, 10], [2, 2, 20], [3, 3, 30], [4, 4, 40]], [4, 4, 0.4, 40]),
    ([[0, 0, 2]], [0, 0, 1.0, 2]),
    ([[1, 2, 100], [2, 2, 100], [3, 3, 100]], [2, 1, 0.3333333333333333, 100]),
    ([[5, 5, 200], [6, 6, 300], [7, 7, 500]], [7, 7, 0.5, 500]),
]


if __name__ == "__main__":
    h = reference_module()
    import whatshap.core as core

    cases = build_cases()
    for c in cases:
        c["want"] = hc.run_module(h, c, core)
        assert hc.run_oracle(c) == c["want"], "the oracle disagrees with the reference"
    # the restated unit tests, checked against the reference's functions
    reads = hc.readset(core, COMPUTE_VOTES["reads"])
    got = h.compute_votes(dict(COMPUTE_VOTES["homozygous"]), reads, {p: dict(m) for p, m in COMPUTE_VOTES["allele_to_id"]})
    assert hc.plain_votes(got) == COMPUTE_VOTES["want"]
    for vote, want in BEST_CANDIDATE:
        assert list(h.best_candidate({(ps, hh): s for ps, hh, s in vote})) == want
    unit = {"compute_votes": COMPUTE_VOTES, "best_candidate": BEST_CANDIDATE}
    np.savez_compressed(os.path.join(HERE, "haplotagphase.npz"), cases=np.frombuffer(json.dumps(cases).encode(), np.uint8),
                        unit=np.frombuffer(json.dumps(unit).encode(), np.uint8))
    errors = sorted(c["want"] for c in cases if isinstance(c["want"], str))
    print(f"{len(cases)} cases, {sum(len(v) for c in cases for v in c['reads'].values())} reads, errors {errors}")
