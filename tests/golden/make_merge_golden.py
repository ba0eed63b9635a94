"""Regenerates tests/golden/merge.npz: the reference's own ReadMerger (whatshap/merge.py, with whatshap.core compiled by
oracle/build_pyref.build() and networkx) on the seeded cases of tests/merge_cases.py, each checked against the plain-Python
oracle oracle/merge_oracle.py before it is stored.  Needs the WhatsHap source tree at $WHATSHAP_REF.

    python tests/golden/make_merge_golden.py

The two fixtures of the reference's tests/test_merge_reads.py are built with its string_to_readset and stored as data."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import merge_cases as mc  # noqa: E402

UNIT_ALLELES = """
      0 000000
      111
      11 00111101
      0 00000
    """
UNIT_WEIGHTS = """
      1 523428
      714
      86 03158958
      8 46626
    """


def main():
    from oracle import build_pyref

    path = build_pyref.build()
    if not path:
        sys.exit("the WhatsHap source tree is needed at $WHATSHAP_REF")
    sys.path.insert(0, path)
    import networkx
    import whatshap.core as core
    import whatshap.merge as ref_merge
    from whatshap.testhelpers import string_to_readset

    unit = [[[v.position, v.allele, v.quality] for v in r] for r in string_to_readset(UNIT_ALLELES, UNIT_WEIGHTS)]
    cases = mc.build_cases(unit)
    for case in cases:
        case["want"] = mc.run(ref_merge.ReadMerger, case, core.Read, core.ReadSet)
        got = mc.run_oracle(case)
        assert got == case["want"], case["name"]
    blob = json.dumps(dict(cases=cases, networkx=networkx.__version__)).encode()
    np.savez_compressed(os.path.join(HERE, "merge.npz"), cases=np.frombuffer(blob, np.uint8))
    merged = sum(1 for c in cases if not isinstance(c["want"], str) and len(c["want"]) < len(c["reads"]))
    print(f"{len(cases)} cases, {merged} with merged reads, networkx {networkx.__version__}")


if __name__ == "__main__":
    main()
