"""Regenerates tests/golden/haplotag.npz: the reference's own prepare_haplotag_information (whatshap/cli/haplotag.py, with
pysam, pyfaidx and xopen stubbed and whatshap.core compiled by oracle/build_pyref.build()) on the seeded cases of
tests/haplotag_cases.py, read through a stand-in variant table and a reader that returns the reference's ReadSets.  Needs the
WhatsHap source tree at $WHATSHAP_REF.

    python tests/golden/make_haplotag_golden.py

Each case stores its inputs, the reference's four results in plain form (or the name of the exception it raised) and the
groups of several reads whose top phase sets tie ("loose": the reference may pick any of them, the oracle lists the choices)."""
import importlib.util
import json
import os
import random
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
STUBS = ("pysam", "pyfaidx", "xopen")

import haplotag_cases as hc  # noqa: E402


class _Any:
    def __init__(self, *a, **k):
        pass


class _StubFinder:
    def find_spec(self, name, path=None, target=None):
        if name.split(".")[0] in STUBS:
            return importlib.util.spec_from_loader(name, self, is_package=True)

    def create_module(self, spec):
        m = types.ModuleType(spec.name)
        m.__path__ = []
        m.__getattr__ = lambda n: _Any
        return m

    def exec_module(self, m):
        pass


def reference_module():
    """The reference's whatshap.cli.haplotag, imported with the stubs (None without the source tree)."""
    from oracle import build_pyref

    path = build_pyref.build()
    if not path:
        return None
    sys.meta_path.insert(0, _StubFinder())
    sys.path.insert(0, path)
    import whatshap.cli.haplotag as h

    return h


def build_cases():
    rng = random.Random(20261018)
    cases = []
    for ploidy in (2, 3, 4):
        for _ in range(30):
            cases.append(hc.make_case(rng, ploidy=ploidy))
    for _ in range(6):
        cases.append(hc.make_case(rng, n_samples=2))
    for error in ("assert", "key", "index", "choice"):
        for _ in range(3):
            cases.append(hc.make_case(rng, error=error))
    for _ in range(3):
        cases.append(hc.make_case(rng, big=True))
    return cases


if __name__ == "__main__":
    h = reference_module()
    import whatshap.core as core

    cases = build_cases()
    for c in cases:
        c["want"] = hc.run(h.prepare_haplotag_information, c, core)
        mine, loose = hc.run_oracle(c)
        c["loose"] = loose
        ok = mine == c["want"] if isinstance(mine, str) or isinstance(c["want"], str) else hc.same(c["want"], mine, loose)
        assert ok, "the oracle disagrees with the reference"
    np.savez_compressed(os.path.join(HERE, "haplotag.npz"), cases=np.frombuffer(json.dumps(cases).encode(), np.uint8))
    errors = [c["want"] for c in cases if isinstance(c["want"], str)]
    print(f"{len(cases)} cases, {sum(len(v) for c in cases for v in c['reads'].values())} reads, errors {sorted(errors)}, "
          f"{sum(len(c['loose']) for c in cases)} loose groups, "
          f"{sum(c['want']['multi'] for c in cases if not isinstance(c['want'], str))} groups with several phase sets")
