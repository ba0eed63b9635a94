"""Allele detection from the CIGAR alone (whmec_detect_alleles_cigar, DESIGN §4.14) on the CPU: the host preparation and chunk plan
of cigar_alleles_plan.cpp with the per-thread code of cigar_alleles.h run by the host emulation tests/emul/emul_cigar_alleles.cpp,
against the reference's answers stored in tests/golden/cigar_alleles.npz and, where oracle/_ref/pyref holds it, the reference's
compiled whatshap._variants live."""
import ctypes as C
import json
import os
import random
import subprocess

import numpy as np
import pytest

from test_realign import reference_variants
from whatshap_b200 import _lib, realign
from whatshap_b200._abi import CQueryQualities

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
_emul = None


def emul():
    global _emul
    if _emul is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "cigar_alleles.mk"], check=True, capture_output=True)
        _emul = _lib.cigar_alleles_signatures(C.CDLL(os.path.join(EMUL_DIR, "libwhemul_cigar_alleles.so")))
    return _emul


class Aln:
    def __init__(self, start, cigar, seq, quals=None):
        self.reference_start = start
        self.cigartuples = None if cigar is None else [tuple(x) for x in cigar]
        self.query_sequence, self.query_qualities = seq, quals


class Var:
    def __init__(self, position, ref, alts):
        self.position, self.reference_allele, self.alts = position, ref, list(alts)

    def get_alt_allele_list(self):
        return self.alts


def golden_cases():
    with np.load(os.path.join(ROOT, "tests", "golden", "cigar_alleles.npz")) as z:
        return json.loads(z["cases"].tobytes())


def check_case(c, run, **extra):
    """The alignments the reference answers give its calls, in order; the whole list raises ValueError naming the first alignment
    the reference raises on and its exception; a preparation the reference fails fails the call."""
    variants = [Var(*v) for v in c["variants"]]
    if c.get("raises"):
        with pytest.raises(ValueError, match=rf"^variant \d+ .*{c['raises']}"):
            run([Aln(*a) for a in c["alignments"]], variants, None, **extra)
        return
    ok = [k for k, w in enumerate(c["want"]) if not isinstance(w, str)]
    got = run([Aln(*c["alignments"][k]) for k in ok], variants, None, **extra)
    assert [[list(t) for t in g] for g in got] == [c["want"][k] for k in ok], c["name"]
    bad = [k for k, w in enumerate(c["want"]) if isinstance(w, str)]
    if bad:
        with pytest.raises(ValueError, match=rf"^alignment {bad[0]}: the reference raises {c['want'][bad[0]]}\b"):
            run([Aln(*a) for a in c["alignments"]], variants, None, **extra)


def reference_python():
    """The reference's compiled whatshap._variants with its variants.py and vcf.py importable (the tree oracle/build_pyref.build()
    makes, pysam and friends stubbed), or None."""
    import sys

    from oracle import build_pyref

    if not os.path.isfile(os.path.join(build_pyref.OUT, "whatshap", "variants.py")) or reference_variants() is None:
        return None
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_realign_golden import _StubFinder

    if not any(isinstance(f, _StubFinder) for f in sys.meta_path):
        sys.meta_path.insert(0, _StubFinder())
    import importlib

    import whatshap  # the shipped binding's package: let it find variants.py and vcf.py in the built tree too

    if os.path.join(build_pyref.OUT, "whatshap") not in whatshap.__path__:
        whatshap.__path__.append(os.path.join(build_pyref.OUT, "whatshap"))
    try:
        importlib.import_module("whatshap.variants")
    except ImportError:
        return None
    return reference_variants()


def emul_detect(*a, **k):
    return realign.detect_alleles(*a, library=emul(), **k)


def test_golden_cases_cover_the_issue():
    cases = golden_cases()
    ops = {op for c in cases for a in c["alignments"] if a[1] for op, _ in a[1]}
    assert set(range(10)) <= ops
    alns = [a for c in cases for a in c["alignments"]]
    assert any(a[3] is None for a in alns) and any(a[3] == [] for a in alns) and any(a[3] for a in alns)
    assert any(a[1] == [] for a in alns) and any(a[1] is None for a in alns) and any(a[2] is None for a in alns)
    assert max(len(a[2] or "") for a in alns) >= 15000
    assert max(len(alt) for c in cases for v in c["variants"] for alt in v[2]) > 1100
    kinds = {w for c in cases if c["want"] for w in c["want"] if isinstance(w, str)}
    assert {"ValueError", "IndexError", "TypeError"} <= kinds
    assert any(c.get("raises") for c in cases) and any(c["running"] for c in cases)


@pytest.mark.parametrize("index", range(len(golden_cases())))
def test_golden_case_emulated(index):
    check_case(golden_cases()[index], emul_detect)


def test_running_index_equals_first_zero():
    """For alignments sorted by reference_start, _alignments_to_reads (with its running index) made the reads that first = 0 gives."""
    for c in golden_cases():
        if not c["running"]:
            continue
        variants = [Var(*v) for v in c["variants"]]
        got = emul_detect([Aln(*a) for a in c["alignments"]], variants, None)
        assert [[[variants[j].position, a, q] for j, a, q in g] for g in got] == c["reads"], c["name"]


def test_live_reference_on_random_alignments():
    """Seeded random alignments with many unsorted, overlapping and duplicate variants, against the compiled _detect_alleles."""
    rv = reference_python()
    if rv is None:
        pytest.skip("the reference's Python package (oracle/build_pyref.build()) is not built here")
    from whatshap.variants import ReadSetReader
    from whatshap.vcf import BiallelicVcfVariant, MultiallelicVcfVariant

    rng = random.Random(3)
    for _ in range(20):
        ref = "".join(rng.choice("ACGT") for _ in range(300))
        raw = []
        for _ in range(rng.randrange(5, 60)):
            p = rng.randrange(0, 290)
            r = ref[p:p + rng.choice([1, 1, 2, 4])]
            alts = [rng.choice(["", ref[p]]) + "".join(rng.choice("ACGT") for _ in range(rng.randrange(0, 4))) for _ in range(rng.choice([1, 1, 2]))]
            alts = [a if a != "" else ref[p] for a in alts]
            raw.append((p, r, alts))
        if rng.random() < 0.7:
            raw.sort(key=lambda v: v[0])
        variants = [BiallelicVcfVariant(p, r, a[0]) if len(a) == 1 else MultiallelicVcfVariant(p, r, a) for p, r, a in raw]
        normalized = [v.normalized() for v in variants]
        valid = ReadSetReader.detect_non_overlapping_variants(None, normalized)
        alns = []
        for _ in range(30):
            start = rng.randrange(0, 250)
            cigar, q = [], 0
            for _ in range(rng.randrange(1, 12)):
                op = rng.choice([0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8])
                n = rng.randrange(0, 12)
                cigar.append((op, n))
                q += n if op in (0, 1, 4, 7, 8) else 0
            seq = "".join(rng.choice("ACGT") for _ in range(max(0, q + rng.choice([0, 0, 0, -2, 3]))))
            quals = rng.choice([None, [], [rng.randrange(0, 50) for _ in seq]])
            alns.append(Aln(start, cigar, seq, quals))
        want = []
        for a in alns:
            vp = [ReadSetReader.build_var_progress(None, normalized, j) for j in valid]
            try:
                want.append([tuple(int(x) for x in t) for t in rv._detect_alleles(normalized, vp, 0, a)])
            except IndexError:
                want.append("IndexError")
        ok = [k for k, w in enumerate(want) if not isinstance(w, str)]
        mine = [Var(*v) for v in raw]
        assert emul_detect([alns[k] for k in ok], mine, None) == [want[k] for k in ok]
        bad = [k for k, w in enumerate(want) if isinstance(w, str)]
        if bad:
            with pytest.raises(ValueError, match=rf"^alignment {bad[0]}: the reference raises IndexError"):
                emul_detect(alns, mine, None)


def test_chunking_down_to_one_item(monkeypatch):
    """Every budget gives the same calls; the smallest runs one item per window, a middling one cuts several chunks."""
    for c in golden_cases():
        if c["name"] not in ("random1", "random5", "rules"):
            continue
        ok = [Aln(*a) for a, w in zip(c["alignments"], c["want"]) if not isinstance(w, str)]
        variants = [Var(*v) for v in c["variants"]]
        st = {}
        whole = emul_detect(ok, variants, None, stats=st)
        assert st["chunks"] == 1 and st["items"] > 0 and st["jobs"] >= st["items"] and st["cells"] == sum(map(len, whole))
        for budget, one in (("1", True), ("200000", False), ("400000", False)):
            monkeypatch.setenv("WHMEC_REALIGN_ARENA_BUDGET", budget)
            st_b = {}
            assert emul_detect(ok, variants, None, stats=st_b) == whole
            assert st_b["items"] == st["items"] and st_b["jobs"] == st["jobs"]
            assert st_b["chunks"] == st["items"] if one else st_b["chunks"] >= 1
        monkeypatch.delenv("WHMEC_REALIGN_ARENA_BUDGET")


def test_options_are_ignored_and_errors():
    v = [Var(5, "A", ["C"])]
    a = [Aln(0, [(0, 10)], "AAAAACAAAA", [20] * 10)]
    assert emul_detect(a, v, None) == [[(0, 1, 20)]]
    assert emul_detect(a, v, None, overhang=3, affine=True, use_kmerald=True, restricted_genotypes=[None]) == [[(0, 1, 20)]]
    assert emul_detect(a, v, None, stats=(st := {})) == [[(0, 1, 20)]] and st["items"] == 1 and st["cells"] == 1
    with pytest.raises(ValueError, match=r"^alignment 0: positions"):
        emul_detect([Aln(2**31 - 5, [(0, 10)], "A" * 10)], v, None)
    with pytest.raises(ValueError, match=r"^variant 0 has no alternative allele"):
        emul_detect(a, [Var(5, "A", [])], None)
    with pytest.raises(ValueError, match=r"^alignment 1: the reference raises TypeError"):
        emul_detect([a[0], Aln(0, None, "A")], v, None)
    assert emul_detect([], v, None) == [] and emul_detect(a, [], None) == [[]]


def test_struct_layout_matches_the_c_compiler(tmp_path):
    name, cls = "whmec_query_qualities", CQueryQualities
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "whmec.h")}"', "int main(void) {",
             f'printf("{name} %zu\\n", sizeof({name}));']
    lines += [f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));' for f, _ in cls._fields_]
    lines.append("return 0; }")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    subprocess.run(["cc", "-o", str(tmp_path / "layout"), str(src)], check=True)
    out = subprocess.run([str(tmp_path / "layout")], check=True, capture_output=True, text=True).stdout.split("\n")
    got = dict(line.split() for line in out if line)
    assert int(got[name]) == C.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f"{name}.{f}"]) == getattr(cls, f).offset, f
