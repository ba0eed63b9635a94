"""Allele detection by re-alignment (whmec_realign, DESIGN §4.11) on the CPU: the host walk and chunk plan of realign_plan.cpp
with the per-job code of realign.h stepped by the host emulation tests/emul/emul_realign.cpp, against the reference's answers
stored in tests/golden/realign.npz and, where oracle/_ref/pyref holds them, the reference's compiled whatshap.align and
whatshap._variants live."""
import ctypes as C
import json
import os
import random
import re
import subprocess
import sys

import numpy as np
import pytest

from whatshap_b200 import _lib, realign
from whatshap_b200._abi import CRealignInput, CRealignOutput, CRealignStats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
PYREF = os.path.join(ROOT, "oracle", "_ref", "pyref")
_emul = None


def emul():
    global _emul
    if _emul is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "realign.mk"], check=True, capture_output=True)
        _emul = _lib.realign_signatures(C.CDLL(os.path.join(EMUL_DIR, "libwhemul_realign.so")))
    return _emul


def reference_align():
    """The reference's compiled whatshap.align, or None."""
    pkg = os.path.join(PYREF, "whatshap")
    if not (os.path.isdir(pkg) and any(f.startswith("align.") for f in os.listdir(pkg))):
        return None
    if PYREF not in sys.path:
        sys.path.insert(0, PYREF)
    import importlib

    return importlib.import_module("whatshap.align")


def reference_variants():
    if reference_align() is None:
        return None
    import importlib

    try:
        return importlib.import_module("whatshap._variants")
    except ImportError:
        return None


class Aln:
    def __init__(self, start, cigar, seq):
        self.reference_start, self.cigartuples, self.query_sequence = start, [tuple(x) for x in cigar], seq


class Var:
    def __init__(self, position, ref, alts):
        self.position, self.reference_allele, self.alts = position, ref, list(alts)

    def get_alt_allele_list(self):
        return self.alts


class Gt:
    def __init__(self, v):
        self.v = list(v)

    def as_vector(self):
        return self.v


def golden_cases():
    with np.load(os.path.join(ROOT, "tests", "golden", "realign.npz")) as z:
        return json.loads(str(z["cases"]))


def case_args(c, alignments=None):
    alns = [Aln(*a) for a in (c["alignments"] if alignments is None else alignments)]
    variants = [Var(*v) for v in c["variants"]]
    kw = dict(restricted_genotypes=[Gt(v) for v in c["restricted"]] if c["restricted"] else None, overhang=c["overhang"],
              affine=c["affine"], gap_start=c["gap_start"], gap_extend=c["gap_extend"], default_mismatch=c["default_mismatch"])
    return alns, variants, c["reference"], kw


def check_case(c, run, **extra):
    """Every golden case: the alignments the reference answers give its calls; the whole list raises ValueError naming the
    first alignment the reference raises on."""
    ok = [k for k, w in enumerate(c["want"]) if not isinstance(w, str)]
    alns, variants, reference, kw = case_args(c, [c["alignments"][k] for k in ok])
    got = run(alns, variants, reference, **kw, **extra)
    assert [[list(t) for t in g] for g in got] == [c["want"][k] for k in ok], c["name"]
    bad = [k for k, w in enumerate(c["want"]) if isinstance(w, str)]
    if bad:
        alns, variants, reference, kw = case_args(c)
        with pytest.raises(ValueError, match=rf"^alignment {bad[0]}\b"):
            run(alns, variants, reference, **kw, **extra)


def emul_detect(*a, **k):
    return realign.detect_alleles(*a, library=emul(), **k)


def test_golden_cases_cover_the_issue():
    cases = golden_cases()
    names = {c["name"] for c in cases}
    assert {"ends", "unsorted", "empty_restriction", "raising_overhang0"} <= names
    assert any(c["affine"] and isinstance(c["gap_start"], float) for c in cases)
    ops = {op for c in cases for a in c["alignments"] for op, _ in a[1]}
    assert {0, 1, 2, 3, 4, 5, 6, 7, 8, 9} <= ops
    assert any(isinstance(w, str) for c in cases for w in c["want"])
    assert max(len(v[2][0]) for c in cases for v in c["variants"]) > 1024


@pytest.mark.parametrize("index", range(len(golden_cases())))
def test_golden_case_emulated(index):
    check_case(golden_cases()[index], emul_detect)


def test_both_paths_and_chunking(monkeypatch):
    """The golden cases with long insertions use both the one-thread and the warp path; one item per chunk equals one chunk."""
    cases = [c for c in golden_cases() if c["name"] in ("random0", "random5", "random11", "random1")]
    for c in cases:
        ok = [c["alignments"][k] for k, w in enumerate(c["want"]) if not isinstance(w, str)]
        alns, variants, reference, kw = case_args(c, ok)
        st = {}
        whole = emul_detect(alns, variants, reference, stats=st, **kw)
        assert st["chunks"] == 1 and st["short_jobs"] > 0
        monkeypatch.setenv("WHMEC_REALIGN_ARENA_BUDGET", "1")
        st1 = {}
        assert emul_detect(alns, variants, reference, stats=st1, **kw) == whole
        assert st1["chunks"] == st1["items"] == st["items"]
        monkeypatch.delenv("WHMEC_REALIGN_ARENA_BUDGET")
    stats = []
    for c in cases:
        ok = [c["alignments"][k] for k, w in enumerate(c["want"]) if not isinstance(w, str)]
        alns, variants, reference, kw = case_args(c, ok)
        st = {}
        emul_detect(alns, variants, reference, stats=st, **kw)
        stats.append(st)
    assert sum(s["long_jobs"] for s in stats) > 0 and sum(s["long_items"] for s in stats) > 0


def test_chunk_budget_cuts():
    """Under a budget of a few items' bytes the chunks hold several items each, and all of them together every item."""
    c = golden_cases()[1]
    ok = [c["alignments"][k] for k, w in enumerate(c["want"]) if not isinstance(w, str)]
    alns, variants, reference, kw = case_args(c, ok)
    whole, st = None, {}
    for budget in (None, 200000, 40000, 8000):
        env = dict(os.environ)
        if budget:
            os.environ["WHMEC_REALIGN_ARENA_BUDGET"] = str(budget)
        try:
            s = {}
            got = emul_detect(alns, variants, reference, stats=s, **kw)
        finally:
            os.environ.clear()
            os.environ.update(env)
        whole = whole or got
        assert got == whole
        st[budget] = s["chunks"]
    assert st[None] == 1 and st[200000] <= st[40000] <= st[8000] and st[8000] > 1


# ---- the two distances -------------------------------------------------------------------------------------------------------

STRING_PAIRS = [("", ""), ("", "A"), ("A", "A"), ("AB", ""), ("AB", "ABC"), ("TGAATCCC", "CCTGAATC"), ("ANANAS", "BANANA"),
                ("SISSI", "MISSISSIPPI"), ("GGAATCCC", "TGAGGGATAAATATTTAGAATTTAGTAGTAGTGTT"), ("TCTGTTCCCTCCCTGTCTCA", "TTTTAGGAAATACGCC"),
                ("TGAGACACGCAACATGGGAAAGGCAAGGCACACAGGGGATAGG",
                 "AATTTATTTTATTGTGATTTTTTGGAGGTTTGGAAGCCACTAAGCTATACTGAGACACGCAACAGGGGAAAGGCAAGGCACA"),
                ("TCCATCTCATCCCTGCGTGTCCCATCTGTTCCCTCCCTGTCTCA", "TTTTAGGAAATACGCCTGGTGGGGTTTGGAGTATAGTGAAAGATAGGTGAGTTGGTCGGGTG"),
                ("A", "TCTGCTCCTGGCCCATGATCGTATAACTTTCAAATTT"), ("GCGCGGACT", "TAAATCCTGG")]
_r = random.Random(10)
STRING_PAIRS += [("".join(_r.choice("AC") for _ in range(_r.randint(0, 10))), "".join(_r.choice("AC") for _ in range(_r.randint(0, 10))))
                 for _ in range(1000)]


def ed(qs, ts, **k):
    return realign.edit_distances(qs, ts, library=emul(), **k)


def ed_aff(qs, ts, mm, gs, ge, **k):
    return realign.edit_distances_affine_gap(qs, ts, mm, gs, ge, library=emul(), **k)


def test_reference_align_cases_restated():
    """The cases of the reference's tests/test_align.py (one mismatch cost per call)."""
    assert list(ed(["", "", "A", "A", "A", "BA"], ["", "A", "B", "A", "AB", "AB"])) == [0, 1, 1, 0, 1, 2]
    assert list(ed(["acgt"], ["ACGT"])) == [4]
    s, t = zip(*STRING_PAIRS)
    assert list(ed(s, [""] * len(s))) == [len(x) for x in s]
    assert list(ed(s, t)) == list(ed(t, s))
    for mm in (1, 10, 30, 40, 50):
        for gs in (1, 10, 30, 40, 50):
            assert list(ed_aff(["", "", "A", "A", "A"], ["", "A", "B", "A", "AB"], mm, gs, 10)) == [0, gs, min(2 * gs, mm), 0, gs]
            assert ed_aff(["BA"], ["AB"], mm, gs, 100)[0] == min(2 * mm, 2 * gs)
            ne = [x for x in s if x]
            assert list(ed_aff(ne, [""] * len(ne), mm, gs, 10)) == [gs + (len(x) - 1) * 10 for x in ne]
            assert list(ed_aff([""] * len(ne), ne, mm, gs, 10)) == [gs + (len(x) - 1) * 10 for x in ne]
            assert list(ed_aff(s, t, mm, gs, 10)) == list(ed_aff(t, s, mm, gs, 10))
    assert ed_aff(["ATCCTC"], ["ATCGGGCTC"], 50, 10, 5)[0] == 20
    assert list(ed(s, t)) == list(ed_aff(s, t, 1, 1, 1))


def random_pairs(rng, n, long_share=0.02):
    qs, ts = [], []
    for _ in range(n):
        if rng.random() < long_share:
            a = "".join(rng.choice("ACGT") for _ in range(rng.randrange(65, 400)))
            b = list(a)
            for _ in range(rng.randrange(0, 40)):
                k = rng.randrange(len(b))
                b[k:k + rng.randrange(0, 3)] = rng.choice(["", "A", "CG", "T" * rng.randrange(1, 100)])
            qs.append(a), ts.append("".join(b))
        else:
            qs.append("".join(rng.choice("ACGTacgN") for _ in range(rng.randrange(0, 50))))
            ts.append("".join(rng.choice("ACGT") for _ in range(rng.randrange(0, 50))))
    return qs, ts


def test_random_pairs_against_reference():
    """10^5 random pairs of both distances, a few of them long (warp path), against the compiled reference."""
    align = reference_align()
    if align is None:
        pytest.skip("the reference's whatshap.align is not shipped under oracle/_ref/pyref")
    rng = random.Random(7)
    qs, ts = random_pairs(rng, 100000)
    st = {}
    got = ed(qs, ts, stats=st)
    assert st["long_jobs"] > 0
    assert list(got) == [align.edit_distance(q, t) for q, t in zip(qs, ts)]
    for mm, gs, ge in ((15.0, 10, 7), (2.5, 10.9, 3.5), (0.3, 1, 1)):
        got = ed_aff(qs[:10000], ts[:10000], mm, gs, ge)
        want = [align.edit_distance_affine_gap(q, t, [mm] * len(q), int(gs), int(ge)) for q, t in zip(qs[:10000], ts[:10000])]
        assert list(got) == want


def test_walk_against_reference_iterate_cigar():
    """The items the walk lists are the (variant, query position) pairs the reference's _iterate_cigar yields, for the golden
    alignments that do not raise."""
    rv = reference_variants()
    if rv is None:
        pytest.skip("the reference's whatshap._variants is not shipped under oracle/_ref/pyref")
    for c in golden_cases():
        if c["restricted"] or c["name"].startswith("raising"):
            continue
        variants = [Var(*v) for v in c["variants"]]
        for k, a in enumerate(c["alignments"]):
            if isinstance(c["want"][k], str):
                continue
            aln = Aln(*a)
            walked = [j for j, i, consumed, qpos in rv._iterate_cigar(variants, 0, aln, aln.cigartuples)] if aln.cigartuples else []
            got = realign.detect_alleles([aln], variants, c["reference"], overhang=c["overhang"], library=emul(), stats=(st := {}))
            symbolic = {j for j, v in enumerate(variants) if any(x.startswith("<") for x in v.alts)}
            assert st["items"] == len([j for j in walked if j not in symbolic])
            assert {i for i, _, _ in got[0]} <= set(walked)


def test_input_errors():
    v = [Var(5, "A", ["C"])]
    with pytest.raises(ValueError, match="affine"):
        realign.detect_alleles([Aln(0, [(0, 10)], "A" * 10)], v, "A" * 20, affine=True, library=emul())
    with pytest.raises(ValueError, match="overhang"):
        realign.detect_alleles([Aln(0, [(0, 10)], "A" * 10)], v, "A" * 20, overhang=-1, library=emul())
    with pytest.raises(ValueError, match="alignment 1, variant 0"):  # the first alignment covers no variant
        realign.detect_alleles([Aln(10, [(0, 5)], "A" * 5), Aln(0, [(0, 10)], "A" * 10)], v, "A" * 20,
                               restricted_genotypes=[Gt([7])], library=emul())
    assert realign.detect_alleles([Aln(0, [], "")], v, "A" * 20, library=emul()) == [[]]


def test_struct_layouts_match_the_c_compiler(tmp_path):
    """offsetof / sizeof of the new ABI types, from the C compiler, equal the ctypes mirrors."""
    fields = {"whmec_realign_input": CRealignInput, "whmec_realign_output": CRealignOutput, "whmec_realign_stats": CRealignStats}
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "whmec.h")}"', "int main(void) {"]
    for name, cls in fields.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        for f, _ in cls._fields_:
            lines.append(f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));')
    lines.append("return 0; }")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    subprocess.run(["cc", "-o", str(tmp_path / "layout"), str(src)], check=True)
    out = subprocess.run([str(tmp_path / "layout")], check=True, capture_output=True, text=True).stdout.split("\n")
    got = dict(line.split() for line in out if line)
    for name, cls in fields.items():
        assert int(got[name]) == C.sizeof(cls), name
        for f, _ in cls._fields_:
            assert int(got[f"{name}.{f}"]) == getattr(cls, f).offset, (name, f)
    assert re.search(r"WHMEC_ABI_VERSION 2", open(os.path.join(ROOT, "include", "whmec.h")).read())
