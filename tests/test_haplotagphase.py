"""Votes of `whatshap haplotagphase` (whmec_haplotagphase, DESIGN §4.16) on the CPU: the phase-set ranks, entry binning, chunk
cut and entry gather of haplotagphase_plan.cpp with the per-entry lookup, per-position walk and choice of haplotagphase.h stepped
by the host emulation tests/emul/emul_haplotagphase.cpp, and the oracle oracle/haplotagphase_oracle.py, against the reference's
answers stored in tests/golden/haplotagphase.npz."""
import ctypes as C
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import haplotagphase_cases as hc
import whatshap_b200
from whatshap_b200 import _lib, haplotagphase as hp
from whatshap_b200._abi import CHaplotagphaseInput, CHaplotagphaseOutput, CHaplotagphaseStats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
_emul = None


def emul():
    global _emul
    if _emul is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "haplotagphase.mk"], check=True, capture_output=True)
        _emul = _lib.haplotagphase_signatures(C.CDLL(os.path.join(EMUL_DIR, "libwhemul_haplotagphase.so")))
    return _emul


with np.load(os.path.join(ROOT, "tests", "golden", "haplotagphase.npz")) as z:
    GOLDEN = json.loads(z["cases"].tobytes())
    UNIT = json.loads(z["unit"].tobytes())


def swapped(library, plain_dicts=False, stats=None):
    """run_haplotagphase's loop around the swap-in pair (consensus on plain dict copies: the runs form)."""
    cv = lambda *a: hp.compute_votes(*a, library=library, stats=stats)
    if plain_dicts:
        cs = lambda *a: hp.consensus(*a[:6], {p: dict(v) for p, v in a[6].items()}, a[7], library=library)
    else:
        cs = lambda *a: hp.consensus(*a, library=library)
    return cv, cs


def emulated(case, **kw):
    return hc.run_functions(*swapped(emul(), **kw), case, whatshap_b200)


def test_golden_covers_what_it_should():
    errors = {c["want"] for c in GOLDEN if isinstance(c["want"], str)}
    assert errors == {"KeyError", "ZeroDivisionError"}
    assert {c["cut_poly"] for c in GOLDEN} >= {-1, 0, 1, 2, 10}
    assert any(c["only_indels"] for c in GOLDEN) and any(c["included"] for c in GOLDEN)
    assert any(len(c["samples"]) > 2 for c in GOLDEN)
    assert any(len({p for p, _ in c["records"]}) < len(c["records"]) for c in GOLDEN)
    assert {hp_ for c in GOLDEN for rs in c["reads"].values() for hp_, _, _ in rs} >= {-1, 0, 1, 2, 3}
    multi = [row for c in GOLDEN if not isinstance(c["want"], str) for s in c["want"] if s for _, row in s["votes"] if len(row) > 2]
    assert len(multi) > 50  # positions with several phase sets
    # homopolymers of more than 10 bases beside voted positions
    assert any("A" * 11 in c["refseq"] or "C" * 11 in c["refseq"] for c in GOLDEN if c["cut_poly"] > 0)


@pytest.mark.parametrize("i", range(len(GOLDEN)))
def test_oracle_and_emulation_equal_the_reference(i):
    case = GOLDEN[i]
    assert hc.run_oracle(case) == case["want"]
    assert emulated(case) == case["want"]


def test_runs_form_equals_the_reference():
    for case in GOLDEN:
        assert emulated(case, plain_dicts=True) == case["want"]


def test_emulation_one_position_per_chunk_equals_the_reference(monkeypatch):
    monkeypatch.setenv("WHMEC_HAPLOTAGPHASE_ARENA_BUDGET", "1")
    for case in GOLDEN:
        assert emulated(case) == case["want"]
        assert emulated(case, plain_dicts=True) == case["want"]


def test_tie_rule():
    """Keys {(5, 0): 7, (5, 1): 9, (3, 0): 9, (3, 1): 1}: the best is (5, 1), inserted before (3, 0) with the same score."""
    case = hc.tie_case()
    want = GOLDEN[0]["want"]
    assert case["reads"] == GOLDEN[0]["reads"] and want[0]["votes"] == [[40, [[5, 0, 7], [5, 1, 9], [3, 0, 9], [3, 1, 1]]]]
    assert want[0]["components"] == [[40, 5]] and want[0]["super"] == [[[40, 1, 9]], [[40, 0, 9]]]
    assert emulated(case) == want and emulated(case, plain_dicts=True) == want


def test_gap_threshold_is_compared_as_a_double():
    """score 29 of total 100: 100 * (29 / 100) is 28.999999999999996, so a gap of 29 drops the position and 28 keeps it."""
    assert 100 * (29 / 100) < 29
    dropped, kept = GOLDEN[1], GOLDEN[2]
    assert (dropped["gap"], kept["gap"]) == (29, 28)
    assert dropped["want"][0]["super"] == [[], []] and dropped["want"][0]["components"] == [[50, 1000]]
    assert kept["want"][0]["super"] == [[[50, 0, 29]], [[50, 1, 29]]]
    for case in (dropped, kept):
        assert emulated(case) == case["want"] and emulated(case, plain_dicts=True) == case["want"]
    (v,) = hp.vote([_sample(dropped)], gap_threshold=29, library=emul())
    assert v.kept.tolist() == [False] and (v.score[0], v.total[0]) == (29, 100)


def test_homopolymer_filter_removes_nothing():
    """The reference counts a homopolymer up to cut_poly bases and drops a position only beyond cut_poly: every stored case
    with cut_poly > 0 has the answer of the same case with the filter off."""
    checked = 0
    for case in GOLDEN:
        if case["cut_poly"] > 0 and not isinstance(case["want"], str):
            assert hc.run_oracle(dict(case, cut_poly=-1)) == case["want"]
            checked += 1
    assert checked >= 10


def _sample(case, name="S0"):
    from oracle import haplotagphase_oracle as o

    records = [(p, snv, gt, ph) for (p, snv), (gt, ph) in zip(case["records"], case["calls"][name])]
    homozygous, a2i, i2a, phased, snv = o.tables(records)
    phased = {p: (1 if f else None) for p, f in phased.items()}
    return hp.Sample(hc.readset(whatshap_b200, case["reads"][name]), homozygous, a2i, i2a, phased, snv)


def test_vote_arrays_equal_the_reference():
    for case in GOLDEN:
        if isinstance(case["want"], str) or case["included"]:
            continue
        got = hp.vote([_sample(case, s) for s in case["samples"]], gap_threshold=case["gap"], only_indels=case["only_indels"], library=emul())
        for v, want in zip(got, case["want"]):
            assert hc.plain_votes(v.as_dict()) == want["votes"]
            assert [[int(p), int(c)] for p, c in zip(v.position, v.phase_set)] == want["components"]
            kept = sorted((int(p), int(a[0]), int(a[1]), int(s)) for p, a, s, k in zip(v.position, v.allele, v.score, v.kept) if k)
            assert [[p, a0, s] for p, a0, _, s in kept] == want["super"][0]
            assert [[p, a1, s] for p, _, a1, s in kept] == want["super"][1]


def test_compute_votes_restated():
    """The reference's test_compute_votes."""
    u = UNIT["compute_votes"]
    for core in (whatshap_b200,):
        got = hp.compute_votes(dict(u["homozygous"]), hc.readset(core, u["reads"]), {p: dict(m) for p, m in u["allele_to_id"]}, library=emul())
        assert got == {1: {(0, 0): 50, (0, 1): 0, (1, 1): 20, (1, 0): 0}, 2: {(0, 0): 10, (0, 1): 30}}
        assert hc.plain_votes(got) == u["want"]


def test_best_candidate_doctests():
    """The reference's best_candidate doctests, through the runs form: (h, ps, q, score)."""
    for vote, (h, ps, q, score) in UNIT["best_candidate"]:
        runs = (np.zeros(1, np.uint32), np.array([9], np.int64), np.array([0, len(vote)], np.uint64),
                *(np.array([r[k] for r in vote], np.int64) for k in range(3)))
        table = ([9], lambda p: 2, lambda p: [], lambda p: [])
        (v,), _ = hp._call(hp._tables([table]), 1, runs=runs, library=emul())
        assert (int(v.haplotype[0]), int(v.phase_set[0]), int(v.score[0]) / int(v.total[0]), int(v.score[0])) == (h, ps, q, score)
        assert v.error.tolist() == [2]  # kept (phased) and id_to_allele is empty: KeyError


def _one(reads, records, **kw):
    from oracle import haplotagphase_oracle as o

    homozygous, a2i, i2a, phased, snv = o.tables(records)
    phased = {p: (1 if f else None) for p, f in phased.items()}
    return hp.vote([hp.Sample(hc.readset(whatshap_b200, reads), homozygous, a2i, i2a, phased, snv)], library=emul(), **kw)


def test_error_order_and_sources():
    records = [(10, True, [0, 1], False), (20, True, [0, 1, 1], False), (30, True, [0, 0], False), (40, True, [0, 1], False)]
    # KeyError: a position without a record, an allele without an id, an id that is not 0 or 1 (polyploid); the first entry
    # in read order decides, and a homozygous position is skipped before its allele is looked up
    for reads, key in (([[1, 1, [[10, 0, 5], [99, 0, 5], [10, 7, 1]]]], 99), ([[1, 1, [[30, 7, 5], [10, 7, 5], [99, 0, 5]]]], 7),
                       ([[2, 3, [[20, 1, 5], [99, 0, 1]]]], (2, 3)), ([[3, 1, [[99, 0, 5]]], [1, 1, [[20, 0, 5], [20, 1, 5]]]], (0, 2))):
        with pytest.raises(KeyError) as e:
            _one(reads, records)
        assert e.value.args[0] == key
    # ZeroDivisionError at a later position in vote order loses to a KeyError of the vote; a zero total raises in consensus
    with pytest.raises(ZeroDivisionError):
        _one([[1, 1, [[40, 0, 0], [10, 0, 3]]]], records)
    with pytest.raises(KeyError):
        _one([[1, 1, [[40, 0, 0], [99, 0, 3]]]], records)
    # a second sample's vote error comes after the first sample's consensus error
    s0 = [[1, 1, [[40, 0, 0]]]]
    from oracle import haplotagphase_oracle as o

    t = o.tables(records)
    mk = lambda reads: hp.Sample(hc.readset(whatshap_b200, reads), t[0], t[1], t[2], {p: None for p in t[3]}, t[4])
    with pytest.raises(ZeroDivisionError):
        hp.vote([mk(s0), mk([[1, 1, [[99, 0, 1]]]])], library=emul())


def test_runs_form_errors_and_ties_in_dict_order():
    change = {5: type("V", (), {"is_snv": lambda self: False})()}
    # dict order decides ties; an empty vote is IndexError; a kept position without its ids is KeyError
    sup, comp = hp.consensus(False, 0, 10, "", change, {5: None}, {5: {(3, 1): 4, (2, 0): 4}}, {5: {0: 7, 1: 8}}, library=emul())
    assert comp == {5: 3} and [(v.position, v.allele, v.quality) for v in sup[0]] == [(5, 8, 4)]
    with pytest.raises(IndexError):
        hp.consensus(False, 0, 10, "", change, {5: None}, {5: {}}, {5: {0: 7, 1: 8}}, library=emul())
    with pytest.raises(KeyError):
        hp.consensus(False, 0, 10, "", change, {5: None}, {5: {(3, 1): 4}}, {5: {1: 8}}, library=emul())
    with pytest.raises(ZeroDivisionError):
        hp.consensus(False, 0, 10, "", change, {5: None}, {5: {(3, 1): 4, (3, 0): -4}}, {5: {0: 7, 1: 8}}, library=emul())
    with pytest.raises(ValueError):
        hp.consensus(False, 0, 10, "", change, {5: None}, {5: {(3, 1): 1 << 53}}, {5: {0: 7, 1: 8}}, library=emul())


def test_skipped_reads_are_logged(caplog):
    records = [(10, True, [0, 1], False)]
    from oracle import haplotagphase_oracle as o

    t = o.tables(records)
    with caplog.at_level("WARNING"):
        hp.compute_votes(t[0], hc.readset(whatshap_b200, [[3, 1, [[10, 0, 1]]], [4, 2, []], [3, 0, []], [1, 1, [[10, 0, 1]]]]), t[1], library=emul())
    assert "2 reads were skipped due incorrect HP" in caplog.text


@pytest.mark.parametrize("seed", [1, 2])
def test_emulation_equals_the_oracle_on_large_inputs(seed, monkeypatch):
    rng = random.Random(seed)
    case = hc.make_case(rng, big=True, n_samples=3, included=[])
    want = hc.run_oracle(case)
    st = {}
    assert emulated(case, stats=st) == want
    assert st["chunks"] == 1 and st["records"] > 0
    monkeypatch.setenv("WHMEC_HAPLOTAGPHASE_ARENA_BUDGET", str(st["entries"] * 60))
    st2 = {}
    assert emulated(case, stats=st2) == want
    assert st2["chunks"] > 1 and (st2["records"], st2["positions"], st2["entries"]) == (st["records"], st["positions"], st["entries"])


def test_live_reference_where_available():
    """The reference's own run_haplotagphase with the swap-in against the same function without it, on fresh seeded cases, in
    a process of its own (its package stubs pysam)."""
    from oracle import build_pyref

    if not build_pyref.build():
        pytest.skip("no WhatsHap source tree at $WHATSHAP_REF")
    code = f"""
import ctypes, random, sys
sys.path[:0] = [{os.path.join(ROOT, "tests", "golden")!r}, {os.path.join(ROOT, "tests")!r}, {ROOT!r}]
import make_haplotagphase_golden as m
h = m.reference_module()
import whatshap.core as core
import whatshap_b200.adapters as a, haplotagphase_cases as hc
from whatshap_b200 import _lib
lib = _lib.haplotagphase_signatures(ctypes.CDLL({os.path.join(EMUL_DIR, "libwhemul_haplotagphase.so")!r}))
cv, cs = a.make_haplotagphase(h)
orig = (h.compute_votes, h.consensus)
rng = random.Random(11)
bad = 0
for i in range(40):
    c = hc.make_case(rng, big=i % 10 == 0, error=[None, None, None, "position", "allele", "haplotype", "zero"][i % 7])
    h.compute_votes, h.consensus = orig
    want = hc.run_module(h, c, core)
    h.compute_votes, h.consensus = (lambda *x: cv(*x, library=lib)), (lambda *x: cs(*x, library=lib))
    got = hc.run_module(h, c, core)
    bad += want != got
    if not isinstance(got, str):
        assert all(type(v) is h.Variant for v in cs(False, 0, 0, "", {{}}, {{5: 1}}, {{5: {{(0, 0): 1}}}}, {{5: {{0: 0, 1: 1}}}}, library=lib)[0][0])
print(bad)
"""
    emul()
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split()[-1] == "0"


def test_struct_layouts_match_the_c_compiler(tmp_path):
    fields = {"whmec_haplotagphase_input": CHaplotagphaseInput, "whmec_haplotagphase_output": CHaplotagphaseOutput,
              "whmec_haplotagphase_stats": CHaplotagphaseStats}
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


def test_malformed_arguments_are_refused():
    records = [(10, True, [0, 1], False)]
    with pytest.raises(ValueError):
        _one([[1, 1, [[10, 0, 1 << 40]]]], records)
    n = C.c_uint64(0)
    off = (C.c_uint64 * 1)()
    ci = CHaplotagphaseInput(n_samples=0, pos_off=C.pointer(n))
    out = CHaplotagphaseOutput(voted_off=off)
    err = C.create_string_buffer(256)
    assert emul().whmec_haplotagphase(C.byref(ci), 0, C.byref(out), None, err, 256) == 0
    emul().whmec_haplotagphase_release(C.byref(out))
    assert emul().whmec_haplotagphase(None, 0, C.byref(out), None, err, 256) == 2
