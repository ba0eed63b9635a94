"""Read assignment of `whatshap haplotag` (whmec_haplotag, DESIGN §4.15) on the CPU: the group walk, block ranks, chunk cut and
entry gather of haplotag_plan.cpp with the per-entry visit and per-group choice of haplotag.h stepped by the host emulation
tests/emul/emul_haplotag.cpp, and the oracle oracle/haplotag_oracle.py, against the reference's answers stored in
tests/golden/haplotag.npz."""
import ctypes as C
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import haplotag_cases as hc
import whatshap_b200
from whatshap_b200 import _lib, adapters, haplotag
from whatshap_b200._abi import CHaplotagInput, CHaplotagOutput, CHaplotagStats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
_emul = None


def emul():
    global _emul
    if _emul is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "haplotag.mk"], check=True, capture_output=True)
        _emul = _lib.haplotag_signatures(C.CDLL(os.path.join(EMUL_DIR, "libwhemul_haplotag.so")))
    return _emul


def golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "haplotag.npz")) as z:
        return json.loads(z["cases"].tobytes())


GOLDEN = golden()


def agrees(want, got, loose):
    if isinstance(want, str) or isinstance(got, str):
        return want == got
    return hc.same(want, got, loose)


def emulated(case, **kw):
    prepare = lambda *a: haplotag.prepare_haplotag_information(*a, library=emul(), **kw)
    return hc.run(prepare, case, whatshap_b200)


def test_golden_covers_what_it_should():
    errors = {c["want"] for c in GOLDEN if isinstance(c["want"], str)}
    assert errors == {"AssertionError", "KeyError", "IndexError"}
    assert {c["ploidy"] for c in GOLDEN} >= {1, 2, 3, 4}
    assert any(c["loose"] for c in GOLDEN)
    assert any(len(c["samples"]) > 1 for c in GOLDEN)
    assert any(r[4] == "" for c in GOLDEN for rs in c["reads"].values() for r in rs)


@pytest.mark.parametrize("i", range(len(GOLDEN)))
def test_oracle_and_emulation_equal_the_reference(i):
    case = GOLDEN[i]
    mine, _ = hc.run_oracle(case)
    assert agrees(case["want"], mine, case["loose"])
    assert agrees(case["want"], emulated(case), case["loose"])


def test_emulation_under_a_small_budget_equals_the_reference(monkeypatch):
    monkeypatch.setenv("WHMEC_HAPLOTAG_ARENA_BUDGET", "1")  # one group per chunk
    for case in GOLDEN[::7]:
        assert agrees(case["want"], emulated(case), case["loose"])


def test_live_reference_where_available():
    """The reference's own function on fresh seeded cases, in a process of its own (its package stubs pysam)."""
    from oracle import build_pyref

    if not build_pyref.build():
        pytest.skip("no WhatsHap source tree at $WHATSHAP_REF")
    code = f"""
import json, random, sys
sys.path[:0] = [{os.path.join(ROOT, "tests", "golden")!r}, {os.path.join(ROOT, "tests")!r}, {ROOT!r}]
import make_haplotag_golden as m
h = m.reference_module()
import whatshap.core as core
import whatshap_b200.adapters as a, haplotag_cases as hc
swap = a.make_prepare_haplotag_information(h)
lib = __import__("whatshap_b200._lib", fromlist=["x"]).haplotag_signatures(__import__("ctypes").CDLL({os.path.join(EMUL_DIR, "libwhemul_haplotag.so")!r}))
rng = random.Random(7)
bad = 0
for _ in range(40):
    c = hc.make_case(rng)
    want = hc.run(h.prepare_haplotag_information, c, core)
    got = hc.run(lambda *x: swap(*x, library=lib), c, core)
    _, loose = hc.run_oracle(c)
    if isinstance(want, str) or isinstance(got, str):
        bad += want != got
    else:
        bad += not hc.same(want, got, loose)
        # the swap-in's keys are the reference module's own dataclasses
        out = swap(hc.VariantTable(c), c["samples"], hc.Reader(c, core), None, c["ignore"], c["cutoff"], c["ploidy"], library=lib)
        assert all(type(k) is h.ReadAlignmentRepresentation for k in out[1]) and all(type(v) is h.PrimaryInfo for v in out[3].values())
        assert type(out[0]).__name__ == "defaultdict"
print(bad)
"""
    emul()
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split()[-1] == "0"


@pytest.mark.parametrize("seed", [1, 2])
def test_emulation_equals_the_oracle_on_large_inputs(seed, monkeypatch):
    rng = random.Random(seed)
    case = hc.make_case(rng, big=True, n_samples=2)
    want, loose = hc.run_oracle(case)
    st = {}
    got = hc.run(lambda *a: haplotag.prepare_haplotag_information(*a, library=emul(), stats=st), case, whatshap_b200)
    assert agrees(want, got, loose)
    assert st["chunks"] == 1 and st["keys"] > 0
    monkeypatch.setenv("WHMEC_HAPLOTAG_ARENA_BUDGET", str(st["entries"] * 50))
    st2 = {}
    got2 = hc.run(lambda *a: haplotag.prepare_haplotag_information(*a, library=emul(), stats=st2), case, whatshap_b200)
    assert st2["chunks"] > 1 and got2 == got
    assert (st2["keys"], st2["runs"], st2["groups"], st2["entries"]) == (st["keys"], st["runs"], st["groups"], st["entries"])


def readset(reads):
    rs = whatshap_b200.ReadSet()
    for k, (bx, start, entries) in enumerate(reads):
        r = whatshap_b200.Read(f"r{k}", 30, 0, 0, start, bx, -1, -1, "chr1", "____1", False, start + 100, False)
        for p, a, q in entries:
            r.add_variant(p, a, q)
        rs.add(r)
    return rs


def test_assign_reads_arrays():
    table = {10: (5, (0, 1)), 20: (5, (1, 0)), 30: (9, (0, 1))}
    rs = readset([("", 0, [(10, 0, 7), (20, 1, 3)]), ("T", 0, [(30, 1, 20)]), ("T", 5, [(10, 1, 4)]), ("", 0, [(30, 0, 6), (10, 0, 6)])])
    a = haplotag.assign_reads([(rs, table)], 2, linked_read_cutoff=10, library=emul())
    assert a.group.tolist() == [0, 1, 1, 3]
    assert a.n_blocks.tolist() == [1, 2, 0, 2]
    # read 1's group: block 9 scores (0, 20), block 5 (0, 4): block 9, haplotype 1, quality 20
    assert (a.block[1], a.haplotype[1], a.quality[1]) == (9, 1, 20)
    assert (a.block[0], a.haplotype[0], a.quality[0]) == (5, 0, 10)
    # read 3: block 9 (6, 0) and block 5 (6, 0) tie; block 9 was matched first
    assert (a.block[3], a.haplotype[3], a.quality[3]) == (9, 0, 6)


@pytest.mark.parametrize("ploidy,reads,exc", [
    (2, [("", 0, [(10, 0, 1), (10, 2, 1), (99, 0, 1)])], AssertionError),
    (2, [("", 0, [(10, 0, 1), (99, 0, 1), (10, 2, 1)])], KeyError),
    (2, [("", 0, [(40, 1, 1), (99, 0, 1)])], IndexError),
    (1, [("", 0, [(10, 0, 1)]), ("", 0, [(99, 0, 1)])], IndexError),
    (1, [("", 0, [(10, 1, 1)])], IndexError),
])
def test_errors_are_the_references(ploidy, reads, exc):
    table = {10: (5, (0, 1)), 40: (5, (0, 0, 1))}
    with pytest.raises(exc):
        haplotag.assign_reads([(readset(reads), table)], ploidy, library=emul())


def test_an_empty_table_and_no_reads():
    a = haplotag.assign_reads([(whatshap_b200.ReadSet(), {})], 2, library=emul())
    assert len(a.group) == 0
    a = haplotag.assign_reads([(readset([("", 0, [])]), {})], 2, library=emul())
    assert a.group.tolist() == [0] and a.haplotype.tolist() == [-1]


def test_representation_quirks():
    assert haplotag.representation("r1____1", "c", False, "____1") == ("r1", "c", False, "____1")
    assert haplotag.representation("r1", "c", False, "") == ("", "c", False, "")
    assert haplotag.representation("r1_s2", "c", True, "_s2", as_primary=True) == ("r1_s2", "c", False, "____1")
    assert haplotag.representation("ab____1", "c", True, "_s2", as_primary=True) == ("ab__", "c", False, "____1")


def test_struct_layouts_match_the_c_compiler(tmp_path):
    fields = {"whmec_haplotag_input": CHaplotagInput, "whmec_haplotag_output": CHaplotagOutput, "whmec_haplotag_stats": CHaplotagStats}
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
    with pytest.raises(ValueError):
        haplotag.assign_reads([(readset([("", 0, [(10, 0, 1 << 40)])]), {10: (1, (0, 1))})], 2, library=emul())
    n = C.c_uint64(0)
    ci = CHaplotagInput(n_samples=0, phase_off=C.pointer(n), n_reads=0)
    out = CHaplotagOutput()
    err = C.create_string_buffer(256)
    assert emul().whmec_haplotag(C.byref(ci), 0, C.byref(out), None, err, 256) == 0
    assert emul().whmec_haplotag(None, 0, C.byref(out), None, err, 256) == 2
