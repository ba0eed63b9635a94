"""Allele detection by k-mer re-alignment (whmec_realign_kmerald, whmec_kmer_align_batch, DESIGN §4.12) on the CPU: the host walk
and chunk plan of realign_plan.cpp with the per-job code of kmerald.h stepped by the host emulation tests/emul/emul_kmerald.cpp,
against the reference's answers stored in tests/golden/kmerald.npz."""
import csv
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest

from whatshap_b200 import _lib, realign
from whatshap_b200._abi import CKmeraldParams, CKmerCosts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
_emul = None


def emul():
    global _emul
    if _emul is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "kmerald.mk"], check=True, capture_output=True)
        L = _lib.realign_signatures(C.CDLL(os.path.join(EMUL_DIR, "libwhemul_kmerald.so")))
        L.whemul_enumerate_kmers.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
        L.whemul_enumerate_kmers.restype = C.c_uint32
        _emul = L
    return _emul


def enumerate_kmers(s: bytes, k: int):
    out = (C.c_uint32 * max(len(s), 1))()
    n = emul().whemul_enumerate_kmers(s, len(s), k, out)
    return list(out[:n])


class Aln:
    def __init__(self, start, cigar, seq):
        self.reference_start, self.cigartuples, self.query_sequence = start, [tuple(x) for x in cigar], seq


class Biallelic:
    def __init__(self, position, ref, alt):
        self.position, self.reference_allele, self.alternative_allele = position, ref, alt

    def get_alt_allele_list(self):
        return [self.alternative_allele]


class Multiallelic:  # no alternative_allele, as the reference's MultiallelicVcfVariant
    def __init__(self, position, ref, alts):
        self.position, self.reference_allele, self.alts = position, ref, list(alts)

    def get_alt_allele_list(self):
        return self.alts


class Gt:
    def __init__(self, v):
        self.v = list(v)

    def as_vector(self):
        return self.v


def golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "kmerald.npz")) as z:
        return json.loads(z["cases"].tobytes())


GOLDEN = golden()


def variant(p, r, alts):
    return Biallelic(p, r, alts[0]) if len(alts) == 1 else Multiallelic(p, r, alts)


def cost_dict(rows):
    """The dict the reference's _alignments_to_reads builds from the file's rows (variants.py:451-454)."""
    d = {}
    for a, b, v in rows:
        d[(int(a), int(b))] = v
    return d


def case_args(c, alignments=None):
    alns = [Aln(*a) for a in (c["alignments"] if alignments is None else alignments)]
    variants = [variant(*v) for v in c["variants"]]
    kw = dict(restricted_genotypes=[Gt(v) for v in c["restricted"]] if c["restricted"] else None, use_kmerald=True,
              kmerald_costs=realign.KmerCosts(cost_dict(c["costs"])), kmer_size=c["k"], kmerald_gappenalty=c["gap"],
              kmerald_window=c["window"])
    return alns, variants, c["reference"], kw


def check_case(c, run, **extra):
    """The alignments the reference answers give its calls; the whole list raises ValueError naming the first alignment the
    reference raises on (and the variant, where the reference fails in realign())."""
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


def as_f32(text):
    return np.float32(float(text))


def same_f32(got, want):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    return got.shape == want.shape and bool(np.all((got == want) | (np.isnan(got) & np.isnan(want))))


def test_golden_covers_the_issue():
    d = GOLDEN["detect"]
    assert {c["k"] for c in d} >= {1, 3, 5, 7, 11, 15}
    assert {c["window"] for c in d} >= {0, 25, 25.7}
    assert any(not float(c["gap"]).is_integer() for c in d)
    assert any(c["restricted"] for c in d)
    assert {"AttributeError", "AssertionError", "ValueError"} <= {w for c in d for w in c["want"] if isinstance(w, str)}
    ops = {op for c in d for a in c["alignments"] for op, _ in a[1]}
    assert {0, 1, 2, 3, 4, 5, 6, 7, 8, 9} <= ops
    assert any("N" in a[2] for c in d for a in c["alignments"]) and any(any(ch.islower() for ch in c["reference"]) for c in d)
    assert any(v[2][0].startswith("<") for c in d for v in c["variants"])
    assert max(len(v[2][0]) for c in d for v in c["variants"]) > 1024
    rows = [r for c in d for r in c["costs"]]
    assert any(r[2] == "nan" for r in rows) and any(r[2] == "inf" for r in rows)
    assert any(len(c["costs"]) > len(cost_dict(c["costs"])) for c in d)  # repeated keys


@pytest.mark.parametrize("index", range(len(GOLDEN["detect"])))
def test_golden_case_emulated(index):
    check_case(GOLDEN["detect"][index], emul_detect)


def test_enumeration_equals_reference():
    for s, k, want in GOLDEN["enumerate"]:
        assert enumerate_kmers(s.encode(), k) == want, (s, k)
    assert enumerate_kmers(b"ACGTNACGT", 3) == [6, 27, 27, 44, 49, 6, 27]
    assert enumerate_kmers(b"acgtACG", 3) == [1, 6]
    assert enumerate_kmers(b"NNNNNNC", 7) == [1]


@pytest.mark.parametrize("table", range(len(GOLDEN["pairs"])))
def test_golden_pairs_emulated(table):
    t = GOLDEN["pairs"][table]
    s1, s2 = zip(*t["seqs"])
    st = {}
    got = realign.kmer_distances(s1, s2, cost_dict(t["costs"]), t["gap"], t["k"], stats=st, library=emul())
    assert same_f32(got, [as_f32(w) for w in t["want"]])
    assert st["short_jobs"] > 0


def test_both_paths_in_golden_pairs():
    st = {}
    for t in GOLDEN["pairs"]:
        s1, s2 = zip(*t["seqs"])
        s = {}
        realign.kmer_distances(s1, s2, cost_dict(t["costs"]), t["gap"], t["k"], stats=s, library=emul())
        for key in ("short_jobs", "long_jobs"):
            st[key] = st.get(key, 0) + s[key]
    assert st["short_jobs"] > 0 and st["long_jobs"] > 0


# the cases of the reference's tests/test_kmeralign.py
REF_COSTS = {(53, 214): 2, (53, 858): 1, (53, 362): 0.5, (215, 53): 0.25, (215, 214): 1, (215, 858): 0.5, (215, 362): 0.25, (862, 53): 1,
             (862, -5): 10, (862, 362): 2.5, (378, 53): 0.1, (378, 214): 0.25, (378, -5): 5}


def test_reference_kmeralign_cases_restated():
    for s in [b"", b"A", b"AC", b"ATCGC", b"NNNNNNNNNNN", b"BANANA", b"MISSISSIPPI"]:
        for k in (9, 7, 6):
            assert enumerate_kmers(s, k) == []
    assert enumerate_kmers(b"TAAATCCTGG", 7) == [12341, 215, 862, 3450]
    assert enumerate_kmers(b"TAAATCCTGG", 11) == []

    def kd(a, b, gap=5):
        return realign.kmer_distances(a, b, REF_COSTS, gap, 5, library=emul())

    assert list(kd(["AATCCTGG", "AATCCGGG"], ["AATCCGGG", "AATCCTGG"])) == [13, 30]
    seq1 = ["AAACCCG", "AAACCCGG", "AAATTTCCCG", "AAAA", ""]
    seq2 = ["GCCCAAA", "GGCCCAAA", "GCCCTTTAAA", "AAAA", ""]
    pairs = [(a, b) for a in seq1 for b in seq2]
    got = kd([a for a, _ in pairs], [b for _, b in pairs])
    for (a, b), d in zip(pairs, got):
        ea, eb = enumerate_kmers(a.encode(), 5), enumerate_kmers(b.encode(), 5)
        assert d == (0 if ea == eb else 5 * (len(ea) + len(eb))), (a, b)


def test_min_keeps_nan_of_match():
    """A NaN cost in match gives NaN even with both gaps finite; a NaN gap only where min meets it first."""
    a, b = enumerate_kmers(b"ACGTA", 5), enumerate_kmers(b"ACGTC", 5)
    got = realign.kmer_distances(["ACGTA"], ["ACGTC"], {(a[0], b[0]): "nan"}, 40, 5, library=emul())
    assert math.isnan(got[0])
    got = realign.kmer_distances(["ACGTA"], ["ACGTC"], {(a[0], -5): "1.5"}, 40, 5, library=emul())
    assert got[0] == np.float32(1.5)
    got = realign.kmer_distances(["ACGTA"], ["ACGTC"], {}, 40, 5, library=emul())
    assert got[0] == 80  # no cost: inf, the gaps win


def test_costs_reader_equals_reference_reader(tmp_path):
    rows = [["7", "3", "1.5"], ["7", "-5", "10"], ["7", "3", "2.25"], ["9", "-5", "nan"], ["0", "-5", "4"], [str(2**30), "1", "3"],
            ["11", "-7", "5"], ["11", "12", " 6.5 "], ["12", "-5", "1e40"]]
    path = tmp_path / "costs.tsv"
    path.write_text("".join("\t".join(r) + "\n" for r in rows))
    want = {}
    with open(path) as f:  # variants.py:451-454
        for line in csv.reader(f, delimiter="\t"):
            want[(int(line[0]), int(line[1]))] = line[2]
    got = realign.KmerCosts.read(path)
    ref = realign.KmerCosts(want)
    assert np.array_equal(got.key, ref.key) and same_f32(got.cost, ref.cost)
    keys = {(int(k) >> 32, int(k) & 0xFFFFFFFF): v for k, v in zip(got.key, got.cost)}
    assert keys.keys() == {(7, 3), (7, 0), (9, 0), (11, 12), (12, 0)}
    assert keys[(7, 3)] == np.float32(2.25) and math.isnan(keys[(9, 0)]) and keys[(11, 12)] == np.float32(6.5) and math.isinf(keys[(12, 0)])
    assert list(got.key) == sorted(got.key)


def test_one_item_per_chunk_equals_one_chunk(monkeypatch):
    for c in GOLDEN["detect"]:
        if c["name"] not in ("random2", "random9", "random14"):
            continue
        ok = [c["alignments"][k] for k, w in enumerate(c["want"]) if not isinstance(w, str)]
        alns, variants, reference, kw = case_args(c, ok)
        st = {}
        whole = emul_detect(alns, variants, reference, stats=st, **kw)
        assert st["chunks"] == 1 and st["short_jobs"] > 0 and st["long_jobs"] > 0 and st["long_items"] > 0
        monkeypatch.setenv("WHMEC_REALIGN_ARENA_BUDGET", "1")
        st1 = {}
        assert emul_detect(alns, variants, reference, stats=st1, **kw) == whole
        assert st1["chunks"] == st1["items"] == st["items"]
        monkeypatch.delenv("WHMEC_REALIGN_ARENA_BUDGET")


def test_use_kmerald_false_is_unchanged():
    c = GOLDEN["detect"][9]
    ok = [c["alignments"][k] for k, w in enumerate(c["want"]) if not isinstance(w, str)]
    alns, variants, reference, kw = case_args(c, ok)
    kw["use_kmerald"] = False
    from test_realign import emul as realign_emul

    assert realign.detect_alleles(alns, variants, reference, library=realign_emul(), **kw) == \
        realign.detect_alleles(alns, variants, reference, library=realign_emul())


def test_input_errors():
    v = [Biallelic(5, "A", "C")]
    a = [Aln(0, [(0, 10)], "A" * 10)]
    costs = {(1, -5): 1}
    with pytest.raises(ValueError, match="kmerald_costs"):
        realign.detect_alleles(a, v, "A" * 20, use_kmerald=True, library=emul())
    for k in (0, 16, -1):
        with pytest.raises(ValueError, match="kmer_size"):
            realign.detect_alleles(a, v, "A" * 20, use_kmerald=True, kmerald_costs=costs, kmer_size=k, library=emul())
        with pytest.raises(ValueError, match="kmer_size"):
            realign.kmer_distances(["A"], ["A"], costs, 5, k, library=emul())
    with pytest.raises(ValueError, match="window"):
        realign.detect_alleles(a, v, "A" * 20, use_kmerald=True, kmerald_costs=costs, kmerald_window=-1, library=emul())
    with pytest.raises(ValueError, match="not a number"):
        realign.KmerCosts({(1, 2): "x"})
    with pytest.raises(ValueError, match="differ"):
        realign.kmer_distances(["A"], [], costs, 5, 3, library=emul())
    # overhang, affine and its costs are not used in k-mer mode
    assert realign.detect_alleles(a, v, "A" * 20, use_kmerald=True, kmerald_costs=costs, overhang=-3, affine=True, library=emul()) == [[(0, 0, 30)]]
    with pytest.raises(ValueError, match=r"^alignment 0, variant 0: the variant has no alternative_allele"):
        realign.detect_alleles([Aln(0, [(0, 20)], "A" * 20)], [Multiallelic(5, "A", ["C", "G"])], "A" * 40, use_kmerald=True,
                               kmerald_costs=costs, kmerald_window=2, library=emul())


def test_library_rejects_unsorted_keys():
    key = np.array([(5 << 32) | 3, (5 << 32) | 3], np.uint64)
    cost = np.array([1, 2], np.float32)
    kc = CKmerCosts(2, key.ctypes.data_as(C.POINTER(C.c_uint64)), cost.ctypes.data_as(C.POINTER(C.c_float)))
    params = CKmeraldParams(5, 5.0, 0, C.pointer(kc), None, None, None)
    out = np.zeros(1, np.float32)
    off = np.array([0, 1], np.uint64)
    s = np.frombuffer(b"A", np.uint8)
    err = C.create_string_buffer(256)
    u64, u8 = C.POINTER(C.c_uint64), C.POINTER(C.c_uint8)
    rc = emul().whmec_kmer_align_batch(1, off.ctypes.data_as(u64), s.ctypes.data_as(u8), off.ctypes.data_as(u64), s.ctypes.data_as(u8),
                                       C.byref(params), out.ctypes.data_as(C.POINTER(C.c_float)), 0, None, err, len(err))
    assert rc == 2 and b"strictly ascending" in err.value


def test_struct_layouts_match_the_c_compiler(tmp_path):
    fields = {"whmec_kmer_costs": CKmerCosts, "whmec_kmerald_params": CKmeraldParams}
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
