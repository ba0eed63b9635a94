"""K-mer pair counts of `whatshap learn` (whmec_learn, DESIGN §4.13) on the CPU: the host walk, floors, variant windows and chunk
cut of learn_plan.cpp with the per-read emit of learn.h stepped by the host emulation tests/emul/emul_learn.cpp, against the
reference's answers stored in tests/golden/learn.npz."""
import ctypes as C
import json
import os
import random
import re
import subprocess

import numpy as np
import pytest

import whatshap_b200
from whatshap_b200 import _lib, learn
from whatshap_b200._abi import CLearnInput, CLearnOutput, CLearnStats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
_emul = None


def emul():
    global _emul
    if _emul is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "learn.mk"], check=True, capture_output=True)
        L = _lib.learn_signatures(C.CDLL(os.path.join(EMUL_DIR, "libwhemul_learn.so")))
        i32p = C.POINTER(C.c_int32)
        L.whemul_learn_intervals.argtypes = [i32p, i32p, C.c_uint32, C.POINTER(C.c_uint32), C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                             C.POINTER(C.c_int64), C.c_uint64]
        L.whemul_learn_intervals.restype = C.c_uint64
        _emul = L
    return _emul


def golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "learn.npz")) as z:
        return json.loads(z["cases"].tobytes())


GOLDEN = golden()


def segments(case):
    return [(ref.encode(), [(p, [tuple(x) for x in cg], q.encode()) for p, cg, q in reads]) for ref, reads in case["segments"]]


def blocks(text):
    """The lines of a counts file as consecutive blocks of one column: [(column, sorted lines)]."""
    out = []
    for line in text.splitlines():
        col = line.split("\t")[0]
        if out and out[-1][0] == col:
            out[-1][1].append(line)
        else:
            out.append((col, [line]))
    return [(c, sorted(lines)) for c, lines in out]


def as_text(rows):
    return "".join("%d\t%d\t%d\t%d\n" % tuple(r) for r in rows.tolist())


def count_case(case, library=None, **kw):
    """The file run_learn writes for the case, through count_kmer_pairs per chromosome run (the last one final)."""
    segs = segments(case)
    text, front = "", 0
    for s, (ref, reads) in enumerate(segs):
        rows, front = learn.count_kmer_pairs(reads, case["variants"], ref, case["k"], case["window"], first_variant=front,
                                             final=s == len(segs) - 1, library=library, **kw)
        text += as_text(rows)
    return text


def caller_case(case, path, library, buffer_bytes=None):
    """The file the swap-in Caller writes for the calls run_learn makes on the case."""
    open(path, "w").close()
    out = str(path).encode()
    caller = None
    for s, (ref, reads) in enumerate(segments(case)):
        caller = learn.Caller(ref, case["k"], case["window"], library=library)
        if buffer_bytes is not None:
            caller.buffer_bytes = buffer_bytes
        if s == 0:
            caller.all_variants(case["variants"])
        for pos, cigar, query in reads:
            caller.add_read(pos, [list(x) for x in cigar], query, out)
    caller.final_pop(out)
    return open(path).read()


def test_golden_covers_the_issue():
    cases = GOLDEN["cases"]
    assert {c["k"] for c in cases} == set(range(1, 16))
    assert {c["window"] for c in cases} >= {0, 25}
    assert sum(len(c["segments"]) > 1 for c in cases) > 50
    reads = [r for c in cases for _, rd in c["segments"] for r in rd]
    ops = {op for _, cg, _ in reads for op, _ in cg}
    assert {0, 1, 2, 3, 4, 5, 7, 8} <= ops
    assert any(cg and cg[0][0] == 1 for _, cg, _ in reads)  # leading insertion
    assert any(any(op == 4 for op, _ in cg[1:-1]) for _, cg, _ in reads)  # mid-read S
    assert any(any(op == 4 and n == 0 for op, n in cg) for _, cg, _ in reads)
    assert any(cg == [[0, c["k"]]] for c in cases for _, rd in c["segments"] for _, cg, _ in rd)  # a single k-mer
    assert any("N" in q for _, _, q in reads) and any(any(ch.islower() for ch in q) for _, _, q in reads)
    assert any(any(a[0] > b[0] for a, b in zip(rd, rd[1:])) for c in cases for _, rd in c["segments"])  # unsorted reads
    assert sum(c["expected"].count("\n") for c in cases) > 10000
    assert GOLDEN["fixture"]["expected"].count("\n") == 28


@pytest.mark.parametrize("index", range(len(GOLDEN["cases"])))
def test_golden_case_emulated(index):
    case = GOLDEN["cases"][index]
    assert blocks(count_case(case, emul())) == blocks(case["expected"])


def test_fixture_byte_for_byte(tmp_path):
    fx = GOLDEN["fixture"]
    assert set(fx["chromosomes"]) == {"chr1"}
    assert count_case(fx, emul()) == fx["expected"]
    ref, reads = fx["segments"][0]
    rows, front = learn.count_kmer_pairs([tuple(r) for r in reads], fx["variants"], ref, library=emul())
    path = tmp_path / "counts.txt"
    learn.write_counts(path, rows, append=False, library=emul())
    assert path.read_text() == fx["expected"]
    assert front == 0


def test_swapin_caller_runs_run_learn_on_the_fixture(tmp_path):
    """run_learn's calls on learn-data (one Caller, all_variants, add_read per mapped read, final_pop) write expected.txt."""
    fx = GOLDEN["fixture"]
    assert caller_case(fx, tmp_path / "out.txt", emul()) == fx["expected"]
    assert whatshap_b200.Caller is learn.Caller


@pytest.mark.parametrize("index", range(0, len(GOLDEN["cases"]), 8))
def test_swapin_caller_on_golden_cases(tmp_path, index):
    case = GOLDEN["cases"][index]
    assert blocks(caller_case(case, tmp_path / "out.txt", emul())) == blocks(case["expected"])


def test_caller_flushed_in_parts_equals_one_flush(tmp_path):
    for case in GOLDEN["cases"][:60]:
        whole = caller_case(case, tmp_path / "a.txt", emul())
        assert caller_case(case, tmp_path / "b.txt", emul(), buffer_bytes=0) == whole, case["name"]


def test_caller_writes_each_pop_to_its_own_file(tmp_path):
    case = next(c for c in GOLDEN["cases"] if len(c["segments"]) == 1 and c["expected"].count("\n") > 200)
    ref, reads = segments(case)[0]
    caller = learn.Caller(ref, case["k"], case["window"], library=emul())
    caller.all_variants(case["variants"])
    files = [tmp_path / f"{i}.txt" for i in range(3)]
    for f in files:
        f.write_text("")
    for i, (pos, cigar, query) in enumerate(reads):
        caller.add_read(pos, cigar, query, str(files[i % 2]).encode())
    caller.final_pop(str(files[2]).encode())
    parts = [f.read_text() for f in files]
    assert blocks("".join(parts)) != [] and sorted(blocks(case["expected"])) == sorted(blocks("".join(parts)))
    top = max([case["k"] - 1] + [p + case["k"] - 1 for p, _, _ in reads])
    assert all(int(line.split("\t")[0]) > top for line in parts[2].splitlines())


def intervals_by_column(pos, length, off, lo, hi, window, k):
    """pop_column's state machine column by column (caller.cpp), with no next variant where one is left."""
    out = []
    for c in range(lo, hi + 1):
        var = (pos[off], length[off])
        if var[0] - window <= c <= var[0] + var[1] - 1 + window + k - 1:
            continue
        if off + 1 < len(pos) and pos[off + 1] - window <= c <= pos[off + 1] + length[off + 1] - 1 + window:
            off += 1
            continue
        out.append(c)
    return out, off


def test_intervals_equal_the_column_state_machine():
    rng = random.Random(7)
    L = emul()
    for _ in range(3000):
        n = rng.randrange(1, 8)
        pos = [rng.randrange(-20, 300) for _ in range(n)]
        if rng.random() < 0.7:
            pos.sort()
        length = [rng.choice([0, 1, 1, 2, 7, 30]) for _ in range(n)]
        window, k = rng.randrange(0, 30), rng.randrange(1, 16)
        off0 = rng.randrange(n)
        lo = rng.randrange(1, 200)
        hi = lo + rng.randrange(-1, 250)
        want, want_off = intervals_by_column(pos, length, off0, lo, hi, window, k)
        p, ln = np.array(pos, np.int32), np.array(length, np.int32)
        buf = np.zeros(1024, np.int64)
        off = C.c_uint32(off0)
        m = L.whemul_learn_intervals(p.ctypes.data_as(C.POINTER(C.c_int32)), ln.ctypes.data_as(C.POINTER(C.c_int32)), n, C.byref(off), lo, hi,
                                     window, k, buf.ctypes.data_as(C.POINTER(C.c_int64)), len(buf))
        got = [c for a, b in buf[:m].reshape(-1, 2).tolist() for c in range(a, b + 1)]
        assert got == want and off.value == want_off
        assert all(b + 1 < a for (_, b), (a, _) in zip(buf[:m].reshape(-1, 2).tolist(), buf[2:m].reshape(-1, 2).tolist()))


def long_reads_case(rng, n_reads=40, length=3000, k=11):
    ref = "".join(rng.choice("ACGT") for _ in range(20000)).encode()
    reads = []
    for _ in range(n_reads):
        p = rng.randrange(0, 20000 - length - 200)
        q = bytearray(ref[p:p + length])
        q[rng.randrange(length)] = ord("N")
        reads.append((p, [(0, 1000), (1, 7), (2, 20), (0, length - 1007), (4, 0), (0, 7)], bytes(q) + b"ACGTACG"))
    reads.sort(key=lambda r: r[0])
    variants = [(v, 1) for v in sorted(rng.sample(range(1, 20000), 30))] + [(10**9, 1)]
    return ref, reads, variants, k


def test_chunk_cut_equals_one_chunk(monkeypatch):
    rng = random.Random(3)
    ref, reads, variants, k = long_reads_case(rng)
    st = {}
    whole, front = learn.count_kmer_pairs(reads, variants, ref, k, 25, stats=st, library=emul())
    assert st["chunks"] == 1 and st["rows"] == len(whole) > 0 and st["kept"] > st["distinct"] >= st["rows"]
    for budget in (1, 64 * 50, 64 * 4000, 64 * 40000):
        monkeypatch.setenv("WHMEC_LEARN_ARENA_BUDGET", str(budget + (0 if budget == 1 else 200000)))  # the reads take ~155 kB
        st_b = {}
        got, f = learn.count_kmer_pairs(reads, variants, ref, k, 25, stats=st_b, library=emul())
        assert np.array_equal(got, whole) and f == front
        assert st_b["chunks"] > 1 and st_b["kept"] == st["kept"]
    monkeypatch.setenv("WHMEC_LEARN_ARENA_BUDGET", "1")  # one column with keys per chunk
    st_b = {}
    learn.count_kmer_pairs(reads, variants, ref, k, 25, stats=st_b, library=emul())
    assert st_b["chunks"] >= len(set(whole[:, 0].tolist()))


def test_golden_cases_chunked(monkeypatch):
    monkeypatch.setenv("WHMEC_LEARN_ARENA_BUDGET", "200")
    for case in GOLDEN["cases"][::5]:
        assert blocks(count_case(case, emul())) == blocks(case["expected"]), case["name"]


@pytest.mark.parametrize("index", range(len(GOLDEN["refusals"])))
def test_refusals(index):
    c = GOLDEN["refusals"][index]
    reads = [(p, [tuple(x) for x in cg], q.encode()) for p, cg, q in c["reads"]]
    with pytest.raises(ValueError) as e:
        learn.count_kmer_pairs(reads, c["variants"], c["reference"].encode(), c["k"], c["window"], library=emul())
    assert re.search(c["error"], str(e.value)), (c["name"], str(e.value))


def test_caller_names_the_read_it_refuses(tmp_path):
    caller = learn.Caller(b"ACGTACGTACGTACGTACGT", 5, 2, library=emul())
    caller.all_variants([(3, 1), (10**9, 1)])
    out = str(tmp_path / "o").encode()
    caller.add_read(0, [(0, 10)], b"ACGTACGTAC", out)
    caller.add_read(2, [(0, 3)], b"ACG", out)
    with pytest.raises(ValueError, match="^read 1 of this Caller: the query has no k-mer"):
        caller.final_pop(out)


def test_caller_names_a_read_beyond_the_reference(tmp_path):
    """pos + k - 1 > L: the flush reaches columns beyond L, and the refusal still names the read, not the column range."""
    caller = learn.Caller(b"ACGTACGTACGTACGTACGT", 5, 2, library=emul())
    caller.all_variants([(3, 1), (10**9, 1)])
    out = str(tmp_path / "o").encode()
    caller.add_read(0, [(0, 10)], b"ACGTACGTAC", out)
    caller.add_read(17, [(1, 5)], b"ACGTA", out)  # five inserted bytes: one k-mer at column 18, target 21 > 20
    with pytest.raises(ValueError, match=r"^read 1 of this Caller: pos \+ k - 1 lies beyond the reference"):
        caller.final_pop(out)


def test_library_rejects_null_arrays():
    starts, off, qoff = (C.c_int32 * 1)(0), (C.c_uint64 * 2)(0, 1), (C.c_uint64 * 2)(0, 5)
    vpos, vlen = (C.c_int32 * 1)(3), (C.c_int32 * 1)(1)
    ref = b"ACGTACGTACGT"
    for cigar_op, query in ((None, b"ACGTA"), ((C.c_uint8 * 1)(0), None)):
        cigar_len = (C.c_int32 * 1)(5)
        ci = CLearnInput(C.cast(C.c_char_p(ref), C.POINTER(C.c_uint8)), len(ref), 1, starts, off,
                         C.cast(cigar_op, C.POINTER(C.c_uint8)), cigar_len, qoff,
                         C.cast(C.c_char_p(query), C.POINTER(C.c_uint8)) if query else None, 1, vpos, vlen, 0, 3, 0, 1, 0, 0, None)
        out, err = CLearnOutput(), C.create_string_buffer(256)
        assert emul().whmec_learn(C.byref(ci), 0, C.byref(out), None, err, len(err)) == 2
        assert b"null or malformed" in err.value


def test_write_counts_formats_as_the_reference(tmp_path):
    rows = np.array([[5, 0, 1023, 2], [2**31 - 1, 7, 0, 1], [-3, 1, 2, 3]], np.int32)
    path = tmp_path / "c.txt"
    path.write_text("x\n")
    learn.write_counts(path, rows, library=emul())
    assert path.read_text() == "x\n5\t0\t1023\t2\n2147483647\t7\t0\t1\n-3\t1\t2\t3\n"
    learn.write_counts(path, rows[:1], append=False, library=emul())
    assert path.read_text() == "5\t0\t1023\t2\n"
    with pytest.raises(OSError):
        learn.write_counts(tmp_path / "no" / "such" / "dir", rows, library=emul())


def test_struct_layouts_match_the_c_compiler(tmp_path):
    fields = {"whmec_learn_input": CLearnInput, "whmec_learn_output": CLearnOutput, "whmec_learn_stats": CLearnStats}
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
