"""Writes tests/golden/learn.npz: the reference's own k-mer pair counts (`whatshap learn`, src/caller.cpp) for the CPU and GPU
tests of whmec_learn (DESIGN §4.13).

It drives the compiled reference binding `whatshap.core.Caller` (oracle/build_pyref.py) with ints, lists and bytes, the calls
`run_learn` makes: one Caller per run of reads on one chromosome, `all_variants` once after the first, `add_read` per read and
`final_pop` on the last Caller only.  Stored, as UTF-8 JSON:

- "fixture": the reference's tests/data/short-genome/learn-data (its BAM parsed here, so pysam is not needed) and expected.txt;
- "cases": seeded cases over every rule of §4.13: several chromosomes that carry the variant list's front and abandon their
  Callers, unsorted and overlapping reads and variants, reads whose k-mers fall under the floor, single-k-mer reads, leading
  insertions, mid-read and zero-length S, H, N, = and X, N and lower-case bases, k = 1..15, windows 0..25, each with the file
  the reference wrote.  Every variant list ends in a far sentinel, so that a next variant always exists;
- "refusals": inputs on which the reference aborts or reads out of bounds, with the error the library must raise.  These are
  made by this script's own checks and never run on the reference.

Run from the repository root: python tests/golden/make_learn_golden.py (needs $WHATSHAP_REF or a shipped binding).
"""
import gzip
import json
import os
import random
import struct
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import build_pyref  # noqa: E402

SENTINEL = (10**9, 1)
FIXTURE = os.path.join(build_pyref.REF, "tests", "data", "short-genome", "learn-data")


class Refused(Exception):
    pass


def walk(pos, cigar, query, k, L):
    """The k-mers (h, column) enumerate_kmers yields for one read, or Refused where the reference aborts or reads out of bounds."""
    mask = (1 << 2 * k) - 1
    out, h, consecutive, i, ci = [], 0, 0, 0, 0
    p = pos
    if query and not cigar:
        raise Refused("the CIGAR ends while query bytes remain")
    op, n = cigar[0] if cigar else (0, 0)
    while i < len(query):
        while True:
            if op in (2, 3):
                p += n
            elif op == 4:
                consecutive = 0
            elif not (n == 0 or op == 5):
                break
            ci += 1
            if ci >= len(cigar):
                raise Refused("the CIGAR ends while query bytes remain")
            op, n = cigar[ci]
        if op not in (0, 1, 7, 8):
            raise Refused(f"CIGAR operation {op} of length {n} while query bytes remain")
        c = "ACGT".find(chr(query[i]))
        if c >= 0:
            h = ((h << 2) | c) & mask
        consecutive += 1
        if consecutive >= k:
            out.append((h, p + 1))
        if op != 1:
            p += 1
        n -= 1
        i += 1
    if not out:
        raise Refused("the query has no k-mer")
    if pos + k - 1 > L:
        raise Refused("pos + k - 1 lies beyond the reference")
    if out[-1][1] > L:
        raise Refused("a k-mer column lies beyond the reference")
    return out


def run_reference(core, segments, variants, k, window):
    """The file run_learn's calls make the reference write: segments = [(reference bytes, [(pos, cigar, query bytes)])]."""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "out.txt")
        open(path, "w").close()
        out = path.encode()
        caller = None
        for s, (ref, reads) in enumerate(segments):
            caller = core.Caller(ref, k, window)
            if s == 0:
                caller.all_variants(variants)
            for pos, cigar, query in reads:
                caller.add_read(pos, [list(x) for x in cigar], query, out)
        caller.final_pop(out)
        return open(path).read()


def random_reference(rng, n):
    s = []
    for _ in range(n):
        r = rng.random()
        s.append("N" if r < 0.04 else rng.choice("acgt") if r < 0.07 else rng.choice("ACGT"))
    if rng.random() < 0.2:  # a run of N
        a, m = rng.randrange(n), rng.randrange(1, 40)
        s[a:a + m] = "N" * len(s[a:a + m])
    return "".join(s).encode()


def random_read(rng, ref, k, single=False):
    L = len(ref)
    for _ in range(1000):
        cigar = []
        if rng.random() < 0.3:
            cigar.append((5, rng.randrange(1, 10)))
        if rng.random() < 0.3:
            cigar.append((4, rng.randrange(0, 6)))
        if rng.random() < 0.1:
            cigar.append((1, rng.randrange(1, 4)))  # a leading insertion
        for _ in range(rng.randrange(1, 6)):
            r = rng.random()
            if r < 0.5:
                cigar.append((rng.choice((0, 0, 0, 7, 8)), rng.randrange(0, 40)))
            elif r < 0.65:
                cigar.append((1, rng.randrange(0, 6)))
            elif r < 0.8:
                cigar.append((2, rng.randrange(0, 6)))
            elif r < 0.87:
                cigar.append((3, rng.randrange(0, 30)))
            elif r < 0.95:
                cigar.append((4, rng.randrange(0, 3)))  # mid-read S (also of length 0)
            else:
                cigar.append((0, 0))
        if rng.random() < 0.3:
            cigar.append((4, rng.randrange(0, 6)))
        if single:
            cigar = [(0, k)]
        qlen = sum(n for op, n in cigar if op in (0, 1, 7, 8))
        query = "".join("N" if rng.random() < 0.03 else rng.choice("acgt") if rng.random() < 0.03 else rng.choice("ACGT")
                        for _ in range(qlen)).encode()
        pos = rng.randrange(-2, L)
        try:
            walk(pos, cigar, query, k, L)
        except Refused:
            continue
        return pos, cigar, query
    raise RuntimeError("no valid read")


def random_case(rng, idx):
    k = [1 + idx % 15, rng.randrange(1, 16)][idx % 2]
    window = rng.choice([0, 1, 3, 7, 25, rng.randrange(0, 26)])
    n_seg = rng.choice([1, 1, 2, 3])
    segments, variants = [], []
    for _ in range(n_seg):
        ref = random_reference(rng, rng.randrange(max(k, 20), 260))
        reads = [random_read(rng, ref, k, single=rng.random() < 0.08) for _ in range(rng.randrange(0, 14))]
        mode = rng.random()
        if mode < 0.6:
            reads.sort(key=lambda r: r[0])
            if reads and rng.random() < 0.5:  # one read out of order: its k-mers fall under the floor
                j = rng.randrange(len(reads))
                reads.insert(rng.randrange(len(reads) + 1), reads.pop(j))
        segments.append((ref, reads))
        vs = sorted((rng.randrange(1, len(ref) + 30), rng.choice([1, 1, 1, 2, 5, 12])) for _ in range(rng.randrange(0, 6)))
        if rng.random() < 0.15:
            rng.shuffle(vs)
        variants += vs
    if not variants:  # the sentinel must not be the front: the reference reads the entry after the front
        variants.append((rng.randrange(1, 300), 1))
    variants.append(SENTINEL)
    return {"name": f"random{idx}", "k": k, "window": window, "variants": variants,
            "segments": [[ref.decode(), [[p, [list(x) for x in cg], q.decode()] for p, cg, q in reads]] for ref, reads in segments]}


def read_bam(path):
    """(reference names, [(name, flag, reference id, pos, cigartuples, query_alignment_sequence)]) of a BAM file."""
    data = gzip.open(path).read()
    assert data[:4] == b"BAM\1"
    (l_text,) = struct.unpack_from("<i", data, 4)
    o = 8 + l_text
    (n_ref,) = struct.unpack_from("<i", data, o)
    o += 4
    names = []
    for _ in range(n_ref):
        (l_name,) = struct.unpack_from("<i", data, o)
        names.append(data[o + 4:o + 4 + l_name - 1].decode())
        o += 4 + l_name + 4
    recs = []
    while o < len(data):
        (size,) = struct.unpack_from("<i", data, o)
        ref_id, pos, l_name, _, _, n_cig, flag, l_seq = struct.unpack_from("<iiBBHHHi", data, o + 4)
        p = o + 36
        name = data[p:p + l_name - 1].decode()
        p += l_name
        cigar = [(v & 15, v >> 4) for v in struct.unpack_from(f"<{n_cig}I", data, p)]
        p += 4 * n_cig
        seq = "".join("=ACMGRSVTWYHKDBN"[(data[p + i // 2] >> (4 * (1 - i % 2))) & 15] for i in range(l_seq))
        qs = 0
        for op, n in cigar:
            if op == 5:
                continue
            if op == 4:
                qs += n
            break
        qe = l_seq
        for op, n in reversed(cigar):
            if op == 5:
                continue
            if op == 4:
                qe -= n
            break
        recs.append((name, flag, ref_id, pos, cigar, seq[qs:qe]))
        o += 4 + size
    return names, recs


def fixture():
    names, recs = read_bam(os.path.join(FIXTURE, "short-reads.bam"))
    lines = open(os.path.join(FIXTURE, "short_ref.fasta")).read().split("\n")
    reference = "".join(x.strip() for x in lines[1:])
    variants = [(int(f[1]), len(f[3])) for f in (x.split("\t") for x in open(os.path.join(FIXTURE, "variant.vcf")) if x and x[0] != "#")]
    reads = [[pos, [list(x) for x in cg], q] for _, flag, _, pos, cg, q in recs if not flag & 4 and q]
    return {"name": "learn-data", "k": 7, "window": 25, "variants": variants, "segments": [[reference, reads]],
            "expected": open(os.path.join(FIXTURE, "expected.txt")).read(), "chromosomes": [names[r[2]] for r in recs if not r[1] & 4]}


def refusals(rng):
    ref = random_reference(rng, 120).replace(b"N", b"A").upper()
    good = [random_read(rng, ref, 5) for _ in range(4)]

    def case(name, bad, err, k=5, reference=ref, variants=((50, 1), SENTINEL), at=2):
        reads = good[:at] + ([bad] if bad else []) + good[at:]
        return {"name": name, "k": k, "window": 5, "variants": [list(v) for v in variants], "reference": reference.decode(),
                "reads": [[p, [list(x) for x in cg], q.decode() if isinstance(q, bytes) else q] for p, cg, q in reads], "error": err}

    out = [
        case("no k-mer", (10, [(0, 4)], b"ACGT"), "^alignment 2: the query has no k-mer"),
        case("S resets below k", (10, [(0, 3), (4, 0), (0, 3)], b"ACGTAC"), "^alignment 2: the query has no k-mer"),
        case("empty query", (10, [(0, 0)], b""), "^alignment 2: the query has no k-mer"),
        case("P", (10, [(0, 3), (6, 2), (0, 5)], b"ACGTACGT"), "^alignment 2: CIGAR operation 6 of length 2"),
        case("B", (10, [(9, 1), (0, 5)], b"ACGTA"), "^alignment 2: CIGAR operation 9 of length 1"),
        case("unknown op", (10, [(0, 5), (12, 3), (0, 2)], b"ACGTACG"), "^alignment 2: CIGAR operation 12 of length 3"),
        case("CIGAR too short", (10, [(0, 5)], b"ACGTACG"), "^alignment 2: the CIGAR ends while query bytes remain"),
        case("no CIGAR", (10, [], b"ACGTACG"), "^alignment 2: the CIGAR ends while query bytes remain"),
        case("target beyond L", (117, [(1, 6)], b"ACGTAC"), r"^alignment 2: pos \+ k - 1 lies beyond the reference"),
        case("column beyond L", (110, [(0, 12)], b"ACGTACGTACGT"), "^alignment 2: a k-mer column lies beyond the reference"),
        case("deletion beyond L", (100, [(0, 5), (2, 30), (0, 2)], b"ACGTACG"), "^alignment 2: a k-mer column lies beyond the reference"),
        case("int32", (10, [(0, 5), (2, 2**31 - 10), (0, 20)], b"ACGTA" * 5), "^alignment 2: a reference position outside int32"),
        case("first of two", (10, [(0, 4)], b"ACGT"), "^alignment 0: the query has no k-mer", at=0),
        case("k = 0", None, "k must lie in 1..15", k=0),
        case("k = 16", None, "k must lie in 1..15", k=16),
        case("L < k", None, "shorter than k", k=15, reference=b"ACGTACGTAC"),
        case("no variants", None, "variant list is empty", variants=()),
    ]
    for c in out:  # the maker's own checks agree on every read before the offending one
        for a, (p, cg, q) in enumerate(c["reads"]):
            if 1 <= c["k"] <= 15 and len(c["reference"]) >= c["k"] and c["variants"]:
                try:
                    walk(p, [tuple(x) for x in cg], q.encode(), c["k"], len(c["reference"]))
                    assert not c["error"].startswith(f"^alignment {a}:"), c["name"]
                except Refused:
                    assert c["error"].startswith(f"^alignment {a}:"), c["name"]
                    break
    return out


def main():
    core = build_pyref.shipped_core()
    assert core is not None, "the reference binding is needed (oracle/build_pyref.py)"
    fx = fixture()
    ref, reads = fx["segments"][0]
    got = run_reference(core, [(ref.encode(), [(p, cg, q.encode()) for p, cg, q in reads])], fx["variants"], 7, 25)
    assert got == fx["expected"], "the reference binding does not reproduce its own learn-data fixture"
    rng = random.Random(20261018)
    cases = []
    for idx in range(320):
        c = random_case(rng, idx)
        segs = [(r.encode(), [(p, [tuple(x) for x in cg], q.encode()) for p, cg, q in rd]) for r, rd in c["segments"]]
        c["expected"] = run_reference(core, segs, c["variants"], c["k"], c["window"])
        cases.append(c)
    blob = {"fixture": fx, "cases": cases, "refusals": refusals(rng)}
    out = os.path.join(ROOT, "tests", "golden", "learn.npz")
    np.savez_compressed(out, cases=np.frombuffer(json.dumps(blob).encode(), np.uint8))
    print(out, os.path.getsize(out), "bytes,", len(cases), "cases,", sum(c["expected"].count("\n") for c in cases), "rows")


if __name__ == "__main__":
    main()
