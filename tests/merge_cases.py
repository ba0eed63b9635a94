"""Seeded cases of read merging (`whatshap phase --merge-reads`), shared by tests/golden/make_merge_golden.py and the tests.

A case is {"name", "reads": [[[position, allele, quality], ...], ...], "params": [error_rate, max_error_rate, positive_threshold,
negative_threshold]}; its answer is the merged reads as [[name, [[position, allele, quality], ...]], ...] or the name of the
exception raised."""
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import merge_oracle  # noqa: E402

DEFAULT = [0.15, 0.25, 1000000, 1000]


def make_reads(rng, n, spacing=1, span=None, max_len=30, error=0.1, sort=True, repeats=0.0, qualities=(1, 40), shuffle=0.0):
    """n reads on two haplotypes: runs of positions `spacing` apart with a per-allele error, optionally repeated positions,
    and, unsorted, a share of reads moved out of order."""
    span = span or max(2, n // 2)
    reads = []
    for _ in range(n):
        start = rng.randrange(span) * spacing
        length = rng.randrange(1, max_len + 1)
        hap = rng.randrange(2)
        read = []
        for x in range(length):
            entry = [start + spacing * x, hap ^ (rng.random() < error), rng.randint(*qualities)]
            read.append(entry)
            if rng.random() < repeats:
                read.append([entry[0], rng.randrange(2), rng.randint(*qualities)])
        reads.append(read)
    if sort:
        reads.sort(key=lambda r: r[0][0])
    for _ in range(int(shuffle * n)):
        a, b = rng.randrange(n), rng.randrange(n)
        reads[a], reads[b] = reads[b], reads[a]
    return [[[int(p), int(a), int(q)] for p, a, q in r] for r in reads]


def build_cases(unit_fixtures):
    """Every stored case; `unit_fixtures` are the reads of the reference's test_merge_reads.py (as data)."""
    rng = random.Random(20261019)
    cases = [dict(name="unit_read_merging", reads=unit_fixtures, params=[0.15, 0.25, 100000, 1000]),
             dict(name="unit_read_merging2", reads=unit_fixtures, params=[0.5, 0.5, 1000, 100000])]
    for k in range(12):
        cases.append(dict(name=f"dense{k}", reads=make_reads(rng, rng.randrange(20, 120), 1, max_len=40), params=DEFAULT))
    for k in range(6):
        cases.append(dict(name=f"sparse{k}", reads=make_reads(rng, rng.randrange(20, 120), 1000, max_len=25), params=DEFAULT))
    for k in range(8):
        cases.append(dict(name=f"unsorted{k}", reads=make_reads(rng, rng.randrange(20, 80), rng.choice([1, 10]), sort=False),
                          params=DEFAULT))
        cases.append(dict(name=f"shuffled{k}", reads=make_reads(rng, rng.randrange(20, 80), 1, shuffle=0.2), params=DEFAULT))
    for k in range(6):
        cases.append(dict(name=f"repeats{k}", reads=make_reads(rng, 60, 1, repeats=0.3, qualities=(-5, 6)), params=DEFAULT))
        cases.append(dict(name=f"ties{k}", reads=make_reads(rng, 60, 1, error=0.02, qualities=(1, 2)), params=[0.15, 0.25, 100, 10]))
    for k in range(3):
        cases.append(dict(name=f"single{k}", reads=make_reads(rng, 80, 1, max_len=1, span=20), params=[0.15, 0.25, 2, 1]))
        cases.append(dict(name=f"long{k}", reads=make_reads(rng, 40, 1, max_len=300, span=200, error=0.03), params=DEFAULT))
    cases.append(dict(name="many", reads=make_reads(rng, 4000, 1, span=3000, max_len=60), params=DEFAULT))
    cases.append(dict(name="many_sparse", reads=make_reads(rng, 3000, 1000, span=3000, max_len=20), params=DEFAULT))
    # not-blue edges: e of 0.8 or 0.9, or thresholds below 1, drive the removal loop
    for k, params in enumerate([[0.8, 0.9, 1000, 1000], [0.9, 0.5, 100, 1000], [0.8, 0.3, 1000, 10], [0.15, 0.25, 0.5, 0.01],
                                [0.15, 0.6, 0.01, 0.001], [0.8, 0.9, 1e6, 1e6]]):
        for m in range(3):
            cases.append(dict(name=f"removal{k}_{m}", reads=make_reads(rng, rng.randrange(10, 40), 1, max_len=12, span=8,
                                                                        sort=m != 2), params=params))
    # errors: the first offending read decides
    base = make_reads(rng, 12, 1)
    for name, edit in (("empty", {5: []}), ("allele2", {3: "2"}), ("allele_minus1", {4: "-1"}), ("allele_then_empty", {2: "2", 6: []}),
                       ("empty_then_allele", {2: [], 6: "-1"})):
        reads = [list(map(list, r)) for r in base]
        for i, e in edit.items():
            if isinstance(e, list):
                reads[i] = []
            else:
                reads[i][len(reads[i]) // 2][1] = int(e)
        cases.append(dict(name=name, reads=reads, params=DEFAULT))
    for name, params in (("e0", [0, 0.25, 1000000, 1000]), ("e075", [0.75, 0.25, 1000000, 1000]), ("e1", [1, 0.25, 1000000, 1000]),
                         ("thr0", [0.15, 0.25, 0, 1000]), ("thr_neg_minus1", [0.15, 0.25, 1000000, -1])):
        cases.append(dict(name=name, reads=base, params=params))
    return cases


def answer(merged_reads):
    """The stored form of a merged ReadSet (any module's)."""
    return [[r.name, [[int(v.position), int(v.allele), int(v.quality)] for v in r]] for r in merged_reads]


def run(merger, case, read_cls, readset_cls):
    """The answer of `merger` (a ReadMerger class) on the case, built from `read_cls` / `readset_cls`."""
    try:
        rs = readset_cls()
        for k, read in enumerate(case["reads"]):
            r = read_cls(f"r{k}", 60, 0, 0)
            for p, a, q in read:
                r.add_variant(p, a, q)
            rs.add(r)
        return answer(merger(*case["params"]).merge(rs))
    except (IndexError, AssertionError, ValueError, ZeroDivisionError) as e:
        return type(e).__name__


def run_oracle(case):
    try:
        return [[name, [list(e) for e in entries]] for name, entries in merge_oracle.merge([[tuple(e) for e in r] for r in case["reads"]],
                                                                                           *case["params"])]
    except (IndexError, AssertionError, ValueError, ZeroDivisionError) as e:
        return type(e).__name__
