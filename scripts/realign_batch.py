"""Allele detection by re-alignment (`realign.detect_alleles`, DESIGN §4.11) on a seeded synthetic chromosome, and how it compares
with the steps around it.

Input: a random chromosome of --mb Mb, variants about every 300 bp (SNVs, insertions, deletions, multiallelic sites), reads from
two haplotypes: 30x of 15 kb reads and 30x of 150 bp reads, each with about 5 % errors (substitutions and 1-3 base indels).
Reported, as medians over --rounds:
  - items (alignment x covered variant) and allele alignments, in unit-cost and affine mode;
  - the device time of the kernels and the end-to-end time of detect_alleles (Python packing of the alignments included);
  - the reference's compiled whatshap.align.edit_distance called once per allele alignment in a Python loop, timed on a
    sample of the call's own (query window, padded allele) pairs and scaled to all of them: a lower bound on the reference's
    realignment, which also walks the CIGARs and cuts the windows in Python (only where oracle/_ref/pyref holds the binary);
  - PedigreeDPTable on the resulting ReadSet of one individual after read selection to coverage 15.
The card's name, power limit and SM clock limit are read in the same run.  Writes JSON to --out.

    python scripts/realign_batch.py --mb 2 --out realign_batch.json
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from whatshap_b200 import NumericSampleIds, Pedigree, PedigreeDPTable, Read, ReadSet, realign  # noqa: E402
from whatshap_b200.readselect import readselection  # noqa: E402
from whatshap_b200.testhelpers import canonic_index_to_biallelic_gt  # noqa: E402

BASES = np.frombuffer(b"ACGT", np.uint8)


class Aln:
    __slots__ = ("reference_start", "cigartuples", "query_sequence")

    def __init__(self, start, cigar, seq):
        self.reference_start, self.cigartuples, self.query_sequence = start, cigar, seq


class Var:
    __slots__ = ("position", "reference_allele", "alts")

    def __init__(self, position, ref, alts):
        self.position, self.reference_allele, self.alts = position, ref, alts

    def get_alt_allele_list(self):
        return self.alts


def synthetic(mb: float, seed: int = 1, long_cov: int = 30, short_cov: int = 30, err: float = 0.05):
    """(reference, variants, alignments)."""
    rng = np.random.default_rng(seed)
    n = int(mb * 1e6)
    ref_arr = BASES[rng.integers(0, 4, n)]
    reference = ref_arr.tobytes().decode()
    variants = []
    pos = int(rng.integers(50, 300))
    while pos < n - 200:
        r = reference[pos]
        k = rng.random()
        if k < 0.7:
            alts = [("ACGT".replace(r, ""))[rng.integers(0, 3)]]
        elif k < 0.82:
            alts = [r + BASES[rng.integers(0, 4, int(rng.integers(1, 12)))].tobytes().decode()]
        elif k < 0.94:
            d = int(rng.integers(1, 12))
            r, alts = reference[pos:pos + d + 1], [reference[pos]]
        else:
            alts = [("ACGT".replace(r, ""))[rng.integers(0, 3)], r + "TG"]
        variants.append(Var(pos, r, alts))
        pos += int(rng.integers(150, 450))
    vpos = np.array([v.position for v in variants])
    # two haplotypes: per variant an allele each (0 = reference)
    hap = [rng.integers(0, 1 + np.array([len(v.alts) for v in variants])) for _ in range(2)]

    def read(start, length, h):
        cigar, seq = [], []
        p, end = start, min(n, start + length)
        lo, hi = np.searchsorted(vpos, start), np.searchsorted(vpos, end)
        events = sorted(set(rng.integers(start, end, int(length * err * 0.4)).tolist()))  # indel errors
        ev = {e: int(rng.integers(1, 4)) * (1 if rng.random() < 0.5 else -1) for e in events}
        stops = sorted(set([int(vpos[i]) for i in range(lo, hi)] + list(ev)))

        def match(upto):
            nonlocal p
            if upto > p:
                s = bytearray(ref_arr[p:upto].tobytes())
                for i in np.nonzero(rng.random(upto - p) < err * 0.6)[0]:
                    s[i] = BASES[rng.integers(0, 4)]
                seq.append(s.decode())
                if cigar and cigar[-1][0] == 0:
                    cigar[-1] = (0, cigar[-1][1] + upto - p)
                else:
                    cigar.append((0, upto - p))
                p = upto

        vi = lo
        for s in stops:
            if s < p or s >= end:
                continue
            match(s)
            while vi < hi and vpos[vi] < s:
                vi += 1
            if vi < hi and vpos[vi] == s:
                v = variants[vi]
                a = hap[h][vi]
                if a:
                    alt = v.alts[a - 1]
                    if len(alt) == len(v.reference_allele) == 1:
                        seq.append(alt), cigar.append((0, 1))
                        p += 1
                    elif len(alt) > 1:
                        seq.append(alt[0]), cigar.append((0, 1)), seq.append(alt[1:]), cigar.append((1, len(alt) - 1))
                        p += 1
                    else:
                        seq.append(alt), cigar.append((0, 1)), cigar.append((2, len(v.reference_allele) - 1))
                        p += len(v.reference_allele)
                continue
            d = ev.get(s, 0)
            if d > 0:
                seq.append(BASES[rng.integers(0, 4, d)].tobytes().decode()), cigar.append((1, d))
            elif d < 0 and p - d < end:
                cigar.append((2, -d))
                p -= d
        match(end)
        merged = []
        for op, k in cigar:
            if merged and merged[-1][0] == op:
                merged[-1] = (op, merged[-1][1] + k)
            else:
                merged.append((op, k))
        return Aln(start, merged, "".join(seq))

    alns = []
    for length, cov in ((15000, long_cov), (150, short_cov)):
        for start in np.sort(rng.integers(0, n - length, int(cov * n / length))):
            alns.append(read(int(start), length, int(rng.integers(0, 2))))
    alns.sort(key=lambda a: a.reference_start)
    return reference, variants, alns


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sample", type=int, default=20000)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    t = time.perf_counter()
    reference, variants, alns = synthetic(args.mb)
    res = {"card": card(), "mb": args.mb, "variants": len(variants), "alignments": len(alns), "generate_s": time.perf_counter() - t}
    print(json.dumps(res), flush=True)
    modes = {"unit": dict(), "affine": dict(affine=True, gap_start=10, gap_extend=7, default_mismatch=15)}
    calls = None
    for name, kw in modes.items():
        realign.detect_alleles(alns[:100], variants, reference, **kw)  # warm-up
        dev, e2e = [], []
        for _ in range(args.rounds):
            st = {}
            t = time.perf_counter()
            got = realign.detect_alleles(alns, variants, reference, stats=st, **kw)
            e2e.append(time.perf_counter() - t)
            dev.append(st["device_ms"])
        calls = calls or got
        res[name] = {"items": st["items"], "jobs": st["jobs"], "long_jobs": st["long_jobs"], "chunks": st["chunks"], "plan_ms": st["plan_ms"],
                     "device_ms": statistics.median(dev), "end_to_end_s": statistics.median(e2e),
                     "calls": sum(len(g) for g in got)}
        print(json.dumps({name: res[name]}), flush=True)
    # the reference's edit_distance per allele alignment, on a sample of this call's own pairs
    pyref = os.path.join(ROOT, "oracle", "_ref", "pyref")
    try:
        sys.path.insert(0, pyref)
        from whatshap import align
    except ImportError:
        align = None
    if align is not None:
        rng = random.Random(3)
        pairs = []
        while len(pairs) < args.sample:
            a = alns[rng.randrange(len(alns))]
            if not a.cigartuples:
                continue
            lo = a.reference_start
            k = rng.randrange(len(variants))
            v = variants[k]
            if not (lo <= v.position < lo + len(a.query_sequence) - 30):
                continue
            off = v.position - lo
            q = a.query_sequence[max(0, off - 10):off + len(v.reference_allele) + 10]
            left, right = reference[v.position - 10:v.position], reference[v.position + len(v.reference_allele):v.position + len(v.reference_allele) + 10]
            pairs.append((q, left + v.reference_allele + right))
            for alt in v.alts:
                pairs.append((q, left + alt + right))
        t = time.perf_counter()
        for q, s in pairs:
            align.edit_distance(q, s)
        per_call = (time.perf_counter() - t) / len(pairs)
        res["reference_edit_distance_loop_s"] = per_call * res["unit"]["jobs"]
        res["reference_edit_distance_per_call_us"] = per_call * 1e6
    # PedigreeDPTable on the ReadSet of the unit-cost calls, one individual, after read selection to coverage 15
    t = time.perf_counter()
    rs = ReadSet()
    for k, g in enumerate(calls):
        if len(g) < 2:
            continue
        r = Read(f"r{k}", 60, 0, 0)
        for vi, allele, q in g:
            r.add_variant(variants[vi].position, allele, q)
        rs.add(r)
    rs.sort()
    selected = readselection(rs, 15)
    sub = rs.subset(sorted(selected))
    positions = sub.get_positions()
    res["readset_build_s"] = time.perf_counter() - t
    ped = Pedigree(NumericSampleIds())
    ped.add_individual("individual0", [canonic_index_to_biallelic_gt(1)] * len(positions))
    PedigreeDPTable(sub, [1] * len(positions), ped)  # warm-up
    dp = []
    for _ in range(args.rounds):
        t = time.perf_counter()
        table = PedigreeDPTable(sub, [1] * len(positions), ped)
        table.get_optimal_cost()
        dp.append(time.perf_counter() - t)
    res["pedigree_dp_s"] = statistics.median(dp)
    res["pedigree_dp_reads"], res["pedigree_dp_columns"] = len(sub), len(positions)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
