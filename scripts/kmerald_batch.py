"""Allele detection by k-mer re-alignment (`realign.detect_alleles(use_kmerald=True)`, DESIGN §4.12) on the seeded synthetic
chromosome of scripts/realign_batch.py, with a seeded costs table.

Input: the chromosome, variants and reads of realign_batch.synthetic(--mb) (every variant biallelic: its first alternative
allele), and a costs table for k = --k with a default (a, -5) for every k-mer a and --per-kmer random (a, b) entries each
(16383 x 64 = 1 M entries for k = 7).  Reported, as medians over --rounds:
  - items and allele alignments, one-thread and warp jobs, chunks;
  - the device time of the kernels and the end-to-end time of detect_alleles (Python packing of the alignments included),
    the costs table packed once beforehand (its packing time is reported apart);
  - where oracle/_ref/pyref holds the reference's compiled whatshap.align: its kmer_align per call, timed on a sample of
    (padded allele, query window) k-mer lists of this workload with the same costs, scaled to all allele alignments.
The card's name, power limit and SM clock limit are read in the same run.  Writes JSON to --out.

    python scripts/kmerald_batch.py --mb 2 --out kmerald_batch.json
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.realign_batch import card, synthetic  # noqa: E402
from whatshap_b200 import realign  # noqa: E402


class Variant:
    __slots__ = ("position", "reference_allele", "alternative_allele")

    def __init__(self, position, ref, alt):
        self.position, self.reference_allele, self.alternative_allele = position, ref, alt

    def get_alt_allele_list(self):
        return [self.alternative_allele]


def workload(mb: float, seed: int = 1):
    reference, variants, alns = synthetic(mb, seed=seed)
    return reference, [Variant(v.position, v.reference_allele, v.alts[0]) for v in variants], alns


def costs_table(k: int, per_kmer: int, seed: int = 2) -> dict:
    """{(a, b): cost string}: a default for every k-mer a and per_kmer random read k-mers b."""
    rng = np.random.default_rng(seed)
    n = 4 ** k - 1
    a = np.repeat(np.arange(1, n + 1), per_kmer)
    b = rng.integers(1, n + 1, a.size)
    v = np.round(rng.uniform(0, 40, a.size), 3)
    d = {(int(x), int(y)): f"{z:.3f}" for x, y, z in zip(a.tolist(), b.tolist(), v.tolist())}
    for x in range(1, n + 1):
        d[(x, -5)] = "45.0"
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=2.0)
    ap.add_argument("--k", type=int, default=7)
    ap.add_argument("--per-kmer", type=int, default=64)
    ap.add_argument("--gap", type=float, default=40)
    ap.add_argument("--window", type=int, default=25)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sample", type=int, default=300)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    t = time.perf_counter()
    reference, variants, alns = workload(args.mb)
    mapping = costs_table(args.k, args.per_kmer)
    res = {"card": card(), "mb": args.mb, "k": args.k, "gap": args.gap, "window": args.window, "variants": len(variants),
           "alignments": len(alns), "cost_entries": len(mapping), "generate_s": time.perf_counter() - t}
    t = time.perf_counter()
    costs = realign.KmerCosts(mapping)
    res["costs_pack_s"] = time.perf_counter() - t
    print(json.dumps(res), flush=True)
    kw = dict(use_kmerald=True, kmerald_costs=costs, kmer_size=args.k, kmerald_gappenalty=args.gap, kmerald_window=args.window)
    realign.detect_alleles(alns[:100], variants, reference, **kw)  # warm-up
    dev, e2e = [], []
    for _ in range(args.rounds):
        st = {}
        t = time.perf_counter()
        got = realign.detect_alleles(alns, variants, reference, stats=st, **kw)
        e2e.append(time.perf_counter() - t)
        dev.append(st["device_ms"])
    res["kmerald"] = {"items": st["items"], "jobs": st["jobs"], "short_jobs": st["short_jobs"], "long_jobs": st["long_jobs"],
                      "chunks": st["chunks"], "plan_ms": st["plan_ms"], "device_ms": statistics.median(dev),
                      "end_to_end_s": statistics.median(e2e), "calls": sum(len(g) for g in got)}
    print(json.dumps({"kmerald": res["kmerald"]}), flush=True)
    pyref = os.path.join(ROOT, "oracle", "_ref", "pyref")
    try:
        sys.path.insert(0, pyref)
        from whatshap.align import enumerate_all_kmers, kmer_align
    except ImportError:
        kmer_align = None
    if kmer_align is not None:
        rng = random.Random(3)
        pairs = []
        w = args.window
        while len(pairs) < args.sample:
            a = alns[rng.randrange(len(alns))]
            if not a.cigartuples:
                continue
            v = variants[rng.randrange(len(variants))]
            if not (a.reference_start + w <= v.position < a.reference_start + len(a.query_sequence) - 2 * w):
                continue
            off = v.position - a.reference_start
            q = a.query_sequence[off - w:off + len(v.reference_allele) + w]
            left, right = reference[v.position - w:v.position], reference[v.position + len(v.reference_allele):v.position + len(v.reference_allele) + w]
            qk = enumerate_all_kmers(q.encode(), args.k)
            for allele in (v.reference_allele, v.alternative_allele):
                pairs.append((enumerate_all_kmers((left + allele + right).encode(), args.k), qk))
        t = time.perf_counter()
        for x, y in pairs:
            kmer_align(x, y, mapping, args.gap)
        per_call = (time.perf_counter() - t) / len(pairs)
        res["reference_kmer_align_per_call_us"] = per_call * 1e6
        res["reference_kmer_align_loop_s"] = per_call * res["kmerald"]["jobs"]
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
