"""Allele detection from the CIGAR alone (`realign.detect_alleles(..., reference=None)`, DESIGN §4.14) on the seeded synthetic
chromosome of realign_batch.py, with base qualities.

Reported, as medians over --rounds: items (enqueued variants) and calls; the device time of the kernels (CUDA events); the host
preparation in the library (normalization, conflict filter, allele targets, operation checks, chunk cut); the Python packing of the
alignment objects; and detect_alleles end to end.  The card's name, power limit and SM clock limit are read in the same run.

With --cpu-only (on a machine with the reference's sources, no GPU needed) it instead times the reference's compiled _detect_alleles
on --sample alignments of the same input, in a Python loop as _alignments_to_reads calls it.  The stub alignments hold plain str
sequences and lists of qualities, so the per-access decoding of a pysam.AlignedSegment is not paid: the figure is a lower bound.

    python scripts/cigar_alleles_batch.py --mb 2 --out cigar_alleles_batch.json
    python scripts/cigar_alleles_batch.py --mb 2 --cpu-only --sample 20000
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.realign_batch import card, synthetic  # noqa: E402
from whatshap_b200 import realign  # noqa: E402


class QAln:
    __slots__ = ("reference_start", "cigartuples", "query_sequence", "query_qualities")

    def __init__(self, start, cigar, seq, quals):
        self.reference_start, self.cigartuples, self.query_sequence, self.query_qualities = start, cigar, seq, quals


def with_qualities(alns, seed=1):
    """The alignments with random base qualities 5..59 (as bytes, what a packer hands over from pysam's array)."""
    rng = np.random.default_rng(seed)
    return [QAln(a.reference_start, a.cigartuples, a.query_sequence, rng.integers(5, 60, len(a.query_sequence), dtype=np.uint8).tobytes())
            for a in alns]


def cpu_reference(variants, alns, sample):
    """Seconds per alignment of the reference's compiled _detect_alleles on the first `sample` alignments."""
    from oracle import build_pyref

    path = build_pyref.build()
    if not path:
        raise SystemExit("the reference tree is not available")
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_realign_golden import _StubFinder

    sys.meta_path.insert(0, _StubFinder())
    sys.path.insert(0, path)
    from whatshap._variants import _detect_alleles
    from whatshap.variants import ReadSetReader
    from whatshap.vcf import BiallelicVcfVariant, MultiallelicVcfVariant

    vs = [BiallelicVcfVariant(v.position, v.reference_allele, v.alts[0]) if len(v.alts) == 1 else
          MultiallelicVcfVariant(v.position, v.reference_allele, v.alts) for v in variants]
    t0 = time.perf_counter()
    normalized = [v.normalized() for v in vs]
    valid = ReadSetReader.detect_non_overlapping_variants(None, normalized)
    vp = [ReadSetReader.build_var_progress(None, normalized, j) for j in valid]
    prep = time.perf_counter() - t0
    stubs = [QAln(a.reference_start, a.cigartuples, a.query_sequence, list(a.query_qualities)) for a in alns[:sample]]
    t0 = time.perf_counter()
    calls = sum(len(list(_detect_alleles(normalized, vp, 0, a))) for a in stubs)
    return prep, (time.perf_counter() - t0) / len(stubs), calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--cpu-only", action="store_true")
    ap.add_argument("--sample", type=int, default=20000)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    reference, variants, alns = synthetic(args.mb)
    alns = with_qualities(alns)
    res = {"mb": args.mb, "alignments": len(alns), "variants": len(variants)}
    if args.cpu_only:
        prep, per, calls = cpu_reference(variants, alns, min(args.sample, len(alns)))
        res.update(reference_prep_s=prep, reference_s_per_alignment=per, reference_sample=min(args.sample, len(alns)),
                   reference_sample_calls=calls, reference_all_s_estimate=per * len(alns))
    else:
        res["card"] = card()
        realign.detect_alleles(alns[:2000], variants, None)  # loads the module and the page-locked staging memory
        rows = []
        for _ in range(args.rounds):
            t0 = time.perf_counter()
            realign.pack_cigar_input(alns, variants)
            pack = time.perf_counter() - t0
            st = {}
            t0 = time.perf_counter()
            got = realign.detect_alleles(alns, variants, None, stats=st)
            rows.append(dict(end_to_end_s=time.perf_counter() - t0, pack_s=pack, device_ms=st["device_ms"], plan_ms=st["plan_ms"],
                             items=st["items"], jobs=st["jobs"], calls=sum(map(len, got)), chunks=st["chunks"],
                             launches=st["kernel_launches"]))
            print(json.dumps(rows[-1]), flush=True)
        res.update({k: statistics.median(r[k] for r in rows) for k in rows[0]})
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
