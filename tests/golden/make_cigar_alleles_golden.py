"""Regenerates tests/golden/cigar_alleles.npz: the reference's own allele detection without a reference (whatshap/_variants.pyx
_detect_alleles, compiled by oracle/build_pyref.build(), with VcfVariant.normalized, detect_non_overlapping_variants and
build_var_progress of whatshap/vcf.py and whatshap/variants.py) on seeded cases.  Needs the WhatsHap source tree at $WHATSHAP_REF;
pysam, pyfaidx and xopen are stubbed as in make_realign_golden.py.

    python tests/golden/make_cigar_alleles_golden.py

Each case holds the variants (position, REF, ALTs) and the alignments (reference_start, cigartuples, query_sequence,
query_qualities, each of the last three possibly None), and per alignment either the list of (variant index, allele, quality) of
_detect_alleles(normalized, var_progress, 0, alignment) or the name of the exception it raised; `raises` names the exception of
the preparation (a variant without alternatives), which fails the whole call.  Cases with `running` were also run through the
reference's ReadSetReader._alignments_to_reads, whose reads (position, allele, quality) are stored per alignment in `reads`."""
import json
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_realign_golden import _StubFinder, make_read, make_variants, rand_seq  # noqa: E402

sys.path.insert(0, os.path.dirname(HERE))


class Aln:
    def __init__(self, start, cigar, seq, quals=None):
        self.reference_start, self.cigartuples, self.query_sequence, self.query_qualities = start, cigar, seq, quals


def with_quals(rng, aln, kind):
    """kind 0: qualities present, 1: None, 2: empty."""
    if kind == 0 and aln.query_sequence is not None:
        aln.query_qualities = [rng.randrange(0, 60) for _ in aln.query_sequence]
    elif kind == 2:
        aln.query_qualities = []
    return aln


def build_cases():
    rng = random.Random(20261019)
    cases = []

    def case(name, variants, alns, running=False):
        cases.append(dict(name=name, variants=[[p, r, list(a)] for p, r, a in variants],
                          alignments=[[a.reference_start, None if a.cigartuples is None else [list(x) for x in a.cigartuples],
                                       a.query_sequence, None if a.query_qualities is None else list(a.query_qualities)] for a in alns],
                          running=running))

    for k in range(12):
        n = rng.choice([400, 1500, 4000]) if k not in (5, 11) else 30000
        ref = rand_seq(rng, n)
        long_ins = {rng.randrange(50, n - 50): 80} if k % 3 == 0 else {}
        if k in (5, 11):
            long_ins[rng.randrange(50, n - 50)] = 1100
        variants = make_variants(rng, ref, rng.choice([15, 40, 100]), long_ins)
        alns = []
        for i in range(rng.choice([10, 30]) if n < 30000 else 12):
            length = rng.choice([60, 150, 600, 1500]) if n < 30000 else 15000
            start = rng.randrange(0, max(1, n - length // 2))
            alns.append(with_quals(rng, make_read(rng, ref, variants, start, length), i % 3))
        alns.append(Aln(rng.randrange(0, n), [], ""))  # empty CIGAR
        if k % 4 == 1:
            alns.sort(key=lambda a: a.reference_start)
        case(f"random{k}", variants, alns, running=k % 4 == 1)

    # hand-made cases: every rule of the op loop and the handlers
    ref = rand_seq(rng, 300)
    b = lambda i: ref[i]  # noqa: E731
    other = lambda c: "A" if c != "A" else "C"  # noqa: E731
    variants = [
        (20, b(20), [b(20) + "GT"]),                      # insertion after a match base: normalizes to an insertion at 21
        (30, b(30), [other(b(30)), b(30) + "TT"]),        # multiallelic: SNV and insertion
        (40, ref[40:44], [b(40)]),                        # deletion, normalizes to 41
        (41, b(41), [other(b(41))]),                      # inside that deletion: conflicting with it
        (60, ref[60:62], [ref[60:62]]),                   # REF == ALT: both alleles empty after normalization
        (70, b(70), ["<DEL>"]),                           # symbolic
        (80, ref[80:83], [ref[80] + "G" + ref[82], ref[80:83] + "A"]),  # normalizes to 81 (MNV-like) and to an insertion at 83
        (80, b(80), [other(b(80))]),                      # duplicate original position
        (100, ref[100:103], [b(100), ref[100:102]]),     # two deletions of different lengths
        (102, b(102), [other(b(102))]),                   # overlaps the deletion at 100
        (150, b(150), [b(150) + "ACGTACGT"]),             # an insertion read through an I operation
        (151, b(151), [other(b(151))]),                   # a SNV right after it
        (200, ref[200:202] + "A", [ref[200:202]]),        # a deletion whose normalized position precedes the next
        (201, b(201), [other(b(201))]),
    ]
    ins = "GT"
    mk = lambda start, cigar, seq: Aln(start, cigar, seq)  # noqa: E731
    alns = [
        mk(10, [(0, 11), (1, 2), (0, 40)], ref[10:21] + ins + ref[21:61]),                 # insertion variant under I
        mk(10, [(0, 11), (1, 3), (0, 40)], ref[10:21] + "GTC" + ref[21:61]),              # longer insertion than the variant
        mk(25, [(0, 5), (1, 2), (0, 30)], ref[25:30] + "TT" + ref[30:60]),                 # an I op at a non-insertion variant
        mk(15, [(0, 6), (2, 3), (0, 30)], ref[15:21] + ref[24:54]),                        # D over the insertion variant at 21
        mk(35, [(0, 6), (2, 3), (0, 30)], ref[35:41] + ref[44:74]),                        # the deletion at 41
        mk(5, [(5, 3), (4, 4), (0, 30), (3, 20), (0, 30), (6, 2), (4, 3)], "NNNN" + ref[5:35] + ref[55:85] + "NNN"),  # H, S, N, P
        mk(55, [(7, 10), (8, 1), (7, 20)], ref[55:65] + other(b(65)) + ref[66:86]),        # = and X
        mk(95, [(0, 5), (2, 2), (0, 20)], ref[95:100] + ref[102:122]),                     # the shorter deletion at 100
        mk(95, [(0, 5), (2, 1), (0, 20)], ref[95:100] + ref[101:121]),
        mk(140, [(0, 11), (1, 8), (0, 30)], ref[140:151] + "ACGTACGT" + ref[151:181]),     # insertion read through, then a SNV
        mk(140, [(0, 11), (1, 4), (0, 30)], ref[140:151] + "ACGT" + ref[151:181]),         # a partial insertion
        mk(140, [(0, 11), (1, 8), (0, 30)], ref[140:151] + "ACGAACGT" + ref[151:181]),     # a mismatching insertion
        mk(190, [(0, 40)], ref[190:230]),                                                  # unsorted normalized positions
        mk(195, [(0, 10), (2, 1), (0, 20)], ref[195:205] + ref[206:226]),
        mk(80, [(0, 10)], ref[80:90]),
        mk(81, [(0, 2), (1, 1), (0, 10)], ref[81:83] + "A" + ref[83:93]),
        mk(75, [], ""),                                                                    # empty CIGAR
    ]
    for i, a in enumerate(alns):
        with_quals(rng, a, i % 3)
    case("rules", variants, alns)
    # variants whose normalized positions are out of order and share positions
    v2 = [(50, "ACGT", ["AC"]), (51, "C", ["G"]), (52, "GT", ["G"]), (49, "TA", ["TAC"]), (53, "T", ["A", "TT"]), (53, "TG", ["T"])]
    ref2 = ref[:49] + "TACGTGA" + ref[56:]
    alns2 = [with_quals(rng, mk(40, [(0, 30)], ref2[40:70]), 0), with_quals(rng, mk(45, [(0, 5), (1, 1), (0, 3), (2, 1), (0, 20)], ref2[45:50] + "C" + ref2[50:53] + ref2[54:74]), 1),
             with_quals(rng, mk(48, [(0, 3), (2, 2), (0, 20)], ref2[48:51] + ref2[53:73]), 2)]
    case("unsorted_normalized", v2, alns2)
    # raising alignments, one per kind, between good ones
    v3 = [(50, b(50), [other(b(50))]), (100, ref[100:104], [b(100)]), (150, b(150), [b(150) + "TT"]), (48, b(48), [other(b(48))])]
    good = with_quals(rng, mk(30, [(0, 40)], ref[30:70]), 0)
    raising = [
        good,
        mk(40, [(0, 20), (9, 3), (0, 20)], ref[40:80]),                                   # unknown op: ValueError
        mk(40, [(0, 20)], ref[40:50]),                                                     # sequence too short: IndexError
        Aln(40, [(0, 20)], ref[40:60], [30] * 5),                                          # qualities too short: IndexError
        Aln(40, [(0, 20)], None),                                                          # no sequence: TypeError
        Aln(40, None, ref[40:60]),                                                         # no CIGAR: TypeError
        Aln(40, [(0, 5), (9, 1)], None),                                                   # no sequence, unknown op before any base
        mk(45, [(0, 20), (1, 500)], ref[45:65]),                                           # an I past the sequence after the variant
        mk(140, [(0, 20), (1, 2), (0, 10), (8, 1)], ref[140:170]),                        # insertion base past the end
        with_quals(rng, mk(45, [(0, 3), (7, 30)], ref[45:78]), 0),
        mk(60, [(0, 10), (42, 2)], ref[60:70]),                                            # unknown op without a covered variant
        good,
    ]
    case("raising", v3, raising)
    case("raising_unsorted", [(50, b(50), [other(b(50))]), (30, b(30), [other(b(30))])], [mk(45, [(0, 20)], ref[45:65]), mk(45, [(0, 20)], "A")])
    # a variant without alternatives: the preparation raises, unless the conflict filter passes over it
    case("no_alts", [(10, "A", []), (20, b(20), [other(b(20))])], [mk(5, [(0, 30)], ref[5:35])])
    case("no_alts_duplicate", [(10, b(10), [other(b(10))]), (10, "A", []), (12, ref[12:15], [b(12)]), (13, "C", [])],
         [with_quals(rng, mk(5, [(0, 30)], ref[5:35]), 0)])
    return cases


def run_reference(cases):
    from oracle import build_pyref

    path = build_pyref.build()
    if not path:
        raise SystemExit("the reference tree is not available")
    sys.meta_path.insert(0, _StubFinder())
    sys.path.insert(0, path)
    from whatshap._variants import _detect_alleles
    from whatshap.variants import ReadSetReader
    from whatshap.vcf import BiallelicVcfVariant, MultiallelicVcfVariant

    for c in cases:
        variants = [BiallelicVcfVariant(p, r, a[0]) if len(a) == 1 else MultiallelicVcfVariant(p, r, a) for p, r, a in c["variants"]]
        c.pop("raises", None)
        try:
            normalized = [v.normalized() for v in variants]
            valid = ReadSetReader.detect_non_overlapping_variants(None, normalized)
        except Exception as e:  # noqa: BLE001 - recorded as the expected outcome
            c["raises"] = type(e).__name__
            c["want"] = None
            continue
        alns = [Aln(*a) for a in c["alignments"]]
        want = []
        for aln in alns:
            var_progress = [ReadSetReader.build_var_progress(None, normalized, j) for j in valid]
            try:
                want.append([[int(i), int(a), int(q)] for i, a, q in _detect_alleles(normalized, var_progress, 0, aln)])
            except Exception as e:  # noqa: BLE001 - recorded as the expected outcome
                want.append(type(e).__name__)
        c["want"] = want
        if c["running"]:
            c["reads"] = run_alignments_to_reads(ReadSetReader, variants, alns)
    return cases


class _Bam:
    """What _alignments_to_reads reads from a pysam.AlignedSegment."""

    def __init__(self, k, aln):
        self.query_name, self.mapq, self.reference_name, self.flag = f"read{k}", 60, "chr1", 0
        self.reference_start, self.cigartuples = aln.reference_start, aln.cigartuples
        self.query_sequence, self.query_qualities = aln.query_sequence, aln.query_qualities
        self.reference_end = aln.reference_start + sum(n for op, n in aln.cigartuples if op in (0, 2, 3, 7, 8))
        self.is_supplementary = self.is_reverse = self.is_secondary = self.is_unmapped = False
        self.cigarstring = "".join(f"{n}{'MIDNSHP=X'[op]}" for op, n in aln.cigartuples)

    def has_tag(self, tag):
        return False


class _Wrapped:
    def __init__(self, k, aln):
        self.bam_alignment, self.source_id = _Bam(k, aln), 0


def run_alignments_to_reads(ReadSetReader, variants, alns):
    """Per alignment, the (position, allele, quality) of the read the reference's _alignments_to_reads yields for it (with its
    running index), or [] where it yields none."""
    reader = ReadSetReader.__new__(ReadSetReader)
    reader._numeric_sample_ids = {}
    reader._use_kmerald = False
    wrapped = [_Wrapped(k, a) for k, a in enumerate(alns)]
    out = {}
    for aligned in reader._alignments_to_reads(wrapped, variants, None, None, None):
        k = int(aligned.read.name[4:])
        out[k] = [[int(v.position), int(v.allele), int(v.quality)] for v in aligned.read]
    return [out.get(k, []) for k in range(len(alns))]


if __name__ == "__main__":
    cases = run_reference(build_cases())
    np.savez_compressed(os.path.join(HERE, "cigar_alleles.npz"), cases=np.frombuffer(json.dumps(cases).encode(), np.uint8))
    calls = sum(len(w) for c in cases if c["want"] for w in c["want"] if isinstance(w, list))
    errors = sum(1 for c in cases if c["want"] for w in c["want"] if isinstance(w, str))
    print(f"{len(cases)} cases, {sum(len(c['alignments']) for c in cases)} alignments, {calls} calls, {errors} raising alignments, "
          f"{sum(1 for c in cases if 'raises' in c)} raising preparations")
