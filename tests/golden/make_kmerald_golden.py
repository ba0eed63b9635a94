"""Regenerates tests/golden/kmerald.npz: the reference's own ReadSetReader.detect_alleles_by_alignment(use_kmerald=True),
kmer_align and enumerate_all_kmers (whatshap/variants.py and whatshap/align.pyx, compiled by oracle/build_pyref.build()) on
seeded cases.  Needs the WhatsHap source tree at $WHATSHAP_REF; the modules variants.py imports but the call never uses are
stubbed as in make_realign_golden.py.

    python tests/golden/make_kmerald_golden.py

Stored (UTF-8 JSON as the uint8 array `cases`):
  - `detect`: per case the reference, the variants (position, ref, alts; one alt: BiallelicVcfVariant, several:
    MultiallelicVcfVariant), the alignments, the restricted genotypes (or none), k, gap, window, the costs as
    [ref k-mer, read k-mer, value string] rows (a file's rows: repeated keys, the last one kept), and per alignment either the
    list of (variant index, allele, quality) or the exception the reference raised for it;
  - `enumerate`: (string, k, the k-mer list);
  - `pairs`: per table, (s1, s2, repr of kmer_align's float32 value) for kmer_align(enum(s1, k), enum(s2, k), costs, gap)."""
import json
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from make_realign_golden import Aln, Gt, _StubFinder, make_read, make_variants, rand_seq  # noqa: E402


def kmers_of(s, k):
    """enumerate_all_kmers restated (only to pick cost keys that the cases look up; the stored answers are the reference's)."""
    mask, h, out = (1 << 2 * k) - 1, 0, []
    for i, c in enumerate(s):
        if c in "ACGT":
            h = ((h << 2) | "ACGT".index(c)) & mask
        if i >= k - 1 and h:
            out.append(h)
    return out


def padded_alleles(ref, variants, w):
    """Every allele of every variant padded with w reference bases on each side: the strings whose k-mers the DP rows look up."""
    out = []
    for p, r, alts in variants:
        left, right = ref[max(0, p - w):p], ref[p + len(r):p + len(r) + w]
        out += [left + a + right for a in [r] + alts]
    return out


def make_costs(rng, strings, k, default_share=0.9, pair_share=0.6, nan=False, dup=True):
    """Rows [a, b, value]: a default (a, -5) for most ref k-mers, specific (a, b) for k-mers one substitution apart, repeated
    keys with differing values, an `inf`, maybe a `nan`."""
    present = sorted({x for s in strings for x in kmers_of(s, k)})
    rows = []
    for a in present:
        if rng.random() < default_share:
            rows.append([a, -5, f"{rng.uniform(5, 60):.2f}"])
        if rng.random() < pair_share:
            for _ in range(rng.randrange(1, 4)):
                pos = rng.randrange(k)
                b = a ^ (rng.randrange(1, 4) << 2 * pos)
                if b:
                    rows.append([a, b, rng.choice([f"{rng.uniform(0, 20):.4f}", str(rng.randrange(0, 30))])])
    if dup and rows:
        for _ in range(max(1, len(rows) // 50)):
            r = rng.choice(rows)
            rows.append([r[0], r[1], f"{rng.uniform(0, 40):.2f}"])
    if rows:
        rows.append([rows[0][0], rows[0][1] if rows[0][1] != -5 else 1, "inf"])
    if nan and rows:  # on defaults, which most rows use
        for r in rng.sample([r for r in rows if r[1] == -5], 3):
            rows.append([r[0], r[1], "nan"])
    rows.append([0, -5, "1.0"])                 # keys no k-mer looks up
    rows.append([(1 << 30) + 5, 3, "2.0"])
    return rows


def build_cases():
    rng = random.Random(20261019)
    detect = []
    ks = [1, 3, 5, 7, 11, 15]
    windows = [25, 0, 25.7]
    gaps = [40, 12.5, 7.3, 3]
    for c in range(18):
        n = rng.choice([300, 600, 1000])
        ref = rand_seq(rng, n)
        if c % 4 == 3:  # soft-masked stretch
            a = rng.randrange(0, n // 2)
            ref = ref[:a] + ref[a:a + n // 3].lower() + ref[a + n // 3:]
        long_ins = {rng.randrange(60, n - 60): 1100} if c in (2, 9, 14) else {}
        variants = make_variants(rng, ref, rng.choice([20, 50, 120]), long_ins, multi=0.0)
        # multiallelic sites (which make the reference raise) in every third case only, and few of them
        variants = [(p, r, a if len(a) == 1 or (c % 3 == 0 and rng.random() < 0.1) else a[:1]) for p, r, a in variants]
        variants.sort(key=lambda v: v[0])
        alns = []
        for _ in range(rng.choice([8, 14])):
            length = rng.choice([60, 150, 600, 1500])
            start = rng.randrange(0, max(1, n - length // 2))
            aln = make_read(rng, ref, variants, start, length)
            if rng.random() < 0.3 and aln.query_sequence:  # N in the read
                s = list(aln.query_sequence)
                for _ in range(rng.randrange(1, 4)):
                    s[rng.randrange(len(s))] = "N"
                aln.query_sequence = "".join(s)
            alns.append(aln)
        if long_ins:
            p = next(iter(long_ins))
            alt = next(v for v in variants if v[0] == p)[2][0]
            lo = max(0, p - 80)
            alns.append(Aln(lo, [(0, p + 1 - lo), (1, len(alt) - 1), (0, 80)], ref[lo:p + 1] + alt[1:] + ref[p + 1:p + 81]))
        alns.append(Aln(rng.randrange(0, n), [], ""))
        k = ks[c % len(ks)]
        window = windows[c % len(windows)]
        gap = gaps[c % len(gaps)]
        costs = make_costs(rng, padded_alleles(ref, variants, int(windows[c % len(windows)]) + 2), k, default_share=0.97 if c % 5 else 0.5, nan=c % 6 == 1)
        rg = None
        if c % 5 == 2:
            rg = [rng.choice([[0, 0], [0, 1], [1, 1], [1, 2]]) for _ in variants]
        multi = any(len(v[2]) > 1 for v in variants)
        detect.append(dict(name=f"random{c}", reference=ref, variants=variants, alignments=[(a.reference_start, a.cigartuples, a.query_sequence) for a in alns],
                           restricted=rg, k=k, gap=gap, window=window, costs=costs, multi=multi))
    # raising alignments, one per alignment: a multiallelic variant covered, an unknown CIGAR op, a window before the start
    ref = rand_seq(rng, 300)
    variants = [(50, ref[50], ["A" if ref[50] != "A" else "C"]), (100, ref[100], ["C", "G"]), (150, ref[150], [ref[150] + "TT"]),
                (200, ref[200], ["<DEL>"])]
    alns = [Aln(30, [(0, 40)], ref[30:70]),                                 # fine
            Aln(80, [(0, 40)], ref[80:120]),                                # covers the multiallelic variant
            Aln(40, [(0, 20), (9, 3), (0, 20)], ref[40:80]),                # unknown CIGAR op after a variant
            Aln(190, [(0, 30)], ref[190:220]),                              # symbolic only: fine
            Aln(45, [(0, 10), (6, 2), (0, 30)], ref[45:85])]                # P inside the window
    strings = [ref]
    for window in (5, 25):
        detect.append(dict(name=f"raising_window{window}", reference=ref, variants=variants, alignments=[(a.reference_start, a.cigartuples, a.query_sequence) for a in alns],
                           restricted=None, k=5, gap=10, window=window, costs=make_costs(rng, strings, 5), multi=True))
    detect.append(dict(name="ends", reference=ref, variants=[(3, ref[3], [ref[3] + "GG"]), (296, ref[296], ["C" if ref[296] != "C" else "A"])],
                       alignments=[(0, [(0, 40)], ref[:40]), (260, [(0, 40)], ref[260:])], restricted=None, k=3, gap=2.5, window=10,
                       costs=make_costs(rng, strings, 3), multi=False))
    # enumerations
    enum = [["ACGTNACGT", 3], ["acgtACG", 3], ["NNNNNNC", 7], ["TAAATCCTGG", 7], ["TAAATCCTGG", 11], ["", 5], ["AAAAAAAA", 3]]
    for _ in range(200):
        s = "".join(rng.choice("ACGTACGTACGTNacgtX") for _ in range(rng.randrange(0, 80)))
        enum.append([s, rng.randrange(1, 16)])
    # pairs, per table
    pairs = []
    for t, k in enumerate([1, 3, 5, 7, 11, 15]):
        seqs = []
        for _ in range(60 if k >= 7 else 150):
            a = rand_seq(rng, rng.randrange(0, 70), "ACGTACGTN" if t % 2 else "ACGT")
            b = list(a)
            for _ in range(rng.randrange(0, 6)):
                if b:
                    p = rng.randrange(len(b))
                    b[p:p + rng.randrange(0, 3)] = rng.choice(["", "A", "G", rand_seq(rng, rng.randrange(1, 5))])
            b = "".join(b)
            if rng.random() < 0.03:
                a = a + rand_seq(rng, rng.randrange(100, 300))
            if rng.random() < 0.03:
                b = rand_seq(rng, rng.randrange(65, 200)) + b
            seqs.append((a, b) if rng.random() < 0.5 else (b, a))
        costs = make_costs(rng, [p[0] for p in seqs], k, pair_share=0.4, nan=t in (1, 3))  # the rows' k-mers
        pairs.append(dict(k=k, gap=[5, 12.5, 40, 7.3, 3, 0.1][t], costs=costs, seqs=seqs))
    pairs.append(dict(k=3, gap=float("inf"), costs=pairs[1]["costs"], seqs=pairs[1]["seqs"][:60]))  # inf * 0 is NaN at score[0][0]
    # a seeded synthetic costs table over all k-mers of k = 5, drawn without regard to the strings
    k = 5
    synth = [[a, -5, f"{rng.uniform(10, 50):.2f}"] for a in range(1, 4 ** k) if rng.random() < 0.9]
    synth += [[rng.randrange(1, 4 ** k), rng.randrange(1, 4 ** k), f"{rng.uniform(0, 30):.3f}"] for _ in range(2000)]
    seqs = [(rand_seq(rng, rng.randrange(20, 70)), rand_seq(rng, rng.randrange(20, 70))) for _ in range(300)]
    pairs.append(dict(k=k, gap=15, costs=synth, seqs=seqs))
    return dict(detect=detect, enumerate=enum, pairs=pairs)


def cost_dict(rows):
    """The dict _alignments_to_reads builds from the file's rows (variants.py:451-454)."""
    d = {}
    for a, b, v in rows:
        d[(int(a), int(b))] = v
    return d


def run_reference(cases):
    from oracle import build_pyref

    path = build_pyref.build()
    if not path:
        raise SystemExit("the reference tree is not available")
    sys.meta_path.insert(0, _StubFinder())
    sys.path.insert(0, path)
    from whatshap.align import enumerate_all_kmers, kmer_align
    from whatshap.variants import ReadSetReader
    from whatshap.vcf import BiallelicVcfVariant, MultiallelicVcfVariant

    for c in cases["detect"]:
        variants = [BiallelicVcfVariant(p, r, a[0]) if len(a) == 1 else MultiallelicVcfVariant(p, r, a) for p, r, a in c["variants"]]
        rg = [Gt(v) for v in c["restricted"]] if c["restricted"] else None
        costs = cost_dict(c["costs"])
        want = []
        calculated, splitted = {}, {}
        for start, cigar, seq in c["alignments"]:
            try:
                got = list(ReadSetReader.detect_alleles_by_alignment(variants, rg, 0, Aln(start, cigar, seq), c["reference"], 10, False, None, None, None,
                                                                     True, costs, c["k"], c["gap"], c["window"], calculated, splitted))
                want.append([[int(i), int(a), int(q)] for i, a, q in got])
            except Exception as e:  # noqa: BLE001 - recorded as the expected outcome
                want.append(type(e).__name__)
        c["want"] = want
    cases["enumerate"] = [[s, k, list(enumerate_all_kmers(s.encode(), k))] for s, k, *_ in cases["enumerate"]]
    for t in cases["pairs"]:
        costs = cost_dict(t["costs"])
        t["want"] = [repr(float(np.float32(kmer_align(enumerate_all_kmers(a.encode(), t["k"]), enumerate_all_kmers(b.encode(), t["k"]), costs, t["gap"]))))
                     for a, b in t["seqs"]]
    return cases


if __name__ == "__main__":
    cases = run_reference(build_cases())
    # the JSON as UTF-8 bytes (a numpy str array would hold 4 bytes per character)
    np.savez_compressed(os.path.join(HERE, "kmerald.npz"), cases=np.frombuffer(json.dumps(cases).encode(), np.uint8))
    d = cases["detect"]
    n_calls = sum(len(w) for c in d for w in c["want"] if isinstance(w, list))
    errors = sum(1 for c in d for w in c["want"] if isinstance(w, str))
    print(f"{len(d)} detect cases, {sum(len(c['alignments']) for c in d)} alignments, {n_calls} calls, {errors} raising alignments; "
          f"{len(cases['enumerate'])} enumerations, {sum(len(t['seqs']) for t in cases['pairs'])} pairs")
