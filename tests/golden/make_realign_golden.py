"""Regenerates tests/golden/realign.npz: the reference's own ReadSetReader.detect_alleles_by_alignment (whatshap/variants.py,
with whatshap._variants and whatshap.align compiled by oracle/build_pyref.build()) on seeded cases.  Needs the WhatsHap source
tree at $WHATSHAP_REF; the modules variants.py imports but the call never uses (pysam, pyfaidx, xopen) are stubbed.

    python tests/golden/make_realign_golden.py

Each case holds the reference, the variants, the alignments, the restricted genotypes (or none) and the mode, and per
alignment either the list of (variant index, allele, quality) or the exception the reference raised for it."""
import importlib.util
import json
import os
import random
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
STUBS = ("pysam", "pyfaidx", "xopen")


class _Any:
    def __init__(self, *a, **k):
        pass


class _StubFinder:
    def find_spec(self, name, path=None, target=None):
        if name.split(".")[0] in STUBS:
            return importlib.util.spec_from_loader(name, self, is_package=True)

    def create_module(self, spec):
        m = types.ModuleType(spec.name)
        m.__path__ = []
        m.__getattr__ = lambda n: _Any
        return m

    def exec_module(self, m):
        pass


class Aln:
    def __init__(self, start, cigar, seq):
        self.reference_start, self.cigartuples, self.query_sequence, self.query_qualities = start, cigar, seq, None


class Gt:
    def __init__(self, v):
        self.v = v

    def as_vector(self):
        return list(self.v)


def rand_seq(rng, n, alphabet="ACGT"):
    return "".join(rng.choice(alphabet) for _ in range(n))


def make_variants(rng, reference, every, long_ins=(), multi=0.15, symbolic=0.03, dup=0.03):
    out, pos = [], rng.randrange(0, every)
    for p in long_ins:
        out.append((p, reference[p], [reference[p] + rand_seq(rng, long_ins[p])]))
    while pos < len(reference) - 1:
        r = reference[pos]
        kind = rng.random()
        if kind < 0.55:
            alts = [rng.choice([c for c in "ACGT" if c != r.upper()])]
        elif kind < 0.7:
            alts = [r + rand_seq(rng, rng.choice([1, 2, 5, 12, 70]))]
        elif kind < 0.85:
            k = min(rng.choice([1, 3, 8, 30, 90]), len(reference) - pos - 1)
            r, alts = reference[pos:pos + k + 1], [reference[pos]]
        else:
            alts = [rng.choice("ACGT"), r + rand_seq(rng, 3)]
        if rng.random() < multi:
            alts = alts + [rng.choice("ACGT") + rand_seq(rng, rng.randrange(0, 3))]
        if rng.random() < symbolic:
            alts = ["<DEL>"]
        out.append((pos, r, alts))
        if rng.random() < dup:
            out.append((pos, reference[pos], [rng.choice("ACGT")]))
        pos += rng.randrange(max(2, every // 2), every * 2)
    out.sort(key=lambda v: v[0])
    return out


def make_read(rng, reference, variants, start, length, err=0.05, clips=True, skip=0.05, ops_extra=()):
    """A read from a haplotype with random alleles, aligned as the haplotype differs from the reference, plus errors."""
    cigar, seq, pos = [], [], start
    if clips and rng.random() < 0.3:
        cigar.append((5, rng.randrange(1, 20)))
    if clips and rng.random() < 0.3:
        k = rng.randrange(1, 15)
        cigar.append((4, k))
        seq.append(rand_seq(rng, k))
    vmap = {}
    for v in variants:
        vmap.setdefault(v[0], v)

    def add(op, n):
        if n <= 0:
            return
        if cigar and cigar[-1][0] == op:
            cigar[-1] = (op, cigar[-1][1] + n)
        else:
            cigar.append((op, n))

    consumed = 0
    while consumed < length and pos < len(reference):
        v = vmap.get(pos)
        if v is not None and rng.random() < 0.5 and not v[2][0].startswith("<"):
            r, a = v[1], rng.choice(v[2])
            if len(r) == 1 and len(a) >= 1 and a[0].upper() == r.upper() and len(a) > 1:
                add(0, 1)
                seq.append(reference[pos].upper())
                add(1, len(a) - 1)
                seq.append(a[1:])
                pos += 1
                consumed += len(a)
                continue
            if len(a) == 1 and len(r) > 1 and a.upper() == r[0].upper() and pos + len(r) <= len(reference):
                add(0, 1)
                seq.append(reference[pos].upper())
                add(2, len(r) - 1)
                pos += len(r)
                consumed += 1
                continue
            if len(a) == 1 and len(r) == 1:
                add(0, 1)
                seq.append(a)
                pos += 1
                consumed += 1
                continue
        x = rng.random()
        if x < err / 3:
            add(8, 1)
            seq.append(rng.choice("ACGT"))
            pos += 1
            consumed += 1
        elif x < 2 * err / 3:
            k = rng.randrange(1, 4)
            add(1, k)
            seq.append(rand_seq(rng, k))
            consumed += k
        elif x < err:
            add(2, rng.randrange(1, 4))
            pos = min(len(reference), pos + cigar[-1][1] if cigar[-1][0] == 2 else pos)
        elif x < err + skip / max(1, length):
            add(3, rng.randrange(5, 60))
            pos += cigar[-1][1]
        else:
            add(rng.choice([0, 0, 0, 7]), 1)
            seq.append(reference[pos].upper())
            pos += 1
            consumed += 1
    if clips and rng.random() < 0.3:
        k = rng.randrange(1, 15)
        add(4, k)
        seq.append(rand_seq(rng, k))
    if clips and rng.random() < 0.2:
        add(5, rng.randrange(1, 9))
    for op in ops_extra:
        cigar.insert(len(cigar) // 2, op)
    return Aln(start, cigar, "".join(seq))


def build_cases():
    rng = random.Random(20261018)
    cases = []

    def case(name, reference, variants, alns, rg=None, overhang=10, affine=False, gs=None, ge=None, mm=None):
        cases.append(dict(name=name, reference=reference, variants=variants, alignments=[(a.reference_start, a.cigartuples, a.query_sequence) for a in alns],
                          restricted=rg, overhang=overhang, affine=affine, gap_start=gs, gap_extend=ge, default_mismatch=mm))

    modes = [dict(), dict(affine=True, gs=10, ge=7, mm=15), dict(affine=True, gs=10.9, ge=3.5, mm=2.5), dict(affine=True, gs=1, ge=1, mm=1)]
    for k in range(16):
        n = rng.choice([400, 1500, 4000])
        ref = rand_seq(rng, n)
        if k % 4 == 3:  # soft-masked stretch
            a = rng.randrange(0, n // 2)
            ref = ref[:a] + ref[a:a + n // 3].lower() + ref[a + n // 3:]
        long_ins = {rng.randrange(50, n - 50): 80} if k % 3 == 0 else {}
        if k in (5, 11):
            long_ins[rng.randrange(50, n - 50)] = 1100
        variants = make_variants(rng, ref, rng.choice([15, 40, 100]), long_ins)
        variants.append((0, ref[0], [rng.choice("ACGT")]))
        variants.append((n - 1, ref[n - 1], [rng.choice("ACGT")]))
        variants.sort(key=lambda v: v[0])
        alns = []
        for _ in range(rng.choice([10, 30])):
            length = rng.choice([60, 150, 600, 1500])
            start = rng.randrange(0, max(1, n - length // 2))
            alns.append(make_read(rng, ref, variants, start, length))
        alns.append(Aln(rng.randrange(0, n), [], ""))  # empty CIGAR
        mode = modes[k % len(modes)]
        overhang = [10, 10, 3, 25, 0, 1][k % 6]
        rg = None
        if k % 5 == 2:
            rg = [rng.choice([[0, 0], [0, 1], [1, 1], [1, 2], [0, 2], [2, 2]]) for _ in variants]
        case(f"random{k}", ref, variants, alns, rg, overhang, **mode)
    # reads at both ends of the chromosome, a read running past its end
    ref = rand_seq(rng, 200)
    variants = [(0, ref[0], ["T" if ref[0] != "T" else "A"]), (3, ref[3], [ref[3] + "GG"]), (196, ref[196], ["C"]), (199, ref[199], ["G"])]
    for mode in modes[:2]:
        case("ends", ref, variants, [Aln(0, [(0, 40)], ref[:40]), Aln(170, [(0, 30)], ref[170:]), Aln(180, [(0, 30)], ref[180:] + "ACGTACGTAC")], **mode)
    # raising cases, one per alignment
    ref = rand_seq(rng, 300)
    variants = [(50, ref[50], ["A" if ref[50] != "A" else "C"]), (100, ref[100:104], [ref[100]]), (150, ref[150], [ref[150] + "TT"])]
    raising = [Aln(40, [(0, 20), (9, 3), (0, 20)], ref[40:80]),                      # unknown CIGAR op after a variant
               Aln(45, [(0, 10), (6, 2), (0, 30)], ref[45:85]),                       # P inside the window
               Aln(50, [(0, 30)], ref[50:80]),                                         # overhang 0: empty left CIGAR
               Aln(30, [(0, 40)], ref[30:70])]                                         # fine
    for overhang in (0, 5):
        case(f"raising_overhang{overhang}", ref, variants, raising, overhang=overhang)
    case("empty_restriction", ref, variants, [Aln(30, [(0, 40)], ref[30:70])], rg=[[3, 4], [0, 1], [0, 1]])
    case("unsorted", ref, [variants[1], variants[0], variants[2]], [Aln(30, [(0, 150)], ref[30:180]), Aln(120, [(0, 50)], ref[120:170])])
    return cases


def run_reference(cases):
    from oracle import build_pyref

    path = build_pyref.build()
    if not path:
        raise SystemExit("the reference tree is not available")
    sys.meta_path.insert(0, _StubFinder())
    sys.path.insert(0, path)
    from whatshap.variants import ReadSetReader
    from whatshap.vcf import BiallelicVcfVariant, MultiallelicVcfVariant

    for c in cases:
        variants = [BiallelicVcfVariant(p, r, a[0]) if len(a) == 1 else MultiallelicVcfVariant(p, r, a) for p, r, a in c["variants"]]
        rg = [Gt(v) for v in c["restricted"]] if c["restricted"] else None
        want = []
        for start, cigar, seq in c["alignments"]:
            try:
                got = list(ReadSetReader.detect_alleles_by_alignment(variants, rg, 0, Aln(start, cigar, seq), c["reference"], c["overhang"],
                                                                     c["affine"], c["gap_start"], c["gap_extend"], c["default_mismatch"]))
                want.append([[int(i), int(a), int(q)] for i, a, q in got])
            except Exception as e:  # noqa: BLE001 - recorded as the expected outcome
                want.append(type(e).__name__)
        c["want"] = want
    return cases


if __name__ == "__main__":
    cases = run_reference(build_cases())
    np.savez_compressed(os.path.join(HERE, "realign.npz"), cases=np.array(json.dumps(cases)))
    n_items = sum(len(w) for c in cases for w in c["want"] if isinstance(w, list))
    errors = sum(1 for c in cases for w in c["want"] if isinstance(w, str))
    print(f"{len(cases)} cases, {sum(len(c['alignments']) for c in cases)} alignments, {n_items} calls, {errors} raising alignments")
