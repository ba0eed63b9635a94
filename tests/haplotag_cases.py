"""Seeded cases for the read assignment of `whatshap haplotag` and the pieces that run them: a variant table and a phased-input
reader as `prepare_haplotag_information` calls them, and the results in a comparable, JSON-friendly form.

A case holds ploidy, ignore (linked reads), cutoff, the chromosome, the variant positions in table order, and per sample the
calls ([genotype alleles, block id or None, phase tuple or None] per variant) and the reads ([name, source_id, chromosome,
is_supplementary, sub_alignment_id, BX tag or '', reference_start, reference_end, is_reverse, [[position, allele, quality]]])."""
import random
from collections import defaultdict


class _Variant:
    def __init__(self, position):
        self.position = position


class _Genotype:
    def __init__(self, alleles):
        self.alleles = alleles

    def is_homozygous(self):
        return len(set(self.alleles)) == 1


class _Phase:
    def __init__(self, block_id, phase):
        self.block_id, self.phase = block_id, phase


class VariantTable:
    def __init__(self, case):
        self.chromosome = case["chromosome"]
        self.variants = [_Variant(p) for p in case["positions"]]
        self.calls = case["calls"]

    def genotypes_of(self, sample):
        return [_Genotype(gt) for gt, _, _ in self.calls[sample]]

    def phases_of(self, sample):
        return [None if phase is None else _Phase(block, tuple(phase)) for _, block, phase in self.calls[sample]]


class Reader:
    """`read(chromosome, variants, sample, regions=...)` -> (ReadSet of `core`'s classes holding the case's reads, None)."""

    def __init__(self, case, core):
        self.case, self.core = case, core

    def read(self, chromosome, variants, sample, regions=None):
        rs = self.core.ReadSet()
        for name, source, chrom, supp, sub, bx, start, end, rev, entries in self.case["reads"][sample]:
            r = self.core.Read(name, 30, source, 0, start, bx, -1, -1, chrom, sub, supp, end, rev)
            for p, a, q in entries:
                r.add_variant(p, a, q)
            rs.add(r)
        return rs, None


def oracle_samples(case):
    """[(phase table, reads)] in the oracle's form (the later record at a position wins)."""
    out = []
    for sample in case["samples"]:
        table = {}
        for p, (_, block, phase) in zip(case["positions"], case["calls"][sample]):
            if phase is not None and block is not None:
                table[p] = (int(block), tuple(phase))
        reads = [(n, c, bool(su), sb, bx, s, e, bool(rv), [tuple(x) for x in en]) for n, _, c, su, sb, bx, s, e, rv, en in case["reads"][sample]]
        out.append((table, reads))
    return out


def as_plain(bx, r2h, multi, primary):
    """The four results in JSON form: keys as field lists, sorted."""
    key = lambda k: [k.read_name, k.chromosome, bool(k.is_supplementary), k.sub_alignment_id] if hasattr(k, "read_name") else list(k)
    info = lambda v: [v.reference_start, v.reference_end, bool(v.is_reverse)] if hasattr(v, "reference_start") else list(v)
    return {
        "bx": {t: [list(map(int, x)) for x in v] for t, v in bx.items() if v},
        "r2h": sorted(key(k) + [int(x) for x in v] for k, v in r2h.items()),
        "multi": int(multi),
        "primary": sorted(key(k) + info(v) for k, v in primary.items()),
    }


def same(want, got, loose=()):
    """Whether got equals want, where the members of each loose group may hold any of its choices (None: nothing recorded)
    and its BX entry any choice at the opening read's start."""
    want, got = dict(want), dict(got)
    free_keys, free_bx = {}, defaultdict(list)
    for members, bx, start, options in loose:
        for m in members:
            free_keys[tuple(m)] = [tuple(o) if o else None for o in options]
        if bx:
            free_bx[bx] += [[start, o[0], o[2]] for o in options if o]
    r2h = []
    for side in (want, got):
        fixed, free = [], {}
        for row in side["r2h"]:
            k = tuple(row[:4])
            if k in free_keys:
                free[k] = tuple(row[4:])
            else:
                fixed.append(row)
        r2h.append((fixed, free))
    if r2h[0][0] != r2h[1][0] or want["multi"] != got["multi"] or want["primary"] != got["primary"]:
        return False
    for k, options in free_keys.items():  # (a later sample's group may have overwritten the key: then it is exact)
        if r2h[1][1].get(k) != r2h[0][1].get(k) and r2h[1][1].get(k) not in options:
            return False
    for side in (want, got):
        side["bx"] = {t: [x for x in v if x not in free_bx.get(t, [])] for t, v in side["bx"].items()}
        side["bx"] = {t: v for t, v in side["bx"].items() if v}
    return want["bx"] == got["bx"]


def make_case(rng: random.Random, ploidy=None, n_samples=None, error=None, big=False):
    """One seeded case; error in (None, 'assert', 'key', 'index', 'choice') plants the first error of that kind."""
    ploidy = ploidy or rng.choice([2, 2, 3, 4])
    n_samples = n_samples or rng.choice([1, 1, 2])
    n_var = rng.randint(200, 400) if big else rng.randint(4, 30)
    positions = sorted(rng.sample(range(100, 100 + 40 * n_var), n_var))
    for _ in range(rng.randint(0, 2)):  # duplicate VCF positions
        i = rng.randrange(n_var)
        positions.insert(i, positions[i])
    samples = [f"S{i}" for i in range(n_samples)]
    blocks = rng.sample([7, 100, 2047, 90001, 5, 12], rng.randint(1, 4))
    calls, reads = {}, {}
    for s in samples:
        row = []
        for _ in positions:
            u = rng.random()
            length = ploidy + (rng.choice([-1, 1]) if rng.random() < 0.1 else 0)
            phase = [rng.choice([0, 1]) for _ in range(max(length, 1))]
            if rng.random() < 0.1:
                phase[rng.randrange(len(phase))] = 2  # a multi-allelic record's allele that no read carries
            if length > ploidy:
                phase[-1] = 2  # a haplotype beyond the ploidy that no read matches
            gt = list(phase) if rng.random() < 0.85 else [phase[0]] * len(phase)
            if u < 0.08:
                row.append([gt, None, None])  # unphased
            elif u < 0.12:
                row.append([gt, None, phase])  # a phase without a block id
            else:
                row.append([gt, rng.choice(blocks), phase])
        calls[s] = row
        phased = sorted({p for p, (_, b, ph) in zip(positions, row) if b is not None and ph is not None})
        n_reads = rng.randint(300, 600) if big else rng.randint(3, 30)
        tags = [f"BX{i}" for i in range(max(1, n_reads // 4))]
        rr = []
        for k in range(n_reads):
            base = f"r{rng.randrange(max(2, n_reads * 2 // 3))}"
            supp = rng.random() < 0.15
            u = rng.random()
            if supp:
                sub = f"_s{rng.randint(2, 4)}"
                name = base + sub if u < 0.6 else base
            else:
                sub = "____1" if u < 0.85 else ("" if u < 0.92 else "_x")
                name = base + sub if rng.random() < 0.5 else base
            bx = rng.choice(tags) if rng.random() < 0.4 else ""
            start = rng.randint(0, 400)
            n_ent = rng.randint(0, min(8, len(phased)) if phased else 0)
            ent = [[p, rng.choice([0, 1]), rng.choice([0, 5, 10, 10, 20, 37])] for p in sorted(rng.sample(phased, n_ent))] if n_ent else []
            rr.append([name, 0, "chr1", supp, sub, bx, start, start + rng.randint(50, 500), rng.random() < 0.5, ent])
        # duplicate names take another source id
        seen = defaultdict(int)
        for r in rr:
            r[1] = seen[r[0]]
            seen[r[0]] += 1
        reads[s] = rr
    s = rng.choice(samples)
    if error in ("assert", "key"):
        r = rng.choice(reads[s])
        bad = [positions[0], 2, 4] if error == "assert" else [positions[-1] + 1, 0, 3]
        r[9].insert(rng.randint(0, len(r[9])), bad)
    elif error == "index":  # the last record at a read's position gets a matching allele beyond the ploidy
        with_entries = [r for r in reads[s] if r[9]]
        if with_entries:
            p, a, _ = rng.choice(rng.choice(with_entries)[9])
            i = max(j for j, q in enumerate(positions) if q == p)
            calls[s][i] = [[0, 1], calls[s][i][1] if calls[s][i][1] is not None else blocks[0], [2] * ploidy + [a]]
    return {"ploidy": 1 if error == "choice" else ploidy, "ignore": rng.random() < 0.15, "cutoff": rng.choice([0, 40, 150, 50000]),
            "chromosome": "chr1", "positions": positions, "samples": samples, "calls": calls, "reads": reads}


def run(prepare, case, core):
    """prepare_haplotag_information (a reference-signature function) on the case: its results in plain form, or the name of
    the exception it raised."""
    try:
        out = prepare(VariantTable(case), case["samples"], Reader(case, core), None, case["ignore"], case["cutoff"], case["ploidy"])
    except (AssertionError, KeyError, IndexError) as e:
        return type(e).__name__
    return as_plain(*out)


def run_oracle(case):
    """The oracle's answer in plain form (or the exception's name) and its loose groups."""
    from oracle import haplotag_oracle

    try:
        bx, r2h, multi, primary, loose = haplotag_oracle.prepare(oracle_samples(case), case["ploidy"], case["ignore"], case["cutoff"])
    except (AssertionError, KeyError, IndexError) as e:
        return type(e).__name__, []
    return as_plain(bx, r2h, multi, primary), [[[list(m) for m in ms], bx_, st, [list(o) if o else None for o in opts]]
                                                for ms, bx_, st, opts in loose]
