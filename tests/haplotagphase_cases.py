"""Seeded cases for the votes of `whatshap haplotagphase` and the pieces that run them: stand-ins for the VCF reader, the
phased-input reader, the VCF writer and the FASTA that `run_haplotagphase` opens, and the per-sample loop of that function for
other compute_votes / consensus pairs.

A case holds the samples of the VCF, the samples to phase ("included", empty for all), gap, cut_poly, only_indels, the reference
sequence, the records ([position, is_snv] in table order, positions may repeat) and per sample the calls ([genotype alleles,
phased] per record) and the reads ([HP_tag, PS_tag, [[position, allele, quality], ...]]).  A result is, per VCF sample, None for
a sample left out or {"votes": [[position, [[ps, h, score], ...]], ...], "super": two lists of [position, allele, quality],
"components": [[position, ps], ...]}; or the name of the exception raised."""
import random

EXCEPTIONS = (KeyError, ZeroDivisionError, IndexError, ValueError)


class _Variant:
    def __init__(self, position, snv):
        self.position, self._snv = position, snv

    def is_snv(self):
        return self._snv


class _Genotype:
    def __init__(self, alleles):
        self.alleles = list(alleles)

    def as_vector(self):
        return list(self.alleles)

    def is_homozygous(self):
        return len(set(self.alleles)) == 1


class _Phase:
    def __init__(self, block_id):
        self.block_id = block_id


class VariantTable:
    def __init__(self, case):
        self.chromosome = "chr1"
        self.variants = [_Variant(p, snv) for p, snv in case["records"]]
        self.calls = case["calls"]

    def genotypes_of(self, sample):
        return [_Genotype(gt) for gt, _ in self.calls[sample]]

    def phases_of(self, sample):
        return [_Phase(1) if ph else None for _, ph in self.calls[sample]]


class VcfReader:
    def __init__(self, case):
        self.case, self.samples = case, list(case["samples"])

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def __iter__(self):
        return iter([VariantTable(self.case)])


class PhasedInputReader:
    def __init__(self, case, core):
        self.case, self.core = case, core

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def read(self, chromosome, variants, sample, restricted_genotypes=None, **kw):
        return readset(self.core, self.case["reads"][sample]), None


class Writer:
    def __init__(self):
        self.written = []

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def write(self, chromosome, sample_to_super_reads, sample_to_components):
        self.written.append((sample_to_super_reads, sample_to_components))

    def write_unchanged(self, chromosome):
        pass


class Fasta(dict):
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def readset(core, reads):
    rs = core.ReadSet()
    for k, (hp, ps, entries) in enumerate(reads):
        r = core.Read(f"r{k}", 60, 0, 0, 0, "", hp, ps)
        for p, a, q in entries:
            r.add_variant(p, a, q)
        rs.add(r)
    return rs


def plain_votes(votes):
    return [[p, [[ps, h, s] for (ps, h), s in v.items()]] for p, v in votes.items()]


def plain_result(votes_by_sample, super_reads, components, samples):
    out = []
    for s in samples:
        if s not in super_reads:
            out.append(None)
            continue
        out.append({"votes": plain_votes(votes_by_sample[s]),
                    "super": [[[v.position, v.allele, v.quality] for v in sr] for sr in super_reads[s]],
                    "components": [[p, c] for p, c in components[s].items()]})
    return out


def run_module(h, case, core):
    """The module's own run_haplotagphase (h: the reference's whatshap.cli.haplotagphase, maybe with swapped-in functions) on
    the case, with the stand-ins assigned into the module; its result in plain form or the exception's name."""
    writer, seen, order = Writer(), {}, []
    h.VcfReader = lambda *a, **k: VcfReader(case)
    h.PhasedInputReader = lambda *a, **k: PhasedInputReader(case, core)
    h.PhasedVcfWriter = lambda *a, **k: writer
    h.IndexedFasta = lambda *a, **k: Fasta(chr1=case["refseq"])
    inner = h.compute_votes

    def compute_votes(*a):
        v = inner(*a)
        order.append(v)
        return v

    h.compute_votes = compute_votes
    try:
        h.run_haplotagphase("in.vcf", "in.bam", output="out.vcf", samples=list(case["included"]), reference="ref.fa",
                            only_indels=case["only_indels"], gap_threshold=case["gap"], cut_poly=case["cut_poly"],
                            write_command_line_header=False)
    except EXCEPTIONS as e:
        return type(e).__name__
    finally:
        h.compute_votes = inner
    (super_reads, components), = writer.written
    included = [s for s in case["samples"] if not case["included"] or s in case["included"]]
    return plain_result(dict(zip(included, order)), super_reads, components, case["samples"])


def run_functions(compute_votes, consensus, case, core):
    """run_haplotagphase's per-sample loop around another compute_votes / consensus pair, with reads of `core`."""
    table = VariantTable(case)
    votes_by, supers, comps = {}, {}, {}
    try:
        for s in case["samples"]:
            if case["included"] and s not in case["included"]:
                continue
            homozygous, change, phased, a2i, i2a = {}, {}, {}, {}, {}
            for v, gt, ph in zip(table.variants, table.genotypes_of(s), table.phases_of(s)):
                for i, a in enumerate(gt.as_vector()):
                    a2i.setdefault(v.position, {})[a] = i
                    i2a.setdefault(v.position, {})[i] = a
                homozygous[v.position], phased[v.position], change[v.position] = gt.is_homozygous(), ph, v
            votes = compute_votes(homozygous, readset(core, case["reads"][s]), a2i)
            votes_by[s] = votes
            supers[s], comps[s] = consensus(case["only_indels"], case["gap"], case["cut_poly"], case["refseq"], change, phased, votes, i2a)
    except EXCEPTIONS as e:
        return type(e).__name__
    return plain_result(votes_by, supers, comps, case["samples"])


def run_oracle(case):
    from oracle import haplotagphase_oracle as o

    samples = []
    for s in case["samples"]:
        records = [(p, snv, gt, ph) for (p, snv), (gt, ph) in zip(case["records"], case["calls"][s])]
        reads = [(hp, ps, [tuple(e) for e in en]) for hp, ps, en in case["reads"][s]]
        samples.append((records, reads, not case["included"] or s in case["included"]))
    try:
        res = o.run(samples, case["gap"], case["only_indels"])
    except EXCEPTIONS as e:
        return type(e).__name__
    out = []
    for r in res:
        if r is None:
            out.append(None)
            continue
        votes, _, sup, comp = r
        out.append({"votes": plain_votes(votes), "super": [[list(x) for x in sr] for sr in sup], "components": [list(c) for c in comp]})
    return out


def homopolymers(rng, n):
    out, bases = [], "ACGT"
    while sum(map(len, out)) < n:
        out.append(rng.choice(bases) * rng.choice([1, 1, 2, 3, 5, 8, 12, 20]))
    return "".join(out)[:n]


def make_case(rng: random.Random, n_samples=None, big=False, error=None, gap=None, cut_poly=None, only_indels=None, included=None):
    """One seeded case; error in (None, 'position', 'allele', 'haplotype', 'zero') plants the first error of that kind."""
    n_samples = n_samples or rng.choice([1, 1, 2, 3])
    n_var = rng.randint(150, 300) if big else rng.randint(3, 25)
    length = 60 * n_var + 200
    positions = sorted(rng.sample(range(5, length - 5), n_var))
    records = [[p, rng.random() < 0.6] for p in positions]
    for _ in range(rng.randint(0, 3)):  # records sharing a position
        i = rng.randrange(len(records))
        records.insert(i + 1, [records[i][0], rng.random() < 0.5])
    samples = [f"S{i}" for i in range(n_samples)]
    calls, reads = {}, {}
    n_ps = rng.choice([1, 2, 3, 5])
    for s in samples:
        row = []
        for _ in records:
            u = rng.random()
            if u < 0.15:
                gt = [rng.choice([0, 1])] * 2  # homozygous
            elif u < 0.2:
                gt = rng.choice([[0, 1, 1], [1, 0, 2], [0, 0, 1]])  # polyploid
            elif u < 0.25:
                gt = [rng.choice([0, 1, 2])]  # haploid
            else:
                gt = rng.choice([[0, 1], [1, 0], [0, 2], [2, 1]])
            row.append([gt, rng.random() < 0.3])
        if error != "haplotype":  # polyploid calls only where a KeyError is wanted (the first one decides otherwise)
            row = [[gt if len(gt) < 3 else gt[:2] if len(set(gt[:2])) > 1 else [0, 1], ph] for gt, ph in row]
        calls[s] = row
        n_reads = rng.randint(300, 500) if big else rng.randint(2, 25)
        rr = []
        for _ in range(n_reads):
            u = rng.random()
            hp = rng.choice([1, 2]) if u < 0.85 else rng.choice([-1, 0, 3, 4])
            ps = rng.randrange(n_ps) * 1000 + 7 if rng.random() < 0.92 else rng.choice([-1, 0])
            i0 = rng.randrange(len(positions))
            ent = []
            for p in positions[i0:i0 + rng.randint(0, 8)]:
                alleles = sorted({a for (q, _), (gt, _) in zip(records, row) if q == p for a in gt})
                ent.append([p, rng.choice(alleles), 0 if rng.random() < 0.01 else rng.choice([1, 5, 10, 10, 20, 30, 37, 60])])
            rr.append([hp, ps, ent])
        reads[s] = rr
    s = rng.choice(samples)
    usable = [r for r in reads[s] if r[0] in (1, 2) and r[1] >= 1]
    if error in ("position", "allele", "zero") and usable:
        r = rng.choice(usable)
        het = [p for (p, _), (gt, _) in zip(records, calls[s]) if len(set(gt)) > 1]
        if error == "position":
            r[2].insert(rng.randint(0, len(r[2])), [length + 3, 0, 5])
        elif error == "allele" and het:
            r[2].insert(rng.randint(0, len(r[2])), [rng.choice(het), 7, 5])
        elif error == "zero" and het:
            p = rng.choice(het)
            for rd in reads[s]:
                rd[2] = [[q, a, 0 if q == p else w] for q, a, w in rd[2]]
            r[2].append([p, calls[s][[q for q, _ in records].index(p)][0][0], 0])
    if included is None:
        included = [] if rng.random() < 0.7 else rng.sample(samples, rng.randint(1, len(samples)))
    return {"samples": samples, "included": included, "gap": rng.choice([0, 29, 50, 70, 70, 90, 101]) if gap is None else gap,
            "cut_poly": rng.choice([-1, 0, 1, 2, 10]) if cut_poly is None else cut_poly,
            "only_indels": rng.random() < 0.3 if only_indels is None else only_indels, "refseq": homopolymers(rng, length),
            "records": records, "calls": calls, "reads": reads}


def boundary_case(gap):
    """One unphased position whose best score is 29 of a total of 100: keys (1000, 0) 29, (1000, 1) 29, (2000, 0) 29, (2000, 1)
    13.  100 * (29 / 100) is 28.999999999999996, below a gap threshold of 29."""
    reads = [[1, 1001, [[50, 0, 29]]], [2, 1001, [[50, 0, 29]]], [1, 2001, [[50, 0, 29]]], [2, 2001, [[50, 0, 13]]]]
    return {"samples": ["S0"], "included": [], "gap": gap, "cut_poly": 10, "only_indels": False, "refseq": "A" * 100,
            "records": [[50, True]], "calls": {"S0": [[[0, 1], False]]}, "reads": {"S0": reads}}


def tie_case():
    """Keys {(5, 0): 7, (5, 1): 9, (3, 0): 9, (3, 1): 1} at position 40: the best is (5, 1), inserted before (3, 0)."""
    reads = [[1, 6, [[40, 0, 7]]], [2, 6, [[40, 0, 9]]], [1, 4, [[40, 0, 9]]], [2, 4, [[40, 0, 1]]]]
    return {"samples": ["S0"], "included": [], "gap": 0, "cut_poly": 2, "only_indels": False, "refseq": "C" * 100,
            "records": [[40, False]], "calls": {"S0": [[[0, 1], False]]}, "reads": {"S0": reads}}
