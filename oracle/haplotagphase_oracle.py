"""Plain-Python restatement of the votes of `whatshap haplotagphase` (compute_votes, best_candidate and consensus), written from
their rules.  The CPU reference for whatshap_b200.haplotagphase and whmec_haplotagphase.

A read is (HP_tag, PS_tag, [(position, allele, quality), ...]).  A sample's variant records are (position, is_snv, genotype
alleles, phased) in table order; several records at one position merge as run_haplotagphase merges them."""


def tables(records):
    """(homozygous, allele_to_id, id_to_allele, phased, is_snv) of one sample's records: the later record wins, except that the
    allele <-> id maps of one position accumulate entry by entry."""
    homozygous, a2i, i2a, phased, snv = {}, {}, {}, {}, {}
    for pos, is_snv, alleles, is_phased in records:
        for i, a in enumerate(alleles):
            a2i.setdefault(pos, {})[a] = i
            i2a.setdefault(pos, {})[i] = a
        homozygous[pos] = len(set(alleles)) == 1
        phased[pos] = is_phased
        snv[pos] = is_snv
    return homozygous, a2i, i2a, phased, snv


def votes_of(homozygous, reads, a2i):
    """(votes as position -> {(ps, h): score} in insertion order, number of reads with HP_tag > 2)."""
    votes, skipped = {}, 0
    for hp, ps_tag, entries in reads:
        ps, ht = ps_tag - 1, hp - 1
        if ps < 0 or ht < 0:
            continue
        if ht > 1:
            skipped += 1
            continue
        for pos, allele, quality in entries:
            if homozygous[pos]:  # KeyError for a position without a record
                continue
            vote = votes.setdefault(pos, {})
            if (ps, 0) not in vote:
                vote[(ps, 0)] = 0
                vote[(ps, 1)] = 0
            key = (ps, ht ^ a2i[pos][allele])  # KeyError for an unknown allele
            vote[key] += quality  # KeyError for a key outside (ps, 0), (ps, 1)
    return votes, skipped


def choose(vote):
    """(ps, h, score, total) of the best key: the highest score, ties to the key inserted first."""
    best = None
    for key, score in vote.items():
        if best is None or score > best[1]:
            best = (key, score)
    (ps, h), score = best
    return ps, h, score, sum(vote.values())


def consensus(votes, phased, snv, i2a, gap_threshold, only_indels):
    """([[(position, allele, quality)] for the two super-reads], [(position, phase set)] in vote order).  The homopolymer filter of
    the reference drops nothing (it counts at most cut_poly bases and asks for more), so it has no counterpart."""
    rows, components = [], []
    for pos, vote in votes.items():
        if not vote:
            raise IndexError("list index out of range")
        ps, h, score, total = choose(vote)
        q = score / total  # ZeroDivisionError
        components.append((pos, ps))
        if not phased[pos]:
            if 100 * q < gap_threshold or (only_indels and snv[pos]):
                continue
        rows.append((pos, i2a[pos][h], i2a[pos][1 - h], score))
    rows.sort()
    return [[(p, a, q) for p, a, _, q in rows], [(p, a, q) for p, _, a, q in rows]], components


def run(samples, gap_threshold, only_indels):
    """Per sample of `samples` ([(records, reads, included)]): None for a sample left out, else (votes, skipped, super-reads,
    components).  Raises what the reference raises first."""
    out = []
    for records, reads, included in samples:
        if not included:
            out.append(None)
            continue
        homozygous, a2i, i2a, phased, snv = tables(records)
        votes, skipped = votes_of(homozygous, reads, a2i)
        out.append((votes, skipped) + consensus(votes, phased, snv, i2a, gap_threshold, only_indels))
    return out
