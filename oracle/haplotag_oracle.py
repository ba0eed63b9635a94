"""Plain-Python restatement of the read assignment of `whatshap haplotag` (prepare_haplotag_information), written from its
rules, with one visit order where the reference has none: a group is its opening read, then its linked reads in read order,
each read's entries in their order.  The CPU reference for whatshap_b200.haplotag and whmec_haplotag.

A read is (name, chromosome, is_supplementary, sub_alignment_id, BX tag or '', reference_start, reference_end, is_reverse,
[(position, allele, quality), ...]); a phase table maps a position to (block id, phase tuple)."""
from collections import defaultdict

PRIMARY = "____1"


def representation(read, as_primary=False):
    name, chrom, supp, sub = read[0], read[1], read[2], read[3]
    used = PRIMARY if as_primary else sub
    if name.endswith(used):
        name = name[: -len(sub)]  # by the length of the read's own id, as the reference cuts
    return (name, chrom, False if as_primary else bool(supp), used)


def groups(reads, ignore_linked_read, linked_read_cutoff):
    """The groups of one sample's reads: [(opening read index, [member indices in visit order])]."""
    by_bx = defaultdict(list)
    if not ignore_linked_read:
        for i, r in enumerate(reads):
            if r[4]:
                by_bx[r[4]].append(i)
    done, out = set(), []
    for i, r in enumerate(reads):
        key = representation(r)
        if key in done:
            continue
        done.add(key)
        members = [i]
        if not ignore_linked_read and r[4]:
            members += [j for j in by_bx[r[4]]
                        if representation(reads[j]) not in done and abs(r[5] - reads[j][5]) <= linked_read_cutoff]
        for j in members:
            done.add(representation(reads[j]))
        out.append((i, members))
    return out


def score(reads, members, table, ploidy):
    """The group's phase sets in the order their first vote arrives: [(block id, [ploidy scores])]."""
    costs = {}
    for j in members:
        for pos, allele, quality in reads[j][8]:
            assert allele in (0, 1)
            block, phase = table[pos]
            for h, a in enumerate(phase):
                if a == allele:
                    if block not in costs:
                        costs[block] = [0] * max(ploidy, 0)
                    costs[block][h] += quality  # IndexError for h >= ploidy
    return list(costs.items())


def choose(block, scores):
    """(haplotype, quality, block): the lowest-index best haplotype and best - second best."""
    ranked = sorted(range(len(scores)), key=lambda h: (-scores[h], h))
    return ranked[0], scores[ranked[0]] - scores[ranked[1]], block


def prepare(samples, ploidy, ignore_linked_read=False, linked_read_cutoff=50000):
    """samples: [(phase table, reads)].  Returns (BX tag -> [(start, haplotype, block)], representation -> (haplotype, quality,
    block), groups with several phase sets, as-primary representation -> (start, end, is_reverse), loose), where loose lists
    the multi-read groups whose top phase sets tie (the reference may pick any of them): (member representations, BX tag or '',
    opening read's start, {choice or None for each tied block})."""
    bx_out, r2h, primary, loose = defaultdict(list), {}, {}, []
    multi = 0
    for table, reads in samples:
        for r in reads:
            if not r[2]:
                primary[representation(r, as_primary=True)] = (r[5], r[6], r[7])
        for i, members in groups(reads, ignore_linked_read, linked_read_cutoff):
            blocks = score(reads, members, table, ploidy)
            if not blocks:
                continue
            if len(blocks) > 1:
                multi += 1
            top = max(max(s) for _, s in blocks)
            choices = [choose(b, s) for b, s in blocks if max(s) == top]  # (IndexError for ploidy < 2)
            ht, q, block = choices[0]
            if len(members) > 1 and len(choices) > 1:
                loose.append(([representation(reads[j]) for j in members], reads[i][4] if not ignore_linked_read else "", reads[i][5],
                              [c if c[1] != 0 else None for c in choices]))
            if q == 0:
                continue
            if not ignore_linked_read and reads[i][4]:
                bx_out[reads[i][4]].append((reads[i][5], ht, block))
            for j in members:
                r2h[representation(reads[j])] = (ht, q, block)
    return bx_out, r2h, multi, primary, loose
