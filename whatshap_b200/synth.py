"""Deterministic synthetic ReadSets for the BASELINE.json configurations (SURVEY.md §8(d)).

There is no reference generator: the reference ships no benchmark for this path.  These
generators emit the *flat* problem (`FlatProblem`, the arrays of the C ABI) directly, in the read
order `ReadSet.sort()` would produce (sorted by first position), which is what `whatshap phase` hands
to `PedigreeDPTable` (whatshap/cli/phase.py:542-610).
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np

from ._abi import FlatProblem, GT_OTHER

#: seeds fixed by SURVEY.md §8(d)
SEEDS = {"cfg2": 20250915, "cfg3": 20250920, "cfg3g": 20250921, "cfg4": 20250925, "cfg5": 20250935}


def _csr_from_spans(first: np.ndarray, last: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """CSR offsets and column indices for reads covering [first, last] without gaps."""
    lens = (last - first + 1).astype(np.int64)
    off = np.zeros(first.size + 1, np.uint64)
    np.cumsum(lens, out=off[1:])
    nnz = int(off[-1])
    rid = np.repeat(np.arange(first.size), lens)
    within = np.arange(nnz) - np.repeat(off[:-1].astype(np.int64), lens)
    cols = (first[rid] + within).astype(np.uint32)
    return off, cols


def geometric_blocks(n: int, mean: float, seed: int, minimum: int = 2) -> np.ndarray:
    """Block lengths ~ Geometric(mean) summing to n (SURVEY.md 8(d): the load-balance variant of cfg3)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    lens, total = [], 0
    while total < n:
        b = max(minimum, int(rng.geometric(1.0 / mean)))
        b = min(b, n - total)
        if n - total - b in range(1, minimum):  # do not leave a stub shorter than `minimum`
            b = n - total
        lens.append(b)
        total += b
    return np.array(lens, np.int64)


def _window_spans(n: int, c: int, stride: int, block_len) -> Tuple[np.ndarray, np.ndarray]:
    """Read spans so that every column has exactly `c` active reads and no read crosses a
    block boundary.  Reads are ordered by (first column, start), i.e. ReadSet order.
    `block_len`: one length for all blocks, or the sequence of block lengths (summing to n)."""
    L = c * stride
    firsts, lasts = [], []
    if np.ndim(block_len) == 0:
        starts = list(range(0, n, int(block_len)))
        lengths = [min(int(block_len), n - b0) for b0 in starts]
    else:
        lengths = [int(b) for b in block_len]
        assert sum(lengths) == n, "block lengths must sum to the number of columns"
        starts = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(int).tolist()
    for b0, B in zip(starts, lengths):
        s = np.arange(-(L - stride), B, stride)
        f = np.maximum(s, 0)
        l = np.minimum(s + L - 1, B - 1)
        keep = (l - f + 1) >= 2  # reads with < 2 variants are dropped upstream (cli/phase.py:518)
        firsts.append(f[keep] + b0)
        lasts.append(l[keep] + b0)
    if not firsts:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(firsts).astype(np.int64), np.concatenate(lasts).astype(np.int64)


def sliding_window(
    n: int,
    c: int,
    stride: int = 1,
    block_len=500,
    err: float = 0.05,
    seed: int = 0,
    gap: float = 0.0,
    max_phred: int = 40,
) -> FlatProblem:
    """Single diploid individual, all sites heterozygous (trusted), coverage exactly `c` (fewer where a
    block is shorter than a read)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    first, last = _window_spans(n, c, stride, block_len)
    off, cols = _csr_from_spans(first, last)
    nnz = cols.size
    lens = (last - first + 1).astype(np.int64)
    truth = rng.integers(0, 2, n, dtype=np.uint8)
    read_hap = rng.integers(0, 2, first.size, dtype=np.uint8)
    flips = (rng.random(nnz) < err).astype(np.uint8)
    allele = truth[cols] ^ np.repeat(read_hap, lens) ^ flips
    phred = rng.integers(1, max_phred + 1, nnz, dtype=np.uint32)
    if gap > 0.0:
        drop = rng.random(nnz) < gap
        starts = off[:-1].astype(np.int64)
        ends = off[1:].astype(np.int64) - 1
        drop[starts] = False
        drop[ends] = False
        keep = ~drop
        new_lens = np.add.reduceat(keep.astype(np.int64), starts)
        off = np.zeros(first.size + 1, np.uint64)
        np.cumsum(new_lens, out=off[1:])
        cols, allele, phred = cols[keep], allele[keep], phred[keep]
    recomb = np.full(n, 49, np.uint32)
    if n:
        recomb[0] = 0
    return FlatProblem(
        positions=(np.arange(n, dtype=np.uint32) + 1) * 1000,
        read_off=off,
        ent_col=cols,
        ent_allele=allele,
        ent_phred=phred,
        read_ind=np.zeros(first.size, np.uint32),
        recombcost=recomb,
        n_ind=1,
        distrust=False,
        gt=np.ones((1, n), np.uint8),
    )


def trio(
    n: int,
    c_per_sample: int = 5,
    block_len: int = 500,
    err: float = 0.05,
    seed: int = 0,
    recomb_every: int = 5000,
    max_phred: int = 40,
) -> FlatProblem:
    """Father, mother, child (indices 0,1,2; one trio), `c_per_sample` reads per sample per column."""
    rng = np.random.Generator(np.random.PCG64(seed))
    f1, l1 = _window_spans(n, c_per_sample, 1, block_len)
    m = f1.size
    first = np.concatenate([f1, f1, f1])
    last = np.concatenate([l1, l1, l1])
    ind = np.repeat(np.arange(3, dtype=np.uint32), m)
    start_key = np.concatenate([np.arange(m)] * 3)
    order = np.lexsort((ind, start_key, first))  # ReadSet order: by first column, then deterministic
    first, last, ind = first[order], last[order], ind[order]
    off, cols = _csr_from_spans(first, last)
    lens = (last - first + 1).astype(np.int64)
    nnz = cols.size
    # parental haplotypes; child inherits one haplotype per parent with rare recombination
    hap = rng.integers(0, 2, (2, 2, n), dtype=np.uint8)  # [parent][haplotype][col]
    sel = np.zeros((2, n), np.uint8)
    for par in range(2):
        cur = int(rng.integers(0, 2))
        brk = rng.random(n) < (1.0 / max(recomb_every, 1))
        for k in range(n):
            if brk[k]:
                cur ^= 1
            sel[par, k] = cur
    child = np.stack([np.where(sel[0] == 0, hap[0, 0], hap[0, 1]), np.where(sel[1] == 0, hap[1, 0], hap[1, 1])])
    haps = np.stack([hap[0], hap[1], child])  # [ind][haplotype][col]
    gt = (haps[:, 0, :] + haps[:, 1, :]).astype(np.uint8)
    read_hap = rng.integers(0, 2, first.size, dtype=np.uint8)
    flips = (rng.random(nnz) < err).astype(np.uint8)
    rid = np.repeat(np.arange(first.size), lens)
    allele = haps[ind[rid], read_hap[rid], cols] ^ flips
    phred = rng.integers(1, max_phred + 1, nnz, dtype=np.uint32)
    recomb = np.full(n, 49, np.uint32)
    if n:
        recomb[0] = 0
    return FlatProblem(
        positions=(np.arange(n, dtype=np.uint32) + 1) * 1000,
        read_off=off,
        ent_col=cols,
        ent_allele=allele.astype(np.uint8),
        ent_phred=phred,
        read_ind=ind,
        recombcost=recomb,
        n_ind=3,
        trios=np.array([0, 1, 2], np.uint32),
        distrust=False,
        gt=gt,
    )


def nuclear_family(
    n: int,
    children: int = 1,
    c_per_sample: int = 5,
    block_len: int = 500,
    err: float = 0.05,
    seed: int = 0,
    recomb_every: int = 5000,
    max_phred: int = 40,
) -> FlatProblem:
    """Father, mother and `children` children (indices 0, 1, 2 ..; one trio per child, T = 4^children), shaped like `trio`:
    `c_per_sample` reads per sample per column.  (`trio` stays as it is: cfg5's inputs must not change.)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    n_ind = 2 + children
    f1, l1 = _window_spans(n, c_per_sample, 1, block_len)
    m = f1.size
    first = np.concatenate([f1] * n_ind)
    last = np.concatenate([l1] * n_ind)
    ind = np.repeat(np.arange(n_ind, dtype=np.uint32), m)
    start_key = np.concatenate([np.arange(m)] * n_ind)
    order = np.lexsort((ind, start_key, first))  # ReadSet order: by first column, then deterministic
    first, last, ind = first[order], last[order], ind[order]
    off, cols = _csr_from_spans(first, last)
    lens = (last - first + 1).astype(np.int64)
    nnz = cols.size
    hap = rng.integers(0, 2, (2, 2, n), dtype=np.uint8)  # [parent][haplotype][col]
    kids = []
    for _ in range(children):  # each child inherits one haplotype per parent with rare recombination
        sel = np.zeros((2, n), np.uint8)
        for par in range(2):
            brk = rng.random(n) < (1.0 / max(recomb_every, 1))
            sel[par] = (int(rng.integers(0, 2)) + np.cumsum(brk)) & 1
        kids.append(np.stack([np.where(sel[0] == 0, hap[0, 0], hap[0, 1]), np.where(sel[1] == 0, hap[1, 0], hap[1, 1])]))
    haps = np.stack([hap[0], hap[1]] + kids)  # [ind][haplotype][col]
    gt = (haps[:, 0, :] + haps[:, 1, :]).astype(np.uint8)
    read_hap = rng.integers(0, 2, first.size, dtype=np.uint8)
    flips = (rng.random(nnz) < err).astype(np.uint8)
    rid = np.repeat(np.arange(first.size), lens)
    allele = haps[ind[rid], read_hap[rid], cols] ^ flips
    phred = rng.integers(1, max_phred + 1, nnz, dtype=np.uint32)
    recomb = np.full(n, 49, np.uint32)
    if n:
        recomb[0] = 0
    return FlatProblem(
        positions=(np.arange(n, dtype=np.uint32) + 1) * 1000,
        read_off=off,
        ent_col=cols,
        ent_allele=allele.astype(np.uint8),
        ent_phred=phred,
        read_ind=ind,
        recombcost=recomb,
        n_ind=n_ind,
        trios=np.array([[0, 1, 2 + i] for i in range(children)], np.uint32).reshape(-1),
        distrust=False,
        gt=gt,
    )


def config(name: str, n: Optional[int] = None) -> FlatProblem:
    """The four GPU configurations of BASELINE.json (cfg2..cfg5) and the ragged variant of cfg3; `n` overrides the column count."""
    if name == "cfg2":
        return sliding_window(n or 10_000, 15, block_len=500, seed=SEEDS[name])
    if name == "cfg3":
        return sliding_window(n or 50_000, 20, block_len=500, seed=SEEDS[name])
    if name == "cfg3g":  # cfg3 with block lengths ~ Geometric(mean 500): load balance over SMs and GPUs (SURVEY.md 8(d))
        nn = n or 50_000
        return sliding_window(nn, 20, block_len=geometric_blocks(nn, 500.0, SEEDS[name]), seed=SEEDS[name])
    if name == "cfg4":
        nn = n or 50_000
        return sliding_window(nn, 25, block_len=nn, seed=SEEDS[name])
    if name == "cfg5":
        return trio(n or 20_000, 5, block_len=500, seed=SEEDS[name])
    raise KeyError(name)


PEDIGREES = {
    # name: (n_ind, trios)
    "single": (1, []),
    "two_unrelated": (2, []),
    "trio": (3, [0, 1, 2]),
    "trio_child_first": (3, [1, 2, 0]),
    "quartet": (4, [0, 1, 2, 0, 1, 3]),
    "three_generations": (5, [0, 1, 2, 2, 3, 4]),
    "three_children": (5, [0, 1, 2, 0, 1, 3, 0, 1, 4]),             # T = 64
    "four_children": (6, [0, 1, 2, 0, 1, 3, 0, 1, 4, 0, 1, 5]),     # T = 256, the largest of the two-pass and genotyping paths (five trios: DESIGN §4.7)
}


def random_problem(
    rng: np.random.Generator,
    n_cols: int,
    max_cov: int,
    pedigree: str = "single",
    distrust: bool = False,
    max_phred: int = 5,
    gap: float = 0.15,
    mean_len: float = 4.0,
    conflict_free: bool = True,
    hom_rate: float = 0.2,
    burst: int = 3,
) -> FlatProblem:
    """Irregular instance for fuzzing: random spans, interior gaps, tie-heavy small weights,
    blank (allele 2) entries, columns without reads, coverage capped at `max_cov`."""
    n_ind, trios = PEDIGREES[pedigree]
    cov = np.zeros(n_cols, np.int64)
    reads = []
    start = 0
    while start < n_cols:
        for _ in range(int(rng.integers(0, burst))):
            L = 1 + int(rng.geometric(1.0 / mean_len))
            end = min(n_cols - 1, start + L)
            if end == start:
                if start == 0:
                    continue
                # single-variant reads are legal input for the DP (tests only need >= 1 entry)
            if cov[start : end + 1].max() >= max_cov:
                continue
            cov[start : end + 1] += 1
            reads.append((start, end))
        start += int(rng.integers(1, 3))
    off = [0]
    cols, alle, phr, inds = [], [], [], []
    for (a, b) in reads:
        span = np.arange(a, b + 1)
        if span.size > 2 and gap > 0:
            keep = rng.random(span.size) >= gap
            keep[0] = keep[-1] = True
            span = span[keep]
        cols.append(span)
        al = rng.integers(0, 2, span.size)
        blank = rng.random(span.size) < 0.03
        al[blank] = 2
        alle.append(al)
        phr.append(rng.integers(0 if rng.random() < 0.2 else 1, max_phred + 1, span.size))
        inds.append(int(rng.integers(0, n_ind)))
        off.append(off[-1] + span.size)
    cat = lambda xs, dt: (np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt))
    # genotypes: Mendelian-consistent by construction unless conflict_free is False
    T = np.array(trios, np.int64).reshape(-1, 3)
    haps = rng.integers(0, 2, (n_ind, 2, n_cols))
    hom = rng.random((n_ind, n_cols)) < hom_rate
    haps[:, 1, :] = np.where(hom, haps[:, 0, :], haps[:, 1, :])
    # children inherit one haplotype per parent (parents are resolved before their children)
    done = set(i for i in range(n_ind) if i not in T[:, 2].tolist()) if T.size else set(range(n_ind))
    while len(done) < n_ind:
        for (f, m, c) in T:
            if c not in done and f in done and m in done:
                sf = rng.integers(0, 2, n_cols)
                sm = rng.integers(0, 2, n_cols)
                haps[c, 0, :] = np.where(sf == 0, haps[f, 0, :], haps[f, 1, :])
                haps[c, 1, :] = np.where(sm == 0, haps[m, 0, :], haps[m, 1, :])
                done.add(int(c))
    gt = (haps[:, 0, :] + haps[:, 1, :]).astype(np.uint8)
    if not conflict_free:
        noise = rng.random((n_ind, n_cols)) < 0.15
        gt = np.where(noise, rng.integers(0, 3, (n_ind, n_cols)), gt).astype(np.uint8)
        other = rng.random((n_ind, n_cols)) < 0.01
        gt = np.where(other, GT_OTHER, gt).astype(np.uint8)
    gl = None
    if distrust:
        gl = rng.integers(0, 12, (n_ind, n_cols, 3)).astype(np.float64)
        if rng.random() < 0.5:
            gl += rng.random((n_ind, n_cols, 3))  # fractional GLs exercise the unsigned += double truncation
    recomb = rng.integers(0, 8, n_cols).astype(np.uint32)
    return FlatProblem(
        positions=(np.arange(n_cols, dtype=np.uint32) + 1) * 10,
        read_off=np.array(off, np.uint64),
        ent_col=cat(cols, np.uint32),
        ent_allele=cat(alle, np.uint8),
        ent_phred=cat(phr, np.uint32),
        read_ind=np.array(inds, np.uint32),
        recombcost=recomb,
        n_ind=n_ind,
        trios=np.array(trios, np.uint32),
        distrust=distrust,
        gt=gt,
        gl=gl,
    )


def het_path_cost(prob: FlatProblem, path_index: np.ndarray) -> int:
    """MEC cost of a given bipartition path for a single individual with trusted genotypes:
    sum over columns of min(D, W - D), D = weight of the reads whose allele disagrees with the
    side they are on (closed form of pedigreecolumncostcomputer.cpp:101-114 for genotype 0/1);
    at a homozygous site (0/0 or 1/1) both sides carry its allele, so D alone.
    Used as a size-independent consistency check of large GPU runs: the reported optimal cost
    must be the cost of the reported path."""
    assert prob.n_ind == 1 and not prob.distrust and np.all(prob.gt <= 2)
    n = prob.n_cols
    lens = np.diff(prob.read_off.astype(np.int64))
    rid = np.repeat(np.arange(prob.n_reads), lens)
    first = prob.ent_col[prob.read_off[:-1].astype(np.int64)].astype(np.int64)
    last = prob.ent_col[prob.read_off[1:].astype(np.int64) - 1].astype(np.int64)
    # bit position of a read in column k = its rank among the active reads (reads are sorted by first position)
    cols = prob.ent_col.astype(np.int64)
    active = []
    nxt = 0
    bitpos = np.zeros(cols.size, np.int64)
    off = prob.read_off.astype(np.int64)
    cursor = off[:-1].copy()
    for k in range(n):
        active = [r for r in active if last[r] >= k]
        while nxt < prob.n_reads and first[nxt] == k:
            active.append(nxt)
            nxt += 1
        for j, r in enumerate(active):
            c = cursor[r]
            if c < off[r + 1] and cols[c] == k:
                bitpos[c] = j
                cursor[r] += 1
    side = (path_index.astype(np.int64)[cols] >> bitpos) & 1
    w = prob.ent_phred.astype(np.int64)
    al = prob.ent_allele.astype(np.int64)
    valid = al < 2
    gt = prob.gt[0].astype(np.int64)
    # het assignment (side 0 -> allele 0, side 1 -> allele 1); homozygous: allele gt / 2 on both sides
    mismatch = np.where(gt[cols] == 1, al != side, al != gt[cols] // 2) & valid
    D = np.bincount(cols, weights=np.where(mismatch, w, 0), minlength=n)
    W = np.bincount(cols, weights=np.where(valid, w, 0), minlength=n)
    return int(np.where(gt == 1, np.minimum(D, W - D), D).sum())


def genotyping_problem(
    rng: np.random.Generator,
    n_cols: int,
    max_cov: int,
    pedigree: str = "single",
    max_phred: int = 40,
    recomb_max: int = 30,
    prior: str = "random",
    **kw,
) -> FlatProblem:
    """Irregular instance for the forward-backward genotyping DP (GenotypeDPTable): as `random_problem`, but every
    read covers at least two variants (the reference asserts that, src/backwardcolumniterator.cpp:41), `gl` holds
    genotype PRIORS (probabilities; `uniform`, `random`, or `sparse` = with exact zeros) and recombination costs
    are phred-scaled probabilities."""
    base = random_problem(rng, n_cols, max_cov, pedigree, distrust=False, max_phred=max_phred, **kw)
    off = base.read_off.astype(np.int64)
    first = base.ent_col[off[:-1]] if base.n_reads else np.zeros(0, np.uint32)
    last = base.ent_col[off[1:] - 1] if base.n_reads else np.zeros(0, np.uint32)
    keep = np.nonzero(last > first)[0]
    sel = np.concatenate([np.arange(off[r], off[r + 1]) for r in keep]) if keep.size else np.zeros(0, np.int64)
    lens = (off[1:] - off[:-1])[keep]
    new_off = np.zeros(keep.size + 1, np.uint64)
    np.cumsum(lens, out=new_off[1:])
    n_ind = base.n_ind
    if prior == "uniform":
        gl = np.full((n_ind, n_cols, 3), 1.0 / 3.0)
    else:
        gl = rng.random((n_ind, n_cols, 3)) + 0.05
        if prior == "sparse":
            gl[rng.random((n_ind, n_cols, 3)) < 0.15] = 0.0
            gl[..., 1] = np.maximum(gl[..., 1], 0.05)  # keep every column feasible for every individual
        gl /= gl.sum(axis=2, keepdims=True)
    return FlatProblem(
        positions=base.positions,
        read_off=new_off,
        ent_col=base.ent_col[sel],
        ent_allele=base.ent_allele[sel],
        ent_phred=base.ent_phred[sel],
        read_ind=base.read_ind[keep],
        recombcost=rng.integers(0, recomb_max + 1, n_cols).astype(np.uint32),
        n_ind=n_ind,
        trios=base.trios,
        distrust=True,
        gt=None,
        gl=gl,
    )


def to_objects(prob: FlatProblem):
    """The container objects a `whatshap phase` run would hand to `PedigreeDPTable` for this flat problem:
    (ReadSet, recombcost list, Pedigree).  Trusted genotypes only (the generators above).  Used by bench.py to time the
    object-level call `PedigreeDPTable(readset, recombcost, pedigree)` + `get_super_reads()`."""
    from array import array

    from .core import Genotype, NumericSampleIds, Pedigree, Read, ReadSet

    positions = prob.positions.tolist()
    rs = ReadSet()
    off = prob.read_off.astype(np.int64)
    cols, alleles, phreds = prob.ent_col, prob.ent_allele.tolist(), prob.ent_phred.tolist()
    pos_of = prob.positions[cols].tolist()
    for r in range(prob.n_reads):
        read = Read("r%07d" % r, 60, 0, int(prob.read_ind[r]))
        a, b = int(off[r]), int(off[r + 1])
        read._pos, read._allele, read._quality = array("q", pos_of[a:b]), array("q", alleles[a:b]), array("q", phreds[a:b])
        rs.add(read)  # already in ReadSet order (sorted by first position)
    ids = NumericSampleIds()
    ped = Pedigree(ids)
    gts = [Genotype([0, 0]), Genotype([0, 1]), Genotype([1, 1])]
    for i in range(prob.n_ind):
        ids[i]
        ped.add_individual(i, [gts[g] for g in prob.gt[i].tolist()])
    tr = prob.trios.tolist()
    for t in range(prob.n_trios):
        ped.add_relationship(tr[3 * t], tr[3 * t + 1], tr[3 * t + 2])
    return rs, prob.recombcost.tolist(), ped
