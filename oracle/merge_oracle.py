"""Plain-Python restatement of ReadMerger.merge (`whatshap phase --merge-reads`), written from its rules without networkx.  The CPU
reference for whatshap_b200.merge and whmec_merge_reads.

A read is a list of (position, allele, quality).  `merge` returns the merged reads as (name, entries) in output order, or raises
what the reference raises first."""
from math import log


def thresholds(error_rate, positive_threshold, negative_threshold):
    base = (1 - error_rate) / (error_rate / 3)
    return 1 + int(log(positive_threshold, base)), 1 + int(log(negative_threshold, base))


def partners(begins, ends):
    """kill[j]: the first k > j with begins[k] >= ends[j] (len(begins) if none); j meets every i in (j, kill[j])."""
    n = len(begins)
    kill = []
    for j in range(n):
        k = j + 1
        while k < n and begins[k] < ends[j]:
            k += 1
        kill.append(k)
    return kill


def overlap(alleles_j, begin_j, alleles_i, begin_i):
    """(match, mismatch) of alleles_j[begin_i - begin_j:] against alleles_i."""
    part = alleles_j[begin_i - begin_j:]
    n = min(len(part), len(alleles_i))
    assert n > 0
    mismatch = sum(1 for a, b in zip(part, alleles_i) if a != b)
    return n - mismatch, mismatch


def shortest_path(adj, u, v):
    """networkx's bidirectional_shortest_path: expand the smaller fringe (forward on ties), neighbours in adjacency order, stop
    at the first node the other side has reached.  None when there is no path."""
    pred, succ = {u: None}, {v: None}
    fwd, rev = [u], [v]
    meet = None
    while fwd and rev and meet is None:
        if len(fwd) <= len(rev):
            level, fwd = fwd, []
            for x in level:
                for w in adj[x]:
                    if w not in pred:
                        fwd.append(w)
                        pred[w] = x
                    if w in succ:
                        meet = w
                        break
                if meet is not None:
                    break
        else:
            level, rev = rev, []
            for x in level:
                for w in adj[x]:
                    if w not in succ:
                        succ[w] = x
                        rev.append(w)
                    if w in pred:
                        meet = w
                        break
                if meet is not None:
                    break
    if meet is None:
        return None
    path, w = [], meet
    while w is not None:
        path.append(w)
        w = pred[w]
    path.reverse()
    w = succ[path[-1]]
    while w is not None:
        path.append(w)
        w = succ[w]
    return path


def components(n, adj):
    """Each node's least component member."""
    rep = list(range(n))
    seen = [False] * n
    for s in range(n):
        if seen[s]:
            continue
        stack, members = [s], []
        seen[s] = True
        while stack:
            x = stack.pop()
            members.append(x)
            for w in adj[x]:
                if not seen[w]:
                    seen[w] = True
                    stack.append(w)
        for x in members:
            rep[x] = s
    return rep


def edges(reads, error_rate, max_error_rate, positive_threshold, negative_threshold):
    """The blue edges {(j, i): match - mismatch} and the not-blue edges [(j, i)], j < i; raises the reference's errors."""
    thr_diff, thr_neg_diff = thresholds(error_rate, positive_threshold, negative_threshold)
    begins, ends, alleles = [], [], []
    for read in reads:
        for _, allele, _ in read:
            assert allele in (0, 1)
        begins.append(read[0][0])  # IndexError for an empty read
        ends.append(begins[-1] + len(read))
        alleles.append([a for _, a, _ in read])
    kill = partners(begins, ends)
    blue, notblue = {}, []
    for j in range(len(reads)):
        for i in range(j + 1, kill[j]):
            m, mm = overlap(alleles[j], begins[j], alleles[i], begins[i])
            if m + mm >= thr_neg_diff and min(m, mm) / (m + mm) <= max_error_rate and m - mm >= thr_diff:
                blue[(j, i)] = m - mm
                if mm - m >= thr_neg_diff:
                    notblue.append((j, i))
    return blue, sorted(notblue)


def merge(reads, error_rate=0.15, max_error_rate=0.25, positive_threshold=1000000, negative_threshold=1000, counters=None):
    n = len(reads)
    blue, notblue = edges(reads, error_rate, max_error_rate, positive_threshold, negative_threshold)
    adj = [[] for _ in range(n)]
    for j, i in sorted(blue):
        adj[j].append(i)
        adj[i].append(j)
    for a in adj:
        a.sort()
    before = components(n, adj)
    removed = 0
    for u, v in notblue:
        if before[u] != before[v]:
            continue
        while True:
            path = shortest_path(adj, u, v)
            if path is None:
                break
            steps = list(zip(path[:-1], path[1:]))
            a, b = min(steps, key=lambda e: blue[(min(e), max(e))])
            adj[a].remove(b)
            adj[b].remove(a)
            removed += 1
    rep = components(n, adj)
    size = {}
    for r in rep:
        size[r] = size.get(r, 0) + 1
    sums = {}
    for r in range(n):
        if size[rep[r]] >= 2:
            for pos, allele, quality in reads[r]:
                z = sums.setdefault(rep[r], {}).setdefault(pos, [0, 0])
                z[allele] += quality
    out = []
    for r in range(n):
        if size[rep[r]] >= 2:
            if rep[r] == r:
                out.append(("read%d" % r, [(p, 0 if z[0] >= z[1] else 1, abs(z[1] - z[0])) for p, z in sorted(sums[r].items())]))
        else:
            out.append(("read%d" % r, list(reads[r])))
    if counters is not None:
        counters.update(blue_edges=len(blue), notblue_edges=len(notblue), removed_edges=removed,
                        merged_components=sum(1 for r, s in size.items() if s >= 2), output_reads=len(out),
                        pairs=sum(k - j - 1 for j, k in enumerate(partners([r[0][0] for r in reads], [r[0][0] + len(r) for r in reads]))))
    return out
