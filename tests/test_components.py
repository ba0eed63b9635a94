"""Post-DP phase-set construction (reference: whatshap/graph.py:35-86, whatshap/cli/phase.py:71-113,
tests/test_graph.py)."""
import random

from whatshap_b200.components import ComponentFinder, find_components
from whatshap_b200.testhelpers import string_to_readset


def test_component_finder_minimum_is_representative():
    cf = ComponentFinder([1, 2, 3, 4, 5, "a", "b"][:5])
    assert [cf.find(i) for i in range(1, 6)] == [1, 2, 3, 4, 5]
    cf.merge(5, 4)
    cf.merge(3, 4)
    assert cf.find(5) == 3 and cf.find(4) == 3 and cf.find(1) == 1
    cf.merge(2, 1)
    cf.merge(5, 1)
    assert {cf.find(i) for i in range(1, 6)} == {1}


def test_find_components_reads_master_block_and_het_filter():
    reads = string_to_readset("""
      11
        00
         11
            01
    """)
    positions = [10, 20, 30, 40, 50, 70, 80]
    assert find_components(positions, reads) == {10: 10, 20: 10, 30: 30, 40: 30, 50: 30, 70: 70, 80: 70}
    merged = find_components(positions, reads, master_block=[20, 70])
    assert merged[80] == 10 and merged[30] == 30
    # restricting to heterozygous positions removes the bridge at 40
    het = {0: {10, 20, 30, 50, 70, 80}}
    assert find_components([10, 20, 30, 50, 70, 80], reads, heterozygous_positions=het)[50] == 50


def test_find_components_equals_graph_search_on_random_reads():
    rng = random.Random(3)
    from whatshap_b200 import Read, ReadSet

    for _ in range(30):
        n = rng.randint(2, 25)
        positions = sorted(rng.sample(range(1, 200), n))
        rs = ReadSet()
        adj = {p: set() for p in positions}
        for r in range(rng.randint(0, 12)):
            cover = sorted(rng.sample(positions, rng.randint(2, min(4, n))))
            read = Read(f"r{r}", 10, 0, 0)
            for p in cover:
                read.add_variant(p, rng.randint(0, 1), 1)
            rs.add(read)
            for p in cover[1:]:
                adj[cover[0]].add(p)
                adj[p].add(cover[0])
        got = find_components(positions, rs)
        for p in positions:  # flood fill
            seen, stack = {p}, [p]
            while stack:
                q = stack.pop()
                for t in adj[q]:
                    if t not in seen:
                        seen.add(t)
                        stack.append(t)
            assert got[p] == min(seen)


def _reference_functions():
    """`find_components` / `compute_overall_components` exactly as the reference defines them: their source text is cut
    out of whatshap/cli/phase.py of the WhatsHap tree at $WHATSHAP_REF (the module itself imports pysam, which is not
    installed) and executed with the reference's own ComponentFinder.  None where that tree is absent."""
    import ast
    import logging
    import os
    import typing

    from oracle.build_pyref import REF

    path = os.path.join(REF, "whatshap", "cli", "phase.py")
    if not os.access(path, os.R_OK):
        return None
    src = open(path).read()
    tree = ast.parse(src)
    wanted = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ("find_components", "compute_overall_components")]
    ns = {"logger": logging.getLogger("ref"), "__name__": "refphase"}
    ns.update({k: getattr(typing, k) for k in ("Sequence", "Optional", "Mapping", "Set", "Dict", "List")})
    gsrc = open(os.path.join(REF, "whatshap", "graph.py")).read()
    gns = {}
    exec(compile(gsrc, "graph.py", "exec"), gns)
    ns["ComponentFinder"] = gns["ComponentFinder"]
    ns["ReadSet"] = ns["NumericSampleIds"] = object
    for node in wanted:
        exec(compile(ast.Module([node], []), path, "exec"), ns)
    return ns["find_components"], ns["compute_overall_components"]


def test_compute_overall_components_equals_the_reference():
    """Against the reference's functions where its tree is present, else against their answers stored in
    tests/golden/components_answers.json (position -> component pairs, sorted)."""
    import golden_io
    from whatshap_b200 import NumericSampleIds, Read, ReadSet
    from whatshap_b200.components import compute_overall_components, phase_calls

    ref = _reference_functions()
    ref_overall = ref[1] if ref is not None else None
    rng = random.Random(11)
    for it in range(60):
        n = rng.randint(4, 30)
        positions = sorted(rng.sample(range(1, 400), n))
        family = ["child", "mother", "father"][: rng.choice([1, 3])]
        ids = NumericSampleIds()
        for s in family:
            ids[s]
        reads = ReadSet()
        for r in range(rng.randint(1, 25)):
            read = Read("r%d" % r, 60, 0, ids[rng.choice(family)])
            start = rng.randrange(n)
            for p in positions[start:start + rng.randint(1, 5)]:
                if rng.random() < 0.85:
                    read.add_variant(p, rng.randint(0, 1), rng.randint(1, 30))
            if len(read):
                reads.add(read)
        accessible = sorted(rng.sample(positions, rng.randint(2, n)))
        superreads_list = []
        for s in family:
            pair = ReadSet()
            alleles = [(rng.choice([0, 1, 3]), rng.choice([0, 1, 3])) for _ in positions]
            for h in range(2):
                sr = Read("superread_%d_0" % h, -1, -1, ids[s])
                for p, a in zip(positions, alleles):
                    sr.add_variant(p, a[h], 5)
                pair.add(sr)
            superreads_list.append(pair)
        homozygous = rng.sample(positions, rng.randint(0, n // 2))
        for distrust in (False, True):
            for genetic in (False, True):
                args = (accessible, reads, distrust, family, genetic, homozygous, ids, superreads_list)
                got = compute_overall_components(*args)
                live = sorted(ref_overall(*args).items()) if ref_overall else None
                want = golden_io.reference_answer("components", f"{it}/{distrust}/{genetic}", live)
                assert sorted([p, c] for p, c in got.items()) == want, (it, distrust, genetic)
        superreads, comps, phases = phase_calls(family, superreads_list, got, ids)
        assert list(superreads) == family and all(comps[s] is got for s in family)
        for s, pair in zip(family, superreads_list):
            assert phases[s] == {v0.position: (v0.allele, v1.allele) for v0, v1 in zip(*pair) if v0.allele != 3 and v1.allele != 3}
