"""The solver swap-in for the reference's OWN objects (whatshap_b200/adapters.py), checked against the real
`whatshap.core` extension (built by oracle/build_pyref.py from the WhatsHap tree at $WHATSHAP_REF, or prebuilt under
oracle/_ref/pyref):

 * real ReadSet / Pedigree objects flatten to exactly the arrays this package's own containers give;
 * the adapter class (constructor + three methods of whatshap/types.py) returns, as real whatshap.core
   Read/ReadSet objects, exactly what the real PedigreeDPTable returns — with the CPU checker standing
   in for the per-call CUDA solve so that the test needs no GPU.

The real classes' answers are stored under tests/golden/ (`golden_io.reference_answer`); without the binding the same
inputs are built from this package's containers and the adapters' answers are compared with the stored ones."""
import json
import sys

import numpy as np
import pytest

import golden_io
import test_pedigreephasing as tp
import test_phasing as ts
from test_gpu_real_containers import check_against_reference
from whatshap_b200 import adapters
from whatshap_b200 import core as mine
from whatshap_b200.testhelpers import string_to_readset, string_to_readset_pedigree


@pytest.fixture(scope="module")
def ref_core():
    """The reference binding, or None where it was neither built nor shipped prebuilt.  Where the WhatsHap tree is present the
    binding is imported from its build directory, which the compiled bridge (integration/) links against."""
    from oracle import build_pyref

    path = build_pyref.build()
    if path:
        sys.path.insert(0, path)
        import whatshap.core as core

        return core
    return build_pyref.shipped_core()


def to_real(core, rs):
    """Copy one of this package's ReadSets into a real whatshap.core.ReadSet."""
    out = core.ReadSet()
    for r in rs:
        read = core.Read(r.name, r.mapqs[0], r.source_id, r.sample_id)
        for v in r:
            read.add_variant(v.position, v.allele, v.quality)
        out.add(read)
    return out


def real_pedigree(core, case, recording):
    cls = adapters.recording_pedigree(core.Pedigree) if recording else core.Pedigree
    ped = cls(core.NumericSampleIds())
    for i, gts in enumerate(case["genotypes"]):
        genotypes = [core.Genotype([0] * (2 - g) + [1] * g) if 0 <= g <= 2 else core.Genotype([]) for g in gts]
        gls = [core.PhredGenotypeLikelihoods(g) for g in case["gls"][i]] if "gls" in case else None
        ped.add_individual("individual{}".format(i), genotypes, gls)
    for f, m, c in case["trios"]:
        ped.add_relationship("individual{}".format(f), "individual{}".format(m), "individual{}".format(c))
    return ped


@pytest.mark.parametrize("recording", [True, False])
@pytest.mark.parametrize("name", sorted(tp.CASES))
def test_adapter_on_real_objects_equals_real_dp_table(ref_core, checker, name, recording):
    case = tp.CASES[name]
    core = ref_core or mine
    my_rs = string_to_readset_pedigree(case["reads"]) if case["reads"].strip() else mine.ReadSet()
    real_rs = to_real(core, my_rs)
    ped = real_pedigree(core, case, recording)
    distrust, positions = case.get("distrust", False), case.get("positions")
    # 1. same flat arrays as this package's own containers
    flat, ids = adapters.flatten_objects(real_rs, case["recomb"], ped, distrust, positions)
    want = mine._flatten(my_rs, case["recomb"], tp.build_pedigree(case), distrust, positions)
    for field in ("positions", "read_off", "ent_col", "ent_allele", "ent_phred", "read_ind", "recombcost", "trios", "gt"):
        assert np.array_equal(getattr(flat, field), getattr(want, field)), field
    assert (flat.gl is None) == (want.gl is None) and (flat.gl is None or np.array_equal(flat.gl, want.gl))
    # 2. the swap-in class answers like the real one, in real objects
    Table = adapters.make_dp_table_class(core, solver=checker.solve)
    a = Table(real_rs, case["recomb"], ped, distrust, positions)
    recomb = list(case["recomb"]) + [case["recomb"][-1]] * 4  # the real class reads recombcost[k] unchecked
    b = ref_core.PedigreeDPTable(real_rs, recomb, ped, distrust, positions) if ref_core else None
    assert a.get_optimal_cost() == case["cost"]
    check_against_reference(f"pedigree/{name}/{recording}", a, b)


def test_single_individual_matrices_through_real_objects(ref_core, checker):
    core = ref_core or mine
    Table = adapters.make_dp_table_class(core, solver=checker.solve)
    for name in sorted(ts.MATRICES):
        reads, weights = ts.MATRICES[name]
        real_rs = to_real(core, string_to_readset(reads, weights))
        positions = real_rs.get_positions()
        for het in (True, False):
            ped = core.Pedigree(core.NumericSampleIds())
            gls = [None if het else core.PhredGenotypeLikelihoods([0, 0, 0])] * len(positions)
            ped.add_individual("individual0", [core.Genotype([0, 1])] * len(positions), gls)
            a = Table(real_rs, [1] * len(positions), ped, not het)
            b = ref_core.PedigreeDPTable(real_rs, [1] * len(positions), ped, not het) if ref_core else None
            check_against_reference(f"matrix/{name}/{het}", a, b)


def _one_individual_pedigree(n):
    ped = mine.Pedigree(mine.NumericSampleIds())
    ped.add_individual("sample", [mine.Genotype([0, 1])] * n)
    return ped


def test_flatten_errors_follow_the_reference_order():
    """The first offending read decides, and within a read the order in which the reference's constructor path
    would stumble: unknown sample, no variants, unsorted reads, unsorted variants, uncovered ends, bad allele."""
    rs = string_to_readset("""
      111
       101
    """)
    ped = _one_individual_pedigree(4)
    prob, ids = adapters.flatten_objects(rs, [1] * 4, ped)
    assert ids == [0] and prob.n_cols == 4 and prob.read_off.tolist() == [0, 3, 6] and prob.ent_col.tolist() == [0, 1, 2, 1, 2, 3]

    def with_read(build, **kw):
        out = mine.ReadSet()
        for r in rs:
            out.add(r)
        read = mine.Read("extra", 50, 0, kw.get("sample", 0))
        build(read)
        out.add(read)
        return out

    cases = [
        (lambda r: [r.add_variant(20, 0, 1), r.add_variant(30, 1, 1)], dict(sample=7), "Individual with ID 7 not present"),
        (lambda r: None, {}, "No variants present"),
        (lambda r: [r.add_variant(10, 0, 1), r.add_variant(30, 1, 1)], {}, "reads in ReadSet are not sorted"),
        (lambda r: [r.add_variant(30, 0, 1), r.add_variant(20, 1, 1), r.add_variant(40, 1, 1)], {}, "read with unsorted variants"),
        (lambda r: [r.add_variant(30, 0, 1), r.add_variant(40, 7, 1)], {}, "allele 7 is not 0, 1 or 2"),
    ]
    for build, kw, text in cases:
        with pytest.raises(RuntimeError, match=text):
            adapters.flatten_objects(with_read(build, **kw), [1] * 4, ped)
    with pytest.raises(RuntimeError, match="first/last variant position is not among the given positions"):
        adapters.flatten_objects(rs, [1] * 3, _one_individual_pedigree(3), positions=[10, 20, 30])
    # interior positions that are not DP columns are dropped (ColumnIterator skips them)
    rs2 = string_to_readset("""
      1111
      1 11
    """)
    prob, _ = adapters.flatten_objects(rs2, [1] * 3, _one_individual_pedigree(3), positions=[10, 30, 40])
    assert prob.read_off.tolist() == [0, 3, 6] and prob.ent_col.tolist() == [0, 1, 2, 0, 1, 2]


def test_compiled_bridge_reads_the_same_arrays_as_the_python_api(monkeypatch):
    """integration/whatshap_bridge.pyx (built against the reference tree) against the public-API walk.  Needs the
    WhatsHap source tree at $WHATSHAP_REF: the bridge is compiled against its .pxd files and headers."""
    import os
    import time

    from oracle import build_pyref

    tree = build_pyref.build()
    if not tree:
        pytest.skip("the WhatsHap source tree ($WHATSHAP_REF) is needed to compile the bridge")
    sys.path.insert(0, tree)
    import whatshap.core as ref_core

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "integration"))
    import build_bridge

    build_bridge.build(tree, tree)
    rng = np.random.default_rng(8)
    rs = ref_core.ReadSet()
    n_var = 3000
    for i in range(4000):
        read = ref_core.Read("r%d" % i, 60, int(rng.integers(0, 2)), 0)
        start = int(rng.integers(0, n_var - 2))
        for v in range(start, min(n_var, start + 2 + int(rng.geometric(0.1)))):
            if v == start or rng.random() > 0.1:
                read.add_variant(50 + 11 * v, int(rng.integers(0, 3)), int(rng.integers(0, 90)))
        if len(read) >= 1:
            rs.add(read)
    rs.sort()
    n = len(rs.get_positions())
    ped = ref_core.Pedigree(ref_core.NumericSampleIds())
    ped.add_individual("sample", [ref_core.Genotype([0, 1])] * n)
    assert adapters._bridge_for(rs) is not None, "the bridge was built but cannot be imported"
    t = time.perf_counter()
    fast, _ = adapters.flatten_objects(rs, [3] * n, ped)
    t_fast = time.perf_counter() - t
    monkeypatch.setattr(adapters, "_bridge_for", lambda readset: None)
    t = time.perf_counter()
    slow, _ = adapters.flatten_objects(rs, [3] * n, ped)
    t_slow = time.perf_counter() - t
    for field in ("positions", "read_off", "ent_col", "ent_allele", "ent_phred", "read_ind", "recombcost", "gt"):
        assert np.array_equal(getattr(fast, field), getattr(slow, field)), field
    print("flatten_objects: compiled bridge %.3f s, public Python API %.3f s" % (t_fast, t_slow))


def test_prior_genotyper_equals_the_real_binding(ref_core):
    """`compute_genotypes` (core.pyx:602-617) of this package and of the real extension on the same reads: same
    Genotype objects (by alleles), same likelihood tuples, bit for bit."""
    rng = np.random.default_rng(17)
    for it in range(20):
        rows = []
        n_cols = int(rng.integers(3, 12))
        for _r in range(int(rng.integers(2, 14))):
            start = int(rng.integers(0, n_cols - 1))
            length = int(rng.integers(2, n_cols - start + 1))
            rows.append(" " * start + "".join(rng.choice(list("01"), length)))
        weights = "\n".join("".join(str(int(rng.integers(1, 10))) if ch != " " else " " for ch in row) for row in rows)
        rs = string_to_readset("\n".join(rows), weights, scale_quality=int(rng.choice([1, 5, 10])))
        rs.sort()
        mine_gt, mine_gl = mine.compute_genotypes(rs)
        live = None
        if ref_core is not None:
            real = to_real(ref_core, rs)
            real.sort()
            real_gt, real_gl = ref_core.compute_genotypes(real)
            live = [[g.as_vector() for g in real_gt], [list(x) for x in real_gl]]
        want = golden_io.reference_answer("adapters", f"genotyper/{it}", live)
        assert [[g.as_vector() for g in mine_gt], [list(x) for x in mine_gl]] == want, it


def test_prior_genotyper_adapter_on_real_objects(ref_core):
    """`adapters.make_compute_genotypes` fed the reference's real ReadSet returns what the real binding returns."""
    rs = string_to_readset("""
      1  11010
      00 00101
      001 01110
       1    111
       111 0101
    """, """
      5  92341
      11 13452
      334 98765
       2    121
       999 1111
    """)
    core = ref_core or mine
    real = to_real(core, rs)
    real.sort()
    compute = adapters.make_compute_genotypes(core)
    for positions in (None, list(real.get_positions())):
        got_gt, got_gl = compute(real, positions)
        live = None
        if ref_core is not None:
            want_gt, want_gl = ref_core.compute_genotypes(real, positions)
            live = [[g.as_vector() for g in want_gt], [list(x) for x in want_gl]]
        want = golden_io.reference_answer("adapters", f"genotyper_adapter/{positions is None}", live)
        assert [[g.as_vector() for g in got_gt], [list(x) for x in got_gl]] == want
        assert all(isinstance(g, core.Genotype) for g in got_gt)


@pytest.mark.parametrize("name", sorted(n for n in tp.CASES if not tp.CASES[n].get("distrust") and tp.CASES[n]["reads"].strip()
                                        and tp.CASES[n].get("positions") is None))
def test_heuristic_adapter_on_real_objects_equals_the_real_class(ref_core, name):
    """`make_heuristic_class` (the host solver `whmec_heuristic`) against the REAL whatshap.core.PedMecHeuristic on real objects:
    same super-reads, transmission vector, bipartition and mutation list (core.pyx:674-734)."""
    case = tp.CASES[name]
    core = ref_core or mine
    my_rs = string_to_readset_pedigree(case["reads"])
    real_rs = to_real(core, my_rs)
    ped = real_pedigree(core, case, False)
    recomb = [max(int(x), 1) for x in case["recomb"]]  # a zero mutation cost leaves the reference undefined with distrusted genotypes
    recomb = recomb + [recomb[-1]] * 4
    Mine = adapters.make_heuristic_class(core)

    def answers(h):
        superreads, tv = h.get_super_reads()
        return {"superreads": [[[x.name, x.sample_id, [[v.position, v.allele, v.quality] for v in x]] for x in rs] for rs in superreads],
                "tv": list(tv), "partitioning": list(h.get_optimal_partitioning()),
                "mutations": [[list(m) for m in ms] for ms in h.get_mutations()], "cost": h.get_optimal_cost()}

    for row_limit in (2, 64):
        a = Mine(real_rs, recomb, ped, row_limit)
        live = None
        if ref_core is not None:
            b = ref_core.PedMecHeuristic(real_rs, recomb[: len(real_rs.get_positions())], ped, row_limit)
            live = answers(b)
        want = golden_io.reference_answer("adapters", f"heuristic/{name}/{row_limit}", live)
        assert json.loads(json.dumps(answers(a))) == want, (name, row_limit)
