"""Data containers of the operator surface (Read, ReadSet, Genotype, PhredGenotypeLikelihoods,
Pedigree, NumericSampleIds): behaviour follows whatshap/core.pyx and the reference's
tests/test_reads.py / tests/test_pedigree.py."""
import copy
import pickle

import pytest

from whatshap_b200 import (
    Genotype, NumericSampleIds, Pedigree, PhredGenotypeLikelihoods, Read, ReadSet, Variant, binomial_coefficient,
)
from whatshap_b200.core import _flatten, _index_to_alleles
from whatshap_b200.testhelpers import canonic_index_list_to_biallelic_gt_list, string_to_readset


def make_read(name, variants, **kw):
    r = Read(name, 15, **kw)
    for v in variants:
        r.add_variant(*v)
    return r


def test_read_basics():
    r = make_read("name", [(100, 1, 37), (23, 0, 99)])
    assert r.name == "name" and r.mapqs == (15,) and len(r) == 2
    assert not r.is_sorted()
    assert r[0] == Variant(position=100, allele=1, quality=37)
    assert r[-1].position == 23
    r.sort()
    assert r.is_sorted() and [v.position for v in r] == [23, 100]
    assert 100 in r and 5 not in r
    r[0] = Variant(position=24, allele=1, quality=3)
    assert r[0].quality == 3
    with pytest.raises(IndexError):
        r[2]
    with pytest.raises(ValueError):
        r[0] = (1, 2, 3)
    r.add_mapq(20)
    assert r.mapqs == (15, 20)
    assert "name='name'" in repr(r)


def test_read_duplicate_variant_raises_on_sort():
    r = make_read("dup", [(10, 0, 1), (10, 1, 1)])
    with pytest.raises(RuntimeError, match="Duplicate variant in read dup at position 10"):
        r.sort()


def test_read_tags_and_pickle():
    r = Read("x", 10, 1, 2, 77, "BX", 1, 5, "chr1", "sub", True, 99, True)
    r.add_variant(5, 1, 9)
    assert (r.source_id, r.sample_id, r.reference_start, r.reference_end) == (1, 2, 77, 99)
    assert r.BX_tag == "BX" and r.HP_tag == 1 and r.PS_tag == 5 and r.chromosome == "chr1"
    assert r.has_BX_tag() and r.is_supplementary and r.is_reverse and r.sub_alignment_id == "sub"
    r2 = pickle.loads(pickle.dumps(r))
    assert repr(r2) == repr(r)


def test_readset_add_copies_and_rejects_duplicates():
    rs = ReadSet()
    r = make_read("a", [(10, 0, 1), (20, 1, 1)])
    rs.add(r)
    r.add_variant(30, 0, 1)
    assert len(rs[0]) == 2  # the set holds a copy
    with pytest.raises(RuntimeError, match="duplicate read name"):
        rs.add(make_read("a", [(10, 0, 1)]))
    rs.add(make_read("a", [(10, 0, 1)], source_id=1))  # same name, other source is fine
    assert rs[(1, "a")].source_id == 1
    with pytest.raises(KeyError):
        rs[(2, "a")]
    with pytest.raises(NotImplementedError):
        rs["a"]


def test_readset_sort_subset_positions():
    rs = ReadSet()
    rs.add(make_read("late", [(30, 0, 1), (50, 1, 1)]))
    rs.add(make_read("early", [(10, 0, 1), (20, 1, 1)]))
    rs.add(make_read("empty", []))
    rs.sort()
    assert [r.name for r in rs] == ["empty", "early", "late"]
    assert rs.get_positions() == [10, 20, 30, 50]
    sub = rs.subset([2, 1, 2])
    assert [r.name for r in sub] == ["early", "late"]
    assert str(rs).startswith("ReadSet:\n")
    assert [r.name for r in pickle.loads(pickle.dumps(rs))] == ["empty", "early", "late"]


def test_readset_sort_ties_follow_the_reference_comparator():
    """Reads with equal first position are ordered by libstdc++'s hash (src/readset.h:39-66): checked against
    ReadSet::sort() itself where the compiled reference is present, else against the order it gave, stored in
    tests/golden/containers_answers.json."""
    import ctypes as C

    import golden_io
    from oracle import checker as ck

    ref = ck.reference()
    names = ["Read {}".format(i) for i in range(40)] + ["r%07d" % i for i in range(40)]
    firsts = [10 * (i % 3) for i in range(len(names))]
    sources = [i % 2 for i in range(len(names))]
    rs = ReadSet()
    for n, f, s in zip(names, firsts, sources):
        rs.add(make_read(n, [(f, 0, 1), (f + 5, 1, 1)], source_id=s))
    rs.sort()
    live = None
    if ref is not None:
        arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
        order = (C.c_uint32 * len(names))()
        ref.lib.whref_sort_order(len(names), arr, (C.c_int32 * len(names))(*sources), (C.c_int32 * len(names))(*firsts), order)
        live = list(order)
    order = golden_io.reference_answer("containers", "sort_ties", live)
    assert [r.name for r in rs] == [names[i] for i in order]


def test_genotype():
    assert str(Genotype([1, 0])) == "0/1" and str(Genotype([])) == "."
    assert Genotype([0, 1]) == Genotype([1, 0]) and Genotype([0, 0]) != Genotype([0, 1])
    assert [Genotype(a).get_index() for a in ([0, 0], [0, 1], [1, 1], [0, 2], [1, 2], [2, 2])] == [0, 1, 2, 3, 4, 5]
    assert Genotype([0, 0, 1, 2]).get_index() == 6
    assert Genotype([1, 0]).as_vector() == [1, 0]
    assert Genotype([1, 1]).is_homozygous() and not Genotype([0, 1]).is_homozygous() and not Genotype([]).is_homozygous()
    assert Genotype([0, 1]).is_diploid_and_biallelic() and not Genotype([0, 2]).is_diploid_and_biallelic()
    assert Genotype([]).is_none() and Genotype([0, 1, 1]).get_ploidy() == 3
    assert Genotype([0, 0]) < Genotype([0, 1])
    assert pickle.loads(pickle.dumps(Genotype([0, 1, 3]))) == Genotype([0, 1, 3])
    assert copy.deepcopy(Genotype([1, 2])) == Genotype([1, 2])
    assert len({Genotype([0, 1]), Genotype([1, 0])}) == 1
    for ploidy in range(1, 5):
        for index in range(12):
            assert Genotype(_index_to_alleles(index, ploidy)).get_index() == index
    with pytest.raises(RuntimeError):
        Genotype([16, 0])
    assert binomial_coefficient(5, 2) == 10 and binomial_coefficient(2, 5) == 0


def test_phred_genotype_likelihoods():
    gl = PhredGenotypeLikelihoods([3, 0, 7.5])
    assert len(gl) == 3 and list(gl) == [3, 0, 7.5]
    assert gl[Genotype([0, 1])] == 0 and gl[Genotype([1, 1])] == 7.5
    assert gl.genotypes() == [Genotype([0, 0]), Genotype([0, 1]), Genotype([1, 1])]
    assert gl == PhredGenotypeLikelihoods([3, 0, 7.5])
    assert len(PhredGenotypeLikelihoods([0] * 6, ploidy=2, nr_alleles=3)) == 6
    with pytest.raises(RuntimeError, match="wrong number"):
        PhredGenotypeLikelihoods([0, 0])


def test_numeric_sample_ids():
    ids = NumericSampleIds()
    assert ids["a"] == 0 and ids["b"] == 1 and ids["a"] == 0 and len(ids) == 2
    assert ids.inverse_mapping() == {0: "a", 1: "b"}
    ids.freeze()
    with pytest.raises(KeyError):
        ids["c"]
    assert pickle.loads(pickle.dumps(ids)).mapping == ids.mapping


def test_pedigree():
    ped = Pedigree(NumericSampleIds())
    ped.add_individual("f", canonic_index_list_to_biallelic_gt_list([0, 1, 2]), [None, PhredGenotypeLikelihoods([1, 2, 3]), None])
    ped.add_individual("m", canonic_index_list_to_biallelic_gt_list([1, 1, 1]))
    ped.add_individual("c", canonic_index_list_to_biallelic_gt_list([0, 1, 1]))
    ped.add_relationship("f", "m", "c")
    assert len(ped) == 3 and ped.variant_count == 3
    assert ped.genotype("f", 2) == Genotype([1, 1])
    assert ped.genotype_likelihoods("f", 0) is None and list(ped.genotype_likelihoods("f", 1)) == [1, 2, 3]
    assert "triples by index (father,mother,child): (0,1,2)" in str(ped)
    with pytest.raises(TypeError):
        ped.add_individual("x", [1, 1, 1])


def test_flatten_restates_column_iterator_inputs():
    """ReadSet -> CSR arrays of the C ABI: columns are ranks of positions, gaps stay implicit,
    interior variants outside `positions` are skipped, reads map to pedigree indices."""
    rs = string_to_readset("""
      1 1
       010
    """)
    ids = NumericSampleIds()
    ped = Pedigree(ids)
    ped.add_individual("s", canonic_index_list_to_biallelic_gt_list([1, 1, 2, 0]))
    p = _flatten(rs, [0, 5, 5, 5], ped, False, None)
    assert p.positions.tolist() == [10, 20, 30, 40]
    assert p.read_off.tolist() == [0, 2, 5] and p.ent_col.tolist() == [0, 2, 1, 2, 3]
    assert p.gt.tolist() == [[1, 1, 2, 0]] and p.read_ind.tolist() == [0, 0]
    # explicit positions: an interior variant whose position is not a column is skipped
    rs2 = string_to_readset("""
      111
      01
    """)
    p2 = _flatten(rs2, [1, 1, 1], ped, False, [10, 20, 30, 40])
    assert p2.n_cols == 4 and p2.ent_col.tolist() == [0, 1, 2, 0, 1]
    rs3 = ReadSet()
    rs3.add(make_read("gap", [(10, 1, 2), (25, 0, 2), (30, 1, 2)]))
    p3 = _flatten(rs3, [1, 1, 1], ped, False, [10, 20, 30])
    assert p3.ent_col.tolist() == [0, 2] and p3.ent_phred.tolist() == [2, 2]
    # short recombination-cost lists are padded with their last value (see core._flatten)
    assert _flatten(rs2, [7], ped, False, [10, 20, 30]).recombcost.tolist() == [7, 7, 7]
    with pytest.raises(RuntimeError, match="not present in pedigree"):
        other = ReadSet()
        other.add(make_read("q", [(10, 0, 1), (20, 0, 1)], sample_id=9))
        _flatten(other, [1, 1], ped, False, None)


def _columns_from_objects(rs):
    """What ReadSet._flat_columns must return: collected again from the Read objects."""
    import numpy as np

    reads = list(rs)
    return (np.array([len(r) for r in reads], np.int64), np.array([r.sample_id for r in reads], np.int64),
            np.array([v.position for r in reads for v in r], np.int64), np.array([v.allele for r in reads for v in r], np.int64),
            np.array([v.quality for r in reads for v in r], np.int64))


def test_readset_columnar_copy_follows_add_sort_and_mutation():
    """ReadSet keeps a columnar copy of all variants (what the DP is flattened from): it must follow add / sort / subset /
    pickling and every change made to a stored read through a reference."""
    import numpy as np
    import random

    rnd = random.Random(5)
    rs = ReadSet()
    for i in range(40):
        r = Read("read{}".format(rnd.randrange(10 ** 6)) + "_%d" % i, 50, rnd.randrange(3), rnd.randrange(2))
        start = rnd.randrange(0, 300, 10)
        for j in range(1 + rnd.randrange(5)):
            r.add_variant(start + 10 * j, rnd.randrange(2), rnd.randrange(1, 40))
        rs.add(r)
        r.add_variant(10 ** 6, 0, 1)  # the set holds a copy: changing the original afterwards does not reach it

    def same():
        got, want = rs._flat_columns(), _columns_from_objects(rs)
        return all(np.array_equal(g, w) for g, w in zip(got, want))

    assert same()
    rs.sort()
    assert rs._columns is not None and same()  # reordered, not rebuilt
    assert rs.get_positions() == sorted({v.position for r in rs for v in r})
    rs[3].add_variant(5000, 1, 7)  # a stored read changed through a reference
    assert rs._columns is None and same()
    rs[5][0] = Variant(rs[5][0].position, 1, 99)
    assert same()
    sub = rs.subset([0, 2, 5, 7])
    assert [r.name for r in sub] == [rs[i].name for i in (0, 2, 5, 7)]
    got, want = sub._flat_columns(), _columns_from_objects(sub)
    assert all(np.array_equal(g, w) for g, w in zip(got, want))
    clone = pickle.loads(pickle.dumps(rs))
    got, want = clone._flat_columns(), _columns_from_objects(rs)
    assert all(np.array_equal(g, w) for g, w in zip(got, want))


def test_flatten_columns_of_reads_with_gaps():
    """`_flatten_reads` maps a read's positions to columns with one binary search per read plus one per entry behind a gap
    (a position of another read that this read skips): compared with a dictionary look-up per entry."""
    import random

    import numpy as np

    from whatshap_b200.core import _flatten_reads

    rnd = random.Random(9)
    all_pos = sorted(rnd.sample(range(1000, 5000), 300))
    rs = ReadSet()
    start = 0
    for i in range(120):
        start += rnd.randrange(0, 4)
        span = all_pos[start : start + rnd.randrange(1, 12)]
        if not span:
            break
        kept = [p for j, p in enumerate(span) if j in (0, len(span) - 1) or rnd.random() < 0.7]  # interior gaps
        r = Read("g%03d" % i, 30, 0, 0)
        for p in kept:
            r.add_variant(p, rnd.randrange(2), rnd.randrange(1, 30))
        rs.add(r)
    pos_list, read_off, ent_col, ent_allele, ent_phred, read_ind = _flatten_reads(rs, None, lambda sid: 0)
    col_of = {p: i for i, p in enumerate(pos_list)}
    want = [col_of[v.position] for r in rs for v in r]
    assert pos_list == sorted({v.position for r in rs for v in r})
    assert np.asarray(ent_col).tolist() == want
    assert np.asarray(read_off).tolist() == [0] + list(np.cumsum([len(r) for r in rs]))
