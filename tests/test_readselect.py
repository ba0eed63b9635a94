"""Coverage-capping read selection (SURVEY.md §8(f) rank 3): the reference's known answers
(tests/test_readselect.py:5-108), golden vectors produced by the unmodified reference module
(tests/golden/make_readselect_golden.py) and, where the reference can be built (machine with the reference),
a live comparison with it -- the SAME reads must be selected, ties included."""
import os
import sys

import numpy as np
import pytest

from whatshap_b200.readselect import readselection, select_reads_csr
from whatshap_b200.testhelpers import string_to_readset

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "readselect.npz")

ROWS = """
  1  1
  00
  0   1
  10  1
  1   1
    11
  0   1
  1    1
"""


@pytest.mark.parametrize("max_cov,bridging,expected", [
    (1, False, {1, 5}), (2, False, {1, 3, 5}), (3, False, {1, 3, 5, 7}),
    (3, True, {1, 3, 5, 7}),  # every position is covered once before bridging starts; coverage 3 is reached by then
])
def test_selection(max_cov, bridging, expected):
    assert readselection(string_to_readset(ROWS), max_cov=max_cov, preferred_source_ids=None, bridging=bridging) == expected


def test_selection_of_nested_reads():
    reads = string_to_readset("""
      1111
         111
         1  111
         1     11
        1      11
    """)
    assert readselection(reads, max_cov=4, preferred_source_ids=None, bridging=False) == {0, 1, 2, 3}


def test_bridging_reads_connect_blocks():
    reads = string_to_readset("""
      111
         000
      00
          00
       1   1
    """)
    assert readselection(reads, max_cov=2, preferred_source_ids=None, bridging=False) == {0, 1, 2, 3}
    assert readselection(reads, max_cov=2, preferred_source_ids=None, bridging=True) == {0, 1, 4}


def test_selection_with_preferred_sources():
    readset = string_to_readset("""
      1        1
    """, source_id=3)
    for read in string_to_readset("""
      1111
         111
            1111
    """, source_id=1):
        readset.add(read)
    assert readselection(readset, max_cov=2, preferred_source_ids=None, bridging=True) == {1, 2, 3}
    assert readselection(readset, max_cov=2, preferred_source_ids={3}, bridging=True) == {0, 1, 3}


def test_single_variant_read_is_rejected():
    from whatshap_b200 import Read, ReadSet

    rs = string_to_readset("""
      11
      11
    """)
    lonely = Read("lonely", 50, 0, 0)
    lonely.add_variant(10, 0, 5)
    rs.add(lonely)
    with pytest.raises(ValueError, match="at least two variants"):
        readselection(rs, 5)
    assert readselection(ReadSet(), 5) == set()


def unragged(z, group, name, i):
    off = z[f"{group}.{name}.off"]
    return z[f"{group}.{name}"][off[i]:off[i + 1]]


def golden_selections():
    z = np.load(GOLDEN)
    for i in range(int(z["sel.n"])):
        j, max_cov, bridging = (int(x) for x in unragged(z, "sel", "args", i))
        preferred = unragged(z, "sel", "preferred", i).tolist()
        positions = unragged(z, "rs", "positions", j)
        yield dict(
            read_off=unragged(z, "rs", "read_off", j), ent_pos=positions[unragged(z, "rs", "ent_var", j)],
            ent_quality=unragged(z, "rs", "ent_quality", j), source_ids=unragged(z, "rs", "source_id", j), max_cov=max_cov,
            preferred_source_ids=None if preferred == [-1] else set(preferred), bridging=bool(bridging),
        ), set(unragged(z, "sel", "selected", i).tolist())


def test_golden_selections():
    """450 selections of the reference on 90 random read sets (gaps, tie-heavy qualities, several sources,
    max_cov 1..15, with and without bridging / preferred sources)."""
    n = 0
    for kwargs, expected in golden_selections():
        assert select_reads_csr(**kwargs) == expected, n
        n += 1
    assert n == 450


def test_selection_respects_the_coverage_cap():
    """Size-independent properties on a large read set: physical coverage never exceeds max_cov, every
    variant that had reads is covered unless capped, the result does not depend on read names."""
    rng = np.random.default_rng(3)
    n_var, reads = 4000, []
    for _ in range(30000):
        start = int(rng.integers(0, n_var - 2))
        reads.append(np.arange(start, min(n_var, start + 2 + int(rng.geometric(0.15)))))
    reads.sort(key=lambda r: int(r[0]))
    off = np.cumsum([0] + [len(r) for r in reads]).astype(np.uint64)
    pos = (np.concatenate(reads) * 7 + 3).astype(np.int32)
    qual = rng.integers(1, 50, len(pos)).astype(np.int32)
    chosen = select_reads_csr(off, pos, qual, np.zeros(len(reads), int), 15)
    coverage = np.zeros(n_var, int)
    for r in chosen:
        coverage[reads[r][0]:reads[r][-1] + 1] += 1
    assert coverage.max() <= 15
    touched = np.zeros(n_var, bool)
    touched[np.concatenate(reads)] = True
    assert np.all(coverage[touched] >= 1)
    assert len(chosen) < len(reads) // 3


# ---- live comparison with the reference module (only where the reference is available) ----
@pytest.fixture(scope="module")
def reference_modules():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from oracle import build_pyref

    path = build_pyref.build()
    if not path:
        pytest.skip("the reference tree is not available here: golden vectors cover this")
    sys.path.insert(0, path)
    import whatshap.core
    import whatshap.readselect

    return whatshap.core, whatshap.readselect


def test_same_selection_as_the_reference_on_its_own_containers(reference_modules):
    """Fresh random read sets held in the REFERENCE's ReadSet: this package's selection, reading them through
    the public container API, picks exactly the reads `whatshap.readselect.readselection` picks."""
    core, ref = reference_modules
    rng = np.random.default_rng(99)
    for it in range(60):
        n_var = int(rng.integers(4, 120))
        rs = core.ReadSet()
        starts = np.sort(rng.integers(0, n_var - 1, int(rng.integers(2, 250))))
        for i, start in enumerate(starts.tolist()):
            read = core.Read("q%d" % i, 60, int(rng.integers(0, 3)), 0)
            for v in range(start, min(n_var, start + 2 + int(rng.geometric(0.3)))):
                if v in (start, start + 1) or rng.random() > 0.2:
                    read.add_variant(100 + 13 * v, int(rng.integers(0, 2)), int(rng.integers(1, 4)))
            rs.add(read)
        for max_cov, preferred, bridging in ((1, None, True), (3, {0}, True), (8, None, False), (4, {1, 2}, False)):
            assert readselection(rs, max_cov, preferred, bridging) == ref.readselection(rs, max_cov, preferred, bridging), (it, max_cov)
