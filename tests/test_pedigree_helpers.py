"""Recombination costs in, recombination events out (whatshap_b200/pedigree.py): the reference's known answers
(tests/test_pedigreephasing.py:432-441, tests/test_pedigree.py:53-80), values recorded from the unmodified
reference module, and a live comparison with it in the machine with the reference."""
import os
import sys

import numpy as np
import pytest

from whatshap_b200 import Genotype
from whatshap_b200.pedigree import (
    GeneticMapRecombinationCostComputer,
    ParseError,
    RecombinationEvent,
    RecombinationMapEntry,
    UniformRecombinationCostComputer,
    centimorgen_to_phred,
    find_recombination,
    mendelian_conflict,
    recombination_cost_map,
)

MAP = ((55550, 0.0), (721290, 0.410292036939447), (752566, 0.4412), (1000000, 0.4412), (2500000, 3.75))
POSITIONS = [100, 55550, 60000, 400000, 721290, 740000, 900000, 1000000, 1000001, 2499999, 2500000, 2600000, 9000000]


def test_centimorgen_to_phred():
    assert round(centimorgen_to_phred(0.10010013353365396)) == 30
    assert round(centimorgen_to_phred(0.0010000100001343354)) == 50
    assert round(centimorgen_to_phred(1e-38)) == 400
    with pytest.raises(ValueError):
        centimorgen_to_phred(0)


def test_costs_from_a_genetic_map(tmp_path):
    """Before, between, on and past the map points, a flat stretch (minimum distance -> cost 120); values of the reference."""
    entries = [RecombinationMapEntry(p, c) for p, c in MAP]
    assert recombination_cost_map(entries, POSITIONS) == [0, 120, 46, 27, 27, 37, 39, 120, 77, 15, 77, 28, 11]
    path = tmp_path / "map.txt"
    path.write_text("position COMBINED_rate(cM/Mb) Genetic_Map(cM)\n" + "\n".join(f"{p} 0.1 {c!r}" for p, c in MAP) + "\n\n")
    assert GeneticMapRecombinationCostComputer(path).compute(POSITIONS) == [0, 120, 46, 27, 27, 37, 39, 120, 77, 15, 77, 28, 11]
    path.write_text("header\n100 1.0\n")
    with pytest.raises(ParseError, match="Found 2 fields instead of 3"):
        GeneticMapRecombinationCostComputer(path)
    path.write_text("header\n100 1.0 abc\n")
    with pytest.raises(ParseError, match="Error at line 2"):
        GeneticMapRecombinationCostComputer(path)


def test_uniform_costs():
    assert UniformRecombinationCostComputer(1.26).compute([1000, 2000, 3000, 1003000, 1003001]) == [0, 49, 49, 19, 79]
    assert UniformRecombinationCostComputer(0.5).compute([10, 11, 500, 100000]) == [0, 83, 56, 33]
    # the benchmark's pedigree workload: 1.26 cM/Mb at 1 kb spacing (SURVEY.md 8(d))
    assert UniformRecombinationCostComputer(1.26).compute([1000 * (k + 1) for k in range(5)]) == [0, 49, 49, 49, 49]


def test_find_recombination():
    events = find_recombination([0, 0, 1, 1, 0], {p: 5303 for p in (5303, 5432, 8307, 9000, 9500)}, [5303, 5432, 8307, 9000, 9500],
                                [0, 3, 3, 1, 1])
    assert events == [RecombinationEvent(5432, 8307, 0, 1, 0, 0, 3), RecombinationEvent(9000, 9500, 1, 0, 0, 0, 1)]
    # mother's haplotype switches (bit 1); two blocks; unphased position 30 is skipped
    events = find_recombination([0, 0, 2, 2, 3, 3, 1], {10: 10, 20: 10, 40: 10, 50: 50, 60: 50, 70: 50}, [10, 20, 30, 40, 50, 60, 70], [0] + [7] * 6)
    assert events == [RecombinationEvent(20, 40, 0, 0, 0, 1, 7), RecombinationEvent(60, 70, 1, 1, 1, 0, 7)]


def test_mendelian_conflict():
    g = lambda *alleles: Genotype(list(alleles))
    assert not mendelian_conflict(g(0, 1), g(0, 1), g(1, 1))
    assert not mendelian_conflict(g(0, 0), g(1, 1), g(0, 1))
    assert mendelian_conflict(g(0, 0), g(0, 0), g(0, 1))
    assert mendelian_conflict(g(1, 1), g(0, 1), g(0, 0))


def test_same_numbers_as_the_reference_module():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from oracle import build_pyref

    path = build_pyref.build()
    if not path:
        pytest.skip("the reference tree is not available here: recorded values cover this")
    sys.path.insert(0, path)
    import whatshap.pedigree as ref

    rng = np.random.default_rng(1)
    for it in range(120):
        m = int(rng.integers(1, 40))
        map_pos = np.sort(rng.choice(np.arange(1, 2_000_000), m, replace=False))
        cum = np.cumsum(rng.random(m) * rng.choice([0, 1e-12, 0.01, 2.0], m))
        pos = np.sort(rng.choice(np.arange(1, 3_000_000), int(rng.integers(1, 200)), replace=False)).tolist()
        if it % 3 == 0:
            pos = sorted(set(pos + [int(map_pos[m // 2])]))
        theirs = ref.recombination_cost_map([ref.RecombinationMapEntry(int(p), float(c)) for p, c in zip(map_pos, cum)], pos)
        assert recombination_cost_map([RecombinationMapEntry(int(p), float(c)) for p, c in zip(map_pos, cum)], pos) == list(theirs)
        rate = float(rng.choice([1.26, 0.01, 50.0]))
        assert UniformRecombinationCostComputer(rate).compute(pos) == list(ref.UniformRecombinationCostComputer(rate).compute(pos))
        tv = rng.integers(0, 4, len(pos)).tolist()
        components, block = {}, pos[0]
        for p in pos:
            block = p if rng.random() < 0.1 else block
            if rng.random() < 0.9:
                components[p] = block
        cost = rng.integers(0, 60, len(pos)).tolist()
        mine = find_recombination(tv, components, pos, cost)
        assert [tuple(vars(e).values()) for e in mine] == [tuple(vars(e).values()) for e in ref.find_recombination(tv, components, pos, cost)]
