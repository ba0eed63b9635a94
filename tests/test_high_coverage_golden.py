"""The stored reference answers at coverage 21-25 (tests/golden/high_coverage.npz, made by make_high_coverage_golden.py), checked
without a GPU.  test_gpu_high_coverage.py holds the tile kernel to these answers; it is only as good as the kernel paths the
instances reach.  So a census of the product's own planner (pack_problem + plan_tiles, tests/emul/emul_census.cpp) must find
every hand-off shape of these coverages in the set: small chunks (gathered element by element) into steady panels mirrored
with km = 0 and with km != 0, small chunks into non-steady panels, unmirrored small-chunk hand-offs, bulk copies from 2^6
producer tiles (the largest that still travel as bulk copies), canonical hand-offs, and many chains in one table.  A planner
change that moves an instance off these paths fails here instead of leaving the GPU test with nothing to check."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import golden_io
from whatshap_b200 import synth
from whatshap_b200._abi import CProblem

sys.path.insert(0, golden_io.HERE)
import make_high_coverage_golden as gen  # noqa: E402

EMUL_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
HANDOFFS = ("fresh", "canonical", "bulk", "small_chunk")
MIRROR = ("unmirrored", "km0", "km_nonzero")


@pytest.fixture(scope="module")
def census_lib():
    subprocess.run(["make", "-C", EMUL_DIR, "-f", "census.mk"], check=True, capture_output=True)
    lib = C.CDLL(os.path.join(EMUL_DIR, "libwhemul_census.so"))
    lib.whemul_census.argtypes = [C.POINTER(CProblem), C.POINTER(C.c_uint64)]
    lib.whemul_census_size.restype = C.c_uint32
    return lib


def census(lib, prob):
    """The planner's schedule of `prob` in numbers (emul_census.cpp); asserts that the tile planner takes the problem."""
    raw = (C.c_uint64 * lib.whemul_census_size())()
    rc = lib.whemul_census(C.byref(prob.as_c()), raw)
    assert rc == 0, rc
    v = np.array(raw[:], np.int64)
    return dict(panels=v[:24].reshape(len(HANDOFFS), 2, len(MIRROR)), km0_cols=v[24], km_nonzero_cols=v[25], max_g=v[26],
                chains=v[27], bulk_at_max_ga=v[28], n_panels=v[29])


def golden():
    return [(label, prob, want) for label, prob, want, _ in golden_io.load("high_coverage")]


def test_census_of_the_stored_instances_reaches_every_handoff_shape(census_lib, monkeypatch):
    monkeypatch.delenv("WHMEC_TILE_MIRROR", raising=False)
    monkeypatch.delenv("WHMEC_TILE_PACKED_BP", raising=False)
    total = np.zeros((len(HANDOFFS), 2, len(MIRROR)), np.int64)
    chains, max_g, bulk_at_max_ga = [], 0, 0
    for label, prob, _ in golden():
        c = census(census_lib, prob)
        total += c["panels"]
        assert c["km0_cols"] + c["km_nonzero_cols"] > 0, label  # every instance has mirrored columns
        chains.append(c["chains"])
        max_g, bulk_at_max_ga = max(max_g, c["max_g"]), bulk_at_max_ga + c["bulk_at_max_ga"]
        assert c["panels"].sum() == c["n_panels"]
        assert c["panels"][1:, :, :].sum() > 0, (label, "a single panel: no hand-off")
    small, canonical = HANDOFFS.index("small_chunk"), HANDOFFS.index("canonical")
    km0, kmx = MIRROR.index("km0"), MIRROR.index("km_nonzero")
    census_text = {f"{h}/{'steady' if s else 'other'}/{m}": int(total[i, s, j])
                   for i, h in enumerate(HANDOFFS) for s in (0, 1) for j, m in enumerate(MIRROR)}
    assert total[small, 1, km0] > 0, census_text      # small chunks into steady mirrored panels, km = 0 (even coverage)
    assert total[small, 1, kmx] > 0, census_text      # ... km != 0 (odd coverage)
    assert total[small, 0, :].sum() > 0, census_text  # small chunks into panels that are not steady
    assert total[canonical].sum() > 0, census_text
    assert bulk_at_max_ga > 0, census_text            # the boundary on the bulk side: 2^6 producer tiles
    assert max(chains) >= 10 and max_g >= 10, (chains, max_g)


def test_census_without_mirrored_panels(census_lib, monkeypatch):
    monkeypatch.setenv("WHMEC_TILE_MIRROR", "0")
    small = HANDOFFS.index("small_chunk")
    total = np.zeros((len(HANDOFFS), 2, len(MIRROR)), np.int64)
    for label, prob, _ in golden():
        c = census(census_lib, prob)
        total += c["panels"]
        assert c["km0_cols"] == c["km_nonzero_cols"] == 0, label
    assert total[:, :, 1:].sum() == 0 and total[small, 1, 0] > 0 and total[small, 0, 0] > 0, total


def test_small_chunk_boundary_lies_between_coverage_21_and_22(census_lib):
    """At coverage 21 the steady state hands 2^6 chunks on (bulk copies), at coverage 22 2^7 (small chunks)."""
    by_label = {label: census(census_lib, prob) for label, prob, _ in golden() if label.startswith("sliding/")}
    bulk, small = HANDOFFS.index("bulk"), HANDOFFS.index("small_chunk")
    c21, c22 = by_label["sliding/n=80/c=21"], by_label["sliding/n=80/c=22"]
    assert c21["panels"][bulk].sum() > 0 and c21["panels"][small].sum() == 0 and c21["bulk_at_max_ga"] > 0
    assert c22["panels"][small].sum() > 0 and c22["panels"][bulk].sum() == 0
    for cov in (23, 24, 25):
        n = 80 if cov == 23 else 60
        c = by_label[f"sliding/n={n}/c={cov}"]
        steady = c["panels"][small, 1]
        assert steady.sum() > 0 and steady[MIRROR.index("km0" if cov % 2 == 0 else "km_nonzero")] == steady.sum(), (cov, c)


def test_stored_costs_are_costs_of_stored_paths():
    n = 0
    for label, prob, want in golden():
        assert want is not None, label
        assert synth.het_path_cost(prob, want.path_index) == want.cost, label
        n += 1
    assert n >= 9 and any(np.any(prob.gt != 1) for _, prob, _ in golden())  # homozygous sites included


def test_stored_problems_are_what_the_generator_makes():
    made = gen.cases()
    stored = golden()
    assert [label for label, _ in made] == [label for label, _, _ in stored]
    for (label, p), (_, q, _) in zip(made, stored):
        for f in gen.PROBLEM_FIELDS:
            a, b = getattr(p, f), getattr(q, f)
            assert (a is None and b is None) or np.array_equal(a, b), (label, f)


def test_smallest_instance_equals_the_reference_live():
    from oracle import checker as ck

    ref = ck.reference()
    if ref is None:
        pytest.skip("the compiled reference (oracle/_ref) is not built here")
    label, prob, want = min(golden(), key=lambda c: np.sum(2.0 ** gen.active_reads(c[1])))  # the reference's DP cells
    got = ref.solve(prob)
    assert got.same_as(want), (label, got.diff(want))
