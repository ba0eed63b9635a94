"""Five-trio pedigrees (T = 1024) on the CPU: the wide column sweep's per-thread code (wide_device.h) stepped by the emulation,
against the reference-generated golden vectors and the compiled reference; its transition transform against transition_min; its
plans; and the refusals that remain (six trios, genotyping, table segments)."""
import os
import sys

import numpy as np
import pytest

import emul_genotype
import emul_wide
import golden_io
from whatshap_b200._abi import Unsupported

sys.path.insert(0, golden_io.HERE)
import make_five_trios_golden as five  # noqa: E402

UMAX = 0xFFFFFFFF


@pytest.mark.parametrize("transform", [-1, 0, 1])
def test_emulated_wide_sweep_matches_golden(transform):
    n = 0
    for label, prob, want, error in golden_io.load("five_trios"):
        assert not error, (label, error)
        if transform == 1 and "wrapping" in label:
            continue  # the transform is exact only without wrapping sums
        got, info = emul_wide.solve(prob, transform)
        assert got.same_as(want), (label, got.diff(want))
        assert info["nowrap"] == ("wrapping" not in label), label
        n += 1
    assert n >= 7


def test_golden_cases_cover_the_shapes():
    labels = [label for label, *_ in golden_io.load("five_trios")]
    assert any(l.startswith("nuclear5") for l in labels) and any(l.startswith("three_gen") for l in labels)
    assert any("distrust=True" in l for l in labels) and any("wrapping" in l for l in labels)


def _ref():
    from oracle import checker

    return checker.reference()


@pytest.mark.skipif(not os.path.exists(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                                                    "libwhref.so")), reason="the compiled reference (oracle/_ref) is not built here")
@pytest.mark.parametrize("seed", range(4))
def test_emulated_wide_sweep_matches_compiled_reference(seed):
    shape = ("nuclear5", "three_gen")[seed % 2]
    prob = five.five_trio_problem(1000 + seed, shape, 12, max_cov=5, distrust=seed == 3, rc_max=3)
    want = _ref().solve(prob)
    got, _ = emul_wide.solve(prob)
    assert got.same_as(want), got.diff(want)


@pytest.mark.parametrize("rc", [0, 1, 2, 37])
@pytest.mark.parametrize("first", [False, True])
def test_transform_equals_transition_min(rc, first):
    rng = np.random.default_rng(rc + 10 * first)
    rows = rng.integers(0, 6, (6, 1024)).astype(np.uint32)  # few distinct values: many ties
    rows[1] = UMAX                                          # all infinite
    rows[2, rng.random(1024) < 0.9] = UMAX
    rows[3] = rng.integers(0, 1 << 30, 1024)
    rows[4] = 0
    rows[5, :1023] = UMAX                                   # one finite entry, at j = 1023
    (vals, args), (rvals, rargs) = emul_wide.xform(rows, rc, first)
    assert np.array_equal(vals, rvals) and np.array_equal(args, rargs)
    assert (vals[1] == (0 if first else UMAX)).all() and (args[1] == (np.arange(1024) if first and rc else 0)).all()


def test_plan_routes_five_trios_to_the_wide_sweep():
    prob = five.five_trio_problem(7, "nuclear5", 40, max_cov=6, rc_max=3)
    res = emul_wide.plan(prob)
    assert res["rc"] == 0 and res["path"] == "wide" and not res["bounded"], res
    # the two-pass sweeps are not for T = 1024, not even when the sequential sweep is possible and chains are many
    assert emul_wide.plan(prob, free_bytes=1 << 36)["path"] == "wide"


@pytest.mark.parametrize("fraction", [2, 4])
def test_plan_bounded_under_the_arena_hook(fraction):
    prob = five.five_trio_problem(8, "three_gen", 40, max_cov=6, rc_max=3)
    full = emul_wide.plan(prob)
    res = emul_wide.plan(prob, hook=full["bp_words"] * 4 // fraction)
    assert res["rc"] == 0 and res["path"] == "wide" and res["bounded"], res
    cuts = res["cuts"]
    assert cuts[0] == 0 and cuts[-1] == prob.n_cols and len(cuts) >= 3
    assert res["arena"] * 4 <= full["bp_words"] * 4 // fraction


def test_plan_refuses_an_impossible_hook_with_its_byte_count():
    prob = five.five_trio_problem(9, "nuclear5", 30, max_cov=6)
    res = emul_wide.plan(prob, hook=64)
    assert res["rc"] == 4 and "needs at least" in res["msg"], res
    need = int(res["msg"].split("needs at least ")[1].split()[0])
    ok = emul_wide.plan(prob, hook=need)
    assert ok["rc"] == 0 and ok["bounded"], ok


def test_plan_under_little_free_memory_takes_the_bounded_sweep():
    prob = five.five_trio_problem(10, "nuclear5", 40, max_cov=6)
    fixed = emul_wide.plan(prob, free_bytes=1 << 40)
    free = (512 << 20) + fixed["bp_words"] * 4 + (64 << 20)  # the reserve, the table's arrays and less than its back-pointers
    res = emul_wide.plan(prob, free_bytes=free - fixed["bp_words"] * 4 // 2)
    assert res["rc"] == 0 and res["path"] == "wide"


def test_six_trios_are_refused():
    prob = five.five_trio_problem(11, "nuclear5", 10, max_cov=4)
    prob.n_ind = 8
    prob.trios = np.concatenate([prob.trios, np.array([0, 1, 7], np.uint32)])
    prob.gt = np.concatenate([prob.gt, prob.gt[:1]])
    with pytest.raises(Unsupported, match="at most 5 trio relationships"):
        emul_wide.solve(prob)


def test_segments_and_genotyping_are_refused():
    prob = five.five_trio_problem(12, "nuclear5", 12, max_cov=4, distrust=True)
    res = emul_wide.plan(prob, segment=1)
    assert res["rc"] == 4, res
    prob.gl = np.full(prob.gl.shape, 1.0 / 3.0)
    with pytest.raises(Unsupported, match="at most 4 trio relationships"):
        emul_genotype.genotype(prob)


def test_cost_functions_beyond_the_limit_are_refused_before_allocation():
    # nine founders' worth of haplotypes (P = 10) with distrusted genotypes: 2^20 functions per column
    prob = five.five_trio_problem(13, "three_gen", 4, max_cov=3, distrust=True)
    prob.n_ind = 10
    prob.trios = np.array([0, 1, 5, 2, 3, 6, 5, 6, 7, 5, 6, 8, 5, 4, 9], np.uint32)
    prob.gt = np.concatenate([prob.gt, prob.gt[:1]])
    prob.gl = np.concatenate([prob.gl, prob.gl[:1]])
    res = emul_wide.plan(prob)
    assert res["rc"] == 0  # four columns fit
    big = five.five_trio_problem(13, "three_gen", 120, max_cov=3, distrust=True)
    big.n_ind, big.trios = prob.n_ind, prob.trios
    big.gt = np.concatenate([big.gt, big.gt[:1]])
    big.gl = np.concatenate([big.gl, big.gl[:1]])
    res = emul_wide.plan(big)
    assert res["rc"] == 4 and "bytes" in res["msg"], res
