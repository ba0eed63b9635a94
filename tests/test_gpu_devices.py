"""One table over several devices from one process, on the GPU: `PedigreeDPTable` / `GenotypeDPTable` with `devices` (three
parts on device 0, and one part per visible GPU) against the single-device call, and the swap-in classes of `adapters` under
WHMEC_DEVICES.  On a box with one GPU the repeated device runs every code path of the driver."""
import sys

import numpy as np
import pytest

import golden_io
from test_devices import objects_with_priors, same_tables
from test_genotype import golden
from whatshap_b200 import _lib, adapters, core, multigpu, synth

sys.path.insert(0, golden_io.HERE)
import make_five_trios_golden as five  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def no_env(monkeypatch):
    monkeypatch.delenv(multigpu.ENV_DEVICES, raising=False)


def device_lists():
    return [[0, 0, 0], list(range(_lib.device_count()))]


def table_args(prob):
    """Constructor arguments of `PedigreeDPTable` for `prob` (likelihoods on the pedigree where genotypes are distrusted)."""
    rs, recomb, ped = objects_with_priors(prob) if prob.distrust else synth.to_objects(prob)
    return rs, recomb, ped, prob.distrust, prob.positions.tolist()


def conflicting_trio():
    prob = synth.trio(600, 3, block_len=40, seed=41)
    prob.gt = prob.gt.copy()
    prob.gt[:, 333] = [0, 0, 2]
    return prob


CASES = {
    "cfg2": lambda: synth.config("cfg2"),
    "cfg5": lambda: synth.config("cfg5"),
    "quartet": lambda: synth.random_problem(np.random.default_rng(3), 300, 5, "quartet", mean_len=3.0),
    "quartet distrusted": lambda: synth.random_problem(np.random.default_rng(4), 300, 5, "quartet", distrust=True, mean_len=3.0),
    "trio distrusted": lambda: synth.random_problem(np.random.default_rng(5), 400, 6, "trio", distrust=True, mean_len=3.0),
    "five trios": lambda: five.five_trio_problem(21, "three_gen", 80, max_cov=7, rc_max=3),
    "conflict": conflicting_trio,
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_pedigree_dp_table_on_devices(gpu, case):
    prob = CASES[case]()
    args = table_args(prob)
    try:
        one, werr = core.PedigreeDPTable(*args), ""
    except RuntimeError as e:
        one, werr = None, "%s: %s" % (type(e).__name__, e)
    assert (werr != "") == (case == "conflict"), werr
    for devices in device_lists():
        try:
            got, gerr = core.PedigreeDPTable(*args, devices=devices), ""
        except RuntimeError as e:
            got, gerr = None, "%s: %s" % (type(e).__name__, e)
        assert gerr == werr, (case, devices, gerr, werr)
        if one is None:
            continue
        assert got._solution.same_as(one._solution), (case, devices, got._solution.diff(one._solution))
        assert same_tables(got, one), (case, devices)
        stats = got.stats
        assert stats["devices"] == devices and all(p["device"] in devices for p in stats["parts"])
        if len(devices) > 1 and len(multigpu.independent_blocks(prob)) > 1:
            want = "blocks" if prob.n_trios == 0 else ("whole" if case == "five trios" else "segments")
            assert stats["mode"] == want, (case, stats["mode"])
            assert len(stats["parts"]) == (1 if want == "whole" else len(devices))


def trio_for_genotyping(cols, c_per_sample, block_len, seed):
    rng = np.random.default_rng(seed)
    prob = synth.trio(cols, c_per_sample, block_len=block_len, seed=seed)
    prob.gl = rng.random((3, prob.n_cols, 3)) + 0.05
    prob.gl /= prob.gl.sum(axis=2, keepdims=True)
    prob.recombcost = rng.integers(0, 30, prob.n_cols).astype(np.uint32)
    prob.distrust = True
    return prob


def likelihoods_close(a, b, tol):
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and bool(np.all((np.abs(a - b) <= tol) | np.isnan(a)))


def genotype_table(prob, **kw):
    rs, recomb, ped = objects_with_priors(prob)
    return core.GenotypeDPTable(ped.numeric_sample_ids, rs, recomb, ped, prob.positions.tolist(), **kw)


def test_genotype_dp_table_on_devices(gpu):
    """The cfg5-shaped trio of DESIGN §4.5 at 4 000 columns, and a single individual cut into runs of chains."""
    single = synth.genotyping_problem(np.random.default_rng(21), 3000, 8, "single", prior="random", burst=3, mean_len=3.0)
    for prob in (trio_for_genotyping(4000, 5, 500, 2), single):
        one = genotype_table(prob)
        for devices in device_lists():
            got = genotype_table(prob, devices=devices)
            assert likelihoods_close(got._likelihoods, one._likelihoods, 1e-12), float(np.nanmax(np.abs(got._likelihoods - one._likelihoods)))
            assert got.stats["devices"] == devices
            for k in (0, prob.n_cols // 2, prob.n_cols - 1):
                assert np.allclose(got.get_genotype_likelihoods(0, k).as_vector(), one.get_genotype_likelihoods(0, k).as_vector(),
                                   rtol=0, atol=1e-12, equal_nan=True)
        if len(multigpu.independent_blocks(prob)) > 1:
            assert genotype_table(prob, devices=[0, 0, 0]).stats["mode"] == ("segments" if prob.n_trios else "blocks")


def test_genotype_golden_vectors_on_devices(gpu):
    n = 0
    for label, prob, want, _ in golden():
        for devices in device_lists():
            got, stats = multigpu.genotype_on_devices(prob, devices)
            assert likelihoods_close(got, want, 1e-9), (label, devices, float(np.nanmax(np.abs(got - want))))
        if prob.n_trios and len(multigpu.independent_blocks(prob)) > 1:
            assert multigpu.genotype_on_devices(prob, [0, 0])[1]["mode"] == "segments", label
            n += 1
    assert n >= 5, n


def test_swap_in_classes_use_the_listed_devices(gpu, monkeypatch):
    """WHMEC_DEVICES=0,0: the swap-in classes of `adapters` (with this package's `core` as the container module) call the
    one-process driver with [0, 0] and answer what the single-device classes answer."""
    calls = []

    def recorded(name):
        real = getattr(multigpu, name)

        def driver(prob, devices, **kw):
            calls.append((name, list(devices)))
            return real(prob, devices, **kw)

        return driver

    for name in ("solve_on_devices", "genotype_on_devices"):
        monkeypatch.setattr(multigpu, name, recorded(name))
    Recording = adapters.recording_pedigree(core.Pedigree)
    prob = synth.trio(600, 3, block_len=40, seed=41)
    rs, recomb, ped = synth.to_objects(prob)
    rec_ped = Recording(ped.numeric_sample_ids)
    for i in range(prob.n_ind):
        rec_ped.add_individual(i, ped._genotypes[i])
    tr = prob.trios.tolist()
    for t in range(prob.n_trios):
        rec_ped.add_relationship(tr[3 * t], tr[3 * t + 1], tr[3 * t + 2])
    gl_prob = trio_for_genotyping(600, 3, 40, 5)
    gl_rs, gl_recomb, gl_ped = objects_with_priors(gl_prob, Recording)
    positions, gl_positions = prob.positions.tolist(), gl_prob.positions.tolist()
    one = core.PedigreeDPTable(rs, recomb, ped, False, positions)
    gl_one = core.GenotypeDPTable(gl_ped.numeric_sample_ids, gl_rs, gl_recomb, gl_ped, gl_positions)
    assert calls == []
    monkeypatch.setenv("WHMEC_DEVICES", "0,0")
    got = adapters.make_dp_table_class(core)(rs, recomb, rec_ped, False, positions)
    gl_got = adapters.make_genotype_table_class(core)(gl_ped.numeric_sample_ids, gl_rs, gl_recomb, gl_ped, gl_positions)
    assert calls == [("solve_on_devices", [0, 0]), ("genotype_on_devices", [0, 0])], calls
    assert same_tables(got, one)
    for i in range(gl_prob.n_ind):
        for k in range(gl_prob.n_cols):
            assert np.allclose(gl_got.get_genotype_likelihoods(i, k).as_vector(), gl_one.get_genotype_likelihoods(i, k).as_vector(),
                               rtol=0, atol=1e-12, equal_nan=True), (i, k)
