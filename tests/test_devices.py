"""One table over several devices from ONE process (`multigpu.solve_on_devices` / `genotype_on_devices`), without a GPU: the
emulated stand-ins take the place of the per-device CUDA calls (the CPU checker for `whmec_solve`, tests/emul for the segments
and the genotyping DP).  The parts run on one host thread per distinct device; the results must equal the whole table's,
bit for bit for phasing and exactly for emulated genotyping of a single individual."""
import threading

import numpy as np
import pytest

import emul_genotype
import emul_genotype_segment
import emul_segment
from oracle import checker
from whatshap_b200 import _lib, multigpu, synth
from whatshap_b200._abi import Unsupported

DEVICE_LISTS = [[0, 1], [0, 1, 2], [0, 0, 0], [0, 1, 0, 1], [3, 1, 2, 0, 1]]


@pytest.fixture(scope="module", autouse=True)
def loaded():
    """The emulation libraries are built and loaded once, before any thread touches them."""
    emul_segment.lib()
    emul_genotype.lib()
    emul_genotype_segment.lib()


def ck_solve(prob, device):
    return checker.best().solve(prob), {"device": device}


def emul_factory(prob, continues, device):
    return emul_segment.EmulSegment(prob, continues)


def gl_factory(prob, continues, continued, device):
    return emul_genotype_segment.Segment(prob, continues, continued)


def solve(prob, devices, solver=ck_solve, factory=emul_factory):
    return multigpu.solve_on_devices(prob, devices, solver=solver, segment_factory=factory)


def genotype(prob, devices, solver=emul_genotype.genotype, factory=gl_factory):
    return multigpu.genotype_on_devices(prob, devices, solver=solver, segment_factory=factory)


def outcome(fn, *args):
    try:
        return fn(*args), ""
    except RuntimeError as e:  # MendelianConflict is a RuntimeError
        return None, "%s: %s" % (type(e).__name__, e)


def pedigree_problems():
    yield "trio", synth.trio(40, 2, block_len=10, seed=6)
    rng = np.random.default_rng(5)
    found = {}
    for it in range(400):
        ped = ("trio", "quartet", "three_generations")[it % 3]
        distrust, conflict_free = it % 2 == 0, it % 7 != 0
        key = (ped, distrust, conflict_free)
        prob = synth.random_problem(rng, int(rng.integers(8, 30)), int(rng.integers(2, 5)), pedigree=ped, distrust=distrust,
                                    conflict_free=conflict_free, mean_len=float(rng.choice([1.5, 3.0])))
        if found.get(key, 0) < 2 and len(multigpu.independent_blocks(prob)) >= 3:
            found[key] = found.get(key, 0) + 1
            yield "%s distrust=%s conflict_free=%s #%d" % (ped, distrust, conflict_free, it), prob
    assert len(found) == 12, sorted(found)


@pytest.mark.parametrize("devices", DEVICE_LISTS)
def test_single_individual_shares(devices):
    for prob in (synth.sliding_window(120, 6, block_len=20, seed=5, gap=0.1), synth.sliding_window(300, 5, block_len=7, seed=2)):
        want = checker.best().solve(prob)
        got, stats = solve(prob, devices)
        assert got.same_as(want), got.diff(want)
        assert stats["mode"] == "blocks" and stats["devices"] == devices
        assert [p["device"] for p in stats["parts"]] == devices[: len(stats["parts"])]
        assert [p["stats"]["device"] for p in stats["parts"]] == [p["device"] for p in stats["parts"]]


@pytest.mark.parametrize("devices", DEVICE_LISTS)
def test_pedigree_segments_equal_the_whole_table(devices):
    """Trios, quartets and three generations, trusted and distrusted genotypes, Mendelian conflicts (same error)."""
    n_conflicts = 0
    for label, prob in pedigree_problems():
        want, werr = outcome(checker.best().solve, prob)
        got, gerr = outcome(solve, prob, devices)
        assert gerr == werr, (label, gerr, werr)
        n_conflicts += bool(werr)
        if want is not None:
            sol, stats = got
            assert sol.same_as(want), (label, sol.diff(want))
            assert stats["mode"] == "segments" and stats["devices"] == devices, label
    assert n_conflicts >= 2


def test_whole_table_cases_run_on_the_first_device():
    one_chain = synth.trio(30, 2, block_len=30, seed=3)
    assert len(multigpu.independent_blocks(one_chain)) == 1
    for prob in (one_chain, synth.sliding_window(0, 3)):
        got, stats = solve(prob, [2, 1])
        assert got.same_as(checker.best().solve(prob))
        assert stats["mode"] == "whole" and stats["parts"] == [{"device": 2, "columns": (0, prob.n_cols), "stats": {"device": 2}}]


@pytest.mark.parametrize("devices", DEVICE_LISTS)
def test_genotyping(devices):
    single = synth.genotyping_problem(np.random.default_rng(21), 160, 5, "single", prior="random", burst=3, mean_len=3.0)
    whole, _ = emul_genotype.genotype(single)
    got, stats = genotype(single, devices)
    assert np.array_equal(got, whole, equal_nan=True) and stats["mode"] == "blocks"
    for ped in ("trio", "quartet", "three_generations"):
        from test_genotype_segments import TOL_WHOLE, close, instance

        prob = instance(ped, "random", 17)
        whole, _ = emul_genotype.genotype(prob)
        got, stats = genotype(prob, devices)
        assert stats["mode"] == "segments", ped
        assert np.array_equal(got, multigpu.genotype_pedigree_segments(prob, len(devices), segment_factory=emul_genotype_segment.Segment),
                              equal_nan=True), ped
        assert close(got, whole, TOL_WHOLE), ped
        assert all(set(p["stats"]) == {"transfer", "run"} for p in stats["parts"])


class Recorder:
    """Counts the parts inside a call per device; `barrier` (optional) must be passed by every distinct device's part at once."""

    def __init__(self, prob, barrier=None):
        self.prob, self.barrier = prob, barrier
        self.lock = threading.Lock()
        self.inside, self.most, self.calls = {}, {}, []

    def __call__(self, part, device, fn):
        with self.lock:
            self.inside[device] = self.inside.get(device, 0) + 1
            self.most[device] = max(self.most.get(device, 0), self.inside[device])
            first = int(np.searchsorted(self.prob.positions, part.positions[0])) if part.n_cols else -1
            self.calls.append((first, device, threading.current_thread().name))
        try:
            if self.barrier is not None:
                self.barrier.wait()
            return fn()
        finally:
            with self.lock:
                self.inside[device] -= 1


def test_parts_run_on_their_devices_at_once():
    """Every part runs on the device it was given, on that device's thread; parts on distinct devices are inside their calls
    at the same time (a barrier no part could pass alone); parts that share a device never overlap."""
    prob = synth.sliding_window(400, 6, block_len=20, seed=9)
    for devices, distinct in (([0, 1, 2], 3), ([0, 0, 1, 1], 2), ([1, 1, 1], 1)):
        rec = Recorder(prob, threading.Barrier(distinct, timeout=60) if distinct > 1 else None)  # every device has as many parts
        got, stats = solve(prob, devices, solver=lambda p, d: rec(p, d, lambda: ck_solve(p, d)))
        assert got.same_as(checker.best().solve(prob))
        assert sorted((first, d) for first, d, _ in rec.calls) == [(p["columns"][0], p["device"]) for p in stats["parts"]]
        assert all(name == "whmec-device-%d" % d for _, d, name in rec.calls)
        assert all(n == 1 for n in rec.most.values()), rec.most
    # pedigree segments: every phase of every segment, with a barrier in the transfer phase
    prob = synth.trio(120, 2, block_len=10, seed=6)
    rec = Recorder(prob, threading.Barrier(3, timeout=60))

    class Held(emul_segment.EmulSegment):
        def __init__(self, p, continues, device):
            super().__init__(p, continues)
            self.device = device

        def transfer(self):
            return rec(self.prob, self.device, super().transfer)

        def sweep(self, vec=None):
            return rec(self.prob, self.device, lambda: super(Held, self).sweep(vec))

    rec_sweeps = rec.calls
    got, stats = solve(prob, [0, 1, 2], factory=Held)
    assert got.same_as(checker.best().solve(prob)) and stats["mode"] == "segments"
    assert len(rec_sweeps) == 6 and all(name == "whmec-device-%d" % d for _, d, name in rec_sweeps)
    for devices in ([0, 0, 0], [1, 0, 1, 0]):
        rec = Recorder(prob)
        got, _ = solve(prob, devices, factory=Held)
        assert got.same_as(checker.best().solve(prob)) and all(n == 1 for n in rec.most.values()), rec.most


def test_genotyping_parts_run_at_once():
    from test_genotype_segments import instance

    prob = instance("trio", "random", 17)
    rec = Recorder(prob, threading.Barrier(3, timeout=60))

    def factory(p, continues, continued, device):
        seg = emul_genotype_segment.Segment(p, continues, continued)
        transfer = seg.transfer
        seg.transfer = lambda: rec(p, device, transfer)
        return seg

    got, stats = genotype(prob, [2, 0, 1], factory=factory)
    assert stats["mode"] == "segments"
    assert np.array_equal(got, multigpu.genotype_pedigree_segments(prob, 3, segment_factory=emul_genotype_segment.Segment), equal_nan=True)
    assert sorted((first, d) for first, d, _ in rec.calls) == [(p["columns"][0], p["device"]) for p in stats["parts"]]


class Tracked(emul_segment.EmulSegment):
    """Fails in `fail_in` for the segments starting at the columns in `failing`; records every segment it opens and closes."""

    open_now: set = set()
    failing: dict = {}
    fail_in = "sweep"
    release = None

    def __init__(self, p, continues, device):
        self.first = int(self.source.positions.searchsorted(p.positions[0]))
        self._fail("create")
        super().__init__(p, continues)
        Tracked.open_now.add(id(self))

    def _fail(self, where):
        if where == self.fail_in and self.first in self.failing:
            exc = self.failing[self.first]
            if self.first == min(self.failing):  # the left part fails last in time
                assert self.release.wait(60)
            else:
                self.release.set()
            raise exc

    def transfer(self):
        self._fail("transfer")
        return super().transfer()

    def sweep(self, vec=None):
        self._fail("sweep")
        return super().sweep(vec)

    def close(self):
        Tracked.open_now.discard(id(self))
        super().close()


@pytest.mark.parametrize("where", ["create", "transfer", "sweep"])
def test_the_left_error_is_raised_after_every_segment_is_closed(where):
    prob = synth.trio(120, 2, block_len=10, seed=6)
    ranges = multigpu.segment_ranges(prob, 4)
    Tracked.source, Tracked.fail_in, Tracked.release = prob, where, threading.Event()
    Tracked.failing = {ranges[1][0]: RuntimeError("left part failed"), ranges[3][0]: MemoryError("right part failed")}
    with pytest.raises(RuntimeError, match="^left part failed$"):
        solve(prob, [0, 1, 2, 3], factory=Tracked)
    assert Tracked.open_now == set()
    # a refusal on the left and an error on the right: the error (a refusal only falls back to the whole table)
    Tracked.failing, Tracked.release = {ranges[0][0]: Unsupported("refused"), ranges[2][0]: RuntimeError("Error: Mendelian conflict")}, threading.Event()
    with pytest.raises(RuntimeError, match="Mendelian conflict"):
        solve(prob, [0, 1, 2, 3], factory=Tracked)
    assert Tracked.open_now == set()


def test_the_left_error_is_raised_for_chain_runs():
    prob = synth.sliding_window(400, 6, block_len=20, seed=9)
    release = threading.Event()

    def solver(p, device):
        if device == 0:
            assert release.wait(60)
            raise RuntimeError("left run failed")
        if device == 2:
            release.set()
            raise Unsupported("right run refused")
        return ck_solve(p, device)

    with pytest.raises(RuntimeError, match="^left run failed$"):
        solve(prob, [0, 1, 2], solver=solver)

    def gl_solver(p, device):  # runs of chains are not segments: a refusal is raised, as the one-device call raises it
        if device == 2:
            raise Unsupported("right run refused")
        return emul_genotype.genotype(p)

    with pytest.raises(Unsupported, match="right run refused"):
        genotype(synth.genotyping_problem(np.random.default_rng(2), 160, 5, "single", burst=3, mean_len=3.0), [1, 1, 2], solver=gl_solver)


@pytest.mark.parametrize("where", ["create", "transfer", "sweep"])
def test_a_refused_segment_falls_back_to_the_whole_table(where):
    prob = synth.trio(120, 2, block_len=10, seed=6)
    ranges = multigpu.segment_ranges(prob, 3)
    Tracked.source, Tracked.fail_in, Tracked.release = prob, where, threading.Event()
    Tracked.failing = {ranges[1][0]: Unsupported("no room")}
    Tracked.release.set()
    got, stats = solve(prob, [2, 0, 1], factory=Tracked)
    assert got.same_as(checker.best().solve(prob)) and Tracked.open_now == set()
    assert stats["mode"] == "whole" and [p["device"] for p in stats["parts"]] == [2]


@pytest.mark.parametrize("where", ["create", "transfer", "run"])
def test_a_refused_genotyping_segment_falls_back_to_the_whole_table(where):
    from test_genotype_segments import instance

    prob = instance("quartet", "random", 17)
    closed = []

    class Refusing(emul_genotype_segment.Segment):
        def __init__(self, p, continues, continued, device):
            if where == "create" and continues and continued:
                raise Unsupported("refused")
            super().__init__(p, continues, continued, budget_doubles=1 if where == "run" and continues and continued else 1 << 62)
            self.refuse = where == "transfer" and continues and continued

        def transfer(self):
            if self.refuse:
                raise Unsupported("refused")
            return super().transfer()

        def close(self):
            closed.append(self)
            super().close()

    got, stats = genotype(prob, [1, 0, 1], factory=Refusing)
    assert np.array_equal(got, emul_genotype.genotype(prob)[0], equal_nan=True)
    assert stats["mode"] == "whole" and stats["parts"][0]["device"] == 1
    assert len(closed) == (2 if where == "create" else 3)


@pytest.fixture
def four_devices(monkeypatch):
    monkeypatch.setattr(_lib, "device_count", lambda: 4)
    monkeypatch.delenv(multigpu.ENV_DEVICES, raising=False)
    return monkeypatch


def test_devices_from_the_environment(four_devices):
    assert multigpu.table_devices() is None
    assert multigpu.table_devices(device=3) is None
    assert multigpu.table_devices(devices=[1, 1, 0]) == [1, 1, 0]
    four_devices.setenv("WHMEC_DEVICES", "")
    assert multigpu.table_devices() is None
    for text, want in (("0,1,2,3", [0, 1, 2, 3]), (" 2, 0 ", [2, 0]), ("1", [1]), ("0,0", [0, 0])):
        four_devices.setenv("WHMEC_DEVICES", text)
        assert multigpu.table_devices() == want, text
        assert multigpu.table_devices(devices=[3]) == [3]  # an explicit list wins
        assert multigpu.table_devices(device=2) is None    # as does a device named by the caller
    for text in ("a", "0,,1", "-1", "1.5", "0;1", "0,1,", "²"):
        four_devices.setenv("WHMEC_DEVICES", text)
        with pytest.raises(ValueError, match="WHMEC_DEVICES"):
            multigpu.table_devices()
    four_devices.setenv("WHMEC_DEVICES", "0,4")
    with pytest.raises(ValueError, match="ordinal 4 "):
        multigpu.table_devices()


def test_device_and_devices_conflict(four_devices):
    with pytest.raises(ValueError, match="not both"):
        multigpu.table_devices(device=1, devices=[0, 1])
    for bad in ([], [0, -1], [0, 1.0], [True], [5]):
        with pytest.raises(ValueError):
            multigpu.table_devices(devices=bad)


def objects_with_priors(prob, pedigree_class=None):
    """(ReadSet, recombcost, Pedigree) of `prob` whose individuals carry `prob.gl` as genotype likelihoods (the priors of
    `GenotypeDPTable`, the likelihoods of distrusted genotypes); the pedigree is a `pedigree_class` (default `core.Pedigree`)."""
    import copy

    from whatshap_b200.core import Genotype, PhredGenotypeLikelihoods

    reads_only = copy.copy(prob)
    reads_only.gt = np.zeros_like(prob.gt)
    rs, recomb, plain = synth.to_objects(reads_only)
    ped = (pedigree_class or type(plain))(plain.numeric_sample_ids)
    alleles = {0: [0, 0], 1: [0, 1], 2: [1, 1]}
    for i in range(prob.n_ind):
        ped.add_individual(i, [Genotype(alleles.get(g, [])) for g in prob.gt[i].tolist()],
                           [PhredGenotypeLikelihoods(prob.gl[i, k].tolist()) for k in range(prob.n_cols)])
    tr = prob.trios.tolist()
    for t in range(prob.n_trios):
        ped.add_relationship(tr[3 * t], tr[3 * t + 1], tr[3 * t + 2])
    return rs, recomb, ped


def same_tables(a, b):
    """Two PedigreeDPTables give the same answers (cost, partitioning, super-reads, transmission vector)."""
    (ra, ta), (rb, tb) = a.get_super_reads(), b.get_super_reads()
    reads = lambda sets: [[(r.name, list(r._pos), list(r._allele), list(r._quality)) for r in rs] for rs in sets]
    return (a.get_optimal_cost() == b.get_optimal_cost() and a.get_optimal_partitioning() == b.get_optimal_partitioning()
            and ta == tb and reads(ra) == reads(rb))


def test_the_public_classes(four_devices):
    """`core`'s classes with `devices`, or with WHMEC_DEVICES, run the one-process driver (here on the emulated stand-ins)
    and give the single-device answers; a single-device call keeps its statistics."""
    from whatshap_b200.core import GenotypeDPTable, PedigreeDPTable

    four_devices.setattr(_lib, "solve", lambda p, device=0: (checker.best().solve(p), {"device": device}))
    four_devices.setattr(_lib, "Segment", emul_factory)
    four_devices.setattr(_lib, "genotype", emul_genotype.genotype)
    four_devices.setattr(_lib, "GenotypeSegment", gl_factory)
    for prob in (synth.trio(120, 2, block_len=10, seed=6), synth.sliding_window(200, 5, block_len=20, seed=4)):
        objects = synth.to_objects(prob) + (False, prob.positions.tolist())
        one = PedigreeDPTable(*objects)
        assert one.stats == {"device": 0}
        for kw in ({"devices": [0, 1, 2]}, {"devices": (3, 3)}):
            got = PedigreeDPTable(*objects, **kw)
            assert same_tables(got, one) and got.stats["devices"] == list(kw["devices"]), kw
        four_devices.setenv("WHMEC_DEVICES", "1,2")
        got = PedigreeDPTable(*objects)
        assert same_tables(got, one) and got.stats["devices"] == [1, 2]
        assert PedigreeDPTable(*objects, device=3).stats == {"device": 3}
        four_devices.delenv("WHMEC_DEVICES")
        with pytest.raises(ValueError, match="not both"):
            PedigreeDPTable(*objects, device=1, devices=[0, 1])
    from test_genotype_segments import instance

    prob = instance("trio", "random", 17)
    rs, recomb, ped = objects_with_priors(prob)
    ids, positions = ped.numeric_sample_ids, prob.positions.tolist()
    one = GenotypeDPTable(ids, rs, recomb, ped, positions)
    got = GenotypeDPTable(ids, rs, recomb, ped, positions, devices=[0, 1])
    assert got.stats["mode"] == "segments" and one.stats.keys() == {"groups"}
    for k in range(prob.n_cols):
        a, b = one.get_genotype_likelihoods(0, k).as_vector(), got.get_genotype_likelihoods(0, k).as_vector()
        assert np.allclose(a, b, rtol=0, atol=1e-11, equal_nan=True), k
    with pytest.raises(ValueError, match="ordinal 7 "):
        GenotypeDPTable(ids, rs, recomb, ped, positions, devices=[0, 7])
