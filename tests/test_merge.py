"""Read merging of `whatshap phase --merge-reads` (whmec_merge_reads, DESIGN §4.17) on the CPU: the validation, partners, chunk
cuts, removal loop and output of merge_plan.cpp with the per-thread code of merge.h stepped by the host emulation
tests/emul/emul_merge.cpp, and the oracle oracle/merge_oracle.py, against the reference's answers stored in
tests/golden/merge.npz."""
import ctypes as C
import json
import logging
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import merge_cases as mc
from oracle import merge_oracle
from whatshap_b200 import Read, ReadSet, _lib, adapters, merge

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
_emul = None


def emul():
    global _emul
    if _emul is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "merge.mk"], check=True, capture_output=True)
        _emul = _lib.merge_reads_signatures(C.CDLL(os.path.join(EMUL_DIR, "libwhemul_merge.so")))
    return _emul


with np.load(os.path.join(ROOT, "tests", "golden", "merge.npz")) as z:
    GOLDEN = json.loads(z["cases"].tobytes())["cases"]


def merger(library, stats=None):
    return lambda *params: merge.ReadMerger(*params, library=library, stats=stats)


def readset(reads):
    rs = ReadSet()
    for k, read in enumerate(reads):
        r = Read(f"r{k}", 60, 0, 0)
        for p, a, q in read:
            r.add_variant(p, a, q)
        rs.add(r)
    return rs


def test_golden_covers_what_it_should():
    wants = {c["want"] for c in GOLDEN if isinstance(c["want"], str)}
    assert wants == {"IndexError", "AssertionError", "ValueError", "ZeroDivisionError"}
    counters = []
    for c in GOLDEN:
        if not isinstance(c["want"], str):
            k = {}
            merge_oracle.merge([[tuple(e) for e in r] for r in c["reads"]], *c["params"], counters=k)
            counters.append(k)
    assert sum(k["removed_edges"] for k in counters) > 50 and sum(k["notblue_edges"] for k in counters) > 50
    assert sum(k["merged_components"] for k in counters) > 500
    assert any(len(c["reads"]) >= 3000 for c in GOLDEN)
    unsorted = lambda c: any(b[0][0] < a[0][0] for a, b in zip(c["reads"], c["reads"][1:]) if a and b)
    assert sum(unsorted(c) for c in GOLDEN) >= 10
    assert any(q < 0 for c in GOLDEN for r in c["reads"] for _, _, q in r)


def test_removal_paths_have_several_edges():
    """Some removal steps pick the least edge of a path longer than the not-blue edge itself."""
    longer = 0
    original = merge_oracle.shortest_path

    def spy(adj, u, v):
        nonlocal longer
        p = original(adj, u, v)
        longer += p is not None and len(p) > 2
        return p

    merge_oracle.shortest_path = spy
    try:
        for c in GOLDEN:
            if c["name"].startswith("removal") and not isinstance(c["want"], str):
                mc.run_oracle(c)
    finally:
        merge_oracle.shortest_path = original
    assert longer > 10


@pytest.mark.parametrize("i", range(len(GOLDEN)))
def test_oracle_and_emulation_equal_the_reference(i):
    case = GOLDEN[i]
    assert mc.run_oracle(case) == case["want"]
    assert mc.run(merger(emul()), case, Read, ReadSet) == case["want"]


def test_emulation_smallest_chunks_equal_the_reference(monkeypatch):
    monkeypatch.setenv("WHMEC_MERGE_ARENA_BUDGET", "1")
    for case in GOLDEN:
        if len(case["reads"]) <= 200:
            assert mc.run(merger(emul()), case, Read, ReadSet) == case["want"], case["name"]


def test_counters_equal_the_oracle(monkeypatch):
    for budget in (None, "1"):
        if budget:
            monkeypatch.setenv("WHMEC_MERGE_ARENA_BUDGET", budget)
        for case in GOLDEN:
            if isinstance(case["want"], str) or len(case["reads"]) > 200:
                continue
            want, st = {}, {}
            merge_oracle.merge([[tuple(e) for e in r] for r in case["reads"]], *case["params"], counters=want)
            mc.run(merger(emul(), st), case, Read, ReadSet)
            assert {k: st[k] for k in want} == want, case["name"]
            assert st["reads"] == len(case["reads"]) and st["entries"] == sum(map(len, case["reads"]))


def queue_partners(begins, ends):
    """The reference's queue, literally: j's partners are the i it is compared with."""
    queue, seen = {}, {j: [] for j in range(len(begins))}
    for i, (b, e) in enumerate(zip(begins, ends)):
        queue[i] = (b, e)
        for x in [x for x in queue if queue[x][1] <= b]:
            del queue[x]
        for j in queue:
            if j != i:
                seen[j].append(i)
    return seen


@pytest.mark.parametrize("seed", range(30))
def test_partners_equal_the_literal_queue(seed):
    rng = random.Random(seed)
    reads = mc.make_reads(rng, rng.randrange(1, 150), rng.choice([1, 3, 100]), sort=seed % 3 != 0, shuffle=0.1 * (seed % 2))
    begins, ends = [r[0][0] for r in reads], [r[0][0] + len(r) for r in reads]
    kill = merge_oracle.partners(begins, ends)
    seen = queue_partners(begins, ends)
    for j in range(len(reads)):
        assert seen[j] == list(range(j + 1, kill[j]))
        for i in seen[j]:  # every compared pair has a non-empty overlap
            m, mm = merge_oracle.overlap([a for _, a, _ in reads[j]], begins[j], [a for _, a, _ in reads[i]], begins[i])
            assert m + mm > 0
    st = {}
    merge.merge_reads([readset(reads)], 0.15, 0.25, 1e6, 1e3, stats=st, library=emul())
    assert st["pairs"] == sum(len(v) for v in seen.values())


def test_several_readsets_in_one_call_equal_one_call_each():
    cases = [c for c in GOLDEN if not isinstance(c["want"], str) and c["params"] == mc.DEFAULT][:12]
    sets = [readset(c["reads"]) for c in cases]
    together = merge.merge_reads(sets, library=emul())
    for rs, got in zip(sets, together):
        (alone,) = merge.merge_reads([rs], library=emul())
        for a, b in zip(got, alone):
            assert np.array_equal(a, b)


def test_errors_and_int32_limits():
    with pytest.raises(ZeroDivisionError):
        merge.merge_reads([readset([[[1, 0, 1]]])], error_rate=0.75, library=emul())
    with pytest.raises(ValueError):
        merge.merge_reads([readset([[[1, 0, 1]]])], positive_threshold=0, library=emul())
    with pytest.raises(ValueError, match="int32"):
        merge.merge_reads([readset([[[1 << 31, 0, 1]]])], library=emul())
    with pytest.raises(ValueError, match="int32"):
        merge.merge_reads([readset([[[1, 0, -(1 << 31) - 1]]])], library=emul())
    with pytest.raises(AssertionError):  # the second set's error, after a clean first set
        merge.merge_reads([readset([[[1, 0, 1]]]), readset([[[1, 0, 1]], [[2, 256, 1]]])], library=emul())
    assert merge.merge_reads([], library=emul()) == []
    (m,) = merge.merge_reads([ReadSet()], library=emul())
    assert len(m.read) == 0 and len(m.representative) == 0


def test_thresholds_follow_the_reference():
    assert merge.thresholds(0.15, 1000000, 1000) == (5, 3)
    assert merge.thresholds(0.8, 1000, 1000) == (-23, -23)


def test_read_merger_logs_and_returns_own_readset(caplog):
    case = next(c for c in GOLDEN if c["name"] == "unit_read_merging")
    caplog.set_level(logging.INFO, logger="whatshap_b200.merge")
    got = merge.ReadMerger(*case["params"], library=emul()).merge(readset(case["reads"]))
    assert isinstance(got, ReadSet) and mc.answer(got) == case["want"]
    assert [r.getMessage() for r in caplog.records] == [
        "Merging 4 reads with error rate 0.15, maximum error rate 0.25, positive threshold 100000 and negative threshold 1000 ...",
        "... after merging: merged 4 reads into 3 reads"]
    assert got.get_positions() == sorted({v.position for r in got for v in r})
    assert isinstance(merge.DoNothingReadMerger().merge(got), ReadSet)


def _pyref():
    from oracle import build_pyref

    return build_pyref.build()


def test_swapin_on_reference_containers():
    if not _pyref():
        pytest.skip("reference tree not available")
    pytest.importorskip("networkx")  # imported by the reference's whatshap/merge.py
    sys.path.insert(0, _pyref())
    import whatshap.core as core
    import whatshap.merge as ref_merge

    cls = adapters.make_read_merger(ref_merge)
    for case in GOLDEN[:40]:
        got = mc.run(lambda *p: cls(*p, library=emul()), case, core.Read, core.ReadSet)
        assert got == case["want"], case["name"]
    assert issubclass(cls, ref_merge.ReadMergerBase)


def test_reference_suite_with_swapin():
    """The reference's own tests/test_merge_reads.py with its ReadMerger replaced by the swap-in (emulated library)."""
    from oracle import build_pyref

    if not _pyref():
        pytest.skip("reference tree not available")
    pytest.importorskip("networkx")
    test_file = os.path.join(build_pyref.REF, "tests", "test_merge_reads.py")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "tests"), _pyref(), ROOT]), PYTHONDONTWRITEBYTECODE="1",
               WHMEC_PYREF=_pyref())
    res = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "swapin_merge_plugin", "-p", "no:cacheprovider", test_file],
                         cwd=build_pyref.REF, env=env, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "2 passed" in res.stdout
