"""Read merging of `whatshap phase --merge-reads` on the device (whmec_merge_reads, DESIGN §4.17): every stored case of
tests/golden/merge.npz resident and in the smallest chunks, a dense chromosome of more than 10^7 pairs against the emulation
and the oracle, chunked against resident runs, several readsets in one call, and the removal path on device-evaluated pairs."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import merge_cases as mc
from oracle import merge_oracle
from whatshap_b200 import Read, ReadSet, _lib, merge

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")

with np.load(os.path.join(ROOT, "tests", "golden", "merge.npz")) as z:
    GOLDEN = json.loads(z["cases"].tobytes())["cases"]

_emul = None


def emul():
    global _emul
    if _emul is None:
        subprocess.run(["make", "-C", EMUL_DIR, "-f", "merge.mk"], check=True, capture_output=True)
        _emul = _lib.merge_reads_signatures(C.CDLL(os.path.join(EMUL_DIR, "libwhemul_merge.so")))
    return _emul


def device_merger(*params):
    return merge.ReadMerger(*params, device=0)


def chromosome(seed, n, span, lengths=(20, 200), error=0.05, spacing=1):
    """A ReadSet of n sorted reads on two haplotypes, built from arrays."""
    rng = np.random.default_rng(seed)
    start = np.sort(rng.integers(0, span, n)) * spacing
    lens = rng.integers(lengths[0], lengths[1] + 1, n)
    off = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    idx = np.arange(off[-1]) - np.repeat(off[:-1], lens)
    pos = np.repeat(start, lens) + idx * spacing
    hap = np.repeat(rng.integers(0, 2, n), lens)
    allele = hap ^ (rng.random(off[-1]) < error)
    quality = rng.integers(1, 40, off[-1])
    m = merge.Merged(np.arange(n), off, pos.astype(np.int64), allele.astype(np.int64), quality.astype(np.int64), None)
    return merge._own_readset(m)


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def comparable(st):
    return {k: v for k, v in st.items() if k not in ("chunks", "kernel_launches", "h2d_bytes", "d2h_bytes", "device_ms", "plan_ms")}


@pytest.mark.parametrize("i", range(len(GOLDEN)))
def test_golden_case_on_the_device(gpu, i):
    case = GOLDEN[i]
    assert mc.run(device_merger, case, Read, ReadSet) == case["want"]


def test_golden_cases_in_the_smallest_chunks(gpu, monkeypatch):
    monkeypatch.setenv("WHMEC_MERGE_ARENA_BUDGET", "1")
    for case in GOLDEN:
        if len(case["reads"]) <= 200:
            assert mc.run(device_merger, case, Read, ReadSet) == case["want"], case["name"]


def test_dense_chromosome_against_emulation_and_oracle(gpu):
    rs = chromosome(7, 60000, 20000)
    st, st_e = {}, {}
    (got,) = merge.merge_reads([rs], device=0, stats=st)
    assert st["pairs"] >= 10 ** 7
    (want,) = merge.merge_reads([rs], stats=st_e, library=emul())
    assert same(got, want) and comparable(st) == comparable(st_e)
    assert st["merged_components"] >= 1 and st["output_reads"] < st["reads"]
    sub = ReadSet()
    for k in range(600):
        sub.add(rs[k])
    (got,) = merge.merge_reads([sub], device=0)
    reads = [[(v.position, v.allele, v.quality) for v in r] for r in sub]
    want = merge_oracle.merge(reads)
    assert [("read%d" % r, list(zip(got.position[a:b].tolist(), got.allele[a:b].tolist(), got.quality[a:b].tolist())))
            for r, a, b in zip(got.read.tolist(), got.entry_off[:-1].tolist(), got.entry_off[1:].tolist())] == want


def test_chunked_runs_equal_the_resident_run(gpu, monkeypatch):
    rs = chromosome(8, 20000, 20000)
    st = {}
    (resident,) = merge.merge_reads([rs], device=0, stats=st)
    for budget in ("8000000", "5000000"):
        monkeypatch.setenv("WHMEC_MERGE_ARENA_BUDGET", budget)
        st_c = {}
        (chunked,) = merge.merge_reads([rs], device=0, stats=st_c)
        assert same(chunked, resident) and comparable(st_c) == comparable(st)
        assert st_c["chunks"] > st["chunks"]


def test_several_readsets_in_one_call(gpu):
    sets = [chromosome(s, 3000, 3000 * (s % 3 + 1), spacing=1 + 999 * (s % 2)) for s in range(6)]
    together = merge.merge_reads(sets, device=0)
    for rs, got in zip(sets, together):
        (alone,) = merge.merge_reads([rs], device=0)
        assert same(got, alone)


def test_removal_path_on_device_pairs(gpu):
    rs = chromosome(9, 120, 60, lengths=(2, 8), error=0.3)
    for params in ((0.8, 0.9, 1000, 1000), (0.15, 0.6, 0.01, 0.001)):
        st = {}
        (got,) = merge.merge_reads([rs], *params, device=0, stats=st)
        (want,) = merge.merge_reads([rs], *params, library=emul())
        assert same(got, want)
        assert st["notblue_edges"] > 0 and st["removed_edges"] > 0
        reads = [[(v.position, v.allele, v.quality) for v in r] for r in rs]
        counters = {}
        merge_oracle.merge(reads, *params, counters=counters)
        assert {k: st[k] for k in counters} == counters


def test_counter_sanity(gpu):
    rs = chromosome(10, 5000, 5000)
    st = {}
    (got,) = merge.merge_reads([rs], device=0, stats=st)
    assert st["reads"] == len(rs) and st["entries"] == sum(len(r) for r in rs)
    assert st["output_reads"] == len(got.read)
    rep = got.representative
    assert st["merged_components"] == int(np.sum((np.bincount(rep, minlength=len(rs)) >= 2)))
    assert st["output_reads"] == len(rs) - int(np.sum(rep != np.arange(len(rs))))
    assert st["notblue_edges"] == 0 and st["removed_edges"] == 0 and st["blue_edges"] >= st["merged_components"]
    assert st["chunks"] >= 2 and st["kernel_launches"] >= 4 and st["device_ms"] > 0 and st["h2d_bytes"] > 0 and st["d2h_bytes"] > 0
