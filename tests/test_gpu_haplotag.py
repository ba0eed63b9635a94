"""Read assignment of `whatshap haplotag` on the GPU (whmec_haplotag, DESIGN §4.15): every stored case of the reference on the
device, a chromosome-sized seeded workload against the emulation and the oracle, budget-chunked runs against resident ones,
several samples in one call, and the call's counters."""
import json
import os
import random

import numpy as np
import pytest

import haplotag_cases as hc
import whatshap_b200
from whatshap_b200 import _lib, haplotag

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

with np.load(os.path.join(ROOT, "tests", "golden", "haplotag.npz")) as z:
    GOLDEN = json.loads(z["cases"].tobytes())


@pytest.fixture(autouse=True)
def gpu(monkeypatch):
    if _lib.device_count() == 0:
        pytest.skip("no CUDA device")
    monkeypatch.delenv("WHMEC_HAPLOTAG_ARENA_BUDGET", raising=False)


def on_device(case, stats=None):
    return hc.run(lambda *a: haplotag.prepare_haplotag_information(*a, device=0, stats=stats), case, whatshap_b200)


def agrees(want, got, loose):
    if isinstance(want, str) or isinstance(got, str):
        return want == got
    return hc.same(want, got, loose)


def test_every_golden_case_on_the_device():
    bad = [i for i, c in enumerate(GOLDEN) if not agrees(c["want"], on_device(c), c["loose"])]
    assert not bad


def test_golden_cases_one_group_per_chunk(monkeypatch):
    monkeypatch.setenv("WHMEC_HAPLOTAG_ARENA_BUDGET", "1")
    bad = [i for i, c in enumerate(GOLDEN) if not agrees(c["want"], on_device(c), c["loose"])]
    assert not bad


def chromosome(seed, n_reads=60000, n_samples=2, ploidy=2):
    """A seeded chromosome: n_reads per sample with about 20 phased heterozygous entries each, 400 blocks, 10 % of the reads
    in BX clouds.  Returns [(ReadSet, phase table)]."""
    rng = np.random.default_rng(seed)
    n_var = n_reads // 4
    pos = np.unique(rng.integers(1, 40 * n_var, n_var))
    block = pos[(np.arange(len(pos)) * 400) // len(pos)]
    samples = []
    for s in range(n_samples):
        phase = rng.integers(0, 2, (len(pos), ploidy))
        table = {int(p): (int(b), tuple(int(x) for x in ph)) for p, b, ph in zip(pos, block, phase)}
        rs = whatshap_b200.ReadSet()
        first = np.sort(rng.integers(0, len(pos) - 25, n_reads))
        for k in range(n_reads):
            bx = f"BX{rng.integers(0, n_reads // 50)}" if rng.random() < 0.1 else ""
            i0 = int(first[k])
            r = whatshap_b200.Read(f"read{k}", 60, 0, s, int(pos[i0]), bx, -1, -1, "chr1", "____1", False, int(pos[i0 + 20]), bool(k & 1))
            for i in range(i0, i0 + 20):
                r.add_variant(int(pos[i]), int(rng.integers(0, 2)), int(rng.integers(0, 40)))
            rs.add(r)
        samples.append((rs, table))
    return samples


@pytest.mark.parametrize("ploidy", [2, 4])
def test_chromosome_equals_the_emulation_and_the_oracle(ploidy, monkeypatch):
    from oracle import haplotag_oracle

    from test_haplotag import emul

    samples = chromosome(ploidy, ploidy=ploidy)
    st = {}
    got = haplotag.assign_reads(samples, ploidy, linked_read_cutoff=50000, stats=st)
    want = haplotag.assign_reads(samples, ploidy, linked_read_cutoff=50000, library=emul())
    for a, b in zip(got[:5], want[:5]):
        assert np.array_equal(a, b)
    assert st["chunks"] == 1 and st["device_ms"] > 0 and st["keys"] >= st["entries"] // 2 and st["runs"] > 0
    assert 0 < st["entries"] <= sum(len(r) for rs, _ in samples for r in rs)
    # the oracle on one sample's reads, through the four results
    reads = [(r.name, "chr1", False, "____1", r.BX_tag, r.reference_start, r.reference_end, r.is_reverse, [(v.position, v.allele, v.quality) for v in r])
             for r in samples[0][0]]
    bx, r2h, multi, _, loose = haplotag_oracle.prepare([(samples[0][1], reads)], ploidy, False, 50000)
    one = haplotag.assign_reads(samples[:1], ploidy)
    tagged = {one.reprs[i]: (int(one.haplotype[g]), int(one.quality[g]), int(one.block[g]))
              for i, g in enumerate(one.group.tolist()) if g >= 0 and one.haplotype[g] >= 0}
    free = {tuple(m) for ms, _, _, _ in loose for m in ms}
    assert {k: v for k, v in tagged.items() if k not in free} == {k: v for k, v in r2h.items() if k not in free}
    assert int(((one.group == np.arange(len(one.group))) & (one.n_blocks > 1)).sum()) == multi
    # budget-chunked runs equal the resident one
    monkeypatch.setenv("WHMEC_HAPLOTAG_ARENA_BUDGET", str(st["entries"] * 40))
    st2 = {}
    chunked = haplotag.assign_reads(samples, ploidy, linked_read_cutoff=50000, stats=st2)
    assert st2["chunks"] > 1
    for a, b in zip(got[:5], chunked[:5]):
        assert np.array_equal(a, b)
    assert (st2["keys"], st2["runs"], st2["groups"]) == (st["keys"], st["runs"], st["groups"])


def test_several_samples_in_one_call_equal_one_call_each():
    rng = random.Random(5)
    cases = [hc.make_case(rng, big=True, n_samples=2) for _ in range(3)]
    for case in cases:
        want, loose = hc.run_oracle(case)
        assert agrees(want, on_device(case), loose)
    samples = chromosome(9, n_reads=5000, n_samples=3)
    all_at_once = haplotag.assign_reads(samples, 2)
    for s in range(3):
        alone = haplotag.assign_reads(samples[s:s + 1], 2)
        lo, hi = all_at_once.sample_off[s], all_at_once.sample_off[s + 1]
        assert np.array_equal(all_at_once.group[lo:hi], np.where(alone.group >= 0, alone.group + lo, -1))
        for a, b in zip(all_at_once[1:5], alone[1:5]):
            assert np.array_equal(a[lo:hi], b)


def test_errors_on_the_device():
    for case in GOLDEN:
        if isinstance(case["want"], str):
            assert on_device(case) == case["want"]
