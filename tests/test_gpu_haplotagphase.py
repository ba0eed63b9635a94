"""Votes of `whatshap haplotagphase` on the GPU (whmec_haplotagphase, DESIGN §4.16): every stored case of the reference on the
device, resident and one position per chunk, in both input forms; a seeded chromosome of 500 000 reads per sample and two
samples against the emulation and the oracle; several samples in one call against one call each; and the call's counters."""
import json
import os

import numpy as np
import pytest

import haplotagphase_cases as hc
import whatshap_b200
from whatshap_b200 import _lib, haplotagphase as hp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

with np.load(os.path.join(ROOT, "tests", "golden", "haplotagphase.npz")) as z:
    GOLDEN = json.loads(z["cases"].tobytes())


@pytest.fixture(autouse=True)
def gpu(monkeypatch):
    if _lib.device_count() == 0:
        pytest.skip("no CUDA device")
    monkeypatch.delenv("WHMEC_HAPLOTAGPHASE_ARENA_BUDGET", raising=False)


def on_device(case, plain_dicts=False, stats=None):
    cv = lambda *a: hp.compute_votes(*a, device=0, stats=stats)
    if plain_dicts:
        cs = lambda *a: hp.consensus(*a[:6], {p: dict(v) for p, v in a[6].items()}, a[7], device=0)
    else:
        cs = lambda *a: hp.consensus(*a, device=0)
    return hc.run_functions(cv, cs, case, whatshap_b200)


def test_every_golden_case_on_the_device():
    assert [i for i, c in enumerate(GOLDEN) if on_device(c) != c["want"]] == []
    assert [i for i, c in enumerate(GOLDEN) if on_device(c, plain_dicts=True) != c["want"]] == []


def test_golden_cases_one_position_per_chunk(monkeypatch):
    monkeypatch.setenv("WHMEC_HAPLOTAGPHASE_ARENA_BUDGET", "1")
    assert [i for i, c in enumerate(GOLDEN) if on_device(c) != c["want"]] == []
    assert [i for i, c in enumerate(GOLDEN) if on_device(c, plain_dicts=True) != c["want"]] == []


def chromosome(seed, n_reads=500000, n_samples=2, entries=20, n_ps=40):
    """A seeded chromosome: n_reads per sample with `entries` entries each over about n_reads / 4 records (15 % homozygous,
    30 % phased), n_ps phase sets, 3 % of the reads with HP or PS missing or HP 3.  Returns [hp.Sample]."""
    rng = np.random.default_rng(seed)
    n_var = n_reads // 4
    pos = np.unique(rng.integers(1, 40 * n_var, n_var))
    samples = []
    for s in range(n_samples):
        homozygous = rng.random(len(pos)) < 0.15
        phased = rng.random(len(pos)) < 0.3
        snv = rng.random(len(pos)) < 0.7
        first = rng.integers(0, 2, len(pos))
        pl = pos.tolist()
        hom = {p: bool(h) for p, h in zip(pl, homozygous.tolist())}
        a2i = {p: ({f: 0} if h else {f: 0, 1 - f: 1}) for p, f, h in zip(pl, first.tolist(), homozygous.tolist())}
        i2a = {p: {i: a for a, i in m.items()} for p, m in a2i.items()}
        rs = whatshap_b200.ReadSet()
        starts = np.sort(rng.integers(0, len(pos) - entries, n_reads))
        hps = np.where(rng.random(n_reads) < 0.97, rng.integers(1, 3, n_reads), rng.choice([-1, 0, 3], n_reads))
        pss = (starts * n_ps) // len(pos) * 100 + 1 + rng.integers(0, 2, n_reads)
        alleles = rng.integers(0, 2, (n_reads, entries))
        quals = rng.integers(1, 60, (n_reads, entries))
        for k in range(n_reads):
            i0 = int(starts[k])
            r = whatshap_b200.Read(f"read{k}", 60, 0, s, pl[i0], "", int(hps[k]), int(pss[k]))
            for j in range(entries):
                r.add_variant(pl[i0 + j], int(alleles[k, j]) if not homozygous[i0 + j] else int(first[i0 + j]), int(quals[k, j]))
            rs.add(r)
        samples.append(hp.Sample(rs, hom, a2i, i2a, {p: (1 if f else None) for p, f in zip(pl, phased.tolist())},
                                 dict(zip(pl, snv.tolist()))))
    return samples


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a[:-1], b[:-1])) and a[-1] == b[-1]


def test_chromosome_equals_the_emulation_and_the_oracle(monkeypatch):
    from oracle import haplotagphase_oracle as o

    from test_haplotagphase import emul

    samples = chromosome(3)
    st = {}
    got = hp.vote(samples, gap_threshold=70, stats=st)
    want = hp.vote(samples, gap_threshold=70, library=emul())
    assert all(same(a, b) for a, b in zip(got, want))
    assert st["chunks"] == 2 and st["device_ms"] > 0 and st["entries"] > 10 ** 7 and st["records"] >= st["positions"] > 0
    # the oracle on the first sample
    s = samples[0]
    reads = [(r.HP_tag, r.PS_tag, [(v.position, v.allele, v.quality) for v in r]) for r in s.reads]
    votes, skipped = o.votes_of(s.homozygous, reads, s.allele_to_id)
    sup, comp = o.consensus(votes, {p: v is not None for p, v in s.phased.items()}, s.is_snv, s.id_to_allele, 70, False)
    assert got[0].as_dict() == votes and got[0].skipped == skipped
    assert [(int(p), int(c)) for p, c in zip(got[0].position, got[0].phase_set)] == comp
    kept = sorted((int(p), int(a[0]), int(sc)) for p, a, sc, k in zip(got[0].position, got[0].allele, got[0].score, got[0].kept) if k)
    assert kept == sup[0]
    # budget-chunked runs equal the resident one
    monkeypatch.setenv("WHMEC_HAPLOTAGPHASE_ARENA_BUDGET", str(st["entries"] * 40))
    st2 = {}
    chunked = hp.vote(samples, gap_threshold=70, stats=st2)
    assert st2["chunks"] > 2 and all(same(a, b) for a, b in zip(got, chunked))
    assert (st2["entries"], st2["positions"], st2["records"]) == (st["entries"], st["positions"], st["records"])


def test_several_samples_in_one_call_equal_one_call_each():
    samples = chromosome(9, n_reads=20000, n_samples=3)
    st = {}
    together = hp.vote(samples, only_indels=True, stats=st)
    assert st["chunks"] == 3 and st["kernel_launches"] == 18
    for s in range(3):
        alone = {}
        (one,) = hp.vote(samples[s:s + 1], only_indels=True, stats=alone)
        assert same(together[s], one)
        assert alone["h2d_bytes"] < st["h2d_bytes"]
