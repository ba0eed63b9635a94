"""`whmec_learn` on the GPU (DESIGN §4.13): every golden case equals the reference's stored file through `count_kmer_pairs` and
through the swap-in `Caller`; chunked runs equal resident ones down to a handful of columns per chunk; reads of 20 kb and more
(one warp each) and a seeded batch of about 10^5 reads equal the host emulation; and, where oracle/_ref/pyref ships it, random
cases equal the reference's compiled Caller live."""
import os
import random
import re
import sys

import numpy as np
import pytest

from test_learn import GOLDEN, blocks, caller_case, count_case, emul, long_reads_case, segments
from whatshap_b200 import learn

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def no_budget(monkeypatch):
    monkeypatch.delenv("WHMEC_LEARN_ARENA_BUDGET", raising=False)


@pytest.mark.parametrize("index", range(len(GOLDEN["cases"])))
def test_golden_case(gpu, index):
    case = GOLDEN["cases"][index]
    assert blocks(count_case(case)) == blocks(case["expected"])


@pytest.mark.parametrize("index", range(len(GOLDEN["cases"])))
def test_golden_case_through_caller(gpu, tmp_path, index):
    case = GOLDEN["cases"][index]
    assert blocks(caller_case(case, tmp_path / "out.txt", None)) == blocks(case["expected"])


def test_fixture_byte_for_byte(gpu, tmp_path):
    fx = GOLDEN["fixture"]
    assert count_case(fx) == fx["expected"]
    assert caller_case(fx, tmp_path / "out.txt", None) == fx["expected"]


@pytest.mark.parametrize("index", range(len(GOLDEN["refusals"])))
def test_refusals(gpu, index):
    c = GOLDEN["refusals"][index]
    reads = [(p, [tuple(x) for x in cg], q.encode()) for p, cg, q in c["reads"]]
    with pytest.raises(ValueError) as e:
        learn.count_kmer_pairs(reads, c["variants"], c["reference"].encode(), c["k"], c["window"])
    assert re.search(c["error"], str(e.value)), (c["name"], str(e.value))


def test_chunked_equals_resident(gpu, monkeypatch):
    rng = random.Random(11)
    ref, reads, variants, k = long_reads_case(rng, n_reads=12, length=1500, k=9)
    ref, reads = ref[:6000], [r for r in reads if r[0] + 1600 < 6000]
    st = {}
    whole, front = learn.count_kmer_pairs(reads, variants, ref, k, 25, stats=st)
    assert st["chunks"] == 1 and len(whole) > 0
    for budget in ("1", "60000", "200000"):  # one column with keys per chunk, then a handful, then more
        monkeypatch.setenv("WHMEC_LEARN_ARENA_BUDGET", budget)
        st_b = {}
        got, f = learn.count_kmer_pairs(reads, variants, ref, k, 25, stats=st_b)
        assert np.array_equal(got, whole) and f == front and st_b["chunks"] > 1, budget


def test_long_reads_on_warps_equal_emulation(gpu):
    rng = random.Random(5)
    ref = "".join(rng.choice("ACGT") for _ in range(80000)).encode()
    reads = []
    for _ in range(30):
        p, n = rng.randrange(0, 80000 - 30000), rng.randrange(20000, 28000)
        q = bytearray(ref[p:p + n])
        for _ in range(40):
            q[rng.randrange(n)] = ord(rng.choice("ACGTNn"))
        reads.append((p, [(4, 5), (0, 5000), (1, 3), (0, 2000), (2, 7), (4, 0), (0, n - 7000)], bytes(q[:7000]) + b"TTT" + bytes(q[7000:])))
    reads.sort(key=lambda r: r[0])
    variants = [(v, rng.choice([1, 3])) for v in sorted(rng.sample(range(1, 80000), 80))] + [(10**9, 1)]
    for k in (7, 15):
        st = {}
        got = learn.count_kmer_pairs(reads, variants, ref, k, 25, stats=st)
        want = learn.count_kmer_pairs(reads, variants, ref, k, 25, library=emul())
        assert np.array_equal(got[0], want[0]) and got[1] == want[1] and len(got[0]) > 100000


def test_large_batch_equals_emulation(gpu):
    sys.path.insert(0, ROOT)
    from scripts.learn_batch import workload

    reference, variants, reads = workload(0.5, seed=4)
    assert len(reads) >= 100000
    st = {}
    got, front = learn.count_kmer_pairs(reads, variants, reference, 7, 25, stats=st)
    want, front_e = learn.count_kmer_pairs(reads, variants, reference, 7, 25, library=emul())
    assert np.array_equal(got, want) and front == front_e
    assert st["kept"] > 10**7 and st["rows"] == len(got)


def test_caller_flushed_in_parts_equals_one_flush(gpu, tmp_path):
    for case in GOLDEN["cases"][:40]:
        whole = caller_case(case, tmp_path / "a.txt", None)
        assert caller_case(case, tmp_path / "b.txt", None, buffer_bytes=40) == whole, case["name"]


def test_random_cases_against_the_compiled_caller(gpu):
    from oracle import build_pyref

    core = build_pyref.shipped_core()
    if core is None:
        pytest.skip("the reference binding is not shipped (oracle/_ref/pyref)")
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_learn_golden as mk

    rng = random.Random(99)
    for idx in range(150):
        case = mk.random_case(rng, idx)
        want = mk.run_reference(core, segments(case), case["variants"], case["k"], case["window"])
        assert blocks(count_case(case)) == blocks(want), case["name"]
