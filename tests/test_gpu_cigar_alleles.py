"""`whmec_detect_alleles_cigar` on the GPU (DESIGN §4.14): every golden case equals the reference's stored answers; a large seeded
workload with 15 kb reads, qualities and several chunks equals the host emulation; budget-chunked runs equal resident ones; the
stats count items, alleles, calls and windows."""
import pytest

from scripts.cigar_alleles_batch import with_qualities
from scripts.realign_batch import synthetic
from test_cigar_alleles import Aln, Var, check_case, emul, golden_cases
from whatshap_b200 import realign

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def no_budget(monkeypatch):
    monkeypatch.delenv("WHMEC_REALIGN_ARENA_BUDGET", raising=False)


@pytest.mark.parametrize("index", range(len(golden_cases())))
def test_golden_case(gpu, index):
    check_case(golden_cases()[index], realign.detect_alleles)


@pytest.fixture(scope="module")
def batch():
    reference, variants, alns = synthetic(1.0, seed=9)
    alns = with_qualities(alns, seed=9)
    # an 1100-base insertion read through, and variants whose normalized positions are out of order
    variants.append(Var(1000, reference[1000], [reference[1000] + "ACGT" * 275]))
    variants.append(Var(5000, reference[5000:5004], [reference[5000]]))
    variants.append(Var(5001, reference[5001], ["A" if reference[5001] != "A" else "C"]))
    variants.sort(key=lambda v: v.position)
    alns.append(Aln(900, [(0, 101), (1, 1100), (0, 300)], reference[900:1001] + "ACGT" * 275 + reference[1001:1301], [35] * 1501))
    return reference, variants, alns


def test_large_batch_equals_emulation(gpu, batch, monkeypatch):
    _, variants, alns = batch
    st, st_e = {}, {}
    got = realign.detect_alleles(alns, variants, None, stats=st)
    want = realign.detect_alleles(alns, variants, None, stats=st_e, library=emul())
    assert got == want
    assert st["items"] == st_e["items"] > 100000 and st["jobs"] == st_e["jobs"] and st["cells"] == sum(map(len, got))
    assert st["chunks"] == 1 and st["device_ms"] > 0
    monkeypatch.setenv("WHMEC_REALIGN_ARENA_BUDGET", str(4 << 20))  # many alignment chunks and item windows
    st_c = {}
    assert realign.detect_alleles(alns, variants, None, stats=st_c) == got
    assert st_c["chunks"] > 4 and st_c["items"] == st["items"]


def test_chunked_equals_resident(gpu, batch, monkeypatch):
    _, variants, alns = batch
    alns = alns[:400] + alns[-1:]
    st = {}
    whole = realign.detect_alleles(alns, variants, None, stats=st)
    for budget in ("1", "100000"):
        monkeypatch.setenv("WHMEC_REALIGN_ARENA_BUDGET", budget)
        st_b = {}
        assert realign.detect_alleles(alns, variants, None, stats=st_b) == whole
        assert st_b["chunks"] > 1 and (budget != "1" or st_b["chunks"] == st["items"])


def test_errors_name_the_first_alignment(gpu):
    ref = "ACGT" * 50
    v = [Var(50, "G", ["C"]), Var(100, "A", ["T"])]
    good = Aln(40, [(0, 30)], ref[40:70], [20] * 30)
    with pytest.raises(ValueError, match=r"^alignment 1: the reference raises ValueError \(Unsupported CIGAR operation: 9\)"):
        realign.detect_alleles([good, Aln(40, [(0, 5), (9, 2), (0, 30)], ref[40:75]), Aln(40, [(0, 30)], ref[40:50])], v, None)
    with pytest.raises(ValueError, match=r"^alignment 2: the reference raises IndexError"):
        realign.detect_alleles([good, good, Aln(40, [(0, 30)], ref[40:50]), Aln(40, [(0, 30)], None)], v, None)
    with pytest.raises(ValueError, match=r"^alignment 0: the reference raises TypeError"):
        realign.detect_alleles([Aln(40, [(0, 30)], None), Aln(40, [(0, 5), (9, 2)], ref[40:45])], v, None)
    assert realign.detect_alleles([good], v, None) == [[(0, 0, 20)]]
