"""The column-kernel plan (col_plan.cpp, DESIGN §4.2) on the CPU: which sweep a problem gets, and the segments of the
memory-bounded sweep under the arena hook (WHMEC_COLUMN_ARENA_BUDGET) and under the free HBM.  The GPU tests
(test_gpu_ped_bounded.py) run these plans; here their invariants are checked for budgets the device cannot be made to show."""
import re

import numpy as np
import pytest

from emul_col_plan import col_plan
from whatshap_b200 import multigpu, synth
from whatshap_b200._abi import WHMEC_ERR_UNSUPPORTED

RESERVE = 512 << 20  # free HBM the plan leaves to everything else
PEDS = ["trio", "trio_child_first", "quartet", "three_generations", "three_children", "four_children"]
COV = {"trio": 9, "trio_child_first": 9, "quartet": 8, "three_generations": 7, "three_children": 6, "four_children": 6}
PATHS = {"default": {}, "batched": {"fused": False}, "sequential": {"sequential": True}}


def instance(ped, chains="several", distrust=False, seed=0):
    """The problems of test_gpu_ped_bounded: a random_problem with at least four chains, or with exactly one."""
    for attempt in range(200):
        rng = np.random.Generator(np.random.PCG64([seed, attempt]))
        if chains == "one":
            prob = synth.random_problem(rng, 40, COV.get(ped, 10), ped, distrust=distrust, gap=0.1, mean_len=8.0, burst=4)
            if len(multigpu.independent_blocks(prob)) == 1:
                return prob
        else:
            prob = synth.random_problem(rng, 90, COV.get(ped, 10), ped, distrust=distrust)
            if len(multigpu.independent_blocks(prob)) >= 4:
                return prob
    raise AssertionError("no instance of the wanted chain structure")


def resident(prob, **kw):
    r = col_plan(prob, **kw)
    assert r["rc"] == 0 and not r["bounded"], r["msg"]
    return r


def check_segments(bounded, res, budget_words):
    """Cuts ascend over the whole table, every segment's offsets are rebased to 0 and fit the arena, the arena fits
    `budget_words` (None: not checked), and the last segment is as large as the budget allowed (returned: its growth by one
    chain or column, in words)."""
    n, cb, cuts = len(res["bp_off"]), bounded["chain_begin"], bounded["cuts"]
    off = np.append(res["bp_off"], res["bp_words"])  # resident offsets, off[n] = the resident size
    two_pass = bounded["path"] != "column"
    assert cuts[0] == 0 and cuts[-1] == (len(cb) - 1 if two_pass else n) and np.all(np.diff(cuts) > 0), cuts
    col_cuts = cb[cuts] if two_pass else cuts
    for k0, k1 in zip(col_cuts[:-1], col_cuts[1:]):
        assert np.array_equal(bounded["bp_off"][k0:k1], off[k0:k1] - off[k0])
        assert off[k1] - off[k0] <= bounded["arena"]
    if budget_words is not None:
        assert bounded["arena"] <= budget_words
    if len(cuts) < 3:
        return None
    before = cb[cuts[-2] - 1] if two_pass else cuts[-2] - 1  # first column of the chain (or the column) before the last segment
    return off[n] - off[before]


def test_path_choice():
    trio = synth.trio(120, 5, block_len=60, seed=20250935)  # cfg5 shape: 2 chains
    assert resident(trio)["path"] == "fused"
    assert resident(trio, fused=False)["path"] == "batched"
    assert resident(trio, sequential=True)["path"] == "column"
    assert resident(instance("trio", distrust=True))["path"] == "batched"  # distrust: more allele assignments than the fused shape holds
    assert resident(synth.nuclear_family(200, 2, 2, block_len=50, seed=3))["path"] == "batched"  # T = 16
    assert resident(instance("trio", chains="one"))["path"] == "column"
    assert resident(synth.sliding_window(120, 12, block_len=120, seed=4))["path"] == "column"  # T = 1
    assert resident(instance("single"))["path"] == "column"


def test_fused_cluster():
    trio = synth.trio(120, 5, block_len=60, seed=20250935)
    assert resident(trio)["cluster"] == 8  # 2 chains on 132 SMs
    assert resident(trio, sms=8)["cluster"] == 4
    assert resident(trio, cluster=2)["cluster"] == 2
    assert resident(trio, cluster=3)["cluster"] == 8  # not a cluster size: automatic


@pytest.mark.parametrize("ped", PEDS + ["single"])
def test_ample_budget_is_resident(ped):
    prob = instance(ped)
    r = resident(prob)
    assert r["arena"] == r["bp_words"] and r["ckpt"] == 0 and len(r["cuts"]) == 0
    assert r["bp_off"][0] == 0 and np.all(np.diff(r["bp_off"]) >= 0) and r["bp_off"][-1] < r["bp_words"]
    assert np.array_equal(resident(prob, hook=4 * r["bp_words"])["bp_off"], r["bp_off"])  # a hook the table fits changes nothing


def least_hook(prob, **kw):
    r = col_plan(prob, hook=8, **kw)
    assert r["rc"] == WHMEC_ERR_UNSUPPORTED and "an arena of 8 bytes holds no segment" in r["msg"], r
    return int(re.search(r"needs at least (\d+) bytes", r["msg"]).group(1))


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("ped", PEDS)
def test_hook_budgets(ped, path):
    prob = instance(ped, seed=PEDS.index(ped) * 4)
    res = resident(prob, **PATHS[path])
    cut = 0
    for hook in sorted({least_hook(prob, **PATHS[path]), res["bp_words"] * 4 * 2 // 3, res["bp_words"] * 4 // 3, res["bp_words"] * 4 // 8}):
        b = col_plan(prob, hook=hook, **PATHS[path])
        if b["rc"] != 0:  # (a divisor below the least budget of this instance)
            assert hook < 4 * max(np.diff(np.append(res["bp_off"], res["bp_words"]))), b["msg"]
            continue
        assert b["bounded"] and not b["over_hbm"] and b["budget"] == hook
        assert b["path"] in {res["path"], "column"}  # (a chain beyond the hook takes the column sweep)
        grown = check_segments(b, res, hook // 4)
        if grown is not None:
            cut += 1
            assert grown > hook // 4  # the last segment is the largest that fits
    assert cut >= 2


@pytest.mark.parametrize("path", ["default", "batched"])
@pytest.mark.parametrize("ped", ["trio", "three_children"])
def test_chain_beyond_the_hook_takes_the_column_sweep(ped, path):
    prob = instance(ped, seed=PEDS.index(ped) * 4)
    res = resident(prob, **PATHS[path])
    assert res["path"] != "column"
    off = np.append(res["bp_off"], res["bp_words"])
    chain_words = max(np.diff(off[res["chain_begin"]]))
    b = col_plan(prob, hook=4 * chain_words, **PATHS[path])
    assert b["rc"] == 0 and b["bounded"] and b["path"] == res["path"]
    b = col_plan(prob, hook=4 * chain_words - 4, **PATHS[path])
    assert b["rc"] == 0 and b["bounded"] and b["path"] == "column"
    check_segments(b, res, chain_words - 1)


def test_refusal_states_a_budget_that_plans():
    prob = synth.nuclear_family(30, 4, 2, block_len=30, seed=1)  # T = 256
    need = least_hook(prob)
    b = col_plan(prob, hook=need)
    assert b["rc"] == 0 and b["bounded"] and b["arena"] * 4 <= need


BIG = {  # large enough for checkpoints to leave room under the free-bytes budget
    "cfg5-shaped trio": lambda: synth.trio(120, 5, block_len=60, seed=20250935),
    "three_children": lambda: synth.nuclear_family(40, 3, 2, block_len=20, seed=7),
    "single": lambda: synth.sliding_window(2000, 12, block_len=400, seed=4),
}


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("key", list(BIG))
def test_free_bytes_budget(key, path):
    """No hook: the free HBM less everything else is the budget of the arena and the checkpoints together."""
    prob = BIG[key]()
    res = resident(prob, **PATHS[path])
    paths = set()
    for divisor in (1.2, 1.5, 2):
        free = res["fixed"] + RESERVE + int(4 * res["bp_words"] / divisor)
        b = col_plan(prob, free_bytes=free, bounded_t1=True, **PATHS[path])
        assert b["rc"] == 0 and b["bounded"] and not b["over_hbm"], b["msg"]
        assert b["budget"] <= free - res["fixed"] - RESERVE
        assert 4 * (b["arena"] + b["ckpt"]) <= b["budget"]
        grown = check_segments(b, res, None)
        # the last segment is the largest that fits: beyond the budget (two-pass), beyond the arena the cut allowed (column)
        assert grown > (b["budget"] // 4 if b["path"] != "column" else b["arena"])
        paths.add(b["path"])
    assert paths == ({"fused"} if (key, path) == ("cfg5-shaped trio", "default") else {"column"})


def test_over_hbm():
    prob = synth.sliding_window(600, 10, block_len=600, seed=4)  # T = 1, one chain
    res = resident(prob)
    free = res["fixed"] + RESERVE + 2 * res["bp_words"]  # half the back-pointers fit
    r = col_plan(prob, free_bytes=free)
    assert r["rc"] == WHMEC_ERR_UNSUPPORTED and r["over_hbm"] and r["msg"] == "back-pointer storage exceeds the free HBM of this device"
    b = col_plan(prob, free_bytes=free, bounded_t1=True)
    assert b["rc"] == 0 and b["bounded"] and not b["over_hbm"]
    trio = BIG["cfg5-shaped trio"]()
    res = resident(trio)
    b = col_plan(trio, free_bytes=res["fixed"] + RESERVE + 2 * res["bp_words"])
    assert b["rc"] == 0 and b["bounded"] and not b["over_hbm"] and b["path"] == "fused"


@pytest.mark.parametrize("segment", [1, 2])
def test_segment_plans(segment):
    trio = instance("trio")
    res = resident(trio, segment=segment)
    assert res["path"] == "fused"
    r = resident(trio, segment=segment, hook=8)  # the hook does not apply to segments
    assert r["arena"] == res["bp_words"] and np.array_equal(r["bp_off"], res["bp_off"])
    r = col_plan(trio, segment=segment, free_bytes=res["fixed"] + RESERVE + 2 * res["bp_words"])
    assert r["rc"] == WHMEC_ERR_UNSUPPORTED and r["over_hbm"] and not r["bounded"]
    # the back-pointers fit, the batch buffers do not: no two-pass sweep, and a segment has no other
    r = col_plan(trio, segment=segment, fused=False, free_bytes=res["fixed"] + RESERVE + 4 * res["bp_words"] + 4096)
    assert r["rc"] == WHMEC_ERR_UNSUPPORTED and not r["over_hbm"] and not r["bounded"]
    assert r["msg"] == "unsupported: this segment cannot run the two-pass pedigree sweep (costs beyond 2^28 or state beyond the budget)"
    assert resident(trio, segment=segment, sequential=True)["path"] == "fused"  # sequential is for whole tables
