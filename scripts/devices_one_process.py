"""One table over several GPUs from one process (`devices=`, DESIGN §6) against the single-device call.

  python scripts/devices_one_process.py [--runs 3] [--out FILE]

Times the container-level calls a `whatshap phase` / `whatshap genotype` run makes: `PedigreeDPTable` on the cfg3 and cfg5
shapes (`synth.config`), and `GenotypeDPTable` on the cfg5-shaped trio of DESIGN §4.5 (`synth.trio(20000, 5)`, random priors,
phred-scaled recombination costs).  Each table is built three ways: `devices=None` (one GPU), every visible GPU, and device 0
repeated as often (at least twice: with one GPU only this row and the single-device row exist).  Wall time around the
constructor, which returns after the device work has been synchronised; --runs rounds after a warm-up round, the ways
alternating within a round.  Every result is compared with the single-device call: phasing bit for bit, genotyping as the
largest absolute difference.

Prints one JSON line per (table, way) with the cards' names and power limits, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from whatshap_b200 import _lib, core, multigpu, synth  # noqa: E402


def cards():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return [dict(zip(("index", "gpu", "power_limit"), (x.strip() for x in line.split(",")))) for line in q.stdout.strip().splitlines()]


def genotyping_trio(cols, seed=20250935):
    rng = np.random.default_rng(seed)
    prob = synth.trio(cols, 5, seed=seed)
    prob.gl = rng.random((3, prob.n_cols, 3)) + 0.05
    prob.gl /= prob.gl.sum(axis=2, keepdims=True)
    prob.recombcost = rng.integers(0, 30, prob.n_cols).astype(np.uint32)
    prob.distrust = True
    return prob


def with_priors(prob):
    """(ReadSet, recombcost, Pedigree) whose individuals carry `prob.gl` as genotype priors."""
    rs, recomb, plain = synth.to_objects(prob)
    ped = core.Pedigree(plain.numeric_sample_ids)
    for i in range(prob.n_ind):
        ped.add_individual(i, plain._genotypes[i], [core.PhredGenotypeLikelihoods(prob.gl[i, k].tolist()) for k in range(prob.n_cols)])
    tr = prob.trios.tolist()
    for t in range(prob.n_trios):
        ped.add_relationship(tr[3 * t], tr[3 * t + 1], tr[3 * t + 2])
    return rs, recomb, ped


def tables(cols_cfg5_genotype):
    """(name, build(devices) -> table, compare(table, single-device table) -> dict, problem)"""
    for name in ("cfg3", "cfg5"):
        prob = synth.config(name)
        rs, recomb, ped = synth.to_objects(prob)
        positions = prob.positions.tolist()
        yield (name + " PedigreeDPTable", lambda devices, rs=rs, recomb=recomb, ped=ped, positions=positions:
               core.PedigreeDPTable(rs, recomb, ped, False, positions, devices=devices),
               lambda got, one: {"same_as_single_device": bool(got._solution.same_as(one._solution))}, prob)
    prob = genotyping_trio(cols_cfg5_genotype)
    rs, recomb, ped = with_priors(prob)
    positions = prob.positions.tolist()
    yield ("cfg5-shaped trio GenotypeDPTable", lambda devices: core.GenotypeDPTable(ped.numeric_sample_ids, rs, recomb, ped, positions, devices=devices),
           lambda got, one: {"max_abs_diff_from_single_device": float(np.nanmax(np.abs(got._likelihoods - one._likelihoods)))}, prob)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--genotype-cols", type=int, default=20_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    visible = _lib.device_count()
    assert visible > 0, "needs a CUDA device"
    os.environ.pop(multigpu.ENV_DEVICES, None)
    hw = cards()
    repeat = max(visible, 2)
    ways = {"one device": None, "device 0 x%d" % repeat: [0] * repeat}
    if visible > 1:
        ways["all %d devices" % visible] = list(range(visible))
    records = []
    for name, build, compare, prob in tables(a.genotype_cols):
        single = build(None)
        for devices in ways.values():  # warm-up round: module loads, memory pools, host threads
            build(devices)
        times = {way: [] for way in ways}
        last = {}
        order = list(ways)
        for r in range(a.runs):
            for way in order[r % len(order):] + order[:r % len(order)]:
                t0 = time.perf_counter()
                last[way] = build(ways[way])
                times[way].append((time.perf_counter() - t0) * 1e3)
        for way, devices in ways.items():
            ms = sorted(times[way])
            rec = {"table": name, "cols": prob.n_cols, "way": way, "devices": devices, "wall_ms_median": round(ms[len(ms) // 2], 2),
                   "wall_ms_min": round(ms[0], 2), "wall_ms_max": round(ms[-1], 2), "runs": a.runs,
                   "mode": last[way].stats.get("mode", "single device"), "cards": hw}
            rec.update(compare(last[way], single))
            records.append(rec)
            print(json.dumps(rec), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(records, f, indent=1)


if __name__ == "__main__":
    main()
