"""Resident vs memory-bounded forward-backward genotyping on the GPU (DESIGN §4.5).

  python scripts/genotype_memory_bounded.py [--cols 20000] [--reps 3] [--out FILE]

A cfg5-shaped trio genotyping problem (`synth.trio(cols, 5)`: 15 reads per column; random priors, phred-scaled recombination
costs, distrusted genotypes): resident, then bounded with WHMEC_GENOTYPE_ARENA_BUDGET at 1/2, 1/4 and 1/8 of the resident
backward tables.  For each: device time (sweep_ms, median of --reps), kernel launches, bytes of backward tables (arena +
checkpoints when bounded), and the largest absolute difference from the resident likelihoods.

Prints one JSON line per measurement, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from whatshap_b200 import _lib, synth  # noqa: E402

HOOK = "WHMEC_GENOTYPE_ARENA_BUDGET"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def problem(cols, seed=20250935):
    rng = np.random.default_rng(seed)
    prob = synth.trio(cols, 5, seed=seed)
    prob.gl = rng.random((3, prob.n_cols, 3)) + 0.05
    prob.gl /= prob.gl.sum(axis=2, keepdims=True)
    prob.recombcost = rng.integers(0, 30, prob.n_cols).astype(np.uint32)
    prob.distrust = True
    return prob


def timed(prob, reps):
    """Median over `reps` calls of the device time (CUDA events around the sweeps), with the last likelihoods."""
    times, got, st = [], None, None
    for _ in range(reps):
        got, st = _lib.genotype(prob)
        times.append(st["sweep_ms"])
    times.sort()
    return got, st, times[len(times) // 2]


def emit(out, rec):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cols", type=int, default=20_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert _lib.device_count() > 0, "needs a CUDA device"
    hw = card()
    os.environ.pop(HOOK, None)
    prob = problem(a.cols)
    try:
        _lib.genotype(prob)  # warm-up: module load, memory pool
        whole, st, ms = timed(prob, a.reps)
        resident = st["backptr_bytes"]
        emit(a.out, dict(hw, case="cfg5-shaped trio genotyping", cols=a.cols, budget="resident", device_ms=round(ms, 3),
                         launches=st["kernel_launches"], backward_bytes=resident, max_abs_diff=0.0))
        for div in (2, 4, 8):
            os.environ[HOOK] = str(resident // div)
            got, st2, ms2 = timed(prob, a.reps)
            emit(a.out, dict(hw, case="cfg5-shaped trio genotyping", cols=a.cols, budget=f"1/{div}", device_ms=round(ms2, 3),
                             launches=st2["kernel_launches"], backward_bytes=st2["backptr_bytes"],
                             max_abs_diff=float(np.nanmax(np.abs(got - whole)))))
    finally:
        os.environ.pop(HOOK, None)


if __name__ == "__main__":
    main()
