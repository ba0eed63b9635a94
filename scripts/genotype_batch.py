"""Many genotyping tables in one call (`whmec_genotype_batch`, DESIGN §4.9) against a loop of single-table calls.

  python scripts/genotype_batch.py [--runs 7] [--out FILE]

Two lists: 32 single-sample tables (`synth.genotyping_problem(rng, 2000, 8, "single")`, what `whatshap genotype` builds for a
multi-sample VCF without a pedigree) and 16 trio tables (`synth.genotyping_problem(rng, 1000, 5, "trio")`), seeded.  Each list is
timed as one `_lib.genotype_batch` against one `_lib.genotype` call per table.  Wall time is a host clock around calls that return
after the device work has been synchronised; device time is the sum of the CUDA-event sweep times the library reports
(`sweep_ms`).  One warm-up round, then --runs rounds in which the two ways alternate (the order flips every round); median, minimum
and maximum are reported, with the largest difference between a batched and a single-call likelihood.

Prints one JSON line per list with the card's name, power limit and SM clock limit, read (never set) in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from whatshap_b200 import _lib, multigpu, synth  # noqa: E402

SEED = 20250915
LISTS = {
    "32 single-sample tables (2000 columns, coverage <= 8)": (32, 2000, 8, "single"),
    "16 trio tables (1000 columns, coverage <= 5)": (16, 1000, 5, "trio"),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(("gpu", "power_limit", "max_sm_clock"), (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))))


def spread(ms):
    ms = sorted(ms)
    return {"median": round(ms[len(ms) // 2], 3), "min": round(ms[0], 3), "max": round(ms[-1], 3)}


def ways(problems):
    def batch():
        out, (_, total) = _lib.genotype_batch(problems, with_stats=True)
        return out, total["sweep_ms"], total["kernel_launches"]

    def loop():
        out, device_ms, launches = [], 0.0, 0
        for p in problems:
            lk, st = _lib.genotype(p)
            out.append(lk)
            device_ms += st["sweep_ms"]
            launches += st["kernel_launches"]
        return out, device_ms, launches

    return batch, loop


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert _lib.device_count() > 0, "needs a CUDA device"
    os.environ.pop(multigpu.ENV_DEVICES, None)
    os.environ.pop("WHMEC_GENOTYPE_ARENA_BUDGET", None)
    hw = card()
    records = []
    for name, (n_tables, n_cols, cov, shape) in LISTS.items():
        rng = np.random.default_rng(SEED)
        problems = [synth.genotyping_problem(rng, n_cols, cov, shape) for _ in range(n_tables)]
        batch, loop = ways(problems)
        got, want = batch()[0], loop()[0]  # warm-up round, and the comparison
        worst = max(float(np.nanmax(np.abs(g - w))) for g, w in zip(got, want))
        wall = {"batch": [], "loop": []}
        device = {"batch": [], "loop": []}
        launches = {}
        for r in range(a.runs):
            for way, fn in (("batch", batch), ("loop", loop))[:: 1 if r % 2 == 0 else -1]:
                t0 = time.perf_counter()
                _, dev_ms, launches[way] = fn()
                wall[way].append((time.perf_counter() - t0) * 1e3)
                device[way].append(dev_ms)
        rec = {"list": name, "runs": a.runs, "max_abs_diff_to_single": worst, "wall_ms_batch": spread(wall["batch"]),
               "wall_ms_loop": spread(wall["loop"]), "device_ms_batch": spread(device["batch"]), "device_ms_loop": spread(device["loop"]),
               "sweep_launches_batch": launches["batch"], "sweep_launches_loop": launches["loop"], "card": hw}
        records.append(rec)
        print(json.dumps(rec), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(records, f, indent=1)


if __name__ == "__main__":
    main()
