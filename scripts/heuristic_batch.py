"""Many heuristic tables in one call (`whmec_heuristic_batch`, one CTA per table, DESIGN §4.10) against the host solver.

  python scripts/heuristic_batch.py [--runs 3] [--lists a,b,...] [--row-limit 256] [--out FILE]

Lists (seeded; `row_limit` 256 unless --row-limit says otherwise):
  cov30x32, cov40x32, cov30x256, cov40x256   single-sample tables of 5000 columns, `synth.sliding_window(5000, c)` (coverage c,
                                            reads of c columns), 32 or 256 of them
  triox16                                   16 trio tables, `synth.trio(2000, 10)` (coverage 10 per individual)
  short10x32                                32 single-sample tables of 200 columns at coverage 10
Each list is run three ways: one `_lib.heuristic_batch` call; `_lib.heuristic` over a host thread pool with one worker per core
(ctypes releases the GIL, so the tables run in parallel); and `_lib.heuristic` one table after the other.  Batch and pool are
timed for --runs rounds (medians, minima and maxima of a host clock; the batch also reports the device time of its launches).
The sequential way is timed once per table on the 32- and 16-table lists; a 256-table list reports 8 x its 32-table list's
sequential time (same generator, the first 32 tables are the same tables), marked "scaled".  Every batched table is compared
with the host solver's answer (`same_as`: bipartition, transmission, haplotypes, mutations).

Prints one JSON line per list with the card's name, power limit and SM clock limit and the host's core count, read in the same
run."""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from whatshap_b200 import _lib, multigpu, synth  # noqa: E402

LISTS = {
    "cov30x32": (32, lambda s: synth.sliding_window(5000, 30, block_len=5000, seed=s)),
    "cov40x32": (32, lambda s: synth.sliding_window(5000, 40, block_len=5000, seed=s)),
    "cov30x256": (256, lambda s: synth.sliding_window(5000, 30, block_len=5000, seed=s)),
    "cov40x256": (256, lambda s: synth.sliding_window(5000, 40, block_len=5000, seed=s)),
    "triox16": (16, lambda s: synth.trio(2000, 10, block_len=2000, seed=s)),
    "short10x32": (32, lambda s: synth.sliding_window(200, 10, block_len=200, seed=s)),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    hw = dict(zip(("gpu", "power_limit", "max_sm_clock"), (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))))
    hw["host_cores"] = os.cpu_count()
    return hw


def spread(ms):
    ms = sorted(ms)
    return {"median": round(ms[len(ms) // 2], 1), "min": round(ms[0], 1), "max": round(ms[-1], 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--lists", default=",".join(LISTS))
    ap.add_argument("--row-limit", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    row_limit = a.row_limit
    assert _lib.device_count() > 0, "needs a CUDA device"
    os.environ.pop(multigpu.ENV_DEVICES, None)
    os.environ.pop("WHMEC_HEURISTIC_ARENA_BUDGET", None)
    hw = card()
    pool = ThreadPoolExecutor(max_workers=os.cpu_count())
    sequential = {}  # per-table host times of the 32-table lists, for their 256-table lists
    records = []
    for name in a.lists.split(","):
        n_tables, make = LISTS[name]
        problems = [make(1000 + s) for s in range(n_tables)]
        _lib.heuristic_batch(problems[:2], row_limit, True)  # warm-up: module load, first launch

        def batch():
            out, (stats, total) = _lib.heuristic_batch(problems, row_limit, True, with_stats=True)
            return out, total["sweep_ms"], sum(st["path_kind"] == 6 for st in stats)

        def pooled():
            return list(pool.map(lambda p: _lib.heuristic(p, row_limit, True), problems))

        rec = {"list": name, "tables": n_tables, "columns": problems[0].n_cols, "row_limit": row_limit, "runs": a.runs}
        wall = {"batch": [], "pool": []}
        device_ms = []
        want = None
        for r in range(a.runs):
            for way in (("batch", "pool") if r % 2 == 0 else ("pool", "batch")):
                t0 = time.perf_counter()
                if way == "batch":
                    got, dev, on_device = batch()
                    device_ms.append(dev)
                else:
                    want = pooled()
                wall[way].append((time.perf_counter() - t0) * 1e3)
        rec["same_as_host"] = sum(g.same_as(w) for g, w in zip(got, want))
        rec["swept_on_device"] = on_device
        rec["wall_ms_batch"] = spread(wall["batch"])
        rec["device_ms_batch"] = spread(device_ms)
        rec["wall_ms_pool"] = spread(wall["pool"])
        if n_tables <= 32:
            per = []
            for p in problems:
                t0 = time.perf_counter()
                _lib.heuristic(p, row_limit, True)
                per.append((time.perf_counter() - t0) * 1e3)
            sequential[name] = per
            rec["wall_ms_sequential"] = round(sum(per), 1)
        else:
            base = name.replace("x256", "x32")
            if base in sequential:
                rec["wall_ms_sequential_scaled"] = round(sum(sequential[base]) * n_tables / len(sequential[base]), 1)
        rec["card"] = hw
        records.append(rec)
        print(json.dumps(rec), flush=True)
    pool.shutdown()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(records, f, indent=1)


if __name__ == "__main__":
    main()
