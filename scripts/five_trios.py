"""A five-trio family on the GPU: the wide column sweep (T = 1024, DESIGN §4.7), resident and memory-bounded.

  python scripts/five_trios.py [--cols 20000] [--out FILE]

Solves synth.nuclear_family(cols, 5, 2) (father, mother, five children, two reads per sample and column: 14 active reads) with the
back-pointers resident, then with WHMEC_COLUMN_ARENA_BUDGET at 1/2 and 1/4 of the resident arena.  Per run: device ms (sweep +
backtrace and copies, CUDA events), columns/s, kernel launches, back-pointer bytes, and the largest difference of any output field
from the resident run (must be 0).  Prints one JSON line per run, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from whatshap_b200 import _lib, synth  # noqa: E402

HOOK = "WHMEC_COLUMN_ARENA_BUDGET"
FIELDS = ("path_index", "path_tv", "partition", "sr_allele", "sr_quality")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def max_diff(a, b):
    d = abs(int(a.cost) - int(b.cost))
    for f in FIELDS:
        d = max(d, int(np.abs(getattr(a, f).astype(np.int64) - getattr(b, f).astype(np.int64)).max(initial=0)))
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cols", type=int, default=20_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert _lib.device_count() > 0, "needs a CUDA device"
    hw = card()
    os.environ.pop(HOOK, None)
    prob = synth.nuclear_family(a.cols, 5, 2)
    resident = None
    for div in (1, 2, 4):
        if div > 1:
            os.environ[HOOK] = str(resident_bytes // div)
        sol, st = _lib.solve(prob)
        ms = st["sweep_ms"] + st["d2h_ms"]
        if resident is None:
            resident, resident_bytes = sol, st["backptr_bytes"]
        rec = dict(hw, case="nuclear_family(5 children, 2 reads per sample)", cols=a.cols, budget="resident" if div == 1 else f"1/{div}",
                   device_ms=round(ms, 3), columns_per_s=round(a.cols / (ms / 1e3), 1), launches=st["kernel_launches"],
                   backptr_bytes=st["backptr_bytes"], path_kind=st["path_kind"], max_diff_from_resident=max_diff(sol, resident),
                   cost=int(sol.cost))
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")
    os.environ.pop(HOOK, None)


if __name__ == "__main__":
    main()
