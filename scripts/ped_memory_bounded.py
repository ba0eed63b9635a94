"""Resident vs memory-bounded pedigree sweeps on the GPU (DESIGN §4.2).

  python scripts/ped_memory_bounded.py [--cfg5-cols 20000] [--reps 3] [--family-cols N] [--leave-free-gb G] [--out FILE]

1. cfg5 (the trio of bench.py): resident, then bounded at 1/2, 1/4 and 1/8 of its arena (WHMEC_COLUMN_ARENA_BUDGET): device
   time of sweep + backtrace (median of --reps), kernel launches, arena bytes, and whether the solution equals the resident one.
2. A `three_children` family (T = 64, 3 reads per sample) whose resident back-pointers exceed the free HBM: solved with the
   budget the free HBM gives, and again with a hook budget of half that arena; the two solutions must be equal.
   --leave-free-gb G first fills the device with a ballast tensor until about G GB are free, so that a family of moderate size
   (and run time) already exceeds the free HBM; the ballast is freed before the script ends.

Prints one JSON line per measurement, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from whatshap_b200 import _lib, synth  # noqa: E402

HOOK = "WHMEC_COLUMN_ARENA_BUDGET"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def timed(prob, reps):
    """Median over `reps` solves of the device time (sweep + backtrace and copies, CUDA events), with the last solution."""
    times, sol, st = [], None, None
    for _ in range(reps):
        sol, st = _lib.solve(prob)
        times.append(st["sweep_ms"] + st["d2h_ms"])
    times.sort()
    return sol, st, times[len(times) // 2]


def emit(out, rec):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg5-cols", type=int, default=20_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--family-cols", type=int, default=0, help="three_children columns (0: skip part 2)")
    ap.add_argument("--leave-free-gb", type=float, default=0.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert _lib.device_count() > 0, "needs a CUDA device"
    hw = card()
    os.environ.pop(HOOK, None)

    prob = synth.config("cfg5", a.cfg5_cols)
    _lib.solve(prob)  # warm-up: module load, memory pool
    whole, st, ms = timed(prob, a.reps)
    resident = st["backptr_bytes"]
    emit(a.out, dict(hw, case="cfg5", cols=a.cfg5_cols, budget="resident", device_ms=round(ms, 3), launches=st["kernel_launches"],
                     arena_bytes=resident, path_kind=st["path_kind"], equal=True))
    for div in (2, 4, 8):
        os.environ[HOOK] = str(resident // div)
        _lib.solve(prob)
        got, st2, ms2 = timed(prob, a.reps)
        emit(a.out, dict(hw, case="cfg5", cols=a.cfg5_cols, budget=f"1/{div}", device_ms=round(ms2, 3), launches=st2["kernel_launches"],
                         arena_bytes=st2["backptr_bytes"], path_kind=st2["path_kind"], equal=bool(got.same_as(whole))))
    os.environ.pop(HOOK, None)

    if a.family_cols:
        ballast = None
        if a.leave_free_gb:
            import torch

            free, _ = torch.cuda.mem_get_info()
            spare = int(free - a.leave_free_gb * 1e9)
            if spare > 0:
                ballast = torch.empty(spare, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
        try:
            fam = synth.nuclear_family(a.family_cols, 3, 3, block_len=a.family_cols, seed=5)
            t0 = time.perf_counter()
            first, st3 = _lib.solve(fam)
            wall = time.perf_counter() - t0
            free_now = None
            if ballast is not None:
                import torch

                free_now = torch.cuda.mem_get_info()[0]
            emit(a.out, dict(hw, case="three_children", cols=a.family_cols, budget="free HBM", free_hbm_bytes=free_now,
                             device_ms=round(st3["sweep_ms"] + st3["d2h_ms"], 3), wall_s=round(wall, 3), launches=st3["kernel_launches"],
                             arena_bytes=st3["backptr_bytes"], path_kind=st3["path_kind"], cost=int(first.cost)))
            os.environ[HOOK] = str(st3["backptr_bytes"] // 2)
            t0 = time.perf_counter()
            second, st4 = _lib.solve(fam)
            wall = time.perf_counter() - t0
            emit(a.out, dict(hw, case="three_children", cols=a.family_cols, budget="1/2 of the first arena",
                             device_ms=round(st4["sweep_ms"] + st4["d2h_ms"], 3), wall_s=round(wall, 3), launches=st4["kernel_launches"],
                             arena_bytes=st4["backptr_bytes"], path_kind=st4["path_kind"], equal=bool(second.same_as(first))))
        finally:
            os.environ.pop(HOOK, None)
            del ballast


if __name__ == "__main__":
    main()
