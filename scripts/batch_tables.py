"""Several tables in one call (`whmec_solve_batch`, DESIGN §4.8) against a loop of single-table calls.

  python scripts/batch_tables.py [--runs 7] [--sizes 1,2,4,8,16,32] [--out FILE]

For B tables of one shape -- cfg2-shaped single individuals (`synth.sliding_window(10000, 15, block_len=500)`, seeds
20250915 + i) and cfg5-shaped trios scaled to 5000 columns (`synth.trio(5000, 5, block_len=500)`, same seeds) -- times
  flat:       one `_lib.solve_batch` of the B tables       against  B `_lib.solve` calls,
  containers: one `PedigreeDPTable.batch` of the B tables  against  B `PedigreeDPTable(...)` constructors.
Wall time is a host clock around calls that return after the device work has been synchronised; device time is the sum of
the sweeps' CUDA-event times the library reports (`sweep_ms`).  One warm-up round, then --runs rounds in which the two ways
alternate (the order flips every round); median, minimum and maximum are reported.  Every batched solution is compared
with the single-table one bit for bit.

Prints one JSON line per (shape, route, B) with the card's name, power limit and SM clock limit, read (never set) in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from whatshap_b200 import PedigreeDPTable, _lib, multigpu, synth  # noqa: E402

SEED = 20250915
SHAPES = {
    "cfg2-shaped (10000 columns, coverage 15)": lambda i: synth.sliding_window(10_000, 15, block_len=500, seed=SEED + i),
    "cfg5-shaped trio (5000 columns)": lambda i: synth.trio(5_000, 5, block_len=500, seed=SEED + i),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(("gpu", "power_limit", "max_sm_clock"), (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))))


def spread(ms):
    ms = sorted(ms)
    return {"median": round(ms[len(ms) // 2], 3), "min": round(ms[0], 3), "max": round(ms[-1], 3)}


def flat_ways(problems):
    def batch():
        out, (_, total) = _lib.solve_batch(problems, with_stats=True)
        return out, total["sweep_ms"], total["kernel_launches"]

    def loop():
        out, device_ms, launches = [], 0.0, 0
        for p in problems:
            sol, st = _lib.solve(p)
            out.append(sol)
            device_ms += st["sweep_ms"]
            launches += st["kernel_launches"]
        return out, device_ms, launches

    return batch, loop, lambda a, b: all(x.same_as(y) for x, y in zip(a, b))


def container_ways(problems):
    tables = [synth.to_objects(p) for p in problems]

    def batch():
        return PedigreeDPTable.batch(tables), 0.0, 0

    def loop():
        return [PedigreeDPTable(*t) for t in tables], 0.0, 0

    return batch, loop, lambda a, b: all(x._solution.same_as(y._solution) for x, y in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--sizes", default="1,2,4,8,16,32")
    ap.add_argument("--container-sizes", default="1,4,16")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert _lib.device_count() > 0, "needs a CUDA device"
    os.environ.pop(multigpu.ENV_DEVICES, None)
    hw = card()
    sizes = [int(x) for x in a.sizes.split(",")]
    container_sizes = [int(x) for x in a.container_sizes.split(",")]
    records = []
    for shape, make in SHAPES.items():
        problems = [make(i) for i in range(max(sizes + container_sizes))]
        columns = sum(p.n_cols for p in problems[:1])
        for route, ways, route_sizes in (("flat", flat_ways, sizes), ("containers", container_ways, container_sizes)):
            for B in route_sizes:
                batch, loop, same = ways(problems[:B])
                got, want = batch()[0], loop()[0]  # warm-up round, and the comparison
                identical = bool(same(got, want))
                wall = {"batch": [], "loop": []}
                device = {"batch": [], "loop": []}
                launches = {}
                for r in range(a.runs):
                    for way, fn in (("batch", batch), ("loop", loop))[:: 1 if r % 2 == 0 else -1]:
                        t0 = time.perf_counter()
                        _, dev_ms, launches[way] = fn()
                        wall[way].append((time.perf_counter() - t0) * 1e3)
                        device[way].append(dev_ms)
                rec = {"shape": shape, "route": route, "tables": B, "runs": a.runs, "identical_to_single": identical,
                       "wall_ms_batch": spread(wall["batch"]), "wall_ms_loop": spread(wall["loop"]),
                       "columns_per_s_batch": round(B * columns / (spread(wall["batch"])["median"] * 1e-3)),
                       "columns_per_s_loop": round(B * columns / (spread(wall["loop"])["median"] * 1e-3)), "card": hw}
                if route == "flat":
                    rec.update({"device_ms_batch": spread(device["batch"]), "device_ms_loop": spread(device["loop"]),
                                "sweep_launches_batch": launches["batch"], "sweep_launches_loop": launches["loop"]})
                records.append(rec)
                print(json.dumps(rec), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(records, f, indent=1)


if __name__ == "__main__":
    main()
