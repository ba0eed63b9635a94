"""Read assignment of `whatshap haplotag` on the GPU (whmec_haplotag, DESIGN §4.15) on a seeded synthetic chromosome: per sample
`--reads` reads with about 20 phased heterozygous entries each, 400 phase sets, 10 % of the reads in BX clouds, two samples,
at ploidy 2 and 4.  Prints, as one JSON line per ploidy: the device time of the call's kernels, the wall time of
`prepare_haplotag_information` (the swap-in, from the variant table to its four results), the wall time of the oracle
(oracle/haplotag_oracle.py, the reference's rules in plain Python) on the same input, whether the two agree, and the card's
name and power limit read in the same run.

    python scripts/haplotag_batch.py [--reads 500000] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import haplotag_cases as hc  # noqa: E402
import whatshap_b200  # noqa: E402
from oracle import haplotag_oracle  # noqa: E402
from whatshap_b200 import haplotag  # noqa: E402


def workload(seed, n_reads, ploidy, n_samples=2, n_blocks=400, entries=20):
    """A case in the form of tests/haplotag_cases.py (variant table rows and reads) built with numpy."""
    rng = np.random.default_rng(seed)
    n_var = max(n_reads // 4, entries + 1)
    pos = np.unique(rng.integers(1, 40 * n_var, n_var))
    block = pos[(np.arange(len(pos)) * n_blocks) // len(pos)].tolist()
    case = {"ploidy": ploidy, "ignore": False, "cutoff": 50000, "chromosome": "chr1", "positions": pos.tolist(), "calls": {}, "reads": {},
            "samples": [f"S{s}" for s in range(n_samples)]}
    for s in case["samples"]:
        phase = rng.integers(0, 2, (len(pos), ploidy))
        phase[:, 0] = 1 - phase[:, 1]  # heterozygous
        case["calls"][s] = [[ph, b, ph] for ph, b in zip(phase.tolist(), block)]
        first = np.sort(rng.integers(0, len(pos) - entries, n_reads))
        alleles, quals = rng.integers(0, 2, (n_reads, entries)).tolist(), rng.integers(1, 40, (n_reads, entries)).tolist()
        in_cloud = rng.random(n_reads) < 0.1
        cloud = rng.integers(0, max(1, n_reads // 100), n_reads)
        pl = pos.tolist()
        case["reads"][s] = [[f"read{k}", 0, "chr1", False, "____1", f"BX{cloud[k]}" if in_cloud[k] else "", pl[i], pl[i + entries], bool(k & 1),
                             [[pl[i + j], alleles[k][j], quals[k][j]] for j in range(entries)]] for k, i in enumerate(first.tolist())]
    return case


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=500000, help="reads per sample")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--ploidy", type=int, nargs="*", default=[2, 4])
    args = ap.parse_args()
    card = gpu_info()
    for ploidy in args.ploidy:
        case = workload(ploidy, args.reads, ploidy)
        table, reader = hc.VariantTable(case), hc.Reader(case, whatshap_b200)
        readsets = {s: reader.read("chr1", None, s)[0] for s in case["samples"]}
        fixed = type("R", (), {"read": lambda self, c, v, s, regions=None: (readsets[s], None)})()
        device_ms, wall = [], []
        for _ in range(args.repeats + 1):  # the first call warms the library and the device up
            st = {}
            t0 = time.perf_counter()
            got = haplotag.prepare_haplotag_information(table, case["samples"], fixed, None, False, 50000, ploidy, stats=st)
            wall.append(time.perf_counter() - t0)
            device_ms.append(st["device_ms"])
        t0 = time.perf_counter()
        want = haplotag_oracle.prepare(hc.oracle_samples(case), ploidy, False, 50000)
        oracle_s = time.perf_counter() - t0
        equal = hc.same(hc.as_plain(*want[:4]), hc.as_plain(*got), [[[list(m) for m in ms], b, s, [list(o) if o else None for o in opts]]
                                                                 for ms, b, s, opts in want[4]])
        print(json.dumps({"ploidy": ploidy, "reads_per_sample": args.reads, "samples": len(case["samples"]), "entries": st["entries"],
                          "groups": st["groups"], "keys": st["keys"], "runs": st["runs"], "chunks": st["chunks"],
                          "device_ms_median": float(np.median(device_ms[1:])), "plan_ms": st["plan_ms"],
                          "swap_in_s_median": float(np.median(wall[1:])), "oracle_s": oracle_s, "equal": bool(equal), "gpu": card}), flush=True)
        if not equal:
            sys.exit(1)


if __name__ == "__main__":
    main()
