"""Read merging of `whatshap phase --merge-reads` on the GPU (whmec_merge_reads, DESIGN §4.17) on seeded synthetic chromosomes:
20 000 sorted reads of 20 to 200 variants on two haplotypes, variants 1 bp apart (dense: every read meets hundreds of later
reads) or 1 kbp apart (sparse, WGS-like: the reference's end = begin + variant count leaves few pairs), and a dense chromosome of
60 000 reads.  Prints one JSON line per shape: the device time of the call's kernels, the host plan time, the wall time of
merge_reads and of ReadMerger.merge (medians of --repeats after a warm-up call), the wall time of the oracle
(oracle/merge_oracle.py, the reference's rules in plain Python) on the same input where it is run, whether the outputs are
equal, and the card's name, power limit and SM clock limit read in the same run.

    python scripts/merge_batch.py [--repeats 3] [--oracle-reads 20000]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from oracle import merge_oracle  # noqa: E402
from test_gpu_merge import chromosome  # noqa: E402
from whatshap_b200 import merge  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--oracle-reads", type=int, default=20000, help="run the oracle on shapes of at most this many reads")
    args = ap.parse_args()
    gpu = gpu_info()
    for name, n, span, spacing in (("dense", 20000, 20000, 1), ("sparse", 20000, 20000, 1000), ("dense60k", 60000, 20000, 1)):
        rs = chromosome(11, n, span, spacing=spacing)
        merge.merge_reads([rs], device=0)  # warm-up
        dev, plan, call, obj = [], [], [], []
        for _ in range(args.repeats):
            st = {}
            t0 = time.perf_counter()
            (got,) = merge.merge_reads([rs], device=0, stats=st)
            call.append(time.perf_counter() - t0)
            dev.append(st["device_ms"])
            plan.append(st["plan_ms"])
            t0 = time.perf_counter()
            merge.ReadMerger(0.15, 0.25, 1000000, 1000, device=0).merge(rs)
            obj.append(time.perf_counter() - t0)
        row = {"shape": name, "reads": st["reads"], "entries": st["entries"], "pairs": st["pairs"], "blue_edges": st["blue_edges"],
               "merged_components": st["merged_components"], "output_reads": st["output_reads"], "chunks": st["chunks"],
               "kernel_launches": st["kernel_launches"], "kernels_ms": statistics.median(dev), "plan_ms": statistics.median(plan),
               "merge_reads_s": statistics.median(call), "read_merger_s": statistics.median(obj), "repeats": args.repeats}
        if n <= args.oracle_reads:
            reads = [[(v.position, v.allele, v.quality) for v in r] for r in rs]
            t0 = time.perf_counter()
            want = merge_oracle.merge(reads)
            row["oracle_s"] = time.perf_counter() - t0
            off = got.entry_off.tolist()
            mine = [("read%d" % r, list(zip(got.position[off[k]:off[k + 1]].tolist(), got.allele[off[k]:off[k + 1]].tolist(),
                                            got.quality[off[k]:off[k + 1]].tolist()))) for k, r in enumerate(got.read.tolist())]
            row["equal"] = mine == want
        row["gpu"] = gpu
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
