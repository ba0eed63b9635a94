"""Votes of `whatshap haplotagphase` on the GPU (whmec_haplotagphase, DESIGN §4.16) on a seeded synthetic chromosome: per sample
`--reads` reads with 20 entries each, two samples, sized as scripts/haplotag_batch.py.  Prints one JSON line: the device time of
the call's kernels (after a warm-up call), the host plan time, the wall time of the swap-in (compute_votes and consensus of
every sample, as run_haplotagphase calls them), the wall time of the oracle (oracle/haplotagphase_oracle.py, the reference's
rules in plain Python) on the same input, whether the outputs are equal, and the card's name, power limit and SM clock limit
read in the same run.

    python scripts/haplotagphase_batch.py [--reads 500000] [--repeats 3]
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

from oracle import haplotagphase_oracle as o  # noqa: E402
from test_gpu_haplotagphase import chromosome  # noqa: E402
from whatshap_b200 import haplotagphase as hp  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=500000)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    samples = chromosome(3, n_reads=args.reads)
    hp.vote(samples)  # warm-up
    dev, plan, swap = [], [], []
    for _ in range(args.repeats):
        st = {}
        hp.vote(samples, stats=st)
        dev.append(st["device_ms"])
        plan.append(st["plan_ms"])
        t0 = time.perf_counter()
        mine = []
        for s in samples:
            votes = hp.compute_votes(s.homozygous, s.reads, s.allele_to_id)
            change = {p: type("V", (), {"is_snv": (lambda v: lambda self: v)(f)})() for p, f in s.is_snv.items()}
            mine.append((votes,) + hp.consensus(False, 70, 10, "", change, s.phased, votes, s.id_to_allele))
        swap.append(time.perf_counter() - t0)
    t0 = time.perf_counter()
    theirs = []
    for s in samples:
        reads = [(r.HP_tag, r.PS_tag, [(v.position, v.allele, v.quality) for v in r]) for r in s.reads]
        votes, _ = o.votes_of(s.homozygous, reads, s.allele_to_id)
        theirs.append((votes,) + o.consensus(votes, {p: v is not None for p, v in s.phased.items()}, s.is_snv, s.id_to_allele, 70, False))
    oracle_s = time.perf_counter() - t0
    equal = all(m[0] == t[0] and [(v.position, v.allele, v.quality) for v in m[1][0]] == t[1][0]
                and [(v.position, v.allele, v.quality) for v in m[1][1]] == t[1][1] and list(m[2].items()) == t[2]
                for m, t in zip(mine, theirs))
    print(json.dumps({"reads_per_sample": args.reads, "samples": len(samples), "entries": st["entries"], "positions": st["positions"],
                      "records": st["records"], "chunks": st["chunks"], "kernels_ms": statistics.median(dev),
                      "plan_ms": statistics.median(plan), "swap_in_s": statistics.median(swap), "oracle_s": oracle_s, "equal": equal,
                      "gpu": gpu_info()}))


if __name__ == "__main__":
    main()
