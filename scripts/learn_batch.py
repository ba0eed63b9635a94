"""K-mer pair counts of `whatshap learn` (`learn.count_kmer_pairs`, DESIGN §4.13) on the seeded synthetic chromosome of
realign_batch.py: 30x of 15 kb reads and 30x of 150 bp reads from two haplotypes, about 5 % errors, variants about every 300 bp.

Reported, as medians over --rounds: the device time of the kernels, the host plan, `count_kmer_pairs` end to end (packing the
Python alignment tuples included), `write_counts` of the rows, and the swap-in `Caller` driven with run_learn's calls.  With
--reference instead, the reference's compiled Caller (oracle/_ref/pyref) on the same reads, once, on the host CPU.  The card's name,
power limit and SM clock limit are read in the same run.  Writes JSON to --out.

    python scripts/learn_batch.py --mb 2 --out learn_batch.json
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.realign_batch import card, synthetic  # noqa: E402
from whatshap_b200 import learn  # noqa: E402

SENTINEL = (10**9, 1)  # the reference reads the entry after the list's front: a far last variant keeps that entry defined


def workload(mb: float, seed: int = 1):
    """(reference bytes, [(VCF position, len(REF))], [(pos, cigartuples, query bytes)]) sorted by position, as run_learn hands
    them over."""
    reference, variants, alns = synthetic(mb, seed)
    vs = [(v.position + 1, len(v.reference_allele)) for v in variants] + [SENTINEL]
    reads = [(a.reference_start, a.cigartuples, a.query_sequence.encode()) for a in alns]
    return reference.encode(), vs, reads


def run_caller(reads, variants, reference, k, window, path, core=None):
    open(path, "w").close()
    out = path.encode()
    caller = (core.Caller if core else learn.Caller)(reference, k, window)
    caller.all_variants(variants)
    for pos, cigar, query in reads:
        caller.add_read(pos, cigar, query, out)
    caller.final_pop(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=2.0)
    ap.add_argument("--k", type=int, default=7)
    ap.add_argument("--window", type=int, default=25)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reference", action="store_true", help="time the reference's compiled Caller instead (host CPU)")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    t = time.perf_counter()
    reference, variants, reads = workload(args.mb)
    res = {"card": card(), "mb": args.mb, "k": args.k, "window": args.window, "variants": len(variants) - 1, "alignments": len(reads),
           "generate_s": time.perf_counter() - t}
    print(json.dumps(res), flush=True)
    if not args.reference:
        learn.count_kmer_pairs(reads[:1000], variants, reference, args.k, args.window)  # warm-up
        dev, plan, e2e, wr, cl = [], [], [], [], []
        with tempfile.TemporaryDirectory() as d:
            for _ in range(args.rounds):
                st = {}
                t = time.perf_counter()
                rows, _ = learn.count_kmer_pairs(reads, variants, reference, args.k, args.window, stats=st)
                e2e.append(time.perf_counter() - t)
                dev.append(st["device_ms"])
                plan.append(st["plan_ms"])
                t = time.perf_counter()
                learn.write_counts(os.path.join(d, "counts.txt"), rows, append=False)
                wr.append(time.perf_counter() - t)
                t = time.perf_counter()
                run_caller(reads, variants, reference, args.k, args.window, os.path.join(d, "caller.txt"))
                cl.append(time.perf_counter() - t)
            same = open(os.path.join(d, "counts.txt"), "rb").read() == open(os.path.join(d, "caller.txt"), "rb").read()
        res["gpu"] = {"kmers": st["kmers"], "kept": st["kept"], "distinct": st["distinct"], "rows": st["rows"], "chunks": st["chunks"],
                      "kernel_launches": st["kernel_launches"], "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"],
                      "device_ms": statistics.median(dev), "plan_ms": statistics.median(plan), "end_to_end_s": statistics.median(e2e),
                      "write_s": statistics.median(wr), "caller_s": statistics.median(cl), "caller_file_equal": same,
                      "kmers_per_s_end_to_end": st["kmers"] / statistics.median(e2e)}
        print(json.dumps({"gpu": res["gpu"]}), flush=True)
    else:
        from oracle import build_pyref

        core = build_pyref.shipped_core()
        if core is not None:
            with tempfile.TemporaryDirectory() as d:
                t = time.perf_counter()
                run_caller(reads, variants, reference, args.k, args.window, os.path.join(d, "ref.txt"), core)
                res["reference_caller_s"] = time.perf_counter() - t
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
