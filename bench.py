#!/usr/bin/env python
"""Benchmark of the weighted-MEC / PedMEC column sweep (the hot path of `whatshap phase`).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--workload cfg3] [--impl ours|reference] [--dump-outputs DIR]

One "step" = one complete forward sweep of the DP over the synthetic workload (all variant
columns of all DP-independent blocks).  Metric: variant-columns per second (BASELINE.json).

  value      device-timed forward sweep + backtrace (+ the 8 bytes / column of the optimal path coming back) with the packed
             ReadSet already resident in HBM: everything the device does for PedigreeDPTable(...) + get_super_reads()
  e2e        the same workload through the C-ABI call `whmec_solve` with HOST buffers:
             packing, allocation, host->device copies, sweep, device backtrace, device->host
             copies and super-read construction are all inside the timed region
  roofline   algorithmic bytes (SURVEY.md §8(d)) / device time of the dominant kernel vs the measured
             HBM copy bandwidth of this pool (MEASURED_PEAKS.json)
  --dump-outputs DIR  writes the solution of the last timed step as DIR/<field>.npy (float64), for comparing two builds
             output for output (the workload is generated from fixed seeds, so the same flags give the same inputs)
  cpu_baseline  the UNMODIFIED reference C++ (oracle/_ref) or the C restatement, single thread,
             on a bounded prefix of the same workload

`--impl reference` times the reference's own CPU implementation on all host cores (independent
block prefixes in parallel; each instance is single-threaded like the reference).
Multi-GPU (torchrun): every rank sweeps its own full-size workload (independent chromosomes /
blocks; weak scaling), no data-path collective; a barrier and max-over-ranks bracket the timing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "variant_columns_per_sec"
UNIT = "columns/s"
WORKLOADS = {
    # name: (description, columns, coverage, T)
    "cfg2": ("synthetic diploid ReadSet: 10k variants, max-coverage 15, single individual", 10_000, 15, 1),
    "cfg3": ("synthetic diploid ReadSet: 50k variants, max-coverage 20, 100 independent blocks", 50_000, 20, 1),
    "cfg3g": ("cfg3 with block lengths ~ Geometric(mean 500) instead of 100 equal blocks (load balance)", 50_000, 20, 1),
    "cfg4": ("synthetic diploid ReadSet: 50k variants, max-coverage 25, one block (2^25 bipartitions)", 50_000, 25, 1),
    "cfg5": ("synthetic trio Pedigree (3 individuals, recombination cost on): 20k variants, coverage 15", 20_000, 15, 4),
}


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workload", default="cfg3", choices=sorted(WORKLOADS))
    ap.add_argument("--cols", type=int, default=None, help="override the number of variant columns")
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed step computed as DIR/<name>.npy (float64, at most 64 MB in all)")
    return ap.parse_args()


class ClockSampler:
    """SM clock / throttle-reason samples DURING the timed region.  The timed region of the default run is a few
    tens of milliseconds, shorter than the start-up of an `nvidia-smi -lms` loop, so the samples are taken through NVML (the library
    nvidia-smi itself reads) every 2 ms by a thread of this process; `nvidia-smi` is the fallback when NVML cannot be loaded."""

    QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, device_index: int):
        self.device_index = device_index
        self.rows = []      # (sm MHz, max MHz, set of reasons)
        self.proc = None
        self.source = None
        self._stop = threading.Event()
        self._thread = None
        self._nvml = None
        try:
            import pynvml

            pynvml.nvmlInit()
            # CUDA_VISIBLE_DEVICES may renumber the devices: resolve the NVML handle through the UUID of the CUDA device
            handle = None
            try:
                import torch

                uuid = "GPU-" + str(torch.cuda.get_device_properties(device_index).uuid)
                handle = pynvml.nvmlDeviceGetHandleByUUID(uuid)
            except Exception:
                handle = None
            if handle is None:
                handle = pynvml.nvmlDeviceGetHandleByIndex(device_index)
            self._nvml, self._handle = pynvml, handle
            self._max = float(pynvml.nvmlDeviceGetMaxClockInfo(handle, pynvml.NVML_CLOCK_SM))
            self.source = "nvml"
        except Exception:
            self._nvml = None

    def _sample_nvml(self):
        nv, h = self._nvml, self._handle
        bits = {"hw_slowdown": nv.nvmlClocksEventReasonHwSlowdown, "hw_thermal_slowdown": nv.nvmlClocksEventReasonHwThermalSlowdown,
                "sw_thermal_slowdown": nv.nvmlClocksEventReasonSwThermalSlowdown, "sw_power_cap": nv.nvmlClocksEventReasonSwPowerCap}
        get_reasons = getattr(nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or getattr(nv, "nvmlDeviceGetCurrentClocksThrottleReasons")
        while not self._stop.is_set():
            try:
                sm = float(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM))
                mask = int(get_reasons(h))
                self.rows.append((sm, self._max, {k for k, b in bits.items() if mask & b}))
            except Exception:
                pass
            self._stop.wait(0.002)

    def start(self):
        if self._nvml is not None:
            self._thread = threading.Thread(target=self._sample_nvml, daemon=True)
            self._thread.start()
            return
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "-i", str(self.device_index), "--query-gpu=" + self.QUERY, "--format=csv,noheader,nounits", "-lms", "20"],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.source = "nvidia-smi"
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:
            self.proc = None

    def _pump(self):
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for line in self.proc.stdout:
            r = [x.strip() for x in line.split(",")]
            try:
                self.rows.append((float(r[1]), float(r[2]), {n for n, v in zip(names, r[4:8]) if v.lower().startswith("active")}))
            except (ValueError, IndexError):
                continue

    def mark(self) -> int:
        """Index of the next sample: the caller brackets its timed region with two marks."""
        return len(self.rows)

    def stop(self, first: int = 0, last: int = None) -> dict:
        if self._thread is not None:
            self._stop.set()
            self._thread.join(timeout=1.0)
        elif self.proc is not None:
            time.sleep(0.05)
            self.proc.terminate()
        else:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no NVML and no nvidia-smi"], "samples": 0}
        rows = self.rows[first:last]
        window = "timed region"
        if len(rows) < 3:  # a slow sampler (nvidia-smi fallback): fall back to everything sampled under load since start()
            rows, window = self.rows, "warm-up + timed region"
        reasons = set()
        for r in rows:
            reasons |= r[2]
        sm = [r[0] for r in rows]
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(r[1] for r in rows) if rows else None,
                "reasons": sorted(reasons), "samples": len(rows), "source": self.source, "window": window}


def hbm_peak():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        return float(json.load(open(path))["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    return 3350.0, "H100 SXM data sheet (HBM3), not measured"


DUMP_BUDGET = 64 * 10**6  # bytes of .npy data --dump-outputs may write


def dump_outputs(out_dir, sol):
    """The FlatSolution the timed path returned (plan.finish() of the last step) as float64 arrays: every uint32 is exact.
    An array larger than its share of DUMP_BUDGET is replaced by a fixed, seeded sample of its flattened elements."""
    import numpy as np

    arrays = {"cost": np.array([sol.cost])}
    for f in ("path_index", "path_tv", "partition", "sr_allele", "sr_quality"):
        arrays[f] = np.asarray(getattr(sol, f))
    share = DUMP_BUDGET // len(arrays)
    os.makedirs(out_dir, exist_ok=True)
    for name, a in arrays.items():
        a = a.astype(np.float64)
        if a.nbytes > share:
            keep = np.sort(np.random.default_rng(0).choice(a.size, share // a.itemsize, replace=False))
            a = a.reshape(-1)[keep]
        np.save(os.path.join(out_dir, name + ".npy"), a)


def make_workload(name, cols, rank):
    from whatshap_b200 import synth

    prob = synth.config(name, cols)
    if rank:  # other ranks phase other chromosomes: same shape, different reads
        from whatshap_b200.synth import SEEDS, sliding_window, trio

        n = prob.n_cols
        if name == "cfg5":
            prob = trio(n, 5, block_len=500, seed=SEEDS[name] + rank)
        elif name == "cfg3g":
            prob = sliding_window(n, 20, block_len=synth.geometric_blocks(n, 500.0, SEEDS[name] + rank), seed=SEEDS[name] + rank)
        else:
            cov = WORKLOADS[name][2]
            prob = sliding_window(n, cov, block_len=(n if name == "cfg4" else 500), seed=SEEDS[name] + rank)
    return prob


def cpu_sample(name, prob, target_cols):
    """A bounded prefix of block 0 with the same structure (reads clipped to the prefix)."""
    from whatshap_b200 import synth
    from whatshap_b200.synth import SEEDS

    cov = WORKLOADS[name][2]
    if name == "cfg5":
        return synth.trio(target_cols, 5, block_len=target_cols, seed=SEEDS[name])
    return synth.sliding_window(target_cols, cov, block_len=target_cols, seed=SEEDS[name])


CPU_SAMPLE_COLS = {"cfg2": 4000, "cfg3": 160, "cfg3g": 160, "cfg4": 6, "cfg5": 1500}
# reference arm (--impl reference): columns per instance and step, one instance per host thread (a step takes seconds)
REF_SAMPLE_COLS = {"cfg2": 400, "cfg3": 16, "cfg3g": 16, "cfg4": 4, "cfg5": 150}
REF_MAX_THREADS = {"cfg4": 32}  # 3 x 128 MiB per stored column and instance in the reference's layout


def run_cpu_baseline(name, prob):
    from oracle import checker

    ref = checker.reference()
    cols = CPU_SAMPLE_COLS[name]
    if ref is None:  # only the C restatement travelled: it is much slower than the reference, shrink the sample
        ck, kind, cols = checker.port(), "port", max(2, cols // 8)
    else:
        ck, kind = ref, "reference"
    sample = cpu_sample(name, prob, cols)
    t0 = time.perf_counter()
    ck.solve(sample)
    dt = ck.last_seconds if kind == "reference" else time.perf_counter() - t0
    return {"value": cols / dt, "unit": UNIT, "cores": 1, "kind": kind,
            "sample": f"{cols}-column prefix of block 0 of {name} (same generator, same coverage), {dt:.2f} s single thread"}


def bench_reference(args, rank, world):
    """Reference arm: the unmodified C++ PedigreeDPTable on all host cores."""
    if rank != 0:
        return
    from oracle import checker

    name = args.workload
    ref = checker.reference()
    threads = os.cpu_count() or 1
    from whatshap_b200 import synth
    from whatshap_b200.synth import SEEDS

    cov = WORKLOADS[name][2]

    def make(cols, count):  # one independent block prefix per host thread
        out = []
        for i in range(count):
            if name == "cfg5":
                out.append(synth.trio(cols, 5, block_len=cols, seed=SEEDS[name] + 1000 + i))
            else:
                out.append(synth.sliding_window(cols, cov, block_len=cols, seed=SEEDS[name] + 1000 + i))
        return out

    # FIXED sample (no time-based calibration: the ratio against this arm must be reproducible): one independent
    # block prefix of REF_SAMPLE_COLS columns per host thread, every instance single-threaded like the reference.
    # A step of that size takes ~20 s at coverage 20 on 128 threads; so that `--steps K --warmup W` still ends within a few
    # minutes whatever K and W the caller picks, the prefix is shortened as a function of K + W alone (deterministic: the same
    # flags give the same sample): full length up to 6 calls, e.g. 4 columns for --steps 20 --warmup 5.
    calls = args.steps + args.warmup + 1
    cols = max(2, min(REF_SAMPLE_COLS[name], (REF_SAMPLE_COLS[name] * 13 // 2) // calls))
    threads = min(threads, REF_MAX_THREADS.get(name, threads))
    probs = make(cols, threads)
    if ref is not None:
        kind = "reference"
        step = lambda: ref.solve_many_timed(probs, threads)
    else:
        kind = "port"
        port = checker.port()

        def step():
            t0 = time.perf_counter()
            for p in probs[:1]:
                port.solve(p)
            return (time.perf_counter() - t0)
        probs = probs[:1]
    step()  # one discarded call (page faults, allocator growth) on top of the requested warm-up
    for _ in range(args.warmup):
        step()
    times = [step() for _ in range(args.steps)]
    total_cols = cols * len(probs)
    value = total_cols * len(times) / sum(times)
    single = None
    if ref is not None:  # the reference is single-threaded: one instance alone on the box
        ref.solve_many_timed(probs[:1], 1)
        single = cols / ref.solve_many_timed(probs[:1], 1)
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": 1e3 * sum(times) / len(times), "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "u32", "data": "synthetic",
        "config": {"workload": name, "description": WORKLOADS[name][0],
                   "sample": f"{len(probs)} independent {cols}-column block prefixes per step, one per host thread "
                             f"(prefix length fixed by --steps + --warmup = {args.steps + args.warmup})"},
        "cpu_baseline": {"value": value, "unit": UNIT, "cores": threads if kind == "reference" else 1, "kind": kind,
                         "sample": f"{len(probs)} x {cols} columns per step (fixed sample)",
                         "single_thread_value": single},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


def main():
    args = parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        if args.dump_outputs:
            raise SystemExit("--dump-outputs writes what the CUDA path computed; --impl reference times the CPU reference only")
        bench_reference(args, rank, world)
        return

    import torch
    import torch.distributed as dist

    from whatshap_b200 import _lib

    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (there is no CPU path in whatshap_b200)")
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))

    name = args.workload
    prob = make_workload(name, args.cols, rank)
    n_cols = prob.n_cols
    flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")  # 10x the 50 MB L2 of an H100

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- device-resident sweep ------------------------------------------------------------
    plan = _lib.Plan(prob, device=local_rank)
    sampler = ClockSampler(local_rank)
    sampler.start()  # before the warm-up, so that even a slow sampler has samples under load
    for _ in range(max(args.warmup, 3)):
        plan.sweep()
        plan.finish()
    barrier()
    mark0 = sampler.mark()
    wall0 = time.perf_counter()
    sweep_ms, step_ms = [], []
    for _ in range(args.steps):
        flush.fill_(1)  # evict the previous step's state / back-pointers from L2 (not timed)
        torch.cuda.synchronize()
        plan.sweep()    # timed on the launching stream with CUDA events inside the library
        sol = plan.finish()  # device: backtrace kernels + D2H of the path (timed with events); host: super-reads (not in `value`, in `e2e`)
        st = plan.stats()
        sweep_ms.append(st["sweep_ms"])
        step_ms.append(st["sweep_ms"] + st["d2h_ms"])
    barrier()
    wall = time.perf_counter() - wall0
    clocks = sampler.stop(mark0, sampler.mark())
    stats = plan.stats()
    plan.close()
    total_ms = sum(step_ms)
    t = torch.tensor([total_ms], dtype=torch.float64, device="cuda")
    cols_t = torch.tensor([float(n_cols)], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.all_reduce(cols_t, op=dist.ReduceOp.SUM)
    max_ms = float(t.item())
    all_cols = float(cols_t.item())
    value = all_cols * args.steps / (max_ms / 1e3)

    # ---- end to end through the C ABI with host buffers ------------------------------------
    _lib.solve(prob, device=local_rank)  # warm-up (context, allocator)
    barrier()
    e2e_t0 = time.perf_counter()
    e2e_steps = max(1, args.steps)
    for _ in range(e2e_steps):
        sol2, st2 = _lib.solve(prob, device=local_rank)
    barrier()
    e2e_dt = time.perf_counter() - e2e_t0
    assert sol2.same_as(sol), "resident and end-to-end runs disagree"
    e2e_t = torch.tensor([e2e_dt], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(e2e_t, op=dist.ReduceOp.MAX)
    e2e_value = all_cols * e2e_steps / float(e2e_t.item())

    # ---- the object-level call a user of the reference makes: PedigreeDPTable(readset, recombcost, pedigree) + get_super_reads()
    # on this package's container objects (rank 0, N = 1): includes the Python-side flattening of the ReadSet
    e2e_api = None
    if world == 1:
        from whatshap_b200 import PedigreeDPTable, synth

        rs, rc_list, ped = synth.to_objects(prob)
        PedigreeDPTable(rs, rc_list, ped).get_super_reads()  # warm-up
        torch.cuda.synchronize()
        api_t0 = time.perf_counter()
        for _ in range(e2e_steps):
            table = PedigreeDPTable(rs, rc_list, ped, device=local_rank)
            superreads, tv = table.get_super_reads()
            cost_api = table.get_optimal_cost()
        api_dt = time.perf_counter() - api_t0
        assert cost_api == int(sol.cost) and list(superreads[0][0]._allele) == sol.sr_allele[0, 0].tolist(), "object-level and flat results disagree"
        e2e_api = {"value": n_cols * e2e_steps / api_dt, "unit": UNIT, "ms_per_step": 1e3 * api_dt / e2e_steps,
                   "note": "PedigreeDPTable(readset, recombcost, pedigree) + get_super_reads() on container objects: flattening of the "
                           "ReadSet (from the columnar copy its add() keeps, numpy passes every call, nothing cached between calls) + "
                           "whmec_solve + super-read objects"}

    # ---- strong scaling: ONE problem (rank 0's) sharded over all ranks, end to end from rank 0's host arrays --------
    sharded = None
    if world > 1:
        from whatshap_b200 import _wire, multigpu

        comm = _wire.Comm()
        comm.warm_up()  # communicator set-up is not part of a solve
        shared = prob if rank == 0 else None
        multigpu.solve_sharded(shared, comm=comm)  # warm-up (contexts, allocators on every rank)
        barrier()
        sh_t0 = time.perf_counter()
        phases = {}
        for _ in range(e2e_steps):
            phases = {}
            sol_sh = multigpu.solve_sharded(shared, comm=comm, timings=phases)
        barrier()
        sh_dt = time.perf_counter() - sh_t0
        sh_t = torch.tensor([sh_dt], dtype=torch.float64, device="cuda")
        dist.all_reduce(sh_t, op=dist.ReduceOp.MAX)
        if rank == 0:
            assert sol_sh.same_as(sol), "sharded and single-GPU solves disagree: " + sol_sh.diff(sol)
            sharded = {"value": n_cols * e2e_steps / float(sh_t.item()), "unit": UNIT, "ms_per_step": 1e3 * float(sh_t.item()) / e2e_steps,
                       "scaling": "strong", "columns": n_cols, "ranks": world, "phases_ms_rank0": {k: round(v, 2) for k, v in phases.items()},
                       "note": "multigpu.solve_sharded: rank 0's host arrays -> cut into blocks (T = 1) or table segments (T > 1) -> tensor "
                               "scatter -> per-rank whmec_solve / whmec_segment_* -> tensor gather -> merged result on rank 0; bit-identical "
                               "to the single-GPU solve (asserted)"}

    if rank == 0:
        peak, peak_src = hbm_peak()
        launches = int(stats["kernel_launches"])
        achieved = stats["algorithmic_bytes"] / (statistics.mean(sweep_ms) / 1e3) / 1e9
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
            "ms_per_step": max_ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "u32", "data": "synthetic",
            "config": {
                "workload": name, "description": WORKLOADS[name][0], "columns_per_gpu": n_cols,
                "coverage": WORKLOADS[name][2], "transmission_vectors": WORKLOADS[name][3],
                "chains": int(stats["n_chains"]), "kernel_path": {1: "tile (mirrored panels)", 2: "column", 3: "pedigree two-pass sweep (fused per chain)" if launches == 3 else "pedigree two-pass sweep (batched)"}.get(int(stats["path_kind"]), "mixed"),
                "value_covers": "forward sweep + backtrace + path D2H, device-timed (CUDA events)",
                "l2": "512 MiB buffer rewritten between timed steps (L2 flush)", "sharding": "one full-size workload per GPU, no collective on the data path",
                "optimal_cost_rank0": int(sol.cost), "wall_s_timed_region": wall,
            },
            "roofline": {
                "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                "peak_source": peak_src,
                "algorithmic_bytes_per_launch": stats["algorithmic_bytes"] / max(launches, 1),
                "kernel": {1: "tile_panel_kernel", 2: "col_direct_kernel", 3: "ped_fused_kernel" if launches == 3 else "col_batched_kernel"}.get(int(stats["path_kind"]), "col_direct_kernel"),
                "algorithmic_bytes_per_step": int(stats["algorithmic_bytes"]), "launches_per_step": launches,
                "bytes_moved_per_step": {"backpointers": int(stats["backptr_bytes"]), "state": int(stats["state_bytes"])},
                "note": ("algorithmic bytes follow the reference's data layout (u32 projection read + u32 value and u32 back-pointer "
                         "written per entry and column, SURVEY.md 8(d)); the tile kernel keeps the projection in shared memory for a "
                         "whole panel of columns and stores 1-bit back-pointers, so its real DRAM traffic is far below "
                         "that and frac can exceed 1: the kernel is bound by integer issue, see dp_cells_per_s"),
                "dp_cells_per_s": stats["cells"] / (statistics.mean(sweep_ms) / 1e3),
                "sweep_ms": statistics.mean(sweep_ms), "backtrace_ms": statistics.mean(step_ms) - statistics.mean(sweep_ms),
            },
            "clocks": clocks,
            "e2e_api": e2e_api,
            "e2e": {"value": e2e_value, "unit": UNIT, "h2d_bytes_per_step": int(st2["h2d_bytes"]), "d2h_bytes_per_step": int(st2["d2h_bytes"]),
                    "ms_per_step": 1e3 * float(e2e_t.item()) / e2e_steps, "steps": e2e_steps,
                    "note": "whmec_solve: host CSR arrays in, host result arrays out (pack + alloc + H2D + sweep + backtrace + D2H)"},
            # forward-sweep kernels + backtrace kernels (1 for a single individual, 3 for a pedigree) per timed step
            "gpu_launches": (launches + (3 if int(stats["transmissions"]) > 1 else 1)) * args.steps,
        }
        if sharded is not None:
            line["e2e_sharded"] = sharded
        if not args.no_cpu_baseline and world == 1:
            line["cpu_baseline"] = run_cpu_baseline(name, prob)
        if args.dump_outputs:
            dump_outputs(args.dump_outputs, sol)
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
