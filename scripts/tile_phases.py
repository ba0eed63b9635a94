"""Where the tile kernel's time goes, per phase of a work item (DESIGN §4.1).

  python scripts/tile_phases.py [--workloads cfg3,cfg4] [--out FILE]

Builds a second copy of libwhmec.so in a temporary directory, with tile.cu compiled under -DWHMEC_TILE_PHASE_CLOCKS and
linked against the in-tree objects of the normal build (run `__graft_entry__.build()` first).  In that build thread 0 of
every CTA of tile_panel_kernel records clock64() at five points of each work item (one tile of one panel):

    start -> input in place -> tables built -> columns done -> end of the item

plus the cycles it spends waiting at the column barrier of steady-state panels and waiting for the completion counter of
the producer panel (an input that was not prefetched).  The normal build's SASS does not change:
every line the macro adds is inside #ifdef.  For each workload the script runs one warm-up sweep, then collects one
sweep + backtrace (step 0) and prints one JSON line with the share of CTA time in each phase:

    input      staging the tile's input (bulk copies / gather) and transposing it into the local order (of which
               `producer_wait`: thread 0 waiting for the producer panel)
    tables     issuing the next tile's prefetch, waiting for the column records (requested when the item started) and
               building the per-column tables
    columns    the column loop (of which `barrier_wait`: thread 0 waiting at the split column barrier)
    writeback  storing the tile for the next panel

`outside_plus_wait` = input + tables + writeback + barrier_wait: the time in which the SM's schedulers have little or
nothing of this CTA to issue.  Shares are of the summed (end - start) of the recorded items; at most 2^20 items are recorded
per collection (cfg4 has more, the first ones are kept).  Needs a CUDA device.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "whatshap_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
OBJS = ["whmec.o", "genotype.o", "col_plan.o", "gl_batch.o", "gl_pack.o", "pack.o", "tile_plan.o", "hostpool.o", "readselect.o", "heuristic.o",
        "heuristic_batch.o", "heuristic_cu.o"]
REC_WORDS = 8  # PhaseRec: t[5], wait, (smid, block), (steady, producer_wait)
CAP = 1 << 20


def build_phase_library(tmp: str) -> str:
    missing = [o for o in OBJS if not os.path.exists(os.path.join(CSRC, o))]
    if missing:
        raise SystemExit(f"objects of the normal build are missing ({', '.join(missing)}): run __graft_entry__.build() first")
    obj = os.path.join(tmp, "tile_phase.o")
    subprocess.run([NVCC, "-O3", "-std=c++17", *ARCH, "-lineinfo", "-ccbin", "/usr/bin/g++", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
                    "-DWHMEC_TILE_PHASE_CLOCKS", "-c", "-o", obj, os.path.join(CSRC, "tile.cu")], check=True, capture_output=True)
    so = os.path.join(tmp, "libwhmec.so")
    subprocess.run([NVCC, "-shared", *ARCH, "-ccbin", "/usr/bin/g++", "-o", so, obj, *[os.path.join(CSRC, o) for o in OBJS],
                    "-cudart", "static"], check=True)
    return so


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clk = (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "sm_clock_max": clk}


def shares(rec: np.ndarray) -> dict:
    t = rec[:, :5].astype(np.int64)
    d = np.diff(t, axis=1)  # input, tables, columns, writeback
    total = float(d.sum())
    wait = float(rec[:, 5].astype(np.int64).sum())
    out = {name: round(float(d[:, i].sum()) / total, 4) for i, name in enumerate(("input", "tables", "columns", "writeback"))}
    out["barrier_wait"] = round(wait / total, 4)
    out["producer_wait"] = round(float((rec[:, 7] >> np.uint64(32)).astype(np.int64).sum()) / total, 4)
    out["outside_plus_wait"] = round((float(d[:, 0].sum() + d[:, 1].sum() + d[:, 3].sum()) + wait) / total, 4)
    out["items"] = int(len(rec))
    out["mean_item_cycles"] = round(total / max(len(rec), 1), 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg4")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="whmec_phase_")
    os.environ["WHMEC_LIBRARY"] = build_phase_library(tmp)
    sys.path.insert(0, ROOT)
    from whatshap_b200 import _lib, synth

    assert _lib.device_count() > 0, "needs a CUDA device"
    L = _lib.lib()
    L.whmec_tile_phase_reset.restype = C.c_int
    L.whmec_tile_phase_read.restype = C.c_longlong
    L.whmec_tile_phase_read.argtypes = [C.c_void_p, C.c_ulonglong]
    buf = np.zeros((CAP, REC_WORDS), dtype=np.uint64)
    info = card()
    for name in a.workloads.split(","):
        prob = synth.config(name)
        plan = _lib.Plan(prob)
        plan.sweep()
        plan.finish()  # warm-up
        assert L.whmec_tile_phase_reset() == 0
        plan.sweep()
        plan.finish()
        n = L.whmec_tile_phase_read(buf.ctypes.data, CAP)
        assert n >= 0, "reading the phase records failed"
        st = plan.stats()
        plan.close()
        rec = buf[:min(n, CAP)]
        steady = (rec[:, 7] & 0xFFFFFFFF) != 0
        line = {"workload": name, "items_seen": int(n), "launches": int(st["kernel_launches"]), "sweep_ms": st["sweep_ms"],
                "all": shares(rec), "steady_panels": shares(rec[steady]) if steady.any() else None,
                "other_panels": shares(rec[~steady]) if (~steady).any() else None, **info}
        s = json.dumps(line)
        print(s, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(s + "\n")


if __name__ == "__main__":
    main()
