"""Float exactness of the device heuristic (DESIGN §4.10), from the SASS and the ptxas report.

  python scripts/heuristic_sass.py [--obj whatshap_b200/csrc/heuristic_cu.o] [--log whatshap_b200/csrc/heuristic.ptxas.log]

heur_batch_kernel must round every float operation on its own, as the host solver does (heuristic.cpp is compiled without
contraction): heuristic.cu is built with -fmad=false.  This disassembles the object (nvdisasm, no GPU needed), counts the kernel's
float opcodes and fails if any fused multiply-add (FFMA) is left; it prints the kernel's registers, stack and spills from the
ptxas log and fails on spills.  Run `__graft_entry__.build()` first (or pass --obj / --log).
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
CSRC = os.path.join(ROOT, "whatshap_b200", "csrc")


def disassemble(obj: str) -> str:
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-xelf", "all", os.path.abspath(obj)], cwd=tmp, check=True,
                       capture_output=True)
        cubins = [f for f in os.listdir(tmp) if f.endswith(".cubin")]
        if not cubins:
            raise SystemExit(f"no cubin in {obj}")
        return subprocess.run([os.path.join(CUDA, "bin", "nvdisasm"), os.path.join(tmp, cubins[0])], check=True, capture_output=True,
                              text=True).stdout


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--obj", default=os.path.join(CSRC, "heuristic_cu.o"))
    ap.add_argument("--log", default=os.path.join(CSRC, "heuristic.ptxas.log"))
    args = ap.parse_args()
    sass = disassemble(args.obj)
    if "heur_batch_kernel" not in sass:
        raise SystemExit("heur_batch_kernel not found in " + args.obj)
    ops = collections.Counter()
    for line in sass.splitlines():
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", line)
        if m:
            ops[m.group(1)] += 1
    fl = {op: n for op, n in sorted(ops.items()) if op.split(".")[0] in ("FADD", "FMUL", "FFMA", "FMNMX", "FSETP", "FSEL", "FCHK", "FFMA32I")}
    print("float opcodes of heur_batch_kernel:", ", ".join(f"{op} {n}" for op, n in fl.items()))
    ffma = sum(n for op, n in ops.items() if op.startswith("FFMA"))
    with open(args.log) as f:
        log = f.read()
    m = re.search(r"Function properties for \S*heur_batch_kernel\S*\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"
                  r"\s+ptxas info\s+: Used (\d+) registers", log)
    if not m:
        raise SystemExit("heur_batch_kernel not found in " + args.log)
    stack, spill_st, spill_ld, regs = (int(g) for g in m.groups())
    print(f"heur_batch_kernel: {regs} registers, {stack} bytes stack frame, {spill_st} bytes spill stores, {spill_ld} bytes spill loads")
    if ffma:
        print(f"{ffma} FFMA instructions: a multiply and an add are fused (is heuristic.cu built with -fmad=false?)")
        return 1
    if spill_st or spill_ld:
        print("the kernel spills")
        return 1
    print("no FFMA, no spills")
    return 0


if __name__ == "__main__":
    sys.exit(main())
