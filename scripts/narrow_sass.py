"""Instruction count of the tile kernel's narrow steady-state column loop (DESIGN §4.1), from the SASS.

  python scripts/narrow_sass.py [--obj whatshap_b200/csrc/tile.o]

Disassembles tile_panel_kernel (nvdisasm, no GPU needed) and finds the column loop of steady_columns_narrow: the loop whose
body holds the VIADDMNMX.U16x2 instructions, and prints the instructions one trip through it issues -- one column of one
thread, 16 outputs -- with a histogram of opcodes; it fails if a halfword operation is not a native .U16x2 one.
Run `__graft_entry__.build()` first (or pass --obj).
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


def disassemble(obj: str) -> list:
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-xelf", "all", os.path.abspath(obj)], cwd=tmp, check=True,
                       capture_output=True)
        cubins = [f for f in os.listdir(tmp) if f.endswith(".cubin")]
        if not cubins:
            raise SystemExit(f"no cubin in {obj}")
        out = subprocess.run([os.path.join(CUDA, "bin", "nvdisasm"), os.path.join(tmp, cubins[0])], check=True,
                             capture_output=True, text=True).stdout
    ins = []  # (address or None, text): None = label
    for line in out.splitlines():
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if m:
            ins.append((int(m.group(1), 16), m.group(2)))
            continue
        m = re.match(r"^(\.L_x_\d+):", line)
        if m:
            ins.append((None, m.group(1)))
    return ins


def opcode(text: str) -> str:
    t = re.sub(r"^@!?U?P\w+\s+", "", text)
    return t.split()[0]


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--obj", default=os.path.join(ROOT, "whatshap_b200", "csrc", "tile.o"))
    args = ap.parse_args()
    ins = disassemble(args.obj)
    dpx = [i for i, (a, t) in enumerate(ins) if a is not None and "VIADDMNMX.U16x2" in t]
    if not dpx:
        raise SystemExit("no VIADDMNMX.U16x2 in the kernel: the narrow column is missing")
    first, last = dpx[0], dpx[-1]
    label_at = {t: i for i, (a, t) in enumerate(ins) if a is None}
    # the loop: the innermost backward branch after the DPX block whose target lies before it
    loop = None
    for i in range(last, len(ins)):
        a, t = ins[i]
        m = re.search(r"BRA\s+`?\(?(\.L_x_\d+)", t) if a is not None else None
        if m and label_at.get(m.group(1), len(ins)) < first and (loop is None or label_at[m.group(1)] > loop[0]):
            loop = (label_at[m.group(1)], i)
    if loop is None:
        raise SystemExit("column loop not found")
    lo, hi = loop
    path = [i for i in range(lo, hi + 1) if ins[i][0] is not None]
    # (the barrier's try-wait and its branch back issue once when the barrier is complete: each counted once)
    hist = collections.Counter(opcode(ins[i][1]) for i in path)
    print(f"narrow column loop: {len(path)} instructions per column and thread (16 outputs)")
    for op, n in hist.most_common():
        print(f"  {op:24s} {n}")
    emulated = [ins[i][1] for i in path if "U16" in ins[i][1] and "U16x2" not in ins[i][1]]
    if emulated:
        print("non-native halfword operations:", emulated)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
