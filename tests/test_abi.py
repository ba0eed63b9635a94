"""The C-ABI shared library loads on a GPU-less machine and exports every symbol that
include/whmec.h declares; host-detectable errors are reported without touching CUDA."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from whatshap_b200 import _lib, synth
from whatshap_b200._abi import CProblem, CStats, MendelianConflict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "whmec.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(whmec_[a-z_]+)\s*\(", text)))


def test_header_and_loader_agree():
    assert declared_symbols() == sorted(_lib.EXPORTS)


def test_library_exports_every_declared_symbol():
    lib = _lib.lib()
    for name in declared_symbols():
        assert hasattr(lib, name), name
    assert lib.whmec_abi_version() == 2
    assert b"sm_90a" in lib.whmec_build_info()


def test_struct_layout_matches_header(tmp_path):
    """sizeof/offsetof as laid out by the C compiler for include/whmec.h == the ctypes mirror."""
    import subprocess

    from whatshap_b200._abi import CHeuristicSolution, CSolution

    src = tmp_path / "layout.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "whmec.h"\n'
        "int main(void){printf(\"%zu %zu %zu %zu %zu %zu %zu %zu\\n\", sizeof(whmec_problem), sizeof(whmec_solution),"
        " sizeof(whmec_stats), offsetof(whmec_problem, gl), offsetof(whmec_stats, sweep_ms), offsetof(whmec_solution, sr_quality),"
        " sizeof(whmec_heuristic_solution), offsetof(whmec_heuristic_solution, mutated));return 0;}\n"
    )
    exe = tmp_path / "layout"
    subprocess.run(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [C.sizeof(CProblem), C.sizeof(CSolution), C.sizeof(CStats), CProblem.gl.offset, CStats.sweep_ms.offset, CSolution.sr_quality.offset,
            C.sizeof(CHeuristicSolution), CHeuristicSolution.mutated.offset]
    assert got == want


def test_host_side_errors_need_no_gpu():
    """Mendelian conflicts and malformed input are detected by the host packer."""
    prob = synth.sliding_window(12, 3, block_len=12, seed=1)
    prob.gt[0, 5] = 255  # no diploid biallelic genotype: no assignment is compatible (trusted genotypes)
    with pytest.raises(MendelianConflict, match="Error: Mendelian conflict"):
        _lib.solve(prob)
    prob = synth.sliding_window(12, 3, block_len=12, seed=1)
    prob.ent_col[1], prob.ent_col[0] = prob.ent_col[0], prob.ent_col[1]
    with pytest.raises(RuntimeError, match="unsorted variants"):
        _lib.solve(prob)


def test_empty_problem_needs_no_gpu():
    sol, stats = _lib.solve(synth.sliding_window(0, 4))
    assert sol.cost == 0 and stats["cells"] == 0


def test_sort_key_is_libstdcxx_hash():
    # std::hash<int> is the identity, so the source id only flips low bits of the name hash
    k0 = _lib.read_sort_key("Read 1", 0)
    assert _lib.read_sort_key("Read 1", 5) == k0 ^ 5
    assert _lib.read_sort_key("Read 2", 0) != k0
