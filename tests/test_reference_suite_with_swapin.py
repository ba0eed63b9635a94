"""The reference's OWN unit tests for this path (tests/test_phasing.py, tests/test_pedigreephasing.py,
tests/test_verification.py — SURVEY.md §4) run unmodified from the WhatsHap tree at $WHATSHAP_REF with
`whatshap.core.PedigreeDPTable` replaced by this repository's swap-in class operating on the real
Cython ReadSet / Pedigree objects, and with the host steps around the DP (read selection, its priority queue,
recombination events) replaced too: tests/test_readselect.py, tests/test_priorityqueue.py, tests/test_pedigree.py; and the
reference's genotyping tests (tests/test_genotyping.py, tests/test_pedigreegenotyping.py) with `GenotypeDPTable` replaced.
These tests run the reference's own test files, which this repository must not copy: they run only where the WhatsHap
source tree is present and skip elsewhere.  The reference's answers that the other tests compare with are stored under
tests/golden/ and checked everywhere."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from oracle.build_pyref import REF  # noqa: E402


def test_reference_tests_pass_with_swapped_dp_table():
    from oracle import build_pyref

    pyref = build_pyref.build()
    if not pyref:
        pytest.skip("reference tree not available")
    env = dict(os.environ, WHMEC_PYREF=pyref, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "tests"), pyref, ROOT]))
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-p", "swapin_plugin",
           "tests/test_phasing.py", "tests/test_pedigreephasing.py", "tests/test_verification.py",
           "tests/test_readselect.py", "tests/test_priorityqueue.py", "tests/test_pedigree.py",
           "tests/test_genotyping.py", "tests/test_pedigreegenotyping.py"]
    res = subprocess.run(cmd, cwd=REF, env=env, capture_output=True, text=True, timeout=900)
    tail = (res.stdout + res.stderr)[-2000:]
    assert res.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail, tail
    # make sure the swap really happened: the plugin module must have been imported by that run
    assert "swapin_plugin" not in res.stderr or "No module" not in res.stderr


def test_reference_tests_pass_on_this_packages_containers():
    """Second run: every class of the path in `whatshap.core` replaced by this package's Python mirror
    (tests/swapin_all_plugin.py), so the reference's data-model tests (tests/test_reads.py, tests/test_pedigree.py,
    tests/test_graph.py), its read-selection / priority-queue tests, the three phasing-DP test files and the two genotyping-DP
    test files (tests/test_genotyping.py, tests/test_pedigreegenotyping.py; `GenotypeDPTable` backed by the emulated kernels) exercise THIS
    package's containers and host steps unmodified.  HapCHAT-parametrised cases are another algorithm (deselected)."""
    from oracle import build_pyref

    pyref = build_pyref.build()
    if not pyref:
        pytest.skip("reference tree not available")
    env = dict(os.environ, WHMEC_PYREF=pyref, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "tests"), pyref, ROOT]))
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-p", "swapin_all_plugin", "-k", "not hapchat",
           "tests/test_reads.py", "tests/test_pedigree.py", "tests/test_geneticmap.py", "tests/test_graph.py", "tests/test_readselect.py", "tests/test_priorityqueue.py",
           "tests/test_phasing.py", "tests/test_pedigreephasing.py", "tests/test_verification.py",
           "tests/test_genotyping.py", "tests/test_pedigreegenotyping.py"]
    res = subprocess.run(cmd, cwd=REF, env=env, capture_output=True, text=True, timeout=900)
    tail = (res.stdout + res.stderr)[-2000:]
    assert res.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail, tail
