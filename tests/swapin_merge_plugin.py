"""pytest plugin used by test_merge.py: before the reference's test modules are imported, replace `whatshap.merge.ReadMerger` by
this repository's swap-in (adapters.make_read_merger), whose device work the host emulation tests/emul/emul_merge.cpp stands in
for (the CUDA path itself is held to the same answers by the GPU tests)."""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ["WHMEC_PYREF"])

import whatshap.merge  # noqa: E402

from whatshap_b200 import _lib, adapters  # noqa: E402

EMUL_DIR = os.path.join(ROOT, "tests", "emul")
subprocess.run(["make", "-C", EMUL_DIR, "-f", "merge.mk"], check=True, capture_output=True)
_emul = _lib.merge_reads_signatures(C.CDLL(os.path.join(EMUL_DIR, "libwhemul_merge.so")))
_SwapIn = adapters.make_read_merger(whatshap.merge)


class ReadMerger(_SwapIn):
    def __init__(self, *args, **kw):
        kw.setdefault("library", _emul)
        super().__init__(*args, **kw)


whatshap.merge.ReadMerger = ReadMerger
