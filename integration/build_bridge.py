"""Builds integration/whatshap_bridge.pyx against a WhatsHap source tree, out of this repository's tree.
    python integration/build_bridge.py [whatshap source dir] [output dir]
Defaults: the scratch copy that oracle/build_pyref.py makes of the WhatsHap tree at $WHATSHAP_REF and its
own directory, so that `import whatshap_bridge` works wherever `import whatshap` does.  Nothing is copied from
WhatsHap: its .pxd files and C++ headers are only on the include paths."""
import os
import shutil
import subprocess
import sys
import sysconfig
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))


def build(whatshap_tree: str, out_dir: str) -> str:
    """Returns the path of the built extension module."""
    import numpy

    suffix = sysconfig.get_config_var("EXT_SUFFIX")
    target = os.path.join(out_dir, "whatshap_bridge" + suffix)
    source = os.path.join(HERE, "whatshap_bridge.pyx")
    if os.path.exists(target) and os.path.getmtime(target) >= os.path.getmtime(source):
        return target
    work = tempfile.mkdtemp(prefix="whmec_bridge_")
    try:
        cpp = os.path.join(work, "whatshap_bridge.cpp")
        subprocess.run([sys.executable, "-m", "cython", "--cplus", "-3", "-I", whatshap_tree, source, "-o", cpp], check=True)
        includes = [sysconfig.get_paths()["include"], numpy.get_include(), os.path.join(whatshap_tree, "src")]
        cmd = ["/usr/bin/g++", "-O2", "-std=c++11", "-fPIC", "-shared", "-w"] + ["-I" + i for i in includes] + [cpp, "-o", target]
        subprocess.run(cmd, check=True)
    finally:
        shutil.rmtree(work, ignore_errors=True)
    return target


if __name__ == "__main__":
    tree = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("WHMEC_PYREF_DIR", "/tmp/whmec_pyref")
    out = sys.argv[2] if len(sys.argv) > 2 else tree
    print(build(tree, out))
