"""TEST INFRASTRUCTURE (only where a WhatsHap source tree is at $WHATSHAP_REF): builds the reference's own Python
extension `whatshap.core` in a scratch directory OUTSIDE this repository so that tests can drive the real Cython
classes.  Nothing is copied into the repo; where the reference is absent, its answers stored under tests/golden/ stand in.

Recipe (SURVEY.md Appendix B): copy src/ whatshap/ setup.py, stub _version.py, skip the polyphase solver
import (needs `pulp`), build_ext --inplace with the distribution compiler (/usr/bin/g++; /opt/gcc links
libstdc++ statically and the module crashes).  Result here: OK, about 45 s, 5 extensions.
"""
import os
import shutil
import subprocess
import sys

REF = os.environ.get("WHATSHAP_REF", "/root/reference")
OUT = os.environ.get("WHMEC_PYREF_DIR", "/tmp/whmec_pyref")


def build() -> str:
    """Returns the directory to put on sys.path, or '' when the reference tree is not available."""
    marker = os.path.join(OUT, "whatshap", ".built")
    if os.path.exists(marker):
        return OUT
    if not os.path.isdir(os.path.join(REF, "src")):
        return ""
    shutil.rmtree(OUT, ignore_errors=True)
    os.makedirs(OUT)
    for item in ("src", "whatshap", "setup.py"):
        src = os.path.join(REF, item)
        dst = os.path.join(OUT, item)
        shutil.copytree(src, dst) if os.path.isdir(src) else shutil.copy(src, dst)
    for root, dirs, files in os.walk(OUT):
        for name in dirs + files:
            os.chmod(os.path.join(root, name), 0o755)
    with open(os.path.join(OUT, "whatshap", "_version.py"), "w") as f:
        f.write('version = "0+oracle"\n')
    init = os.path.join(OUT, "whatshap", "__init__.py")
    text = open(init).read().replace("    import whatshap.polyphase.solver  # noqa", "    pass")
    open(init, "w").write(text)
    env = dict(os.environ, CC="/usr/bin/gcc", CXX="/usr/bin/g++", CFLAGS="-O2", CXXFLAGS="-O2")
    subprocess.run([sys.executable, "setup.py", "build_ext", "--inplace", "-j", "8"], cwd=OUT, env=env, check=True,
                   capture_output=True)
    open(marker, "w").write("ok\n")
    return OUT


if __name__ == "__main__":
    print(build() or "reference tree not found")


SHIP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "pyref")


def ship() -> str:
    """Puts the COMPILED reference binding next to oracle/_ref/libwhref.so (oracle/_ref is git-ignored):
    oracle/_ref/pyref/whatshap/core.*.so plus two stub modules
    of our own (`__init__`, `variant` — core.pyx imports `.variant.Variant`, a three-field dataclass).  No reference
    source is copied.  Returns the directory to put on sys.path ('' when neither a build nor a prebuilt copy exists)."""
    pkg = os.path.join(SHIP, "whatshap")
    have = os.path.isdir(pkg) and any(f.startswith("core.") and f.endswith(".so") for f in os.listdir(pkg))
    built = build()
    if built:
        os.makedirs(pkg, exist_ok=True)
        for f in os.listdir(os.path.join(built, "whatshap")):
            if f.startswith("core.") and f.endswith(".so"):
                src, dst = os.path.join(built, "whatshap", f), os.path.join(pkg, f)
                if not os.path.exists(dst) or os.path.getmtime(dst) < os.path.getmtime(src):
                    shutil.copy(src, dst)
                have = True
    if have:
        with open(os.path.join(pkg, "__init__.py"), "w") as f:
            f.write('"""Stub package (test infrastructure): only the compiled reference binding whatshap.core lives here."""\n')
        with open(os.path.join(pkg, "variant.py"), "w") as f:
            f.write('"""Stub: the dataclass whatshap.core imports as `.variant.Variant` (same three fields)."""\n'
                    "from whatshap_b200.variant import Variant  # noqa: F401\n")
        return SHIP
    return ""


def shipped_core():
    """The compiled reference binding `whatshap.core` (built here or a prebuilt copy under oracle/_ref), or None."""
    if "whatshap.core" in sys.modules:  # already imported (e.g. from the full out-of-tree build): the same binding
        return sys.modules["whatshap.core"]
    path = ship()
    if not path:
        return None
    import importlib

    if path not in sys.path:
        sys.path.insert(0, path)
    return importlib.import_module("whatshap.core")
