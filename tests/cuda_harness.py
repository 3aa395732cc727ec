"""Compiles a test harness (a .cu file under tests/ that includes the library's headers and exports C functions) with
the library's own nvcc flags (tinsel_b200.build) into a temporary directory keyed by its sources and flags: the
repository tree may be read-only.  TEST INFRASTRUCTURE."""
import hashlib
import os
import subprocess
import tempfile

from tinsel_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tinsel_b200", "csrc")
HEADERS = [os.path.join(CSRC, h) for h in build.HEADERS] + [os.path.join(ROOT, "include", h) for h in ("tinsel_b200.h", "tb200_detmath.h")]


def _compile_cmd(src, out):
    return [build._nvcc(), "-ccbin", build._host_compiler(), *build.NVCC_FLAGS, "-I", os.path.join(ROOT, "include"),
            "-I", CSRC, "-shared", "-o", out, src, "-lcudart"]


def harness_path(name):
    """tests/<name>.cu compiled into a shared library, on first use; returns its path."""
    src = os.path.join(ROOT, "tests", name + ".cu")
    h = hashlib.sha1(" ".join(_compile_cmd(src, "")).encode())
    for p in [src] + HEADERS:
        with open(p, "rb") as f:
            h.update(f.read())
    path = os.path.join(tempfile.gettempdir(), "tinsel_b200_%s_%s.so" % (name, h.hexdigest()[:16]))
    if not os.path.exists(path):
        tmp = "%s.%d.tmp" % (path, os.getpid())
        subprocess.check_call(_compile_cmd(src, tmp))
        os.replace(tmp, path)
    return path
