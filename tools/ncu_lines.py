#!/usr/bin/env python
"""Attribute an ncu source-page capture (SASS level) to source functions and lines.

    python tools/ncu_lines.py prof.ncu-rep [kernel-mangled-substring]

Joins `ncu --page source --csv` (per-SASS-instruction executed counts and stall samples) with
`nvdisasm -g` line info of the in-tree library, then aggregates by innermost source line and by
the function that line belongs to.  Needs the library built with -lineinfo (it is).
"""
import csv
import io
import os
import re
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.environ.get("TINSEL_B200_LIB") or os.path.join(ROOT, "tinsel_b200", "libtinsel_b200.so")


def sass_listing(kernel):
    """[(section, address, (file, line) or None, instruction)] of the kernels whose section names contain `kernel`.
    A kernel's out-of-line callees are copied into its section, so they are part of the listing."""
    tmp = tempfile.mkdtemp()
    subprocess.check_call(["cuobjdump", "-xelf", "all", LIB], cwd=tmp, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    listing = []
    for f in os.listdir(tmp):
        if not f.startswith("kernels"):
            continue
        out = subprocess.check_output(["nvdisasm", "-g", "-c", os.path.join(tmp, f)], text=True, stderr=subprocess.DEVNULL)
        cur = None
        inside = False
        section = None
        for ln in out.splitlines():
            if ln.startswith(".text."):
                inside = kernel in ln
                section = ln[len(".text."):].rstrip(":")
                cur = None
                continue
            if not inside:
                continue
            m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
            if m:
                cur = (os.path.basename(m.group(1)), int(m.group(2)))
                continue
            m = re.match(r"\s+/\*([0-9a-f]{4,6})\*/\s*(.*?)\s*;?\s*$", ln)
            if m:
                listing.append((section, int(m.group(1), 16), cur, m.group(2)))
    return listing


def line_table(kernel):
    return {addr: key for _, addr, key, _ in sass_listing(kernel)}


def function_of_line():
    """(file, line) -> enclosing function name, from a light parse of the sources."""
    funcs = {}
    srcs = [os.path.join(ROOT, "tinsel_b200", "csrc", f) for f in os.listdir(os.path.join(ROOT, "tinsel_b200", "csrc"))]
    srcs.append(os.path.join(ROOT, "include", "tb200_detmath.h"))
    for path in srcs:
        if not path.endswith((".cuh", ".cu", ".h")):
            continue
        name = os.path.basename(path)
        cur = None
        table = []
        for i, ln in enumerate(open(path, errors="ignore"), 1):
            m = re.match(r"^(?:TB_DEV|TB_HD|TBM_HD|__global__|static|inline|void|template)?.*?\b([A-Za-z_][A-Za-z0-9_]*)\s*\([^;]*$", ln)
            if m and not ln.startswith((" ", "\t", "//", "#", "}")) and "(" in ln:
                cur = m.group(1)
            table.append(cur)
        funcs[name] = table
    return funcs


def mangled_fragment(rep, kernel):
    """The mangled name of the profiled kernel (`_ZN6wf2_lq12k_wavefront2ILi512ELi0EEEv12LaunchParamsy`), so that
    the line table of exactly that instantiation is used: the library holds the same template in several
    namespaces (the layouts of wf2_common.cuh) and with several arguments."""
    raw = subprocess.check_output(["ncu", "-i", rep, "--page", "raw", "--csv", "--print-kernel-base", "mangled"], text=True, stderr=subprocess.DEVNULL)
    rows = list(csv.reader(io.StringIO(raw)))
    name = rows[2][rows[0].index("Kernel Name")]
    return name if kernel in name else kernel


def main():
    rep = sys.argv[1]
    kernel = sys.argv[2] if len(sys.argv) > 2 else "k_wavefront"
    kernel = mangled_fragment(rep, kernel)
    raw = subprocess.check_output(["ncu", "-i", rep, "--page", "source", "--csv"], text=True, stderr=subprocess.DEVNULL)
    rows = list(csv.reader(io.StringIO(raw)))
    # first row: kernel name, second: header
    hdr_idx = next(i for i, r in enumerate(rows) if r and r[0] == "Address")
    hdr = rows[hdr_idx]
    col = {h: i for i, h in enumerate(hdr)}
    table = line_table(kernel)
    funcs = function_of_line()
    base = None
    by_line = defaultdict(lambda: [0, 0, 0])
    by_func = defaultdict(lambda: [0, 0, 0])
    stall_cols = [h for h in hdr if h.startswith("stall_") and "Not Issued" not in h]
    stalls = defaultdict(int)
    stall_by_func = defaultdict(lambda: defaultdict(int))
    tot = [0, 0, 0]
    for r in rows[hdr_idx + 1:]:
        if len(r) < len(hdr):
            continue
        addr = int(r[col["Address"]], 16)
        if base is None:
            base = addr
        key = table.get(addr - base)
        inst = int(r[col["Instructions Executed"]] or 0)
        thr = int(r[col["Thread Instructions Executed"]] or 0)
        smp = int(r[col["# Samples"]] or 0)
        fname = None
        if key:
            t = funcs.get(key[0])
            if t and key[1] - 1 < len(t):
                fname = t[key[1] - 1]
        for agg, k in ((by_line, key), (by_func, (key[0] if key else None, fname))):
            agg[k][0] += inst
            agg[k][1] += thr
            agg[k][2] += smp
        tot[0] += inst
        tot[1] += thr
        tot[2] += smp
        for s in stall_cols:
            v = int(r[col[s]] or 0)
            stalls[s] += v
            stall_by_func[(key[0] if key else None, fname)][s] += v
    print("total warp-inst %d, thread-inst %d (%.1f/32 lanes), samples %d" % (tot[0], tot[1], tot[1] / max(1, tot[0]), tot[2]))
    print("\nstall reasons (all samples):")
    for s, v in sorted(stalls.items(), key=lambda x: -x[1])[:10]:
        print("  %-28s %6.2f %%" % (s, 100.0 * v / max(1, tot[2])))
    print("\nby function: %inst  lanes  %samples")
    for k, v in sorted(by_func.items(), key=lambda x: -x[1][2])[:28]:
        top = sorted(stall_by_func[k].items(), key=lambda x: -x[1])[:3]
        print("  %-18s %-26s %5.1f %5.1f %5.1f   %s" % (k[0], k[1], 100.0 * v[0] / tot[0], v[1] / max(1, v[0]), 100.0 * v[2] / max(1, tot[2]),
                                                   " ".join("%s:%d%%" % (a.replace("stall_", ""), 100 * b // max(1, v[2])) for a, b in top)))
    print("\nby line: %inst lanes %samples")
    for k, v in sorted(by_line.items(), key=lambda x: -x[1][2])[:30]:
        print("  %-34s %5.1f %5.1f %5.1f" % ("%s:%s" % k if k else "?", 100.0 * v[0] / tot[0], v[1] / max(1, v[0]), 100.0 * v[2] / max(1, tot[2])))
    only = os.environ.get("NCU_LINES_FILE")   # e.g. wf2_lanes.cuh: every line of that file, in line order
    if only:
        print("\nevery line of %s: %%inst lanes %%samples" % only)
        for k, v in sorted((kv for kv in by_line.items() if kv[0] and kv[0][0] == only), key=lambda x: x[0][1]):
            print("  %-34s %5.2f %5.1f %5.2f" % ("%s:%s" % k, 100.0 * v[0] / tot[0], v[1] / max(1, v[0]), 100.0 * v[2] / max(1, tot[2])))


if __name__ == "__main__":
    main()
