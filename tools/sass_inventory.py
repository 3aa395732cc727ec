#!/usr/bin/env python
"""Count the IEEE division and square-root sites of a kernel's SASS, per inlined source function.

With -prec-div=true -prec-sqrt=true (tinsel_b200/build.py) every `x / y` and `1 / y` is a MUFU.RCP with a
refinement chain, a division adds an FCHK range check, and every square root is a MUFU.RSQ with its own chain;
each of them has a CALL to a slow path.  Those sites are the fixed-latency poles of a kernel that keeps its scene on
chip.  This counts MUFU.RCP, MUFU.RSQ, FCHK and CALL per SASS function (a kernel, or a __noinline__ function inside
it), and splits each count over the source functions the instructions were inlined from, using the -lineinfo
records the build keeps (`nvdisasm -gi`).

    python tools/sass_inventory.py OBJ [--function SUBSTR ...] [--depth N]

OBJ is an object file or library holding sm_90a code (tinsel_b200/build/default/kernels.cu.o, or the .so), or a
cubin.  --function keeps the SASS functions whose demangled name contains every SUBSTR (default: all); --depth N
shows the N innermost source functions of each inline chain (default 2: function <- its caller)."""
import argparse
import collections
import glob
import os
import re
import shutil
import subprocess
import sys
import tempfile

OPS = ["MUFU.RCP", "MUFU.RSQ", "FCHK", "CALL"]
FILE_RE = re.compile(r'^\s*//## File "([^"]+)", line (\d+)')
LABEL_RE = re.compile(r"^(\$?[A-Za-z_][\w$.]*):\s*$")
INSN_RE = re.compile(r"^\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)")
# a function definition: a line at column 0 that declares a device function, then its name before the first '('
DEF_RE = re.compile(r"^(?:template\s*<.*>\s*)?(?:static\s+)?(?:TB_DEV|TB_HD|TB_NOINLINE|TB_COLD|TB_ORDERED_ATTR|__device__|__global__)\b")
NOT_NAMES = {"__launch_bounds__", "__align__", "alignas", "__noinline__", "__forceinline__"}


def tool(name):
    path = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    if not os.path.exists(path):
        raise SystemExit("%s not found" % name)
    return path


def cubins(obj, tmp):
    if obj.endswith(".cubin"):
        return [obj]
    subprocess.check_call([tool("cuobjdump"), "-xelf", "all", os.path.abspath(obj)], cwd=tmp, stdout=subprocess.DEVNULL)
    found = sorted(glob.glob(os.path.join(tmp, "*.cubin")))
    if not found:
        raise SystemExit("%s holds no cubin" % obj)
    return found


def demangle(names):
    filt = shutil.which("cu++filt") or os.path.join("/usr/local/cuda/bin", "cu++filt")
    out = subprocess.run([filt], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return dict(zip(names, out))


class SourceMap:
    """file:line -> the name of the function whose definition precedes that line"""

    def __init__(self):
        self.defs = {}

    def name(self, path, line):
        if path not in self.defs:
            table = []
            try:
                with open(path, encoding="utf-8", errors="replace") as f:
                    for i, text in enumerate(f, 1):
                        if DEF_RE.match(text):
                            names = [n for n in re.findall(r"(\w+)\s*\(", text) if n not in NOT_NAMES]
                            if names:
                                table.append((i, names[0]))
            except OSError:
                pass
            self.defs[path] = table
        best = None
        for i, n in self.defs[path]:
            if i > line:
                break
            best = n
        return best or "%s:%d" % (os.path.basename(path), line)


def inventory(cubin, src):
    """{sass function: {op: Counter(chain tuple -> count)}}, and the SASS functions' instruction counts"""
    text = subprocess.run([tool("nvdisasm"), "-gi", cubin], capture_output=True, text=True, check=True).stdout
    counts = collections.defaultdict(lambda: {op: collections.Counter() for op in OPS})
    sizes = collections.Counter()
    func = None
    frames, fresh = [], False
    for line in text.split("\n"):
        m = FILE_RE.match(line)
        if m:
            if not fresh:
                frames = []
                fresh = True
            frames.append(src.name(m.group(1), int(m.group(2))))
            continue
        m = LABEL_RE.match(line)
        if m and not m.group(1).startswith(".L"):
            func = m.group(1)
            frames, fresh = [], False
            continue
        m = INSN_RE.match(line)
        if not m or func is None:
            continue
        fresh = False
        sizes[func] += 1
        opcode = m.group(1)
        for op in OPS:
            if opcode == op or opcode.startswith(op + "."):
                counts[func][op][tuple(frames)] += 1
    return counts, sizes


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("obj")
    ap.add_argument("--function", action="append", default=[], help="keep SASS functions whose name contains this")
    ap.add_argument("--depth", type=int, default=2)
    args = ap.parse_args()

    src = SourceMap()
    tmp = tempfile.mkdtemp(prefix="sass_inventory_")
    try:
        counts, sizes = {}, collections.Counter()
        for c in cubins(args.obj, tmp):
            cc, ss = inventory(c, src)
            counts.update(cc)
            sizes.update(ss)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)

    names = demangle(sorted(sizes))
    shown = 0
    for func in sorted(sizes, key=lambda f: names[f]):
        pretty = names[func]
        if not all(s in pretty for s in args.function):
            continue
        shown += 1
        per = counts.get(func, {op: collections.Counter() for op in OPS})
        totals = {op: sum(per[op].values()) for op in OPS}
        print("%s\n  %d instructions; %s" % (pretty, sizes[func], ", ".join("%s %d" % (op, totals[op]) for op in OPS)))
        rows = collections.defaultdict(lambda: [0] * len(OPS))
        for k, op in enumerate(OPS):
            for chain, n in per[op].items():
                rows[" <- ".join(chain[: args.depth]) or "(no line info)"][k] += n
        if rows:
            print("    %-72s %s" % ("source function <- caller", " ".join("%8s" % op for op in OPS)))
            for key in sorted(rows, key=lambda r: (-sum(rows[r][:2]), r)):
                print("    %-72s %s" % (key[:72], " ".join("%8d" % n for n in rows[key])))
        print()
    if not shown:
        raise SystemExit("no SASS function matches %s" % " and ".join(args.function))


if __name__ == "__main__":
    sys.exit(main())
