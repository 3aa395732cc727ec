#!/usr/bin/env python
"""Static code size of one kernel instantiation by source function (SASS instructions, 16 B each):
where the bytes are that compete for the 32 KB L1.5 instruction cache.
    python tools/code_size.py [mangled-substring, default _ZN6wf2_lq12k_wavefront2ILi512ELi0ELj0E, the lane-owned kernel cornell runs]

With --local: the local-memory instructions (LDL / STL) of one kernel instantiation, out-of-line callees
included, by source function and line.  Needs no GPU.
    python tools/code_size.py --local [mangled-substring, default _ZN6wf2_lq12k_wavefront2ILi512ELi0ELj0E]"""
import re
import sys
from collections import Counter

import ncu_lines


def func_name(funcs, key):
    if key:
        t = funcs.get(key[0])
        if t and key[1] - 1 < len(t):
            return t[key[1] - 1]
    return None


def code_size(kernel):
    table = ncu_lines.line_table(kernel)
    funcs = ncu_lines.function_of_line()
    by_func = Counter()
    for addr, key in table.items():
        by_func[(key[0] if key else None, func_name(funcs, key))] += 1
    total = sum(by_func.values())
    print("%s: %d instructions = %.1f KB" % (kernel, total, total * 16 / 1024.0))
    for (f, n), c in by_func.most_common(45):
        print("  %-18s %-28s %5d  %5.1f KB" % (f, n, c, c * 16 / 1024.0))


def local_accesses(kernel):
    listing = ncu_lines.sass_listing(kernel)
    sections = sorted(set(sec for sec, _, _, _ in listing))
    if len(sections) != 1:
        sys.exit("%r matches %d kernels%s: pass a longer substring of the mangled name" %
                 (kernel, len(sections), "".join("\n  " + s for s in sections)))
    funcs = ncu_lines.function_of_line()
    by_line = {}
    by_func = Counter()
    for _, _, key, ins in listing:
        m = re.match(r"(?:@!?U?P\w+\s+)?(LDL|STL)\b", ins)
        if not m:
            continue
        fn = func_name(funcs, key)
        row = by_line.setdefault((key, fn), Counter())
        row[m.group(1)] += 1
        by_func[(key[0] if key else None, fn, m.group(1))] += 1
    n_ld = sum(c for (_, _, op), c in by_func.items() if op == "LDL")
    n_st = sum(c for (_, _, op), c in by_func.items() if op == "STL")
    print("%s: %d LDL, %d STL of %d instructions" % (sections[0], n_ld, n_st, len(listing)))
    print("\nby function:                                    LDL   STL")
    names = sorted(set((f, n) for f, n, _ in by_func), key=lambda k: (str(k[0]), str(k[1])))
    for f, n in names:
        print("  %-18s %-28s %5d %5d" % (f, n, by_func[(f, n, "LDL")], by_func[(f, n, "STL")]))
    print("\nby line:                                        LDL   STL")
    for (key, fn), c in sorted(by_line.items(), key=lambda kv: (kv[0][0] or ("", 0), str(kv[0][1]))):
        print("  %-34s %-12s %5d %5d" % ("%s:%d" % key if key else "?", fn, c["LDL"], c["STL"]))


if __name__ == "__main__":
    args = sys.argv[1:]
    if "--local" in args:
        args.remove("--local")
        local_accesses(args[0] if args else "_ZN6wf2_lq12k_wavefront2ILi512ELi0ELj0E")
    else:
        code_size(args[0] if args else "_ZN6wf2_lq12k_wavefront2ILi512ELi0ELj0E")
