#!/usr/bin/env python
"""Where the cycles of the lane-owned wavefront kernel go, per stage.  Cornell runs its instantiation without the
scene features (wf2_lq::k_wavefront2<512, generic, TB_FEAT_NONE>; TINSEL_B200_SPECIALIZE=0: the generic one), and
the clock accounting is compiled into both; the table's first line names the kernel that ran.

Builds the development variant with the kernel's own clock64() accounting (-DTB_WF2_STAGE_CLOCKS, off in the
product build) as tinsel_b200/libtinsel_b200_clocks.so, renders cornell in the benchmark's shape with it
(1024x1024, 32 spp per render_device call, TINSEL_B200_LIB pointing at the variant) and prints per stage:
SM cycles per camera sample, visits (warp chunks) per sample and the mean number of lanes active per chunk.
Stage R is also split into its parts: the splat of the finished sample, the claim of new sample indices (from
the vote to the index) and the regeneration (the camera rays).  So is stage A: the hit prologue, the light samples,
the shadow traces, the connections and the BSDF sample.  A's lanes leave the NEE loop at different times, so each
of its parts counts, per chunk, the longest any lane spent in it; the parts can add up to a little more than the
stage where lanes run different parts side by side.

    python tools/stage_clocks.py [--steps N] [--lib PATH | --no-build]

"SM cycles per sample" is warp cycles / warps per CTA / samples: the share of an SM's time a stage takes,
per sample, so that the rows add up to the kernel's SM cycles per sample (one CTA per SM).  claim counts the
claims that got slots, idle the empty claims and their back-off.  The clock reads themselves cost a little:
compare two builds with this tool, and absolute speed with bench.py."""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANT = "libtinsel_b200_clocks.so"
WORDS = 23                     # tb_kernels.cuh: TB_WF2_STAGE_CLOCK_WORDS
WARPS_PER_CTA = 512 // 32
STAGES = ["R", "T", "A", "B"]  # counter order (wf2_lanes.cuh: Wf2Clocks)
R_PARTS = ["splat", "claim", "regenerate"]   # wf2_common.cuh: WF2_R_*
A_PARTS = ["hit", "light", "shadow", "connect", "scatter"]   # wf2_lanes.cuh: WF2_A_*
PARTS = {"R": (15, R_PARTS), "A": (18, A_PARTS)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--spp", type=int, default=32)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--lib", help="an already built clock variant (default: build tinsel_b200/%s)" % VARIANT)
    ap.add_argument("--no-build", action="store_true", help="use tinsel_b200/%s as it is" % VARIANT)
    args = ap.parse_args()

    lib = args.lib or os.path.join(ROOT, "tinsel_b200", VARIANT)
    if not args.lib and not args.no_build:
        subprocess.check_call([sys.executable, "-m", "tinsel_b200.build", "--out", VARIANT, "-DTB_WF2_STAGE_CLOCKS"], cwd=ROOT)
    os.environ["TINSEL_B200_LIB"] = os.path.abspath(lib)
    os.environ.pop("TINSEL_B200_PIPELINE", None)
    sys.path.insert(0, ROOT)
    import tinsel_b200 as tb

    native = tb.load_library()
    if not hasattr(native, "tb200_stage_clocks"):
        raise SystemExit("%s was not built with -DTB_WF2_STAGE_CLOCKS" % lib)
    native.tb200_stage_clocks.restype = C.c_int
    native.tb200_stage_clocks.argtypes = [C.POINTER(C.c_ulonglong), C.c_int, C.c_int]
    counters = (C.c_ulonglong * WORDS)()

    def read(reset):
        if native.tb200_stage_clocks(counters, WORDS, 1 if reset else 0) != WORDS:
            raise SystemExit("tb200_stage_clocks failed")
        return list(counters)

    w = h = args.size
    snap = tb.Snapshot(tb.scene_path("cornell"))
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = w, h
    r = tb.Renderer(snap.scene)
    r.Init(w, h)
    for _ in range(args.warmup):
        r.render_device(cam, opt, args.spp)
    read(True)
    gpu_ms = 0.0
    for _ in range(args.steps):
        r.render_device(cam, opt, args.spp)
        gpu_ms += r.stats().gpuMs
    c = read(True)
    kernel = r.last_kernel()
    r.close()
    snap.close()

    samples = w * h * args.spp * args.steps
    per = float(WARPS_PER_CTA) * samples
    claim, idle = c[0], c[1]
    cyc, chunks, lanes = c[2:6], c[6:10], c[10:14]
    total = claim + idle + sum(cyc)
    print("cornell %dx%d, %d spp x %d steps, %s: %.1f Msamples/s with the clock reads, %d warps" % (
        w, h, args.spp, args.steps, kernel, samples / gpu_ms / 1e3, c[14]))
    print("%-10s %14s %8s %16s %12s" % ("stage", "SM cyc/sample", "share", "visits/sample", "mean lanes"))
    print("%-10s %14.1f %7.1f%%" % ("claim", claim / per, 100.0 * claim / total))
    print("%-10s %14.1f %7.1f%%" % ("idle", idle / per, 100.0 * idle / total))
    for k, name in enumerate(STAGES):
        if chunks[k] == 0:
            continue
        print("%-10s %14.1f %7.1f%% %16.3f %12.2f" % (name, cyc[k] / per, 100.0 * cyc[k] / total, lanes[k] / samples,
                                                     lanes[k] / chunks[k]))
        if name in PARTS:
            # the stage's parts; what is left is the bookkeeping between them (flags, the claim loop's vote, the
            # slot state's loads and stores)
            first, parts = PARTS[name]
            for p, part in enumerate(parts):
                print("%-10s %14.1f %7.1f%%" % ("  " + part, c[first + p] / per, 100.0 * c[first + p] / total))
    print("%-10s %14.1f" % ("total", total / per))


if __name__ == "__main__":
    main()
