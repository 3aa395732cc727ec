#!/usr/bin/env python
"""What a new sky costs a live renderer, one JSON line per scene:
    python tools/sky_bench.py [--scenes env_like,envmini] [--reps 10] [--table-reps 50]

env_like is bigscene's stand-in for env (a 4000 x 2000 probe, a glass torus of 12 288 triangles), written to a
temporary directory; envmini is the checked-in snapshot (a 128 x 64 probe).  Per scene:
  (a) what a caller pays without tb200_set_sky: tb200_create of the whole scene with the probe's tables (create_ms),
      after building those tables on the host.  The host build is timed on bigscene.build_cdf, the numpy float32
      restatement of Probe::BuildCDF (host_build_cdf_numpy_ms), not on the C++ loop a tinsel host runs, so
      today_ms = the two together is an estimate of that path; create_ms alone is measured as it is.  Each is the
      median of --reps runs;
  (b) set_sky_host_ms: Renderer.set_sky from a numpy probe (upload, table build, swap), median wall time;
  (c) set_sky_device_ms: Renderer.set_sky from a CUDA tensor on the renderer's device, median wall time;
  (d) tables_ms: tb200_probe_tables alone, the mean of --table-reps calls' stats.gpuMs (CUDA events around the three
      kernels) after --warmup calls.  Its bytes are those the build must move at least: 16 read and 8 written per
      texel, and 4 read and 8 written per row (the row total and pdfY, cdfY); tables_gbps is those bytes over
      tables_ms, and hbm_share that rate over the H100 SXM's 3.35 TB/s.  The kernels also re-read and re-write pdfX
      and cdfX once to scale them (8 + 8 bytes per texel, mostly from L2), which the floor leaves out.
The device's tables are checked bit for bit against bigscene.build_cdf in the same run.  The GPU's name, power limit and
maximum SM clock are read in the same run.  Needs a GPU."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import tinsel_b200 as tb  # noqa: E402
from tinsel_b200 import abi  # noqa: E402
import bigscene  # noqa: E402
import ray_query_bench as rqb  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _exact(got, want):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    return bool(((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))).all())


def _median_ms(fn, reps):
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times)


def bench(name, path, args, torch):
    snap = tb.Snapshot(path)
    k = snap.scene.contents.sky
    W, H = k.probeWidth, k.probeHeight
    probe = np.ctypeslib.as_array(k.probeData, (W * H * 4,)).reshape(H, W, 4).copy()
    horizon, zenith = list(k.horizon), list(k.zenith)
    line = {"scene": name, "probe": [W, H], "tris": sum(snap.scene.contents.meshes[m].numIndices // 3
                                                         for m in range(snap.scene.contents.numMeshes))}

    # (a) the tables on the host (the numpy restatement), then tb200_create with them
    tables = []
    line["host_build_cdf_numpy_ms"] = _median_ms(lambda: tables.append(bigscene.build_cdf(probe)), args.reps)
    sc = abi.copy_struct(snap.scene.contents)
    keep = [np.ascontiguousarray(t, np.float32) for t in tables[-1]]
    for f, a in zip(("pdfValuesX", "cdfValuesX", "pdfValuesY", "cdfValuesY"), keep):
        setattr(sc.sky, f, a.ctypes.data_as(abi.c_float_p))

    def create():
        tb.Renderer(C.pointer(sc)).close()
    create()
    line["create_ms"] = _median_ms(create, args.reps)
    line["today_ms"] = line["host_build_cdf_numpy_ms"] + line["create_ms"]

    # (b), (c) set_sky from host pixels and from a CUDA tensor
    r = tb.Renderer(C.pointer(sc))
    dev = torch.from_numpy(probe).cuda()
    for _ in range(args.warmup):
        r.set_sky(horizon, zenith, probe)
        r.set_sky(horizon, zenith, dev)
    line["set_sky_host_ms"] = _median_ms(lambda: r.set_sky(horizon, zenith, probe), args.reps)
    line["set_sky_device_ms"] = _median_ms(lambda: r.set_sky(horizon, zenith, dev), args.reps)
    line["set_sky_build_gpu_ms"] = r.stats().gpuMs

    # (d) the table build alone
    out = [torch.empty((H, W), device="cuda"), torch.empty((H, W), device="cuda"), torch.empty(H, device="cuda"),
           torch.empty(H, device="cuda")]
    for _ in range(args.warmup):
        r.probe_tables(dev, *out)
    gpu_ms = []
    for _ in range(args.table_reps):
        r.probe_tables(dev, *out)
        gpu_ms.append(r.stats().gpuMs)
    tables_ms = sum(gpu_ms) / len(gpu_ms)
    nbytes = 24 * W * H + 12 * H
    line.update(tables_ms=tables_ms, tables_ms_min=min(gpu_ms), tables_ms_max=max(gpu_ms), tables_bytes=nbytes,
                tables_gbps=nbytes / (tables_ms * 1e-3) / 1e9, hbm_share=nbytes / (tables_ms * 1e-3) / HBM_BYTES_PER_S)
    want = bigscene.build_cdf(probe)
    line["bit_exact"] = all(_exact(o.cpu().numpy(), w) for o, w in zip(out, want))
    line["create_over_set_sky_host"] = line["create_ms"] / line["set_sky_host_ms"]
    line["create_over_set_sky_device"] = line["create_ms"] / line["set_sky_device_ms"]
    r.close()
    snap.close()
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--scenes", default="env_like,envmini")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--table-reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("sky_bench: no CUDA device (the times are GPU measurements)")
    gpu, power, clock = rqb.gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        for name in args.scenes.split(","):
            if name == "env_like":
                path = os.path.join(tmp, "env_like.tsnap")
                bigscene.env_like(path)
            else:
                path = tb.scene_path(name)
            line = bench(name, path, args, torch)
            line.update(gpu=gpu, power_limit=power, max_sm_clock=clock)
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
