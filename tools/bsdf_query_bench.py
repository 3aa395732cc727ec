#!/usr/bin/env python
"""Throughput of the batched BSDF queries (Renderer.bsdf_eval / tb200_bsdf_eval and Renderer.bsdf_sample /
tb200_bsdf_sample), one JSON line per scene:
    python tools/bsdf_query_bench.py [--scenes cornell,veach,meshlight] [--calls 10] [--warmup 3]

Per scene: 2^24 queries built on the device from the hits of raster-order camera rays (misses left out, the hits
repeated to fill the batch): the hit primitive's own material, n = the hit normal, v = -dir, l uniform on the sphere,
and PathTrace's etas (entering, (1, ior), or leaving, (ior, 1), half each).  Eval and sample are timed separately
with CUDA events around `--calls` calls after the warm-up; the kernel's own time is stats.gpuMs.  Reported: ms per
call, kernel ms, Gqueries/s, the bytes each query moves (eval 48 in + 16 out = 64, sample 48 + 4 in + 32 out = 84)
against the H100 SXM's 3.35 TB/s, a bit-exact check of the first 2^16 queries against the CPU restatement, the
restatement's own rate on those queries (oracle_bsdf_cases, one host thread), and the GPU's name, power limit and
maximum SM clock, read in the same run.  Needs a GPU."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import tinsel_b200 as tb  # noqa: E402
import ray_query_bench as rqb  # noqa: E402
import test_bsdf_gpu as bsdf  # noqa: E402
import test_bsdf_query_gpu as bq  # noqa: E402

EVAL_BYTES = 48 + 16
SAMPLE_BYTES = 48 + 4 + 32


def hit_queries(torch, r, snap, mats, n, seed):
    """(queries (n, 12), seeds (n,) int32) on the device from camera-ray hits, as the module docstring describes."""
    side = 1 << (int(np.log2(n)) // 2)
    rays = rqb.camera_rays_device(torch, snap.camera, side, seed)
    hits, prims = r.trace_rays(rays)
    keep = torch.nonzero(prims >= 0).squeeze(1)
    idx = keep[torch.arange(n, device="cuda") % len(keep)]
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    prim = prims[idx]
    ior = torch.from_numpy(tb.material_ior(mats["eta"], mats["specular"])).cuda()[prim.long()]
    leaving = torch.rand(n, device="cuda", generator=g) < 0.5
    one = torch.ones(n, device="cuda")
    l = torch.randn((n, 3), device="cuda", generator=g)
    l = l / l.norm(dim=1, keepdim=True)
    q = tb.bsdf_queries(prim, hits[idx, 1:4].contiguous(), (-rays[idx, 4:7]).contiguous(),
                        torch.where(leaving, ior, one), torch.where(leaving, one, ior), l)
    seeds = torch.randint(-2 ** 31, 2 ** 31 - 1, (n,), device="cuda", generator=g, dtype=torch.int32)
    return q, seeds


def cases_of(q, seeds):
    """The CASE_DTYPE cases of query records (numpy (k, 12)) and seeds, for the restatement."""
    c = np.zeros(len(q), bsdf.CASE_DTYPE)
    c["n"], c["v"], c["l"] = q[:, 0:3], q[:, 4:7], q[:, 8:11]
    c["mat"] = q[:, 3].view(np.int32)
    c["etaI"], c["etaO"] = q[:, 7], q[:, 11]
    c["seed"] = seeds
    return c


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--scenes", default="cornell,veach,meshlight")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--log2-queries", type=int, default=24)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bsdf_query_bench: no CUDA device (the rates are GPU measurements)")
    gpu, power, clock = rqb.gpu_info()
    n = 1 << args.log2_queries
    for name in args.scenes.split(","):
        path = tb.scene_path(name)
        if not os.path.exists(path):
            continue
        snap = tb.Snapshot(path)
        mats = bq.materials_of(snap.scene.contents)
        r = tb.Renderer(snap.scene)
        q, seeds = hit_queries(torch, r, snap, mats, n, 1)
        ev = torch.empty((n, 4), device="cuda")
        sm = torch.empty((n, 8), device="cuda")
        line = {"scene": name, "queries": n, "gpu": gpu, "power_limit": power, "max_sm_clock": clock}
        k = min(n, 1 << 16)
        c = cases_of(q[:k].cpu().numpy(), seeds[:k].cpu().numpy())
        t0 = time.perf_counter()
        wev, ws = bq.expected(mats, c)
        cpu_rate = k / (time.perf_counter() - t0) / 1e6
        for arm, call, nbytes in (("eval", lambda: r.bsdf_eval(q, ev), EVAL_BYTES),
                                  ("sample", lambda: r.bsdf_sample(q, seeds, sm), SAMPLE_BYTES)):
            ms, kms = rqb.time_calls(torch, r, call, args.warmup, args.calls)
            out = rqb.rates(n, ms, kms, nbytes)
            out["gqueries_per_s"] = round(n / ms / 1e6, 2)
            del out["mrays_per_s"]
            out["bytes_per_query"] = out.pop("bytes_per_ray")
            got = (ev if arm == "eval" else sm)[:k].cpu().numpy()
            out["bit_exact_2^16"] = not bq.mismatches(got, wev if arm == "eval" else ws).any()
            line[arm] = out
        line["cpu_restatement_mqueries_per_s"] = round(cpu_rate, 3)
        line["cpu_threads"] = 1
        print(json.dumps(line), flush=True)
        r.close()
        snap.close()


if __name__ == "__main__":
    main()
