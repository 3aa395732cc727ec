#!/usr/bin/env python
"""Throughput of the emitter and probe sample queries (Renderer.sample_emitters / tb200_sample_emitters and
Renderer.sample_probe / tb200_sample_probe), one JSON line per scene:
    python tools/emitter_query_bench.py [--scenes cornell,veach,envmini] [--log2-n 24] [--calls 10]

Per scene, 2^log2-n queries: emitter queries over the scene's lights (each record a light picked uniformly at random,
a time uniform in [0, 1) and a random seed), and as many probe seeds when the sky has a probe.  Each query kind is timed
with CUDA events around `--calls` calls after `--warmup`; its kernel time is stats.gpuMs.  The HBM floor counts the
bytes each query streams at the H100 SXM's 3.35 TB/s: 44 per emitter query (the 8-byte record, the 4-byte seed, the
32-byte output) and 36 per probe query (seed and output).  It leaves out the gathers (a light's primitive record, a
mesh light's CDF search and triangle, the probe's CDF searches and texel), which mostly hit L2, so the floor is an
estimate from below.  The first 2^14 results of each kind are checked bit for bit against the CPU restatement.  The
GPU's name, power limit and maximum SM clock are read in the same run.  Needs a GPU."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import tinsel_b200 as tb  # noqa: E402
import emitteroracle  # noqa: E402
import ray_query_bench as rqb  # noqa: E402

EMITTER_BYTES = 8 + 4 + 32
PROBE_BYTES = 4 + 32


def _exact(got, want):
    return bool(((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))).all())


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--scenes", default="cornell,veach,envmini")
    ap.add_argument("--log2-n", type=int, default=24)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("emitter_query_bench: no CUDA device (the rates are GPU measurements)")
    gpu, power, clock = rqb.gpu_info()
    n = 1 << args.log2_n
    k = min(n, 1 << 14)
    for name in args.scenes.split(","):
        snap = tb.Snapshot(tb.scene_path(name))
        sc = snap.scene.contents
        r = tb.Renderer(snap.scene)
        g = torch.Generator(device="cuda").manual_seed(1)
        seeds = torch.randint(-2 ** 31, 2 ** 31 - 1, (n,), device="cuda", generator=g, dtype=torch.int32)
        line = {"scene": name, "gpu": gpu, "power_limit": power, "max_sm_clock": clock, "queries": n}
        lights = [i for i in range(sc.numPrimitives) if sc.primitives[i].lightSamples > 0]
        if lights:
            pick = torch.randint(0, len(lights), (n,), device="cuda", generator=g)
            prims = torch.tensor(lights, dtype=torch.int32, device="cuda")[pick]
            q = tb.emitter_queries(prims, torch.rand(n, device="cuda", generator=g))
            out = torch.empty((n, 8), device="cuda")
            ms, kms = rqb.time_calls(torch, r, lambda: r.sample_emitters(q, seeds, out), args.warmup, args.calls)
            e = rqb.rates(n, ms, kms, EMITTER_BYTES)
            e["gqueries_per_s"] = round(n / kms / 1e6, 2)
            del e["mrays_per_s"]
            e["lights"] = {"sphere": sum(sc.primitives[i].type == tb.abi.SPHERE for i in lights),
                           "mesh": sum(sc.primitives[i].type == tb.abi.MESH for i in lights)}
            want = emitteroracle.sample_emitters(snap.scene, q[:k].cpu().numpy(), seeds[:k].cpu().numpy())
            e["bit_exact_2^14"] = _exact(out[:k].cpu().numpy(), want)
            line["sample_emitters"] = e
        if sc.sky.probeValid:
            out = torch.empty((n, 8), device="cuda")
            ms, kms = rqb.time_calls(torch, r, lambda: r.sample_probe(seeds, out), args.warmup, args.calls)
            p = rqb.rates(n, ms, kms, PROBE_BYTES)
            p["gqueries_per_s"] = round(n / kms / 1e6, 2)
            del p["mrays_per_s"]
            p["probe"] = "%dx%d" % (sc.sky.probeWidth, sc.sky.probeHeight)
            want = emitteroracle.sample_probe(snap.scene, seeds[:k].cpu().numpy())
            p["bit_exact_2^14"] = _exact(out[:k].cpu().numpy(), want)
            line["sample_probe"] = p
        print(json.dumps(line), flush=True)
        r.close()
        snap.close()


if __name__ == "__main__":
    main()
