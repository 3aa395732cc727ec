#!/usr/bin/env python
"""Throughput of the light queries (Renderer.sample_lights / tb200_sample_lights and Renderer.sky / tb200_sky_eval),
one JSON line per scene:
    python tools/light_query_bench.py [--scenes cornell:1024x1024,veach:1920x1080,envmini:1024x1024] [--calls 10]

Per scene: the first hits of one frame of the image's own camera samples at the given size (camera_rays, then
trace_rays; misses left out), with PathTrace's first-bounce etas (1, the material's ior) and random seeds.  NEE is
timed with CUDA events around `--calls` calls after `--warmup`; its kernel time is stats.gpuMs.  Reported: ms per
call, kernel ms, Mqueries/s and shadow rays/s (each query traces the probe sample when the sky has one, plus every
light's lightSamples), and as the comparison point trace_rays' kernel time over as many shadow rays of the same kind
built in torch: from each hit point, offset along the face-forwarded normal, to the centre of each light once per
sample, and in a uniform direction for the probe sample.  The first 2^14 NEE results are checked bit for bit against
the CPU restatement.  The sky is timed over 2^24 uniform directions against the HBM floor of the bytes it moves (the
32-byte sector holding each ray's direction in, 16 bytes out) at the H100 SXM's 3.35 TB/s.  The GPU's name, power
limit and maximum SM clock are read in the same run.  Needs a GPU."""
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
import lightoracle  # noqa: E402
import ray_query_bench as rqb  # noqa: E402

SKY_BYTES = 32 + 16


def first_hit_queries(torch, r, snap, W, H, seed):
    """(queries (n, 16), seeds (n,), hits, normals) at the hits of frame 0's camera samples of a W x H image."""
    opt = snap.options
    opt.width, opt.height = W, H
    rays, _ = r.camera_rays(snap.camera, opt, tb.frame_samples(W, H, 0, device="cuda"))
    hits, prims = r.trace_rays(rays)
    keep = torch.nonzero(prims >= 0).squeeze(1)
    rays, hits, prims = rays[keep], hits[keep], prims[keep]
    sc = snap.scene.contents
    eta = np.array([sc.primitives[i].material.eta for i in range(sc.numPrimitives)], np.float32)
    spec = np.array([sc.primitives[i].material.specular for i in range(sc.numPrimitives)], np.float32)
    ior = torch.from_numpy(tb.material_ior(eta, spec).reshape(-1)).cuda()[prims.long()]
    d = rays[:, 4:7]
    p = rays[:, 0:3] + d * hits[:, 0:1]
    n = hits[:, 1:4].contiguous()
    q = tb.light_queries(prims, p, n, -d, 1.0, ior, rays[:, 3].contiguous())
    g = torch.Generator(device="cuda").manual_seed(seed)
    seeds = torch.randint(-2 ** 31, 2 ** 31 - 1, (len(prims),), device="cuda", generator=g, dtype=torch.int32)
    return q, seeds, p, n


def shadow_rays(torch, snap, p, n, seed):
    """The comparison rays: per hit, one ray to each light's centre per light sample, one uniform probe direction."""
    sc = snap.scene.contents
    g = torch.Generator(device="cuda").manual_seed(seed)
    targets = []
    for i in range(sc.numPrimitives):
        targets += [list(sc.primitives[i].start.p)] * sc.primitives[i].lightSamples
    dirs = []
    for c in targets:
        w = torch.tensor(c, device="cuda") - p
        dirs.append(w / w.norm(dim=1, keepdim=True))
    if sc.sky.probeValid:
        w = torch.randn(p.shape, device="cuda", generator=g)
        dirs.append(w / w.norm(dim=1, keepdim=True))
    out = []
    for w in dirs:
        side = torch.where((n * w).sum(1, keepdim=True) < 0.0, -1.0, 1.0)
        rays = torch.zeros((len(p), 8), device="cuda")
        rays[:, 0:3] = p + n * side * 1e-4
        rays[:, 4:7] = w
        out.append(rays)
    return torch.cat(out) if out else torch.zeros((0, 8), device="cuda")


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--scenes", default="cornell:1024x1024,veach:1920x1080,envmini:1024x1024")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--log2-sky", type=int, default=24)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("light_query_bench: no CUDA device (the rates are GPU measurements)")
    gpu, power, clock = rqb.gpu_info()
    for spec in args.scenes.split(","):
        name, size = spec.split(":")
        W, H = (int(x) for x in size.split("x"))
        snap = tb.Snapshot(tb.scene_path(name))
        sc = snap.scene.contents
        r = tb.Renderer(snap.scene)
        q, seeds, p, n = first_hit_queries(torch, r, snap, W, H, 1)
        nq = len(q)
        per_query = int(bool(sc.sky.probeValid)) + sum(sc.primitives[i].lightSamples for i in range(sc.numPrimitives))
        out = torch.empty((nq, 3), device="cuda")
        ms, kms = rqb.time_calls(torch, r, lambda: r.sample_lights(q, seeds, out), args.warmup, args.calls)
        line = {"scene": name, "image": size, "gpu": gpu, "power_limit": power, "max_sm_clock": clock}
        k = min(nq, 1 << 14)
        want = lightoracle.sample_lights(snap.scene, q[:k].cpu().numpy(), seeds[:k].cpu().numpy())
        got = out[:k].cpu().numpy()
        exact = ((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))).all()
        nee = {"queries": nq, "shadow_rays_per_query": per_query, "ms_per_call": round(ms, 4),
               "kernel_ms": round(kms, 4), "mqueries_per_s": round(nq / kms / 1e3, 1),
               "mshadow_rays_per_s": round(nq * per_query / kms / 1e3, 1), "bit_exact_2^14": bool(exact)}
        sr = shadow_rays(torch, snap, p, n, 2)
        if len(sr):
            hits, prims = torch.empty((len(sr), 4), device="cuda"), torch.empty(len(sr), dtype=torch.int32, device="cuda")
            _, tkms = rqb.time_calls(torch, r, lambda: r.trace_rays(sr, hits, prims), args.warmup, args.calls)
            nee["trace_rays_same_count_kernel_ms"] = round(tkms, 4)
            nee["trace_rays_mrays_per_s"] = round(len(sr) / tkms / 1e3, 1)
        line["sample_lights"] = nee
        ns = 1 << args.log2_sky
        g = torch.Generator(device="cuda").manual_seed(3)
        rays = torch.zeros((ns, 8), device="cuda")
        d = torch.randn((ns, 3), device="cuda", generator=g)
        rays[:, 4:7] = d / d.norm(dim=1, keepdim=True)
        sky = torch.empty((ns, 4), device="cuda")
        ms, kms = rqb.time_calls(torch, r, lambda: r.sky(rays, sky), args.warmup, args.calls)
        s = rqb.rates(ns, ms, kms, SKY_BYTES)
        s["gqueries_per_s"] = round(ns / kms / 1e6, 2)
        del s["mrays_per_s"]
        s["probe"] = bool(sc.sky.probeValid)
        line["sky"] = s
        print(json.dumps(line), flush=True)
        r.set_stream(None)
        r.close()
        snap.close()


if __name__ == "__main__":
    main()
