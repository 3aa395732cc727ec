#!/usr/bin/env python
"""Throughput of the batched closest-hit and occlusion queries (Renderer.trace_rays / tb200_trace_rays,
Renderer.trace_rays_tri / tb200_trace_rays_tri and Renderer.occluded / tb200_occluded_rays), one JSON line per scene:
    python tools/ray_query_bench.py [--scenes cornell,veach,meshlight,ajax,env] [--calls 10] [--warmup 3]

Closest hit, per scene: Mrays/s for 2^24 coherent camera rays (a raster-order 4096 x 4096 grid, jittered) and 2^24
random rays (origins in and around the scene bounds, uniform directions), from CUDA events around `--calls` timed
calls after the warm-up; the bytes each ray moves (32 in, 20 out) against the H100 SXM's 3.35 TB/s; the CPU
restatement's rate on every host core (tests/rayoracle.py); a bit-exact check of 2^16 rays against it; and the GPU's
name, power limit and maximum SM clock, read in the same run.

Closest hit with the hit triangle (key "tri"), on the same camera and random batches: the same rates (68 bytes per
ray: 32 in, 16 + 4 + 16 out), the kernel time against trace_rays' on the same rays, the fraction of rays that hit a
mesh, and a bit-exact check of 2^16 rays (hits, primitives, triangles and weights) against the restatement
(tests/trioracle.py).

Occlusion (key "occluded"), on the same batches: the camera rays with tmax = +inf, the random rays with tmax uniform
in [0, the scene's diagonal), and point-to-point segments built on the device from the camera rays' hit points to
those of the same rays in another order (dir = target - origin, tmax = 1).  Each reports the same rates (33 bytes
per ray: 32 in, 1 out), the occluded fraction, the kernel time against trace_rays' on the same rays, and an exact check
of 2^16 rays against the restatement's closest hits.  ajax and env are skipped when their snapshots are not present.
Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import tinsel_b200 as tb  # noqa: E402
import occlusionsets  # noqa: E402
import rayoracle  # noqa: E402
import raysets  # noqa: E402
import trioracle  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BYTES_PER_RAY = 32 + 16 + 4
OCC_BYTES_PER_RAY = 32 + 1
TRI_BYTES_PER_RAY = 32 + 16 + 4 + 16


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return name, power, clock
    except Exception as e:   # the rates are still measured; the line says what could not be read
        import torch
        unknown = "unknown (%s)" % type(e).__name__
        return torch.cuda.get_device_name(0), unknown, unknown


def camera_rays_device(torch, camera, side, seed):
    """side*side camera rays in raster order (neighbouring rays are neighbouring pixels), on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = side * side
    idx = torch.arange(n, device="cuda")
    px = (idx % side).float() + torch.rand(n, device="cuda", generator=g)
    py = (idx // side).float() + torch.rand(n, device="cuda", generator=g)
    f = float(np.tan(camera.fov * 0.5))
    d = torch.stack([(2.0 * px / side - 1.0) * f, (1.0 - 2.0 * py / side) * f, -torch.ones(n, device="cuda")], 1)
    d = d / d.norm(dim=1, keepdim=True)
    q = torch.tensor(camera.rotation[:], device="cuda")
    u = q[:3].expand(n, 3)
    t = 2.0 * torch.cross(u, d, dim=1)
    d = d + q[3] * t + torch.cross(u, t, dim=1)
    rays = torch.zeros((n, 8), device="cuda")
    rays[:, 0:3] = torch.tensor(camera.position[:], device="cuda")
    rays[:, 3] = camera.shutterStart + (camera.shutterEnd - camera.shutterStart) * torch.rand(n, device="cuda", generator=g)
    rays[:, 4:7] = d
    return rays


def random_rays_device(torch, scene, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lo, hi = raysets.scene_bounds(scene)
    pad = 0.2 * (hi - lo) + 1e-3
    lo_t = torch.tensor(lo - pad, device="cuda", dtype=torch.float32)
    span = torch.tensor((hi - lo) + 2 * pad, device="cuda", dtype=torch.float32)
    d = torch.randn((n, 3), device="cuda", generator=g)
    rays = torch.zeros((n, 8), device="cuda")
    rays[:, 0:3] = lo_t + span * torch.rand((n, 3), device="cuda", generator=g)
    rays[:, 3] = torch.rand(n, device="cuda", generator=g)
    rays[:, 4:7] = d / d.norm(dim=1, keepdim=True)
    return rays


def time_calls(torch, r, call, warmup, calls):
    """ms per call from CUDA events around `calls` calls of call() on the caller's stream, and the kernel's own median time."""
    stream = torch.cuda.current_stream()
    r.set_stream(stream.cuda_stream)
    for _ in range(warmup):
        call()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kernel = []
    start.record(stream)
    for _ in range(calls):
        call()
        kernel.append(r.stats().gpuMs)
    end.record(stream)
    end.synchronize()
    r.set_stream(None)
    return start.elapsed_time(end) / calls, float(np.median(kernel))


def rates(n, ms, kms, bytes_per_ray):
    floor = n * bytes_per_ray / HBM_BYTES_PER_S * 1e3
    return {"ms_per_call": round(ms, 4), "kernel_ms": round(kms, 4), "mrays_per_s": round(n / ms / 1e3, 1),
            "bytes_per_ray": bytes_per_ray, "hbm_floor_ms": round(floor, 4),
            "share_of_hbm_floor": round(floor / kms, 4) if kms > 0 else None}


def point_to_point_device(torch, rays, hits, prims, seed):
    """Segments from the hit points of `rays` (offset by 1e-4 along the face-forwarded normal, towards the target)
    to the hit points of the same rays in a random order: dir = target - origin, tmax = 1.  Misses are left out."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    keep = torch.nonzero(prims >= 0).squeeze(1)
    p = rays[keep, 0:3] + rays[keep, 4:7] * hits[keep, 0:1]
    nrm = hits[keep, 1:4]
    target = p[torch.randperm(len(keep), device="cuda", generator=g)]
    side = torch.where((nrm * (target - p)).sum(1, keepdim=True) < 0.0, -1.0, 1.0)
    o = p + nrm * side * 1e-4
    out = torch.zeros((len(keep), 8), device="cuda")
    out[:, 0:3] = o
    out[:, 3] = rays[keep, 3]
    out[:, 4:7] = target - o
    out[:, 7] = 1.0
    return out


def occlusion_arm(torch, r, port, rays, occ, trace_kms, args):
    """The occlusion query on `rays` (tmax in column 7): rates, occluded fraction, kernel time against trace_rays'
    (trace_kms, on the same rays) and an exact check of the first 2^16 rays against the restatement."""
    n = len(rays)
    ms, kms = time_calls(torch, r, lambda: r.occluded(rays, occ[:n]), args.warmup, args.calls)
    out = rates(n, ms, kms, OCC_BYTES_PER_RAY)
    out["rays"] = n
    out["occluded_fraction"] = round(float(occ[:n].float().mean()), 4)
    out["trace_rays_kernel_ms"] = round(trace_kms, 4)
    out["kernel_ms_over_trace_rays"] = round(kms / trace_kms, 4) if trace_kms > 0 else None
    k = min(n, 1 << 16)
    sub = rays[:k].cpu().numpy()
    want_h, want_p = port.trace_rays(sub)
    out["bit_exact_2^16"] = bool((occ[:k].cpu().numpy() == occlusionsets.occluded(want_h, want_p, sub[:, 7])).all())
    return out


def tri_arm(torch, r, port, rays, hits, prims, tris, trace_kms, args):
    """The closest-hit query with the hit triangle on `rays`: rates, kernel time against trace_rays' (trace_kms, on the
    same rays), the mesh-hit fraction and a bit-exact check of the first 2^16 rays against the restatement."""
    n = len(rays)
    ms, kms = time_calls(torch, r, lambda: r.trace_rays_tri(rays, hits, prims, tris), args.warmup, args.calls)
    out = rates(n, ms, kms, TRI_BYTES_PER_RAY)
    out["trace_rays_kernel_ms"] = round(trace_kms, 4)
    out["kernel_ms_over_trace_rays"] = round(kms / trace_kms, 4) if trace_kms > 0 else None
    out["mesh_hit_fraction"] = round(float((tris[:, 0] >= 0).float().mean()), 4)
    k = min(n, 1 << 16)
    want_h, want_p, want_tri, want_uvw = port.trace_rays_tri(rays[:k].cpu().numpy())
    got = tris[:k].cpu().numpy()
    out["bit_exact_2^16"] = (len(raysets.mismatches(hits[:k].cpu().numpy(), prims[:k].cpu().numpy(), want_h, want_p)) == 0 and
                             bool((got[:, 0] == want_tri).all()) and bool((got[:, 1:] == want_uvw.view(np.int32)).all()))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--scenes", default="cornell,veach,meshlight,ajax,env")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--log2-rays", type=int, default=24)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ray_query_bench: no CUDA device (the rates are GPU measurements)")
    rayoracle.load()
    trioracle.load()
    gpu, power, clock = gpu_info()
    n = 1 << args.log2_rays
    side = 1 << (args.log2_rays // 2)
    for name in args.scenes.split(","):
        path = tb.scene_path(name)
        if not os.path.exists(path):
            continue
        snap = tb.Snapshot(path)
        scene = snap.scene.contents
        r = tb.Renderer(snap.scene)
        port = rayoracle.RayOracle.from_snapshot(path)
        tri_port = trioracle.TriOracle.from_snapshot(path)
        line = {"scene": name, "rays": n, "gpu": gpu, "power_limit": power, "max_sm_clock": clock,
                "library": os.path.basename(os.environ.get("TINSEL_B200_LIB", tb.LIB_PATH))}
        hits = torch.empty((n, 4), device="cuda")
        prims = torch.empty((n,), device="cuda", dtype=torch.int32)
        occ = torch.empty((n,), device="cuda", dtype=torch.bool)
        tris = torch.empty((n, 4), device="cuda", dtype=torch.int32)
        lo, hi = raysets.scene_bounds(scene)
        diagonal = float(np.linalg.norm(hi - lo))
        line["occluded"] = {}
        line["tri"] = {}
        for kind in ("camera", "random"):
            rays = camera_rays_device(torch, snap.camera, side, 1) if kind == "camera" else random_rays_device(torch, scene, n, 2)
            ms, kms = time_calls(torch, r, lambda: r.trace_rays(rays, hits, prims), args.warmup, args.calls)
            line[kind] = rates(n, ms, kms, BYTES_PER_RAY)
            # the CPU restatement on every host core, on the first 2^20 rays of the same batch
            sub = rays[: min(n, 1 << 20)].cpu().numpy()
            t0 = time.perf_counter()
            want_h, want_p = port.trace_rays(sub)
            line[kind]["cpu_mrays_per_s"] = round(len(sub) / (time.perf_counter() - t0) / 1e6, 2)
            k = min(n, 1 << 16)
            got_h, got_p = hits[:k].cpu().numpy(), prims[:k].cpu().numpy()
            line[kind]["bit_exact_2^16"] = len(raysets.mismatches(got_h, got_p, want_h[:k], want_p[:k])) == 0
            line[kind]["hit_fraction"] = round(float((prims >= 0).float().mean()), 4)
            # the query with the hit triangle on the same rays (it writes the same hits and prims)
            line["tri"][kind] = tri_arm(torch, r, tri_port, rays, hits, prims, tris, kms, args)
            # the occlusion query on the same rays
            if kind == "camera":
                rays[:, 7] = float("inf")
            else:
                g = torch.Generator(device="cuda").manual_seed(3)
                rays[:, 7] = diagonal * torch.rand(n, device="cuda", generator=g)
            line["occluded"][kind] = occlusion_arm(torch, r, port, rays, occ, kms, args)
            if kind == "camera":   # hits / prims still hold these rays' closest hits
                p2p = point_to_point_device(torch, rays, hits, prims, 4)
            del rays
        m = len(p2p)
        _, kms = time_calls(torch, r, lambda: r.trace_rays(p2p, hits[:m], prims[:m]), args.warmup, args.calls)
        line["occluded"]["point_to_point"] = occlusion_arm(torch, r, port, p2p, occ, kms, args)
        del p2p
        line["cpu_threads"] = os.cpu_count()
        print(json.dumps(line), flush=True)
        r.close()
        port.close()
        tri_port.close()
        snap.close()


if __name__ == "__main__":
    main()
