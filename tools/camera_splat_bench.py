#!/usr/bin/env python
"""Throughput of the camera-sample and splat queries (Renderer.camera_rays / tb200_camera_rays and Renderer.splat /
tb200_splat), one JSON line per scene:
    python tools/camera_splat_bench.py [--scenes cornell:1024x1024,veach:1920x1080] [--calls 10] [--warmup 3]

Per scene: 2^24 samples, the whole frames frame_samples gives from frame 0 at the given image size (cut at 2^24).
Camera rays: ms per call and the kernel's own time (stats.gpuMs), Gsamples/s, and the HBM floor of the 8 bytes read
and 40 written per sample against the H100 SXM's 3.35 TB/s.  Splat: the same rays' raster positions with uniform
radiance in [0, 1), splatted with the scene's own filter into a zeroed film, in frame-major order and in a shuffled
order; kernel ms, Gsamples/s and the filter reductions per sample, counted from each sample's footprint (the
Gaussian's zero-weight pixels, which the kernel skips, included).  Every line carries a bit-exact check on 2^16
samples: the camera rays against the CPU restatement (tests/camera_oracle.cpp); the splat, in the line's order, in
counting mode (box filter of width 0: at most two terms per pixel, whose float32 sum has one value) against the
same sums formed on the host.  The GPU's name, power limit and maximum SM clock are read in the same run.  Needs a
GPU."""
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
import cameraoracle  # noqa: E402
import filmref  # noqa: E402
import ray_query_bench as rqb  # noqa: E402

CAMERA_BYTES = 8 + 32 + 8
CHECK = 1 << 16


def footprint_pixels(torch, raster, o):
    """Pixels of each sample's AddSample footprint (render.cpp:404-407), as float64 on the device."""
    W, H, w = o.width, o.height, float(o.filterWidth)
    rx, ry = raster[:, 0].double(), raster[:, 1].double()
    sx = torch.clamp(torch.trunc(rx - w), min=0)
    sy = torch.clamp(torch.trunc(ry - w), min=0)
    ex = torch.clamp(torch.trunc(rx + w), max=W - 1)
    ey = torch.clamp(torch.trunc(ry + w), max=H - 1)
    return torch.clamp(ex - sx + 1, min=0) * torch.clamp(ey - sy + 1, min=0)


def counting_exact(torch, r, o, raster, radiance):
    """The counting-mode splat of the given samples on the device, bit for bit against float32 sums on the host."""
    c = filmref.counting_options(o)
    acc = torch.zeros((o.height, o.width, 4), device="cuda")
    r.splat(c, raster, radiance, acc)
    ras, rad = raster.cpu().numpy(), radiance.cpu().numpy()
    keep = (ras[:, 0] < o.width) & (ras[:, 1] < o.height)
    idx = ras[keep, 1].astype(np.int64) * o.width + ras[keep, 0].astype(np.int64)
    want = np.zeros((o.height * o.width, 4), np.float32)
    np.add.at(want, idx, np.concatenate([rad[keep], np.ones((int(keep.sum()), 1), np.float32)], 1))
    got = acc.cpu().numpy().reshape(-1, 4)
    return bool((got.view(np.uint32) == want.view(np.uint32)).all())


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--scenes", default="cornell:1024x1024,veach:1920x1080")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--log2-samples", type=int, default=24)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("camera_splat_bench: no CUDA device (the rates are GPU measurements)")
    gpu, power, clock = rqb.gpu_info()
    n = 1 << args.log2_samples
    for spec in args.scenes.split(","):
        name, size = spec.split(":")
        W, H = [int(v) for v in size.split("x")]
        snap = tb.Snapshot(tb.scene_path(name))
        cam, o = snap.camera, snap.options
        o.width, o.height = W, H
        r = tb.Renderer(snap.scene)
        frames = -(-n // (W * H))
        samples = tb.frame_samples(W, H, 0, frames, device="cuda")[:n].contiguous()
        rays = torch.empty((n, 8), device="cuda")
        raster = torch.empty((n, 2), device="cuda")
        line = {"scene": name, "width": W, "height": H, "samples": n, "gpu": gpu, "power_limit": power,
                "max_sm_clock": clock, "filter": {"type": int(o.filterType), "width": float(o.filterWidth)}}

        ms, kms = rqb.time_calls(torch, r, lambda: r.camera_rays(cam, o, samples, rays, raster), args.warmup, args.calls)
        out = rqb.rates(n, ms, kms, CAMERA_BYTES)
        del out["mrays_per_s"]
        out["gsamples_per_s"] = round(n / kms / 1e6, 2)
        out["bytes_per_sample"] = out.pop("bytes_per_ray")
        s16 = samples[:CHECK].cpu().numpy()
        org, d, t, ras = cameraoracle.camera_samples(cam, W, H, s16)
        want = np.concatenate([org, t[:, None], d, np.full((CHECK, 1), np.inf, np.float32)], 1)
        out["bit_exact_2^16"] = bool((rays[:CHECK].cpu().numpy().view(np.uint32) == want.view(np.uint32)).all() and
                                     (raster[:CHECK].cpu().numpy().view(np.uint32) == ras.view(np.uint32)).all())
        line["camera_rays"] = out

        g = torch.Generator(device="cuda").manual_seed(7)
        radiance = torch.rand((n, 3), device="cuda", generator=g)
        perm = torch.randperm(n, device="cuda", generator=g)
        reductions = float(footprint_pixels(torch, raster, o).mean())
        acc = torch.zeros((H, W, 4), device="cuda")
        for order, (ras_o, rad_o) in (("frame_major", (raster, radiance)),
                                      ("shuffled", (raster[perm].contiguous(), radiance[perm].contiguous()))):
            ms, kms = rqb.time_calls(torch, r, lambda: r.splat(o, ras_o, rad_o, acc), args.warmup, args.calls)
            # the line's bit-exact check: the 2^16 samples of frame 0's first pixels, in the line's order
            sel = torch.nonzero(perm < CHECK).squeeze(1) if order == "shuffled" else torch.arange(CHECK, device="cuda")
            line["splat_" + order] = {"ms_per_call": round(ms, 4), "kernel_ms": round(kms, 4),
                                      "gsamples_per_s": round(n / kms / 1e6, 2),
                                      "reductions_per_sample": round(reductions, 3),
                                      "bit_exact_2^16": counting_exact(torch, r, o, ras_o[sel].contiguous(),
                                                                       rad_o[sel].contiguous())}
        print(json.dumps(line), flush=True)
        r.close()
        snap.close()


if __name__ == "__main__":
    main()
