"""Ray batches for the closest-hit query tests and tools/ray_query_bench.py: (N, 8) float32 arrays in the layout of
tb200_ray (origin.xyz, time, dir.xyz, pad).  The rays are inputs only -- the device and the CPU restatement are
compared on the same array -- so the camera rays here come from a numpy pinhole model, not the renderer's
GenerateRay."""
import ctypes as C

import numpy as np

from tinsel_b200 import abi


def pack(o, d, time):
    """(N, 8) float32 rays from origins (N, 3), directions (N, 3) and times (N,) or a scalar."""
    o = np.asarray(o, np.float32).reshape(-1, 3)
    d = np.asarray(d, np.float32).reshape(-1, 3)
    out = np.zeros((len(o), 8), np.float32)
    out[:, 0:3] = o
    out[:, 3] = time
    out[:, 4:7] = d
    return out


def scene_bounds(scene):
    """(lo, hi) over the finite boxes of the scene-level BVH (planes' +-1e8 boxes are left out)."""
    nodes = C.cast(scene.bvhNodes, C.POINTER(abi.BvhNode * scene.numBvhNodes)).contents
    lo, hi = np.full(3, np.inf), np.full(3, -np.inf)
    for n in nodes:
        a, b = np.array(n.lower[:]), np.array(n.upper[:])
        if np.all(np.abs(a) < 5e7) and np.all(np.abs(b) < 5e7):
            lo, hi = np.minimum(lo, a), np.maximum(hi, b)
    if not np.all(np.isfinite(lo)):
        lo, hi = np.full(3, -1.0), np.full(3, 1.0)
    return lo, hi


def _rotate(q, v):
    """Rotates the vectors v (N, 3) by the quaternion q = (x, y, z, w)."""
    u, w = np.asarray(q[:3], np.float64), float(q[3])
    t = 2.0 * np.cross(u, v)
    return v + w * t + np.cross(u, t)


def camera_rays(camera, n, rng, width=640, height=480, time=None):
    """n rays of `camera` through jittered raster positions, times in the shutter interval unless given."""
    px = rng.uniform(0.0, width, n)
    py = rng.uniform(0.0, height, n)
    f = np.tan(camera.fov * 0.5)
    d = np.stack([(2.0 * px / width - 1.0) * f * width / height, (1.0 - 2.0 * py / height) * f, -np.ones(n)], 1)
    d = _rotate(camera.rotation, d / np.linalg.norm(d, axis=1, keepdims=True))
    if time is None:
        time = rng.uniform(camera.shutterStart, camera.shutterEnd, n)
    return pack(np.tile(camera.position[:], (n, 1)), d, time)


def _directions(rng, n):
    d = rng.normal(size=(n, 3))
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def random_rays(scene, n, rng, time=(0.0, 1.0)):
    """Origins uniform in and around the scene's finite bounds, uniform directions; half of them scaled to a length
    in [0.25, 4) (the query uses dir as given)."""
    lo, hi = scene_bounds(scene)
    pad = 0.2 * (hi - lo) + 1e-3
    o = rng.uniform(lo - pad, hi + pad, (n, 3))
    d = _directions(rng, n)
    scale = np.where(rng.uniform(size=n) < 0.5, 1.0, rng.uniform(0.25, 4.0, n))
    return pack(o, d * scale[:, None], rng.uniform(time[0], time[1], n))


def secondary_rays(rays, hits, prims, rng):
    """Rays that leave the hit points of `rays` (hits / prims as the query returns them) in uniform directions,
    from the point offset along FaceForward(n, d) * 1e-4 as the path tracer does."""
    keep = prims >= 0
    r, h = rays[keep], hits[keep]
    p = r[:, 0:3] + r[:, 4:7] * h[:, 0:1]
    d = _directions(rng, len(r)).astype(np.float32)
    n = h[:, 1:4]
    side = np.where(np.sum(n * d, axis=1, keepdims=True) < 0.0, -1.0, 1.0).astype(np.float32)
    return pack(p + n * side * np.float32(1e-4), d, r[:, 3])


def fallback_rays(scene, rng, n=512):
    """Rays that trace_closest hands to the ordered walk or that stress the slab tests: origins beyond 1e7, NaN and
    zero direction components, axis-aligned directions."""
    lo, hi = scene_bounds(scene)
    c = 0.5 * (lo + hi)
    far = c + _directions(rng, n) * rng.uniform(1.1e7, 1.0e8, (n, 1))
    far_d = (c - far) + rng.normal(size=(n, 3)) * 1e5
    inside = rng.uniform(lo, hi, (n, 3))
    nan_d = _directions(rng, n)
    nan_d[np.arange(n), rng.randint(0, 3, n)] = np.nan
    zero_d = _directions(rng, n)
    col = rng.randint(0, 3, n)
    zero_d[np.arange(n), col] = 0.0
    zero_d[np.arange(n // 4), (col[: n // 4] + 1) % 3] = 0.0   # a quarter with two zero components
    axes = np.concatenate([np.eye(3), -np.eye(3)])[rng.randint(0, 6, n)]
    t = rng.uniform(0.0, 1.0, n)
    return np.concatenate([pack(far, far_d, t), pack(inside, nan_d, t), pack(inside, zero_d, t), pack(inside, axes, t),
                           pack(far, axes, t)])


def mismatches(a_hits, a_prims, b_hits, b_prims):
    """Indices where two query results differ: the primitive, or the bits of t / normal (NaN matches NaN)."""
    bits = (a_hits.view(np.uint32) == b_hits.view(np.uint32)) | (np.isnan(a_hits) & np.isnan(b_hits))
    return np.nonzero((a_prims != b_prims) | ~bits.all(axis=1))[0]
