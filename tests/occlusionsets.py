"""Ray batches and the expected answers for the occlusion query tests (tests/test_occlusion_gpu.py) and
tools/ray_query_bench.py: tmax columns for rays in the layout of tb200_ray (column 7, `pad`, is the occlusion query's
tmax), segment rays between two batches' hit points, and the verdict derived from the closest-hit query's answer.
The ray batches themselves come from tests/raysets.py."""
import numpy as np

from raysets import pack


def with_tmax(rays, tmax):
    """A copy of `rays` with column 7 (tb200_ray::pad, the occlusion query's tmax) set to `tmax` (N,) or a scalar."""
    out = np.array(rays, np.float32, copy=True)
    out[:, 7] = tmax
    return out


def occluded(hits, prims, tmax):
    """The occlusion query's answer from the closest-hit query's: a primitive was hit and its t < tmax."""
    return (prims >= 0) & (hits[:, 0] < np.asarray(tmax, np.float32))


def tmax_sets(hits, prims, rng):
    """tmax columns (N,) float32 for rays whose closest hits are hits / prims: +inf; uniform in [0, 2 t]; and the edge
    values around each ray's own t (a miss's t is FLT_MAX) and at the ends of the float range."""
    t = hits[:, 0].astype(np.float32)
    n = len(t)
    fmax = np.finfo(np.float32).max
    with np.errstate(over="ignore"):   # a miss's 2 t and the float above FLT_MAX round to +inf, as they should
        uniform = rng.uniform(0.0, 2.0 * t.astype(np.float64)).astype(np.float32)
        t_up = np.nextafter(t, np.float32(np.inf))
    return {
        "inf": np.full(n, np.inf, np.float32),
        "uniform": uniform,
        "t": t,
        "t_up": t_up,
        "t_down": np.nextafter(t, np.float32(0.0)),
        "zero": np.zeros(n, np.float32),
        "minus_zero": np.full(n, -0.0, np.float32),
        "negative": -rng.uniform(1e-3, 10.0, n).astype(np.float32),
        "denormal": np.full(n, np.nextafter(np.float32(0.0), np.float32(1.0)), np.float32),
        "flt_max": np.full(n, fmax, np.float32),
        "nan": np.full(n, np.nan, np.float32),
    }


def point_to_point_rays(a_rays, a_hits, a_prims, b_rays, b_hits, b_prims, rng, tmax):
    """Segment rays between the hit points of two batches: from each hit point of `a_rays`, offset along its
    FaceForward'ed normal by 1e-4 towards the target as secondary_rays does, to a hit point of `b_rays`, with
    dir = target - origin and the given tmax (1 ends the segment at the target)."""
    ka, kb = a_prims >= 0, b_prims >= 0
    pa = a_rays[ka, 0:3] + a_rays[ka, 4:7] * a_hits[ka, 0:1]
    pb = b_rays[kb, 0:3] + b_rays[kb, 4:7] * b_hits[kb, 0:1]
    m = min(len(pa), len(pb))
    pa, pb, na = pa[:m], pb[rng.permutation(len(pb))[:m]], a_hits[ka, 1:4][:m]
    side = np.where(np.sum(na * (pb - pa), axis=1, keepdims=True) < 0.0, -1.0, 1.0).astype(np.float32)
    o = pa + na * side * np.float32(1e-4)
    out = pack(o, pb - o, a_rays[ka, 3][:m])
    out[:, 7] = tmax
    return out
