"""Stand-ins, written by the tests themselves, for the two large scenes of BASELINE.json whose snapshots a checkout does
not hold (they are git-ignored: tools/make_snapshots.py): ajax (C3, a mesh of about 545 000 triangles) and env (C5,
lit by a 4000 x 2000 HDR probe).

  ajax_like  a bumpy torus of 512 000 triangles (closed, non-convex, high-frequency displacement: overlapping boxes
             and grazing rays) with a balanced median-split BVH of 19 interior levels, instanced twice (a static
             diffuse instance, and a rotated, scaled mesh light whose area CDF has 512 000 entries), on a diffuse
             floor under a sphere light
  env_like   a glass torus (transmission, absorption) of 12 288 triangles on a floor, lit only by a synthetic
             4000 x 2000 probe: a sky gradient, a sun disc 10^4 times brighter than the sky, a mountain horizon (runs
             of black texels inside rows: runs of equal values in cdfX), black ground rows (NaN rows of cdfX, as
             BuildCDF makes them), a block of identical texels and one isolated hot texel

Everything is vectorised numpy: fuzzscene.MeshData and _build_bvh loop over triangles in Python.  The snapshots go
through fuzzscene._save (tb200_snapshot_save) to wherever the caller asks, a temporary directory in the tests."""
import ctypes as C
import time

import numpy as np

from tinsel_b200 import abi
import fuzzscene

LEAF = fuzzscene.LEAF
NODE_DTYPE = np.dtype([("lower", np.float32, 3), ("upper", np.float32, 3), ("left", np.uint32), ("right_leaf", np.uint32)])
AJAX_GRID = (800, 320)    # torus segments around the major and the minor circle: 2 * 800 * 320 = 512 000 triangles
ENV_GRID = (128, 48)      # 12 288 triangles
PROBE_SIZE = (4000, 2000)


def torus(nu, nv, major, minor, bumps):
    """A closed torus of 2 nu nv triangles, its tube radius displaced by `bumps` times a sum of high-frequency sines;
    float64 positions (V, 3), unit normals of the undisplaced torus (V, 3), int32 indices (T, 3)."""
    u = np.arange(nu) * (2.0 * np.pi / nu)
    v = np.arange(nv) * (2.0 * np.pi / nv)
    U, V = np.meshgrid(u, v, indexing="ij")
    r = minor * (1.0 + bumps * (np.sin(37.0 * U) * np.sin(11.0 * V) + 0.5 * np.sin(91.0 * U + 29.0 * V)))
    ring = major + r * np.cos(V)
    pos = np.stack([ring * np.cos(U), r * np.sin(V), ring * np.sin(U)], -1).reshape(-1, 3)
    nrm = np.stack([np.cos(V) * np.cos(U), np.sin(V), np.cos(V) * np.sin(U)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    a = i * nv + j
    b = ((i + 1) % nu) * nv + j
    c = ((i + 1) % nu) * nv + (j + 1) % nv
    d = i * nv + (j + 1) % nv
    idx = np.stack([np.stack([a, b, c], -1), np.stack([a, c, d], -1)], 2).reshape(-1, 3)
    return pos, nrm, idx.astype(np.int32)


def median_bvh(lo, hi):
    """A BVH in the reference's node format (preorder, root at 0; interior: left child index, right child index;
    leaf: triangle index, LEAF) over boxes lo/hi (T, 3) float32: every node splits its triangles in half at the median
    centroid along the longest axis of their centroids, so the tree has ceil(log2 T) interior levels.  Boxes are the
    exact float32 unions of the triangles' boxes.  Returns a NODE_DTYPE array of 2T - 1 nodes."""
    n = lo.shape[0]
    cen = (lo.astype(np.float64) + hi.astype(np.float64)) * 0.5
    order = np.arange(n)
    nodes = np.zeros(2 * n - 1, NODE_DTYPE)
    node_start, node_size = np.zeros(2 * n - 1, np.int64), np.zeros(2 * n - 1, np.int64)
    start, size, node = np.array([0]), np.array([n]), np.array([0])
    while start.size:
        node_start[node], node_size[node] = start, size
        inner = size > 1
        start, size, node = start[inner], size[inner], node[inner]
        if not start.size:
            break
        # the elements of every segment, segment by segment
        seg = np.repeat(np.arange(start.size), size)
        at = np.repeat(start - np.concatenate([[0], np.cumsum(size)[:-1]]), size) + np.arange(seg.size)
        c = cen[order[at]]
        ext = _segment_reduce(np.maximum, c, size) - _segment_reduce(np.minimum, c, size)
        axis = np.argmax(ext, 1)
        key = c[np.arange(seg.size), axis[seg]]
        order[at] = order[at][np.lexsort((key, seg))]
        half = size // 2
        nodes["left"][node] = node + 1
        nodes["right_leaf"][node] = node + 2 * half
        start, size, node = np.concatenate([start, start + half]), np.concatenate([half, size - half]), \
            np.concatenate([node + 1, node + 2 * half])
    leaf = node_size == 1
    nodes["left"][leaf] = order[node_start[leaf]]
    nodes["right_leaf"][leaf] = LEAF
    slo, shi = lo[order], hi[order]
    nodes["lower"] = _range_reduce(np.minimum, slo, node_start, node_size)
    nodes["upper"] = _range_reduce(np.maximum, shi, node_start, node_size)
    return nodes


def _segment_reduce(op, a, sizes):
    """op.reduce of a's consecutive segments of the given sizes (all > 0)."""
    return op.reduceat(a, np.concatenate([[0], np.cumsum(sizes)[:-1]]), axis=0)


def _range_reduce(op, a, starts, sizes):
    """op.reduce of a[s:s + k] for every (s, k), k > 0."""
    pad = np.concatenate([a, a[-1:]])
    pairs = np.stack([starts, starts + sizes], 1).reshape(-1)
    return op.reduceat(pad, pairs, axis=0)[0::2]


def tree_levels(nodes):
    """Interior levels of a NODE_DTYPE tree (root at 0)."""
    leaf = (nodes["right_leaf"] >> 31) != 0
    frontier, levels = np.array([0]), -1
    while frontier.size:
        levels += 1
        f = frontier[~leaf[frontier]]
        frontier = np.concatenate([nodes["left"][f], nodes["right_leaf"][f]]).astype(np.int64)
    return levels


def area_cdf(pos, idx):
    """Mesh::RebuildCDF as fuzzscene.MeshData computes it: float32 triangle areas, their sequential float32 running
    sum (np.cumsum adds in order), divided by the total.  Returns (cdf, total area, areas)."""
    tri = pos[idx]
    e1, e2 = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    areas = (np.float32(0.5) * np.linalg.norm(np.cross(e1, e2), axis=1)).astype(np.float32)
    run = np.cumsum(areas, dtype=np.float32)
    return (run / run[-1]).astype(np.float32), float(run[-1]), areas


class BigMesh:
    """A mesh for fuzzscene.make_scene_struct (its `struct()` and `radius`), with the BVH of median_bvh."""

    def __init__(self, pos, nrm, idx):
        self.pos = np.ascontiguousarray(pos, np.float32)
        self.nrm = np.ascontiguousarray(nrm, np.float32)
        self.idx = np.ascontiguousarray(idx, np.int32)
        tri = self.pos[self.idx]
        self.nodes = median_bvh(tri.min(1), tri.max(1))
        self.cdf, self.area, self.areas = area_cdf(self.pos, self.idx)

    @property
    def radius(self):
        return float(np.linalg.norm(self.pos, axis=1).max())

    def struct(self):
        m = abi.Mesh()
        m.positions = self.pos.ctypes.data_as(abi.c_float_p)
        m.normals = self.nrm.ctypes.data_as(abi.c_float_p)
        m.indices = self.idx.ctypes.data_as(abi.c_int_p)
        m.nodes = self.nodes.ctypes.data_as(C.POINTER(abi.BvhNode))
        m.cdf = self.cdf.ctypes.data_as(abi.c_float_p)
        m.numVertices, m.numIndices, m.numNodes = len(self.pos), self.idx.size, len(self.nodes)
        m.area = self.area
        return m, self


def _diffuse(rng):
    m = fuzzscene._material(rng, False)
    m.transmission = 0.0
    return m


def ajax_like(path):
    """Writes ajax_like to `path`; returns a dict of its facts (the mesh is under "mesh")."""
    t0 = time.perf_counter()
    rng = np.random.RandomState(2024)
    mesh = BigMesh(*torus(*AJAX_GRID, 0.75, 0.3, 0.08))
    P = (abi.Primitive * 4)()
    bounds = [fuzzscene._floor(P[0], rng)]
    P[1].material = _diffuse(rng)
    tilt = (np.sin(np.pi / 6), 0.0, 0.0, np.cos(np.pi / 6))     # 60 degrees about x: the ring faces the camera
    bounds.append(fuzzscene._instance(P[1], 0, mesh, (-0.9, 1.1, 0.0), tilt, 1.0))
    light = abi.Material.default()
    light.emission[:] = [1.5, 1.3, 1.0]
    light.color[:] = [0.0, 0.0, 0.0]
    light.specular = 0.0
    P[2].material = light
    P[2].lightSamples = 1
    q = np.array([0.3, 0.5, -0.2, 0.8])
    bounds.append(fuzzscene._instance(P[2], 0, mesh, (1.1, 1.1, -0.6), q / np.linalg.norm(q), 0.7))
    bounds.append(fuzzscene._sphere(P[3], (0.0, 3.2, 1.5), 0.3, fuzzscene._material(rng, True), 1))
    fuzzscene._save(rng, path, P, fuzzscene._build_bvh(bounds), [mesh], 1024, 1024, camera=(0.0, 1.3, 5.0), max_depth=5)
    return dict(tris=len(mesh.idx), levels=tree_levels(mesh.nodes), mesh=mesh, seconds=time.perf_counter() - t0)


def probe_image(width=PROBE_SIZE[0], height=PROBE_SIZE[1]):
    """The env_like probe, (height, width, 4) float32 (row 0 is the zenith, as ProbeUVToDir maps it)."""
    v = (np.arange(height) + 0.5) / height
    phi = (np.arange(width) + 0.5) / width * 2.0 * np.pi
    up = np.clip(np.cos(v * np.pi), 0.0, 1.0)[:, None, None]
    zenith, horizon = np.array([0.15, 0.3, 0.8]), np.array([0.7, 0.75, 0.8])
    img = np.zeros((height, width, 4), np.float32)
    img[..., :3] = np.broadcast_to(horizon + (zenith - horizon) * np.sqrt(up), (height, width, 3))
    # mountains: each column is black below its horizon row, so the rows they cross hold runs of black texels
    ridge = 0.5 - 0.06 * np.abs(np.sin(3.0 * phi) * np.cos(7.0 * phi)) - 0.01 * (np.sin(41.0 * phi) > 0.3)
    img[v[:, None] > ridge[None, :], :3] = 0.0
    img[v >= 0.52, :3] = 0.0                                      # black ground rows
    rows, cols = np.ogrid[:height, :width]
    sun = (rows - 360) ** 2 + (cols - 2600) ** 2 <= 25            # a small disc, about 10^4 times the sky
    img[sun, :3] = np.float32(6.0e3)
    img[600:660, 900:1400, :3] = np.float32([0.7, 0.5, 0.3])      # a block of identical texels
    img[820, 333, :3] = np.float32(2.0e5)                         # one isolated hot texel
    return img


def env_like(path):
    """Writes env_like to `path`; returns a dict of its facts (the probe image is under "probe")."""
    t0 = time.perf_counter()
    rng = np.random.RandomState(2025)
    mesh = BigMesh(*torus(*ENV_GRID, 0.8, 0.35, 0.1))
    probe = probe_image()
    P = (abi.Primitive * 2)()
    bounds = [fuzzscene._floor(P[0], rng)]
    glass = abi.Material.default()
    glass.color[:] = [1.0, 1.0, 1.0]
    glass.transmission, glass.eta, glass.roughness = 1.0, 1.5, 0.02
    glass.absorption[:] = [0.6, 0.2, 0.05]
    P[1].material = glass
    q = np.array([0.4, 0.1, 0.2, 0.9])
    bounds.append(fuzzscene._instance(P[1], 0, mesh, (0.0, 1.3, 0.0), q / np.linalg.norm(q), 1.0))
    fuzzscene._save(rng, path, P, fuzzscene._build_bvh(bounds), [mesh], 2048, 2048, probe=probe, camera=(0.0, 1.2, 5.0),
                    max_depth=6)
    return dict(tris=len(mesh.idx), levels=tree_levels(mesh.nodes), probe=probe, mesh=mesh,
                seconds=time.perf_counter() - t0)


def build_cdf(probe):
    """Probe::BuildCDF (src/probe.h:31-79) in numpy, in the reference's float32 operation order: the luminance
    weight (r * 0.3 + g * 0.6) + b * 0.1, each row's sequential running sum, then pdf and cdf times 1 / the row total
    (0 * inf: NaN in a black row), the row totals' running sum divided by its total.  Returns pdfX, cdfX (H, W),
    pdfY, cdfY (H,) float32."""
    f = np.float32
    c = probe[..., :3].astype(np.float32)
    w = (c[..., 0] * f(0.3) + c[..., 1] * f(0.6)) + c[..., 2] * f(0.1)
    run = np.cumsum(w, axis=1, dtype=np.float32)
    total = run[:, -1]
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = f(1.0) / total
        pdf_x, cdf_x = w * inv[:, None], run * inv[:, None]
    run_y = np.cumsum(total, dtype=np.float32)
    return pdf_x, cdf_x, total / run_y[-1], run_y / run_y[-1]


def probe_tables(sky):
    """pdfX, cdfX (H, W), pdfY, cdfY (H,) of a tb200_sky as the snapshot built them, and the slack elements past
    each (cdfX, pdfX, cdfY, pdfY)."""
    W, H = sky.probeWidth, sky.probeHeight
    arr = [np.ctypeslib.as_array(p, (n + 1,)).copy() for p, n in
           ((sky.pdfValuesX, W * H), (sky.cdfValuesX, W * H), (sky.pdfValuesY, H), (sky.cdfValuesY, H))]
    return (arr[0][:-1].reshape(H, W), arr[1][:-1].reshape(H, W), arr[2][:-1], arr[3][:-1],
            np.array([a[-1] for a in arr], np.float32))


def equal_runs(cdf_x):
    """Pairs of equal neighbours in the rows of cdfX that are not NaN (the steps a black texel adds nothing at)."""
    ok = ~np.isnan(cdf_x).any(1)
    return int((cdf_x[ok, 1:] == cdf_x[ok, :-1]).sum())
