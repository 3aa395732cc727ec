"""Random small scenes (planes, static and moving spheres, sphere lights, the whole Disney parameter
space, gradient sky) written as .tsnap snapshots, for the fuzz parity tests: the same file is loaded
into a reference `Scene` (oracle/_ref), the CPU restatement and the CUDA renderer.  The scene-level
BVH is a median-split tree built here; any valid BVH gives the three implementations the same walk.
make_mesh_scene adds triangle meshes: instancing, degenerate triangles, exact ties, big meshes, an HDR probe
and caterpillar BVHs that fill the traversal stack."""
import ctypes as C

import numpy as np

import tinsel_b200 as tb
from tinsel_b200 import abi

LEAF = 1 << 31


def _material(rng, light):
    m = abi.Material.default()
    if light:
        e = float(rng.uniform(4.0, 40.0))
        m.emission[:] = [e, e * float(rng.uniform(0.6, 1.0)), e * float(rng.uniform(0.4, 1.0))]
        m.color[:] = [0.0, 0.0, 0.0]
        m.specular = 0.0
        return m
    m.color[:] = [float(x) for x in rng.uniform(0.05, 1.0, 3)]
    m.metallic = float(rng.choice([0.0, 1.0, rng.uniform()]))
    m.subsurface = float(rng.choice([0.0, rng.uniform()]))
    m.specular = float(rng.uniform())
    m.roughness = float(rng.uniform(0.02, 1.0))
    m.specularTint = float(rng.uniform())
    m.sheen = float(rng.choice([0.0, rng.uniform()]))
    m.sheenTint = float(rng.uniform())
    m.clearcoat = float(rng.choice([0.0, rng.uniform()]))
    m.clearcoatGloss = float(rng.uniform())
    m.transmission = float(rng.choice([0.0, 0.0, rng.uniform(), 1.0]))
    if m.transmission > 0.0:
        m.eta = float(rng.uniform(1.1, 1.9))
        m.absorption[:] = [float(x) for x in rng.choice([0.0, 1.0]) * rng.uniform(0.0, 2.0, 3)]
    return m


def _xf(t, p, q, s):
    t.p[:] = [float(x) for x in p]
    t.r[:] = [float(x) for x in q]
    t.s = float(s)


def _build_bvh(bounds):
    """Median split over the x centre; preorder array of (lower, upper, left, right_leaf)."""
    nodes = []

    def rec(items):
        me = len(nodes)
        nodes.append(None)
        lo = np.min([bounds[i][0] for i in items], axis=0)
        hi = np.max([bounds[i][1] for i in items], axis=0)
        if len(items) == 1:
            nodes[me] = (lo, hi, items[0], LEAF)
            return me
        items = sorted(items, key=lambda i: float(bounds[i][0][0] + bounds[i][1][0]))
        half = len(items) // 2
        left = rec(items[:half])
        right = rec(items[half:])
        nodes[me] = (lo, hi, left, right)
        return me

    rec(list(range(len(bounds))))
    return nodes


def make_scene(seed, path, width=40, height=30):
    """Writes a random scene to `path` (a .tsnap) and returns a short description."""
    rng = np.random.RandomState(seed)
    nspheres = int(rng.randint(3, 7))
    nlights = int(rng.randint(1, 3))
    nplanes = int(rng.randint(1, 3))
    n = nplanes + nspheres + nlights
    prims = (abi.Primitive * n)()
    bounds = []
    k = 0
    for i in range(nplanes):
        p = prims[k]
        p.type = abi.PLANE
        p.plane[:] = [0.0, 1.0, 0.0, 0.0] if i == 0 else [0.0, 0.0, 1.0, 3.0]
        _xf(p.start, (0, 0, 0), (0, 0, 0, 1), 1.0)
        _xf(p.end, (0, 0, 0), (0, 0, 0, 1), 1.0)
        p.mesh = -1
        p.material = _material(rng, False)
        p.material.transmission = 0.0
        bounds.append((np.full(3, -1.0e8, np.float32), np.full(3, 1.0e8, np.float32)))   # PrimitiveBounds, intersection.h:919-924
        k += 1
    for i in range(nspheres + nlights):
        light = i >= nspheres
        p = prims[k]
        p.type = abi.SPHERE
        p.radius = float(rng.uniform(0.2, 0.7)) if not light else float(rng.uniform(0.15, 0.4))
        pos = np.array([rng.uniform(-2.2, 2.2), rng.uniform(0.3, 1.8) if not light else rng.uniform(2.0, 3.5), rng.uniform(-2.0, 1.5)])
        q = rng.normal(size=4)
        q = q / np.linalg.norm(q) if rng.uniform() < 0.5 else np.array([0.0, 0.0, 0.0, 1.0])
        s = float(rng.choice([1.0, rng.uniform(0.6, 1.5)]))
        end = pos + (rng.uniform(-0.4, 0.4, 3) if (rng.uniform() < 0.3 and not light) else 0.0)
        _xf(p.start, pos, q, s)
        _xf(p.end, end, q, s)
        p.mesh = -1
        p.material = _material(rng, light)
        p.lightSamples = int(rng.randint(1, 3)) if light else 0
        r = p.radius * s * 1.001 + 1e-4
        bounds.append((np.minimum(pos, end).astype(np.float32) - np.float32(r), np.maximum(pos, end).astype(np.float32) + np.float32(r)))
        k += 1
    opt = _save(rng, path, prims, _build_bvh(bounds), [], width, height)
    return "seed %d: %d planes, %d spheres, %d lights, maxDepth %d" % (seed, nplanes, nspheres, nlights, opt.maxDepth)


def _nodes(tree):
    nodes = (abi.BvhNode * len(tree))()
    for i, (lo, hi, left, right) in enumerate(tree):
        nodes[i].lower[:] = [float(x) for x in lo]
        nodes[i].upper[:] = [float(x) for x in hi]
        nodes[i].left = int(left)
        nodes[i].right_leaf = int(right)
    return nodes


def _save(rng, path, prims, tree, meshes, width, height, probe=None, camera=None):
    """Sky, camera and options drawn from `rng`, then the snapshot.  meshes: list of MeshData."""
    scene, keep = make_scene_struct(prims, tree, meshes)
    scene.sky.horizon[:] = [float(x) for x in rng.uniform(0.0, 1.0, 3)]
    scene.sky.zenith[:] = [float(x) for x in rng.uniform(0.0, 1.0, 3)]
    if probe is not None:
        scene.sky.probeValid = 1
        scene.sky.probeHeight, scene.sky.probeWidth = probe.shape[:2]
        scene.sky.probeData = probe.ctypes.data_as(abi.c_float_p)
    base = tb.Snapshot(tb.scene_path("cornell"))
    cam, opt = abi.copy_struct(base.camera), abi.copy_struct(base.options)
    base.close()
    cam.position[:] = [0.0, 1.2, 6.0]
    cam.rotation[:] = [0.0, 0.0, 0.0, 1.0]
    cam.fov = float(np.radians(rng.uniform(35.0, 60.0))) if cam.fov < 3.2 else float(rng.uniform(35.0, 60.0))
    cam.shutterStart, cam.shutterEnd = 0.0, 1.0
    if camera is not None:
        cam.position[:] = camera
    opt.width, opt.height = width, height
    opt.maxDepth = int(rng.randint(2, 6))
    opt.filterType, opt.filterWidth, opt.filterFalloff, opt.filterOffset = abi.FILTER_GAUSSIAN, 0.75, 1.0, 0.5697828531265259
    if tb.load_library().tb200_snapshot_save(str(path).encode(), C.byref(scene), C.byref(cam), C.byref(opt)) != 0:
        raise RuntimeError(tb.last_error())
    return opt


def make_scene_struct(prims, tree, meshes):
    """A tb200_scene over `prims` (a ctypes array), a scene BVH `tree` (_build_bvh / _chain_bvh format) and
    MeshData `meshes`; returns (scene, keepalive)."""
    nodes = _nodes(tree)
    arr = (abi.Mesh * max(1, len(meshes)))()
    keep = [prims, nodes, arr]
    for i, m in enumerate(meshes):
        arr[i], k = m.struct()
        keep.append(k)
    scene = abi.Scene()
    scene.primitives = C.cast(prims, C.POINTER(abi.Primitive))
    scene.numPrimitives = len(prims)
    scene.meshes = C.cast(arr, C.POINTER(abi.Mesh))
    scene.numMeshes = len(meshes)
    scene.bvhNodes = C.cast(nodes, C.POINTER(abi.BvhNode))
    scene.numBvhNodes = len(tree)
    return scene, keep


# ---- meshes ------------------------------------------------------------------------------------------

def _chain_bvh(bounds):
    """A caterpillar: interior node k has item k as one child and the subtree over items k+1.. as the other, so
    len(bounds) items give len(bounds) - 1 interior levels.  With the items ordered far to near along the ray,
    the ray hits both children at every level and near-first traversal leaves one far leaf pending per level:
    the stack holds levels + 1 entries at the bottom."""
    n = len(bounds)
    nodes = []
    for k in range(n - 1):
        lo = np.min([b[0] for b in bounds[k:]], axis=0)
        hi = np.max([b[1] for b in bounds[k:]], axis=0)
        last = k == n - 2
        me = len(nodes)
        # children: leaf of item k at me + 1, the rest at me + 2 (an interior node, or the last item's leaf)
        nodes.append((lo, hi, me + 1, me + 2))
        nodes.append((bounds[k][0], bounds[k][1], k, LEAF))
        if last:
            nodes.append((bounds[k + 1][0], bounds[k + 1][1], k + 1, LEAF))
    if n == 1:
        nodes.append((bounds[0][0], bounds[0][1], 0, LEAF))
    return nodes


def tree_levels(tree):
    """Interior levels of a _build_bvh / _chain_bvh tree (node 0 is the root)."""
    def rec(i):
        lo, hi, left, right = tree[i]
        return 0 if right == LEAF else 1 + max(rec(left), rec(right))
    return rec(0)


class MeshData:
    """float32 positions / normals (V,3), int32 indices (T,3), a BVH over the triangles, the area CDF."""

    def __init__(self, pos, nrm, idx, bvh="median"):
        self.pos = np.ascontiguousarray(pos, np.float32)
        self.nrm = np.ascontiguousarray(nrm, np.float32)
        self.idx = np.ascontiguousarray(idx, np.int32)
        tri = self.pos[self.idx]                                        # (T, 3, 3)
        self.tri_bounds = [(t.min(0), t.max(0)) for t in tri]
        self.tree = _chain_bvh(self.tri_bounds) if bvh == "chain" else _build_bvh(self.tri_bounds)
        # Mesh::RebuildCDF: per-triangle areas summed in float, the running sums divided by the total
        e1, e2 = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
        areas = (np.float32(0.5) * np.linalg.norm(np.cross(e1, e2), axis=1)).astype(np.float32)
        run = np.zeros(len(areas), np.float32)
        total = np.float32(0.0)
        for i, a in enumerate(areas):
            total = np.float32(total + a)
            run[i] = total
        self.area = float(total)
        self.cdf = (run / total).astype(np.float32) if total > 0 else run
        self.zero_area = int((areas == 0).sum())

    @property
    def radius(self):
        return float(np.linalg.norm(self.pos, axis=1).max())

    def struct(self):
        m = abi.Mesh()
        nodes = _nodes(self.tree)
        m.positions = self.pos.ctypes.data_as(abi.c_float_p)
        m.normals = self.nrm.ctypes.data_as(abi.c_float_p)
        m.indices = self.idx.ctypes.data_as(abi.c_int_p)
        m.nodes = C.cast(nodes, C.POINTER(abi.BvhNode))
        m.cdf = self.cdf.ctypes.data_as(abi.c_float_p)
        m.numVertices, m.numIndices, m.numNodes = len(self.pos), self.idx.size, len(self.tree)
        m.area = self.area
        return m, (self, nodes)


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _icosphere(sub, rng=None, bump=0.0):
    t = (1.0 + 5.0 ** 0.5) / 2.0
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
         (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    verts = [np.array(x, np.float64) / np.linalg.norm(x) for x in v]
    for _ in range(sub):
        mid = {}
        nf = []

        def m(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                verts.append(_unit(verts[a] + verts[b]))
                mid[key] = len(verts) - 1
            return mid[key]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    p = np.array(verts)
    if bump:
        p = p * (1.0 + bump * rng.uniform(-1.0, 1.0, (len(p), 1)))
    return p, _unit(np.array(verts)), np.array(f)


def _box():
    p = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64) * 0.8
    f = [(0, 1, 3), (0, 3, 2), (4, 6, 7), (4, 7, 5), (0, 4, 5), (0, 5, 1), (2, 3, 7), (2, 7, 6), (0, 2, 6), (0, 6, 4), (1, 5, 7), (1, 7, 3)]
    return p, _unit(p), np.array(f)


def _grid(n):
    """An axis-aligned n x n quad grid in the z = 0 plane: every box has zero z extent, vertices are shared."""
    s = np.linspace(-1.0, 1.0, n + 1)
    p = np.array([[x, y, 0.0] for y in s for x in s])
    f = []
    for j in range(n):
        for i in range(n):
            a = j * (n + 1) + i
            f += [(a, a + 1, a + n + 2), (a, a + n + 2, a + n + 1)]
    return p, np.tile([0.0, 0.0, 1.0], (len(p), 1)), np.array(f)


def _soup(rng, n):
    c = rng.uniform(-0.7, 0.7, (n, 1, 3))
    p = (c + rng.uniform(-0.4, 0.4, (n, 3, 3))).reshape(-1, 3)
    return p, _unit(rng.normal(size=(3 * n, 3))), np.arange(3 * n).reshape(n, 3)


def _with_degenerates(rng, p, nrm, f):
    """Adds a sliver, two zero-area triangles (a repeated vertex; three collinear points) and a duplicate of
    an existing triangle on new vertices with the same positions but different normals."""
    p, nrm, f = list(p), list(nrm), [tuple(x) for x in f]
    base, src = len(p), f[int(rng.randint(0, len(f)))]
    a = rng.uniform(-0.6, 0.6, 3)
    d = _unit(rng.normal(size=3))
    p += [a, a + d, a + d * 0.5 + _unit(rng.normal(size=3)) * 1e-4,      # sliver
          a + 0.1, a + 0.1 + d * 0.3, a + 0.1 + d * 0.6]                 # collinear
    nrm += [_unit(rng.normal(size=3)) for _ in range(6)]
    f += [(base, base + 1, base + 2), (base, base, base + 1), (base + 3, base + 4, base + 5)]
    k = len(p)
    p += [p[i] for i in src]
    nrm += [-np.asarray(nrm[i]) + _unit(rng.normal(size=3)) * 0.3 for i in src]
    f.append((k, k + 1, k + 2))
    return np.array(p), _unit(np.array(nrm)), np.array(f)


def _random_mesh(rng):
    kind = rng.choice(["soup", "box", "ico", "grid"])
    if kind == "soup":
        p, n, f = _soup(rng, int(rng.randint(4, 40)))
    elif kind == "box":
        p, n, f = _box()
    elif kind == "ico":
        p, n, f = _icosphere(int(rng.randint(1, 3)))
    else:
        p, n, f = _grid(int(rng.randint(2, 6)))
    p, n, f = _with_degenerates(rng, p, n, f)
    return kind, MeshData(p, n, f)


def _quat(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def _instance(p, mesh_index, mesh, pos, q, s, end_pos=None, end_s=None):
    p.type = abi.MESH
    p.mesh = mesh_index
    _xf(p.start, pos, q, s)
    _xf(p.end, pos if end_pos is None else end_pos, q, s if end_s is None else end_s)
    r = mesh.radius * max(s, s if end_s is None else end_s) * 1.001 + 1e-4
    e = pos if end_pos is None else end_pos
    return (np.minimum(pos, e).astype(np.float32) - np.float32(r), np.maximum(pos, e).astype(np.float32) + np.float32(r))


def _sphere(p, pos, radius, material, light_samples=0):
    p.type = abi.SPHERE
    p.radius = float(radius)
    p.mesh = -1
    _xf(p.start, pos, (0, 0, 0, 1), 1.0)
    _xf(p.end, pos, (0, 0, 0, 1), 1.0)
    p.material = material
    p.lightSamples = light_samples
    r = float(radius) * 1.001 + 1e-4
    return (np.asarray(pos, np.float32) - np.float32(r), np.asarray(pos, np.float32) + np.float32(r))


def _floor(p, rng):
    p.type = abi.PLANE
    p.plane[:] = [0.0, 1.0, 0.0, 0.0]
    _xf(p.start, (0, 0, 0), (0, 0, 0, 1), 1.0)
    _xf(p.end, (0, 0, 0), (0, 0, 0, 1), 1.0)
    p.mesh = -1
    p.material = _material(rng, False)
    p.material.transmission = 0.0
    return (np.full(3, -1.0e8, np.float32), np.full(3, 1.0e8, np.float32))


def _probe(rng):
    """A small HDR probe: random radiance, a few black rows, one texel far brighter than the rest."""
    h, w = int(rng.randint(6, 17)), int(rng.randint(8, 33))
    img = np.zeros((h, w, 4), np.float32)
    img[..., :3] = np.exp(rng.normal(-1.0, 1.0, (h, w, 3)))
    img[rng.choice(h, size=max(1, h // 4), replace=False)] = 0.0
    img[int(rng.randint(0, h)), int(rng.randint(0, w)), :3] = 5.0e4
    return img


FAMILIES = ("instanced", "ties", "many", "big", "probe", "caterpillar")


def make_mesh_scene(seed, path, family, width=40, height=30, swap_ties=False, levels=None):
    """Writes a random scene with triangle meshes to `path` and returns a dict describing what it holds.
      instanced    1-3 meshes (soups, closed boxes, icospheres, axis-aligned flat grids, each with a sliver,
                   zero-area triangles and a duplicated triangle with other normals), each instanced 1-3 times
                   with rotation, uniform scale and motion (scale too); some are lights (area CDF with flat
                   steps).  Odd seeds: an unrotated axis-aligned grid squarely in front of the camera.
      ties         exact duplicates with different materials: a mesh instanced twice at one transform, a
                   sphere twice, a sphere light on a diffuse sphere (swap_ties swaps each pair's materials)
      many         17-40 primitives: the scene level runs the reference-order walk, not the flat program
      big          one mesh of more than 4096 triangles (a bumpy icosphere): the default heuristics pick the
                   free-running wavefront, 768-thread CTAs, the mesh-split queue and its tuner
      probe        `instanced` lit by a small random HDR probe
      caterpillar  a stack of parallel triangles in front of the camera, nearer ones deeper in a chain BVH of
                   `levels` interior levels: the traversal stack fills to levels + 1 entries"""
    rng = np.random.RandomState(10007 * (FAMILIES.index(family) + 1) + seed)
    prims, bounds, meshes, info = [], [], [], {"family": family, "seed": seed}
    P = (abi.Primitive * 64)()
    camera = None

    def add():
        prims.append(P[len(prims)])
        return prims[-1]

    bounds.append(_floor(add(), rng))
    if family == "caterpillar":
        n = (levels or 30) + 1
        z = -1.0 - 0.05 * np.arange(n)[::-1]                   # item 0 farthest
        p = np.array([[[-3.0, -2.0, zz], [3.0, -2.0, zz], [0.0, 4.0, zz]] for zz in z]).reshape(-1, 3)
        p[:, 1] += 1.2
        nrm = np.tile([0.0, 0.0, 1.0], (len(p), 1))
        m = MeshData(p, nrm, np.arange(3 * n).reshape(n, 3), bvh="chain")
        meshes.append(m)
        mat = _material(rng, False)
        mat.transmission = 1.0                                  # rays go on through the stack
        mat.eta = 1.0
        q = add()
        q.material = mat
        bounds.append(_instance(q, 0, m, (0.0, 0.0, 0.0), (0, 0, 0, 1), 1.0))
        bounds.append(_sphere(add(), (0.0, 3.0, 2.0), 0.3, _material(rng, True), 1))
        info["levels"] = tree_levels(m.tree)
    elif family == "ties":
        kind, m = _random_mesh(rng)
        meshes.append(m)
        mats = [_material(rng, False) for _ in range(4)]
        pos, qq, s = rng.uniform(-1.0, 1.0, 3) + (0, 1.0, 0), _quat(rng), float(rng.uniform(0.5, 0.9))
        for k in range(2):
            q = add()
            q.material = mats[k ^ int(swap_ties)]
            bounds.append(_instance(q, 0, m, pos, qq, s))
        c = rng.uniform(-1.5, 1.5, 3) + (0, 1.2, 0)
        for k in range(2):
            bounds.append(_sphere(add(), c, 0.5, mats[2 + (k ^ int(swap_ties))]))
        c2 = rng.uniform(-1.5, 1.5, 3) + (0, 1.5, -0.5)
        pair = [(_material(rng, True), 1), (_material(rng, False), 0)]
        for k in range(2):
            mat, ls = pair[k ^ int(swap_ties)]
            bounds.append(_sphere(add(), c2, 0.35, mat, ls))
        bounds.append(_sphere(add(), (0.0, 3.5, 1.0), 0.3, _material(rng, True), 1))
        info["ties"] = 3
    else:
        if family == "big":
            p, n, f = _icosphere(4, rng, bump=0.05)
            p, n, f = _with_degenerates(rng, p, n, f)
            meshes.append(MeshData(p, n, f))
        elif family == "instanced" and seed % 2 == 1:
            p, n, f = _grid(4)
            meshes.append(MeshData(p, n, f))
            camera = (0.0, 1.0, 6.0)
        nm = int(rng.randint(1, 4)) if family != "many" else int(rng.randint(2, 4))
        while len(meshes) < nm:
            meshes.append(_random_mesh(rng)[1])
        target = int(rng.randint(17, 41)) if family == "many" else 0
        for mi, m in enumerate(meshes):
            for _ in range(int(rng.randint(1, 4))):
                q = add()
                light = rng.uniform() < 0.25 and m.area > 0
                q.material = _material(rng, light)
                q.lightSamples = int(rng.randint(1, 3)) if light else 0
                if camera is not None and mi == 0 and len(prims) == 2:
                    bounds.append(_instance(q, mi, m, (0.0, 1.0, 0.0), (0, 0, 0, 1), 1.0))   # axis-aligned, unrotated
                    continue
                pos = rng.uniform(-2.0, 2.0, 3) * (1, 0.4, 1) + (0, 1.0, 0)
                s = float(rng.uniform(0.3, 0.8))
                moving = rng.uniform() < 0.4
                end = pos + rng.uniform(-0.3, 0.3, 3) if moving else None
                end_s = s * float(rng.uniform(0.7, 1.3)) if moving or light else None
                bounds.append(_instance(q, mi, m, pos, _quat(rng), s, end, end_s))
        while len(prims) < max(target, 3):
            light = len(prims) == 2 or rng.uniform() < 0.15
            pos = rng.uniform(-2.5, 2.5, 3) * (1, 0.5, 1) + (0, 1.5 if light else 0.8, 0)
            bounds.append(_sphere(add(), pos, rng.uniform(0.1, 0.4), _material(rng, light), int(rng.randint(1, 3)) if light else 0))
        if not any(q.lightSamples > 0 for q in prims):
            bounds.append(_sphere(add(), (0.0, 3.2, 1.0), 0.3, _material(rng, True), 1))
    arr = (abi.Primitive * len(prims))()
    for i, q in enumerate(prims):
        arr[i] = q
    tree = _build_bvh(bounds)
    probe = _probe(rng) if family == "probe" else None
    opt = _save(rng, path, arr, tree, meshes, width, height, probe=probe, camera=camera)
    info.update(prims=len(prims), meshes=len(meshes), tris=[len(m.idx) for m in meshes], maxDepth=opt.maxDepth,
                moving_scale=sum(1 for q in prims if q.type == abi.MESH and q.start.s != q.end.s),
                mesh_lights=sum(1 for q in prims if q.type == abi.MESH and q.lightSamples > 0),
                zero_area=sum(m.zero_area for m in meshes), probe=probe is not None)
    return info
