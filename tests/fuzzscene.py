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


def _save(rng, path, prims, tree, meshes, width, height, probe=None, camera=None, max_depth=None, shutter=(0.0, 1.0)):
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
    cam.shutterStart, cam.shutterEnd = shutter
    if camera is not None:
        cam.position[:] = camera
    opt.width, opt.height = width, height
    opt.maxDepth = int(rng.randint(2, 6))
    if max_depth is not None:
        opt.maxDepth = max_depth
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


def _instance(p, mesh_index, mesh, pos, q, s, end_pos=None, end_s=None, end_q=None):
    p.type = abi.MESH
    p.mesh = mesh_index
    _xf(p.start, pos, q, s)
    _xf(p.end, pos if end_pos is None else end_pos, q if end_q is None else end_q, s if end_s is None else end_s)
    r = mesh.radius * max(s, s if end_s is None else end_s) * 1.001 + 1e-4
    e = pos if end_pos is None else end_pos
    return (np.minimum(pos, e).astype(np.float32) - np.float32(r), np.maximum(pos, e).astype(np.float32) + np.float32(r))


def _sphere(p, pos, radius, material, light_samples=0, q=(0, 0, 0, 1), end_q=None, end_pos=None):
    p.type = abi.SPHERE
    p.radius = float(radius)
    p.mesh = -1
    e = pos if end_pos is None else end_pos
    _xf(p.start, pos, q, 1.0)
    _xf(p.end, e, q if end_q is None else end_q, 1.0)
    p.material = material
    p.lightSamples = light_samples
    r = float(radius) * 1.001 + 1e-4
    return (np.minimum(pos, e).astype(np.float32) - np.float32(r), np.maximum(pos, e).astype(np.float32) + np.float32(r))


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


FAMILIES = ("instanced", "ties", "many", "big", "probe", "caterpillar", "rotating", "signed_zero")
# rotation pairs of the rotating family, by what the reference's quaternion lerp a + (b - a) t does with them
ROTATIONS = ("random", "antipodal", "near_antipodal", "tiny_lerp", "one_ulp")
SHUTTER = (-0.5, 0.5)      # the camera shutter of the rotating and signed_zero families: half the times are negative


def rotation_pair(rng, kind):
    """(start, end) float32 quaternions of the kind:
      random          two random unit quaternions
      antipodal       q and -q: the lerp is exactly 0 at t = 0.5, where the reference's transform is NaN
      near_antipodal  -q with one component moved by 1e-3 or by 1-8 ulps: a lerp length near 0 at t = 0.5
      tiny_lerp       q with a +0 component k and -q with 2e-21 at k: the lerp at t = 0.5 is 1e-21 in component k and
                      exactly 0 elsewhere, a length below 1e-20 whose normalisation still gives a unit quaternion
      one_ulp         q and q with one component one ulp away: at t = +-FLT_MAX the lerp overflows"""
    q = _quat(rng).astype(np.float32)
    k = int(rng.randint(0, 4))
    if kind == "random":
        return q, _quat(rng).astype(np.float32)
    if kind == "antipodal":
        return q, -q
    e = -q
    if kind == "near_antipodal":
        if rng.uniform() < 0.5:
            e[k] += np.float32(1e-3)
        else:
            for _ in range(int(rng.randint(1, 9))):
                e[k] = np.nextafter(e[k], np.float32(np.inf))
        return q, e
    if kind == "tiny_lerp":
        q[k] = 0.0
        e = -q
        e[k] = np.float32(2e-21)
        return q, e
    assert kind == "one_ulp"
    e = q.copy()
    e[k] = np.nextafter(q[k], np.float32(rng.choice([-np.inf, np.inf])))
    return q, e


def _has_negative_zero(t):
    return any(np.signbit(x) and x == 0.0 for x in list(t.p) + list(t.r) + [t.s])


def is_static(p):
    """Whether the renderer takes primitive p's transform without interpolating it (api.cu: image_from_scene): start and
    end are the same bit for bit and no component of p, r or s is -0."""
    return bytes(p.start) == bytes(p.end) and not _has_negative_zero(p.start)


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
                   `levels` interior levels: the traversal stack fills to levels + 1 entries
      rotating     a mesh instance and a sphere for each kind of rotation_pair, all rotating over the shutter
                   SHUTTER; some instances also move and scale, some are mesh lights, some spheres sphere lights
      signed_zero  static spheres, sphere lights, mesh instances and mesh lights with -0 in their position
                   (on the x = 0 plane) and rotation, each beside a twin written with +0, under SHUTTER"""
    rng = np.random.RandomState(10007 * (FAMILIES.index(family) + 1) + seed)
    prims, bounds, meshes, info = [], [], [], {"family": family, "seed": seed}
    P = (abi.Primitive * 64)()
    camera = None

    def add():
        prims.append(P[len(prims)])
        return prims[-1]

    bounds.append(_floor(add(), rng))
    shutter = (0.0, 1.0)
    if family == "rotating":
        shutter = SHUTTER
        for _ in range(int(rng.randint(1, 3))):
            meshes.append(_random_mesh(rng)[1])
        kinds = []
        for k, kind in enumerate(ROTATIONS):
            qa, qb = rotation_pair(rng, kind)
            mi = int(rng.randint(0, len(meshes)))
            q = add()
            light = (k + seed) % 2 == 0
            q.material = _material(rng, light)
            q.lightSamples = int(rng.randint(1, 3)) if light else 0
            pos = rng.uniform(-2.0, 2.0, 3) * (1, 0.4, 1) + (0, 1.0, 0)
            s = float(rng.uniform(0.3, 0.8))
            end = pos + rng.uniform(-0.3, 0.3, 3) if rng.uniform() < 0.5 else None
            end_s = s * float(rng.uniform(0.7, 1.3)) if rng.uniform() < 0.5 else None
            bounds.append(_instance(q, mi, meshes[mi], pos, qa, s, end, end_s, qb))
            qa, qb = rotation_pair(rng, kind)
            light = (k + seed) % 2 == 1
            pos = rng.uniform(-2.5, 2.5, 3) * (1, 0.5, 1) + (0, 1.5 if light else 0.8, 0)
            end = pos + rng.uniform(-0.3, 0.3, 3) if rng.uniform() < 0.5 else None
            bounds.append(_sphere(add(), pos, rng.uniform(0.1, 0.4), _material(rng, light), int(rng.randint(1, 3)) if light else 0,
                                  qa, qb, end))
            kinds += [kind, kind]
        info["rotations"] = kinds
    elif family == "signed_zero":
        shutter = SHUTTER
        p, n, f = _grid(2)                       # normals (0, 0, 1): rotations of exact zeros
        meshes.append(MeshData(p, n, f))
        meshes.append(_random_mesh(rng)[1])
        rots = [(-0.0, 0.0, 0.0, 1.0), (0.0, -0.0, 0.0, 1.0), (0.0, 0.0, -0.0, 1.0), (-0.0, -0.0, -0.0, 1.0), (-0.0, 0.6, 0.0, 0.8),
                (0.0, -0.0, 0.6, 0.8)]
        for k, kind in enumerate(("sphere", "sphere light", "mesh", "mesh light")):
            qz = rots[int(rng.randint(0, len(rots)))]
            y, z = 0.4 + 0.6 * k, float(rng.uniform(-1.5, 0.5))
            light = kind.endswith("light")
            mat = _material(rng, light)
            for twin in (False, True):            # the twin is the same primitive written with +0, 2.2 to the right
                rot = tuple(abs(c) for c in qz) if twin else qz
                pos = (2.2 if twin else -0.0, y, z if k % 2 or twin else -0.0)
                q = add()
                if kind.startswith("mesh"):
                    q.material = mat
                    q.lightSamples = 1 if light else 0
                    bounds.append(_instance(q, k % 2, meshes[k % 2], pos, rot, 0.5))
                else:
                    bounds.append(_sphere(q, pos, 0.3, mat, 1 if light else 0, rot))
    elif family == "caterpillar":
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
    opt = _save(rng, path, arr, tree, meshes, width, height, probe=probe, camera=camera, shutter=shutter)
    info.update(prims=len(prims), meshes=len(meshes), tris=[len(m.idx) for m in meshes], maxDepth=opt.maxDepth,
                moving_scale=sum(1 for q in prims if q.type == abi.MESH and q.start.s != q.end.s),
                mesh_lights=sum(1 for q in prims if q.type == abi.MESH and q.lightSamples > 0),
                zero_area=sum(m.zero_area for m in meshes), probe=probe is not None,
                rotating=[i for i, q in enumerate(prims) if bytes(q.start)[12:28] != bytes(q.end)[12:28]],
                negative_zero=[i for i, q in enumerate(prims) if _has_negative_zero(q.start) or _has_negative_zero(q.end)],
                static=[i for i, q in enumerate(prims) if is_static(q)], shutter=shutter)
    return info


# ---- the limits tb200_create accepts -------------------------------------------------------------

MAX_PRIMS = 4095            # TB200_MAX_PRIMITIVES
MAX_LIGHT_SAMPLES = 4095    # TB200_MAX_LIGHT_SAMPLES
LIMIT_CASES = ("prims40", "prims41", "prims42", "prims600", "prims4095", "nee255", "nee256", "nee257", "nee300",
               "nee300_odd", "probe255", "meshlight300")


def _wall(p, rng):
    """A plane at z = -3 behind everything: with the floor, every camera ray hits a surface."""
    p.type = abi.PLANE
    p.plane[:] = [0.0, 0.0, 1.0, 3.0]
    _xf(p.start, (0, 0, 0), (0, 0, 0, 1), 1.0)
    _xf(p.end, (0, 0, 0), (0, 0, 0, 1), 1.0)
    p.mesh = -1
    p.material = _material(rng, False)
    p.material.transmission = 0.0
    return (np.full(3, -1.0e8, np.float32), np.full(3, 1.0e8, np.float32))


def nee_order(light_samples):
    """(primitive, sample) of every shadow ray a surface hit draws, in order, after the probe sample if there is one."""
    return [(i, k) for i, n in enumerate(light_samples) for k in range(n)]


def make_limit_scene(case, path, width=48, height=32):
    """Writes one of LIMIT_CASES to `path` and returns a dict describing what it holds.  Floor and back wall
    first (every camera ray hits a surface, and every surface hit draws all numNee shadow rays), then:
      prims40/41/42  spheres, about a quarter of them lights with 1-2 samples: 40 primitives stage their
                     records and the 39 BVH pairs on chip, 41 stage the 40 pairs only, 42 neither
      prims600       lights at even and odd indices with 1-12 samples each; the 256th shadow ray is a sample
                     of a light at an even index that is not that light's last one
      prims4095      the most primitives tb200_create accepts; the last one is a light with the most lightSamples
                     it accepts
      neeN           8 primitives, one sphere light with N samples at index 2
      nee300_odd     the light at index 3
      probe255       an HDR probe (no black rows) and a 255-sample light at index 3: 256 shadow rays per hit
      meshlight300   an icosphere mesh light at index 2 with 300 samples"""
    rng = np.random.RandomState(7919 * (LIMIT_CASES.index(case) + 1))
    counts = {"prims40": 40, "prims41": 41, "prims42": 42, "prims600": 600, "prims4095": MAX_PRIMS}
    n = counts.get(case, 8)
    P = (abi.Primitive * n)()
    bounds = [_floor(P[0], rng), _wall(P[1], rng)]
    meshes, probe, max_depth = [], None, None
    if case in counts:
        r_lo, r_hi = {40: (0.15, 0.35), 41: (0.15, 0.35), 42: (0.15, 0.35), 600: (0.05, 0.14), MAX_PRIMS: (0.02, 0.05)}[n]
        if case == "prims600":
            while True:       # lights at random indices until the 256th shadow ray falls inside an even-index light
                lights = set(int(i) for i in rng.choice(np.arange(2, n), 60, replace=False))
                samples = [int(rng.randint(1, 13)) if i in lights else 0 for i in range(n)]
                prim, k = nee_order(samples)[255]
                if prim % 2 == 0 and k + 1 < samples[prim] and any(i % 2 for i in lights) and max(lights) > prim:
                    break
        elif case == "prims4095":
            samples = [0] * n
            samples[n - 1] = MAX_LIGHT_SAMPLES
            max_depth = 2
        else:
            samples = [int(rng.randint(1, 3)) if rng.uniform() < 0.25 else 0 for i in range(n)]
            samples[0] = samples[1] = 0
            samples[2] = max(samples[2], 1)
        for i in range(2, n):
            light = samples[i] > 0
            if case == "prims4095" and light:
                bounds.append(_sphere(P[i], (0.0, 3.2, 1.0), 0.3, _material(rng, True), samples[i]))
                continue
            pos = rng.uniform(-2.8, 2.8, 3) * (1, 0.4, 1) + (0, 2.5 if light else 1.0, -0.2)
            bounds.append(_sphere(P[i], pos, rng.uniform(r_lo, r_hi), _material(rng, light), samples[i]))
    else:
        spp = int("".join(ch for ch in case if ch.isdigit()))
        at = 3 if case in ("nee300_odd", "probe255") else 2
        samples = [0] * n
        samples[at] = spp
        if case == "meshlight300":
            p, nrm, f = _icosphere(2)
            meshes.append(MeshData(p, nrm, f))
        for i in range(2, n):
            if i == at and meshes:
                P[i].material = _material(rng, True)
                P[i].lightSamples = spp
                bounds.append(_instance(P[i], 0, meshes[0], (0.3, 2.6, 0.5), _quat(rng), 0.35))
            elif i == at:
                bounds.append(_sphere(P[i], (0.3, 2.6, 0.5), 0.3, _material(rng, True), spp))
            else:
                pos = rng.uniform(-1.8, 1.8, 3) * (1, 0.3, 1) + (0, 0.8, 0)
                bounds.append(_sphere(P[i], pos, rng.uniform(0.25, 0.5), _material(rng, False)))
        if case == "probe255":
            probe = _probe(rng)
            probe[..., :3] = np.maximum(probe[..., :3], np.float32(0.05))     # black rows would give NaN samples
    opt = _save(rng, path, P, _build_bvh(bounds), meshes, width, height, probe=probe, max_depth=max_depth)
    samples = [int(q.lightSamples) for q in P]
    lights = [i for i, s in enumerate(samples) if s > 0]
    order = [(-1, 0)] * int(probe is not None) + nee_order(samples)      # (-1, 0): the probe sample
    info = {"case": case, "prims": n, "meshes": len(meshes), "tris": [len(m.idx) for m in meshes], "probe": probe is not None,
            "lights": lights, "light_samples": {i: samples[i] for i in lights}, "maxDepth": opt.maxDepth,
            "numNee": len(order), "lightBegin": lights[0], "lightEnd": lights[-1] + 1}
    if len(order) >= 256:
        info["ray256"] = order[255]       # (primitive, sample) of the 256th shadow ray
    return info
