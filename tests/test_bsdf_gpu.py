"""The Disney BSDF on the device (tb_shade.cuh: bsdf_pdf, bsdf_eval, bsdf_eval_pdf, bsdf_sample_dir, with the
per-material constants of tb_scene.cuh: make_material) against the CPU restatement (oracle_bsdf_eval /
oracle_bsdf_sample) and, where oracle/_ref is built, the reference's own code, one call per case, bit for bit.

tests/bsdf_harness.cu runs one case per thread in both instantiations the kernels use: TB_FEAT_ALL on every case,
TB_FEAT_NONE on the cases whose material scene_features counts as featureless.  Every output must have the
restatement's bits -- f, pdf, the sampled direction, its pdf (taken from bsdf_eval_pdf when bsdf_sample_dir says so,
as path_scatter does), its type and the RNG state after sampling -- with two exceptions:
  * a NaN matches any NaN (payloads are not compared);
  * +0 matches -0 in f where the clearcoat lobe is skipped (TB_MAT_NO_CLEARCOAT) and in a pdf where Fr is skipped
    (TB_MAT_NO_FRESNEL): adding the skipped +-0 term can only change the sign of a zero.  The renderer never observes
    that sign: a pdf is only compared with 0 before it divides anything, and a zero f only reaches the radiance
    through sums that start at +0, which +0 + -0 leaves +0.
The materials take the edge values of every parameter the loader accepts without checking (roughness 0 and 0.001 +-
1 ulp, specular 12.5 and -0.5 whose ior is infinite or NaN, eta 0, negative, infinite or NaN, clearcoat glosses where
the clearcoat alpha is -1, near 0 or of either sign huge, negative colours, subsurface above 1), and the directions the call sites
produce: N face-forwarded towards V (dot(N, V) >= 0), with V at grazing angles, along N and one ulp off unit length,
and L over the whole sphere, along N, perpendicular to it, along the mirror direction and along -V.

The edge-materials scenes at the end trace the same materials per sample through the renderer in every route."""
import ctypes as C
import os

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import cuda_harness
import fuzzscene
import refdrv
import schedenv

F32 = np.float32
INF = F32(np.inf)
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# tb200_material
MAT_DTYPE = np.dtype([("emission", "<f4", 3), ("color", "<f4", 3), ("absorption", "<f4", 3), ("eta", "<f4"),
                      ("metallic", "<f4"), ("subsurface", "<f4"), ("specular", "<f4"), ("roughness", "<f4"),
                      ("specularTint", "<f4"), ("anisotropic", "<f4"), ("sheen", "<f4"), ("sheenTint", "<f4"),
                      ("clearcoat", "<f4"), ("clearcoatGloss", "<f4"), ("transmission", "<f4")])
# struct BsdfCase in bsdf_harness.cu, struct oracle_bsdf_case in oracle/tinsel_oracle.cpp
CASE_DTYPE = np.dtype([("mat", "<i4"), ("seed", "<i4"), ("etaI", "<f4"), ("etaO", "<f4"), ("n", "<f4", 3),
                       ("v", "<f4", 3), ("l", "<f4", 3)])
# struct BsdfOut in bsdf_harness.cu
OUT_DTYPE = np.dtype([("f", "<f4", 3), ("pdf", "<f4"), ("fp", "<f4", 3), ("pdfp", "<f4"), ("light", "<f4", 3),
                      ("spdf", "<f4"), ("type", "<i4"), ("fromBsdf", "<i4"), ("rng", "<u4", 2)])
# struct oracle_bsdf_result in oracle/tinsel_oracle.cpp
REF_DTYPE = np.dtype([("f", "<f4", 3), ("pdf", "<f4"), ("light", "<f4", 3), ("spdf", "<f4"), ("type", "<i4"),
                      ("rng", "<u4", 2)])
assert MAT_DTYPE.itemsize == C.sizeof(abi.Material)

# tb_scene.cuh: TB_MAT_*, TB_FEAT_*
GTR1_WIDE, NO_CLEARCOAT, NO_FRESNEL = 1, 2, 4
FEAT_TRANSMISSION, FEAT_SUBSURFACE, FEAT_CLEARCOAT, FEAT_ABSORPTION = 4, 8, 16, 32

BATCH = 1 << 16
BATCHES = 16          # 2^20 cases
SCENES = BATCH // 4   # materials per batch: scenes of two, each shared by eight cases


def _gloss_near_zero_alpha():
    """The float glosses around 1/.99, where the clearcoat alpha float(.1 + (.001-.1)*gloss) crosses 0."""
    g = F32(0.1 / 0.099)
    out = [g]
    for _ in range(4):
        out += [np.nextafter(out[-1], INF)]
    lo = [g]
    for _ in range(4):
        lo += [np.nextafter(lo[-1], -INF)]
    return sorted(set(float(x) for x in out + lo))


GLOSS_A_MINUS_1 = float(F32(11.111112))     # the clearcoat alpha is exactly -1: a2 == 1, GTR1 is 0/0
GLOSS_NEAR_ZERO = _gloss_near_zero_alpha()
R001 = F32(0.001)


def clearcoat_alpha(gloss):
    return (0.1 + (0.001 - 0.1) * np.asarray(gloss, np.float64)).astype(F32)


# ---- the harness ----

_lib = None


def harness():
    global _lib
    if _lib is None:
        lib = C.CDLL(cuda_harness.harness_path("bsdf_harness"))
        lib.bsdf_sizeof_material.restype = C.c_int
        u32p = C.POINTER(C.c_uint32)
        lib.bsdf_make_materials.restype = None
        lib.bsdf_make_materials.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, u32p, u32p, C.POINTER(C.c_float)]
        lib.bsdf_run.restype = C.c_int
        lib.bsdf_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        _lib = lib
    return _lib


def make_materials(mats, scene_size):
    """The renderer's host code over `mats` (MAT_DTYPE) in scenes of scene_size consecutive materials:
    (DMaterial records as bytes (n, size), flags, features, ior)."""
    lib = harness()
    mats = np.ascontiguousarray(mats, MAT_DTYPE)
    n = mats.size
    out = np.zeros((n, lib.bsdf_sizeof_material()), np.uint8)
    flags, feats, ior = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, F32)
    lib.bsdf_make_materials(mats.ctypes.data, n, scene_size, out.ctypes.data, flags.ctypes.data_as(C.POINTER(C.c_uint32)),
                            feats.ctypes.data_as(C.POINTER(C.c_uint32)), ior.ctypes.data_as(C.POINTER(C.c_float)))
    return out, flags, feats, ior


def material(**kw):
    """One MAT_DTYPE record: abi.Material.default() with the given fields."""
    m = np.zeros(1, MAT_DTYPE)
    C.memmove(m.ctypes.data, C.byref(abi.Material.default()), MAT_DTYPE.itemsize)
    for k, v in kw.items():
        m[k] = v
    return m


# ---- the cases ----


def _pick(rng, n, edges, uniform, p_edge=0.7):
    edges = np.asarray(edges, F32)
    v = edges[rng.integers(0, edges.size, n)]
    return np.where(rng.random(n) < p_edge, v, uniform(n).astype(F32)).astype(F32)


def edge_materials(rng, n):
    """n materials, each parameter from its edge values or a uniform draw."""
    m = np.zeros(n, MAT_DTYPE)
    u01 = lambda k: rng.random(k)
    m["roughness"] = _pick(rng, n, [0.0, R001, np.nextafter(R001, INF), np.nextafter(R001, F32(0)), 1.0, 4.0], u01)
    for name in ("metallic", "specularTint", "transmission"):
        m[name] = _pick(rng, n, [0.0, 0.0, 1.0], u01)
    m["subsurface"] = _pick(rng, n, [0.0, 0.0, 1.0, 1.5, 3.0], u01)
    m["specular"] = _pick(rng, n, [0.0, 1.0, 12.5, -0.5, 50.0, 0.5], u01)
    m["eta"] = _pick(rng, n, [0.0, 0.0, 0.0, 1.0, 0.5, 1.5, -1.5, np.inf, np.nan], lambda k: 1.0 + rng.random(k))
    m["clearcoat"] = _pick(rng, n, [0.0, 0.0, 1.0], u01)
    m["clearcoatGloss"] = _pick(rng, n, [0.0, 1.0, GLOSS_A_MINUS_1, -1e20, 1e20, 1e21, np.nan, 50.0, -20.0] + GLOSS_NEAR_ZERO, u01)
    kind = rng.integers(0, 5, n)
    color = rng.random((n, 3)).astype(F32)
    color[kind == 0] = 0.0                               # Cdlum 0: Ctint 1
    color[kind == 1] = 1.0
    color[kind == 2] = -color[kind == 2]
    m["color"] = color
    m["sheen"], m["sheenTint"] = rng.random(n), rng.random(n)
    return m


def _dot(a, b):
    """dot() as the device computes it, in float32."""
    a, b = a.astype(F32), b.astype(F32)
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def _unit(v):
    return (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(F32)


def make_cases(seed):
    """BATCH cases over 2 * SCENES materials (MAT_DTYPE) in scenes of two; returns (materials, cases, kinds)."""
    rng = np.random.default_rng(seed)
    n = BATCH
    mats = edge_materials(rng, 2 * SCENES)
    # the second material of a scene: half of the time a copy of the first, so that its ior alone decides the scene
    copy = rng.random(SCENES) < 0.5
    mats[1::2][copy] = mats[0::2][copy]
    scene = rng.integers(0, SCENES, n)
    c = np.zeros(n, CASE_DTYPE)
    c["mat"] = 2 * scene
    c["seed"] = rng.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64).astype(np.int32)
    # N: random, axis-aligned with signed zeros, |x| == |y| (basis_from_vector's branch), one signed-zero component
    nk = rng.integers(0, 4, n)
    N = _unit(rng.normal(size=(n, 3)))
    sgn = lambda k: np.where(rng.random(k) < 0.5, F32(-1), F32(1))
    ax = np.zeros((n, 3), F32) * sgn((n, 3))
    ax[np.arange(n), rng.integers(0, 3, n)] = sgn(n)
    a = F32(np.sqrt(0.5)) * rng.uniform(0.2, 1.0, n).astype(F32)
    xy = np.stack([a * sgn(n), a * sgn(n), np.sqrt(np.maximum(0, 1 - 2 * a.astype(np.float64) ** 2)).astype(F32) * sgn(n)], 1)
    z0 = _unit(rng.normal(size=(n, 3)))
    z0[np.arange(n), rng.integers(0, 3, n)] = F32(0) * sgn(n)
    N = np.choose(nk[:, None], [N, ax, xy, z0]).astype(F32)
    vk = rng.integers(0, 5, n)
    lk = rng.integers(0, 6, n)
    # an exactly perpendicular V or L needs N of the axis-aligned or the |x| == |y| kind: N = (a, s a, c), V = (b, -s b, 0)
    perp = ((vk == 2) | (lk == 2)) & ~np.isin(nk, [1, 2])
    N[perp] = xy[perp]
    # V with dot(N, V) >= 0: random, V == N, dot(N, V) == 0 exactly, grazing, one ulp off unit length
    V = _unit(rng.normal(size=(n, 3)))
    b = F32(np.sqrt(0.5))
    s = np.where(N[:, 0] * N[:, 1] < 0, F32(-1), F32(1))
    vperp = np.stack([np.full(n, b), -s * b, np.zeros(n, F32)], 1) * sgn(n)[:, None]
    axz = (N[:, 0] == 0) & (N[:, 1] == 0)                  # N along z: any V in the xy plane
    t = rng.uniform(0, 2 * np.pi, n)
    vperp[axz] = np.stack([np.cos(t), np.sin(t), np.zeros(n)], 1)[axz].astype(F32)
    vperp[(N[:, 2] == 0) & ~axz] = np.stack([np.zeros(n, F32), np.zeros(n, F32), np.ones(n, F32)], 1)[(N[:, 2] == 0) & ~axz]
    tang = _unit(np.cross(N, rng.normal(size=(n, 3))))
    eps = np.array([1e-2, 1e-4, 1e-7, 1e-30])[rng.integers(0, 4, n)]
    graze = _unit(tang.astype(np.float64) + eps[:, None] * N)
    off = V * np.where(rng.random((n, 1)) < 0.5, F32(1) + F32(2 ** -23), F32(1) - F32(2 ** -24))
    V = np.choose(vk[:, None], [V, N, vperp, graze, off]).astype(F32)
    V[_dot(N, V) < 0] *= F32(-1)
    # L: the whole sphere, L == N, dot(N, L) == 0 exactly, the mirror direction, -V, one ulp beside N
    L = _unit(rng.normal(size=(n, 3)))
    lperp = vperp * sgn(n)[:, None]
    lperp[axz] = np.stack([np.cos(t + 1.0), np.sin(t + 1.0), np.zeros(n)], 1)[axz].astype(F32)
    ndv = _dot(N, V)
    mirror = (F32(2) * ndv)[:, None] * N - V
    beside = np.nextafter(N, INF)
    L = np.choose(lk[:, None], [L, N, lperp, mirror, -V, beside]).astype(F32)
    c["n"], c["v"], c["l"] = N, V, L
    _, _, _, ior = make_materials(mats, 2)
    # (etaI, etaO) as path_hit makes them: entering the material (1, ior), or leaving into the air from the medium
    # of the scene's other material (ior', 1)
    leaving = rng.random(n) < 1.0 / 3.0
    c["etaI"] = np.where(leaving, ior[2 * scene + 1], F32(1))
    c["etaO"] = np.where(leaving, F32(1), ior[2 * scene])
    kinds = {"N": nk, "V": vk, "L": lk, "leaving": leaving}
    return mats, c, kinds


def all_batches():
    for k in range(BATCHES):
        yield make_cases(20261016 + k)


def classify(mats, c, kinds, flags, feats):
    """The case classes, as boolean masks."""
    m = mats[c["mat"]]
    fl, fe = flags[c["mat"]], feats[c["mat"]]
    N, V, L = c["n"], c["v"], c["l"]
    a = clearcoat_alpha(m["clearcoatGloss"])
    with np.errstate(all="ignore"):
        ior_nonfinite = ~np.isfinite(c["etaI"]) | ~np.isfinite(c["etaO"])
        return {
            "roughness 0": m["roughness"] == 0,
            "roughness 0.001 +- 1 ulp": (m["roughness"] != R001) & (np.abs(m["roughness"] - R001) < 1e-9),
            "roughness 4": m["roughness"] == 4,
            "subsurface > 1": m["subsurface"] > 1,
            "transmission 1": m["transmission"] == 1,
            "transmission in (0, 1)": (m["transmission"] > 0) & (m["transmission"] < 1),
            "ior NaN (specular < 0)": (m["eta"] == 0) & (m["specular"] < 0),
            "ior inf (specular 12.5)": (m["eta"] == 0) & (m["specular"] == 12.5),
            "ior 1 (specular 0)": (m["eta"] == 0) & (m["specular"] == 0),
            "eta negative": m["eta"] < 0,
            "eta inf": np.isinf(m["eta"]),
            "eta NaN": np.isnan(m["eta"]),
            "non-finite eta pair": ior_nonfinite,
            "clearcoat alpha -1": a == -1,
            "clearcoat alpha near 0": np.abs(a) < 1e-5,
            "clearcoat gloss NaN": np.isnan(m["clearcoatGloss"]),
            "clearcoat alpha huge": np.abs(a) > 1e10,
            "gtr1 wide": (fl & GTR1_WIDE) != 0,
            "colour 0": (m["color"] == 0).all(1),
            "colour negative": (m["color"] < 0).all(1),
            "Fr skipped": (fl & NO_FRESNEL) != 0,
            "Fr kept, transmission 0": ((fl & NO_FRESNEL) == 0) & (m["transmission"] == 0),
            "clearcoat skipped": (fl & NO_CLEARCOAT) != 0,
            "clearcoat 0 kept": ((fl & NO_CLEARCOAT) == 0) & (m["clearcoat"] == 0),
            "featureless": fe == 0,
            "N axis-aligned, signed zeros": kinds["N"] == 1,
            "N |x| == |y|": np.abs(N[:, 0]) == np.abs(N[:, 1]),
            "dot(N, V) == 0": _dot(N, V) == 0,
            "V == N": (V == N).all(1),
            "V grazing": kinds["V"] == 3,
            "V off unit": kinds["V"] == 4,
            "L == N": (L == N).all(1),
            "dot(N, L) == 0": _dot(N, L) == 0,
            "L mirror": kinds["L"] == 3,
            "L == -V": (L == -V).all(1),
            "L below": _dot(N, L) < 0,
            "leaving (ior', 1)": kinds["leaving"],
        }


MIN_PER_CLASS = 2000


def test_bsdf_harness_compiles_for_sm90a():
    """The harness against the headers as they are (no GPU needed): a header change that breaks it fails here."""
    cuda_harness.harness_path("bsdf_harness")


def test_case_coverage():
    """Every class of case occurs often enough, so that an edit of the generator cannot quietly drop one."""
    counts = {}
    for mats, c, kinds in all_batches():
        _, flags, feats, _ = make_materials(mats, 2)
        for name, m in classify(mats, c, kinds, flags, feats).items():
            counts[name] = counts.get(name, 0) + int(m.sum())
    print("bsdf cases per class: %s" % counts)
    low = {name: v for name, v in counts.items() if v < MIN_PER_CLASS}
    assert not low, low


# ---- the host-side flags, without a GPU ----


def _flags_of(**kw):
    _, flags, feats, ior = make_materials(material(**kw), 1)
    return int(flags[0]), int(feats[0]), float(ior[0])


def test_material_flags_decide_the_skips():
    """TB_MAT_NO_FRESNEL and TB_MAT_NO_CLEARCOAT on the materials where the skipped term is NaN in the reference,
    and the scene features that keep such a material off the kernel that skips unconditionally."""
    flags, feats, _ = _flags_of(color=[0.5] * 3)
    assert flags == NO_FRESNEL | NO_CLEARCOAT and feats == 0
    # ior NaN / inf from the specular: Fr is NaN, so is the reference's pdf
    for spec in (-0.5, 12.5, 50.0):
        flags, feats, ior = _flags_of(specular=spec)
        assert not np.isfinite(ior) or ior < 0 or ior > 256, (spec, ior)
        assert not flags & NO_FRESNEL and feats & FEAT_TRANSMISSION, spec
    for eta in (-1.5, np.inf, np.nan, 1e-30, 1e30):
        flags, feats, _ = _flags_of(eta=eta)
        assert not flags & NO_FRESNEL and feats & FEAT_TRANSMISSION, eta
    for eta in (0.5, 1.0, 1.5, 1.0 / 256, 256.0):
        flags, feats, _ = _flags_of(eta=eta)
        assert flags & NO_FRESNEL and feats == 0, eta
    flags, feats, _ = _flags_of(transmission=0.5)
    assert not flags & NO_FRESNEL and feats & FEAT_TRANSMISSION
    # the clearcoat lobe: 0/0 at alpha -1, NaN gloss, alpha near 0 (GTR1's t reaches 0), alpha^2 infinite (1e21)
    for gloss in [GLOSS_A_MINUS_1, np.nan, 1e21] + [g for g in GLOSS_NEAR_ZERO if abs(clearcoat_alpha(g)) < 1e-4]:
        flags, feats, _ = _flags_of(clearcoatGloss=gloss)
        assert not flags & NO_CLEARCOAT and feats & FEAT_CLEARCOAT, gloss
    for gloss in (0.0, 0.5, 1.0, 50.0, 1e10, 1e20):
        flags, feats, _ = _flags_of(clearcoatGloss=gloss)
        assert flags & NO_CLEARCOAT and feats == 0, gloss
    for gloss in (-20.0, -1e20):                            # alpha >= 1: GTR1 is kInvPi
        flags, feats, _ = _flags_of(clearcoatGloss=gloss)
        assert flags & GTR1_WIDE and flags & NO_CLEARCOAT and feats == 0, gloss
    flags, feats, _ = _flags_of(clearcoat=0.5)
    assert not flags & NO_CLEARCOAT and feats & FEAT_CLEARCOAT
    # one material with a NaN ior takes the skip from every material of its scene: etaI can be its ior
    two = np.concatenate([material(), material(specular=-0.5)])
    _, flags, feats, _ = make_materials(two, 2)
    assert not (flags & NO_FRESNEL).any() and (feats & FEAT_TRANSMISSION).all()
    _, flags, feats, _ = make_materials(two, 1)
    assert flags[0] & NO_FRESNEL and not flags[1] & NO_FRESNEL


def _fresnel32(vdn, etaI, etaT):
    """Fr (tb_shade.cuh: fresnel_dielectric) in float32."""
    q = etaI / etaT
    s2 = (q * q) * (F32(1) - vdn * vdn)
    ldn = np.sqrt(F32(1) - s2)
    eta = etaT / etaI
    r1 = (vdn - eta * ldn) / (vdn + eta * ldn)
    r2 = (ldn - eta * vdn) / (ldn + eta * vdn)
    return np.where(s2 > F32(1), F32(1), F32(0.5) * (r1 * r1 + r2 * r2))


def test_fresnel_is_finite_over_the_skipped_ior_range():
    """Fr is finite for every front-facing VDotN (denormal, tiny, one ulp beside 1 on both sides) and every pair of
    etas in [1/256, 256], the range set_fresnel_flags allows; just outside it, it is not."""
    rng = np.random.default_rng(5)
    one = F32(1)
    vdn = np.concatenate([np.array([1e-45, 1e-40, 1e-38, 1e-30, 1e-20, 1e-7, 0.5, np.nextafter(one, F32(0)), 1.0,
                                    np.nextafter(one, INF), np.nextafter(np.nextafter(one, INF), INF)], F32),
                          rng.random(200).astype(F32)])
    lo, hi = F32(1.0 / 256), F32(256)
    etas = np.concatenate([np.array([lo, np.nextafter(lo, INF), hi, np.nextafter(hi, F32(0)), 1.0, np.nextafter(one, INF),
                                     np.nextafter(one, F32(0)), 0.5, 1.5, 2.0], F32),
                           np.exp(rng.uniform(np.log(lo), np.log(hi), 60)).astype(F32)])
    with np.errstate(all="ignore"):
        a, b, v = np.meshgrid(etas, etas, vdn, indexing="ij")
        assert np.isfinite(_fresnel32(v, a, b)).all()
        v = vdn[None, :]
        assert not np.isfinite(_fresnel32(v, F32(1e30), F32(1e-30))).all()


def test_clearcoat_skip_needs_a_finite_gtr1():
    """Where TB_MAT_NO_CLEARCOAT is set, GTR1 (disney.h:56-62, as the restatement computes it in float32) is finite
    for every NDotH up to 1 + 2^-22 in magnitude; on the glosses of the table it is not set."""
    rng = np.random.default_rng(6)
    g = np.concatenate([np.array([0, 1, 50, 1e10, -20, -1e20, 1e20, 1e21, GLOSS_A_MINUS_1, np.nan] + GLOSS_NEAR_ZERO, F32),
                        rng.uniform(-30, 30, 400).astype(F32), rng.uniform(1.0, 1.02, 400).astype(F32)])
    mats = np.concatenate([material(clearcoatGloss=x) for x in g])
    _, flags, _, _ = make_materials(mats, 1)
    c = np.concatenate([np.linspace(-1, 1, 2001, dtype=F32), np.array([1 + 2 ** -23, 1 + 2 ** -22, -1 - 2 ** -22], F32)])
    a = clearcoat_alpha(g)
    with np.errstate(all="ignore"):
        a2 = a * a
        t = F32(1) + ((a2 - F32(1))[:, None] * c[None, :]) * c[None, :]
        gtr1 = np.where((a >= 1)[:, None], F32(1 / np.pi), (a2 - F32(1))[:, None] / ((F32(np.pi) * np.log(a2))[:, None] * t))
    finite = np.isfinite(gtr1).all(1)
    skip = (flags & NO_CLEARCOAT) != 0
    assert finite[skip].all(), g[skip & ~finite]
    assert not skip[np.isin(g, [GLOSS_A_MINUS_1, F32(1e21)]) | np.isnan(g)].any()
    # and it is set wherever the alpha is no nearer 0 than a gloss of 1 gives, not -1 and not so large its square overflows
    assert skip[(np.abs(a) >= R001) & (a != -1) & (np.abs(a) < 1e19)].all()


# ---- the GPU side ----


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype.kind == "f":
        return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
    return a == b


def _oracle(mats, c):
    out = np.zeros(c.size, REF_DTYPE)
    lib = refdrv.load_port()
    lib.oracle_bsdf_cases.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.oracle_bsdf_cases(mats.ctypes.data, c.ctypes.data, c.size, out.ctypes.data)
    return out


def _reference(mats, c, every):
    """The reference's own BSDFEval / BSDFPdf / BSDFSample (oracle/_ref) on every `every`-th case."""
    lib = refdrv.load_ref("detmath")
    idx = np.arange(0, c.size, every)
    out = np.zeros(idx.size, REF_DTYPE)
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    for j, k in enumerate(idx):
        m = abi.Material()
        C.memmove(C.byref(m), mats[c["mat"][k]:c["mat"][k] + 1].ctypes.data, MAT_DTYPE.itemsize)
        n, v, l = c["n"][k].copy(), c["v"][k].copy(), c["l"][k].copy()
        f, ls = np.zeros(3, F32), np.zeros(3, F32)
        pdf, spdf, stype, after = C.c_float(), C.c_float(), C.c_int(), (C.c_uint32 * 2)()
        lib.ref_bsdf_eval(C.byref(m), c["etaI"][k], c["etaO"][k], fp(n), fp(v), fp(l), fp(f), C.byref(pdf))
        lib.ref_bsdf_sample(C.byref(m), c["etaI"][k], c["etaO"][k], fp(n), fp(v), int(c["seed"][k]), fp(ls), C.byref(spdf),
                            C.byref(stype), after)
        out[j] = (f, pdf.value, ls, spdf.value, stype.value, (after[0], after[1]))
    return idx, out


def _device(dmats, c, all_features):
    import torch
    dm = torch.from_numpy(dmats.reshape(-1)).cuda()
    dc = torch.from_numpy(np.ascontiguousarray(c).view(np.uint8)).cuda()
    do = torch.zeros(c.size * OUT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    rc = harness().bsdf_run(dm.data_ptr(), dc.data_ptr(), c.size, do.data_ptr(), int(all_features))
    assert rc == 0, "bsdf_run: cudaError %d" % rc
    return do.cpu().numpy().view(OUT_DTYPE)


def _mismatches(dev, ref, flags):
    """Per output, a mask of the cases whose device value differs from `ref` under the rules of the module docstring."""
    zero_f = ((flags & NO_CLEARCOAT) != 0)[:, None] & (dev["f"] == 0) & (ref["f"] == 0)
    fresnel = (flags & NO_FRESNEL) != 0
    bad = {
        "f": ~(_bits_equal(dev["f"], ref["f"]) | zero_f).all(1),
        "pdf": ~(_bits_equal(dev["pdf"], ref["pdf"]) | (fresnel & (dev["pdf"] == 0) & (ref["pdf"] == 0))),
        "light": ~_bits_equal(dev["light"], ref["light"]).all(1),
        "sample pdf": ~(_bits_equal(dev["spdf"], ref["spdf"]) | (fresnel & (dev["spdf"] == 0) & (ref["spdf"] == 0))),
        "type": dev["type"] != ref["type"],
        "rng": ~(dev["rng"] == ref["rng"]).all(1),
        # bsdf_eval_pdf is the pair of the separate calls
        "bsdf_eval_pdf": ~(_bits_equal(dev["fp"], dev["f"]).all(1) & _bits_equal(dev["pdfp"], dev["pdf"])),
    }
    return bad


def _report(what, bad, dev, ref, mats, c):
    lines = []
    for name, m in bad.items():
        if m.any():
            k = int(np.argmax(m))
            lines.append("%s: %d cases differ, first: material %s, case %s, device %s, restatement %s" % (
                name, int(m.sum()), mats[c["mat"][k]], c[k], dev[k], ref[k]))
    return "%s:\n  %s" % (what, "\n  ".join(lines))


@pytest.mark.gpu
def test_bsdf_matches_restatement():
    totals = {}
    failures = []
    ran = {"TB_FEAT_ALL": 0, "TB_FEAT_NONE": 0}
    for b, (mats, c, kinds) in enumerate(all_batches()):
        dmats, flags, feats, _ = make_materials(mats, 2)
        ref = _oracle(mats, c)
        fl = flags[c["mat"]]
        featureless = feats[c["mat"]] == 0
        for inst, sel in (("TB_FEAT_ALL", np.ones(c.size, bool)), ("TB_FEAT_NONE", featureless)):
            cs = np.ascontiguousarray(c[sel])
            dev = _device(dmats, cs, inst == "TB_FEAT_ALL")
            checks = [("restatement", _mismatches(dev, ref[sel], fl[sel]), ref[sel], cs)]
            if inst == "TB_FEAT_ALL" and refdrv.have_ref("detmath"):
                idx, rref = _reference(mats, c, 64)
                checks.append(("reference", _mismatches(dev[idx], rref, fl[idx]), rref, c[idx]))
            ran[inst] += cs.size
            for against, bad, expect, cc in checks:
                for name, m in bad.items():
                    totals[(inst, against, name)] = totals.get((inst, against, name), 0) + int(m.sum())
                if any(m.any() for m in bad.values()) and len(failures) < 4:
                    failures.append(_report("batch %d, %s against the %s" % (b, inst, against), bad, dev, expect, mats, cc))
    print("bsdf: %d cases in TB_FEAT_ALL, %d featureless ones in TB_FEAT_NONE; mismatches %s" % (
        ran["TB_FEAT_ALL"], ran["TB_FEAT_NONE"], {k: v for k, v in totals.items() if v}))
    assert not any(totals.values()), "\n".join(failures) + "\nmismatch counts: %s" % {k: v for k, v in totals.items() if v}


@pytest.mark.gpu
def test_golden_bsdf_kats_on_the_device():
    """kats.npz["bsdf"]: the reference's own BSDFEval / BSDFPdf / BSDFSample outputs, run on the device directly."""
    g = np.load(os.path.join(GOLD, "kats.npz"))
    mats = np.ascontiguousarray(g["materials"].astype(F32)).view(MAT_DTYPE).reshape(-1)
    dmats, flags, _, _ = make_materials(mats, 1)
    rec = g["bsdf"]
    c = np.zeros(len(rec), CASE_DTYPE)
    c["mat"] = rec[:, 0].astype(np.int32)
    c["etaI"], c["etaO"] = rec[:, 1].astype(F32), rec[:, 2].astype(F32)
    c["n"], c["v"], c["l"] = rec[:, 3:6].astype(F32), rec[:, 6:9].astype(F32), rec[:, 9:12].astype(F32)
    c["seed"] = rec[:, 16].astype(np.int64).astype(np.int32)
    ref = np.zeros(len(rec), REF_DTYPE)
    ref["f"], ref["pdf"] = rec[:, 12:15].astype(F32), rec[:, 15].astype(F32)
    ref["light"], ref["spdf"] = rec[:, 17:20].astype(F32), rec[:, 20].astype(F32)
    ref["type"], ref["rng"] = rec[:, 21].astype(np.int32), rec[:, 22:24].astype(np.int64).astype(np.uint32)
    dev = _device(dmats, c, True)
    bad = _mismatches(dev, ref, flags[c["mat"]])
    # the records hold the sampled direction and type only where the sample's pdf is positive (tools/make_golden.py)
    unsampled = ~(ref["spdf"] > 0)
    bad["light"] &= ~unsampled
    bad["type"] &= ~unsampled
    assert not any(m.any() for m in bad.values()), _report("kats.npz", bad, dev, ref, mats, c)


# ---- edge materials in whole renders ----


def _edge_scene_materials(rng, unsafe):
    """Materials for one scene.  unsafe=False: edge values whose skips are exact (the scene is featureless, so the
    lane-owned kernel compiled without features runs it).  unsafe=True: the values where the skipped terms are NaN."""
    out = []
    for _ in range(6):
        m = abi.Material.default()
        m.color[:] = [float(x) for x in rng.choice([0.0, 1.0, -0.3, rng.uniform()], 3)]
        m.metallic = float(rng.choice([0.0, 1.0, rng.uniform()]))
        m.specularTint = float(rng.choice([0.0, 1.0, rng.uniform()]))
        m.roughness = float(rng.choice([0.0, float(R001), float(np.nextafter(R001, INF)), float(np.nextafter(R001, F32(0))), 1.0, 4.0]))
        if unsafe:
            kind = int(rng.randint(0, 4))
            if kind == 0:
                m.specular, m.eta = float(rng.choice([-0.5, 12.5, 50.0])), 0.0
            elif kind == 1:
                m.eta = float(rng.choice([-1.5, np.inf, np.nan]))
                m.transmission = float(rng.choice([0.0, 0.5, 1.0]))
            elif kind == 2:
                m.clearcoatGloss = float(rng.choice([GLOSS_A_MINUS_1, np.nan, 1e21] + GLOSS_NEAR_ZERO))
            else:
                m.subsurface = float(rng.choice([1.5, 3.0]))
                m.clearcoat = float(rng.choice([0.0, 1.0]))
        else:
            m.specular = float(rng.choice([0.0, 1.0, 0.5, 10.0]))
            m.eta = float(rng.choice([0.0, 1.0, 0.5, 1.5]))
            m.clearcoatGloss = float(rng.choice([0.0, 1.0, 50.0, -20.0, 1e20, -1e20]))
        out.append(m)
    return out


def make_edge_scene(seed, path, unsafe, width=96, height=64):
    """A floor, five spheres and two sphere lights, every surface with an edge material (_edge_scene_materials)."""
    rng = np.random.RandomState(4099 * (2 + int(unsafe)) + seed)
    mats = _edge_scene_materials(rng, unsafe)
    prims = (abi.Primitive * 8)()
    bounds = [fuzzscene._floor(prims[0], rng)]
    prims[0].material = mats[0]
    for i in range(5):
        pos = (rng.uniform(-2.0, 2.0), rng.uniform(0.3, 1.4), rng.uniform(-1.5, 1.0))
        bounds.append(fuzzscene._sphere(prims[1 + i], pos, rng.uniform(0.3, 0.6), mats[1 + i]))
    for i in range(2):
        light = fuzzscene._material(rng, True)
        bounds.append(fuzzscene._sphere(prims[6 + i], (rng.uniform(-1.5, 1.5), rng.uniform(2.2, 3.2), rng.uniform(-1.0, 1.5)),
                                        0.3, light, int(rng.randint(1, 3))))
    fuzzscene._save(rng, path, prims, fuzzscene._build_bvh(bounds), [], width, height, max_depth=5)
    return mats


EDGE_ROUTES = {r: schedenv.ROUTES[r] for r in ("mega", "wavefront", "lanes", "lanes-generic")}
EDGE_ROUTES["SPECIALIZE=0"] = dict(SPECIALIZE="0")
EDGE_SCENES = [(False, s) for s in range(3)] + [(True, s) for s in range(3)]


def _trace_routes(path, routes, frames):
    """{(route, frame): samples that differ from the restatement}, {route: kernel that ran}, NaN samples per frame.
    routes: {route: its knob settings}."""
    port = refdrv.PortScene.from_snapshot(path)
    expect = {f: port.trace_frame(f, 8) for f in frames}
    port.close()
    snap = tb.Snapshot(path)
    cam, opt = snap.camera, snap.options
    bad, kernels = {}, {}
    try:
        for route, settings in routes.items():
            with schedenv.knobs(**settings):
                r = tb.Renderer(snap.scene)
            r.Init(opt.width, opt.height)
            for f in frames:
                rad, ras = r.trace_frame(cam, opt, f)
                prad, pras = expect[f]
                assert np.array_equal(ras, pras)
                n = int((~_bits_equal(rad, prad).all(-1)).sum())
                if n:
                    bad[(route, f)] = n
            kernels[route] = r.last_kernel()
            r.close()
    finally:
        snap.close()
    return bad, kernels, {f: int(np.isnan(expect[f][0]).any(-1).sum()) for f in frames}


@pytest.mark.gpu
@pytest.mark.parametrize("unsafe,seed", EDGE_SCENES)
def test_edge_material_scenes_match_restatement(unsafe, seed, tmp_path):
    """Per sample and bit for bit (NaN as NaN) in the megakernel, the default wavefront route, the lane-owned kernel
    and with the specialised kernel switched off.  Scenes whose skips are all exact run the specialised kernel; the
    others never do, and their NaN samples land where the restatement's do."""
    path = str(tmp_path / "edge.tsnap")
    make_edge_scene(seed, path, unsafe)
    bad, kernels, nan = _trace_routes(path, EDGE_ROUTES, (0, 3))
    assert not bad, "samples differ: %s" % bad
    assert kernels["lanes"] == ("wf2_lq.generic" if unsafe else "wf2_lq.specialized"), kernels
    assert kernels["lanes-generic"] == "wf2_lq.generic", kernels
    print("edge scene unsafe=%s seed %d: kernels %s, NaN samples per frame %s" % (unsafe, seed, kernels, nan))


@pytest.mark.gpu
@pytest.mark.parametrize("sched,cta", [(s, c) for s in schedenv.SCHEDS for c in schedenv.CTAS])
def test_edge_material_scenes_under_every_scheduler_variant(sched, cta, tmp_path):
    for unsafe, seed in EDGE_SCENES[::2]:
        path = str(tmp_path / ("edge%d%d.tsnap" % (unsafe, seed)))
        make_edge_scene(seed, path, unsafe)
        bad, _, _ = _trace_routes(path, {sched: schedenv.sched_knobs(sched, cta)}, (3, 4))
        assert not bad, "unsafe=%s seed %d: samples differ %s" % (unsafe, seed, bad)


def test_edge_scenes_hold_what_they_claim(tmp_path):
    """The featureless scenes are featureless by the renderer's own rule and the others are not; the restatement
    renders every scene lit, and the unsafe ones with NaN samples."""
    nan = 0
    for unsafe, seed in EDGE_SCENES:
        path = str(tmp_path / "e.tsnap")
        mats = make_edge_scene(seed, path, unsafe)
        arr = np.zeros(len(mats), MAT_DTYPE)
        for i, m in enumerate(mats):
            C.memmove(arr[i:i + 1].ctypes.data, C.byref(m), MAT_DTYPE.itemsize)
        _, _, feats, _ = make_materials(arr, len(mats))
        assert (feats != 0).any() == unsafe, (unsafe, seed, feats)
        port = refdrv.PortScene.from_snapshot(path)
        rad, _ = port.trace_frame(0, 4)
        port.close()
        assert float(np.nansum(np.abs(rad))) > 0.0, (unsafe, seed)
        if unsafe:
            nan += int(np.isnan(rad).any(-1).sum())
    assert nan > 0
