"""Which primitives the renderer may take as static, without a GPU.  The device takes a static primitive's transform as
computed once at t = 0 (DPrim::fixed) instead of the reference's InterpolateTransform(start, end, t), whose components
are Lerp(a, b, t) = a + (b - a) * t.  With start == end bit for bit that is a + 0 * t: here the rule is restated in
numpy float32 over component values and ray times, the scene cache is checked to record exactly the primitives the
rule calls static, and a cache written before the rule is refused."""
import numpy as np

import tinsel_b200 as tb
import fuzzscene
from queryscenes import TIMES   # the finite ray times of test_motion_time_gpu.py

F32 = np.float32
COMPONENTS = np.array([0.0, -0.0, 1.0, -1.0, np.finfo(F32).max, np.inf, np.nan], F32)
PRIM_BYTES_IS_STATIC = 96    # DPrim: Xf start, end, fixed (32 bytes each), then int isStatic


def _same(a, b):
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def test_lerp_of_equal_ends_is_time_independent_exactly_without_negative_zero():
    """a + (a - a) * t equals its value at t = 0 for every finite t exactly when a is not -0; a -0 keeps its sign at
    t < 0 and t = -0, where the value at t = 0 is +0."""
    with np.errstate(invalid="ignore"):
        for a in COMPONENTS:
            lerp = a + (a - a) * TIMES
            at0 = a + (a - a) * F32(0.0)
            same = _same(lerp, np.full_like(lerp, at0))
            negative_zero = a == 0 and np.signbit(a)
            if negative_zero:
                assert (same == ~np.signbit(TIMES)).all(), (a, TIMES[~same])
            else:
                assert same.all(), (a, TIMES[~same])


def test_rule_restated_on_transforms():
    """fuzzscene.is_static, the rule the tests rely on, is the numpy restatement over whole transforms."""
    prims = (fuzzscene.abi.Primitive * 3)()
    fuzzscene._xf(prims[0].start, (0.0, 1.0, 2.0), (0.0, 0.0, 0.0, 1.0), 1.0)
    fuzzscene._xf(prims[0].end, (0.0, 1.0, 2.0), (0.0, 0.0, 0.0, 1.0), 1.0)
    fuzzscene._xf(prims[1].start, (0.0, 1.0, 2.0), (0.0, -0.0, 0.0, 1.0), 1.0)
    fuzzscene._xf(prims[1].end, (0.0, 1.0, 2.0), (0.0, -0.0, 0.0, 1.0), 1.0)
    fuzzscene._xf(prims[2].start, (0.0, 1.0, 2.0), (0.0, 0.0, 0.0, 1.0), 1.0)
    fuzzscene._xf(prims[2].end, (0.0, 1.0, 2.0), (0.0, 0.0, 0.0, 1.0), 0.5)
    with np.errstate(invalid="ignore"):
        for p, static in zip(prims, (True, False, False)):
            assert fuzzscene.is_static(p) == static
            a = np.frombuffer(bytes(p.start), F32)
            b = np.frombuffer(bytes(p.end), F32)
            lerp = a[None, :] + (b - a)[None, :] * TIMES[:, None]
            at0 = a + (b - a) * F32(0.0)
            assert _same(lerp, np.broadcast_to(at0, lerp.shape)).all() == static


def _cached_prims(tmp_path, family, seed):
    path = str(tmp_path / "s.tsnap")
    info = fuzzscene.make_mesh_scene(seed, path, family)
    snap = tb.Snapshot(path)
    cache = str(tmp_path / "s.tcache")
    tb.scene_cache_save(snap.scene, cache)       # needs no GPU
    sc = snap.scene.contents
    want = [fuzzscene.is_static(sc.primitives[i]) for i in range(sc.numPrimitives)]
    snap.close()
    data = open(cache, "rb").read()
    version, size_prim = (int.from_bytes(data[o:o + 4], "little") for o in (8, 12))
    assert data[:8] == b"TB2CACHE" and version == 5
    n = int.from_bytes(data[24:32], "little")
    assert n == len(want)
    recs = [data[32 + i * size_prim:32 + (i + 1) * size_prim] for i in range(n)]
    got = [int.from_bytes(r[PRIM_BYTES_IS_STATIC:PRIM_BYTES_IS_STATIC + 4], "little") for r in recs]
    return info, want, got, recs, data, cache


def test_cache_marks_primitives_with_negative_zero_as_moving(tmp_path):
    for seed in range(3):
        info, want, got, recs, _, _ = _cached_prims(tmp_path, "signed_zero", seed)
        assert info["negative_zero"] and len(info["negative_zero"]) < info["prims"]
        assert got == [0 if i in info["negative_zero"] else 1 for i in range(info["prims"])], (seed, got)
        assert got == [int(w) for w in want]
        for r in recs:                  # start and end stored as given, -0 included
            assert r[0:32] == r[32:64]


def test_cache_marks_rotating_primitives_as_moving(tmp_path):
    info, want, got, _, _, _ = _cached_prims(tmp_path, "rotating", 0)
    assert got == [int(w) for w in want] and got.count(1) == 1     # only the floor is static


def test_version_4_cache_is_refused(tmp_path):
    _, _, _, _, data, _ = _cached_prims(tmp_path, "signed_zero", 0)
    old = bytearray(data)
    old[8:12] = (4).to_bytes(4, "little")
    path = str(tmp_path / "v4.tcache")
    open(path, "wb").write(bytes(old))
    lib = tb.load_library()
    h = lib.tb200_create_cached(path.encode(), 0)
    if h:
        lib.tb200_destroy(h)
    assert not h and "another build" in tb.last_error(), tb.last_error()
