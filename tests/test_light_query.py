"""The light queries without a GPU: the tb200_light_query record of include/tinsel_b200.h, the entry points, the
packing of tinsel_b200.light_queries, tinsel_b200.primitive_areas against the restatement's PrimitiveArea, and the
CPU arm the device's SampleLights query is checked against (tests/light_oracle.cpp)."""
import ctypes as C
import glob
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import lightoracle

F32 = np.float32
HEADER = tb.ROOT + "/include/tinsel_b200.h"


def test_light_query_layout_matches_the_header():
    src = r'''
#include <stddef.h>
#include <stdio.h>
#include "tinsel_b200.h"
#define F(f) printf("tb200_light_query." #f " %zu\n", offsetof(tb200_light_query, f));
int main(void)
{
    printf("tb200_light_query %zu\n", sizeof(tb200_light_query));
    F(p) F(time) F(n) F(prim) F(wo) F(etaI) F(etaO) F(pad)
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        with open(c, "w") as f:
            f.write(src)
        subprocess.check_call(["cc", "-I", os.path.dirname(HEADER), c, "-o", exe])
        got = dict(re.findall(r"^(\S+) (\d+)$", subprocess.check_output([exe], text=True), re.M))
    assert int(got["tb200_light_query"]) == C.sizeof(abi.LightQuery) == 64
    for field, _ in abi.LightQuery._fields_:
        assert int(got["tb200_light_query." + field]) == getattr(abi.LightQuery, field).offset, field
    # the (N, 16) float32 columns light_queries documents
    assert [getattr(abi.LightQuery, f).offset // 4 for f in ("p", "time", "n", "prim", "wo", "etaI", "etaO", "pad")] == \
        [0, 3, 4, 7, 8, 11, 12, 13]


def test_entry_points_are_declared_and_exported():
    text = open(HEADER).read()
    for name in ("tb200_sample_lights", "tb200_sky_eval"):
        assert re.search(r"\bint %s\(" % name, text), name
        assert name in abi.EXPORTS
    lib = tb.load_library()
    assert hasattr(lib, "tb200_sample_lights") and hasattr(lib, "tb200_sky_eval")


def test_light_queries_packs_the_records():
    torch = pytest.importorskip("torch")
    n = 7
    rng = np.random.default_rng(5)
    prims = torch.tensor([-1, 0, 5, 2 ** 31 - 1, -2 ** 31, 4095, 123456789], dtype=torch.int32)
    p, nn, wo = (torch.from_numpy(rng.normal(size=(n, 3)).astype(F32)) for _ in range(3))
    eta_i, t = (torch.from_numpy(rng.random(n).astype(F32)) for _ in range(2))
    q = tb.light_queries(prims, p, nn, wo, eta_i, 1.5, t)
    assert q.dtype == torch.float32 and tuple(q.shape) == (n, 16) and q.is_contiguous() and q.device == prims.device
    rec = np.ascontiguousarray(q.numpy()).view(np.uint8).reshape(n, 64)
    for i in range(n):
        r = abi.LightQuery.from_buffer_copy(rec[i].tobytes())
        assert r.prim == int(prims[i])           # the int32 bits survive, NaN patterns included
        assert list(r.p) == p[i].tolist() and list(r.n) == nn[i].tolist() and list(r.wo) == wo[i].tolist()
        assert r.time == t[i].item() and r.etaI == eta_i[i].item() and r.etaO == F32(1.5)
        assert list(r.pad) == [0.0, 0.0, 0.0]
    q = tb.light_queries(prims, p, nn, wo, 1.0, 2.0, 0.25)
    assert (q[:, 11] == 1).all() and (q[:, 12] == 2).all() and (q[:, 3] == 0.25).all()
    assert (q[:, 7].view(torch.int32) == prims).all()
    with pytest.raises(ValueError):
        tb.light_queries(prims.long(), p, nn, wo, 1.0, 1.0, 0.0)
    with pytest.raises(ValueError):
        tb.light_queries(prims[:, None], p, nn, wo, 1.0, 1.0, 0.0)
    with pytest.raises(ValueError):
        tb.light_queries(prims, p[:, :2], nn, wo, 1.0, 1.0, 0.0)
    with pytest.raises(ValueError):
        tb.light_queries(prims, p, nn, wo.double(), 1.0, 1.0, 0.0)
    with pytest.raises(ValueError):
        tb.light_queries(prims, p, nn, wo, eta_i[:3], 1.0, 0.0)
    with pytest.raises(ValueError):
        tb.light_queries(prims, p, nn, wo, 1.0, 1.0, t.double())


def _snapshots():
    return sorted(glob.glob(os.path.join(tb.SCENE_DIR, "*.tsnap")))


@pytest.mark.parametrize("path", _snapshots(), ids=lambda p: os.path.basename(p)[:-6])
def test_primitive_areas_match_the_restatement(path):
    snap = tb.Snapshot(path)
    try:
        got = tb.primitive_areas(snap.scene)
        want = lightoracle.primitive_areas(snap.scene)
        assert got.dtype == F32 and got.shape == want.shape
        assert (got.view(np.uint32) == want.view(np.uint32)).all(), (got, want)
        assert (tb.primitive_areas(snap.scene.contents).view(np.uint32) == want.view(np.uint32)).all()
    finally:
        snap.close()


def test_sample_lights_oracle_without_lights_or_probe_gives_zeros():
    sphere = abi.Primitive()
    sphere.type, sphere.radius, sphere.mesh = abi.SPHERE, 1.0, -1
    sphere.start.r[3] = sphere.end.r[3] = 1.0
    sphere.start.s = sphere.end.s = 1.0
    sphere.material = abi.Material.default()
    prims = (abi.Primitive * 1)(sphere)
    sc = abi.Scene()
    sc.primitives, sc.numPrimitives = prims, 1
    sc.sky.horizon[:] = [0.5, 0.6, 0.7]
    sc.sky.zenith[:] = [0.1, 0.2, 0.3]
    rec = np.zeros((4, 16), F32)
    rec[:, 0:3] = [0.0, 0.0, 1.0]
    rec[:, 4:7] = [0.0, 0.0, 1.0]
    rec[:, 8:11] = [0.0, 0.6, 0.8]
    rec[:, 11], rec[:, 12] = 1.0, 1.5
    rec[:, 7] = np.array([0, 0, -1, 1], np.int32).view(F32)
    out = lightoracle.sample_lights(C.pointer(sc), rec, np.arange(4, dtype=np.uint32))
    assert (out == 0).all()
