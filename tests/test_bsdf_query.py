"""The BSDF queries without a GPU: the record layouts of include/tinsel_b200.h, the packing of tinsel_b200.bsdf_queries
and tinsel_b200.material_ior against the restatement's Material::GetIndexOfRefraction (oracle_material_ior)."""
import ctypes as C
import re

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import abi
import refdrv

F32 = np.float32
HEADER = tb.ROOT + "/include/tinsel_b200.h"


def _header_offsets():
    """Offsets and sizes of the three records, as a C compiler lays them out from the header."""
    src = r'''
#include <stddef.h>
#include <stdio.h>
#include "tinsel_b200.h"
#define F(T, f) printf(#T "." #f " %zu\n", offsetof(T, f));
int main(void)
{
    printf("tb200_bsdf_query %zu\n", sizeof(tb200_bsdf_query));
    printf("tb200_bsdf_value %zu\n", sizeof(tb200_bsdf_value));
    printf("tb200_bsdf_sampled %zu\n", sizeof(tb200_bsdf_sampled));
    F(tb200_bsdf_query, n) F(tb200_bsdf_query, prim) F(tb200_bsdf_query, v) F(tb200_bsdf_query, etaI)
    F(tb200_bsdf_query, l) F(tb200_bsdf_query, etaO)
    F(tb200_bsdf_value, f) F(tb200_bsdf_value, pdf)
    F(tb200_bsdf_sampled, l) F(tb200_bsdf_sampled, pdf) F(tb200_bsdf_sampled, f) F(tb200_bsdf_sampled, type)
    printf("REFLECTED %d TRANSMITTED %d SPECULAR %d\n", TB200_BSDF_REFLECTED, TB200_BSDF_TRANSMITTED, TB200_BSDF_SPECULAR);
    return 0;
}
'''
    import os
    import subprocess
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        with open(c, "w") as f:
            f.write(src)
        subprocess.check_call(["cc", "-I", os.path.dirname(HEADER), c, "-o", exe])
        return subprocess.check_output([exe], text=True)


def test_record_layouts_match_the_header():
    out = _header_offsets()
    got = dict(re.findall(r"^(\S+) (\d+)$", out, re.M))
    for name, cls, size in (("tb200_bsdf_query", abi.BsdfQuery, 48), ("tb200_bsdf_value", abi.BsdfValue, 16),
                            ("tb200_bsdf_sampled", abi.BsdfSampled, 32)):
        assert int(got[name]) == C.sizeof(cls) == size, name
        for field, _ in cls._fields_:
            assert int(got["%s.%s" % (name, field)]) == getattr(cls, field).offset, (name, field)
    # the (N, 12) / (N, 4) / (N, 8) float32 columns the Python interface documents
    assert [abi.BsdfQuery.n.offset, abi.BsdfQuery.prim.offset, abi.BsdfQuery.v.offset, abi.BsdfQuery.etaI.offset,
            abi.BsdfQuery.l.offset, abi.BsdfQuery.etaO.offset] == [0, 12, 16, 28, 32, 44]
    assert [abi.BsdfSampled.l.offset, abi.BsdfSampled.pdf.offset, abi.BsdfSampled.f.offset,
            abi.BsdfSampled.type.offset] == [0, 12, 16, 28]
    m = re.search(r"REFLECTED (\d+) TRANSMITTED (\d+) SPECULAR (\d+)", out)
    assert tuple(int(x) for x in m.groups()) == (abi.BSDF_REFLECTED, abi.BSDF_TRANSMITTED, abi.BSDF_SPECULAR)


def test_entry_points_are_declared_and_exported():
    text = open(HEADER).read()
    for name in ("tb200_bsdf_eval", "tb200_bsdf_sample"):
        assert re.search(r"\bint %s\(" % name, text), name
        assert name in abi.EXPORTS
    lib = tb.load_library()
    assert hasattr(lib, "tb200_bsdf_eval") and hasattr(lib, "tb200_bsdf_sample")


def test_bsdf_queries_packs_the_records():
    torch = pytest.importorskip("torch")
    n = 7
    rng = np.random.default_rng(1)
    prims = torch.tensor([-1, 0, 5, 2 ** 31 - 1, -2 ** 31, 4095, 123456789], dtype=torch.int32)
    nn, v, l = (torch.from_numpy(rng.normal(size=(n, 3)).astype(F32)) for _ in range(3))
    eta_i = torch.from_numpy(rng.random(n).astype(F32))
    q = tb.bsdf_queries(prims, nn, v, eta_i, 1.5, l)
    assert q.dtype == torch.float32 and tuple(q.shape) == (n, 12) and q.is_contiguous() and q.device == prims.device
    rec = np.ascontiguousarray(q.numpy()).view(np.uint8).reshape(n, 48)
    for i in range(n):
        r = abi.BsdfQuery.from_buffer_copy(rec[i].tobytes())
        assert r.prim == int(prims[i])           # the int32 bits survive, NaN patterns included
        assert list(r.n) == nn[i].tolist() and list(r.v) == v[i].tolist() and list(r.l) == l[i].tolist()
        assert r.etaI == eta_i[i].item() and r.etaO == F32(1.5)
    # l defaults to zeros; the etas may be scalars
    q = tb.bsdf_queries(prims, nn, v, 1.0, 2.0)
    assert (q[:, 8:11] == 0).all() and (q[:, 7] == 1).all() and (q[:, 11] == 2).all()
    assert (q[:, 3].view(torch.int32) == prims).all()
    with pytest.raises(ValueError):
        tb.bsdf_queries(prims.long(), nn, v, 1.0, 1.0)
    with pytest.raises(ValueError):
        tb.bsdf_queries(prims, nn[:, :2], v, 1.0, 1.0)
    with pytest.raises(ValueError):
        tb.bsdf_queries(prims, nn, v, eta_i.double(), 1.0)


def _edge_values():
    x = [0.0, -0.0, 0.5, -0.5, 12.5, float(np.nextafter(F32(12.5), F32(0))), float(np.nextafter(F32(12.5), F32(20))),
         1.0, 1.5, 50.0, -12.5, np.nan, np.inf, -np.inf, 1e-45, 1e30, float(np.nextafter(F32(0.5), F32(1)))]
    return np.array(x, F32)


def test_material_ior_matches_restatement():
    lib = refdrv.load_port()
    ev = _edge_values()
    rng = np.random.default_rng(3)
    spec = np.concatenate([ev, rng.uniform(-1, 13, 2000).astype(F32)])
    eta = np.concatenate([ev, np.array([1.5, 2.0, 1e-30], F32)])
    E, S = np.meshgrid(eta, spec, indexing="ij")
    E, S = E.ravel(), S.ravel()
    got = tb.material_ior(E, S)
    assert got.dtype == F32 and got.shape == E.shape
    want = np.empty_like(got)
    m = abi.Material.default()
    for k in range(E.size):
        m.eta, m.specular = float(E[k]), float(S[k])
        want[k] = lib.oracle_material_ior(C.byref(m))
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    assert same.all(), (E[~same][:5], S[~same][:5], got[~same][:5], want[~same][:5])
    # the reference's default material: eta 0, specular 0.5 -> 1.5 (as near as float32 gets)
    assert abs(float(tb.material_ior(0.0, 0.5)) - 1.5) < 1e-6
    assert tb.material_ior(0.0, 12.5) == np.inf and np.isnan(tb.material_ior(0.0, -0.5))
    assert tb.material_ior(np.float32(1.33), 0.5) == np.float32(1.33)
