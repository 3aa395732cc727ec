"""bsdf_eval_pdf with the view terms computed once per bounce (tb_shade.cuh: bsdf_view and the bsdf_eval_pdf overload
that takes them, which the lane-owned wavefront kernel calls) against bsdf_eval_pdf itself, bit for bit: every f and
pdf, NaNs included (a NaN matches only a NaN).

tests/bsdf_view_harness.cu runs one case per thread in both instantiations the kernels use, TB_FEAT_ALL and
TB_FEAT_NONE, each on every case (the two evaluations are one instantiation's, whatever the material holds).  The
cases are test_bsdf_gpu's materials and directions, plus the edges that the hoisted evaluation treats apart:
  * dot(N, V) <= 0 (V flipped or perpendicular), where the view terms take their other branches;
  * L + V == 0 (L == -V), and L + V nonzero with |L + V|^2 == 0 in float32, where bsdf_pdf's half vector falls back to
    0 and bsdf_eval's normalize gives inf and NaN;
  * a NaN or an infinity in N, V or L."""
import ctypes as C

import numpy as np
import pytest

import cuda_harness
import test_bsdf_gpu as bsdf

F32 = np.float32
OUT_DTYPE = np.dtype([("f", "<f4", 3), ("pdf", "<f4"), ("fv", "<f4", 3), ("pdfv", "<f4")])
BATCHES = 4

_lib = None


def harness():
    global _lib
    if _lib is None:
        lib = C.CDLL(cuda_harness.harness_path("bsdf_view_harness"))
        lib.view_run.restype = C.c_int
        lib.view_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        _lib = lib
    return _lib


def with_edges(c, seed):
    """test_bsdf_gpu's cases with a share of them moved to the edges of the module docstring; returns (cases, kinds)."""
    rng = np.random.default_rng(seed)
    c = c.copy()
    n = c.size
    kind = rng.integers(0, 8, n)
    N, V, L = c["n"].copy(), c["v"].copy(), c["l"].copy()
    V[kind == 1] *= F32(-1)                                   # dot(N, V) < 0 (or -0 where V is perpendicular)
    L[kind == 2] = -V[kind == 2]                              # L + V == 0
    # |L + V|^2 underflows to 0 with L + V != 0: V = (1, 2e-30, 0), L = (-1, -1e-30, 0), in N's frame of axes
    tiny = kind == 3
    V[tiny] = np.array([1.0, 2e-30, 0.0], F32)
    L[tiny] = np.array([-1.0, -1e-30, 0.0], F32)
    N[tiny] = np.array([0.0, 0.0, 1.0], F32) * np.where(rng.random((int(tiny.sum()), 1)) < 0.5, F32(1), F32(-1))
    bad = np.array([np.nan, np.inf, -np.inf], F32)[rng.integers(0, 3, n)]
    comp = rng.integers(0, 3, n)
    for k, arr in ((4, N), (5, V), (6, L)):
        sel = np.flatnonzero(kind == k)
        arr[sel, comp[sel]] = bad[sel]
    c["n"], c["v"], c["l"] = N, V, L
    return c, kind


def _device(dmats, c, all_features):
    import torch
    dm = torch.from_numpy(dmats.reshape(-1)).cuda()
    dc = torch.from_numpy(np.ascontiguousarray(c).view(np.uint8)).cuda()
    do = torch.zeros(c.size * OUT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    rc = harness().view_run(dm.data_ptr(), dc.data_ptr(), c.size, do.data_ptr(), int(all_features))
    assert rc == 0, "view_run: cudaError %d" % rc
    return do.cpu().numpy().view(OUT_DTYPE)


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def test_bsdf_view_harness_compiles_for_sm90a():
    """The harness against the headers as they are (no GPU needed)."""
    cuda_harness.harness_path("bsdf_view_harness")


def test_edge_cases_are_there():
    """The edges the module docstring names occur in every batch (no GPU needed)."""
    mats, c, _ = bsdf.make_cases(20261016)
    c, _ = with_edges(c, 1)
    N, V, L = (c[k].astype(np.float64) for k in ("n", "v", "l"))
    with np.errstate(invalid="ignore"):
        ndv = (c["n"] * c["v"]).sum(1, dtype=F32)
    s = (c["l"] + c["v"]).astype(F32)
    m = (s * s).sum(1, dtype=F32)
    assert (ndv < 0).sum() > 1000 and (ndv == 0).sum() > 100
    assert ((m == 0) & (s == 0).all(1)).sum() > 1000
    assert ((m == 0) & (s != 0).any(1)).sum() > 1000
    for arr in (N, V, L):
        assert np.isnan(arr).any(1).sum() > 100 and np.isinf(arr).any(1).sum() > 100


@pytest.mark.gpu
def test_bsdf_view_matches_bsdf_eval_pdf():
    totals = {"TB_FEAT_ALL": 0, "TB_FEAT_NONE": 0}
    ran = 0
    first = None
    for b in range(BATCHES):
        mats, c, _ = bsdf.make_cases(20261016 + b)
        c, kind = with_edges(c, b)
        dmats, _, _, _ = bsdf.make_materials(mats, 2)
        for inst in totals:
            dev = _device(dmats, c, inst == "TB_FEAT_ALL")
            bad = ~(_same(dev["f"], dev["fv"]).all(1) & _same(dev["pdf"], dev["pdfv"]))
            totals[inst] += int(bad.sum())
            if bad.any() and first is None:
                k = int(np.argmax(bad))
                first = "%s, batch %d, edge kind %d: material %s, case %s: %s" % (inst, b, kind[k], mats[c["mat"][k]], c[k], dev[k])
        ran += c.size
    print("bsdf_view: %d cases per instantiation; mismatches %s" % (ran, totals))
    assert not any(totals.values()), "mismatches %s, first: %s" % (totals, first)
