"""The emitter and probe sample queries without a GPU: the tb200_emitter_query, tb200_emitter_sampled and
tb200_probe_sampled records of include/tinsel_b200.h, the entry points, the packing of tinsel_b200.emitter_queries, and
the CPU arms the device's queries are checked against (tests/emitter_oracle.cpp) against the restatement's single-call
oracle_primitive_sample and oracle_probe_sample."""
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
import emitteroracle
import fuzzscene
import lightoracle

F32 = np.float32
HEADER = tb.ROOT + "/include/tinsel_b200.h"
RECORDS = {"tb200_emitter_query": (abi.EmitterQuery, 8), "tb200_emitter_sampled": (abi.EmitterSampled, 32),
           "tb200_probe_sampled": (abi.ProbeSampled, 32)}


def test_edge_seeds_draw_what_they_claim():
    for (k, value), seed in emitteroracle.EDGE_SEEDS.items():
        assert emitteroracle.randf(seed, 4)[k] == value, (k, value, seed)
    for seed in emitteroracle.COL_END_SEEDS:
        assert emitteroracle.randf(seed, 2)[1] == 1.0


def test_records_match_the_header():
    src = ['#include <stddef.h>', '#include <stdio.h>', '#include "tinsel_b200.h"', 'int main(void)', '{']
    for name, (cls, _) in RECORDS.items():
        src.append('    printf("%s %%zu\\n", sizeof(%s));' % (name, name))
        for field, _ in cls._fields_:
            src.append('    printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (name, field, name, field))
    src += ['    return 0;', '}']
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        with open(c, "w") as f:
            f.write("\n".join(src) + "\n")
        subprocess.check_call(["cc", "-I", os.path.dirname(HEADER), c, "-o", exe])
        got = dict(re.findall(r"^(\S+) (\d+)$", subprocess.check_output([exe], text=True), re.M))
    for name, (cls, size) in RECORDS.items():
        assert int(got[name]) == C.sizeof(cls) == size, name
        for field, _ in cls._fields_:
            assert int(got[name + "." + field]) == getattr(cls, field).offset, (name, field)
    # the float32 columns Renderer.sample_emitters / sample_probe slice
    assert [abi.EmitterSampled.pos.offset, abi.EmitterSampled.normal.offset] == [0, 16]
    assert [abi.ProbeSampled.dir.offset, abi.ProbeSampled.pdf.offset, abi.ProbeSampled.color.offset] == [0, 12, 16]


def test_entry_points_are_declared_and_exported():
    text = open(HEADER).read()
    for name in ("tb200_sample_emitters", "tb200_sample_probe"):
        assert re.search(r"\bint %s\(" % name, text), name
        assert name in abi.EXPORTS
    lib = tb.load_library()
    assert hasattr(lib, "tb200_sample_emitters") and hasattr(lib, "tb200_sample_probe")


def test_emitter_queries_packs_the_records():
    torch = pytest.importorskip("torch")
    prims = torch.tensor([-1, 0, 5, 2 ** 31 - 1, -2 ** 31, 4095, 123456789], dtype=torch.int32)
    t = torch.tensor([0.0, -0.0, 0.5, 1.0, -3.0, 1e30, float("nan")], dtype=torch.float32)
    q = tb.emitter_queries(prims, t)
    assert q.dtype == torch.float32 and tuple(q.shape) == (7, 2) and q.is_contiguous() and q.device == prims.device
    rec = np.ascontiguousarray(q.numpy()).view(np.uint8).reshape(7, 8)
    for i in range(7):
        r = abi.EmitterQuery.from_buffer_copy(rec[i].tobytes())
        assert r.prim == int(prims[i])                  # the int32 bits survive, NaN patterns included
        assert np.array(r.time, F32).view(np.uint32) == t[i:i + 1].numpy().view(np.uint32)[0]
    q = tb.emitter_queries(prims, 0.25)
    assert (q[:, 1] == 0.25).all() and (q[:, 0].view(torch.int32) == prims).all()
    with pytest.raises(ValueError):
        tb.emitter_queries(prims.long(), t)
    with pytest.raises(ValueError):
        tb.emitter_queries(prims[:, None], t)
    with pytest.raises(ValueError):
        tb.emitter_queries(prims, t[:3])
    with pytest.raises(ValueError):
        tb.emitter_queries(prims, t.double())
    with pytest.raises(ValueError):
        tb.emitter_queries(prims, t[:, None])


def _snapshots():
    return sorted(glob.glob(os.path.join(tb.SCENE_DIR, "*.tsnap")))


def _seeds(rng, n):
    return np.concatenate([np.array(list(emitteroracle.EDGE_SEEDS.values()), np.uint32),
                           rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)])


@pytest.mark.parametrize("path", _snapshots(), ids=lambda p: os.path.basename(p)[:-6])
def test_batch_oracles_match_the_single_calls(path):
    snap = tb.Snapshot(path)
    try:
        sc = snap.scene.contents
        rng = np.random.default_rng(31)
        seeds = _seeds(rng, 24)
        lights = [i for i in range(sc.numPrimitives) if sc.primitives[i].lightSamples > 0]
        for prim in lights:
            for time in (F32(0.0), F32(0.5), F32(1.0), F32(-2.0)):
                rec = np.zeros((len(seeds), 2), F32)
                rec[:, 0] = np.int32(prim).view(F32)
                rec[:, 1] = time
                got = emitteroracle.sample_emitters(snap.scene, rec, seeds)
                assert (got[:, 3] == 0).all() and (got[:, 7] == 0).all()
                for k, s in enumerate(seeds):
                    pos, nrm = emitteroracle.primitive_sample(snap.scene, prim, time, s)
                    assert (got[k, 0:3].view(np.uint32) == pos.view(np.uint32)).all(), (prim, time, s)
                    assert (got[k, 4:7].view(np.uint32) == nrm.view(np.uint32)).all(), (prim, time, s)
        # non-lights, out-of-range prims: zeros
        others = [i for i in range(sc.numPrimitives) if i not in lights] + [-1, sc.numPrimitives, -2 ** 31]
        rec = np.zeros((len(others), 2), F32)
        rec[:, 0] = np.array(others, np.int32).view(F32)
        assert (emitteroracle.sample_emitters(snap.scene, rec, seeds[:len(others)]).view(np.uint32) == 0).all()
        got = emitteroracle.sample_probe(snap.scene, seeds)
        if not sc.sky.probeValid:
            assert (got.view(np.uint32) == 0).all()
        else:
            for k, s in enumerate(seeds):
                d, pdf, c = emitteroracle.probe_sample(snap.scene, s)
                want = np.concatenate([d, [pdf], c, [0]]).astype(F32)
                assert (got[k].view(np.uint32) == want.view(np.uint32)).all(), s
    finally:
        snap.close()


def test_probe_batch_oracle_on_a_probe_with_black_rows(tmp_path):
    path = str(tmp_path / "p.tsnap")
    assert fuzzscene.make_mesh_scene(0, path, "probe")["probe"]
    snap = tb.Snapshot(path)
    try:
        seeds = np.concatenate([_seeds(np.random.default_rng(32), 200), np.array(emitteroracle.COL_END_SEEDS, np.uint32)])
        got = emitteroracle.sample_probe(snap.scene, seeds)
        for k, s in enumerate(seeds):
            d, pdf, c = emitteroracle.probe_sample(snap.scene, s)
            want = np.concatenate([d, [pdf], c, [0]]).astype(F32)
            assert ((got[k].view(np.uint32) == want.view(np.uint32)) | (np.isnan(got[k]) & np.isnan(want))).all(), s
    finally:
        snap.close()


def test_per_slot_oracle_with_one_seed_per_record_and_slot_is_sample_lights_on_one_slot_scenes():
    # with a single slot (cornell: one light sample and no probe; envmini: the probe and no light), the per-slot arm
    # draws from the same Random as sample_lights, so the two must agree bit for bit
    for name in ("cornell", "envmini"):
        snap = tb.Snapshot(tb.scene_path(name))
        try:
            assert emitteroracle.num_slots(snap.scene.contents) == 1, name
            rng = np.random.default_rng(33)
            n = 64
            rec = np.zeros((n, 16), F32)
            rec[:, 0:3] = rng.normal(size=(n, 3)) * (1, 0.2, 1) + (0, 0.5, 0)
            nrm = rng.normal(size=(n, 3))
            rec[:, 4:7] = nrm / np.linalg.norm(nrm, axis=1, keepdims=True)
            rec[:, 8:11] = rec[:, 4:7]
            rec[:, 11], rec[:, 12] = 1.0, 1.5
            rec[:, 7] = np.zeros(n, np.int32).view(F32)
            seeds = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
            rad, hit, acc = emitteroracle.sample_lights_per_slot(snap.scene, rec, seeds)
            want = lightoracle.sample_lights(snap.scene, rec, seeds)
            assert (rad.view(np.uint32) == want.view(np.uint32)).all(), name
            assert hit.shape == (n, 1) and (hit >= -1).all() and (acc <= (hit >= 0) ^ (name == "envmini")).all()
        finally:
            snap.close()
