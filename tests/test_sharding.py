"""N>1 host logic on CPU (gloo, world_size 2): each rank renders ITS shard of the image with the
oracle (the product has no CPU path), the accumulators are sum-reduced onto rank 0 exactly as
bench.py does with NCCL, and the result must equal the unsharded oracle image."""
import os
import socket
import sys

import numpy as np
import pytest

import tinsel_b200 as tb
from tinsel_b200 import sharding
import refdrv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_shards_partition_the_image():
    for h in (1, 3, 4, 5, 70, 256, 1080):
        for n in (1, 2, 3, 8):
            rows = sorted(r for s in range(n) for r in sharding.shard_rows(h, s, n))
            assert rows == list(range(h)), (h, n)
    assert sharding.shard_rows(10, 0, 2) == [0, 1, 2, 3, 8, 9]
    assert sharding.shard_rows(10, 1, 2) == [4, 5, 6, 7]
    assert sum(sharding.shard_sample_count(100, 70, s, 3, 2) for s in range(3)) == 100 * 70 * 2


def _worker(rank, world, port, w, h, spp, out_path):
    import torch
    import torch.distributed as dist
    for p in (ROOT, os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    oracle = refdrv.PortScene.from_snapshot(tb.scene_path("cornell"))
    oracle.set_size(w, h)
    # render only this rank's rows: per-sample radiance -> filter splat of the owned samples
    acc = np.zeros((h, w, 4), np.float32)
    mine = set(sharding.shard_rows(h, rank, world))
    lib = oracle.lib
    for k in range(spp):
        rad, ras = oracle.trace_frame(k, 2)
        for j in sorted(mine):
            for i in range(w):
                _splat(acc, oracle.options, ras[j, i, 0], ras[j, i, 1], rad[j, i], lib)
    t = torch.from_numpy(acc)
    dist.reduce(t, dst=0, op=dist.ReduceOp.SUM)
    if rank == 0:
        np.save(out_path, t.numpy())
    dist.destroy_process_group()
    oracle.close()


def _splat(acc, o, rx, ry, c, lib):
    """AddSample (render.cpp:401-445) in numpy-free python, using the oracle's filter hook."""
    h, w = acc.shape[:2]
    fw = o.filterWidth
    for x in range(max(0, int(rx - fw)), min(int(rx + fw), w - 1) + 1):
        for y in range(max(0, int(ry - fw)), min(int(ry + fw), h - 1) + 1):
            wt = lib.oracle_filter_eval(o.filterType, fw, o.filterFalloff, o.filterOffset,
                                        np.float32(np.float32(x) - rx), np.float32(np.float32(y) - ry))
            acc[y, x, :3] += np.float32(wt) * c
            acc[y, x, 3] += np.float32(wt)


def test_two_rank_gloo_reduce_equals_full_image(tmp_path):
    import torch.multiprocessing as mp
    import subprocess
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "port"])
    w, h, spp = 24, 18, 2
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "sum.npy")
    mp.spawn(_worker, args=(2, port, w, h, spp, out), nprocs=2, join=True)
    got = np.load(out)
    oracle = refdrv.PortScene.from_snapshot(tb.scene_path("cornell"))
    oracle.set_size(w, h)
    full = oracle.render_seeded(0, spp, 1)
    oracle.close()
    assert np.allclose(got, full, rtol=1e-5, atol=1e-6)
    assert got[..., 3].sum() > 0


# ---------------------------------------------------------------------------------------------------
# Owner-computes row slabs (tb200_create_multi / tb200_set_slab): the host rule, and the whole scheme
# on CPU -- every rank traces its slab plus the filter's reach with the oracle, splats into the rows it
# owns only, and the ranks' rows are GATHERED (no reduction): the result must be the unsharded image.
# ---------------------------------------------------------------------------------------------------
def test_slab_rule_matches_the_c_abi():
    import ctypes as C
    lib = tb.load_library()
    for h in (1, 3, 4, 5, 70, 256, 1024, 1080, 2048):
        for n in (1, 2, 3, 4, 8):
            covered = []
            for k in range(n):
                a, b = C.c_int(), C.c_int()
                lib.tb200_slab_rows(h, k, n, C.byref(a), C.byref(b))
                assert (a.value, b.value) == sharding.slab_rows(h, k, n), (h, k, n)
                assert a.value % 4 == 0 or a.value == h
                covered.extend(range(a.value, a.value + b.value))
                for fw in (0.0, 0.75, 1.0, 3.5):
                    t0, tn = C.c_int(), C.c_int()
                    lib.tb200_slab_traced_rows(h, a.value, b.value, fw, C.byref(t0), C.byref(tn))
                    assert (t0.value, tn.value) == sharding.slab_traced_rows(h, a.value, b.value, fw)
                    if b.value:
                        assert t0.value <= a.value and t0.value + tn.value >= a.value + b.value
            assert covered == list(range(h)), (h, n)
    assert sharding.slab_rows(1024, 3, 8) == (384, 128)
    assert sharding.slab_traced_rows(1024, 384, 128, 1.0) == (382, 132)   # reach = ceil(1) + 1 = 2 rows
    assert sharding.slab_traced_rows(1024, 0, 128, 0.75) == (0, 130)


def test_slab_traced_rows_of_unbounded_widths_stay_in_the_image():
    """tb200_slab_traced_rows takes a width that no fill_params has checked: infinite, NaN and huge widths must give
    traced rows inside the image (the whole image, or the slab alone for NaN), never an int overflow."""
    import ctypes as C
    lib = tb.load_library()
    for fw in (float("inf"), float("-inf"), float("nan"), 1e30, -1e30, 2.0 ** 30, 3e38):
        for h, row0, rows in ((1, 0, 1), (70, 0, 68), (70, 32, 20), (1080, 1076, 4), (2048, 512, 512), (64, 13, 0)):
            t0, tn = C.c_int(), C.c_int()
            lib.tb200_slab_traced_rows(h, row0, rows, fw, C.byref(t0), C.byref(tn))
            what = (fw, h, row0, rows, t0.value, tn.value)
            assert (t0.value, tn.value) == sharding.slab_traced_rows(h, row0, rows, fw), what
            assert 0 <= t0.value <= h and 0 <= tn.value and t0.value + tn.value <= h, what
            if rows:
                assert t0.value <= row0 and t0.value + tn.value >= row0 + rows, what
            if fw > 1e6:
                assert (t0.value, tn.value) == ((0, h) if rows else (max(0, row0 - 2 ** 30 - 1), 0)), what


def _slab_worker(rank, world, port, w, h, spp, out_path):
    import torch
    import torch.distributed as dist
    for p in (ROOT, os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    oracle = refdrv.PortScene.from_snapshot(tb.scene_path("cornell"))
    oracle.set_size(w, h)
    row0, rows = sharding.slab_rows(h, rank, world)
    t0, tn = sharding.slab_traced_rows(h, row0, rows, oracle.options.filterWidth)
    full = np.zeros((h, w, 4), np.float32)
    for k in range(spp):
        rad, ras = oracle.trace_frame(k, 2)
        for j in range(t0, t0 + tn):
            for i in range(w):
                _splat(full, oracle.options, ras[j, i, 0], ras[j, i, 1], rad[j, i], oracle.lib)
    # owned rows only (the halo rows' partial sums are discarded), padded to the largest slab: gloo's
    # gather wants equal shapes
    sizes = [sharding.slab_rows(h, r, world)[1] for r in range(world)]
    mine = torch.zeros((max(sizes), w, 4), dtype=torch.float32)
    mine[:rows] = torch.from_numpy(full[row0:row0 + rows])
    parts = [torch.zeros_like(mine) for _ in range(world)] if rank == 0 else None
    dist.gather(mine, parts, dst=0)
    if rank == 0:
        np.save(out_path, torch.cat([parts[r][:sizes[r]] for r in range(world)], 0).numpy())
    dist.destroy_process_group()
    oracle.close()


def test_two_rank_row_slabs_gather_to_the_full_image(tmp_path):
    import torch.multiprocessing as mp
    import subprocess
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "port"])
    w, h, spp = 20, 22, 2      # 22 rows: slabs of 8 and 14 rows, cut at a tile row
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "gather.npy")
    mp.spawn(_slab_worker, args=(2, port, w, h, spp, out), nprocs=2, join=True)
    got = np.load(out)
    oracle = refdrv.PortScene.from_snapshot(tb.scene_path("cornell"))
    oracle.set_size(w, h)
    full = oracle.render_seeded(0, spp, 1)
    oracle.close()
    # same contributions per pixel (the halo samples are bit-identical duplicates), another summation order
    assert np.allclose(got, full, rtol=1e-5, atol=1e-6)
    assert got.shape == full.shape and got[..., 3].sum() > 0
