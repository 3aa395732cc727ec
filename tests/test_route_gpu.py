"""Which of the seven wavefront kernels a scene runs (kernels.cu: wavefront2_route, launch_wavefront2), pinned by
name through tb200_last_kernel.  Every kernel gives the same bits, so no image test notices a scene sent to the
wrong one: this test restates the rule and checks the kernel that ran against it, under the default knobs and
every scheduler variant of schedenv, at a small launch and at one of at least six samples per slot."""
import math

import pytest
import torch

import tinsel_b200 as tb
from tinsel_b200 import abi
import fuzzscene
import schedenv

pytestmark = pytest.mark.gpu

SMALL = (64, 64)   # one frame of these is a small launch
TUNE_SIZE = (256, 256)   # 4 frames of these are the 2^18 image samples a launch needs to advance the tuner
SETTINGS = [None] + [(s, c) for s in schedenv.SCHEDS for c in schedenv.CTAS]


@pytest.fixture(autouse=True)
def default_knobs():
    with schedenv.knobs():
        yield


@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    paths = {n: tb.scene_path(n) for n in ("cornell", "glass", "veach")}
    paths["big"] = str(tmp_path_factory.mktemp("route") / "big.tsnap")
    assert max(fuzzscene.make_mesh_scene(0, paths["big"], "big")["tris"]) > 4096
    return paths


@pytest.fixture(scope="module")
def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def facts(path):
    """What the route reads from a scene: shadow rays per hit, the largest mesh's triangles, whether the scene BVH
    has a leaf for that mesh's primitive (its box), and whether the scene has any TB_FEAT_* feature."""
    snap = tb.Snapshot(path)
    s = snap.scene.contents
    prims = [s.primitives[i] for i in range(s.numPrimitives)]
    tris = [s.meshes[m].numIndices // 3 for m in range(s.numMeshes)]
    big, big_tris = -1, 0
    for i, p in enumerate(prims):
        if p.type == abi.MESH and 0 <= p.mesh < s.numMeshes and tris[p.mesh] > big_tris:
            big, big_tris = i, tris[p.mesh]
    box = any(s.bvhNodes[n].right_leaf >> 31 and s.bvhNodes[n].left == big for n in range(s.numBvhNodes)) and big >= 0
    features = bool(s.sky.probeValid) or any(
        bytes(p.start) != bytes(p.end) or p.material.transmission != 0.0 or p.material.subsurface != 0.0
        or p.material.clearcoat != 0.0 or any(a != 0.0 for a in p.material.absorption) for p in prims)
    out = dict(numNee=int(bool(s.sky.probeValid)) + sum(max(p.lightSamples, 0) for p in prims),
               maxTris=max(tris, default=0), box=box, features=features)
    snap.close()
    return out


def route(f, knobs):
    """The per-scene part of the rule, from the scene's facts and the knob settings schedenv.knobs applied."""
    sched, split, cta, queues, spec = (knobs.get(k) for k in ("SCHED", "SPLIT", "CTA", "QUEUES", "SPECIALIZE"))
    hard = {"hard": True, "free": False}.get(sched, f["numNee"] > 1 and f["maxTris"] <= 4096)
    wide = {"768": True, "512": False}.get(cta, not hard and f["maxTris"] > 4096)
    in_use = f["box"] and (f["maxTris"] > 4096 or split == "1") and split != "0"
    return dict(hard=hard, wide=wide, split=not hard and in_use, tune=not hard and in_use and split is None,
                lanes={"ring": 0, "lanes": 2}.get(queues, 1), specialized=not f["features"] and spec != "0")


def kernel(r, samples, num_sms):
    """The per-launch part: the kernel a launch of `samples` samples runs on route r."""
    small = samples < 6 * num_sms * 1024
    if r["wide"]:
        return "wf2_l2.split" if r["split"] else "wf2_l2.generic"
    if not r["hard"] and not r["split"] and (r["lanes"] == 2 or (r["lanes"] == 1 and not small)):
        return "wf2_lq.specialized" if r["specialized"] else "wf2_lq.generic"
    return "wf2_smem.hard" if r["hard"] else "wf2_smem.split" if r["split"] else "wf2_smem.generic"


def run(path, size, spp):
    """The kernel each launch ran: one timed launch (render_device) of size[0] x size[1] x k samples per k in spp,
    on one renderer."""
    snap = tb.Snapshot(path)
    cam, opt = snap.camera, snap.options
    opt.width, opt.height = size
    r = tb.Renderer(snap.scene)
    r.Init(*size)
    names = []
    for frames in spp:
        r.render_device(cam, opt, frames)
        names.append(r.last_kernel())
    r.close()
    snap.close()
    return names


def large_spp(size, num_sms):
    return math.ceil(6 * num_sms * 1024 / (size[0] * size[1]))


def test_defaults(scenes, num_sms):
    """The default knobs on the scenes whose routes are documented."""
    spp = large_spp(SMALL, num_sms)
    assert run(scenes["cornell"], SMALL, [1])[0] == "wf2_smem.generic"
    assert run(scenes["cornell"], SMALL, [spp])[0] == "wf2_lq.specialized"
    assert run(scenes["glass"], SMALL, [1])[0] == "wf2_smem.generic"
    assert run(scenes["glass"], SMALL, [spp])[0] == "wf2_lq.generic"
    assert run(scenes["veach"], SMALL, [1, spp]) == ["wf2_smem.hard"] * 2


@pytest.mark.parametrize("setting", SETTINGS, ids=["default"] + ["%s-%s" % s for s in SETTINGS[1:]])
@pytest.mark.parametrize("name", ["cornell", "glass", "veach", "big"])
def test_route_matches_rule(name, setting, scenes, num_sms):
    f = facts(scenes[name])
    for spp in (1, large_spp(SMALL, num_sms)):
        with schedenv.sched_env(*setting) if setting else schedenv.knobs() as knobs:
            want = kernel(route(f, knobs), SMALL[0] * SMALL[1] * spp, num_sms)
            ran = run(scenes[name], SMALL, [spp])[0]
        assert ran == want, "%s %s, %d spp: ran %s, the rule says %s (facts %s)" % (name, setting, spp, ran, want, f)


def test_tuner_default(scenes):
    """The tuner times phase 1 with the split queue and phase 2 without it, then keeps the faster."""
    assert route(facts(scenes["big"]), {})["tune"]
    ran = run(scenes["big"], TUNE_SIZE, [4] * 6)
    assert ran[:3] == ["wf2_l2.split", "wf2_l2.split", "wf2_l2.generic"], ran
    assert ran[3] in ("wf2_l2.split", "wf2_l2.generic") and ran[3:] == [ran[3]] * 3, ran


@pytest.mark.parametrize("split,name", [("0", "wf2_l2.generic"), ("1", "wf2_l2.split")])
def test_tuner_off_when_split_is_set(split, name, scenes):
    with schedenv.knobs(SPLIT=split):
        assert run(scenes["big"], TUNE_SIZE, [4] * 6) == [name] * 6


@pytest.mark.parametrize("size", ["small", "large"])
def test_tuner_phase2_takes_rule_2(size, scenes, num_sms):
    """With 512-thread CTAs the split queue runs on wf2_smem; phase 2 turns it off, so rule 2 applies: a launch of
    at least six samples per slot runs the lane-owned kernel, a smaller one the generic ring kernel."""
    spp = 4 if size == "small" else large_spp(TUNE_SIZE, num_sms)
    samples = TUNE_SIZE[0] * TUNE_SIZE[1] * spp
    assert samples >= 1 << 18 and (samples < 6 * num_sms * 1024) == (size == "small")
    f = facts(scenes["big"])
    with schedenv.knobs(CTA="512") as knobs:
        without = kernel(dict(route(f, knobs), split=False), samples, num_sms)
        ran = run(scenes["big"], TUNE_SIZE, [spp] * 6)
    assert without == ("wf2_smem.generic" if size == "small" else
                       "wf2_lq.generic" if f["features"] else "wf2_lq.specialized")
    assert ran[:3] == ["wf2_smem.split", "wf2_smem.split", without], ran
    assert ran[3] in ("wf2_smem.split", without) and ran[3:] == [ran[3]] * 3, ran
