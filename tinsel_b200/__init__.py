"""tinsel_b200 -- H100-native wavefront path tracer behind tinsel's Renderer interface.

This package is the Python-side host mirror used by the tests and bench.py: it loads the
in-tree C-ABI library (tinsel_b200/libtinsel_b200.so: hand-written sm_90a kernels + host
runtime, built by tinsel_b200/build.py) and wraps it in a `Renderer` with the reference's
`Init(width, height)` / `Render(camera, options, output)` shape (src/render.h:66-73).
There is no CPU fallback: if the library or a CUDA device is missing, creation fails loudly.
"""
import ctypes as C
import os

import numpy as np

from . import abi
from .abi import Camera, Options, Scene, Stats  # noqa: F401

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libtinsel_b200.so")
ROOT = os.path.dirname(_PKG)
SCENE_DIR = os.path.join(ROOT, "scenes")

_lib = None


class TinselB200Error(RuntimeError):
    pass


def load_library():
    """Loads libtinsel_b200.so (never builds implicitly: use tinsel_b200.build.build_native)."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("TINSEL_B200_LIB", LIB_PATH)   # development: alternative builds of the same library
    if not os.path.exists(path):
        raise TinselB200Error(
            "native library %s is missing: run `python -m tinsel_b200.build` (needs nvcc); "
            "there is no CPU fallback" % path)
    lib = C.CDLL(path)
    f32p = C.POINTER(C.c_float)
    lib.tb200_create.restype = C.c_void_p
    lib.tb200_create.argtypes = [C.POINTER(Scene), C.c_int]
    lib.tb200_init.restype = C.c_int
    lib.tb200_init.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.tb200_render.restype = C.c_int
    lib.tb200_render.argtypes = [C.c_void_p, C.POINTER(Camera), C.POINTER(Options), f32p]
    lib.tb200_render_device.restype = C.c_int
    lib.tb200_render_device.argtypes = [C.c_void_p, C.POINTER(Camera), C.POINTER(Options), C.c_int, C.c_int, C.c_int]
    lib.tb200_set_shard.restype = C.c_int
    lib.tb200_set_shard.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.tb200_set_stream.restype = C.c_int
    lib.tb200_set_stream.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    lib.tb200_create_multi.restype = C.c_void_p
    lib.tb200_create_multi.argtypes = [C.POINTER(Scene), C.POINTER(C.c_int), C.c_int]
    lib.tb200_num_devices.restype = C.c_int
    lib.tb200_num_devices.argtypes = [C.c_void_p]
    lib.tb200_slab_rows.restype = None
    lib.tb200_slab_rows.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.tb200_divisor_magic.restype = None
    lib.tb200_divisor_magic.argtypes = [C.c_uint, C.POINTER(C.c_uint), C.POINTER(C.c_uint)]
    lib.tb200_slab_traced_rows.restype = None
    lib.tb200_slab_traced_rows.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.tb200_set_slab.restype = C.c_int
    lib.tb200_set_slab.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.tb200_pin_output.restype = C.c_int
    lib.tb200_pin_output.argtypes = [C.c_void_p, f32p, C.c_size_t]
    lib.tb200_unpin_output.restype = C.c_int
    lib.tb200_unpin_output.argtypes = [C.c_void_p]
    lib.tb200_gather_device.restype = C.c_int
    lib.tb200_gather_device.argtypes = [C.c_void_p]
    lib.tb200_bind_accumulator.restype = C.c_int
    lib.tb200_bind_accumulator.argtypes = [C.c_void_p, C.c_void_p]
    lib.tb200_device_accumulator.restype = C.c_void_p
    lib.tb200_device_accumulator.argtypes = [C.c_void_p]
    lib.tb200_read_accumulator.restype = C.c_int
    lib.tb200_read_accumulator.argtypes = [C.c_void_p, f32p]
    lib.tb200_render_n.restype = C.c_int
    lib.tb200_render_n.argtypes = [C.c_void_p, C.POINTER(Camera), C.POINTER(Options), C.c_int, f32p]
    lib.tb200_finish.restype = C.c_int
    lib.tb200_finish.argtypes = [C.c_void_p, C.c_float, C.c_float, f32p, C.POINTER(C.c_ubyte)]
    lib.tb200_nlm.restype = C.c_int
    lib.tb200_nlm.argtypes = [C.c_void_p, C.c_float, C.c_int, f32p]
    lib.tb200_trace_frame.restype = C.c_int
    lib.tb200_trace_frame.argtypes = [C.c_void_p, C.POINTER(Camera), C.POINTER(Options), C.c_int, f32p, f32p]
    lib.tb200_trace_rays.restype = C.c_int
    lib.tb200_trace_rays.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    lib.tb200_trace_rays_tri.restype = C.c_int
    lib.tb200_trace_rays_tri.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    lib.tb200_occluded_rays.restype = C.c_int
    lib.tb200_occluded_rays.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    lib.tb200_set_frame.restype = None
    lib.tb200_set_frame.argtypes = [C.c_void_p, C.c_int]
    lib.tb200_get_stats.restype = None
    lib.tb200_get_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
    lib.tb200_last_kernel.restype = C.c_char_p
    lib.tb200_last_kernel.argtypes = [C.c_void_p]
    lib.tb200_get_member_stats.restype = C.c_int
    lib.tb200_get_member_stats.argtypes = [C.c_void_p, C.c_int, C.POINTER(Stats), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.tb200_destroy.restype = None
    lib.tb200_destroy.argtypes = [C.c_void_p]
    lib.tb200_last_error.restype = C.c_char_p
    lib.tb200_last_error.argtypes = []
    lib.tb200_scene_cache_save.restype = C.c_int
    lib.tb200_scene_cache_save.argtypes = [C.POINTER(Scene), C.c_char_p]
    lib.tb200_create_cached.restype = C.c_void_p
    lib.tb200_create_cached.argtypes = [C.c_char_p, C.c_int]
    lib.tb200_bvh_build.restype = C.c_int
    lib.tb200_bvh_build.argtypes = [f32p, C.c_int, C.POINTER(C.c_int32), C.c_int, C.c_void_p, C.c_int, C.POINTER(abi.BvhBuildInfo)]
    lib.tb200_bvh_build_error.restype = C.c_char_p
    lib.tb200_bvh_build_error.argtypes = []
    abi.declare_snapshot_api(lib)
    _lib = lib
    return lib


def last_error():
    return load_library().tb200_last_error().decode()


def sample_seed(pixel, frame):
    return load_library().tb200_sample_seed(pixel, frame)


def scene_cache_save(scene, path):
    """Writes the device-layout scene cache of `scene` (tb200_scene_cache_save; no GPU needed)."""
    if load_library().tb200_scene_cache_save(scene, path.encode()) != 0:
        raise TinselB200Error("tb200_scene_cache_save failed: " + last_error())


def bvh_build(positions, indices, nodes, device=0):
    """Mesh BVH construction on the GPU (tb200_bvh_build): positions (nv,3) float32, indices (nt,3) int32,
    nodes: a writable array of 2*nt-1 records of 32 bytes (the reference's BVHNode).  Returns the build info."""
    lib = load_library()
    positions = np.ascontiguousarray(positions, np.float32)
    indices = np.ascontiguousarray(indices, np.int32)
    assert nodes.nbytes >= (2 * indices.shape[0] - 1) * 32 and nodes.flags["C_CONTIGUOUS"]
    info = abi.BvhBuildInfo()
    rc = lib.tb200_bvh_build(_fp(positions), positions.shape[0], indices.ctypes.data_as(C.POINTER(C.c_int32)), indices.size,
                             nodes.ctypes.data_as(C.c_void_p), device, C.byref(info))
    if rc != 0:
        raise TinselB200Error("tb200_bvh_build failed: " + lib.tb200_bvh_build_error().decode())
    return info


def scene_path(name):
    return os.path.join(SCENE_DIR, name + ".tsnap")


class Snapshot:
    """A .tsnap scene snapshot: tb200_scene + the camera and options the .tin file specified."""

    def __init__(self, path):
        self.lib = load_library()
        self.h = self.lib.tb200_snapshot_load(path.encode())
        if not self.h:
            raise TinselB200Error("cannot load snapshot %s: %s" % (path, last_error()))
        self.path = path

    @property
    def scene(self):
        return self.lib.tb200_snapshot_scene(self.h)

    @property
    def camera(self):
        return abi.copy_struct(self.lib.tb200_snapshot_camera(self.h).contents)

    @property
    def options(self):
        return abi.copy_struct(self.lib.tb200_snapshot_options(self.h).contents)

    def close(self):
        if self.h:
            self.lib.tb200_snapshot_free(self.h)
            self.h = None


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


class Renderer:
    """Host mirror of tinsel's `Renderer` (src/render.h:66-73) over the C ABI.

    Renderer(scene)            <-> CreateGpuWavefrontRenderer(const Scene*)
    Init(width, height)        <-> Renderer::Init
    Render(camera, options, o) <-> Renderer::Render: adds one sample per pixel, `o` (H,W,4 float32)
                                   receives the running sums (sum w*rgb, sum w)
    """

    def __init__(self, scene, device=0, devices=None, cache=None):
        """devices: a list of CUDA ordinals -> one renderer spread over several GPUs (tb200_create_multi).
        cache: path of a scene cache written by scene_cache_save (tb200_create_cached); `scene` is ignored."""
        self.lib = load_library()
        if cache is not None:
            self.h = self.lib.tb200_create_cached(cache.encode(), device)
        elif devices is not None:
            arr = (C.c_int * len(devices))(*devices)
            self.h = self.lib.tb200_create_multi(scene, arr, len(devices))
        else:
            self.h = self.lib.tb200_create(scene, device)
        if not self.h:
            raise TinselB200Error("tb200_create failed: " + last_error())
        self.device = devices[0] if devices is not None and cache is None else device   # the head: trace_rays runs there
        self.width = self.height = 0
        self._pinned = None
        self._external_stream = False

    def _check(self, rc, what):
        if rc != 0:
            raise TinselB200Error("%s failed: %s" % (what, last_error()))

    def Init(self, width, height):
        self._check(self.lib.tb200_init(self.h, width, height), "tb200_init")
        self.width, self.height = width, height

    def Render(self, camera, options, output):
        assert output.dtype == np.float32 and output.flags["C_CONTIGUOUS"]
        assert output.size == options.width * options.height * 4
        self._check(self.lib.tb200_render(self.h, C.byref(camera), C.byref(options), _fp(output)), "tb200_render")

    # batch / device-resident extensions (not part of the reference interface)
    def render_device(self, camera, options, spp, first_row=0, num_rows=-1):
        self._check(self.lib.tb200_render_device(self.h, C.byref(camera), C.byref(options), spp, first_row, num_rows),
                    "tb200_render_device")

    def set_shard(self, shard, num_shards):
        self._check(self.lib.tb200_set_shard(self.h, shard, num_shards), "tb200_set_shard")

    def set_stream(self, cuda_stream_handle):
        """None: the renderer's private stream; an int (0 = CUDA's legacy default stream): the caller's."""
        if cuda_stream_handle is None:
            self._check(self.lib.tb200_set_stream(self.h, None, 0), "tb200_set_stream")
        else:
            self._check(self.lib.tb200_set_stream(self.h, C.c_void_p(cuda_stream_handle), 1), "tb200_set_stream")
        self._external_stream = cuda_stream_handle is not None

    def set_slab(self, first_row, num_rows):
        self._check(self.lib.tb200_set_slab(self.h, first_row, num_rows), "tb200_set_slab")

    def pin_output(self, array):
        """Page-locks `array` (which the caller keeps alive until unpin_output / close) for fast read-backs."""
        assert array.dtype == np.float32 and array.flags["C_CONTIGUOUS"]
        self._check(self.lib.tb200_pin_output(self.h, _fp(array), array.nbytes), "tb200_pin_output")
        self._pinned = array   # keeps the buffer alive while it is registered

    def unpin_output(self):
        self.lib.tb200_unpin_output(self.h)
        self._pinned = None

    def gather_device(self):
        self._check(self.lib.tb200_gather_device(self.h), "tb200_gather_device")

    def num_devices(self):
        return self.lib.tb200_num_devices(self.h)

    def member_stats(self, member):
        """(Stats, first_row, num_rows) of one device of a multi-device renderer."""
        st, a, b = Stats(), C.c_int(), C.c_int()
        self._check(self.lib.tb200_get_member_stats(self.h, member, C.byref(st), C.byref(a), C.byref(b)), "tb200_get_member_stats")
        return st, a.value, b.value

    def bind_accumulator(self, device_ptr):
        self._check(self.lib.tb200_bind_accumulator(self.h, C.c_void_p(device_ptr)), "tb200_bind_accumulator")

    def read_accumulator(self, out=None):
        if out is None:
            out = np.empty((self.height, self.width, 4), np.float32)
        self._check(self.lib.tb200_read_accumulator(self.h, _fp(out)), "tb200_read_accumulator")
        return out

    def render_n(self, camera, options, n, output):
        """n x Render with one read-back (the `numSamples` loop of src/main.cpp:242-251)."""
        assert output.dtype == np.float32 and output.flags["C_CONTIGUOUS"]
        assert output.size == options.width * options.height * 4
        self._check(self.lib.tb200_render_n(self.h, C.byref(camera), C.byref(options), n, _fp(output)), "tb200_render_n")

    def finish(self, exposure, limit, filtered=True, rgb8=True):
        """Display/finish step on the device (src/main.cpp:258-271, src/png.cpp:329-343):
        returns (filtered float32 (H,W,4) or None, rgb8 uint8 (H,W,3) or None)."""
        f = np.empty((self.height, self.width, 4), np.float32) if filtered else None
        b = np.empty((self.height, self.width, 3), np.uint8) if rgb8 else None
        self._check(self.lib.tb200_finish(self.h, exposure, limit, _fp(f) if filtered else None,
                                          b.ctypes.data_as(C.POINTER(C.c_ubyte)) if rgb8 else None), "tb200_finish")
        return f, b

    def nlm(self, falloff, radius):
        """NonLocalMeansFilter (src/nlm.cpp:36-73) of the image the last finish() produced: (H,W,4) float32."""
        out = np.empty((self.height, self.width, 4), np.float32)
        self._check(self.lib.tb200_nlm(self.h, falloff, radius, _fp(out)), "tb200_nlm")
        return out

    def device_accumulator_ptr(self):
        return self.lib.tb200_device_accumulator(self.h)

    def trace_frame(self, camera, options, frame):
        rad = np.empty((options.height, options.width, 3), np.float32)
        ras = np.empty((options.height, options.width, 2), np.float32)
        self._check(self.lib.tb200_trace_frame(self.h, C.byref(camera), C.byref(options), frame, _fp(rad), _fp(ras)),
                    "tb200_trace_frame")
        return rad, ras

    def _check_tensor(self, x, name, shape, dtype):
        """What the ray queries require of a tensor argument: its type, dtype, shape, device (the head) and layout."""
        import torch
        if not isinstance(x, torch.Tensor):
            raise TypeError("%s must be a torch tensor" % name)
        if x.dtype != dtype:
            raise TypeError("%s must be %s, not %s" % (name, dtype, x.dtype))
        if tuple(x.shape) != shape:
            raise ValueError("%s must have shape %s, not %s" % (name, shape, tuple(x.shape)))
        dev = torch.device("cuda", self.device)
        if x.device != dev:
            raise ValueError("%s must be on %s (the renderer's head device), not %s" % (name, dev, x.device))
        if not x.is_contiguous():
            raise ValueError("%s must be contiguous" % name)

    def _check_rays(self, rays):
        """Checks a (N, 8) float32 ray tensor and returns N."""
        import torch
        if not isinstance(rays, torch.Tensor) or rays.dim() != 2:
            raise ValueError("rays must be a (N, 8) tensor")
        n = rays.shape[0]
        self._check_tensor(rays, "rays", (n, 8), torch.float32)
        return n

    def _wait_for_torch(self):
        """On the renderer's private stream, waits for torch's current stream, so that tensors written there are complete."""
        import torch
        if not self._external_stream:
            torch.cuda.current_stream(torch.device("cuda", self.device)).synchronize()

    def _query(self, entry, rays, outputs):
        """What the ray queries share: checks `rays` (N rays) and each output (tensor or None, name, shape after N,
        dtype), allocating on the head device those not given; when N > 0, waits for torch and calls the library's
        `entry` on the rays and the outputs, raising on a refusal.  Returns the output tensors."""
        import torch
        n = self._check_rays(rays)
        out = []
        for x, name, shape, dtype in outputs:
            if x is None:
                x = torch.empty((n,) + shape, dtype=dtype, device=torch.device("cuda", self.device))
            self._check_tensor(x, name, (n,) + shape, dtype)
            out.append(x)
        if n > 0:
            self._wait_for_torch()
            self._check(getattr(self.lib, entry)(self.h, rays.data_ptr(), *[x.data_ptr() for x in out], n), entry)
        return out

    def trace_rays(self, rays, hits=None, prims=None):
        """Closest hit of every ray (tb200_trace_rays): Trace (src/render.cpp:17-62) bit for bit.
        rays: contiguous float32 CUDA tensor (N, 8) on the head device -- origin.xyz, time, dir.xyz, pad.
        Returns (hits (N, 4) float32: t, normal.xyz; prims (N,) int32: closest primitive, -1 on a miss), in
        `hits` / `prims` when given.  On the renderer's private stream the call first waits for torch's current
        stream, so that tensors written there are complete; after set_stream the work is ordered on that stream."""
        import torch
        hits, prims = self._query("tb200_trace_rays", rays, [(hits, "hits", (4,), torch.float32), (prims, "prims", (), torch.int32)])
        return hits, prims

    def trace_rays_tri(self, rays, hits=None, prims=None, tris=None):
        """trace_rays, plus the triangle each mesh hit lies on (tb200_trace_rays_tri).  Returns (hits, prims) as
        trace_rays does, bit for bit, and (tri (N,) int32, uvw (N, 3) float32): the hit triangle's index in its mesh
        and its barycentric weights, u*N[i0] + v*N[i1] + w*N[i2] over the triangle's vertices i0, i1, i2 in the mesh's
        own space; tri = -1 and uvw = 0 for a sphere hit, a plane hit or a miss.  Both are views of one (N, 4) int32
        tensor, the tb200_tri_hit records, which `tris` gives when it is passed.  Stream behaviour as for trace_rays."""
        import torch
        hits, prims, tris = self._query("tb200_trace_rays_tri", rays, [(hits, "hits", (4,), torch.float32),
                                                                        (prims, "prims", (), torch.int32),
                                                                        (tris, "tris", (4,), torch.int32)])
        return hits, prims, tris[:, 0], tris[:, 1:].view(torch.float32)

    def occluded(self, rays, out=None):
        """Whether anything blocks each ray before its tmax (tb200_occluded_rays): exactly `Trace (src/render.cpp:17-62)
        hits a primitive and its t < tmax`.  rays: as for trace_rays, with column 7 = tmax in units of |dir| (so
        dir = target - origin, tmax = 1 asks about the segment between two points).  Returns a (N,) torch.bool
        tensor, `out` when given.  Stream behaviour as for trace_rays."""
        import torch
        out, = self._query("tb200_occluded_rays", rays, [(out, "out", (), torch.bool)])
        return out

    def set_frame(self, frame):
        self.lib.tb200_set_frame(self.h, frame)

    def stats(self):
        s = Stats()
        self.lib.tb200_get_stats(self.h, C.byref(s))
        return s

    def last_kernel(self):
        """Name of the kernel the last launch ran (tb200_last_kernel)."""
        return self.lib.tb200_last_kernel(self.h).decode()

    def close(self):
        if self.h:
            self.lib.tb200_destroy(self.h)   # unpins
            self.h = None
            self._pinned = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
