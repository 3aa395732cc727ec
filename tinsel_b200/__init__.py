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
    lib.tb200_bsdf_eval.restype = C.c_int
    lib.tb200_bsdf_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    lib.tb200_bsdf_sample.restype = C.c_int
    lib.tb200_bsdf_sample.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    lib.tb200_camera_rays.restype = C.c_int
    lib.tb200_camera_rays.argtypes = [C.c_void_p, C.POINTER(Camera), C.POINTER(Options), C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int64]
    lib.tb200_splat.restype = C.c_int
    lib.tb200_splat.argtypes = [C.c_void_p, C.POINTER(Options), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    lib.tb200_sample_lights.restype = C.c_int
    lib.tb200_sample_lights.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    lib.tb200_sky_eval.restype = C.c_int
    lib.tb200_sky_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    lib.tb200_sample_emitters.restype = C.c_int
    lib.tb200_sample_emitters.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    lib.tb200_sample_probe.restype = C.c_int
    lib.tb200_sample_probe.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    lib.tb200_probe_tables.restype = C.c_int
    lib.tb200_probe_tables.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.tb200_set_sky.restype = C.c_int
    lib.tb200_set_sky.argtypes = [C.c_void_p, f32p, f32p, C.c_void_p, C.c_int, C.c_int]
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


def material_ior(eta, specular):
    """Material::GetIndexOfRefraction (src/scene.h:72-78) in float32, elementwise: `eta` where it is not 0, else
    2 / (1 - sqrt(float(0.08 * specular))) - 1 with the product in double, as the reference rounds it.  The etaO of
    a path entering a material (PathTrace's eta convention, include/tinsel_b200.h: tb200_bsdf_eval).  Returns a
    float32 numpy array (a 0-d one for scalars)."""
    eta = np.asarray(eta, np.float32)
    specular = np.asarray(specular, np.float32)
    with np.errstate(all="ignore"):
        k = np.sqrt((0.08 * specular.astype(np.float64)).astype(np.float32))
        from_specular = np.float32(2) / (np.float32(1) - k) - np.float32(1)
    return np.where(eta == 0, from_specular, eta).astype(np.float32)


def bsdf_queries(prims, n, v, eta_i, eta_o, l=None):
    """Packs tb200_bsdf_query records for Renderer.bsdf_eval / bsdf_sample: an (N, 12) float32 tensor on `prims`'
    device with n.xyz, the int32 primitive's bits, v.xyz, etaI, l.xyz, etaO per row.  prims: (N,) int32 tensor
    (trace_rays' prims can be passed as they are); n, v, l: (N, 3) float32 tensors (l None: zeros, which sampling
    ignores); eta_i, eta_o: (N,) float32 tensors or Python numbers."""
    return _pack_records(prims, 12, 3, [(0, n, 3, "n"), (4, v, 3, "v"), (7, eta_i, 1, "eta_i"),
                                        (8, l if l is not None else 0.0, 3, "l"), (11, eta_o, 1, "eta_o")])


def light_queries(prims, p, n, wo, eta_i, eta_o, time):
    """Packs tb200_light_query records for Renderer.sample_lights: an (N, 16) float32 tensor on `prims`' device with
    p.xyz, time, n.xyz, the int32 primitive's bits, wo.xyz, etaI, etaO and three zeros per row.  prims: (N,) int32
    tensor (trace_rays' prims can be passed as they are); p, n, wo: (N, 3) float32 tensors (the hit point, the normal
    trace_rays returns and -dir of the incoming ray); eta_i, eta_o, time: (N,) float32 tensors or Python numbers."""
    return _pack_records(prims, 16, 7, [(0, p, 3, "p"), (3, time, 1, "time"), (4, n, 3, "n"), (8, wo, 3, "wo"),
                                        (11, eta_i, 1, "eta_i"), (12, eta_o, 1, "eta_o"), (13, 0.0, 3, "pad")])


def emitter_queries(prims, time):
    """Packs tb200_emitter_query records for Renderer.sample_emitters: an (N, 2) float32 tensor on `prims`' device with
    the int32 primitive's bits and the time per row.  prims: (N,) int32 tensor (trace_rays' prims can be passed as they
    are); time: (N,) float32 tensor or a Python number."""
    return _pack_records(prims, 2, 0, [(1, time, 1, "time")])


def _pack_records(prims, width, prim_col, fields):
    """An (N, width) float32 tensor on `prims`' device with the int32 prims' bits in column prim_col and each field
    (col, x, cols, name) in columns [col, col + cols): x a float32 tensor of shape (N, cols), or (N,) for one column,
    or a Python number for every row."""
    import torch
    if not isinstance(prims, torch.Tensor) or prims.dtype != torch.int32 or prims.dim() != 1:
        raise ValueError("prims must be an (N,) int32 tensor")
    count, dev = prims.shape[0], prims.device
    q = torch.empty((count, width), dtype=torch.float32, device=dev)
    for col, x, cols, name in fields:
        if not isinstance(x, torch.Tensor):
            q[:, col:col + cols] = float(x)
            continue
        shape = (count, cols) if cols > 1 else (count,)
        if x.dtype != torch.float32 or tuple(x.shape) != shape:
            raise ValueError("%s must be a float32 tensor of shape %s" % (name, shape))
        q[:, col:col + cols] = x.to(dev).reshape(count, cols)
    q[:, prim_col] = prims.view(torch.float32)
    return q


def primitive_areas(scene):
    """PrimitiveArea (src/intersection.h:833-853) of every primitive of `scene` (a tb200_scene or a pointer to one),
    as the renderer computes it in float32: 4 pi r^2 for a sphere, the mesh's area times the end transform's scale
    for a mesh, 0 for a plane.  With a primitive's lightSamples and emission, it is what PathTrace's emission MIS
    weight at a hit needs (src/render.cpp:255-310).  Returns an (numPrimitives,) float32 numpy array."""
    sc = scene.contents if isinstance(scene, C._Pointer) else scene
    out = np.zeros(sc.numPrimitives, np.float32)
    pi = np.float32(3.14159265358979323846)
    for i in range(sc.numPrimitives):
        p = sc.primitives[i]
        if p.type == abi.SPHERE:
            r = np.float32(p.radius)
            out[i] = np.float32(4) * pi * r * r
        elif p.type == abi.MESH:
            out[i] = np.float32(sc.meshes[p.mesh].area) * np.float32(p.end.s)
    return out


def frame_samples(width, height, frame0, num_frames=1, device="cuda"):
    """The (pixel, frame) records of whole frames for Renderer.camera_rays: an (num_frames * width * height, 2) int32
    tensor on `device`, frames frame0, frame0 + 1, ... one after the other, each with its pixels in row-major order.
    Frame numbers wrap as the renderer's int32 frame counter does."""
    import torch
    if width <= 0 or height <= 0 or num_frames < 0:
        raise ValueError("frame_samples needs a positive width and height and num_frames >= 0, not %r, %r, %r"
                         % (width, height, num_frames))
    npix = width * height
    frames = (torch.arange(num_frames, dtype=torch.int64) + int(frame0) + 2 ** 31) % 2 ** 32 - 2 ** 31
    out = torch.empty((num_frames, npix, 2), dtype=torch.int32)
    out[:, :, 0] = torch.arange(npix, dtype=torch.int32)
    out[:, :, 1] = frames.to(torch.int32)[:, None]
    return out.reshape(num_frames * npix, 2).to(device)


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

    def _check_records(self, x, name, width, dtype):
        """Checks a (N, width) tensor of query records, or with width None an (N,) one, and returns N."""
        import torch
        shape = "(N,)" if width is None else "(N, %d)" % width
        if not isinstance(x, torch.Tensor) or x.dim() != (1 if width is None else 2):
            raise ValueError("%s must be a %s tensor" % (name, shape))
        n = x.shape[0]
        self._check_tensor(x, name, (n,) if width is None else (n, width), dtype)
        return n

    def _wait_for_torch(self):
        """On the renderer's private stream, waits for torch's current stream, so that tensors written there are complete."""
        import torch
        if not self._external_stream:
            torch.cuda.current_stream(torch.device("cuda", self.device)).synchronize()

    def _query(self, entry, records, inputs, outputs, before=(), after=()):
        """What the batched queries share.  records: (tensor, name, width, dtype), the (N, width) records that set N
        ((N,) with width None);
        inputs: further input arrays and outputs: output arrays, each (tensor or None, name, shape after N, dtype).
        Checks them all, allocating on the head device the outputs not given (an input must be given); when N > 0,
        waits for torch and calls the library's `entry` on the `before` arguments, the records, the inputs, the
        outputs and the `after` arguments, raising on a refusal.  Returns the output tensors."""
        import torch
        x, name, width, dtype = records
        n = self._check_records(x, name, width, dtype)
        args = [x]
        for y, yname, shape, ydtype in inputs:
            self._check_tensor(y, yname, (n,) + shape, ydtype)
            args.append(y)
        out = []
        for y, yname, shape, ydtype in outputs:
            if y is None:
                y = torch.empty((n,) + shape, dtype=ydtype, device=torch.device("cuda", self.device))
            self._check_tensor(y, yname, (n,) + shape, ydtype)
            out.append(y)
        if n > 0:
            self._wait_for_torch()
            self._check(getattr(self.lib, entry)(self.h, *before, *[y.data_ptr() for y in args + out], *after, n), entry)
        return out

    def trace_rays(self, rays, hits=None, prims=None):
        """Closest hit of every ray (tb200_trace_rays): Trace (src/render.cpp:17-62) bit for bit.
        rays: contiguous float32 CUDA tensor (N, 8) on the head device -- origin.xyz, time, dir.xyz, pad.
        Returns (hits (N, 4) float32: t, normal.xyz; prims (N,) int32: closest primitive, -1 on a miss), in
        `hits` / `prims` when given.  On the renderer's private stream the call first waits for torch's current
        stream, so that tensors written there are complete; after set_stream the work is ordered on that stream."""
        import torch
        hits, prims = self._query("tb200_trace_rays", (rays, "rays", 8, torch.float32), [],
                                  [(hits, "hits", (4,), torch.float32), (prims, "prims", (), torch.int32)])
        return hits, prims

    def trace_rays_tri(self, rays, hits=None, prims=None, tris=None):
        """trace_rays, plus the triangle each mesh hit lies on (tb200_trace_rays_tri).  Returns (hits, prims) as
        trace_rays does, bit for bit, and (tri (N,) int32, uvw (N, 3) float32): the hit triangle's index in its mesh
        and its barycentric weights, u*N[i0] + v*N[i1] + w*N[i2] over the triangle's vertices i0, i1, i2 in the mesh's
        own space; tri = -1 and uvw = 0 for a sphere hit, a plane hit or a miss.  Both are views of one (N, 4) int32
        tensor, the tb200_tri_hit records, which `tris` gives when it is passed.  Stream behaviour as for trace_rays."""
        import torch
        hits, prims, tris = self._query("tb200_trace_rays_tri", (rays, "rays", 8, torch.float32), [],
                                        [(hits, "hits", (4,), torch.float32), (prims, "prims", (), torch.int32),
                                         (tris, "tris", (4,), torch.int32)])
        return hits, prims, tris[:, 0], tris[:, 1:].view(torch.float32)

    def occluded(self, rays, out=None):
        """Whether anything blocks each ray before its tmax (tb200_occluded_rays): exactly `Trace (src/render.cpp:17-62)
        hits a primitive and its t < tmax`.  rays: as for trace_rays, with column 7 = tmax in units of |dir| (so
        dir = target - origin, tmax = 1 asks about the segment between two points).  Returns a (N,) torch.bool
        tensor, `out` when given.  Stream behaviour as for trace_rays."""
        import torch
        out, = self._query("tb200_occluded_rays", (rays, "rays", 8, torch.float32), [], [(out, "out", (), torch.bool)])
        return out

    def bsdf_eval(self, queries, out=None):
        """The Disney BSDF of every query (tb200_bsdf_eval): BSDFEval and BSDFPdf (src/disney.h) bit for bit, with the
        material the renderer shades primitive `prim` with.  queries: contiguous float32 CUDA tensor (N, 12) on the
        head device, the tb200_bsdf_query records n.xyz, prim, v.xyz, etaI, l.xyz, etaO, with column 3 holding the
        int32 primitive index's bits (bsdf_queries packs them).  n, v, l are used as given, never normalised.
        Returns (N, 4) float32: f.rgb, pdf, in `out` when given; a prim outside the scene gives zeros.  Stream
        behaviour as for trace_rays."""
        import torch
        out, = self._query("tb200_bsdf_eval", (queries, "queries", 12, torch.float32), [],
                           [(out, "out", (4,), torch.float32)])
        return out

    def bsdf_sample(self, queries, seeds, out=None):
        """One BSDF sampling step of PathTrace per query (tb200_bsdf_sample): BSDFSample with BasisFromVector(n) and
        Random(seed), then f = BSDFEval of the sampled direction where its pdf > 0, else 0; bit for bit.  queries:
        as for bsdf_eval (their l is ignored); seeds: (N,) int32 tensor whose bits are the uint32 seeds.  Returns
        (l (N, 3) float32, pdf (N,) float32, f (N, 3) float32, type (N,) int32: abi.BSDF_*, -1 for a prim outside
        the scene, whose other outputs are 0), views of one (N, 8) tensor of tb200_bsdf_sampled records, which `out`
        (float32) gives when it is passed.  Stream behaviour as for trace_rays."""
        import torch
        out, = self._query("tb200_bsdf_sample", (queries, "queries", 12, torch.float32), [(seeds, "seeds", (), torch.int32)],
                           [(out, "out", (8,), torch.float32)])
        return out[:, 0:3], out[:, 3], out[:, 4:7], out[:, 7].view(torch.int32)

    def camera_rays(self, camera, options, samples, rays=None, raster=None):
        """The renderer's camera sample of every (pixel, frame) record (tb200_camera_rays): Random(sample_seed(pixel,
        frame)), the draws x, y, t (src/render.cpp:476-482) and GenerateRay through the camera of an options.width x
        options.height image, bit for bit.  samples: (N, 2) int32 tensor on the head device, the pixel (row-major) and
        the frame (frame_samples makes whole frames).  Returns (rays (N, 8) float32: origin.xyz, time, dir.xyz, +inf,
        ready for trace_rays and occluded; raster (N, 2) float32: the position the renderer splats the sample at), in
        `rays` / `raster` when given.  A pixel outside the image gives a zero ray and a NaN raster.  Stream behaviour
        as for trace_rays."""
        import torch
        rays, raster = self._query("tb200_camera_rays", (samples, "samples", 2, torch.int32), [],
                                   [(rays, "rays", (8,), torch.float32), (raster, "raster", (2,), torch.float32)],
                                   before=(C.byref(camera), C.byref(options)))
        return rays, raster

    def splat(self, options, raster, radiance, accum=None):
        """AddSample (src/render.cpp:401-445) of every sample into a film (tb200_splat), with the options' filter and
        clamp, as the renderer splats its own samples.  raster (N, 2) and radiance (N, 3): float32 tensors on the head
        device; a raster coordinate that is NaN or 2^30 or more in magnitude is skipped.  accum: a contiguous
        (options.height, options.width, 4) float32 tensor on the head device, added to (the caller zeroes it); None:
        the renderer's own accumulator, which finish(), nlm() and read_accumulator() then see, and options.width /
        height must be those of the last Init.  Returns `accum` (None for the renderer's own).  Stream behaviour as
        for trace_rays."""
        import torch
        W, H = options.width, options.height
        if accum is None:
            if (W, H) != (self.width, self.height) or not self.width:
                raise ValueError("splat into the renderer's accumulator: options.width/height %dx%d differ from the last "
                                 "Init (%dx%d)" % (W, H, self.width, self.height))
            ptr = self.device_accumulator_ptr()
        else:
            self._check_tensor(accum, "accum", (H, W, 4), torch.float32)
            ptr = accum.data_ptr()
        self._query("tb200_splat", (raster, "raster", 2, torch.float32), [(radiance, "radiance", (3,), torch.float32)], [],
                    before=(C.byref(options),), after=(C.c_void_p(ptr),))
        return accum

    def sample_lights(self, queries, seeds, out=None):
        """Next-event estimation at every surface record (tb200_sample_lights): SampleLights (src/render.cpp:103-227)
        with Random(seed), bit for bit -- the probe sample, every light's samples with their closest-hit shadow rays
        and MIS -- the `sum` PathTrace multiplies by the throughput at a hit.  queries: contiguous float32 CUDA tensor
        (N, 16) on the head device, the tb200_light_query records (light_queries packs them); seeds: (N,) int32
        tensor whose bits are the uint32 seeds.  Returns (N, 3) float32 radiance, `out` when given; a prim outside
        the scene gives zeros.  Stream behaviour as for trace_rays."""
        import torch
        out, = self._query("tb200_sample_lights", (queries, "queries", 16, torch.float32),
                           [(seeds, "seeds", (), torch.int32)], [(out, "out", (3,), torch.float32)])
        return out

    def sky(self, rays, out=None, split=False):
        """The sky of a miss for every ray (tb200_sky_eval): Sky::Eval(dir) (src/scene.h:168-178) and ProbePdf(dir)
        (src/probe.h:136-160), 0 without a probe, bit for bit.  rays: as for trace_rays, of which only dir is read.
        Returns (N, 4) float32: rgb, pdf, in `out` when given; with split, (rgb (N, 3), pdf (N,)) views of it.  The
        miss's MIS weight depends on path state and is the caller's.  Stream behaviour as for trace_rays."""
        import torch
        out, = self._query("tb200_sky_eval", (rays, "rays", 8, torch.float32), [], [(out, "out", (4,), torch.float32)])
        return (out[:, :3], out[:, 3]) if split else out

    def sample_emitters(self, queries, seeds, out=None):
        """A point on each query's light (tb200_sample_emitters): PrimitiveSample (src/intersection.h:855-904) of
        primitive `prim` at `time` from Random(seed), bit for bit -- what SampleLights draws for one light sample.
        queries: contiguous float32 CUDA tensor (N, 2) on the head device, the tb200_emitter_query records, with
        column 0 holding the int32 primitive index's bits (emitter_queries packs them); seeds: (N,) int32 tensor
        whose bits are the uint32 seeds.  Returns (pos (N, 3) float32, normal (N, 3) float32), views of one (N, 8)
        tensor of tb200_emitter_sampled records, which `out` (float32) gives when it is passed.  Only primitives with
        lightSamples > 0 are sampled; any other prim, or one outside the scene, gives zeros.  The sample's area pdf
        is 1 / primitive_areas(scene)[prim].  Stream behaviour as for trace_rays."""
        import torch
        out, = self._query("tb200_sample_emitters", (queries, "queries", 2, torch.float32),
                           [(seeds, "seeds", (), torch.int32)], [(out, "out", (8,), torch.float32)])
        return out[:, 0:3], out[:, 4:7]

    def sample_probe(self, seeds, out=None):
        """A direction drawn from the sky's probe per seed (tb200_sample_probe): ProbeSample (src/probe.h:205-236)
        from Random(seed), bit for bit -- what SampleLights draws for its probe sample.  seeds: (N,) int32 CUDA
        tensor on the head device whose bits are the uint32 seeds.  Returns (dir (N, 3) float32, pdf (N,) float32,
        color (N, 3) float32), views of one (N, 8) tensor of tb200_probe_sampled records, which `out` (float32)
        gives when it is passed; zeros when the sky has no probe.  pdf is 0 where sin(theta) is 0; sky() gives the
        matching ProbePdf of any direction.  Stream behaviour as for trace_rays."""
        import torch
        out, = self._query("tb200_sample_probe", (seeds, "seeds", None, torch.int32), [],
                           [(out, "out", (8,), torch.float32)])
        return out[:, 0:3], out[:, 3], out[:, 4:7]

    def _probe_image(self, probe, device_only):
        """Checks an (H, W, 4) float32 C-contiguous probe image: a numpy array or a CPU tensor (unless device_only), or
        a CUDA tensor on the head device.  Returns (pointer, W, H, whether it is on the device)."""
        import torch
        if isinstance(probe, np.ndarray):
            if device_only:
                raise TypeError("probe must be a CUDA tensor, not a numpy array")
            if probe.dtype != np.float32:
                raise TypeError("probe must be float32, not %s" % probe.dtype)
            if probe.ndim != 3 or probe.shape[2] != 4:
                raise ValueError("probe must have shape (H, W, 4), not %s" % (probe.shape,))
            if not probe.flags["C_CONTIGUOUS"]:
                raise ValueError("probe must be C-contiguous")
            return probe.ctypes.data, probe.shape[1], probe.shape[0], False
        if not isinstance(probe, torch.Tensor):
            raise TypeError("probe must be a numpy array or a torch tensor")
        if probe.dim() != 3 or probe.shape[2] != 4:
            raise ValueError("probe must have shape (H, W, 4), not %s" % (tuple(probe.shape),))
        if probe.device.type == "cpu" and not device_only:
            if probe.dtype != torch.float32:
                raise TypeError("probe must be torch.float32, not %s" % probe.dtype)
            if not probe.is_contiguous():
                raise ValueError("probe must be contiguous")
        else:
            self._check_tensor(probe, "probe", tuple(probe.shape), torch.float32)
        return probe.data_ptr(), probe.shape[1], probe.shape[0], probe.device.type == "cuda"

    def set_sky(self, horizon, zenith, probe=None):
        """Replaces the renderer's sky (tb200_set_sky): the gradient colours horizon and zenith (3 floats each) and,
        unless probe is None, an HDR probe of (H, W, 4) float32 RGBA texels, row 0 at the zenith -- a C-contiguous
        numpy array, a CPU tensor, or a contiguous CUDA tensor on the head device.  The renderer copies the texels and
        builds the probe's sampling tables on the device; afterwards it renders and answers every query as one created
        from the same scene with this sky would.  The accumulated image and the frame counter stay as they are (Init
        restarts them).  A CUDA probe is read after torch's current stream, as the queries read their inputs."""
        colours = []
        for name, c in (("horizon", horizon), ("zenith", zenith)):
            c = [float(v) for v in c]
            if len(c) != 3:
                raise ValueError("%s must have 3 values (r, g, b), not %d" % (name, len(c)))
            colours.append((C.c_float * 3)(*c))
        h, z = colours
        if probe is None:
            self._check(self.lib.tb200_set_sky(self.h, h, z, None, 0, 0), "tb200_set_sky")
            return
        ptr, width, height, on_device = self._probe_image(probe, False)
        if on_device:
            self._wait_for_torch()
        self._check(self.lib.tb200_set_sky(self.h, h, z, C.c_void_p(ptr), width, height), "tb200_set_sky")

    def probe_tables(self, probe, pdf_x=None, cdf_x=None, pdf_y=None, cdf_y=None):
        """Probe::BuildCDF (src/probe.h:31-79) of a probe on the device (tb200_probe_tables), bit for bit: probe is an
        (H, W, 4) float32 contiguous CUDA tensor on the head device.  Returns (pdf_x (H, W), cdf_x (H, W), pdf_y (H,),
        cdf_y (H,)) float32 tensors, the given ones when passed.  It does not change the renderer's sky.  Stream
        behaviour as for trace_rays."""
        import torch
        ptr, width, height, _ = self._probe_image(probe, True)
        dev = torch.device("cuda", self.device)
        out = []
        for y, name, shape in ((pdf_x, "pdf_x", (height, width)), (cdf_x, "cdf_x", (height, width)),
                               (pdf_y, "pdf_y", (height,)), (cdf_y, "cdf_y", (height,))):
            if y is None:
                y = torch.empty(shape, dtype=torch.float32, device=dev)
            self._check_tensor(y, name, shape, torch.float32)
            out.append(y)
        self._wait_for_torch()
        self._check(self.lib.tb200_probe_tables(self.h, C.c_void_p(ptr), width, height, *[y.data_ptr() for y in out]),
                    "tb200_probe_tables")
        return tuple(out)

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
