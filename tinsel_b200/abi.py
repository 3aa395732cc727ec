"""ctypes mirrors of include/tinsel_b200.h (the C ABI).  Field order and types must match the header."""
import ctypes as C

import numpy as np

c_float_p = C.POINTER(C.c_float)
c_int_p = C.POINTER(C.c_int32)


class Transform(C.Structure):
    _fields_ = [("p", C.c_float * 3), ("r", C.c_float * 4), ("s", C.c_float)]


class Material(C.Structure):
    _fields_ = [
        ("emission", C.c_float * 3),
        ("color", C.c_float * 3),
        ("absorption", C.c_float * 3),
        ("eta", C.c_float),
        ("metallic", C.c_float),
        ("subsurface", C.c_float),
        ("specular", C.c_float),
        ("roughness", C.c_float),
        ("specularTint", C.c_float),
        ("anisotropic", C.c_float),
        ("sheen", C.c_float),
        ("sheenTint", C.c_float),
        ("clearcoat", C.c_float),
        ("clearcoatGloss", C.c_float),
        ("transmission", C.c_float),
    ]

    @classmethod
    def default(cls):
        """Material() defaults, src/scene.h:47-70."""
        m = cls()
        m.color[:] = [0.82, 0.67, 0.16]
        m.specular = 0.5
        m.roughness = 0.5
        m.clearcoatGloss = 1.0
        return m


class Primitive(C.Structure):
    _fields_ = [
        ("start", Transform),
        ("end", Transform),
        ("type", C.c_int32),
        ("radius", C.c_float),
        ("plane", C.c_float * 4),
        ("mesh", C.c_int32),
        ("material", Material),
        ("lightSamples", C.c_int32),
    ]


class BvhNode(C.Structure):
    _fields_ = [("lower", C.c_float * 3), ("upper", C.c_float * 3), ("left", C.c_uint32), ("right_leaf", C.c_uint32)]


class Mesh(C.Structure):
    _fields_ = [
        ("positions", c_float_p),
        ("normals", c_float_p),
        ("indices", c_int_p),
        ("nodes", C.POINTER(BvhNode)),
        ("cdf", c_float_p),
        ("numVertices", C.c_int32),
        ("numIndices", C.c_int32),
        ("numNodes", C.c_int32),
        ("area", C.c_float),
    ]


class Sky(C.Structure):
    _fields_ = [
        ("horizon", C.c_float * 3),
        ("zenith", C.c_float * 3),
        ("probeValid", C.c_int32),
        ("probeWidth", C.c_int32),
        ("probeHeight", C.c_int32),
        ("probeData", c_float_p),
        ("pdfValuesX", c_float_p),
        ("cdfValuesX", c_float_p),
        ("pdfValuesY", c_float_p),
        ("cdfValuesY", c_float_p),
    ]


class Scene(C.Structure):
    _fields_ = [
        ("primitives", C.POINTER(Primitive)),
        ("numPrimitives", C.c_int32),
        ("meshes", C.POINTER(Mesh)),
        ("numMeshes", C.c_int32),
        ("bvhNodes", C.POINTER(BvhNode)),
        ("numBvhNodes", C.c_int32),
        ("sky", Sky),
    ]


class Camera(C.Structure):
    _fields_ = [
        ("position", C.c_float * 3),
        ("rotation", C.c_float * 4),
        ("fov", C.c_float),
        ("shutterStart", C.c_float),
        ("shutterEnd", C.c_float),
    ]


FILTER_BOX, FILTER_GAUSSIAN = 0, 1
MODE_NORMALS, MODE_COMPLEXITY, MODE_PATHTRACE = 0, 1, 2
SPHERE, PLANE, MESH = 0, 1, 2


class Options(C.Structure):
    _fields_ = [
        ("mode", C.c_int32),
        ("width", C.c_int32),
        ("height", C.c_int32),
        ("filterType", C.c_int32),
        ("filterWidth", C.c_float),
        ("filterFalloff", C.c_float),
        ("filterOffset", C.c_float),
        ("exposure", C.c_float),
        ("limit", C.c_float),
        ("clamp", C.c_float),
        ("maxDepth", C.c_int32),
        ("maxSamples", C.c_int32),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("frames", C.c_uint64),
        ("samples", C.c_uint64),
        ("kernelLaunches", C.c_uint64),
        ("d2hBytes", C.c_uint64),
        ("h2dBytes", C.c_uint64),
        ("gpuMs", C.c_double),
    ]


class Ray(C.Structure):
    """tb200_ray: one ray of tb200_trace_rays and tb200_occluded_rays (32 bytes; `pad` is the occlusion query's tmax)."""
    _fields_ = [("origin", C.c_float * 3), ("time", C.c_float), ("dir", C.c_float * 3), ("pad", C.c_float)]


class Hit(C.Structure):
    """tb200_hit: what tb200_trace_rays returns per ray besides the primitive index (16 bytes)."""
    _fields_ = [("t", C.c_float), ("normal", C.c_float * 3)]


class TriHit(C.Structure):
    """tb200_tri_hit: the hit triangle and its barycentric weights, from tb200_trace_rays_tri (16 bytes)."""
    _fields_ = [("tri", C.c_int32), ("u", C.c_float), ("v", C.c_float), ("w", C.c_float)]


class BsdfQuery(C.Structure):
    """tb200_bsdf_query: one query of tb200_bsdf_eval and tb200_bsdf_sample (48 bytes; `l` is ignored when sampling)."""
    _fields_ = [("n", C.c_float * 3), ("prim", C.c_int32), ("v", C.c_float * 3), ("etaI", C.c_float),
                ("l", C.c_float * 3), ("etaO", C.c_float)]


class BsdfValue(C.Structure):
    """tb200_bsdf_value: BSDFEval and BSDFPdf of one query, from tb200_bsdf_eval (16 bytes)."""
    _fields_ = [("f", C.c_float * 3), ("pdf", C.c_float)]


class BsdfSampled(C.Structure):
    """tb200_bsdf_sampled: the sampled direction, its pdf, BSDFEval of it and its BSDFType, from tb200_bsdf_sample
    (32 bytes)."""
    _fields_ = [("l", C.c_float * 3), ("pdf", C.c_float), ("f", C.c_float * 3), ("type", C.c_int32)]


# BSDFType (src/disney.h:27-32), tb200_bsdf_sampled.type
BSDF_REFLECTED, BSDF_TRANSMITTED, BSDF_SPECULAR = 0, 1, 2


class CameraSample(C.Structure):
    """tb200_camera_sample: one record of tb200_camera_rays, a pixel (row-major index) and a frame (8 bytes)."""
    _fields_ = [("pixel", C.c_int32), ("frame", C.c_int32)]


class LightQuery(C.Structure):
    """tb200_light_query: one query of tb200_sample_lights, a surface point as PathTrace reaches it (64 bytes)."""
    _fields_ = [("p", C.c_float * 3), ("time", C.c_float), ("n", C.c_float * 3), ("prim", C.c_int32),
                ("wo", C.c_float * 3), ("etaI", C.c_float), ("etaO", C.c_float), ("pad", C.c_float * 3)]


class EmitterQuery(C.Structure):
    """tb200_emitter_query: one query of tb200_sample_emitters, a light primitive and a time (8 bytes)."""
    _fields_ = [("prim", C.c_int32), ("time", C.c_float)]


class EmitterSampled(C.Structure):
    """tb200_emitter_sampled: a point PrimitiveSample drew on a light and the normal there, from tb200_sample_emitters
    (32 bytes)."""
    _fields_ = [("pos", C.c_float * 3), ("pad0", C.c_float), ("normal", C.c_float * 3), ("pad1", C.c_float)]


class ProbeSampled(C.Structure):
    """tb200_probe_sampled: a direction ProbeSample drew, its pdf and the probe's colour there, from tb200_sample_probe
    (32 bytes)."""
    _fields_ = [("dir", C.c_float * 3), ("pdf", C.c_float), ("color", C.c_float * 3), ("pad", C.c_float)]


# tb200_camera_sample as a numpy record (Renderer.camera_rays takes the same records as an (N, 2) int32 tensor)
CAMERA_SAMPLE_DTYPE = np.dtype([("pixel", "<i4"), ("frame", "<i4")])


class BvhBuildInfo(C.Structure):
    _fields_ = [("numNodes", C.c_int32), ("rounds", C.c_int32), ("kernelLaunches", C.c_uint64), ("buildMs", C.c_double)]


def copy_struct(s):
    """Value copy of a ctypes structure."""
    out = type(s)()
    C.memmove(C.byref(out), C.byref(s), C.sizeof(s))
    return out


# Every symbol include/tinsel_b200.h declares (tests/test_abi.py checks the library exports them all).
EXPORTS = [
    "tb200_create",
    "tb200_bvh_build",
    "tb200_bvh_build_error",
    "tb200_create_multi",
    "tb200_create_cached",
    "tb200_scene_cache_save",
    "tb200_num_devices",
    "tb200_get_member_stats",
    "tb200_slab_rows",
    "tb200_slab_traced_rows",
    "tb200_divisor_magic",
    "tb200_set_slab",
    "tb200_pin_output",
    "tb200_unpin_output",
    "tb200_gather_device",
    "tb200_init",
    "tb200_render",
    "tb200_render_device",
    "tb200_set_shard",
    "tb200_set_stream",
    "tb200_bind_accumulator",
    "tb200_device_accumulator",
    "tb200_read_accumulator",
    "tb200_render_n",
    "tb200_finish",
    "tb200_nlm",
    "tb200_trace_frame",
    "tb200_trace_rays",
    "tb200_trace_rays_tri",
    "tb200_occluded_rays",
    "tb200_bsdf_eval",
    "tb200_bsdf_sample",
    "tb200_camera_rays",
    "tb200_splat",
    "tb200_sample_lights",
    "tb200_sky_eval",
    "tb200_sample_emitters",
    "tb200_sample_probe",
    "tb200_probe_tables",
    "tb200_set_sky",
    "tb200_set_frame",
    "tb200_get_stats",
    "tb200_last_kernel",
    "tb200_destroy",
    "tb200_last_error",
    "tb200_sample_seed",
    "tb200_snapshot_load",
    "tb200_snapshot_scene",
    "tb200_snapshot_camera",
    "tb200_snapshot_options",
    "tb200_snapshot_save",
    "tb200_snapshot_free",
    "tb200_mesh_bin_load",
    "tb200_mesh_bin_mesh",
    "tb200_mesh_bin_save",
    "tb200_mesh_bin_free",
]


def declare_snapshot_api(lib):
    lib.tb200_mesh_bin_load.restype = C.c_void_p
    lib.tb200_mesh_bin_load.argtypes = [C.c_char_p]
    lib.tb200_mesh_bin_mesh.restype = C.POINTER(Mesh)
    lib.tb200_mesh_bin_mesh.argtypes = [C.c_void_p]
    lib.tb200_mesh_bin_save.restype = C.c_int
    lib.tb200_mesh_bin_save.argtypes = [C.c_char_p, C.POINTER(Mesh)]
    lib.tb200_mesh_bin_free.restype = None
    lib.tb200_mesh_bin_free.argtypes = [C.c_void_p]
    lib.tb200_snapshot_load.restype = C.c_void_p
    lib.tb200_snapshot_load.argtypes = [C.c_char_p]
    lib.tb200_snapshot_scene.restype = C.POINTER(Scene)
    lib.tb200_snapshot_scene.argtypes = [C.c_void_p]
    lib.tb200_snapshot_camera.restype = C.POINTER(Camera)
    lib.tb200_snapshot_camera.argtypes = [C.c_void_p]
    lib.tb200_snapshot_options.restype = C.POINTER(Options)
    lib.tb200_snapshot_options.argtypes = [C.c_void_p]
    lib.tb200_snapshot_save.restype = C.c_int
    lib.tb200_snapshot_save.argtypes = [C.c_char_p, C.POINTER(Scene), C.POINTER(Camera), C.POINTER(Options)]
    lib.tb200_snapshot_free.restype = None
    lib.tb200_snapshot_free.argtypes = [C.c_void_p]
    lib.tb200_sample_seed.restype = C.c_uint32
    lib.tb200_sample_seed.argtypes = [C.c_uint32, C.c_uint32]
