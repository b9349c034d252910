"""Struct layouts of the visibility path as numpy dtypes and ctypes structures.

Mirrors include/niagara_cull.h, which mirrors the reference's src/shaders/mesh.h:11-123,
src/scene.h:10-93 and src/niagara.cpp:227-260 (sizes 24/20/208/48/24/20/144 bytes).
"""
import ctypes

import numpy as np

TASK_WGSIZE = 64  # src/config.h:2
TASK_WGLIMIT = 1 << 22  # src/config.h:25
CLUSTER_LIMIT = 1 << 24  # src/config.h:28
CLUSTER_TILE = 16  # src/config.h:22
MAX_DISPATCH_GROUPS = 65535  # tasksubmit.comp.glsl:36
MAX_LODS = 8
MAX_HIZ_LEVELS = 16

MESHLET_DTYPE = np.dtype(
    [
        ("center", "<u2", (3,)),  # binary16 bits
        ("radius", "<u2"),
        ("cone_axis", "i1", (3,)),
        ("cone_cutoff", "i1"),
        ("dataOffset", "<u4"),
        ("baseVertex", "<u4"),
        ("vertexCount", "u1"),
        ("triangleCount", "u1"),
        ("shortRefs", "u1"),
        ("padding", "u1"),
    ]
)

MESHLOD_DTYPE = np.dtype(
    [("indexOffset", "<u4"), ("indexCount", "<u4"), ("meshletOffset", "<u4"), ("meshletCount", "<u4"), ("error", "<f4")]
)

MESH_DTYPE = np.dtype(
    [
        ("center", "<f4", (3,)),
        ("radius", "<f4"),
        ("vertexOffset", "<u4"),
        ("vertexCount", "<u4"),
        ("ommIndexData", "<u4"),
        ("ommIndexBase", "<u4"),
        ("lodCount", "<u4"),
        ("lodRT", "<u4"),
        ("padding", "<u4", (2,)),
        ("lods", MESHLOD_DTYPE, (MAX_LODS,)),
    ]
)

MESHDRAW_DTYPE = np.dtype(
    [
        ("position", "<f4", (3,)),
        ("scale", "<f4"),
        ("orientation", "<f4", (4,)),  # x, y, z, w
        ("meshIndex", "<u4"),
        ("meshletVisibilityOffset", "<u4"),
        ("postPass", "<u4"),
        ("materialIndex", "<u4"),
    ]
)

MESHDRAWCOMMAND_DTYPE = np.dtype(
    [
        ("drawId", "<u4"),
        ("indexCount", "<u4"),
        ("instanceCount", "<u4"),
        ("firstIndex", "<u4"),
        ("vertexOffset", "<u4"),
        ("firstInstance", "<u4"),
    ]
)

MESHTASKCOMMAND_DTYPE = np.dtype(
    [
        ("drawId", "<u4"),
        ("taskOffset", "<u4"),
        ("taskCount", "<u4"),
        ("lateDrawVisibility", "<u4"),
        ("meshletVisibilityOffset", "<u4"),
    ]
)

CULLDATA_DTYPE = np.dtype(
    [
        ("view", "<f4", (16,)),  # column-major
        ("P00", "<f4"),
        ("P11", "<f4"),
        ("znear", "<f4"),
        ("zfar", "<f4"),
        ("frustum", "<f4", (4,)),
        ("lodTarget", "<f4"),
        ("pyramidWidth", "<f4"),
        ("pyramidHeight", "<f4"),
        ("drawCount", "<u4"),
        ("cullingEnabled", "<i4"),
        ("lodEnabled", "<i4"),
        ("occlusionEnabled", "<i4"),
        ("clusterOcclusionEnabled", "<i4"),
        ("clusterBackfaceEnabled", "<i4"),
        ("postPass", "<u4"),
        ("pad_", "<u4", (2,)),
    ]
)

assert MESHLET_DTYPE.itemsize == 24
assert MESHLOD_DTYPE.itemsize == 20
assert MESH_DTYPE.itemsize == 208
assert MESHDRAW_DTYPE.itemsize == 48
assert MESHDRAWCOMMAND_DTYPE.itemsize == 24
assert MESHTASKCOMMAND_DTYPE.itemsize == 20
assert CULLDATA_DTYPE.itemsize == 144


class CullData(ctypes.Structure):
    _fields_ = [
        ("view", ctypes.c_float * 16),
        ("P00", ctypes.c_float),
        ("P11", ctypes.c_float),
        ("znear", ctypes.c_float),
        ("zfar", ctypes.c_float),
        ("frustum", ctypes.c_float * 4),
        ("lodTarget", ctypes.c_float),
        ("pyramidWidth", ctypes.c_float),
        ("pyramidHeight", ctypes.c_float),
        ("drawCount", ctypes.c_uint32),
        ("cullingEnabled", ctypes.c_int32),
        ("lodEnabled", ctypes.c_int32),
        ("occlusionEnabled", ctypes.c_int32),
        ("clusterOcclusionEnabled", ctypes.c_int32),
        ("clusterBackfaceEnabled", ctypes.c_int32),
        ("postPass", ctypes.c_uint32),
        ("pad_", ctypes.c_uint32 * 2),
    ]

    def copy(self):
        out = CullData()
        ctypes.memmove(ctypes.byref(out), ctypes.byref(self), ctypes.sizeof(CullData))
        return out

    def to_numpy(self):
        return np.frombuffer(bytes(self), dtype=CULLDATA_DTYPE)[0].copy()


class HiZ(ctypes.Structure):
    _fields_ = [
        ("texels", ctypes.c_void_p),
        ("width", ctypes.c_uint32),
        ("height", ctypes.c_uint32),
        ("levels", ctypes.c_uint32),
        ("level_offset", ctypes.c_uint32 * MAX_HIZ_LEVELS),
        ("total_texels", ctypes.c_uint32),
    ]

    def level_size(self, level):
        return max(1, self.width >> level), max(1, self.height >> level)

    def with_texels(self, ptr):
        out = HiZ()
        ctypes.memmove(ctypes.byref(out), ctypes.byref(self), ctypes.sizeof(HiZ))
        out.texels = ptr
        return out


class Limits(ctypes.Structure):
    _fields_ = [("task_wglimit", ctypes.c_uint32), ("cluster_limit", ctypes.c_uint32)]


class Camera(ctypes.Structure):
    _fields_ = [
        ("position", ctypes.c_float * 3),
        ("orientation", ctypes.c_float * 4),
        ("fovY", ctypes.c_float),
        ("znear", ctypes.c_float),
    ]


class GltfInfo(ctypes.Structure):
    _fields_ = [
        ("node_count", ctypes.c_uint32),
        ("mesh_count", ctypes.c_uint32),
        ("primitive_count", ctypes.c_uint32),
        ("draw_count", ctypes.c_uint32),
        ("animation_count", ctypes.c_uint32),
        ("keyframe_count", ctypes.c_uint32),
        ("material_count", ctypes.c_uint32),
        ("point_light_count", ctypes.c_uint32),
        ("has_camera", ctypes.c_uint32),
        ("has_sun", ctypes.c_uint32),
        ("camera", Camera),
        ("sun_direction", ctypes.c_float * 3),
    ]


class CullOptions(ctypes.Structure):
    _fields_ = [
        ("draw_distance", ctypes.c_float),
        ("culling", ctypes.c_int32),
        ("lod", ctypes.c_int32),
        ("occlusion", ctypes.c_int32),
        ("cluster_occlusion", ctypes.c_int32),
        ("mesh_shading", ctypes.c_int32),
        ("debug_lod_step", ctypes.c_int32),
    ]


assert ctypes.sizeof(CullData) == 144

# scene.h:141-161 — animation tracks of the scene cache (widening N3)
KEYFRAME_DTYPE = np.dtype([("translation", "<f4", (3,)), ("scale", "<f4"), ("rotation", "<f4", (4,))])
ANIMATION_DTYPE = np.dtype([("drawIndex", "<i4"), ("lightIndex", "<i4"), ("startTime", "<f4"), ("period", "<f4"), ("keyframeOffset", "<u4"), ("keyframeCount", "<u4")])
assert KEYFRAME_DTYPE.itemsize == 32 and ANIMATION_DTYPE.itemsize == 24

CACHE_SECTIONS = ["vertices", "indices", "meshlets", "meshletdata", "meshletvtx0", "meshes", "materials", "draws", "lights", "animations", "keyframes", "omm_data", "omm_indices", "omm_descs", "texture_paths"]


class SceneCacheHeader(ctypes.Structure):  # scenecache.cpp:16-55
    _fields_ = [
        ("magic", ctypes.c_uint32),
        ("version", ctypes.c_uint32),
        ("hashMeta", ctypes.c_uint64),
        ("meshletMaxVertices", ctypes.c_uint32),
        ("meshletMaxTriangles", ctypes.c_uint32),
        ("clrtMode", ctypes.c_uint8),
        ("compressed", ctypes.c_uint8),
        ("pad0_", ctypes.c_uint8 * 2),
        ("compressedVertexBytes", ctypes.c_uint32),
        ("compressedIndexBytes", ctypes.c_uint32),
        ("compressedMeshletDataBytes", ctypes.c_uint32),
        ("compressedMeshletVtx0Bytes", ctypes.c_uint32),
        ("vertexCount", ctypes.c_uint32),
        ("indexCount", ctypes.c_uint32),
        ("meshletCount", ctypes.c_uint32),
        ("meshletdataCount", ctypes.c_uint32),
        ("meshletvtx0Count", ctypes.c_uint32),
        ("meshCount", ctypes.c_uint32),
        ("materialCount", ctypes.c_uint32),
        ("drawCount", ctypes.c_uint32),
        ("texturePathCount", ctypes.c_uint32),
        ("lightCount", ctypes.c_uint32),
        ("animationCount", ctypes.c_uint32),
        ("keyframeCount", ctypes.c_uint32),
        ("ommArrayDataSize", ctypes.c_uint32),
        ("ommIndexDataSize", ctypes.c_uint32),
        ("ommDescCount", ctypes.c_uint32),
        ("ommStates", ctypes.c_uint32),
        ("camera", Camera),
        ("sunDirection", ctypes.c_float * 3),
        ("pad1_", ctypes.c_uint32),
    ]


class SceneCacheSection(ctypes.Structure):
    _fields_ = [
        ("offset", ctypes.c_uint64),
        ("stored_bytes", ctypes.c_uint64),
        ("decoded_bytes", ctypes.c_uint64),
        ("count", ctypes.c_uint32),
        ("element_size", ctypes.c_uint32),
        ("compressed", ctypes.c_uint32),
        ("pad_", ctypes.c_uint32),
    ]


class SceneCacheInfo(ctypes.Structure):
    _fields_ = [("header", SceneCacheHeader), ("sections", SceneCacheSection * len(CACHE_SECTIONS))]


class SceneCacheWriteDesc(ctypes.Structure):  # nvc_scene_cache_write
    _fields_ = [
        ("hashMeta", ctypes.c_uint64),
        ("clrtMode", ctypes.c_uint32),
        ("compressed", ctypes.c_uint32),
        ("ommStates", ctypes.c_uint32),
        ("device_sections", ctypes.c_uint32),
        ("camera", Camera),
        ("sunDirection", ctypes.c_float * 3),
        ("data", ctypes.c_void_p * len(CACHE_SECTIONS)),
        ("count", ctypes.c_uint32 * len(CACHE_SECTIONS)),
    ]


assert ctypes.sizeof(SceneCacheHeader) == 160 and ctypes.sizeof(SceneCacheSection) == 40 and ctypes.sizeof(SceneCacheWriteDesc) == 256


def load_nvcg(path):
    """Reads a geometry dump written by oracle/refscene/dump_scene (the reference's own scene.cpp output):
    returns (meshes, meshlets, draws) as structured numpy arrays."""
    raw = open(path, "rb").read()
    header = np.frombuffer(raw, dtype="<u4", count=8)
    if header[0] != 0x4743564E or header[1] != 1:
        raise ValueError("%s: not an NVCG v1 file" % path)
    nmesh, nmeshlet, ndraw = int(header[2]), int(header[3]), int(header[4])
    off = 32
    meshes = np.frombuffer(raw, dtype=MESH_DTYPE, count=nmesh, offset=off).copy()
    off += nmesh * MESH_DTYPE.itemsize
    meshlets = np.frombuffer(raw, dtype=MESHLET_DTYPE, count=nmeshlet, offset=off).copy()
    off += nmeshlet * MESHLET_DTYPE.itemsize
    draws = np.frombuffer(raw, dtype=MESHDRAW_DTYPE, count=ndraw, offset=off).copy()
    return meshes, meshlets, draws
