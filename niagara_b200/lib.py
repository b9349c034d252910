"""ctypes binding of the C ABI in include/niagara_cull.h (libniagara_cull.so).

There is NO CPU fallback: if the shared library is missing, or no CUDA device is present when a context is
created, this module raises.  The oracle under oracle/ is never imported from here."""
import ctypes
import os

from . import _build
from .layout import Camera, CullData, CullOptions, GltfInfo, HiZ, Limits, SceneCacheInfo, SceneCacheWriteDesc

_LIB = None

c_void_p = ctypes.c_void_p
c_u32_p = ctypes.POINTER(ctypes.c_uint32)


class NvcError(RuntimeError):
    pass


# every symbol include/niagara_cull.h declares: (name, restype, argtypes)
SIGNATURES = [
    ("nvc_create", ctypes.c_int, [ctypes.c_int, ctypes.POINTER(Limits), ctypes.POINTER(c_void_p)]),
    ("nvc_destroy", None, [c_void_p]),
    ("nvc_status_string", ctypes.c_char_p, [ctypes.c_int]),
    ("nvc_last_error", ctypes.c_char_p, [c_void_p]),
    ("nvc_version", ctypes.c_char_p, []),
    ("nvc_prepare_meshes", ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_uint32]),
    ("nvc_prepare_meshlets", ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_uint32]),
    ("nvc_set_hiz_staging", ctypes.c_int, [c_void_p, ctypes.c_uint32]),
    ("nvc_prepare_hiz", ctypes.c_int, [c_void_p, ctypes.POINTER(HiZ)]),
    ("nvc_set_cluster_filter", ctypes.c_int, [c_void_p, ctypes.c_int]),
    ("nvc_gltf_import", ctypes.c_int, [c_void_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(c_void_p)]),
    ("nvc_gltf_free", None, [c_void_p]),
    ("nvc_gltf_info", ctypes.c_int, [c_void_p, ctypes.POINTER(GltfInfo)]),
    ("nvc_gltf_scene_arrays", ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("nvc_gltf_primitive_size", ctypes.c_int, [c_void_p, ctypes.c_uint32, c_u32_p, c_u32_p]),
    ("nvc_gltf_primitive_data", ctypes.c_int, [c_void_p, ctypes.c_uint32, c_void_p, c_void_p]),
    ("nvc_raster_depth", ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.POINTER(CullData), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, ctypes.c_uint32, c_void_p]),
    ("nvc_raster_depth_tasks", ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.POINTER(CullData), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, ctypes.c_uint32, c_void_p]),
    ("nvc_raster_depth_indexed", ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.POINTER(CullData), c_void_p, c_void_p, ctypes.c_uint32, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, ctypes.c_uint32, c_void_p]),
    ("nvc_filter_stats", ctypes.c_int, [c_void_p, ctypes.POINTER(ctypes.c_uint64), ctypes.c_int]),
    ("nvc_filter_approx", ctypes.c_int, [c_void_p, c_void_p, ctypes.c_int, c_void_p, c_void_p, ctypes.c_uint64]),
    ("nvc_set_mesh_cull", ctypes.c_int, [c_void_p, ctypes.c_int]),
    ("nvc_mesh_cull_stats", ctypes.c_int, [c_void_p, ctypes.POINTER(ctypes.c_uint64), ctypes.c_int]),
    ("nvc_set_task_cull", ctypes.c_int, [c_void_p, ctypes.c_int]),
    ("nvc_previous_pow2", ctypes.c_uint32, [ctypes.c_uint32]),
    ("nvc_image_mip_levels", ctypes.c_uint32, [ctypes.c_uint32, ctypes.c_uint32]),
    ("nvc_hiz_layout", ctypes.c_int, [ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(HiZ)]),
    (
        "nvc_drawcull",
        ctypes.c_int,
        [c_void_p, c_void_p, ctypes.POINTER(CullData), ctypes.c_int, ctypes.c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.POINTER(HiZ)],
    ),
    (
        "nvc_clustercull",
        ctypes.c_int,
        [c_void_p, c_void_p, ctypes.POINTER(CullData), ctypes.c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.POINTER(HiZ)],
    ),
    (
        "nvc_taskcull",
        ctypes.c_int,
        [c_void_p, c_void_p, ctypes.POINTER(CullData), ctypes.c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.POINTER(HiZ)],
    ),
    ("nvc_decode_clusters", ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("nvc_depth_pyramid", ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(HiZ)]),
    ("nvc_host_random_draws", None, [c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_float]),
    ("nvc_host_visibility_offsets", ctypes.c_uint32, [c_void_p, ctypes.c_uint32, c_void_p, c_u32_p]),
    (
        "nvc_host_cull_data",
        None,
        [ctypes.POINTER(Camera), ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(CullOptions), ctypes.POINTER(CullData), c_void_p],
    ),
    ("nvc_host_pass_data", None, [ctypes.POINTER(CullData), ctypes.c_int, ctypes.c_uint32, ctypes.POINTER(CullData)]),
    ("nvc_scene_cache_parse", ctypes.c_int, [c_void_p, ctypes.c_size_t, ctypes.POINTER(SceneCacheInfo)]),
    ("nvc_scene_cache_read", ctypes.c_int, [c_void_p, ctypes.c_size_t, ctypes.POINTER(SceneCacheInfo), ctypes.c_int, c_void_p, ctypes.c_size_t]),
    ("nvc_scene_cache_read_device", ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_size_t, ctypes.POINTER(SceneCacheInfo), ctypes.c_int, c_void_p, ctypes.c_size_t]),
    ("nvc_scene_cache_write_bound", ctypes.c_int, [ctypes.POINTER(SceneCacheWriteDesc), ctypes.POINTER(ctypes.c_size_t)]),
    ("nvc_scene_cache_write", ctypes.c_int, [c_void_p, c_void_p, ctypes.POINTER(SceneCacheWriteDesc), c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]),
    ("nvc_decode_vertex_stream", ctypes.c_int, [c_void_p, ctypes.c_uint32, ctypes.c_uint32, c_void_p, ctypes.c_size_t]),
    ("nvc_decode_index_stream", ctypes.c_int, [c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_size_t]),
    ("nvc_decode_meshlet_stream", ctypes.c_int, [c_void_p, ctypes.c_uint32, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_size_t]),
    ("nvc_decode_index_buffer", ctypes.c_int, [c_void_p, ctypes.c_uint32, ctypes.c_uint32, c_void_p, ctypes.c_size_t]),
    ("nvc_decode_index_sequence", ctypes.c_int, [c_void_p, ctypes.c_uint32, ctypes.c_uint32, c_void_p, ctypes.c_size_t]),
    ("nvc_decode_vertex_filter", ctypes.c_int, [ctypes.c_int, c_void_p, ctypes.c_uint32, ctypes.c_uint32]),
    (
        "nvc_host_animate",
        ctypes.c_int,
        [c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, ctypes.c_double, c_void_p, ctypes.c_uint32, c_void_p, c_void_p, ctypes.c_uint32],
    ),
    ("nvc_update_draws", ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, c_void_p, ctypes.c_uint32]),
    ("nvc_cook_meshlet_bounds", ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p]),
    (
        "nvc_cook_meshlets",
        ctypes.c_int,
        [c_void_p, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p],
    ),
    ("nvc_cook_meshlets_capacity", ctypes.c_int, [c_void_p, ctypes.c_uint32, c_u32_p, ctypes.POINTER(ctypes.c_uint64)]),
    (
        "nvc_cook_meshlets_clrt",
        ctypes.c_int,
        [c_void_p, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p,
         ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p],
    ),
    ("nvc_cook_meshlets_clrt_capacity", ctypes.c_int, [c_void_p, c_void_p, ctypes.c_uint32, c_u32_p, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64)]),
    ("nvc_cook_mesh_lods_capacity", ctypes.c_int, [c_void_p, ctypes.c_uint32, c_u32_p]),
    (
        "nvc_cook_mesh_lods",
        ctypes.c_int,
        [c_void_p, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, c_void_p,
         ctypes.c_uint32, c_void_p],
    ),
    (
        "nvc_cook_mesh_vertices",
        ctypes.c_int,
        [c_void_p, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint32, c_void_p, c_void_p, ctypes.c_uint32,
         c_void_p, ctypes.c_uint32, c_void_p],
    ),
    ("nvc_obj_load", ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_uint32, c_void_p, ctypes.c_uint64, c_void_p]),
    ("nvc_nccl_unique_id", ctypes.c_int, [c_void_p]),
    ("nvc_nccl_init", ctypes.c_int, [c_void_p, c_void_p, ctypes.c_int, ctypes.c_int]),
    ("nvc_allgather_visible", ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_size_t, c_void_p, c_void_p, c_void_p]),
    ("nvc_hiz_footprints", ctypes.c_int, [c_void_p, ctypes.POINTER(c_void_p), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint32)]),
    ("nvc_gather_create", ctypes.c_int, [c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, c_void_p]),
    ("nvc_gather_connect", ctypes.c_int, [c_void_p, c_void_p]),
    ("nvc_gather_push", ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    ("nvc_gather_wait", ctypes.c_int, [c_void_p, c_void_p]),
    ("nvc_gather_set_mode", ctypes.c_int, [c_void_p, ctypes.c_int]),
    ("nvc_gather_region_bytes", ctypes.c_size_t, [ctypes.c_size_t, ctypes.c_int]),
    ("nvc_gather_attach", ctypes.c_int, [c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.POINTER(c_void_p), c_void_p]),
    ("nvc_gather_fuse_next_drawcull", ctypes.c_int, [c_void_p, c_void_p]),
    ("nvc_gather_buffers", ctypes.c_int, [c_void_p, ctypes.POINTER(c_void_p), ctypes.POINTER(c_void_p)]),
    ("nvc_gather_graph_advance", ctypes.c_int, [c_void_p, c_void_p, ctypes.c_uint32]),
    ("nvc_gather_status", ctypes.c_int, [c_void_p, ctypes.POINTER(ctypes.c_int)]),
]


def library_path():
    # NVC_LIB_PATH selects another build of the library (e.g. one of another revision, made with _build.build(out=...), for an
    # A/B); default = the product build
    return os.environ.get("NVC_LIB_PATH") or _build.LIB_PATH


def load_library():
    """Loads libniagara_cull.so (must have been built: `python -m niagara_b200._build` or __graft_entry__.build())."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not os.path.exists(path):
        raise NvcError(
            "%s is missing: the CUDA extension has not been built (run `python -c 'import __graft_entry__ as g; g.build()'`). "
            "There is no CPU fallback." % path
        )
    lib = ctypes.CDLL(path)
    for name, restype, argtypes in SIGNATURES:
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    _LIB = lib
    return lib


def check(status, ctx=None, what=""):
    if status != 0:
        lib = load_library()
        msg = lib.nvc_status_string(status).decode()
        if ctx:
            detail = lib.nvc_last_error(ctx).decode()
            if detail:
                msg += " (" + detail + ")"
        raise NvcError("%s failed: %s" % (what or "nvc call", msg))
