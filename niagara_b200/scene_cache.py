"""Reader and writer of the reference's scene cache (.cache v7, src/scenecache.cpp) through the C ABI (nvc_scene_cache_*):
SURVEY §8(f) row N2 — the on-disk format that feeds the visibility path.  `section` decodes on the host;
`section_device` reads a section straight into device memory, decoding the vertex and meshlet streams on the GPU;
`write_scene_cache` makes the file saveSceneCache writes, encoding the vertex and meshlet streams on the GPU."""
import ctypes
import mmap

import numpy as np

from . import host, layout
from .lib import NvcError, check, load_library

_DTYPES = {
    "meshlets": layout.MESHLET_DTYPE,
    "meshes": layout.MESH_DTYPE,
    "draws": layout.MESHDRAW_DTYPE,
    "animations": layout.ANIMATION_DTYPE,
    "keyframes": layout.KEYFRAME_DTYPE,
    "meshletdata": np.dtype("<u4"),
    "indices": np.dtype("<u4"),
    "omm_descs": np.dtype("<u4"),
    "meshletvtx0": np.dtype("<u2"),
}


class SceneCache:
    """A parsed cache file.  `section(name)` returns a numpy array (a copy; the meshopt streams of a compressed cache —
    vertices, indices, meshlet data, RT positions — are decoded)."""

    def __init__(self, path):
        self.path = path
        self._file = open(path, "rb")
        self._map = mmap.mmap(self._file.fileno(), 0, access=mmap.ACCESS_READ)
        self._buf = (ctypes.c_char * len(self._map)).from_buffer_copy(self._map) if len(self._map) < (1 << 20) else None
        self.size = len(self._map)
        self.info = layout.SceneCacheInfo()
        self._lib = load_library()
        status = self._lib.nvc_scene_cache_parse(self._address(), self.size, ctypes.byref(self.info))
        if status != 0:
            raise NvcError("%s: %s" % (path, self._lib.nvc_status_string(status).decode()))
        self.header = self.info.header
        self._contexts = {}  # device index -> NvcContext of section_device

    def _address(self):
        if self._buf is not None:
            return ctypes.addressof(self._buf)
        # large files: hand the mapping itself to the library (read-only mmap -> numpy view -> address)
        self._view = np.frombuffer(self._map, dtype=np.uint8)
        return self._view.ctypes.data

    def section_info(self, name):
        return self.info.sections[layout.CACHE_SECTIONS.index(name)]

    def section(self, name):
        idx = layout.CACHE_SECTIONS.index(name)
        sec = self.info.sections[idx]
        raw = np.zeros(int(sec.decoded_bytes), dtype=np.uint8)
        status = self._lib.nvc_scene_cache_read(self._address(), self.size, ctypes.byref(self.info), idx, raw.ctypes.data, raw.nbytes)
        if status != 0:
            raise NvcError("%s[%s]: %s" % (self.path, name, self._lib.nvc_status_string(status).decode()))
        if name == "texture_paths":
            return [bytes(raw[i * 256 : (i + 1) * 256]).split(b"\0", 1)[0].decode() for i in range(sec.count)]
        return raw.view(_DTYPES[name]) if name in _DTYPES else raw

    def section_device(self, name, device="cuda"):
        """The section's decoded bytes as a torch.uint8 tensor on `device`, equal to `section(name)`'s bytes
        (nvc_scene_cache_read_device: the compressed vertex streams, indices and meshlet data go up as stored and are
        decoded by kernels).  Runs on the device's current stream and synchronises the device."""
        import torch

        idx = layout.CACHE_SECTIONS.index(name)
        sec = self.info.sections[idx]
        dev = torch.device(device)
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        out = torch.empty(int(sec.decoded_bytes), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            ctx = self._contexts.get(dev.index)
            if ctx is None:
                ctx = ctypes.c_void_p()
                check(self._lib.nvc_create(dev.index, None, ctypes.byref(ctx)), None, "nvc_create")
                self._contexts[dev.index] = ctx
            stream = torch.cuda.current_stream(dev).cuda_stream
            status = self._lib.nvc_scene_cache_read_device(ctx, stream, self._address(), self.size, ctypes.byref(self.info), idx, out.data_ptr() if out.numel() else None, out.numel())
        if status != 0:
            detail = self._lib.nvc_last_error(ctx).decode()
            raise NvcError("%s[%s]: %s%s" % (self.path, name, self._lib.nvc_status_string(status).decode(), " (%s)" % detail if detail else ""))
        return out

    def camera(self):
        c = self.header.camera
        return host.make_camera(tuple(c.position), tuple(c.orientation), float(c.fovY), float(c.znear))

    def close(self):
        for ctx in self._contexts.values():
            self._lib.nvc_destroy(ctx)
        self._contexts = {}
        self._view = None
        self._map.close()
        self._file.close()


_ELEMENT_SIZE = dict(zip(layout.CACHE_SECTIONS, (16, 4, 24, 4, 2, 208, 64, 48, 32, 24, 32, 1, 1, 4, 256)))
_WRITE_CONTEXTS = {}  # device index -> NvcContext of write_scene_cache


def _write_context(lib, index):
    ctx = _WRITE_CONTEXTS.get(index)
    if ctx is None:
        ctx = ctypes.c_void_p()
        check(lib.nvc_create(index, None, ctypes.byref(ctx)), None, "nvc_create")
        _WRITE_CONTEXTS[index] = ctx
    return ctx


def write_scene_cache(sections, compressed=True, hash_meta=0, clrt_mode=False, omm_states=0, camera=None, sun_direction=(0.0, 0.0, 0.0), device=None):
    """The bytes of the scene cache saveSceneCache writes for `sections` (nvc_scene_cache_write).  `sections` maps names of
    layout.CACHE_SECTIONS to numpy arrays or torch tensors (CUDA tensors are read where they lie), whose bytes are the
    section's elements; missing sections are empty; "texture_paths" may also be a list of str.  `camera` is a
    layout.Camera.  A compressed cache encodes the vertex and meshlet streams on `device` (default: the device of the
    CUDA tensors given, else the current one), on its current stream; the call synchronises that device."""
    lib = load_library()
    desc = layout.SceneCacheWriteDesc()
    desc.hashMeta, desc.clrtMode, desc.compressed, desc.ommStates = int(hash_meta), int(bool(clrt_mode)), int(bool(compressed)), int(omm_states)
    if camera is not None:
        desc.camera = camera
    desc.sunDirection[:] = [float(x) for x in sun_direction]
    keep = []
    cuda_index = None
    for name, value in sections.items():
        idx = layout.CACHE_SECTIONS.index(name)
        if name == "texture_paths" and isinstance(value, (list, tuple)):
            value = np.frombuffer(b"".join(p.encode()[:256].ljust(256, b"\0") for p in value), np.uint8)
        if hasattr(value, "is_cuda") and value.is_cuda:
            value = value.contiguous()
            cuda_index = value.device.index if cuda_index is None else cuda_index
            if value.device.index != cuda_index:
                raise NvcError("write_scene_cache: CUDA tensors on more than one device")
            nbytes, ptr = value.numel() * value.element_size(), value.data_ptr()
            desc.device_sections |= 1 << idx
        else:
            value = np.ascontiguousarray(value.cpu().numpy() if hasattr(value, "cpu") else value)
            nbytes, ptr = value.nbytes, value.ctypes.data
        if nbytes % _ELEMENT_SIZE[name]:
            raise NvcError("write_scene_cache: %s holds %d bytes, not a multiple of its %d-byte elements" % (name, nbytes, _ELEMENT_SIZE[name]))
        keep.append(value)
        desc.data[idx], desc.count[idx] = (ptr if nbytes else None), nbytes // _ELEMENT_SIZE[name]
    bound = ctypes.c_size_t()
    check(lib.nvc_scene_cache_write_bound(ctypes.byref(desc), ctypes.byref(bound)), None, "nvc_scene_cache_write_bound")
    out = np.empty(max(int(bound.value), 1), np.uint8)
    size = ctypes.c_size_t()
    needs_device = desc.device_sections != 0 or (compressed and (desc.count[0] or desc.count[2] or desc.count[4]))
    if not needs_device:
        check(lib.nvc_scene_cache_write(None, None, ctypes.byref(desc), out.ctypes.data, out.nbytes, ctypes.byref(size)), None, "nvc_scene_cache_write")
        return out[: size.value].tobytes()
    import torch

    dev = torch.device(device) if device is not None else torch.device("cuda", cuda_index if cuda_index is not None else torch.cuda.current_device())
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        ctx = _write_context(lib, dev.index)
        stream = torch.cuda.current_stream(dev).cuda_stream
        check(lib.nvc_scene_cache_write(ctx, stream, ctypes.byref(desc), out.ctypes.data, out.nbytes, ctypes.byref(size)), ctx, "nvc_scene_cache_write")
    return out[: size.value].tobytes()


def load_scene(path, screen=(1024, 768), depth=None, name=None):
    """Scene (niagara_b200.scenes.Scene) from a cache file: Mesh[] / Meshlet[] / MeshDraw[] exactly as stored, the
    cache's camera, meshletVisibilityOffset as stored (niagara.cpp:1003-1020 assigns it before saving)."""
    from . import scenes

    c = SceneCache(path)
    meshes, meshlets, draws = c.section("meshes"), c.section("meshlets"), c.section("draws")
    bits = 0
    if len(draws):
        counts = meshes["lods"]["meshletCount"].max(axis=1)[draws["meshIndex"]]
        bits = int((draws["meshletVisibilityOffset"].astype(np.int64) + counts).max())
    cam = c.camera()
    if depth is None:
        depth = scenes.synthetic_depth(screen[0], screen[1], cam.znear, occluders=40, seed=9)
    s = scenes.Scene(name or path, meshes, meshlets, draws, depth, cam, screen, bits)
    s.animations, s.keyframes = c.section("animations"), c.section("keyframes")
    c.close()
    return s
