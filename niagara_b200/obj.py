"""OBJ import on the device through the C ABI (nvc_obj_load): what the reference's loadMesh gets from loadObj
(src/scene.cpp:117-168), one Vertex[] record per triangle corner, ready for nvc_cook_mesh_vertices."""
import ctypes
import os

import numpy as np

from .lib import NvcError, check, load_library


class ObjFile(ctypes.Structure):
    _fields_ = [("data", ctypes.c_void_p), ("size", ctypes.c_uint64)]


class ObjInfo(ctypes.Structure):
    _fields_ = [
        ("bytes_parsed", ctypes.c_uint64),
        ("position_count", ctypes.c_uint32),
        ("texcoord_count", ctypes.c_uint32),
        ("normal_count", ctypes.c_uint32),
        ("face_count", ctypes.c_uint32),
        ("index_count", ctypes.c_uint64),
        ("corner_offset", ctypes.c_uint64),
        ("corner_count", ctypes.c_uint64),
    ]


assert ctypes.sizeof(ObjFile) == 16 and ctypes.sizeof(ObjInfo) == 48


def info_dict(info):
    return {name: int(getattr(info, name)) for name, _ in ObjInfo._fields_}


def file_table(blobs):
    """(ObjFile array, the numpy buffers it points into: keep them alive) for a list of bytes objects"""
    bufs = [np.frombuffer(b, np.uint8) if len(b) else None for b in blobs]
    table = (ObjFile * max(len(blobs), 1))()
    for k, b in enumerate(bufs):
        table[k].data = b.ctypes.data if b is not None else None
        table[k].size = 0 if b is None else len(b)
    return table, bufs


def load_obj(files, stream=None, ctx=None):
    """files: paths or bytes.  Returns (vertices, infos): a (n, 8) torch.uint16 tensor on the current CUDA device (the Vertex[]
    of every file, file after file) and one dict per file (NvcObjInfo: bytes_parsed, the v / vt / vn / face / index record counts,
    corner_offset and corner_count, the file's rows of `vertices`).  Raises NvcError when the call refuses the files."""
    import torch

    lib = load_library()
    blobs = [f if isinstance(f, (bytes, bytearray)) else open(os.fspath(f), "rb").read() for f in files]
    own = ctx is None
    if own:
        ctx = ctypes.c_void_p()
        check(lib.nvc_create(torch.cuda.current_device(), None, ctypes.byref(ctx)), None, "nvc_create")
    try:
        table, _keep = file_table(blobs)
        infos = (ObjInfo * max(len(blobs), 1))()
        s = stream.cuda_stream if stream is not None else None
        check(lib.nvc_obj_load(ctx, s, table, len(blobs), None, 0, infos), ctx, "nvc_obj_load")
        total = sum(int(infos[k].corner_count) for k in range(len(blobs)))
        out = torch.empty((max(total, 1), 16), dtype=torch.uint8, device="cuda")
        check(lib.nvc_obj_load(ctx, s, table, len(blobs), out.data_ptr(), total, infos), ctx, "nvc_obj_load")
        if own:
            torch.cuda.synchronize()
        return out[:total].view(torch.uint16), [info_dict(infos[k]) for k in range(len(blobs))]
    finally:
        if own:
            lib.nvc_destroy(ctx)


__all__ = ["ObjFile", "ObjInfo", "NvcError", "load_obj"]
