"""The PRODUCT's kernels executed on the CPU: niagara_b200/csrc/nvc_kernels.cu + nvc_api.cu compiled by g++ against
tests/cuda_emu (a SIMT emulation: fibers per CUDA thread, rendezvous for warp collectives and __syncthreads) into
tests/_build/emu/libniagara_cull_emu.so, driven through the SAME C ABI with host pointers.  Test infrastructure: it lets
the CPU tier check kernel logic (indexing, scans, compaction, epilogues, arithmetic order) when no GPU is at hand; the
parity tests proper remain the -m gpu ones."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_lib
from niagara_b200 import layout
from niagara_b200 import lib as product_lib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "niagara_b200", "csrc")
EMU = os.path.join(HERE, "cuda_emu")
OUT = os.path.join(HERE, "_build", "emu")
_LIB = None


def load():
    """Builds (when stale) and loads the emulated library: the translated kernels and API, the emulation, the host sources
    (nvc_host, the scene-cache reader and writer and their codecs) and cuda_emu/guard_alloc.cpp.  Its calloc / free are
    wrapped: after emu_guard_allocations(1) every device allocation ends exactly at an inaccessible page, so that a kernel
    that reads past a context-owned buffer faults; until then every call goes to the C library."""
    global _LIB
    so = os.path.join(OUT, "libniagara_cull_emu.so")
    if _LIB is not None:
        return _LIB
    os.makedirs(OUT, exist_ok=True)
    emu = [os.path.join(EMU, f) for f in ("emu.cpp", "emu_stubs.cpp", "guard_alloc.cpp")]
    host = [os.path.join(CSRC, f + ".cpp") for f in ("nvc_host", "nvc_scene_cache", "nvc_scene_cache_device", "nvc_scene_cache_write", "nvc_meshopt_decode", "nvc_meshopt_encode")]
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + emu + [os.path.join(EMU, "gen_emu.py")] + [os.path.join(EMU, "include", f) for f in os.listdir(os.path.join(EMU, "include"))] + [os.path.join(ROOT, "include", "niagara_cull.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        for name in ("nvc_kernels", "nvc_api"):
            subprocess.run(["python3", os.path.join(EMU, "gen_emu.py"), os.path.join(CSRC, name + ".cu"), os.path.join(OUT, name + ".cpp")], check=True)
        cmd = ["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-w", "-I", os.path.join(EMU, "include"), "-I", CSRC]
        cmd += ["-Wl,--wrap=calloc,--wrap=free", "-o", so, os.path.join(OUT, "nvc_kernels.cpp"), os.path.join(OUT, "nvc_api.cpp")] + emu + host
        subprocess.run(cmd, check=True)
    lib = ctypes.CDLL(so)
    for name, restype, argtypes in product_lib.SIGNATURES:
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
    lib.emu_guard_allocations.argtypes = [ctypes.c_int]
    lib.emu_guard_allocations.restype = None
    lib.emu_guarded_live.restype = ctypes.c_int
    _LIB = lib
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


class EmuPath(oracle_lib.OraclePath):
    """OraclePath's buffers, every pass executed by the product's kernels under the SIMT emulation."""

    def __init__(self, *args, prepare_meshes=True, prepare_hiz=True, **kwargs):
        super().__init__(*args, **kwargs)
        self.emu = load()
        self.ctx = ctypes.c_void_p()
        limits = layout.Limits(self.limits.task_wglimit, self.limits.cluster_limit)
        assert self.emu.nvc_create(0, ctypes.byref(limits), ctypes.byref(self.ctx)) == 0
        if prepare_meshes:
            assert self.emu.nvc_prepare_meshes(self.ctx, None, _p(self.meshes), len(self.meshes)) == 0
        if prepare_hiz:
            assert self.emu.nvc_prepare_hiz(self.ctx, ctypes.byref(self.hiz)) == 0

    def _check(self, status, what):
        assert status == 0, (what, status, self.emu.nvc_last_error(self.ctx))

    def cull(self, cull_data, late, post_pass=0, task=None):
        task = self.mesh_shading if task is None else task
        pd = self._pass_data(cull_data, 1, post_pass)
        self._check(self.emu.nvc_drawcull(self.ctx, None, ctypes.byref(pd), int(late), int(task), _p(self.draws), _p(self.meshes), _p(self.dvb), _p(self.dcb), _p(self.dccb), ctypes.byref(self.hiz)), "nvc_drawcull")

    def render_clusters(self, cull_data, late, post_pass=0, cluster_backface=None):
        pd = self._pass_data(cull_data, 0, post_pass)
        if cluster_backface is not None:
            pd.clusterBackfaceEnabled = int(cluster_backface)
        self._check(self.emu.nvc_clustercull(self.ctx, None, ctypes.byref(pd), int(late), _p(self.dcb), _p(self.dccb), _p(self.draws), _p(self.meshlets), _p(self.mvb), _p(self.cib), _p(self.ccb), ctypes.byref(self.hiz)), "nvc_clustercull")

    def task_shading(self, cull_data, late, payloads, emit_counts, post_pass=0, cluster_backface=None):
        pd = self._pass_data(cull_data, 0, post_pass)
        if cluster_backface is not None:
            pd.clusterBackfaceEnabled = int(cluster_backface)
        self._check(self.emu.nvc_taskcull(self.ctx, None, ctypes.byref(pd), int(late), _p(self.dcb), _p(self.dccb), _p(self.draws), _p(self.meshlets), _p(self.mvb), _p(payloads), _p(emit_counts), ctypes.byref(self.hiz)), "nvc_taskcull")

    def pyramid(self, depth):
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        self._check(self.emu.nvc_depth_pyramid(self.ctx, None, _p(depth), self.depth_width, self.depth_height, ctypes.byref(self.hiz)), "nvc_depth_pyramid")

    def raster_depth(self, cull_data, projection16, vertices, meshletdata, depth, cib=None, ccb=None, dcb=None):
        """nvc_raster_depth over (cib, ccb) (default: this path's own); returns stats[4]"""
        cib = self.cib if cib is None else np.ascontiguousarray(cib, dtype=np.uint32)
        ccb = self.ccb if ccb is None else np.ascontiguousarray(ccb, dtype=np.uint32)
        dcb = self.dcb if dcb is None else dcb
        pd = self._pass_data(cull_data, 0, 0)
        proj = np.ascontiguousarray(projection16, dtype=np.float32)
        md = np.ascontiguousarray(meshletdata, dtype=np.uint32)
        vb = np.ascontiguousarray(vertices)
        stats = np.zeros(4, np.uint32)
        self._check(self.emu.nvc_raster_depth(self.ctx, None, _p(proj), ctypes.byref(pd), _p(cib), _p(ccb), _p(dcb), _p(self.draws), _p(self.meshlets), _p(md), len(md), _p(vb), vb.nbytes // 16, _p(depth), depth.shape[1], depth.shape[0], _p(stats)), "nvc_raster_depth")
        return stats

    def close(self):
        if self.ctx:
            self.emu.nvc_destroy(self.ctx)
            self.ctx = None
