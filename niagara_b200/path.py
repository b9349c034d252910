"""VisibilityPath — the host-side mirror of the reference's hot-path call sites (src/niagara.cpp):

    cull(late, post_pass)             niagara.cpp:1530-1574   cull lambda   (drawcull [+ tasksubmit])
    render_clusters(late, post_pass)  niagara.cpp:1582-1610   cluster block of the render lambda (clustercull + clustersubmit)
    pyramid(depth)                    niagara.cpp:1703-1733   pyramid lambda (depthreduce per mip)
    frame(...)                        niagara.cpp:1765-1788   pass order: early cull/render, pyramid, late cull/render[, post]

Buffers carry the reference's names (db, mb, mlb, dvb, mvb, dcb, dccb, cib, ccb, depthPyramid; niagara.cpp:1027-1090).
PyTorch is only used to own device memory and streams; every pass goes through the C ABI (libniagara_cull.so)."""
import ctypes
import os

import numpy as np
import torch

from . import layout
from .lib import check, load_library


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _round_up(v, m):
    return (v + m - 1) // m * m


class VisibilityPath:
    def __init__(self, meshes, meshlets, draws, depth_width, depth_height, device="cuda:0", task_wglimit=layout.TASK_WGLIMIT, cluster_limit=layout.CLUSTER_LIMIT, mesh_shading=True, hiz_stage_texels=None, prepare_meshes=True, prepare_meshlets=True, prepare_hiz=True):
        """meshes / meshlets / draws: structured numpy arrays (layout.MESH_DTYPE / MESHLET_DTYPE / MESHDRAW_DTYPE) or
        already-resident torch uint8 tensors.  draws must already carry meshletVisibilityOffset
        (host.visibility_offsets)."""
        if not torch.cuda.is_available():
            raise RuntimeError("VisibilityPath needs a CUDA device; there is no CPU fallback")
        self.lib = load_library()
        self.device = torch.device(device)
        self.mesh_shading = bool(mesh_shading)
        torch.cuda.set_device(self.device)

        limits = layout.Limits(task_wglimit, cluster_limit)
        ctx = ctypes.c_void_p()
        check(self.lib.nvc_create(self.device.index or 0, ctypes.byref(limits), ctypes.byref(ctx)), None, "nvc_create")
        self.ctx = ctx
        if hiz_stage_texels is not None:
            check(self.lib.nvc_set_hiz_staging(self.ctx, int(hiz_stage_texels)), self.ctx, "nvc_set_hiz_staging")
        self.task_wglimit = int(task_wglimit)
        self.cluster_limit = int(cluster_limit)

        self.draw_count = int(len(draws)) if not isinstance(draws, torch.Tensor) else draws.numel() // layout.MESHDRAW_DTYPE.itemsize
        self.mb = self._upload(meshes)
        self.mlb = self._upload(meshlets)
        self.db = self._upload(draws)
        if prepare_meshes:  # derived cull view of Mesh[] (once per geometry upload)
            mesh_count = self.mb.numel() // layout.MESH_DTYPE.itemsize
            check(self.lib.nvc_prepare_meshes(self.ctx, self._stream(), _ptr(self.mb), mesh_count), self.ctx, "nvc_prepare_meshes")
        if prepare_meshlets:  # derived cull view of Meshlet[]: the 12 bytes the cluster passes read, as two dense arrays
            meshlet_count = self.mlb.numel() // layout.MESHLET_DTYPE.itemsize
            check(self.lib.nvc_prepare_meshlets(self.ctx, self._stream(), _ptr(self.mlb), meshlet_count), self.ctx, "nvc_prepare_meshlets")

        # niagara.cpp:1062-1090
        self.dvb = torch.zeros(max(1, self.draw_count), dtype=torch.int32, device=self.device)
        cmd_bytes = max(_round_up(self.task_wglimit, 64) * layout.MESHTASKCOMMAND_DTYPE.itemsize, self.draw_count * layout.MESHDRAWCOMMAND_DTYPE.itemsize)
        self.dcb = torch.zeros(cmd_bytes, dtype=torch.uint8, device=self.device)
        self.dccb = torch.zeros(4, dtype=torch.int32, device=self.device)
        self.cib = torch.zeros(_round_up(self.cluster_limit, 256), dtype=torch.int32, device=self.device)
        self.ccb = torch.zeros(4, dtype=torch.int32, device=self.device)
        self.mvb = None  # sized by set_visibility_bits()

        self.depth_width, self.depth_height = int(depth_width), int(depth_height)
        self.hiz = layout.HiZ()
        check(self.lib.nvc_hiz_layout(self.depth_width, self.depth_height, ctypes.byref(self.hiz)), self.ctx, "nvc_hiz_layout")
        self.depthPyramid = torch.zeros(self.hiz.total_texels, dtype=torch.float32, device=self.device)
        self.hiz.texels = self.depthPyramid.data_ptr()
        if prepare_hiz and os.environ.get("NVC_PREPARE_HIZ", "1") != "0":  # derived footprint image of the pyramid (rebuilt by every nvc_depth_pyramid call)
            check(self.lib.nvc_prepare_hiz(self.ctx, ctypes.byref(self.hiz)), self.ctx, "nvc_prepare_hiz")

    # -- buffers ------------------------------------------------------------------------------------------
    def _upload(self, arr):
        if isinstance(arr, torch.Tensor):
            return arr.to(self.device)
        raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
        return torch.from_numpy(raw.copy()).to(self.device)

    def set_visibility_bits(self, meshlet_visibility_count):
        """mvb: (count + 31) / 32 words, zeroed on the first frame (niagara.cpp:1020,1081,1460-1468)."""
        words = max(1, (int(meshlet_visibility_count) + 31) // 32)
        self.mvb = torch.zeros(words, dtype=torch.int32, device=self.device)

    def update_draws(self, draws):
        """The reference rewrites the host-visible `db` when animating (niagara.cpp:1362-1411)."""
        raw = torch.from_numpy(np.ascontiguousarray(draws).view(np.uint8).reshape(-1))
        self.db.copy_(raw, non_blocking=True)

    def scatter_draws(self, indices, values):
        """Incremental form (N3): only the animated draws travel — one packed H2D copy of {index, MeshDraw} and one
        scatter launch (nvc_update_draws) instead of rewriting the whole buffer."""
        n = int(len(indices))
        if n == 0:
            return
        idx = torch.from_numpy(np.ascontiguousarray(indices, dtype=np.uint32).view(np.int32)).pin_memory().to(self.device, non_blocking=True)
        val = torch.from_numpy(np.ascontiguousarray(values).view(np.uint8).reshape(-1)).pin_memory().to(self.device, non_blocking=True)
        check(self.lib.nvc_update_draws(self.ctx, self._stream(), _ptr(self.db), self.draw_count, _ptr(idx), _ptr(val), n), self.ctx, "nvc_update_draws")

    def close(self):
        if getattr(self, "ctx", None):
            self.lib.nvc_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # -- passes -------------------------------------------------------------------------------------------
    def cull(self, cull_data, late, post_pass=0, task=None):
        """cull lambda, niagara.cpp:1530-1574.  task defaults to meshSubmit (mesh shading on)."""
        task = self.mesh_shading if task is None else task
        pass_data = layout.CullData()
        self.lib.nvc_host_pass_data(ctypes.byref(cull_data), 1, post_pass, ctypes.byref(pass_data))
        check(
            self.lib.nvc_drawcull(self.ctx, self._stream(), ctypes.byref(pass_data), int(late), int(task), _ptr(self.db), _ptr(self.mb), _ptr(self.dvb), _ptr(self.dcb), _ptr(self.dccb), ctypes.byref(self.hiz)),
            self.ctx,
            "nvc_drawcull",
        )

    def render_clusters(self, cull_data, late, post_pass=0, cluster_backface=None):
        """clusterSubmit block of the render lambda, niagara.cpp:1582-1610.  cluster_backface=None keeps the
        reference's wiring (flag stays 0 for this pass, SURVEY F8); True/False overrides it."""
        pass_data = layout.CullData()
        self.lib.nvc_host_pass_data(ctypes.byref(cull_data), 0, post_pass, ctypes.byref(pass_data))
        if cluster_backface is not None:
            pass_data.clusterBackfaceEnabled = int(cluster_backface)
        check(
            self.lib.nvc_clustercull(self.ctx, self._stream(), ctypes.byref(pass_data), int(late), _ptr(self.dcb), _ptr(self.dccb), _ptr(self.db), _ptr(self.mlb), _ptr(self.mvb), _ptr(self.cib), _ptr(self.ccb), ctypes.byref(self.hiz)),
            self.ctx,
            "nvc_clustercull",
        )

    def task_shading(self, cull_data, late, payloads, emit_counts, post_pass=0, cluster_backface=None):
        """taskShadingEnabled path, niagara.cpp:1666-1679 (meshlet.task.glsl)."""
        pass_data = layout.CullData()
        self.lib.nvc_host_pass_data(ctypes.byref(cull_data), 0, post_pass, ctypes.byref(pass_data))
        if cluster_backface is not None:
            pass_data.clusterBackfaceEnabled = int(cluster_backface)
        check(
            self.lib.nvc_taskcull(self.ctx, self._stream(), ctypes.byref(pass_data), int(late), _ptr(self.dcb), _ptr(self.dccb), _ptr(self.db), _ptr(self.mlb), _ptr(self.mvb), _ptr(payloads), _ptr(emit_counts), ctypes.byref(self.hiz)),
            self.ctx,
            "nvc_taskcull",
        )

    def pyramid(self, depth):
        """pyramid lambda, niagara.cpp:1703-1733.  depth: float32 device tensor [depth_height, depth_width]."""
        assert depth.dtype == torch.float32 and depth.is_contiguous() and depth.numel() == self.depth_width * self.depth_height
        check(self.lib.nvc_depth_pyramid(self.ctx, self._stream(), _ptr(depth), self.depth_width, self.depth_height, ctypes.byref(self.hiz)), self.ctx, "nvc_depth_pyramid")

    def set_mesh_cull(self, enabled):
        """The mesh shader's per-triangle cull stage (meshlet.mesh.glsl with MESH_CULL = 1) in raster_depth and raster_depth_tasks
        calls made after this one: back-facing, zero-area and small triangles are not sampled.  Off by default, as in the reference;
        raster_depth_indexed is not affected."""
        check(self.lib.nvc_set_mesh_cull(self.ctx, int(bool(enabled))), self.ctx, "nvc_set_mesh_cull")

    def set_task_cull(self, enabled):
        """The reference's TASK_CULL switch for cull, render_clusters and task_shading calls made after this one.
        Off: the late drawcull emits only draws not visible last frame (plus post-pass draws), and the cluster and task passes pass
        every meshlet of every command through without a test, leaving mvb untouched.  On by default, as in the reference."""
        check(self.lib.nvc_set_task_cull(self.ctx, int(bool(enabled))), self.ctx, "nvc_set_task_cull")

    def mesh_cull_stats(self, reset=False):
        """(triangles tested, triangles culled) by the mesh-cull stage since the last reset (synchronises the device)."""
        out = (ctypes.c_uint64 * 2)()
        check(self.lib.nvc_mesh_cull_stats(self.ctx, out, int(bool(reset))), self.ctx, "nvc_mesh_cull_stats")
        return int(out[0]), int(out[1])

    def raster_depth(self, cull_data, projection16, vertices, meshletdata, depth, stats=None):
        """Depth-only consumer of this path's cib / ccb / dcb on the device (nvc_raster_depth): what the reference's mesh stage +
        rasteriser do to the depth target between the cull passes.  vertices: uint8 device tensor of 16-byte Vertex records;
        meshletdata: int32 device tensor; depth: float32 device tensor [height, width], cleared by the caller before the early pass."""
        pass_data = layout.CullData()
        self.lib.nvc_host_pass_data(ctypes.byref(cull_data), 0, 0, ctypes.byref(pass_data))
        proj = (ctypes.c_float * 16)(*[float(v) for v in projection16])
        check(
            self.lib.nvc_raster_depth(self.ctx, self._stream(), proj, ctypes.byref(pass_data), _ptr(self.cib), _ptr(self.ccb), _ptr(self.dcb), _ptr(self.db), _ptr(self.mlb), _ptr(meshletdata), meshletdata.numel(), _ptr(vertices), vertices.numel() // 16, _ptr(depth), depth.shape[1], depth.shape[0], _ptr(stats)),
            self.ctx,
            "nvc_raster_depth",
        )

    def raster_depth_tasks(self, cull_data, projection16, payloads, emit_counts, vertices, meshletdata, depth, stats=None):
        """raster_depth in the task-shading mode (nvc_raster_depth_tasks): draws the clusters that task_shading() put into
        payloads / emit_counts for this path's dcb / dccb."""
        pass_data = layout.CullData()
        self.lib.nvc_host_pass_data(ctypes.byref(cull_data), 0, 0, ctypes.byref(pass_data))
        proj = (ctypes.c_float * 16)(*[float(v) for v in projection16])
        check(
            self.lib.nvc_raster_depth_tasks(self.ctx, self._stream(), proj, ctypes.byref(pass_data), _ptr(payloads), _ptr(emit_counts), _ptr(self.dccb), _ptr(self.dcb), _ptr(self.db), _ptr(self.mlb), _ptr(meshletdata), meshletdata.numel(), _ptr(vertices), vertices.numel() // 16, _ptr(depth), depth.shape[1], depth.shape[0], _ptr(stats)),
            self.ctx,
            "nvc_raster_depth_tasks",
        )

    def raster_depth_indexed(self, cull_data, projection16, vertices, indices, depth, stats=None):
        """raster_depth in the indexed-draw mode (nvc_raster_depth_indexed): draws this path's MeshDrawCommand[] (cull(task=False))
        with max_draw_count = draw_count.  indices: int32 device tensor of the uint32 index buffer."""
        pass_data = layout.CullData()
        self.lib.nvc_host_pass_data(ctypes.byref(cull_data), 0, 0, ctypes.byref(pass_data))
        proj = (ctypes.c_float * 16)(*[float(v) for v in projection16])
        check(
            self.lib.nvc_raster_depth_indexed(self.ctx, self._stream(), proj, ctypes.byref(pass_data), _ptr(self.dcb), _ptr(self.dccb), self.draw_count, _ptr(self.db), _ptr(indices), indices.numel(), _ptr(vertices), vertices.numel() // 16, _ptr(depth), depth.shape[1], depth.shape[0], _ptr(stats)),
            self.ctx,
            "nvc_raster_depth_indexed",
        )

    def frame(self, cull_data, depth, post_passes=False, cluster_backface=None):
        """One frame of the hot path in the reference's order (niagara.cpp:1765-1788).  `depth` stands in for the
        depth target the early render would have produced."""
        self.cull(cull_data, late=False)
        if self.mesh_shading:
            self.render_clusters(cull_data, late=False, cluster_backface=cluster_backface)
        self.pyramid(depth)
        self.cull(cull_data, late=True)
        if self.mesh_shading:
            self.render_clusters(cull_data, late=True, cluster_backface=cluster_backface)
        if post_passes:
            self.cull(cull_data, late=True, post_pass=1)
            if self.mesh_shading:
                self.render_clusters(cull_data, late=True, post_pass=1, cluster_backface=cluster_backface)

    def decode_clusters(self, want_records=True):
        """consumer-side walk of cib/ccb/dcb like meshlet.mesh.glsl:89-105 (nvc_decode_clusters); returns
        (records[slots, 4] uint32 or None, stats[4] = decoded, skipped, invalid, triangles)"""
        torch.cuda.current_stream(self.device).synchronize()
        ccb = self.ccb.cpu().numpy().astype(np.uint32)
        slots = int(ccb[2]) * 256
        records = torch.empty((max(slots, 1), 4), dtype=torch.int32, device=self.device) if want_records else None
        stats = torch.zeros(4, dtype=torch.int32, device=self.device)
        check(self.lib.nvc_decode_clusters(self.ctx, self._stream(), _ptr(self.cib), _ptr(self.ccb), _ptr(self.dcb), _ptr(self.mlb), _ptr(records), _ptr(stats)), self.ctx, "nvc_decode_clusters")
        torch.cuda.current_stream(self.device).synchronize()
        rec = records[:slots].cpu().numpy().astype(np.uint32) if want_records else None
        return rec, stats.cpu().numpy().astype(np.uint32)

    # -- readback helpers (tests / e2e) -----------------------------------------------------------------------
    def read_counts(self):
        return self.dccb.cpu().numpy().astype(np.uint32), self.ccb.cpu().numpy().astype(np.uint32)

    def read_task_commands(self, count):
        n = int(count) * layout.MESHTASKCOMMAND_DTYPE.itemsize
        return self.dcb[:n].cpu().numpy().view(layout.MESHTASKCOMMAND_DTYPE)

    def read_draw_commands(self, count):
        n = int(count) * layout.MESHDRAWCOMMAND_DTYPE.itemsize
        return self.dcb[:n].cpu().numpy().view(layout.MESHDRAWCOMMAND_DTYPE)

    def read_cluster_indices(self, count):
        return self.cib[: int(count)].cpu().numpy().astype(np.uint32)
