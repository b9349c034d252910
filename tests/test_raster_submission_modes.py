"""Depth production in the task-shading and indexed-draw submission modes (nvc_raster_depth_tasks, nvc_raster_depth_indexed).

CPU tier: the product's kernels under the SIMT emulation (tests/cuda_emu) against the reference's own mesh shader (TASK = true) and
vertex shader (mesh.vert) + the sequential test rasteriser (oracle/refshader), bit for bit; the cluster-submit producer on the same
clusters; closed two-phase loops on produced depth against the oracle loop; hostile and edge inputs.
GPU tier (-m gpu): the same loops with the CUDA path against the oracle + reference-shader pipeline, a larger C3-style frame per mode,
and the hostile inputs on the device."""
import ctypes
import os

import numpy as np
import pytest

import emu_lib
import oracle_lib
import refshader_lib
from niagara_b200 import host, scenes
from test_end_to_end_raster import _kitten_scene

needs_refshader = pytest.mark.skipif(not refshader_lib.available(), reason="needs /root/reference or a prebuilt oracle/_ref/librefshader.so")

CAMS = [host.make_camera((0, 0, 0)), host.make_camera((2.5, -1.0, 2.0), host.quat_from_axis_angle((0, 1, 0), 0.2)), host.make_camera((4.0, 0.5, 3.0), host.quat_from_axis_angle((0, 1, 0), 0.25))]
INDEXED = dict(mesh_shading=False, cluster_occlusion=False)


class _EmuPath(emu_lib.EmuPath):
    """EmuPath with the task-shading and indexed-draw depth producers (the product's kernels under the emulation)"""

    def raster_depth_tasks(self, cull_data, projection16, payloads, emit_counts, vertices, meshletdata, depth):
        """nvc_raster_depth_tasks over (payloads, emit_counts) for this path's dcb / dccb; returns stats[4]"""
        pd = self._pass_data(cull_data, 0, 0)
        proj = np.ascontiguousarray(projection16, dtype=np.float32)
        md = np.ascontiguousarray(meshletdata, dtype=np.uint32)
        vb = np.ascontiguousarray(vertices)
        stats = np.zeros(4, np.uint32)
        p = emu_lib._p
        self._check(self.emu.nvc_raster_depth_tasks(self.ctx, None, p(proj), ctypes.byref(pd), p(payloads), p(emit_counts), p(self.dccb), p(self.dcb), p(self.draws), p(self.meshlets), p(md), len(md), p(vb), vb.nbytes // 16, p(depth), depth.shape[1], depth.shape[0], p(stats)), "nvc_raster_depth_tasks")
        return stats

    def raster_depth_indexed(self, cull_data, projection16, vertices, indices, depth):
        """nvc_raster_depth_indexed over this path's dcb / dccb with max_draw_count = the draw count; returns stats[4]"""
        pd = self._pass_data(cull_data, 0, 0)
        proj = np.ascontiguousarray(projection16, dtype=np.float32)
        ib = np.ascontiguousarray(indices, dtype=np.uint32)
        vb = np.ascontiguousarray(vertices)
        stats = np.zeros(4, np.uint32)
        p = emu_lib._p
        self._check(self.emu.nvc_raster_depth_indexed(self.ctx, None, p(proj), ctypes.byref(pd), p(self.dcb), p(self.dccb), len(self.draws), p(self.draws), p(ib), len(ib), p(vb), vb.nbytes // 16, p(depth), depth.shape[1], depth.shape[0], p(stats)), "nvc_raster_depth_indexed")
        return stats


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _cache_geometry(golden_dir):
    from niagara_b200 import scene_cache

    cache = scene_cache.SceneCache(os.path.join(golden_dir, "kitten.z.cache"))
    return cache.section("vertices"), cache.section("indices"), cache.section("meshes")


def _task_buffers(n):
    return np.zeros((max(n, 1), 64), np.uint32), np.zeros(max(n, 1), np.uint32)


def _payload_table(cmds, payloads, counts, n):
    """order-independent view of a task pass: command contents -> sorted lanes it emitted (payload order is unspecified)"""
    out = {}
    for i in range(n):
        if cmds["taskCount"][i]:
            c = min(int(counts[i]), 64)
            out[tuple(cmds[i].tolist())] = tuple(sorted(int(v) >> 24 for v in payloads[i][:c]))
    return out


def _payloads_from_cib(cib, count, commands):
    """task payloads holding the cluster pass's own clusters: each command's cluster indices in ascending lane order"""
    ci = np.asarray(cib[:count], dtype=np.uint32)
    ci = ci[np.lexsort((ci >> 24, ci & 0xFFFFFF))]
    cmd = (ci & 0xFFFFFF).astype(np.int64)
    emit = np.bincount(cmd, minlength=commands).astype(np.uint32)[:commands]
    first = np.cumsum(emit.astype(np.int64)) - emit
    payloads = np.full((max(commands, 1), 64), 0xFFFFFFFF, np.uint32)
    payloads[cmd, np.arange(len(ci)) - first[cmd]] = ci
    counts = np.zeros(max(commands, 1), np.uint32)
    counts[:commands] = emit
    return payloads, counts


# ---- CPU tier: the product's kernels under the emulation ---------------------------------------------------------------------


@needs_refshader
def test_task_mode_matches_the_reference_mesh_shader(golden_dir):
    """nvc_raster_depth_tasks over the emulated path's payloads == meshlet.mesh (TASK = true) + the test rasteriser, early and late pass"""
    screen = (320, 240)
    s, vertices, meshletdata = _kitten_scene(golden_dir, 120, screen)
    o = _EmuPath(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    o.set_visibility_bits(s.visibility_bits)
    drawn_total = 0
    for cam in CAMS[:2]:
        s.camera = cam
        cd = s.cull_data()
        proj = host.projection(cam, *screen)
        ms = refshader_lib.MeshStage(o, vertices, meshletdata, proj)
        want = np.zeros((screen[1], screen[0]), np.float32)
        got = np.zeros_like(want)
        for late in (False, True):
            if late:
                o.pyramid(got)
            o.cull(cd, late)
            n = int(o.dccb[1]) * 64
            payloads, emit = _task_buffers(n)
            o.task_shading(cd, late, payloads, emit)
            rec, pos, tri = ms.run_payloads(cd, payloads[:n], emit[:n])
            ms.rasterize(rec, pos, tri, want)
            stats = o.raster_depth_tasks(cd, proj, payloads, emit, vertices, meshletdata, got)
            assert int(stats[0]) == int(np.minimum(emit[:n], 64).sum()) and int(stats[2]) == 0, stats
            drawn_total += int(stats[0])
            assert np.array_equal(_bits(want), _bits(got)), (late, int((want != got).sum()))
    assert drawn_total > 300 and (want > 0).mean() > 0.05
    o.close()


@needs_refshader
def test_indexed_mode_matches_mesh_vert(golden_dir):
    """nvc_raster_depth_indexed over the emulated path's MeshDrawCommand[] == mesh.vert under vkCmdDrawIndexedIndirectCount + the test
    rasteriser; geometry from the reference-written kitten.z.cache"""
    screen = (320, 240)
    vertices, indices, meshes = _cache_geometry(golden_dir)
    s, _, _ = _kitten_scene(golden_dir, 80, screen)
    assert np.array_equal(s.meshes, meshes)
    o = _EmuPath(meshes, s.meshlets, s.draws, *screen, mesh_shading=False, threads=4)
    lods = set()
    for cam in CAMS[:2]:
        s.camera = cam
        cd = s.cull_data(**INDEXED)
        proj = host.projection(cam, *screen)
        vs = refshader_lib.VertexStage(o, vertices, indices, proj)
        want = np.zeros((screen[1], screen[0]), np.float32)
        got = np.zeros_like(want)
        for late in (False, True):
            if late:
                o.pyramid(got)
            o.cull(cd, late, task=False)
            n = int(o.dccb[0])
            vs.draw(cd, want)
            stats = o.raster_depth_indexed(cd, proj, vertices, indices, got)
            cmds = o.read_draw_commands(n)
            lods.update(cmds["indexCount"].tolist())
            assert int(stats[0]) == n and int(stats[2]) == 0 and int(stats[3]) == 0, stats
            assert np.array_equal(_bits(want), _bits(got)), (late, int((want != got).sum()))
    assert len(lods) >= 2 and (want > 0).mean() > 0.05
    o.close()


def test_task_mode_equals_cluster_submit_on_the_same_clusters(golden_dir):
    """payloads built from the cluster pass's own cib (per command, ascending lane): nvc_raster_depth_tasks gives the image and the
    statistics nvc_raster_depth gives on cib"""
    screen = (320, 240)
    s, vertices, meshletdata = _kitten_scene(golden_dir, 120, screen)
    o = _EmuPath(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    o.set_visibility_bits(s.visibility_bits)
    s.camera = CAMS[1]
    cd = s.cull_data()
    proj = host.projection(s.camera, *screen)
    by_cib = np.zeros((screen[1], screen[0]), np.float32)
    by_tasks = np.zeros_like(by_cib)
    for late in (False, True):
        if late:
            o.pyramid(by_cib)
        o.cull(cd, late)
        o.render_clusters(cd, late)
        payloads, emit = _payloads_from_cib(o.cib, int(o.ccb[0]), int(o.dccb[1]) * 64)
        a = o.raster_depth(cd, proj, vertices, meshletdata, by_cib)
        b = o.raster_depth_tasks(cd, proj, payloads, emit, vertices, meshletdata, by_tasks)
        assert int(a[0]) == int(o.ccb[0]) and np.array_equal(a, b), (late, a, b)
        assert np.array_equal(_bits(by_cib), _bits(by_tasks)), late
    assert (by_cib > 0).mean() > 0.05
    o.close()


def _closed_loop(golden_dir, mode, frames):
    """early cull -> device raster -> pyramid of that depth -> late cull -> device raster over a moving camera, the product's kernels
    (emulated) against the oracle + the reference's shaders; depth images, draw / task passes and visibility state must agree"""
    screen = (256, 192)
    if mode == "tasks":
        s, vertices, meshletdata = _kitten_scene(golden_dir, 100, screen)
        kw = {}
    else:
        vertices, indices, meshes = _cache_geometry(golden_dir)
        s, _, _ = _kitten_scene(golden_dir, 60, screen)
        kw = dict(mesh_shading=False)
    e = _EmuPath(s.meshes, s.meshlets, s.draws, *screen, threads=4, **kw)
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *screen, threads=4, **kw)
    e.set_visibility_bits(s.visibility_bits)
    o.set_visibility_bits(s.visibility_bits)
    late_total = 0
    for f in range(frames):
        s.camera = CAMS[f % len(CAMS)]
        cd = s.cull_data(**(INDEXED if mode == "indexed" else {}))
        proj = host.projection(s.camera, *screen)
        want = np.zeros((screen[1], screen[0]), np.float32)
        got = np.zeros_like(want)
        for late in (False, True):
            if late:
                e.pyramid(got)
                o.pyramid(want)
                assert np.array_equal(e.pyramid_texels.view(np.uint32), o.pyramid_texels.view(np.uint32)), ("pyramid", f)
            e.cull(cd, late)
            o.cull(cd, late)
            assert np.array_equal(e.dccb, o.dccb) and np.array_equal(e.dvb, o.dvb), ("cull", f, late)
            if mode == "tasks":
                n = int(o.dccb[1]) * 64
                cmds = o.read_task_commands(n)
                assert np.array_equal(oracle_lib.sorted_commands(e.read_task_commands(n)), oracle_lib.sorted_commands(cmds)), ("cull", f, late)
                ep, ee = _task_buffers(n)
                op, oe = _task_buffers(n)
                e.task_shading(cd, late, ep, ee)
                o.task_shading(cd, late, op, oe)
                assert _payload_table(e.read_task_commands(n), ep, ee, n) == _payload_table(cmds, op, oe, n) and np.array_equal(e.mvb, o.mvb), ("tasks", f, late)
                ms = refshader_lib.MeshStage(o, vertices, meshletdata, proj, threads=4)
                rec, pos, tri = ms.run_payloads(cd, op[:n], oe[:n])
                ms.rasterize(rec, pos, tri, want)
                stats = e.raster_depth_tasks(cd, proj, ep, ee, vertices, meshletdata, got)
                assert int(stats[0]) == int(oe[:n].sum()) and int(stats[2]) == 0, stats
                late_total += int(oe[:n].sum()) if late else 0
            else:
                n = int(o.dccb[0])
                assert np.array_equal(oracle_lib.sorted_commands(e.read_draw_commands(n)), oracle_lib.sorted_commands(o.read_draw_commands(n))), ("cull", f, late)
                refshader_lib.VertexStage(o, vertices, indices, proj).draw(cd, want)
                stats = e.raster_depth_indexed(cd, proj, vertices, indices, got)
                assert int(stats[0]) == n and int(stats[2]) == 0 and int(stats[3]) == 0, stats
                late_total += n if late else 0
            assert np.array_equal(_bits(want), _bits(got)), ("depth", f, late, int((want != got).sum()))
    assert late_total > 0 and (want > 0).mean() > 0.05
    e.close()


@needs_refshader
@pytest.mark.parametrize("mode", ["tasks", "indexed"])
def test_closed_loop_on_emulated_produced_depth(golden_dir, mode):
    _closed_loop(golden_dir, mode, frames=3)


# ---- hostile and edge inputs, on the emulation and on the device -------------------------------------------------------------


class _EmuCalls:
    """the C ABI of the emulated library on host arrays"""

    def __init__(self):
        self.lib = emu_lib.load()
        self.ctx = ctypes.c_void_p()
        assert self.lib.nvc_create(0, None, ctypes.byref(self.ctx)) == 0

    def __call__(self, name, *args):
        return getattr(self.lib, name)(self.ctx, None, *[a.ctypes.data_as(ctypes.c_void_p) if isinstance(a, np.ndarray) else a for a in args])

    def close(self):
        self.lib.nvc_destroy(self.ctx)


class _CudaCalls:
    """the C ABI of the CUDA library: every numpy argument is copied to the device for the call and copied back after it"""

    def __init__(self):
        import torch
        from niagara_b200.lib import load_library

        assert torch.cuda.is_available()
        self.torch, self.lib = torch, load_library()
        self.ctx = ctypes.c_void_p()
        assert self.lib.nvc_create(0, None, ctypes.byref(self.ctx)) == 0

    def __call__(self, name, *args):
        torch = self.torch
        moved, conv = [], []
        for a in args:
            if isinstance(a, np.ndarray):
                t = torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).cuda()
                moved.append((a, t))
                conv.append(ctypes.c_void_p(t.data_ptr()))
            else:
                conv.append(a)
        status = getattr(self.lib, name)(self.ctx, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream), *conv)
        torch.cuda.synchronize()
        for a, t in moved:
            a.view(np.uint8).reshape(-1)[:] = t.cpu().numpy()
        return status

    def close(self):
        self.lib.nvc_destroy(self.ctx)


def _hostile_cases(golden_dir, call):
    screen = (128, 96)
    s, vertices, meshletdata = _kitten_scene(golden_dir, 40, screen)
    cvert, indices, _ = _cache_geometry(golden_dir)
    cd = s.cull_data(culling=False, occlusion=False, cluster_occlusion=False)
    proj = (ctypes.c_float * 16)(*[float(v) for v in host.projection(s.camera, *screen)])
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    o.dvb[:] = 1
    o.cull(cd, False)
    pd = o._pass_data(cd, 0, 0)
    dccb = o.dccb.copy()
    ncmd = int(dccb[1]) * 64
    tcmds = o.read_task_commands(ncmd)
    dcb = o.dcb[: max(ncmd * 20, 20)].copy()
    draws, md = np.ascontiguousarray(s.draws), np.ascontiguousarray(meshletdata, dtype=np.uint32)
    vb = np.ascontiguousarray(vertices)

    # every lane of every command in its payload, padded with ~0 (which draws nothing)
    lane = np.arange(64, dtype=np.uint32)
    live = lane[None, :] < tcmds["taskCount"][:, None]
    payloads = np.where(live, np.arange(ncmd, dtype=np.uint32)[:, None] | (lane[None, :] << 24), 0xFFFFFFFF).astype(np.uint32)

    def tasks(emit, meshlets=s.meshlets, payloads=payloads, width=screen[0]):
        depth, stats = np.zeros((screen[1], screen[0]), np.float32), np.zeros(4, np.uint32)
        st = call("nvc_raster_depth_tasks", proj, ctypes.byref(pd), payloads, np.ascontiguousarray(emit, dtype=np.uint32), dccb, dcb, draws, np.ascontiguousarray(meshlets), md, len(md), vb, vb.nbytes // 16, depth, width, screen[1], stats)
        return st, stats, depth

    emit = tcmds["taskCount"].astype(np.uint32)
    st, base, img = tasks(emit)
    assert st == 0 and int(base[0]) == int(emit.sum()) > 50 and int(base[2]) == 0 and (img > 0).mean() > 0.01
    # emit counts past 64 are clamped: the padded lanes (~0) draw nothing either way
    for big in (np.full_like(emit, 64), np.full_like(emit, 1000), np.full_like(emit, 0xFFFFFFFF)):
        st, stats, d = tasks(big)
        assert st == 0 and np.array_equal(stats, base) and np.array_equal(_bits(d), _bits(img))
    # meshlet data out of range: every cluster rejected and counted, nothing written
    bad = s.meshlets.copy()
    bad["dataOffset"][:] = 0x7FFFFFF0
    st, stats, d = tasks(emit, meshlets=bad)
    assert st == 0 and int(stats[0]) == 0 and int(stats[2]) == int(base[0]) and not d.any()
    # NULL / zero-size arguments
    assert tasks(emit, payloads=None)[0] == -1 and tasks(emit, width=0)[0] == -1

    # ---- indexed draws: every draw at its LOD
    oi = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *screen, mesh_shading=False, threads=4)
    oi.dvb[:] = 1
    oi.cull(s.cull_data(culling=False, occlusion=False, **INDEXED), False, task=False)
    n = int(oi.dccb[0])
    assert n == len(s.draws)
    cmds = oi.read_draw_commands(n)
    cv, ib = np.ascontiguousarray(cvert), np.ascontiguousarray(indices, dtype=np.uint32)

    def indexed(cmds=cmds, count=n, max_draw_count=n, ib=ib, idx_arg=True, height=screen[1]):
        depth, stats = np.zeros((screen[1], screen[0]), np.float32), np.zeros(4, np.uint32)
        c4 = np.array([count, 0, 0, 0], np.uint32)
        st = call("nvc_raster_depth_indexed", proj, ctypes.byref(pd), np.ascontiguousarray(cmds), c4, max_draw_count, draws, ib if idx_arg else None, len(ib), cv, cv.nbytes // 16, depth, screen[0], height, stats)
        return st, stats, depth

    def changed(**fields):
        c = cmds.copy()
        for f, v in fields.items():
            c[f][k] = v
        return c

    st, base, img = indexed()
    assert st == 0 and int(base[0]) == n and int(base[2]) == 0 and int(base[3]) == 0 and (img > 0).mean() > 0.01
    for k in range(n):  # a command that owns pixels; without_k = the image of every other command
        _, _, without_k = indexed(changed(instanceCount=0))
        if not np.array_equal(_bits(without_k), _bits(img)):
            break
    assert k < n - 1
    # instanceCount 0 draws nothing; 3 instances give the image and the counts of one
    none = cmds.copy()
    none["instanceCount"] = 0
    st, stats, d = indexed(none)
    assert st == 0 and not stats.any() and not d.any()
    three = cmds.copy()
    three["instanceCount"] = 3
    st, stats, d = indexed(three)
    assert st == 0 and np.array_equal(stats, base) and np.array_equal(_bits(d), _bits(img))
    # an index range past index_count: the command is rejected whole
    c0 = cmds[k]
    st, stats, d = indexed(changed(firstIndex=len(ib) - int(c0["indexCount"]) + 3))
    assert st == 0 and int(stats[0]) == n - 1 and int(stats[2]) == 1 and np.array_equal(_bits(d), _bits(without_k))
    st, stats, d = indexed(changed(firstIndex=0xFFFFFFF0))
    assert st == 0 and int(stats[2]) == 1 and np.array_equal(_bits(d), _bits(without_k))
    # vertex indices past vertex_count: those triangles are rejected and counted
    st, stats, d = indexed(changed(vertexOffset=cv.nbytes // 16))
    assert st == 0 and int(stats[0]) == n and int(stats[3]) == int(c0["indexCount"]) // 3 and np.array_equal(_bits(d), _bits(without_k))
    # vertexOffset wraps in uint32: indices + 7 with vertexOffset - 7 is the same geometry
    shifted = cmds.copy()
    shifted["vertexOffset"] = (shifted["vertexOffset"].astype(np.int64) - 7) & 0xFFFFFFFF
    st, stats, d = indexed(shifted, ib=ib + np.uint32(7))
    assert st == 0 and np.array_equal(stats, base) and np.array_equal(_bits(d), _bits(img))
    # trailing indices that make no whole triangle are not drawn
    fits = [i for i in range(n) if int(cmds["firstIndex"][i]) + int(cmds["indexCount"][i]) + 2 <= len(ib)]
    longer = cmds.copy()
    longer["indexCount"][fits] += 2
    st, stats, d = indexed(longer)
    assert fits and st == 0 and np.array_equal(stats, base) and np.array_equal(_bits(d), _bits(img))
    # command_count4[0] > max_draw_count: clamped
    st, stats, d = indexed(count=10**6)
    assert st == 0 and np.array_equal(stats, base) and np.array_equal(_bits(d), _bits(img))
    st, stats, d = indexed(max_draw_count=1)
    assert st == 0 and int(stats[0]) == 1
    # NULL / zero-size arguments
    assert indexed(idx_arg=False)[0] == -1 and indexed(height=0)[0] == -1


def test_hostile_and_edge_inputs(golden_dir):
    call = _EmuCalls()
    _hostile_cases(golden_dir, call)
    call.close()


# ---- GPU tier --------------------------------------------------------------------------------------------------------------------


def _device_loop(golden_dir, mode):
    """test_two_phase_on_device_produced_depth for the task-shading and indexed-draw modes"""
    import torch
    from test_gpu_parity import _compare_draw_pass, _compare_pyramid, _paths

    screen = (512, 384)
    if mode == "tasks":
        s, vertices, meshletdata = _kitten_scene(golden_dir, 300, screen)
        g, o, _ = _paths(s)
        md = torch.from_numpy(np.ascontiguousarray(meshletdata, dtype=np.uint32).view(np.int32)).cuda()
    else:
        vertices, indices, _ = _cache_geometry(golden_dir)
        s, _, _ = _kitten_scene(golden_dir, 160, screen)
        g, o, _ = _paths(s, mesh_shading=False)
        ib = torch.from_numpy(np.ascontiguousarray(indices, dtype=np.uint32).view(np.int32)).cuda()
    vb = torch.from_numpy(np.ascontiguousarray(vertices)).cuda()
    stats = torch.zeros(4, dtype=torch.int32, device="cuda")
    cams = [host.make_camera((0, 0, 0)), host.make_camera((0, 0, 0)), host.make_camera((3.5, -1.0, 2.0), host.quat_from_axis_angle((0, 1, 0), 0.18)),
            host.make_camera((7.0, 1.5, 5.0), host.quat_from_axis_angle((0.1, 1, 0), 0.42))]
    late_total, lods = 0, set()
    for f, cam in enumerate(cams):
        s.camera = cam
        cd = s.cull_data(**(INDEXED if mode == "indexed" else {}))
        proj = host.projection(cam, *screen)
        want = np.zeros((screen[1], screen[0]), np.float32)
        got = torch.zeros((screen[1], screen[0]), dtype=torch.float32, device="cuda")
        for late in (False, True):
            if late:
                g.pyramid(got)
                o.pyramid(want)
                _compare_pyramid(g, o, ("pyramid of produced depth", f))
            g.cull(cd, late)
            o.cull(cd, late)
            _compare_draw_pass(g, o, mode == "tasks", ("cull", f, late))
            if mode == "tasks":
                n = int(o.dccb[1]) * 64
                gp = torch.zeros((max(n, 1), 64), dtype=torch.int32, device="cuda")
                ge = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
                op, oe = _task_buffers(n)
                g.task_shading(cd, late, gp, ge)
                o.task_shading(cd, late, op, oe)
                torch.cuda.synchronize()
                gpn, gen = gp.cpu().numpy().astype(np.uint32), ge.cpu().numpy().astype(np.uint32)
                assert _payload_table(g.read_task_commands(n), gpn, gen, n) == _payload_table(o.read_task_commands(n), op, oe, n), ("tasks", f, late)
                assert np.array_equal(g.mvb.cpu().numpy().astype(np.uint32), o.mvb), ("mvb", f, late)
                ms = refshader_lib.MeshStage(o, vertices, meshletdata, proj)
                rec, pos, tri = ms.run_payloads(cd, op[:n], oe[:n])
                ms.rasterize(rec, pos, tri, want)
                g.raster_depth_tasks(cd, proj, gp, ge, vb, md, got, stats)
                torch.cuda.synchronize()
                st = stats.cpu().numpy()
                assert int(st[0]) == int(oe[:n].sum()) and int(st[2]) == 0, (f, late, st)
                late_total += int(oe[:n].sum()) if late else 0
            else:
                n = int(o.dccb[0])
                lods.update(o.read_draw_commands(n)["indexCount"].tolist())
                refshader_lib.VertexStage(o, vertices, indices, proj).draw(cd, want)
                g.raster_depth_indexed(cd, proj, vb, ib, got, stats)
                torch.cuda.synchronize()
                st = stats.cpu().numpy()
                assert int(st[0]) == n and int(st[2]) == 0 and int(st[3]) == 0, (f, late, st)
                late_total += n if late else 0
            assert np.array_equal(got.cpu().numpy().view(np.uint32), want.view(np.uint32)), ("depth image", f, late)
    assert late_total > 0 and (want > 0).mean() > 0.2
    assert mode == "tasks" or len(lods) >= 2


@pytest.mark.gpu
@needs_refshader
def test_task_shading_loop_on_device_produced_depth(golden_dir):
    _device_loop(golden_dir, "tasks")


@pytest.mark.gpu
@needs_refshader
def test_indexed_draw_loop_on_device_produced_depth(golden_dir):
    _device_loop(golden_dir, "indexed")


@pytest.mark.gpu
@needs_refshader
@pytest.mark.parametrize("mode", ["tasks", "indexed"])
def test_c3_style_frame_per_mode(golden_dir, mode):
    """~2 000 C3-style draws at 1024^2, two-phase frames on produced depth in each mode: the device's depth equals the CPU
    reference-shader pipeline's bit for bit, and running the last frame again from the same visibility state gives the same bits"""
    import torch
    from niagara_b200.path import VisibilityPath

    screen = (1024, 1024)
    s = scenes.config3_scene(golden_dir, draw_count=2000, screen=screen)
    tasks = mode == "tasks"
    if tasks:
        vertices, meshletdata = s.vertices, s.meshletdata
        md = torch.from_numpy(meshletdata.view(np.int32)).cuda()
    else:
        vertices, indices, _ = _cache_geometry(golden_dir)
        ib = torch.from_numpy(np.ascontiguousarray(indices, dtype=np.uint32).view(np.int32)).cuda()
    g = VisibilityPath(s.meshes, s.meshlets, s.draws, *screen, mesh_shading=tasks)
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *screen, mesh_shading=tasks, threads=os.cpu_count() or 8)
    g.set_visibility_bits(s.visibility_bits)
    o.set_visibility_bits(s.visibility_bits)
    vb = torch.from_numpy(np.ascontiguousarray(vertices)).cuda()
    cd = s.cull_data(**({} if tasks else INDEXED))
    proj = host.projection(s.camera, *screen)
    stats = torch.zeros(4, dtype=torch.int32, device="cuda")

    def device_frame():
        got = torch.zeros((screen[1], screen[0]), dtype=torch.float32, device="cuda")
        drawn = []
        for late in (False, True):
            if late:
                g.pyramid(got)
            g.cull(cd, late)
            if tasks:
                n = int(g.dccb[1].item()) * 64
                gp = torch.zeros((max(n, 1), 64), dtype=torch.int32, device="cuda")
                ge = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
                g.task_shading(cd, late, gp, ge)
                g.raster_depth_tasks(cd, proj, gp, ge, vb, md, got, stats)
            else:
                g.raster_depth_indexed(cd, proj, vb, ib, got, stats)
            torch.cuda.synchronize()
            st = stats.cpu().numpy()
            assert int(st[2]) == 0 and (tasks or int(st[3]) == 0), st
            drawn.append(int(st[0]))
        return got.cpu().numpy(), drawn

    def cpu_frame():
        want = np.zeros((screen[1], screen[0]), np.float32)
        for late in (False, True):
            if late:
                o.pyramid(want)
            o.cull(cd, late)
            if tasks:
                n = int(o.dccb[1]) * 64
                op, oe = _task_buffers(n)
                o.task_shading(cd, late, op, oe)
                ms = refshader_lib.MeshStage(o, vertices, meshletdata, proj, threads=os.cpu_count() or 8)
                rec, pos, tri = ms.run_payloads(cd, op[:n], oe[:n])
                ms.rasterize(rec, pos, tri, want)
            else:
                refshader_lib.VertexStage(o, vertices, indices, proj).draw(cd, want)
        return want

    # frame 0 draws everything in the late pass (nothing was visible before), frame 1 mostly in the early pass
    for f in range(2):
        if f == 1:
            dvb, mvb = g.dvb.clone(), g.mvb.clone()
        got, drawn = device_frame()
        want = cpu_frame()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (f, int((got != want).sum()))
        assert drawn[1 - f] > 500 and (want > 0).mean() > 0.05, (f, drawn)
    g.dvb.copy_(dvb)
    g.mvb.copy_(mvb)
    again, drawn_again = device_frame()
    assert drawn_again == drawn and np.array_equal(again.view(np.uint32), got.view(np.uint32))


@pytest.mark.gpu
def test_hostile_and_edge_inputs_on_device(golden_dir):
    """the kernels bounds-check: these inputs exercise the counting, they never fault"""
    call = _CudaCalls()
    _hostile_cases(golden_dir, call)
    call.close()
