"""The mesh shader's per-triangle cull stage (meshlet.mesh.glsl with MESH_CULL = 1) in the cluster-submit and task-shading depth
producers (nvc_set_mesh_cull, nvc_mesh_cull_stats).

The oracle is the reference's own shader with its own switch flipped: oracle/refshader_cull generates meshlet_mesh_cull from
meshlet.mesh.glsl with `#define CULL 1` (oracle/_ref/librefshader_cull.so), and its rs_rasterize_culled leaves out the primitives
the shader flags gl_CullPrimitiveEXT.
CPU tier: the product's kernels under the SIMT emulation (tests/cuda_emu) against that shader + the test rasteriser, bit for bit:
whole frames in both modes, single decisions on constructed triangles, closed two-phase loops against the brute-force image, the
switch turned off again, and hostile meshlet data in guarded memory.
GPU tier (-m gpu): the same loops and a 2 000-draw frame per mode on the device."""
import ctypes
import os

import numpy as np
import pytest

import emu_lib
import oracle_lib
import refshader_lib
from niagara_b200 import host, layout, scenes
from test_end_to_end_raster import _all_clusters, _kitten_scene
from test_kernels_emulated import _guarded
from test_raster_submission_modes import _EmuPath as _ModesEmuPath
from test_raster_submission_modes import _bits, _cache_geometry, _payloads_from_cib, _task_buffers

CAMS = [host.make_camera((0, 0, 0)), host.make_camera((1.0, -0.5, -2.0), host.quat_from_axis_angle((0, 1, 0), 0.15))]  # the second one is close to the nearest kittens
MOVING = [host.make_camera((0, 0, 0)), host.make_camera((0.5, 0, -1.0)), host.make_camera((2.5, -1.0, 2.0), host.quat_from_axis_angle((0, 1, 0), 0.2)),
          host.make_camera((1.0, -0.5, -2.0), host.quat_from_axis_angle((0, 1, 0), 0.15)), host.make_camera((4.0, 0.5, 3.0), host.quat_from_axis_angle((0, 1, 0), 0.25))]
INDEXED = dict(mesh_shading=False, cluster_occlusion=False)

vp, sz, f32, u32, i32 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_float, ctypes.c_uint32, ctypes.c_int

CULL_SO = os.path.join(refshader_lib.ROOT, "oracle", "_ref", "librefshader_cull.so")
_CULL_LIB = []


def _available():
    return os.path.exists(CULL_SO) or os.path.isdir(os.path.join(refshader_lib.REFERENCE, "src", "shaders"))


needs_refshader = pytest.mark.skipif(not (refshader_lib.available() and _available()), reason="needs /root/reference or prebuilt oracle/_ref/librefshader.so and librefshader_cull.so")


def _rs():
    """oracle/_ref/librefshader_cull.so (oracle/refshader_cull: the reference-shader library plus meshlet.mesh.glsl with MESH_CULL = 1)
    with the argument types of its MESH_CULL entry points; built from the reference where that exists, as refshader_lib.load() does"""
    if _CULL_LIB:
        return _CULL_LIB[0]
    if os.path.isdir(os.path.join(refshader_lib.REFERENCE, "src", "shaders")):
        import subprocess

        subprocess.run(["make", "-s", "-C", os.path.join(refshader_lib.ROOT, "oracle", "refshader_cull"), "REF=" + refshader_lib.REFERENCE], check=True)
    rs = ctypes.CDLL(CULL_SO)
    cd = ctypes.POINTER(layout.CullData)
    rs.rs_mesh_clusters_cull.restype = i32
    rs.rs_mesh_clusters_cull.argtypes = [vp, cd, f32, f32, vp, sz, vp, sz, vp, sz, vp, sz, vp, sz, vp, sz, vp, vp, vp, vp, vp, i32]
    rs.rs_mesh_payloads_cull.restype = i32
    rs.rs_mesh_payloads_cull.argtypes = [vp, cd, f32, f32, vp, sz, u32, vp, sz, vp, sz, vp, sz, vp, sz, vp, vp, vp, vp, vp, vp, vp, i32]
    rs.rs_rasterize_culled.restype = i32
    rs.rs_rasterize_culled.argtypes = [vp, vp, vp, vp, u32, u32, u32, vp, vp, i32]
    _CULL_LIB.append(rs)
    return rs


_p, _n = refshader_lib._p, refshader_lib._n


class _EmuPath(_ModesEmuPath):
    """the emulated path with the mesh-cull switch and counters"""

    def set_mesh_cull(self, enabled):
        self._check(self.emu.nvc_set_mesh_cull(self.ctx, int(enabled)), "nvc_set_mesh_cull")

    def mesh_cull_stats(self, reset=True):
        out = (ctypes.c_uint64 * 2)()
        self._check(self.emu.nvc_mesh_cull_stats(self.ctx, out, int(reset)), "nvc_mesh_cull_stats")
        return int(out[0]), int(out[1])


class _CullStage(refshader_lib.MeshStage):
    """meshlet.mesh.glsl with CULL = 1 (meshlet_mesh_cull) + the test rasteriser that skips gl_CullPrimitiveEXT primitives"""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.rc = _rs()

    def run_cull(self, cull_data, cib=None, ccb=None, dcb=None):
        """as MeshStage.run, plus culled[slots, 96] (1 = gl_CullPrimitiveEXT)"""
        p = self.p
        cib = p.cib if cib is None else np.ascontiguousarray(cib, dtype=np.uint32)
        ccb = p.ccb if ccb is None else np.ascontiguousarray(ccb, dtype=np.uint32)
        dcb = p.dcb if dcb is None else dcb
        slots = int(ccb[1]) * int(ccb[2]) * int(ccb[3])
        rec, pos = np.zeros((max(slots, 1), 4), np.uint32), np.zeros((max(slots, 1), 64, 4), np.float32)
        tri, culled = np.zeros((max(slots, 1), 96, 3), np.uint8), np.zeros((max(slots, 1), 96), np.uint8)
        pd = p._pass_data(cull_data, 0, 0)
        s = self.rc.rs_mesh_clusters_cull(_p(self.projection), ctypes.byref(pd), float(p.depth_width), float(p.depth_height), _p(dcb), _n(dcb), _p(p.draws), _n(p.draws), _p(p.meshlets), _n(p.meshlets),
                                          _p(self.meshletdata), _n(self.meshletdata), _p(self.vertices), _n(self.vertices), _p(cib), _n(cib), _p(ccb), _p(rec), _p(pos), _p(tri), _p(culled), self.threads)
        assert s == 0, s
        return rec[:slots], pos[:slots], tri[:slots], culled[:slots]

    def run_payloads_cull(self, cull_data, payloads, emit_counts, dcb=None):
        """as MeshStage.run_payloads, plus culled[slots, 96]"""
        p = self.p
        dcb = p.dcb if dcb is None else dcb
        emit = np.minimum(np.ascontiguousarray(emit_counts, dtype=np.uint32), 64)
        first = (np.cumsum(emit) - emit).astype(np.uint32)
        slots = int(emit.sum())
        rec, pos = np.zeros((max(slots, 1), 4), np.uint32), np.zeros((max(slots, 1), 64, 4), np.float32)
        tri, culled = np.zeros((max(slots, 1), 96, 3), np.uint8), np.zeros((max(slots, 1), 96), np.uint8)
        payloads = np.ascontiguousarray(payloads, dtype=np.uint32)
        pd = p._pass_data(cull_data, 0, 0)
        s = self.rc.rs_mesh_payloads_cull(_p(self.projection), ctypes.byref(pd), float(p.depth_width), float(p.depth_height), _p(dcb), _n(dcb), len(emit), _p(p.draws), _n(p.draws), _p(p.meshlets), _n(p.meshlets),
                                          _p(self.meshletdata), _n(self.meshletdata), _p(self.vertices), _n(self.vertices), _p(payloads), _p(emit), _p(first), _p(rec), _p(pos), _p(tri), _p(culled), self.threads)
        assert s == 0, s
        return rec[:slots], pos[:slots], tri[:slots], culled[:slots]

    def rasterize_culled(self, rec, pos, tri, culled, depth):
        s = self.rc.rs_rasterize_culled(_p(pos), _p(tri), _p(rec), _p(np.ascontiguousarray(culled, dtype=np.uint8)), len(rec), depth.shape[1], depth.shape[0], _p(depth), None, 0)
        assert s == 0, s

    def owners_culled(self, rec, pos, tri, culled, depth):
        hit = np.zeros(max(len(rec), 1), np.uint8)
        s = self.rc.rs_rasterize_culled(_p(pos), _p(tri), _p(rec), _p(np.ascontiguousarray(culled, dtype=np.uint8)), len(rec), depth.shape[1], depth.shape[0], _p(depth), _p(hit), 1)
        assert s == 0, s
        return hit[: len(rec)].astype(bool)


def _flagged(rec, culled):
    """primitives the shader flagged (the driver writes 0 past each slot's triangleCount)"""
    assert not any(culled[i, int(rec[i, 1]):].any() for i in range(len(rec)))
    return int(culled.sum())


def _sensitive(cs, rec, pos, tri, culled, with_cull, without_cull):
    """the MESH_CULL = 1 image differs from the MESH_CULL = 0 one, or no flagged primitive covers a sample at all"""
    if not np.array_equal(_bits(with_cull), _bits(without_cull)):
        return True
    only_flagged = np.zeros_like(with_cull)
    cs.rasterize_culled(rec, pos, tri, 1 - culled, only_flagged)
    return not only_flagged.any()


# ---- CPU tier: whole frames ------------------------------------------------------------------------------------------------------


@needs_refshader
@pytest.mark.parametrize("mode", ["clusters", "tasks"])
def test_frames_match_the_reference_mesh_shader_with_mesh_cull(golden_dir, mode):
    """nvc_raster_depth / nvc_raster_depth_tasks with the stage on == meshlet.mesh.glsl (CULL = 1) + the test rasteriser skipping flagged
    primitives, early and late pass, two cameras; the device's culled count == the shader's flags"""
    screen = (320, 240)
    s, vertices, meshletdata = _kitten_scene(golden_dir, 120, screen)
    o = _EmuPath(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    o.set_visibility_bits(s.visibility_bits)
    o.set_mesh_cull(1)
    flagged_total, sensitive = 0, False
    for cam in CAMS:
        s.camera = cam
        cd = s.cull_data()
        proj = host.projection(cam, *screen)
        cs = _CullStage(o, vertices, meshletdata, proj, threads=4)
        want, got, plain = (np.zeros((screen[1], screen[0]), np.float32) for _ in range(3))
        for late in (False, True):
            if late:
                o.pyramid(got)
            o.cull(cd, late)
            if mode == "clusters":
                o.render_clusters(cd, late)
                rec, pos, tri, culled = cs.run_cull(cd)
                stats = o.raster_depth(cd, proj, vertices, meshletdata, got)
                assert int(stats[0]) == int(o.ccb[0]), stats
            else:
                n = int(o.dccb[1]) * 64
                payloads, emit = _task_buffers(n)
                o.task_shading(cd, late, payloads, emit)
                rec, pos, tri, culled = cs.run_payloads_cull(cd, payloads[:n], emit[:n])
                stats = o.raster_depth_tasks(cd, proj, payloads, emit, vertices, meshletdata, got)
                assert int(stats[0]) == len(rec), stats
            cs.rasterize_culled(rec, pos, tri, culled, want)
            cs.rasterize(rec, pos, tri, plain)
            tested, culled_n = o.mesh_cull_stats(reset=True)
            assert int(stats[2]) == 0 and tested == int(rec[:, 1].sum()) and culled_n == _flagged(rec, culled), (late, stats, tested, culled_n, _flagged(rec, culled))
            flagged_total += culled_n
            assert np.array_equal(_bits(want), _bits(got)), (cam, late, int((want != got).sum()))
        sensitive = sensitive or _sensitive(cs, rec, pos, tri, culled, want, plain)
        assert (want > 0).mean() > 0.05
    assert flagged_total > 0 and sensitive
    o.close()


# ---- CPU tier: single decisions --------------------------------------------------------------------------------------------------

W = H = 64  # the depth target of the single-decision launches (= the shader's screenWidth / screenHeight)


def _screen(px, py, w=1.0, z=0.5):
    """clip corner whose screen position (x / w * 0.5 + 0.5) * 64 is (px, py) for w = 1 (exact for the values used below)"""
    return (np.float32((px / W - 0.5) * 2 * w), np.float32((py / H - 0.5) * 2 * w), np.float32(z), np.float32(w))


def _p32(v, wv):
    """the float screen coordinate of one clip component (what the kernel and the shader compute)"""
    f = np.float32
    return f(f(f(f(v) / f(wv)) * f(0.5)) + f(0.5)) * f(W)


def _up(v, k=1):
    v = np.float32(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, np.float32(np.inf if k > 0 else -np.inf), dtype=np.float32)
    return float(v)


S = 1.0 / 256.0
NAN, INF = float("nan"), float("inf")


def _decision_cases():
    c = {}
    c["front"] = [_screen(10, 10), _screen(50, 10), _screen(10, 50)]
    c["back"] = [_screen(10, 10), _screen(10, 50), _screen(50, 10)]
    c["zero area"] = [_screen(20, 20), _screen(20, 20), _screen(40, 30)]
    c["collinear"] = [_screen(10, 10), _screen(20, 20), _screen(30, 30)]
    # eb.x * ec.y == eb.y * ec.x only after rounding: (1 + 2^-12)^2 rounds to 1 + 2^-11 (exactly: front facing)
    c["equal after rounding"] = [_screen(32, 32), _screen(33 + 2**-12, 33 + 2**-11), _screen(33, 33 + 2**-12)]
    # small-primitive test: bmin.x - 1/256 on x.5 and 1 ulp either side; bmax.y + 1/256 on x.5 and 1 ulp either side
    for k in (-1, 0, 1):
        bx = _up(40.5 + S, k)
        c["bmin.x - 1/256 = 40.5 %+d ulp" % k] = [_screen(bx, 10), _screen(40.9, 10), _screen(bx, 50)]
        by = _up(40.5 - S, k)
        c["bmax.y + 1/256 = 40.5 %+d ulp" % k] = [_screen(10, 39.7), _screen(50, 39.7), _screen(10, by)]
    # halfway cases that half-to-even (2.5 -> 2) and floor(x + 0.5) (-0.5 -> 0) decide differently from half away from zero
    c["bmin.x - 1/256 = 2.5"] = [_screen(2.5 + S, 10), _screen(2.9, 10), _screen(2.5 + S, 50)]
    c["bmin.x - 1/256 = -0.5"] = [_screen(-0.5 + S, 10), _screen(-0.7, 10), _screen(-0.5 + S, 50)]
    small = [_screen(30.1, 30.1), _screen(30.4, 30.1), _screen(30.1, 30.4)]  # inside one pixel: culled as long as every w > 0
    c["small"] = small
    c["small, w = 0"] = small[:2] + [(np.float32(0), np.float32(0), np.float32(0.5), np.float32(0))]
    c["small, w < 0"] = small[:2] + [(np.float32(-0.01), np.float32(-0.01), np.float32(0.5), np.float32(-1))]
    c["small, w = -0"] = small[:2] + [(np.float32(0), np.float32(0), np.float32(0.5), np.float32(-0.0))]
    c["back, w < 0"] = [_screen(10, 10), _screen(10, 50), (np.float32(-0.5), np.float32(-0.9), np.float32(0.5), np.float32(-1))]
    c["small, x NaN"] = small[:2] + [(np.float32(NAN), small[2][1], small[2][2], small[2][3])]
    c["small, y NaN"] = small[:2] + [(small[2][0], np.float32(NAN), small[2][2], small[2][3])]
    c["small, w NaN"] = small[:2] + [(small[2][0], small[2][1], small[2][2], np.float32(NAN))]
    c["front, x NaN"] = [_screen(10, 10), _screen(50, 10), (np.float32(NAN), np.float32(0.5), np.float32(0.5), np.float32(1))]
    c["small, x inf"] = small[:2] + [(np.float32(INF), small[2][1], small[2][2], small[2][3])]
    c["small, x -inf"] = small[:2] + [(np.float32(-INF), small[2][1], small[2][2], small[2][3])]
    c["small, x / w overflows"] = small[:2] + [(np.float32(3e38), small[2][1], small[2][2], np.float32(1e-5))]
    c["thin, y / w overflows"] = [_screen(10, 10), _screen(50, 10), (np.float32(-0.5), np.float32(3e38), np.float32(0.5), np.float32(1e-5))]
    c["far right, small"] = [_screen(1e7, 30), _screen(1e7 + 0.25, 30), _screen(1e7, 30.25)]
    c["far left, large"] = [_screen(-1e7, -1e7), _screen(-1e7 + 5e6, -1e7), _screen(-1e7, -1e7 + 5e6)]
    c["far both sides"] = [_screen(-1e9, 30), _screen(1e9, 30), _screen(0, 1e9)]
    c["far both sides, back"] = [_screen(-1e9, 30), _screen(0, 1e9), _screen(1e9, 30)]
    c["huge, products overflow"] = [(np.float32(-3e37), np.float32(-3e37), np.float32(0.5), np.float32(1)), (np.float32(3e37), np.float32(-3e37), np.float32(0.5), np.float32(1)),
                                     (np.float32(-3e37), np.float32(3e37), np.float32(0.5), np.float32(1))]
    return c


def _single_triangle_scene(corners):
    """One meshlet of three vertices (1,0,0), (0,1,0), (0,0,1) and one triangle, one draw at the origin, view = identity; the
    projection's columns 0-2 are the three clip corners, column 3 is 0, so corner k's clip position is exactly corners[k]."""
    vertices = np.zeros((3, 8), np.uint16)
    vertices[0, 0] = vertices[1, 1] = vertices[2, 2] = 0x3C00  # binary16 1.0
    meshletdata = np.array([0, 1, 2, 0 | (1 << 8) | (2 << 16)], np.uint32)
    meshlets = np.zeros(1, layout.MESHLET_DTYPE)
    meshlets["vertexCount"], meshlets["triangleCount"] = 3, 1
    draws = np.zeros(1, layout.MESHDRAW_DTYPE)
    draws["scale"], draws["orientation"] = 1.0, (0, 0, 0, 1)
    commands = np.zeros(1, layout.MESHTASKCOMMAND_DTYPE)
    commands["taskCount"] = 1
    proj = np.zeros(16, np.float32)
    for k in range(3):
        proj[4 * k: 4 * k + 4] = corners[k]
    cib = np.full(256, 0xFFFFFFFF, np.uint32)
    cib[0] = 0
    return vertices.view(np.uint8).reshape(-1), meshletdata, meshlets, draws, commands, proj, cib, np.array([1, 1, 1, 1], np.uint32)


@needs_refshader
def test_single_decisions_match_the_shader():
    """one triangle per cluster, one launch each: the device's decision (nvc_mesh_cull_stats) == the shader's gl_CullPrimitiveEXT, for
    halfway rounding, facing at the rounding limit, w <= 0, NaN / inf corners and far off-screen coordinates"""
    rs = _rs()
    lib = emu_lib.load()
    ctx = ctypes.c_void_p()
    assert lib.nvc_create(0, None, ctypes.byref(ctx)) == 0
    assert lib.nvc_set_mesh_cull(ctx, 1) == 0
    pd = layout.CullData()
    for i in range(16):
        pd.view[i] = 1.0 if i % 5 == 0 else 0.0
    decisions = {}
    for name, corners in _decision_cases().items():
        vb, md, meshlets, draws, commands, proj, cib, ccb = _single_triangle_scene(corners)
        rec, pos = np.zeros((1, 4), np.uint32), np.zeros((1, 64, 4), np.float32)
        tri, flags = np.zeros((1, 96, 3), np.uint8), np.zeros((1, 96), np.uint8)
        s = rs.rs_mesh_clusters_cull(_p(proj), ctypes.byref(pd), float(W), float(H), _p(commands), _n(commands), _p(draws), _n(draws), _p(meshlets), _n(meshlets), _p(md), _n(md), _p(vb), _n(vb),
                                     _p(cib), _n(cib), _p(ccb), _p(rec), _p(pos), _p(tri), _p(flags), 1)
        assert s == 0 and rec[0, 1] == 1
        got_clip = pos[0, :3].astype(np.float32)
        want_clip = np.array(corners, np.float32)
        # (-0 arrives as +0; a NaN or inf entry of the projection reaches the other corners as NaN through 0 * NaN: those are NaN cases)
        assert not np.isfinite(want_clip).all() or np.array_equal(got_clip, want_clip), name
        depth, stats, out = np.zeros((H, W), np.float32), np.zeros(4, np.uint32), (ctypes.c_uint64 * 2)()
        assert lib.nvc_raster_depth(ctx, None, _p(proj), ctypes.byref(pd), _p(cib), _p(ccb), _p(commands), _p(draws), _p(meshlets), _p(md), len(md), _p(vb), 3, _p(depth), W, H, _p(stats)) == 0
        assert lib.nvc_mesh_cull_stats(ctx, out, 1) == 0
        assert int(out[0]) == 1 and int(stats[0]) == 1, (name, list(out), stats)
        assert int(out[1]) == int(flags[0, 0]), (name, int(out[1]), int(flags[0, 0]), corners)
        # a culled triangle is not sampled; one that is not culled goes through the sampler unchanged
        want = np.zeros_like(depth)
        assert rs.rs_rasterize_culled(_p(pos), _p(tri), _p(rec), _p(flags), 1, W, H, _p(want), None, 0) == 0
        assert np.array_equal(_bits(want), _bits(depth)) and (int(stats[1]) == 0 or not flags[0, 0]), name
        decisions[name] = bool(flags[0, 0])
    lib.nvc_destroy(ctx)
    # the cases land where intended (the screen positions computed as the kernel does hit the halfway points exactly; at 40.5 the
    # float grid is fine enough for 1 ulp steps) and decide as half away from zero does
    f = np.float32
    assert f(_p32(_screen(_up(40.5 + S, 0), 0)[0], 1) - f(S)) == f(40.5) and f(_p32(_screen(0, _up(40.5 - S, 0))[1], 1) + f(S)) == f(40.5)
    assert f(_p32(_screen(-0.5 + S, 0)[0], 1) - f(S)) == f(-0.5) and f(_p32(_screen(2.5 + S, 0)[0], 1) - f(S)) == f(2.5)
    assert decisions["bmin.x - 1/256 = 40.5 +0 ulp"] and not decisions["bmin.x - 1/256 = 40.5 -1 ulp"] and decisions["bmin.x - 1/256 = 40.5 +1 ulp"]
    assert not decisions["bmax.y + 1/256 = 40.5 +0 ulp"] and decisions["bmax.y + 1/256 = 40.5 -1 ulp"]
    assert decisions["bmin.x - 1/256 = 2.5"] and decisions["bmin.x - 1/256 = -0.5"]
    assert decisions["equal after rounding"] and decisions["back"] and decisions["zero area"] and decisions["collinear"] and not decisions["front"]
    assert decisions["small"] and not decisions["small, w = 0"] and not decisions["small, w < 0"] and not decisions["back, w < 0"]
    assert not decisions["small, w NaN"] and not decisions["front, x NaN"]


# ---- CPU tier: closed two-phase loops --------------------------------------------------------------------------------------------


def _closed_loop(golden_dir, mode, frames, e_factory, cams, screen=(256, 192), kittens=100, device=None):
    """early cull -> produced depth (mesh cull on) -> pyramid of it -> late cull -> produced depth, over a moving camera.  Each pass's
    depth == the reference shader (CULL = 1) + the test rasteriser over the same clusters; after the late pass the image == the
    brute-force image of ALL clusters (CULL = 1); every pixel-owning cluster was emitted; early and late sets are disjoint."""
    s, vertices, meshletdata = _kitten_scene(golden_dir, kittens, screen)
    e = e_factory(s)
    gt = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    gt.set_visibility_bits(s.visibility_bits)
    owners_total, late_total, flagged_total = 0, 0, 0
    for f in range(frames):
        s.camera = cams[f % len(cams)]
        cd = s.cull_data()
        proj = host.projection(s.camera, *screen)
        cs = _CullStage(e.shader_view(), vertices, meshletdata, proj, threads=4)
        want = np.zeros((screen[1], screen[0]), np.float32)
        got = e.new_depth()
        sets = []
        for late in (False, True):
            if late:
                e.pyramid(got)
            e.cull(cd, late)
            cmds = e.task_commands()
            if mode == "clusters":
                e.render_clusters(cd, late)
                cib, count = e.cluster_indices()
                ci = cib[:count]
                ccb = np.array([count, 16, (count + 255) // 256, 16], np.uint32)
                padded = np.full(max((count + 255) // 256 * 256, 256), 0xFFFFFFFF, np.uint32)
                padded[:count] = ci
                rec, pos, tri, culled = cs.run_cull(cd, cib=padded, ccb=ccb, dcb=e.dcb_host())
                stats = e.raster(cd, proj, vertices, meshletdata, got)
            else:
                payloads, emit, n = e.task_shading(cd, late)
                ci = np.concatenate([payloads[c, : min(int(emit[c]), 64)] for c in range(n)]) if n else np.zeros(0, np.uint32)
                rec, pos, tri, culled = cs.run_payloads_cull(cd, payloads[:n], emit[:n], dcb=e.dcb_host())
                stats = e.raster_tasks(cd, proj, vertices, meshletdata, got)
            cs.rasterize_culled(rec, pos, tri, culled, want)
            tested, culled_n = e.mesh_cull_stats()
            assert int(stats[2]) == 0 and culled_n == _flagged(rec, culled) and tested == int(rec[:, 1].sum()), (f, late, stats, tested, culled_n)
            flagged_total += culled_n
            assert np.array_equal(_bits(want), _bits(e.host_depth(got))), ("depth", f, late)
            sets.append(oracle_lib.cluster_pairs(ci, cmds))
        early, late_set = sets
        assert len(np.intersect1d(early, late_set)) == 0, f
        late_total += len(late_set)
        # brute force: every meshlet of the selected LODs, no culling, through the same shader with CULL = 1
        gt.dvb[:] = 1
        gt.cull(s.cull_data(culling=False, occlusion=False, cluster_occlusion=False), late=False)
        all_cmds = gt.read_task_commands(int(gt.dccb[1]) * 64)
        cib, ccb, ci = _all_clusters(all_cmds, int(gt.dccb[0]))
        bs = _CullStage(gt, vertices, meshletdata, proj, threads=4)
        rec, pos, tri, culled = bs.run_cull(cd, cib=cib, ccb=ccb, dcb=gt.dcb)
        truth = np.zeros_like(want)
        bs.rasterize_culled(rec, pos, tri, culled, truth)
        assert np.array_equal(_bits(truth), _bits(want)), ("brute force", f, int((truth != want).sum()))
        own = bs.owners_culled(rec, pos, tri, culled, truth)
        owner_pairs = oracle_lib.cluster_pairs(ci[own[: len(ci)]], all_cmds)
        assert np.isin(owner_pairs, np.union1d(early, late_set)).all(), f
        owners_total += len(owner_pairs)
        assert (truth > 0).mean() > 0.05
    assert late_total > 0 and owners_total > 100 and flagged_total > 0
    e.close()


class _EmuLoop:
    """the emulated product path as _closed_loop drives it"""

    def __init__(self, s):
        self.p = _EmuPath(s.meshes, s.meshlets, s.draws, *s.screen, threads=4)
        self.p.set_visibility_bits(s.visibility_bits)
        self.p.set_mesh_cull(1)

    def shader_view(self):
        return self.p

    def new_depth(self):
        return np.zeros((self.p.depth_height, self.p.depth_width), np.float32)

    def host_depth(self, d):
        return d

    def pyramid(self, d):
        self.p.pyramid(d)

    def cull(self, cd, late):
        self.p.cull(cd, late)

    def task_commands(self):
        return self.p.read_task_commands(int(self.p.dccb[1]) * 64)

    def render_clusters(self, cd, late):
        self.p.render_clusters(cd, late)

    def cluster_indices(self):
        n = int(self.p.ccb[0])
        return self.p.read_cluster_indices(n), n

    def dcb_host(self):
        return self.p.dcb

    def task_shading(self, cd, late):
        n = int(self.p.dccb[1]) * 64
        self.payloads, self.emit = _task_buffers(n)
        self.p.task_shading(cd, late, self.payloads, self.emit)
        return self.payloads, self.emit, n

    def raster(self, cd, proj, vertices, meshletdata, got):
        return self.p.raster_depth(cd, proj, vertices, meshletdata, got)

    def raster_tasks(self, cd, proj, vertices, meshletdata, got):
        return self.p.raster_depth_tasks(cd, proj, self.payloads, self.emit, vertices, meshletdata, got)

    def mesh_cull_stats(self):
        return self.p.mesh_cull_stats(reset=True)

    def close(self):
        self.p.close()


@needs_refshader
@pytest.mark.parametrize("mode", ["clusters", "tasks"])
def test_closed_loop_with_mesh_cull_on_emulated_produced_depth(golden_dir, mode):
    _closed_loop(golden_dir, mode, 5, _EmuLoop, MOVING)


# ---- CPU tier: the switch, hostile data ------------------------------------------------------------------------------------------


def test_switching_off_restores_the_default_producer(golden_dir):
    """after nvc_set_mesh_cull(ctx, 0) both cluster producers give the default producer's bits; the indexed producer gives the same bits
    with the switch on or off"""
    screen = (256, 192)
    s, vertices, meshletdata = _kitten_scene(golden_dir, 80, screen)
    s.camera = CAMS[1]
    cd = s.cull_data()
    proj = host.projection(s.camera, *screen)
    default = _EmuPath(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    switched = _EmuPath(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    images = {}
    for name, p in (("default", default), ("switched", switched)):
        p.set_visibility_bits(s.visibility_bits)
        p.dvb[:] = 1  # everything visible last frame: the early pass draws
        p.mvb[:] = 0xFFFFFFFF
        p.cull(cd, False)
        p.render_clusters(cd, False)
        n = int(p.dccb[1]) * 64
        payloads, emit = _payloads_from_cib(p.cib, int(p.ccb[0]), n)
        for on in ((0,) if name == "default" else (1, 0)):
            if name == "switched":
                p.set_mesh_cull(on)
            a, b = np.zeros((screen[1], screen[0]), np.float32), np.zeros((screen[1], screen[0]), np.float32)
            sa = p.raster_depth(cd, proj, vertices, meshletdata, a)
            sb = p.raster_depth_tasks(cd, proj, payloads, emit, vertices, meshletdata, b)
            images[(name, on)] = (a, b, sa, sb)
    (a0, b0, sa0, sb0), (a1, b1, sa1, sb1), (a2, b2, sa2, sb2) = images[("default", 0)], images[("switched", 1)], images[("switched", 0)]
    assert np.array_equal(_bits(a0), _bits(a2)) and np.array_equal(_bits(b0), _bits(b2)) and np.array_equal(sa0, sa2) and np.array_equal(sb0, sb2)
    assert np.array_equal(_bits(a0), _bits(b0)) and np.array_equal(_bits(a1), _bits(b1))
    assert int(sa1[1]) < int(sa0[1]) and int(sa1[0]) == int(sa0[0])  # the stage was on: fewer triangles sampled, same clusters
    assert switched.mesh_cull_stats()[1] > 0
    default.close()
    switched.close()

    cvert, indices, meshes = _cache_geometry(golden_dir)
    cdi = s.cull_data(**INDEXED)
    p = _EmuPath(meshes, s.meshlets, s.draws, *screen, mesh_shading=False, threads=4)
    p.set_visibility_bits(s.visibility_bits)
    p.dvb[:] = 1
    p.cull(cdi, False, task=False)
    out = []
    for on in (0, 1, 0):
        p.set_mesh_cull(on)
        d = np.zeros((screen[1], screen[0]), np.float32)
        out.append((d, p.raster_depth_indexed(cdi, proj, cvert, indices, d)))
    assert all(np.array_equal(_bits(d), _bits(out[0][0])) and np.array_equal(st, out[0][1]) for d, st in out) and (out[0][0] > 0).mean() > 0.05
    assert p.mesh_cull_stats() == (0, 0)
    p.close()


def test_hostile_meshlets_with_mesh_cull_in_guarded_memory(golden_dir):
    """out-of-range meshlet data, vertex references and triangle indices with the stage on: the same rejections, stats4[2] and image as
    with it off, with every input array ending at an inaccessible page (any read past an end faults)"""
    screen = (128, 96)
    s, vertices, meshletdata = _kitten_scene(golden_dir, 40, screen)
    cd = s.cull_data(culling=False, occlusion=False, cluster_occlusion=False)
    proj = (ctypes.c_float * 16)(*[float(v) for v in host.projection(s.camera, *screen)])
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    o.dvb[:] = 1
    o.cull(cd, False)
    o.render_clusters(cd, False)
    pd = o._pass_data(cd, 0, 0)
    ncmd = int(o.dccb[1]) * 64
    tcmds = o.read_task_commands(ncmd)
    count = int(o.ccb[0])
    cib_live = o.cib[:count].copy()
    payloads, emit = _payloads_from_cib(o.cib, count, ncmd)
    lib = emu_lib.load()
    ctx = ctypes.c_void_p()
    lib.emu_guard_allocations(1)  # the context's device allocations (the counters among them) end at a guard page too
    try:
        assert lib.nvc_create(0, None, ctypes.byref(ctx)) == 0
    finally:
        lib.emu_guard_allocations(0)

    md_words = np.ascontiguousarray(meshletdata, dtype=np.uint32)
    mls = s.meshlets.copy()
    variants = {"as cooked": (mls, md_words)}
    bad = mls.copy()
    bad["dataOffset"][::3] = len(md_words) - 2  # references / triangles past the end of meshletdata
    variants["data past the end"] = (bad, md_words)
    bad = mls.copy()
    bad["baseVertex"][1::4] = len(vertices) // 16 - 5  # vertex references past vertex_count
    variants["vertices past the end"] = (bad, md_words)
    bad = mls.copy()
    bad["vertexCount"][2::5] = 65
    bad["triangleCount"][3::5] = 97
    variants["counts past 64 / 96"] = (bad, md_words)
    bad_md = md_words.copy()
    used = mls[mls["triangleCount"] > 0][:50]
    for m in used:  # triangle indices >= vertexCount
        first = int(m["dataOffset"]) + (int(m["vertexCount"]) + 1) // 2 if m["shortRefs"] else int(m["dataOffset"]) + int(m["vertexCount"])
        bad_md[first] = np.uint32(0xFFFEFD00) | np.uint32(bad_md[first] & 0xFF)
    variants["triangle indices past vertexCount"] = (mls, bad_md)

    def run(meshlets, md, on, tasks):
        assert lib.nvc_set_mesh_cull(ctx, on) == 0
        depth, stats = np.zeros((screen[1], screen[0]), np.float32), np.zeros(4, np.uint32)
        g = [_guarded(a) for a in (np.ascontiguousarray(meshlets), md, np.ascontiguousarray(vertices), np.ascontiguousarray(s.draws), o.dcb[: max(ncmd * 20, 20)].copy())]
        gm, gmd, gvb, gdraws, gdcb = g
        if tasks:
            gp, ge, gc4 = _guarded(payloads), _guarded(emit), _guarded(o.dccb.copy())
            st = lib.nvc_raster_depth_tasks(ctx, None, proj, ctypes.byref(pd), _p(gp), _p(ge), _p(gc4), _p(gdcb), _p(gdraws), _p(gm), _p(gmd), len(gmd), _p(gvb), len(gvb) // 16, _p(depth), screen[0], screen[1], _p(stats))
        else:
            cib = np.full((count + 255) // 256 * 256, 0xFFFFFFFF, np.uint32)
            cib[:count] = cib_live
            gcib, gccb = _guarded(cib), _guarded(o.ccb.copy())
            st = lib.nvc_raster_depth(ctx, None, proj, ctypes.byref(pd), _p(gcib), _p(gccb), _p(gdcb), _p(gdraws), _p(gm), _p(gmd), len(gmd), _p(gvb), len(gvb) // 16, _p(depth), screen[0], screen[1], _p(stats))
        assert st == 0
        out = (ctypes.c_uint64 * 2)()
        assert lib.nvc_mesh_cull_stats(ctx, out, 1) == 0
        return depth, stats, (int(out[0]), int(out[1]))

    rejections = 0
    for name, (meshlets, md) in variants.items():
        for tasks in (False, True):
            d0, s0, c0 = run(meshlets, md, 0, tasks)
            d1, s1, c1 = run(meshlets, md, 1, tasks)
            assert c0 == (0, 0) and c1[0] > 0, (name, tasks, c0, c1)
            # the same clusters drawn and rejected; fewer triangles sampled, by at most the number culled
            assert int(s1[0]) == int(s0[0]) and int(s1[2]) == int(s0[2]) and int(s1[3]) <= int(s0[3]), (name, tasks, s0, s1)
            assert int(s1[1]) <= int(s0[1]) <= int(s1[1]) + c1[1], (name, tasks, s0, s1, c1)
            assert ((d1 > 0) <= (d0 > 0)).all() and (d1 <= d0).all(), (name, tasks)
            rejections += int(s0[2])
            if name == "as cooked":
                assert int(s0[2]) == 0 and int(s0[0]) == count
    assert rejections > 0
    lib.nvc_destroy(ctx)


# ---- GPU tier --------------------------------------------------------------------------------------------------------------------


class _DeviceLoop:
    """the CUDA path (VisibilityPath) as _closed_loop drives it, the oracle path's buffers mirrored for the shader"""

    def __init__(self, s):
        import torch
        from niagara_b200.path import VisibilityPath

        self.torch = torch
        self.g = VisibilityPath(s.meshes, s.meshlets, s.draws, *s.screen)
        self.g.set_visibility_bits(s.visibility_bits)
        self.g.set_mesh_cull(True)
        self.view = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *s.screen, threads=4)
        self.stats = torch.zeros(4, dtype=torch.int32, device="cuda")
        self.vb = self.md = None

    def shader_view(self):
        return self.view

    def new_depth(self):
        return self.torch.zeros((self.g.depth_height, self.g.depth_width), dtype=self.torch.float32, device="cuda")

    def host_depth(self, d):
        return d.cpu().numpy()

    def pyramid(self, d):
        self.g.pyramid(d)

    def cull(self, cd, late):
        self.g.cull(cd, late)

    def task_commands(self):
        n = int(self.g.dccb[1].item()) * 64
        return self.g.read_task_commands(n)

    def render_clusters(self, cd, late):
        self.g.render_clusters(cd, late)

    def cluster_indices(self):
        n = int(self.g.ccb[0].item())
        return self.g.cib[:n].cpu().numpy().astype(np.uint32), n

    def dcb_host(self):
        return self.g.dcb.cpu().numpy()

    def task_shading(self, cd, late):
        torch = self.torch
        n = int(self.g.dccb[1].item()) * 64
        self.gp = torch.zeros((max(n, 1), 64), dtype=torch.int32, device="cuda")
        self.ge = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
        self.g.task_shading(cd, late, self.gp, self.ge)
        torch.cuda.synchronize()
        return self.gp.cpu().numpy().astype(np.uint32), self.ge.cpu().numpy().astype(np.uint32), n

    def _geometry(self, vertices, meshletdata):
        if self.vb is None:
            self.vb = self.torch.from_numpy(np.ascontiguousarray(vertices)).cuda()
            self.md = self.torch.from_numpy(np.ascontiguousarray(meshletdata, dtype=np.uint32).view(np.int32)).cuda()

    def raster(self, cd, proj, vertices, meshletdata, got):
        self._geometry(vertices, meshletdata)
        self.g.raster_depth(cd, proj, self.vb, self.md, got, self.stats)
        self.torch.cuda.synchronize()
        return self.stats.cpu().numpy().astype(np.uint32)

    def raster_tasks(self, cd, proj, vertices, meshletdata, got):
        self._geometry(vertices, meshletdata)
        self.g.raster_depth_tasks(cd, proj, self.gp, self.ge, self.vb, self.md, got, self.stats)
        self.torch.cuda.synchronize()
        return self.stats.cpu().numpy().astype(np.uint32)

    def mesh_cull_stats(self):
        return self.g.mesh_cull_stats(reset=True)

    def close(self):
        self.g.close()


@pytest.mark.gpu
@needs_refshader
@pytest.mark.parametrize("mode", ["clusters", "tasks"])
def test_closed_loop_with_mesh_cull_on_device_produced_depth(golden_dir, mode):
    _closed_loop(golden_dir, mode, 5, _DeviceLoop, MOVING, screen=(512, 384), kittens=300)


@pytest.mark.gpu
@needs_refshader
@pytest.mark.parametrize("mode", ["clusters", "tasks"])
def test_c3_style_frame_with_mesh_cull(golden_dir, mode):
    """~2 000 C3-style draws at 1024^2 with the stage on: two frames of the two-phase loop on device depth equal the CPU reference-shader
    pipeline (CULL = 1) bit for bit with the same culled count; the last frame run again from the same visibility state gives the same
    bits and counts; with the stage switched off the same frame gives the default producer's bits"""
    import torch
    from niagara_b200.path import VisibilityPath

    screen = (1024, 1024)
    s = scenes.config3_scene(golden_dir, draw_count=2000, screen=screen)
    tasks = mode == "tasks"
    vertices, meshletdata = s.vertices, s.meshletdata
    md = torch.from_numpy(meshletdata.view(np.int32)).cuda()
    vb = torch.from_numpy(np.ascontiguousarray(vertices)).cuda()
    g = VisibilityPath(s.meshes, s.meshlets, s.draws, *screen)
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *screen, threads=os.cpu_count() or 8)
    g.set_visibility_bits(s.visibility_bits)
    o.set_visibility_bits(s.visibility_bits)
    cd = s.cull_data()
    proj = host.projection(s.camera, *screen)
    stats = torch.zeros(4, dtype=torch.int32, device="cuda")
    cs = _CullStage(o, vertices, meshletdata, proj, threads=os.cpu_count() or 8)

    def device_frame():
        got = torch.zeros((screen[1], screen[0]), dtype=torch.float32, device="cuda")
        sampled = []
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
                g.render_clusters(cd, late)
                g.raster_depth(cd, proj, vb, md, got, stats)
            torch.cuda.synchronize()
            st = stats.cpu().numpy()
            assert int(st[2]) == 0, st
            sampled.append(tuple(int(v) for v in st))
        return got.cpu().numpy(), sampled, g.mesh_cull_stats(reset=True)

    def cpu_frame():
        want = np.zeros((screen[1], screen[0]), np.float32)
        flagged = 0
        for late in (False, True):
            if late:
                o.pyramid(want)
            o.cull(cd, late)
            if tasks:
                n = int(o.dccb[1]) * 64
                op, oe = _task_buffers(n)
                o.task_shading(cd, late, op, oe)
                rec, pos, tri, culled = cs.run_payloads_cull(cd, op[:n], oe[:n])
            else:
                o.render_clusters(cd, late)
                rec, pos, tri, culled = cs.run_cull(cd)
            cs.rasterize_culled(rec, pos, tri, culled, want)
            flagged += _flagged(rec, culled)
        return want, flagged

    g.set_mesh_cull(True)
    g.mesh_cull_stats(reset=True)
    for f in range(2):
        if f == 1:
            dvb, mvb = g.dvb.clone(), g.mvb.clone()
        got, sampled, counts = device_frame()
        want, flagged = cpu_frame()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (f, int((got != want).sum()))
        assert counts[1] == flagged > 0 and (want > 0).mean() > 0.05, (f, counts, flagged)
    g.dvb.copy_(dvb)
    g.mvb.copy_(mvb)
    again, sampled_again, counts_again = device_frame()
    assert sampled_again == sampled and counts_again == counts and np.array_equal(again.view(np.uint32), got.view(np.uint32))
    # the same frame with the stage off == a path that never had it on
    g.dvb.copy_(dvb)
    g.mvb.copy_(mvb)
    g.set_mesh_cull(False)
    off, sampled_off, counts_off = device_frame()
    d = VisibilityPath(s.meshes, s.meshlets, s.draws, *screen)
    d.set_visibility_bits(s.visibility_bits)
    d.dvb.copy_(dvb)
    d.mvb.copy_(mvb)
    g, g_on = d, g
    default, sampled_default, _ = device_frame()
    assert counts_off == (0, 0) and sampled_off == sampled_default and np.array_equal(off.view(np.uint32), default.view(np.uint32))
    assert sum(v[1] for v in sampled_default) > sum(v[1] for v in sampled)
    g_on.close()
    d.close()
