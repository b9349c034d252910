"""The reference's TASK_CULL = 0 build (nvc_set_task_cull): the late drawcull emits only draws not visible last frame (plus post-pass
draws), and the cluster and task passes pass every meshlet of every command through without a test.

The oracle is the reference's own shaders with its own switch flipped: oracle/refshader_taskcull generates drawcull, clustercull and
meshlet.task with `#define TASK_CULL 0` (oracle/_ref/librefshader_taskcull.so).
CPU tier: the product's kernels under the SIMT emulation (tests/cuda_emu) against those shaders, bit for bit: the drawcull flag
matrix, the cluster and task passes (early, late, post), edge inputs (small cluster_limit, hostile taskCount, no commands, guarded
memory), five-frame closed loops on produced depth against the brute-force image, and switching back on.
GPU tier (-m gpu): the same loops on the device, a C4-size frame against a numpy expansion of the commands, and a captured graph."""
import ctypes
import mmap
import os

import numpy as np
import pytest

import emu_lib
import oracle_lib
import refshader_lib
from niagara_b200 import host, layout
from test_end_to_end_raster import _all_clusters, _kitten_scene
from test_kernels_emulated import _guarded
from test_mesh_cull import MOVING
from test_raster_submission_modes import _EmuPath as _ModesEmuPath
from test_raster_submission_modes import _bits, _task_buffers

vp, sz, i32 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int

SO = os.path.join(refshader_lib.ROOT, "oracle", "_ref", "librefshader_taskcull.so")
_LIB = []


def _available():
    return os.path.exists(SO) or os.path.isdir(os.path.join(refshader_lib.REFERENCE, "src", "shaders"))


needs_refshader = pytest.mark.skipif(not (refshader_lib.available() and _available()), reason="needs /root/reference or prebuilt oracle/_ref/librefshader.so and librefshader_taskcull.so")


def _rs0():
    """oracle/_ref/librefshader_taskcull.so with the argument types of its TASK_CULL = 0 entry points; built from the reference where
    that exists, as refshader_lib.load() does"""
    if _LIB:
        return _LIB[0]
    if os.path.isdir(os.path.join(refshader_lib.REFERENCE, "src", "shaders")):
        import subprocess

        subprocess.run(["make", "-s", "-C", os.path.join(refshader_lib.ROOT, "oracle", "refshader_taskcull"), "REF=" + refshader_lib.REFERENCE], check=True)
    rs = ctypes.CDLL(SO)
    cd, hz = ctypes.POINTER(layout.CullData), ctypes.POINTER(layout.HiZ)
    rs.rs_drawcull_taskcull0.restype = i32
    rs.rs_drawcull_taskcull0.argtypes = [cd, i32, i32, vp, sz, vp, sz, vp, sz, vp, sz, vp, hz, i32]
    rs.rs_clustercull_taskcull0.restype = i32
    rs.rs_clustercull_taskcull0.argtypes = [cd, i32, vp, sz, vp, vp, sz, vp, sz, vp, sz, vp, sz, vp, hz, i32]
    rs.rs_taskcull_taskcull0.restype = i32
    rs.rs_taskcull_taskcull0.argtypes = [cd, i32, vp, sz, vp, vp, sz, vp, sz, vp, sz, vp, vp, hz, i32]
    _LIB.append(rs)
    return rs


_p, _n = refshader_lib._p, refshader_lib._n


class _RefPath0(refshader_lib.RefShaderPath):
    """RefShaderPath with drawcull, clustercull and meshlet.task as a TASK_CULL = 0 build compiles them"""

    def cull(self, cull_data, late, post_pass=0, task=None):
        task = self.mesh_shading if task is None else task
        pd = self._pass_data(cull_data, 1, post_pass)
        s = _rs0().rs_drawcull_taskcull0(ctypes.byref(pd), int(late), int(task), _p(self.draws), _n(self.draws), _p(self.meshes), _n(self.meshes), _p(self.dvb), _n(self.dvb), _p(self.dcb), _n(self.dcb), _p(self.dccb), ctypes.byref(self.hiz), self.threads)
        assert s == 0, s

    def render_clusters(self, cull_data, late, post_pass=0, cluster_backface=None):
        pd = self._pass_data(cull_data, 0, post_pass)
        if cluster_backface is not None:
            pd.clusterBackfaceEnabled = int(cluster_backface)
        s = _rs0().rs_clustercull_taskcull0(ctypes.byref(pd), int(late), _p(self.dcb), _n(self.dcb), _p(self.dccb), _p(self.draws), _n(self.draws), _p(self.meshlets), _n(self.meshlets), _p(self.mvb), _n(self.mvb), _p(self.cib), _n(self.cib), _p(self.ccb), ctypes.byref(self.hiz), self.threads)
        assert s == 0, s

    def task_shading(self, cull_data, late, payloads, emit_counts, post_pass=0, cluster_backface=None):
        pd = self._pass_data(cull_data, 0, post_pass)
        if cluster_backface is not None:
            pd.clusterBackfaceEnabled = int(cluster_backface)
        s = _rs0().rs_taskcull_taskcull0(ctypes.byref(pd), int(late), _p(self.dcb), _n(self.dcb), _p(self.dccb), _p(self.draws), _n(self.draws), _p(self.meshlets), _n(self.meshlets), _p(self.mvb), _n(self.mvb), _p(payloads), _p(emit_counts), ctypes.byref(self.hiz), self.threads)
        assert s == 0, s


class _EmuPath(_ModesEmuPath):
    """the emulated path with the task-cull switch"""

    def set_task_cull(self, enabled):
        self._check(self.emu.nvc_set_task_cull(self.ctx, int(enabled)), "nvc_set_task_cull")


def _expand(cmds, ncmd):
    """what a TASK_CULL = 0 cluster pass appends for commands[0..ncmd): c | (mgi << 24) for every mgi < min(taskCount, 64), in command
    order"""
    counts = np.minimum(cmds["taskCount"][:ncmd].astype(np.int64), 64)
    cid = np.repeat(np.arange(ncmd, dtype=np.int64), counts)
    mgi = np.arange(int(counts.sum()), dtype=np.int64) - np.repeat(np.cumsum(counts) - counts, counts)
    return (cid | (mgi << 24)).astype(np.uint32)


def _task_expected(cmds, ncmd):
    """what a TASK_CULL = 0 task pass writes for commands[0..ncmd): every payload entry c | (lane << 24), emit = taskCount as stored"""
    lanes = np.arange(64, dtype=np.uint32)
    payloads = (np.arange(ncmd, dtype=np.uint32)[:, None] | (lanes[None, :] << 24)).astype(np.uint32)
    return payloads, cmds["taskCount"][:ncmd].astype(np.uint32)


def _sorted_cmds(path, task):
    n = int(path.dccb[0])
    if task:
        n = min(n, path.limits.task_wglimit)
        return oracle_lib.sorted_commands(path.read_task_commands(n))
    return oracle_lib.sorted_commands(path.read_draw_commands(n))


def _cluster_result(path):
    """(sorted cib prefix, ccb, the padding up to the dispatch's end)"""
    count = min(int(path.ccb[0]), len(path.cib))
    end = int(path.ccb[2]) * 256
    return np.sort(path.cib[:count]), path.ccb.copy(), path.cib[count:end].copy()


def _scene(golden_dir, n=120, screen=(320, 240)):
    s, vertices, meshletdata = _kitten_scene(golden_dir, n, screen)
    s.camera = MOVING[1]
    return s, vertices, meshletdata


def _depth(screen, seed=7):
    """a reverse-Z depth image with structure at several scales, so that the late passes' occlusion tests go both ways"""
    rng = np.random.default_rng(seed)
    d = np.zeros((screen[1], screen[0]), np.float32)
    for _ in range(40):
        x0, y0 = rng.integers(0, screen[0]), rng.integers(0, screen[1])
        w, h = rng.integers(8, screen[0] // 2), rng.integers(8, screen[1] // 2)
        d[y0: y0 + h, x0: x0 + w] = np.maximum(d[y0: y0 + h, x0: x0 + w], np.float32(rng.uniform(0.002, 0.05)))
    return d


def _paths(s, screen, **kwargs):
    e = _EmuPath(s.meshes, s.meshlets, s.draws, *screen, threads=4, **kwargs)
    e.set_task_cull(0)
    r = _RefPath0(s.meshes, s.meshlets, s.draws, *screen, threads=4, **kwargs)
    for p in (e, r):
        p.set_visibility_bits(s.visibility_bits)
    return e, r


def _copy_state(src, dst):
    dst.dvb[:] = src.dvb
    dst.mvb[:] = src.mvb
    dst.dcb[:] = src.dcb
    dst.dccb[:] = src.dccb


# ---- CPU tier: the switch is live ------------------------------------------------------------------------------------------------


@needs_refshader
def test_task_cull_0_shaders_differ_from_the_default_build(golden_dir):
    """on the kitten scene the TASK_CULL = 0 shaders give another late command set and another cluster set than the TASK_CULL = 1
    ones, so the comparisons below cannot pass by accident"""
    screen = (320, 240)
    s, _, _ = _scene(golden_dir)
    cd = s.cull_data()
    r0 = _RefPath0(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    r1 = refshader_lib.RefShaderPath(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    rng = np.random.default_rng(3)
    dvb = (rng.random(len(s.draws)) < 0.5).astype(np.uint32)
    out = {}
    for name, r in (("0", r0), ("1", r1)):
        r.set_visibility_bits(s.visibility_bits)
        r.mvb[:] = rng.integers(0, 2**32, len(r.mvb), dtype=np.uint64).astype(np.uint32) if name == "0" else r0.mvb
        r.dvb[:] = dvb
        r.pyramid(_depth(screen))
        r.cull(cd, False)
        r.render_clusters(cd, False)
        early = oracle_lib.cluster_pairs(r.cib[: int(r.ccb[0])], r.read_task_commands(int(r.dccb[1]) * 64))
        r.dvb[:] = dvb
        r.cull(cd, True)
        out[name] = (_sorted_cmds(r, True), early)
    assert len(out["0"][0]) and len(out["1"][0]) > len(out["0"][0]) and not np.array_equal(out["0"][0], out["1"][0])
    assert len(out["0"][1]) > len(out["1"][1]) > 0 and np.isin(out["1"][1], out["0"][1]).all()


# ---- CPU tier: drawcull ----------------------------------------------------------------------------------------------------------


@needs_refshader
def test_drawcull_matches_the_task_cull_0_shader(golden_dir):
    """commands (sorted), dccb and dvb == drawcull.comp.glsl with TASK_CULL = 0 for late x task x postPass x clusterOcclusionEnabled"""
    screen = (320, 240)
    s, _, _ = _scene(golden_dir)
    e, r = _paths(s, screen)
    depth = _depth(screen)
    e.pyramid(depth)
    r.pyramid(depth)
    assert np.array_equal(e.pyramid_texels, r.pyramid_texels)
    dvb = (np.random.default_rng(5).random(len(s.draws)) < 0.5).astype(np.uint32)
    emitted = {}
    for late in (0, 1):
        for task in (0, 1):
            for post in (0, 1):
                for cocc in (0, 1):
                    cd = s.cull_data(cluster_occlusion=bool(cocc))
                    for p in (e, r):
                        p.dvb[:] = dvb
                        p.cull(cd, late, post_pass=post, task=task)
                    key = (late, task, post, cocc)
                    k = 4 if task else 1  # (draw mode: drawcull writes only dccb[0]; the product sets [1..3] to 0)
                    assert np.array_equal(e.dccb[:k], r.dccb[:k]), (key, e.dccb, r.dccb)
                    assert np.array_equal(_sorted_cmds(e, task), _sorted_cmds(r, task)), key
                    assert np.array_equal(e.dvb, r.dvb), key
                    emitted[key] = int(e.dccb[0])
    # the late rule: without post pass, only draws not visible last frame are emitted, whatever clusterOcclusionEnabled says
    assert emitted[(1, 1, 0, 1)] == emitted[(1, 1, 0, 0)] and emitted[(1, 0, 0, 1)] == emitted[(1, 0, 0, 0)]
    assert emitted[(1, 0, 0, 1)] > 0 and emitted[(0, 0, 0, 1)] > 0
    e.close()


# ---- CPU tier: cluster and task passes -------------------------------------------------------------------------------------------


def _commands(golden_dir, screen=(320, 240)):
    """task commands of a real drawcull (every draw visible last frame and now) in a path pair, and the scene"""
    s, _, _ = _scene(golden_dir)
    e, r = _paths(s, screen)
    cd = s.cull_data(culling=False, occlusion=False)
    r.dvb[:] = 1
    r.cull(cd, False)
    _copy_state(r, e)
    return s, e, r


@needs_refshader
@pytest.mark.parametrize("phase", ["early", "late", "post"])
def test_cluster_pass_matches_the_task_cull_0_shader(golden_dir, phase):
    """the sorted cib prefix, ccb, the ~0 padding and an untouched mvb == clustercull.comp.glsl (TASK_CULL = 0) + clustersubmit, and the
    output depends neither on clusterOcclusionEnabled, backface culling nor the Hi-Z contents"""
    screen = (320, 240)
    s, e, r = _commands(golden_dir, screen)
    late, post = phase != "early", int(phase == "post")
    rng = np.random.default_rng(11)
    mvb = rng.integers(0, 2**32, len(e.mvb), dtype=np.uint64).astype(np.uint32)
    ncmd = int(r.dccb[1]) * 64
    want_codes = np.sort(_expand(r.read_task_commands(ncmd), ncmd))
    results = []
    for cocc, bf, depth in ((1, 1, _depth(screen)), (0, 0, _depth(screen, 9)), (1, 0, np.zeros((screen[1], screen[0]), np.float32))):
        cd = s.cull_data(cluster_occlusion=bool(cocc))
        for p in (e, r):
            p.pyramid(depth)
            p.mvb[:] = mvb
            p.cib[:] = 0x12345678
            p.render_clusters(cd, late, post_pass=post, cluster_backface=bool(bf))
            assert np.array_equal(p.mvb, mvb)
        got, want = _cluster_result(e), _cluster_result(r)
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), (phase, cocc, bf, got[1], want[1])
        assert np.array_equal(got[0], want_codes) and (got[2] == 0xFFFFFFFF).all() and len(got[2]) < 256
        results.append(got)
    assert all(all(np.array_equal(a, b) for a, b in zip(results[0], x)) for x in results[1:])
    assert len(want_codes) > 1000
    e.close()


@needs_refshader
@pytest.mark.parametrize("phase", ["early", "late", "post"])
def test_task_pass_matches_the_task_cull_0_shader(golden_dir, phase):
    """all 64 payload entries and the raw emit counts of every command c < X * 64, padding commands included, == meshlet.task.glsl
    (TASK_CULL = 0); mvb is not written"""
    screen = (320, 240)
    s, e, r = _commands(golden_dir, screen)
    late, post = phase != "early", int(phase == "post")
    cd = s.cull_data()
    mvb = np.random.default_rng(12).integers(0, 2**32, len(e.mvb), dtype=np.uint64).astype(np.uint32)
    ncmd = int(r.dccb[1]) * 64
    out = []
    for p in (e, r):
        p.pyramid(_depth(screen))
        p.mvb[:] = mvb
        payloads, emit = _task_buffers(ncmd)
        payloads[:] = 0x12345678
        emit[:] = 0x12345678
        p.task_shading(cd, late, payloads, emit, post_pass=post)
        assert np.array_equal(p.mvb, mvb)
        out.append((payloads, emit))
    (gp, ge), (wp, we) = out
    assert np.array_equal(gp, wp) and np.array_equal(ge, we)
    xp, xe = _task_expected(r.read_task_commands(ncmd), ncmd)
    assert np.array_equal(gp, xp) and np.array_equal(ge, xe)
    assert int(r.dccb[0]) < ncmd and (ge[int(r.dccb[0]):] == 0).all()  # padding commands exist and emit 0
    e.close()


# ---- CPU tier: edge inputs -------------------------------------------------------------------------------------------------------


def _hostile_commands(counts, ncmd_groups=1):
    cmds = np.zeros(ncmd_groups * 64, layout.MESHTASKCOMMAND_DTYPE)
    cmds["taskCount"][: len(counts)] = counts
    cmds["drawId"] = np.arange(len(cmds)) % 3
    cmds["taskOffset"] = 7
    return cmds


HOSTILE = [0, 64, 65, 0xFFFFFFFF, 1, 63, 0xFFFFFFFF, 0, 65, 64]


@needs_refshader
def test_hostile_task_counts_and_no_commands(golden_dir):
    """taskCount 0, 64, 65 and 0xffffffff in both passes (the cluster pass takes min(taskCount, 64), the task pass emits the raw
    value), and command_count4[1] = 0 (no clusters, ccb {0, 16, 0, 16}, no payload written)"""
    screen = (64, 64)
    s, _, _ = _scene(golden_dir, 4, screen)
    cd = s.cull_data()
    e, r = _paths(s, screen)
    cmds = _hostile_commands(HOSTILE)
    for groups in (1, 0):
        for p in (e, r):
            p.dcb[:] = 0
            p.dcb[: cmds.nbytes] = cmds.view(np.uint8)
            p.dccb[:] = [len(HOSTILE), groups, 64, 1]
            p.render_clusters(cd, False)
        got, want = _cluster_result(e), _cluster_result(r)
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), (groups, got[1], want[1])
        assert np.array_equal(got[0], np.sort(_expand(cmds, groups * 64)))
        out = []
        for p in (e, r):
            payloads, emit = _task_buffers(64)
            payloads[:] = 0x12345678
            emit[:] = 0x12345678
            p.task_shading(cd, False, payloads, emit)
            out.append((payloads, emit))
        assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
        if groups:
            xp, xe = _task_expected(cmds, 64)
            assert np.array_equal(out[0][0], xp) and np.array_equal(out[0][1], xe) and int(out[0][1][3]) == 0xFFFFFFFF
        else:
            assert list(got[1]) == [0, 16, 0, 16] and (out[0][0] == 0x12345678).all() and (out[0][1] == 0x12345678).all()
    e.close()


@needs_refshader
@pytest.mark.parametrize("limit", [1, 300, 1000])
def test_small_cluster_limit(golden_dir, limit):
    """with cluster_limit below the pass's cluster count, ccb[0] is the full count, the stored entries are distinct members of the
    expected set, and the padding follows the clamped count"""
    screen = (320, 240)
    s, e0, r = _commands(golden_dir, screen)
    e0.close()
    e = _EmuPath(s.meshes, s.meshlets, s.draws, *screen, threads=4, cluster_limit=limit, cluster_capacity=(limit + 255) // 256 * 256)
    e.set_task_cull(0)
    e.set_visibility_bits(s.visibility_bits)
    _copy_state(r, e)
    ncmd = int(r.dccb[1]) * 64
    want = _expand(r.read_task_commands(ncmd), ncmd)
    e.render_clusters(s.cull_data(), True)
    assert int(e.ccb[0]) == len(want) > limit and int(e.ccb[2]) == (limit + 255) // 256
    stored = e.cib[:limit]
    assert len(np.unique(stored)) == limit and np.isin(stored, want).all() and (e.cib[limit:] == 0xFFFFFFFF).all()
    e.close()


def _no_access(nbytes):
    """the address of a fresh mapping of at least nbytes that faults on any access (PROT_NONE)"""
    libc = ctypes.CDLL(None, use_errno=True)
    libc.mmap.restype = ctypes.c_void_p
    libc.mmap.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_long]
    addr = libc.mmap(None, max(nbytes, 1), 0, mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS, -1, 0)  # PROT_NONE
    assert addr is not None and addr != ctypes.c_void_p(-1).value, ctypes.get_errno()
    return ctypes.c_void_p(addr)


def test_pass_through_in_guarded_memory(golden_dir):
    """in guarded memory: outputs sized exactly and ending at an inaccessible page, draws, meshlets and mvb inaccessible as a
    whole (the passes must not read them), the context's own allocations guarded too"""
    screen = (64, 64)
    s, _, _ = _scene(golden_dir, 4, screen)
    cd = s.cull_data(cluster_occlusion=False)
    lib = emu_lib.load()
    ctx = ctypes.c_void_p()
    lib.emu_guard_allocations(1)
    try:
        assert lib.nvc_create(0, None, ctypes.byref(ctx)) == 0
    finally:
        lib.emu_guard_allocations(0)
    assert lib.nvc_set_task_cull(ctx, 0) == 0
    hiz = host.hiz_layout(*screen)
    texels = np.zeros(hiz.total_texels, np.float32)
    hiz.texels = texels.ctypes.data
    draws, meshlets, mvb = (_no_access(1 << 20) for _ in range(3))
    for groups, counts in ((2, HOSTILE + [64] * 70), (1, [65] * 64), (0, [])):
        cmds = _hostile_commands(counts, max(groups, 1))
        ncmd = groups * 64
        want = _expand(cmds, ncmd)
        pad = (len(want) + 255) // 256 * 256
        gcmds, gc4 = _guarded(cmds[: max(ncmd, 1)]), _guarded(np.array([len(counts), groups, 64, 1], np.uint32))
        for late in (0, 1):
            pd = layout.CullData()
            ctypes.memmove(ctypes.byref(pd), ctypes.byref(cd), ctypes.sizeof(pd))
            cib, ccb = _guarded(np.zeros(max(pad, 1), np.uint32)), _guarded(np.zeros(4, np.uint32))
            assert lib.nvc_clustercull(ctx, None, ctypes.byref(pd), late, _p(gcmds), _p(gc4), draws, meshlets, mvb, _p(cib), _p(ccb), ctypes.byref(hiz)) == 0
            assert int(ccb[0]) == len(want) and np.array_equal(np.sort(cib[: len(want)]), np.sort(want)) and (cib[len(want): pad] == 0xFFFFFFFF).all()
            payloads, emit = _guarded(np.zeros((max(ncmd, 1), 64), np.uint32)), _guarded(np.zeros(max(ncmd, 1), np.uint32))
            assert lib.nvc_taskcull(ctx, None, ctypes.byref(pd), late, _p(gcmds), _p(gc4), draws, meshlets, mvb, _p(payloads), _p(emit), ctypes.byref(hiz)) == 0
            if ncmd:
                xp, xe = _task_expected(cmds, ncmd)
                assert np.array_equal(payloads, xp) and np.array_equal(emit, xe)
    lib.nvc_destroy(ctx)


# ---- CPU tier: closed loops and the switch ---------------------------------------------------------------------------------------


def _closed_loop(golden_dir, mode, frames, e_factory, cams, screen=(256, 192), kittens=100):
    """TASK_CULL = 0 two-phase frames on produced depth over a moving camera: the product path against the TASK_CULL = 0 shaders ->
    the reference's mesh shader -> the test rasteriser.  Depth bit-identical after every pass, the same dvb, disjoint early / late
    draw sets, and the early + late image == the brute-force image of every meshlet of every draw at its selected LOD."""
    s, vertices, meshletdata = _kitten_scene(golden_dir, kittens, screen)
    e = e_factory(s)
    r = _RefPath0(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    r.set_visibility_bits(s.visibility_bits)
    gt = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *screen, threads=4)
    gt.set_visibility_bits(s.visibility_bits)
    late_draws = 0
    for f in range(frames):
        s.camera = cams[f % len(cams)]
        cd = s.cull_data()
        proj = host.projection(s.camera, *screen)
        ms = refshader_lib.MeshStage(r, vertices, meshletdata, proj, threads=4)
        want = np.zeros((screen[1], screen[0]), np.float32)
        got = e.new_depth()
        draw_sets = []
        for late in (False, True):
            if late:
                e.pyramid(got)
                r.pyramid(want)
            e.cull(cd, late)
            r.cull(cd, late)
            cmds = r.read_task_commands(int(r.dccb[1]) * 64)
            assert np.array_equal(e.dccb(), r.dccb) and np.array_equal(oracle_lib.sorted_commands(e.task_commands()), oracle_lib.sorted_commands(cmds)), (f, late)
            n = int(r.dccb[1]) * 64
            if mode == "clusters":
                r.render_clusters(cd, late)
                e.render_clusters(cd, late)
                rec, pos, tri = ms.run(cd)
                stats = e.raster(cd, proj, vertices, meshletdata, got)
                assert int(stats[0]) == int(r.ccb[0]), (f, late, stats)
            else:
                payloads, emit = _task_buffers(n)
                r.task_shading(cd, late, payloads, emit)
                rec, pos, tri = ms.run_payloads(cd, payloads[:n], emit[:n])
                stats = e.raster_tasks(cd, late, proj, vertices, meshletdata, got, n)
                assert int(stats[0]) == len(rec), (f, late, stats)
            ms.rasterize(rec, pos, tri, want)
            assert int(stats[2]) == 0
            assert np.array_equal(_bits(want), _bits(e.host_depth(got))), ("depth", f, late)
            assert np.array_equal(e.dvb(), r.dvb), ("dvb", f, late)
            draw_sets.append(np.unique(cmds["drawId"][: int(r.dccb[0])]))
        assert len(np.intersect1d(*draw_sets)) == 0, f
        late_draws += len(draw_sets[1])
        gt.dvb[:] = 1
        gt.cull(s.cull_data(culling=False, occlusion=False, cluster_occlusion=False), late=False)
        all_cmds = gt.read_task_commands(int(gt.dccb[1]) * 64)
        cib, ccb, _ = _all_clusters(all_cmds, int(gt.dccb[0]))
        bs = refshader_lib.MeshStage(gt, vertices, meshletdata, proj, threads=4)
        rec, pos, tri = bs.run(cd, cib=cib, ccb=ccb, dcb=gt.dcb)
        truth = np.zeros_like(want)
        bs.rasterize(rec, pos, tri, truth)
        assert np.array_equal(_bits(truth), _bits(want)), ("brute force", f, int((truth != want).sum()))
        assert (truth > 0).mean() > 0.05
    assert late_draws > 0
    e.close()


class _EmuLoop:
    """the emulated product path with the switch off, as _closed_loop drives it"""

    def __init__(self, s):
        self.p = _EmuPath(s.meshes, s.meshlets, s.draws, *s.screen, threads=4)
        self.p.set_visibility_bits(s.visibility_bits)
        self.p.set_task_cull(0)

    def new_depth(self):
        return np.zeros((self.p.depth_height, self.p.depth_width), np.float32)

    def host_depth(self, d):
        return d

    def pyramid(self, d):
        self.p.pyramid(d)

    def cull(self, cd, late):
        self.p.cull(cd, late)

    def dccb(self):
        return self.p.dccb

    def dvb(self):
        return self.p.dvb

    def task_commands(self):
        return self.p.read_task_commands(int(self.p.dccb[1]) * 64)

    def render_clusters(self, cd, late):
        self.p.render_clusters(cd, late)

    def raster(self, cd, proj, vertices, meshletdata, got):
        return self.p.raster_depth(cd, proj, vertices, meshletdata, got)

    def raster_tasks(self, cd, late, proj, vertices, meshletdata, got, n):
        payloads, emit = _task_buffers(n)
        self.p.task_shading(cd, late, payloads, emit)
        return self.p.raster_depth_tasks(cd, proj, payloads, emit, vertices, meshletdata, got)

    def close(self):
        self.p.close()


@needs_refshader
@pytest.mark.parametrize("mode", ["clusters", "tasks"])
def test_closed_loop_with_task_cull_off_on_emulated_produced_depth(golden_dir, mode):
    _closed_loop(golden_dir, mode, 5, _EmuLoop, MOVING)


def test_switching_back_on_restores_the_default_path(golden_dir):
    """nvc_set_task_cull(ctx, 1) after 0: drawcull, the cluster pass and the task pass on the same inputs give the default path's
    output; with the switch off they give something else"""
    screen = (320, 240)
    s, _, _ = _scene(golden_dir)
    cd = s.cull_data()
    depth = _depth(screen)
    dvb = (np.random.default_rng(5).random(len(s.draws)) < 0.5).astype(np.uint32)
    mvb = None
    results = []
    for switch in (None, 0, 1):
        p = _ModesEmuPath(s.meshes, s.meshlets, s.draws, *screen, threads=4) if switch is None else _EmuPath(s.meshes, s.meshlets, s.draws, *screen, threads=4)
        p.set_visibility_bits(s.visibility_bits)
        if switch is not None:
            p.set_task_cull(0)
            p.set_task_cull(switch)
        mvb = np.random.default_rng(6).integers(0, 2**32, len(p.mvb), dtype=np.uint64).astype(np.uint32) if mvb is None else mvb
        p.pyramid(depth)
        p.dvb[:] = dvb
        p.mvb[:] = mvb
        p.cull(cd, True)
        p.render_clusters(cd, True)
        n = int(p.dccb[1]) * 64
        payloads, emit = _task_buffers(n)
        p.mvb[:] = mvb
        p.task_shading(cd, True, payloads, emit)
        results.append((_sorted_cmds(p, True), np.sort(p.cib[: int(p.ccb[0])]), p.ccb.copy(), p.mvb.copy(), payloads, emit, p.dvb.copy()))
        p.close()
    default, off, on = results
    same = lambda a, b: all(np.array_equal(x, y) for x, y in zip(a, b))  # noqa: E731
    assert same(default, on) and not same(default, off)
    assert not np.array_equal(default[0], off[0]) and not np.array_equal(default[1], off[1]) and not np.array_equal(default[3], off[3])


# ---- GPU tier --------------------------------------------------------------------------------------------------------------------


class _DeviceLoop:
    """the CUDA path (VisibilityPath) with the switch off, as _closed_loop drives it"""

    def __init__(self, s):
        import torch
        from niagara_b200.path import VisibilityPath

        self.torch = torch
        self.g = VisibilityPath(s.meshes, s.meshlets, s.draws, *s.screen)
        self.g.set_visibility_bits(s.visibility_bits)
        self.g.set_task_cull(False)
        self.stats = torch.zeros(4, dtype=torch.int32, device="cuda")
        self.vb = self.md = None

    def new_depth(self):
        return self.torch.zeros((self.g.depth_height, self.g.depth_width), dtype=self.torch.float32, device="cuda")

    def host_depth(self, d):
        return d.cpu().numpy()

    def pyramid(self, d):
        self.g.pyramid(d)

    def cull(self, cd, late):
        self.g.cull(cd, late)

    def dccb(self):
        return self.g.dccb.cpu().numpy().astype(np.uint32)

    def dvb(self):
        return self.g.dvb.cpu().numpy().astype(np.uint32)

    def task_commands(self):
        return self.g.read_task_commands(int(self.g.dccb[1].item()) * 64)

    def render_clusters(self, cd, late):
        self.g.render_clusters(cd, late)

    def _geometry(self, vertices, meshletdata):
        if self.vb is None:
            self.vb = self.torch.from_numpy(np.ascontiguousarray(vertices)).cuda()
            self.md = self.torch.from_numpy(np.ascontiguousarray(meshletdata, dtype=np.uint32).view(np.int32)).cuda()

    def raster(self, cd, proj, vertices, meshletdata, got):
        self._geometry(vertices, meshletdata)
        self.g.raster_depth(cd, proj, self.vb, self.md, got, self.stats)
        self.torch.cuda.synchronize()
        return self.stats.cpu().numpy().astype(np.uint32)

    def raster_tasks(self, cd, late, proj, vertices, meshletdata, got, n):
        torch = self.torch
        self._geometry(vertices, meshletdata)
        gp = torch.zeros((max(n, 1), 64), dtype=torch.int32, device="cuda")
        ge = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
        self.g.task_shading(cd, late, gp, ge)
        self.g.raster_depth_tasks(cd, proj, gp, ge, self.vb, self.md, got, self.stats)
        torch.cuda.synchronize()
        return self.stats.cpu().numpy().astype(np.uint32)

    def close(self):
        self.g.close()


@pytest.mark.gpu
@needs_refshader
@pytest.mark.parametrize("mode", ["clusters", "tasks"])
def test_closed_loop_with_task_cull_off_on_device_produced_depth(golden_dir, mode):
    _closed_loop(golden_dir, mode, 5, _DeviceLoop, MOVING, screen=(512, 384), kittens=300)


def _c4_commands():
    """a C4-size scene (1 M draws) and its early drawcull on the device with the switch off"""
    import torch
    from niagara_b200 import scenes
    from niagara_b200.path import VisibilityPath

    s = scenes.config4_scene()
    g = VisibilityPath(s.meshes, s.meshlets, s.draws, *s.screen)
    g.set_visibility_bits(s.visibility_bits)
    g.set_task_cull(False)
    g.dvb.fill_(1)
    cd = s.cull_data()
    g.cull(cd, False)
    torch.cuda.synchronize()
    ncmd = int(g.dccb[1].item()) * 64
    return s, g, cd, ncmd, g.read_task_commands(ncmd)


@pytest.mark.gpu
def test_c4_frame_with_task_cull_off_is_the_expansion_of_its_commands():
    """1 M draws: the cluster set and every payload entry / emit count equal a numpy expansion of the command array, and mvb is not
    written"""
    import torch

    s, g, cd, ncmd, cmds = _c4_commands()
    mvb = g.mvb.clone()
    g.render_clusters(cd, False)
    torch.cuda.synchronize()
    want = _expand(cmds, ncmd)
    count = int(g.ccb[0].item())
    assert count == len(want) > 1_000_000
    assert np.array_equal(np.sort(g.cib[:count].cpu().numpy().astype(np.uint32)), np.sort(want))
    pad = (count + 255) // 256 * 256
    assert (g.cib[count:pad].cpu().numpy().astype(np.uint32) == 0xFFFFFFFF).all()
    assert g.ccb.cpu().numpy().astype(np.uint32).tolist() == [count, 16, pad // 256, 16]
    gp = torch.zeros((ncmd, 64), dtype=torch.int32, device="cuda")
    ge = torch.zeros(ncmd, dtype=torch.int32, device="cuda")
    g.task_shading(cd, True, gp, ge)
    torch.cuda.synchronize()
    xp, xe = _task_expected(cmds, ncmd)
    assert np.array_equal(gp.cpu().numpy().astype(np.uint32), xp) and np.array_equal(ge.cpu().numpy().astype(np.uint32), xe)
    assert torch.equal(g.mvb, mvb)
    g.close()


@pytest.mark.gpu
def test_graph_captured_with_task_cull_off_keeps_passing_through():
    """a CUDA graph of the cluster and task passes captured with the switch off still produces pass-through output when replayed after
    the switch is turned on"""
    import torch

    s, g, cd, ncmd, cmds = _c4_commands()
    gp = torch.zeros((ncmd, 64), dtype=torch.int32, device="cuda")
    ge = torch.zeros(ncmd, dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # warm-up outside the capture
        g.render_clusters(cd, False)
        g.task_shading(cd, False, gp, ge)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g.render_clusters(cd, False)
        g.task_shading(cd, False, gp, ge)
    g.set_task_cull(True)
    g.cib.fill_(0)
    gp.fill_(0)
    ge.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    want = _expand(cmds, ncmd)
    count = int(g.ccb[0].item())
    assert count == len(want) and np.array_equal(np.sort(g.cib[:count].cpu().numpy().astype(np.uint32)), np.sort(want))
    xp, xe = _task_expected(cmds, ncmd)
    assert np.array_equal(gp.cpu().numpy().astype(np.uint32), xp) and np.array_equal(ge.cpu().numpy().astype(np.uint32), xe)
    # and an uncaptured call now culls again (the early pass keeps only meshlets whose visibility bit is set: none here)
    g.render_clusters(cd, False)
    torch.cuda.synchronize()
    assert int(g.ccb[0].item()) < len(want)
    del graph
    g.close()
