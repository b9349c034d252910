"""CPU-only: the PRODUCT's CUDA kernels executed under the SIMT emulation of tests/cuda_emu (nvc_kernels.cu + nvc_api.cu compiled
by g++, same C ABI, host pointers) against the oracle — the -m gpu parity suite in miniature for a machine without a GPU.  It checks
kernel logic (indexing, block / warp scans, flattening, compaction, staging, epilogues, arithmetic order); what only hardware can
show (memory model, timing) stays with the GPU tests."""
import ctypes
import os

import numpy as np
import pytest

import emu_lib
import oracle_lib
from niagara_b200 import host, layout, scenes


def _pair(s, threads=4, **kw):
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *s.screen, threads=threads, **kw)
    e = emu_lib.EmuPath(s.meshes, s.meshlets, s.draws, *s.screen, **kw)
    o.set_visibility_bits(s.visibility_bits)
    e.set_visibility_bits(s.visibility_bits)
    return o, e


def _compare_draw(o, e, task, what):
    assert np.array_equal(o.dccb, e.dccb), (what, o.dccb, e.dccb)
    if task:
        n = int(o.dccb[1]) * 64
        assert np.array_equal(oracle_lib.sorted_commands(o.read_task_commands(n)), oracle_lib.sorted_commands(e.read_task_commands(n))), what
    else:
        n = int(o.dccb[0])
        assert np.array_equal(oracle_lib.sorted_commands(o.read_draw_commands(n)), oracle_lib.sorted_commands(e.read_draw_commands(n))), what
    assert np.array_equal(o.dvb, e.dvb), what


def _compare_clusters(o, e, what):
    assert np.array_equal(o.ccb, e.ccb), (what, o.ccb, e.ccb)
    n = int(o.ccb[0])
    oc, ec = o.read_task_commands(int(o.dccb[1]) * 64), e.read_task_commands(int(e.dccb[1]) * 64)
    assert np.array_equal(oracle_lib.cluster_pairs(o.read_cluster_indices(n), oc), oracle_lib.cluster_pairs(e.read_cluster_indices(n), ec)), what
    pad = (n + 255) // 256 * 256
    assert (e.cib[n:pad] == 0xFFFFFFFF).all(), what
    assert np.array_equal(o.mvb, e.mvb), what


def _frames(s, frames=2, toggles=None, cluster_backface=True, cameras=None, post_passes=False, **kw):
    o, e = _pair(s, **kw)
    emitted = 0
    for f in range(frames):
        if cameras:
            s.camera = cameras[f % len(cameras)]
        cd = s.cull_data(**(toggles or {}))
        passes = [(False, 0), (True, 0)] + ([(True, 1)] if post_passes else [])
        for late, post in passes:
            if late and post == 0:
                o.pyramid(s.depth)
                e.pyramid(s.depth)
                assert np.array_equal(o.pyramid_texels.view(np.uint32), e.pyramid_texels.view(np.uint32)), ("pyramid", f)
            o.cull(cd, late, post_pass=post)
            e.cull(cd, late, post_pass=post)
            _compare_draw(o, e, o.mesh_shading, ("cull", f, late, post))
            if o.mesh_shading:
                o.render_clusters(cd, late, post_pass=post, cluster_backface=cluster_backface)
                e.render_clusters(cd, late, post_pass=post, cluster_backface=cluster_backface)
                _compare_clusters(o, e, ("clusters", f, late, post))
                emitted += int(o.ccb[0])
            else:
                emitted += int(o.dccb[0])
    e.close()
    return emitted


def _kp(golden_dir, n, screen=(640, 480)):
    return scenes.instanced_scene(os.path.join(golden_dir, "kitten_pirate.nvcg"), n, screen=screen)


@pytest.mark.parametrize("toggles", [dict(), dict(lod=False), dict(culling=False), dict(occlusion=False), dict(cluster_occlusion=False), dict(debug_lod_step=3)])
def test_two_phase_frames(golden_dir, toggles):
    assert _frames(_kp(golden_dir, 5000), frames=2, toggles=toggles) > 500


@pytest.mark.parametrize("backface", [False, None])
def test_cluster_backface_wiring(golden_dir, backface):
    _frames(_kp(golden_dir, 3000), cluster_backface=backface)


def test_moving_camera_and_post_pass(golden_dir):
    s = _kp(golden_dir, 6000, screen=(800, 600))
    s.draws["postPass"][::5] = 1
    cams = [host.make_camera((0, 0, 0)), host.make_camera((12, -4, 9), host.quat_from_axis_angle((0, 1, 0), 0.35)), host.make_camera((25, 3, -14), host.quat_from_axis_angle((0.1, 1, 0), 0.9))]
    assert _frames(s, frames=3, cameras=cams, post_passes=True) > 500


def test_draw_path(golden_dir):
    assert _frames(_kp(golden_dir, 8000), frames=2, toggles=dict(mesh_shading=False, cluster_occlusion=False), mesh_shading=False) > 100


def test_without_prepared_mesh_heads(golden_dir):
    _frames(_kp(golden_dir, 3000), prepare_meshes=False) if False else None
    s = _kp(golden_dir, 3000)
    o, _ = _pair(s)
    e = emu_lib.EmuPath(s.meshes, s.meshlets, s.draws, *s.screen, prepare_meshes=False)
    e.set_visibility_bits(s.visibility_bits)
    cd = s.cull_data()
    for late in (False, True):
        if late:
            o.pyramid(s.depth)
            e.pyramid(s.depth)
        o.cull(cd, late)
        e.cull(cd, late)
        _compare_draw(o, e, True, late)


def test_synthetic_c4_and_c2():
    """uniform meshlet counts (the multiply-high flatten), 4-LOD meshes with several task groups per draw"""
    assert _frames(scenes.config4_scene(draw_count=20000, screen=(1024, 1024)), frames=2, cmd_capacity=40000) > 10000
    assert _frames(scenes.config2_scene(draw_count=30000, num_meshes=128, screen=(512, 512)), frames=2) > 100


@pytest.mark.parametrize("size", [(64, 64), (100, 60), (30, 17), (129, 257), (2, 2), (1, 1), (256, 8), (1920, 1080), (1000, 3)])
def test_pyramid_sizes(size):
    w, h = size
    depth = np.random.default_rng(w * 7 + h).random((h, w), dtype=np.float32)
    blank = (np.zeros(1, layout.MESH_DTYPE), np.zeros(1, layout.MESHLET_DTYPE), np.zeros(1, layout.MESHDRAW_DTYPE))
    o = oracle_lib.OraclePath(*blank, w, h)
    e = emu_lib.EmuPath(*blank, w, h, prepare_meshes=False)
    o.pyramid(depth)
    e.pyramid(depth)
    assert np.array_equal(o.pyramid_texels.view(np.uint32), e.pyramid_texels.view(np.uint32))


@pytest.mark.parametrize("size", [(64, 64), (100, 60), (30, 17), (129, 257), (2, 2), (1, 1), (256, 8), (1920, 1080), (1000, 3), (4096, 16)])
def test_footprint_image(size):
    """the derived footprint image (nvc_prepare_hiz): every entry of every mip = min of the clamped 2 x 2 texel footprint, for
    pyramids whose rows take the 16-byte path of footprint_kernel and for shapes that do not (widths 1, 2, 3 mod 4, tiny mips)"""
    import ctypes

    w, h = size
    depth = np.random.default_rng(w * 11 + h).random((h, w), dtype=np.float32)
    blank = (np.zeros(1, layout.MESH_DTYPE), np.zeros(1, layout.MESHLET_DTYPE), np.zeros(1, layout.MESHDRAW_DTYPE))
    e = emu_lib.EmuPath(*blank, w, h, prepare_meshes=False)
    e.pyramid(depth)
    image, first, total = ctypes.c_void_p(), ctypes.c_uint32(), ctypes.c_uint32()
    offsets = (ctypes.c_uint32 * 16)()
    assert e.emu.nvc_hiz_footprints(e.ctx, ctypes.byref(image), ctypes.byref(first), offsets, ctypes.byref(total)) == 0
    assert image.value and total.value > 0
    fp = np.ctypeslib.as_array(ctypes.cast(image.value, ctypes.POINTER(ctypes.c_float)), shape=(total.value,))  # emulated device memory is host memory
    hz = e.hiz
    for l in range(first.value, hz.levels):
        lw, lh = max(1, hz.width >> l), max(1, hz.height >> l)
        t = e.pyramid_texels[hz.level_offset[l] : hz.level_offset[l] + lw * lh].reshape(lh, lw)
        pad = np.pad(t, 1, mode="edge")  # texel (-1) = texel 0, texel w = texel w - 1
        want = np.minimum(np.minimum(pad[:-1, :-1], pad[:-1, 1:]), np.minimum(pad[1:, :-1], pad[1:, 1:]))  # (lh + 1, lw + 1)
        pitch = (lw + 4) & ~3
        got = fp[offsets[l] : offsets[l] + pitch * (lh + 1)].reshape(lh + 1, pitch)[:, : lw + 1]
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (size, l)
    e.close()


def test_tiny_and_empty_inputs(golden_dir):
    _frames(_kp(golden_dir, 1))
    s = _kp(golden_dir, 3)
    o, e = _pair(s)
    cd = s.cull_data()
    cd.drawCount = 0
    for late in (False, True):
        o.cull(cd, late)
        e.cull(cd, late)
        _compare_draw(o, e, True, late)
        o.render_clusters(cd, late)
        e.render_clusters(cd, late)
        _compare_clusters(o, e, late)


def test_overflow_limits(golden_dir):
    """TASK_WGLIMIT / CLUSTER_LIMIT drop-and-clamp: counters keep counting, writes stop, group counts clamp"""
    s = _kp(golden_dir, 4000)
    cd = s.cull_data(occlusion=False, cluster_occlusion=False)
    o, e = _pair(s, task_wglimit=64, cluster_limit=512)
    o.dvb[:] = 1
    e.dvb[:] = 1
    o.cull(cd, False)
    e.cull(cd, False)
    assert np.array_equal(o.dccb, e.dccb) and int(o.dccb[0]) > 64
    # WHICH commands land below the limit depends on the order of the counter's atomics (unspecified in the reference too; the
    # persistent drawcull walks tiles in another order than the sequential checker): everything written must be a command of
    # the unlimited run, and the cluster pass is compared on the same 64 commands
    o_full, _ = _pair(s)
    o_full.dvb[:] = 1
    o_full.cull(cd, False)
    allowed = set(map(tuple, o_full.read_task_commands(int(o_full.dccb[0])).tolist()))
    assert all(tuple(c) in allowed for c in e.read_task_commands(64).tolist())
    o.dcb[: 64 * 20] = e.dcb[: 64 * 20]
    o.render_clusters(cd, False)
    e.render_clusters(cd, False)
    assert np.array_equal(o.ccb, e.ccb)


def test_taskcull_payloads(golden_dir):
    s = _kp(golden_dir, 3000)
    o, e = _pair(s)
    cd = s.cull_data()
    for f in range(2):
        for late in (False, True):
            if late:
                o.pyramid(s.depth)
                e.pyramid(s.depth)
            o.cull(cd, late)
            e.cull(cd, late)
            n = int(o.dccb[1]) * 64
            op, oe = np.zeros((max(n, 1), 64), np.uint32), np.zeros(max(n, 1), np.uint32)
            ep, ee = np.zeros((max(n, 1), 64), np.uint32), np.zeros(max(n, 1), np.uint32)
            o.task_shading(cd, late, op, oe, cluster_backface=True)
            e.task_shading(cd, late, ep, ee, cluster_backface=True)
            ot, et = o.read_task_commands(n), e.read_task_commands(n)

            def table(cmds, payloads, counts):
                return {tuple(cmds[i].tolist()): tuple(sorted(int(v) >> 24 for v in payloads[i][: counts[i]])) for i in range(n) if cmds["taskCount"][i]}

            assert table(ot, op, oe) == table(et, ep, ee)
            assert np.array_equal(o.mvb, e.mvb)


def test_hostile_inputs(golden_dir):
    import warnings

    import hostile

    s = hostile.hostile_scene(golden_dir, 6000)
    cams = [host.make_camera((0, 0, 0)), host.make_camera((5, 2, -3), host.quat_from_axis_angle((0.3, 1, 0), 0.9))]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _frames(s, frames=2, cameras=cams)
        _frames(s, frames=2, toggles=dict(culling=False))


def test_kitten_config4_and_moving_camera_frames(golden_dir):
    """the cluster kernels' item -> command mappings on the kitten / pirate and C4 scenes and on frames with a moving camera,
    where the early pass sees sparse, changing visibility masks"""
    assert _frames(_kp(golden_dir, 3000)) > 300
    assert _frames(scenes.config4_scene(draw_count=6000, screen=(512, 512)), cmd_capacity=12000) > 3000
    cams = [host.make_camera((0, 0, 0)), host.make_camera((12, -4, 9), host.quat_from_axis_angle((0, 1, 0), 0.35)), host.make_camera((25, 3, -14), host.quat_from_axis_angle((0.1, 1, 0), 0.9))]
    assert _frames(_kp(golden_dir, 2500, screen=(800, 600)), frames=4, cameras=cams) > 300
    # task commands with taskCount 0 between non-empty ones (drawcull never writes them): without visibility tracking the
    # filtered kernel then maps items to commands by the scan search
    s = _kp(golden_dir, 2500)
    cd = s.cull_data(cluster_occlusion=False)
    o, e = _pair(s)
    for p in (o, e):
        p.pyramid(s.depth)
        p.cull(cd, True)
    _compare_draw(o, e, True, "empty commands")
    for p in (o, e):
        p.dcb.view(np.uint32)[2 : 5 * int(p.dccb[0]) : 15] = 0  # taskCount of every third command
    o.render_clusters(cd, True, cluster_backface=True)
    e.render_clusters(cd, True, cluster_backface=True)
    _compare_clusters(o, e, "empty commands")
    assert 0 < int(e.ccb[0]) < int(np.minimum(e.dcb.view(np.uint32)[2 : 5 * int(e.dccb[0]) : 5], 64).sum())


def test_tma_staged_hiz(golden_dir):
    """nvc_set_hiz_staging: the late cluster pass reads the coarse mips from the staged shared-memory copy"""
    s = _kp(golden_dir, 3000)
    o, e = _pair(s)
    assert e.emu.nvc_set_hiz_staging(e.ctx, 5461) == 0
    cd = s.cull_data()
    for late in (False, True):
        if late:
            o.pyramid(s.depth)
            e.pyramid(s.depth)
        o.cull(cd, late)
        e.cull(cd, late)
        o.render_clusters(cd, late, cluster_backface=True)
        e.render_clusters(cd, late, cluster_backface=True)
        _compare_clusters(o, e, late)


def test_decode_update_and_cook(golden_dir):
    """the smaller kernels: consumer walk, animated-draw scatter, meshlet bounds"""
    s = _kp(golden_dir, 2500)
    o, e = _pair(s)
    cd = s.cull_data()
    o.frame(cd, s.depth, cluster_backface=True)
    e.frame(cd, s.depth, cluster_backface=True)
    slots = int(e.ccb[2]) * 256
    rec, stats = np.zeros((max(slots, 1), 4), np.uint32), np.zeros(4, np.uint32)
    assert e.emu.nvc_decode_clusters(e.ctx, None, e.cib.ctypes.data, e.ccb.ctypes.data, e.dcb.ctypes.data, e.meshlets.ctypes.data, rec.ctypes.data, stats.ctypes.data) == 0
    _, ostats = o.decode_clusters()
    assert np.array_equal(stats, ostats) and stats[2] == 0

    draws = s.draws.copy()
    idx = np.array([5, 17, 2400, 99999], np.uint32)
    val = np.zeros(4, layout.MESHDRAW_DTYPE)
    val["scale"] = [1.5, 2.5, 3.5, 4.5]
    assert e.emu.nvc_update_draws(e.ctx, None, draws.ctypes.data, len(draws), idx.ctypes.data, val.ctypes.data, 4) == 0
    want = s.draws.copy()
    want[idx[:3]] = val[:3]
    assert np.array_equal(draws, want)

    z = np.load(os.path.join(golden_dir, "kitten_cook.npz"))
    positions, data = z["positions"], z["meshletdata"]
    _, want_ml, _ = layout.load_nvcg(os.path.join(golden_dir, "kitten.nvcg"))
    vertices = np.zeros((len(positions), 8), np.uint16)
    vertices[:, :3] = positions
    got = want_ml.copy()
    got.view(np.uint8).reshape(len(got), 24)[:, :12] = 0xCD
    rej = np.full(1, 9, np.uint32)
    assert e.emu.nvc_cook_meshlet_bounds(e.ctx, None, vertices.ctypes.data, len(vertices), data.ctypes.data, len(data), got.ctypes.data, len(got), rej.ctypes.data) == 0
    assert rej[0] == 0 and np.array_equal(got, want_ml)
    e.close()


def _guarded(arr):
    """A copy of `arr` that ends exactly at an inaccessible page: any read or write past its end faults (the CPU counterpart of
    compute-sanitizer's memcheck for the emulated kernels)."""
    import mmap

    page = mmap.PAGESIZE
    raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    n = max(len(raw), 1)
    span = (n + page - 1) // page * page
    m = mmap.mmap(-1, span + page, flags=mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS, prot=mmap.PROT_READ | mmap.PROT_WRITE)
    libc = ctypes.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
    base = ctypes.addressof(ctypes.c_char.from_buffer(m))
    assert libc.mprotect(base + span, page, 0) == 0, ctypes.get_errno()  # PROT_NONE
    view = np.frombuffer(m, dtype=np.uint8, count=n, offset=span - n)
    view[: len(raw)] = raw
    out = view[: len(raw)].view(arr.dtype).reshape(arr.shape) if len(raw) else view[:0].view(arr.dtype)
    _guarded.keep.append(m)
    return out


_guarded.keep = []


def test_no_access_past_buffer_ends(golden_dir):
    """Every device buffer of the passes (draws, meshes, meshlets, dvb, dcb, dccb, cib, ccb, mvb, depth, pyramid) ends at a
    PROT_NONE page while the emulated kernels run two frames + the small kernels: an overrun would be a SIGSEGV."""
    s = _kp(golden_dir, 2047, screen=(333, 217))  # odd sizes: ragged last blocks / tiles
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *s.screen, threads=4)
    o.set_visibility_bits(s.visibility_bits)
    e = emu_lib.EmuPath(s.meshes, s.meshlets, s.draws, *s.screen, prepare_meshes=False)
    e.set_visibility_bits(s.visibility_bits)
    for name in ("meshes", "meshlets", "draws", "dvb", "dcb", "dccb", "cib", "ccb", "mvb", "pyramid_texels"):
        setattr(e, name, _guarded(getattr(e, name)))
    e.hiz.texels = e.pyramid_texels.ctypes.data
    assert e.emu.nvc_prepare_meshes(e.ctx, None, e.meshes.ctypes.data, len(e.meshes)) == 0
    depth = _guarded(s.depth)
    cd = s.cull_data()
    for f in range(2):
        for late in (False, True):
            if late:
                o.pyramid(s.depth)
                e.pyramid(depth)
            o.cull(cd, late)
            e.cull(cd, late)
            _compare_draw(o, e, True, (f, late))
            o.render_clusters(cd, late, cluster_backface=True)
            e.render_clusters(cd, late, cluster_backface=True)
            _compare_clusters(o, e, (f, late))
    n = int(e.dccb[1]) * 64
    payloads, emit = _guarded(np.zeros((max(n, 1), 64), np.uint32)), _guarded(np.zeros(max(n, 1), np.uint32))
    e.task_shading(cd, True, payloads, emit, cluster_backface=True)
    slots = int(e.ccb[2]) * 256
    rec, stats = _guarded(np.zeros((max(slots, 1), 4), np.uint32)), _guarded(np.zeros(4, np.uint32))
    assert e.emu.nvc_decode_clusters(e.ctx, None, e.cib.ctypes.data, e.ccb.ctypes.data, e.dcb.ctypes.data, e.meshlets.ctypes.data, rec.ctypes.data, stats.ctypes.data) == 0
    idx, val = _guarded(np.array([3, 2046, 5000], np.uint32)), _guarded(np.zeros(3, layout.MESHDRAW_DTYPE))
    assert e.emu.nvc_update_draws(e.ctx, None, e.draws.ctypes.data, len(e.draws), idx.ctypes.data, val.ctypes.data, 3) == 0
    z = np.load(os.path.join(golden_dir, "kitten_cook.npz"))
    _, want_ml, _ = layout.load_nvcg(os.path.join(golden_dir, "kitten.nvcg"))
    vertices = np.zeros((len(z["positions"]), 8), np.uint16)
    vertices[:, :3] = z["positions"]
    gv, gd, gm = _guarded(vertices), _guarded(z["meshletdata"]), _guarded(want_ml.copy())
    assert e.emu.nvc_cook_meshlet_bounds(e.ctx, None, gv.ctypes.data, len(gv), gd.ctypes.data, len(gd), gm.ctypes.data, len(gm), None) == 0
    assert np.array_equal(gm, want_ml)
    e.close()
