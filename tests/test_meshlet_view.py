"""CPU-only: the prepared meshlet cull view (nvc_prepare_meshlets) under the kernel emulation.  The cluster passes read the
12 cull bytes of every meshlet either from the view's two dense arrays or from the 24-byte records; both must give the
oracle's results bit for bit, in the filtered and the exact kernel, for cluster-index and task-shading output, and a pass
whose Meshlet[] pointer is not the prepared one must read the records."""
import ctypes
import os

import numpy as np
import pytest

import emu_lib
import oracle_lib
from niagara_b200 import layout, scenes
from test_kernels_emulated import _compare_clusters, _compare_draw, _guarded


def _kitten(golden_dir, n=2500):
    return scenes.instanced_scene(os.path.join(golden_dir, "kitten_pirate.nvcg"), n, screen=(640, 480))


def _c4():
    return scenes.config4_scene(draw_count=6000, screen=(512, 512))


SCENES = {"kitten": (_kitten, {}), "c4": (lambda golden_dir: _c4(), {"cmd_capacity": 12000})}


def _prepare(e, meshlets=None):
    m = e.meshlets if meshlets is None else meshlets
    assert e.emu.nvc_prepare_meshlets(e.ctx, None, m.ctypes.data, len(m)) == 0


def _paths(s, view, **kw):
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *s.screen, threads=4, **kw)
    e = emu_lib.EmuPath(s.meshes, s.meshlets, s.draws, *s.screen, **kw)
    if view:
        _prepare(e)
    o.set_visibility_bits(s.visibility_bits)
    e.set_visibility_bits(s.visibility_bits)
    return o, e


def _task_table(p, n, payloads, counts):
    cmds = p.read_task_commands(n)
    return {tuple(cmds[i].tolist()): tuple(sorted(int(v) >> 24 for v in payloads[i][: counts[i]])) for i in range(n) if cmds["taskCount"][i]}


def _frame(o, e, s, cd, what, task=False):
    """one two-phase frame on both paths, every output compared after every pass; returns the clusters emitted"""
    emitted = 0
    for late in (False, True):
        if late:
            o.pyramid(s.depth)
            e.pyramid(s.depth)
            assert np.array_equal(o.pyramid_texels.view(np.uint32), e.pyramid_texels.view(np.uint32)), what
        o.cull(cd, late)
        e.cull(cd, late)
        _compare_draw(o, e, True, (what, late))
        if task:
            n = int(o.dccb[1]) * 64
            op, oe = np.zeros((max(n, 1), 64), np.uint32), np.zeros(max(n, 1), np.uint32)
            ep, ee = np.zeros((max(n, 1), 64), np.uint32), np.zeros(max(n, 1), np.uint32)
            o.task_shading(cd, late, op, oe, cluster_backface=True)
            e.task_shading(cd, late, ep, ee, cluster_backface=True)
            assert _task_table(o, n, op, oe) == _task_table(e, n, ep, ee), (what, late)
            assert np.array_equal(o.mvb, e.mvb), (what, late)
            emitted += int(oe[:n].sum())
        else:
            o.render_clusters(cd, late, cluster_backface=True)
            e.render_clusters(cd, late, cluster_backface=True)
            _compare_clusters(o, e, (what, late))
            emitted += int(o.ccb[0])
    return emitted


@pytest.mark.parametrize("scene", sorted(SCENES))
@pytest.mark.parametrize("view", [True, False])
@pytest.mark.parametrize("cluster_filter", [1, 0])
def test_two_phase_frames_with_and_without_view(golden_dir, scene, view, cluster_filter):
    """filtered (1) and exact (0) cluster kernel, meshlet view prepared or absent: two frames, every pass bit-exact"""
    make, kw = SCENES[scene]
    s = make(golden_dir)
    o, e = _paths(s, view, **kw)
    assert e.emu.nvc_set_cluster_filter(e.ctx, cluster_filter) == 0
    cd = s.cull_data()
    assert sum(_frame(o, e, s, cd, (scene, view, cluster_filter, f)) for f in range(2)) > 300
    e.close()


@pytest.mark.parametrize("view", [True, False])
def test_task_shading_with_and_without_view(golden_dir, view):
    s = _kitten(golden_dir)
    o, e = _paths(s, view)
    cd = s.cull_data()
    assert sum(_frame(o, e, s, cd, (view, f), task=True) for f in range(2)) > 300
    e.close()


def test_other_meshlet_pointer_reads_the_records(golden_dir):
    """the view is keyed by the Meshlet[] pointer it was built from: a pass over another buffer must not use it.  The view is
    built from a copy whose cull bytes are garbage; passes over the real records must still match the oracle."""
    s = _kitten(golden_dir)
    o, e = _paths(s, False)
    decoy = s.meshlets.copy()
    decoy.view(np.uint8).reshape(len(decoy), layout.MESHLET_DTYPE.itemsize)[:, :12] = 0x7B
    _prepare(e, decoy)
    cd = s.cull_data()
    _frame(o, e, s, cd, "records")
    _frame(o, e, s, cd, "records", task=True)
    e.close()


@pytest.mark.parametrize("cluster_filter", [1, 0])
def test_prepared_passes_read_only_the_view(golden_dir, cluster_filter):
    """with the view prepared, the cluster passes (filter, exact fallback, exact kernel, task shading) take the cull bytes from
    it alone: overwriting the records' bytes 0-11 afterwards must not change any result"""
    s = _kitten(golden_dir)
    o, e = _paths(s, False)
    e.meshlets = s.meshlets.copy()
    _prepare(e)
    e.meshlets.view(np.uint8).reshape(len(e.meshlets), layout.MESHLET_DTYPE.itemsize)[:, :12] = 0x7B
    assert e.emu.nvc_set_cluster_filter(e.ctx, cluster_filter) == 0
    cd = s.cull_data()
    _frame(o, e, s, cd, "view only")
    _frame(o, e, s, cd, "view only", task=True)
    e.close()


def test_release_and_prepare_again(golden_dir):
    """NULL releases the view (passes read the records), preparing again after a re-upload uses the new contents"""
    s = _kitten(golden_dir)
    o, e = _paths(s, True)
    cd = s.cull_data()
    _frame(o, e, s, cd, "prepared")
    assert e.emu.nvc_prepare_meshlets(e.ctx, None, None, 0) == 0
    _frame(o, e, s, cd, "released")
    # re-upload: the same buffer gets other contents (fewer meshlets pass), then the view is prepared again from it
    e.meshlets["cone_cutoff"] = np.int8(127)
    o.meshlets["cone_cutoff"] = np.int8(127)
    _prepare(e)
    _frame(o, e, s, cd, "prepared again")
    _prepare(e)  # prepare over a prepared view
    _frame(o, e, s, cd, "prepared twice")
    e.close()


def test_view_arrays_end_at_guard_page(golden_dir):
    """the view's two arrays are allocated exactly meshlet_count entries long, each ending at an inaccessible page; the source
    records end at one too.  Two frames of cluster passes, the exact kernel and task shading read through the view: a read
    past either array's end would fault."""
    s = _kitten(golden_dir, 2047)
    o, e = _paths(s, False)
    e.close()  # the same buffers, driven through a fresh context
    e.ctx = ctypes.c_void_p()
    limits = layout.Limits(e.limits.task_wglimit, e.limits.cluster_limit)
    assert e.emu.nvc_create(0, ctypes.byref(limits), ctypes.byref(e.ctx)) == 0
    assert e.emu.nvc_prepare_meshes(e.ctx, None, e.meshes.ctypes.data, len(e.meshes)) == 0
    assert e.emu.nvc_prepare_hiz(e.ctx, ctypes.byref(e.hiz)) == 0
    e.meshlets = _guarded(e.meshlets)
    e.emu.emu_guard_allocations(1)
    try:
        _prepare(e)
    finally:
        e.emu.emu_guard_allocations(0)
    assert e.emu.emu_guarded_live() == 2  # sphere[n] and cone[n]
    cd = s.cull_data()
    for f in range(2):
        _frame(o, e, s, cd, ("guarded", f))
    _frame(o, e, s, cd, "guarded task", task=True)
    assert e.emu.nvc_set_cluster_filter(e.ctx, 0) == 0
    _frame(o, e, s, cd, "guarded exact")
    e.close()
    assert e.emu.emu_guarded_live() == 0  # nvc_destroy freed both
