"""Every cull decision at its rounding boundary (tests/boundary_scenes.py): ladders of items at +-{0..4, 8, ..., 2^24} ulps of
the flip of each threshold comparison of the shaders.  Random scenes put almost no item within a few ulps of a threshold, so
a `>` written as `>=`, a `<= 2.0` written as `< 2.0`, a zero-weight texel counted by the MIN sampler or a filter margin that
is too small passes them; here each of those changes the verdict of an item.

CPU tier: the generator's scenes are hot (both outcomes within +-4 ulps of every flip, by the oracle), the checkers agree
(oracle, numpy restatement, the reference's own GLSL), and the product's kernels under the SIMT emulation reproduce the
oracle bit for bit in every kernel variant: filtered cluster kernel with and without the footprint image, the exact kernel
unstaged and staged, task shading with the filter on and off, drawcull's filtered occlusion stage (NVC_DRAW_FILTER=1),
backface and cluster occlusion off, the post pass.  -m gpu: the same matrix on the device."""
import ctypes
import functools
import time

import numpy as np
import pytest

import boundary_scenes as bs
import emu_lib
import numpy_ref as nr
import oracle_lib


@functools.lru_cache(maxsize=None)
def _families():
    t = time.perf_counter()
    fams = bs.generate(bases_per_setup=8)
    n = sum(len(s.draws) for v in fams.values() for s in v)
    print("boundary scenes: %d families, %d draws, generated in %.2f s" % (len(fams), n, time.perf_counter() - t))
    return fams


def _scenes():
    return [s for v in _families().values() for s in v]


# configuration: product-path options and what the frame loop does
CONFIGS = {
    "filtered": dict(),
    "filtered_no_footprint_image": dict(prepare_hiz=False),
    "exact": dict(cluster_filter=0),
    "exact_staged": dict(cluster_filter=0, stage_texels=5461),
    "no_backface": dict(backface=False),
    "no_cluster_occlusion": dict(toggles=dict(cluster_occlusion=False)),
    "post_pass": dict(post=True),
    "draw_filter": dict(draw_filter=True),
    "task_filtered": dict(task=True),
    "task_exact": dict(task=True, cluster_filter=0),
}
FILTERED = ("filtered", "filtered_no_footprint_image", "no_backface", "post_pass", "draw_filter", "task_filtered")


def _scene_for(s, cfg):
    draws = s.draws
    if cfg.get("post"):
        draws = s.draws.copy()
        draws["postPass"][::3] = 1
    return draws


def _verdicts(s):
    """The oracle's outcome per draw after the first frame's late pass: meshlet visible (cluster kind) or LOD index / 255."""
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *s.screen, threads=4)
    o.set_visibility_bits(s.visibility_bits)
    cd = s.cull_data()
    o.cull(cd, False)
    o.render_clusters(cd, False, cluster_backface=s.backface)
    o.pyramid(s.depth)
    o.cull(cd, True)
    if s.kind == "draw":
        return o.lod_out[: len(s.draws)].astype(np.int64)
    o.render_clusters(cd, True, cluster_backface=s.backface)
    n = int(o.ccb[0])
    pairs = oracle_lib.cluster_pairs(o.read_cluster_indices(n), o.read_task_commands(int(o.dccb[1]) * 64))
    out = np.zeros(len(s.draws), np.int64)
    out[(pairs >> np.uint64(32)).astype(np.int64)] = 1
    return out


def test_every_family_is_hot():
    """Within +-4 ulps of every flip the oracle's verdicts include both outcomes: the ladders sit on their boundaries."""
    fams = _families()
    assert set(fams) == set(bs.FAMILIES)
    total = 0
    for s in _scenes():
        v = _verdicts(s)
        total += len(s.draws)
        for b in range(len(s.bases)):
            inner = v[(s.base == b) & (np.abs(s.rung) <= bs.HOT)]
            assert len(np.unique(inner)) >= 2, (s.name, b, s.bases[b].indicator, s.bases[b].sweep, inner)
    assert total <= 60000


def test_numpy_ref_lod_distance_is_maxnum():
    """max(NaN, 0) = 0 in the LOD distance (IEEE maxNum, like the kernels and the oracle): a NaN draw position selects the
    LODs whose error is below threshold 0"""
    s = _families()["lod_edge"][0]
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *s.screen)
    o.set_visibility_bits(s.visibility_bits)
    cd = s.cull_data()
    pd = bs._pass_data(cd, 1)
    o.cull(cd, True)
    _, _, emit, lod = nr.drawcull_decisions(pd, True, s.draws, s.meshes, o.dvb * 0, None)
    assert np.isnan(s.draws["position"]).any(axis=1).all() and emit.all()
    assert np.array_equal(o.lod_out[: len(s.draws)], lod.astype(np.uint8))
    assert set(np.unique(lod)) == {0, 1}


def _pass_data(cd, for_drawcull, backface=None):
    return bs._pass_data(cd, for_drawcull, backface)


@pytest.mark.parametrize("toggles", [dict(), dict(cluster_occlusion=False)])
def test_oracle_agrees_with_numpy_restatement(toggles):
    """Two frames on every family: each per-draw and per-meshlet decision of the oracle (visible, LOD, dvb, mvb, counters)
    equals the numpy restatement's."""
    for s in _scenes():
        cd = s.cull_data(**toggles)
        o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *s.screen, threads=4)
        o.set_visibility_bits(s.visibility_bits)
        levels = s.setup.levels
        for frame in range(2):
            for late in (False, True):
                what = (s.name, frame, late)
                if late:
                    o.pyramid(s.depth)
                dvb_before = o.dvb.copy()
                reached, visible, emit, lod = nr.drawcull_decisions(_pass_data(cd, 1), late, s.draws, s.meshes, dvb_before, levels)
                o.cull(cd, late)
                assert np.array_equal(o.lod_out[: len(s.draws)] != 0xFF, emit), what
                assert np.array_equal(o.lod_out[: len(s.draws)][emit], lod[emit].astype(np.uint8)), what
                want_dvb = np.where(reached, visible.astype(np.uint32), dvb_before[: len(s.draws)]) if late else dvb_before
                assert np.array_equal(o.dvb[: len(want_dvb)], want_dvb), what
                cmds = o.read_task_commands(o.dccb[1] * 64)
                assert o.dccb[0] == emit.sum(), what  # one meshlet per LOD: one task command per emitted draw
                mvb_before = o.mvb.copy()
                cid, mgi, mi, mvi, vis, out = nr.cluster_decisions(_pass_data(cd, 0, s.backface), late, cmds[: o.dccb[0]], s.draws, s.meshlets, mvb_before, levels)
                o.render_clusters(cd, late, cluster_backface=s.backface)
                assert o.ccb[0] == out.sum(), what
                assert np.array_equal(o.read_cluster_indices(o.ccb[0]), (cid[out] | (mgi[out] << 24)).astype(np.uint32)), what
                if late and cd.clusterOcclusionEnabled == 1:
                    want = mvb_before.copy()
                    np.bitwise_or.at(want, mvi[vis] >> 5, np.uint32(1) << (mvi[vis] & 31).astype(np.uint32))
                    np.bitwise_and.at(want, mvi[~vis] >> 5, ~(np.uint32(1) << (mvi[~vis] & 31).astype(np.uint32)))
                    assert np.array_equal(o.mvb, want), what
                else:
                    assert np.array_equal(o.mvb, mvb_before), what


def test_oracle_agrees_with_reference_shaders():
    """Two frames on every family: the oracle against the reference's own GLSL, buffer for buffer."""
    import refshader_lib

    if not refshader_lib.available():
        pytest.skip("needs oracle/_ref/librefshader.so")
    for s in _scenes():
        cd = s.cull_data()
        o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *s.screen, threads=4)
        r = refshader_lib.RefShaderPath(s.meshes, s.meshlets, s.draws, *s.screen, threads=4)
        for p in (o, r):
            p.set_visibility_bits(s.visibility_bits)
        for frame in range(2):
            for late in (False, True):
                what = (s.name, frame, late)
                if late:
                    o.pyramid(s.depth)
                    r.pyramid(s.depth)
                    assert np.array_equal(o.pyramid_texels.view(np.uint32), r.pyramid_texels.view(np.uint32)), what
                o.cull(cd, late)
                r.cull(cd, late)
                _compare_draw(o, r, what)
                o.render_clusters(cd, late, cluster_backface=s.backface)
                r.render_clusters(cd, late, cluster_backface=s.backface)
                _compare_clusters(o, r, what)


# ---- the product: comparison helpers shared by the emulated and the device runs -----------------------------------------


def _np(a):
    return a.cpu().numpy().astype(np.uint32) if hasattr(a, "cpu") else np.asarray(a).view(np.uint32)


def _compare_draw(o, p, what):
    dccb = _np(p.dccb)
    assert np.array_equal(o.dccb, dccb), (what, o.dccb, dccb)
    n = int(o.dccb[1]) * 64
    assert np.array_equal(oracle_lib.sorted_commands(o.read_task_commands(n)), oracle_lib.sorted_commands(p.read_task_commands(n))), what
    assert np.array_equal(o.dvb, _np(p.dvb)[: len(o.dvb)]), what


def _compare_clusters(o, p, what):
    ccb = _np(p.ccb)
    assert np.array_equal(o.ccb, ccb), (what, o.ccb, ccb)
    n = int(o.ccb[0])
    ot, pt = o.read_task_commands(int(o.dccb[1]) * 64), p.read_task_commands(int(o.dccb[1]) * 64)
    assert np.array_equal(oracle_lib.cluster_pairs(o.read_cluster_indices(n), ot), oracle_lib.cluster_pairs(p.read_cluster_indices(n), pt)), what
    assert np.array_equal(o.mvb, _np(p.mvb)), what


def _task_table(path, cd, late, s, zeros):
    # n = 0 (no command this pass): the one slot read and allocated holds a command of an earlier pass, in an order the
    # device does not fix, so it is not compared
    n = int(_np(path.dccb)[1]) * 64
    cmds = path.read_task_commands(max(n, 1)).copy()
    payloads, emit = zeros((max(n, 1), 64)), zeros(max(n, 1))
    path.task_shading(cd, late, payloads, emit, cluster_backface=s.backface)
    pl, em = _np(payloads), _np(emit)
    return {tuple(cmds[i].tolist()): tuple(sorted(int(v) >> 24 for v in pl[i][: em[i]])) for i in range(n) if cmds["taskCount"][i]}


def _run(s, cfg, make_path, sync=lambda: None, zeros=None):
    """Two frames (+ post passes) of the product path against the oracle; returns the filter counters (items, undecided)."""
    draws = _scene_for(s, cfg)
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, draws, *s.screen, threads=4)
    p = make_path(draws)
    lib = p.emu if hasattr(p, "emu") else p.lib
    if "cluster_filter" in cfg:
        assert lib.nvc_set_cluster_filter(p.ctx, cfg["cluster_filter"]) == 0
    if "stage_texels" in cfg:
        assert lib.nvc_set_hiz_staging(p.ctx, cfg["stage_texels"]) == 0
    stats = (ctypes.c_uint64 * 2)()
    assert lib.nvc_filter_stats(p.ctx, stats, 1) == 0
    for q in (o, p):
        q.set_visibility_bits(s.visibility_bits)
    backface = cfg.get("backface", s.backface)
    cd = s.cull_data(**cfg.get("toggles", {}))
    passes = [(False, 0), (True, 0)] + ([(True, 1)] if cfg.get("post") else [])
    for frame in range(2):
        for late, post in passes:
            what = (s.name, frame, late, post)
            if late and post == 0:
                o.pyramid(s.depth)
                p.pyramid(p.depth_input)
            o.cull(cd, late, post_pass=post)
            p.cull(cd, late, post_pass=post)
            sync()
            _compare_draw(o, p, what)
            if cfg.get("task"):
                want = _task_table(o, cd, late, s, lambda shape: np.zeros(shape, np.uint32))
                got = _task_table(p, cd, late, s, zeros)
                assert want == got, what
                sync()
                assert np.array_equal(o.mvb, _np(p.mvb)), what
            else:
                o.render_clusters(cd, late, post_pass=post, cluster_backface=backface)
                p.render_clusters(cd, late, post_pass=post, cluster_backface=backface)
                sync()
                _compare_clusters(o, p, what)
    assert lib.nvc_filter_stats(p.ctx, stats, 1) == 0
    p.close()
    return int(stats[0]), int(stats[1])


def _check_filter(name, results):
    """Per cluster family: the filter decided some items and handed some to the exact path: the ladder straddles its margin."""
    by = {}
    for s, (items, undecided) in results:
        if s.kind == "cluster":
            a = by.setdefault(s.family, [0, 0])
            a[0] += items
            a[1] += undecided
    print(name, {f: "%d/%d undecided (%.1f %%)" % (u, i, 100.0 * u / max(i, 1)) for f, (i, u) in by.items()})
    for f, (items, undecided) in by.items():
        assert 0 < undecided < items, (name, f, items, undecided)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_emulated_kernels_at_boundaries(config, monkeypatch):
    """The product's kernels under the SIMT emulation against the oracle, bit for bit, on every family."""
    cfg = CONFIGS[config]
    if cfg.get("draw_filter"):
        monkeypatch.setenv("NVC_DRAW_FILTER", "1")  # read by nvc_create

    def make(s):
        def f(draws):
            e = emu_lib.EmuPath(s.meshes, s.meshlets, draws, *s.screen, prepare_hiz=cfg.get("prepare_hiz", True))
            e.depth_input = s.depth
            return e

        return f

    results = [(s, _run(s, cfg, make(s), zeros=lambda shape: np.zeros(shape, np.uint32))) for s in _scenes()]
    if config in FILTERED:
        _check_filter(config, results)
    elif cfg.get("cluster_filter") == 0:
        assert all(r[1] == (0, 0) for r in results), config  # the exact kernels do not count


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
def test_device_kernels_at_boundaries(config, monkeypatch):
    """The same families and configurations through VisibilityPath on the device, bit for bit against the oracle."""
    import torch

    from niagara_b200.path import VisibilityPath

    assert torch.cuda.is_available()
    cfg = CONFIGS[config]
    if cfg.get("draw_filter"):
        monkeypatch.setenv("NVC_DRAW_FILTER", "1")  # read by nvc_create

    def make(s):
        def f(draws):
            g = VisibilityPath(s.meshes, s.meshlets, draws, *s.screen, prepare_hiz=cfg.get("prepare_hiz", True))
            g.depth_input = torch.from_numpy(s.depth).cuda()
            return g

        return f

    zeros = lambda shape: torch.zeros(shape, dtype=torch.int32, device="cuda")
    results = [(s, _run(s, cfg, make(s), sync=torch.cuda.synchronize, zeros=zeros)) for s in _scenes()]
    if config in FILTERED:
        _check_filter("H100 " + config, results)
