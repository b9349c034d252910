"""CPU-only checks of the conservative meshlet filter (niagara_b200/csrc/nvc_filter.cuh):
  * tests/filter_harness.cpp — millions of random / hostile meshlets through filter_meshlet (both Hi-Z access variants) against
    the exact per-meshlet test, with the approximate reciprocals / roots perturbed by +-2 ulp and flushed as the device's .ftz
    instructions flush (the "subnormal" scenario puts znear, scale and view-space magnitudes there): no decided item may disagree,
    the margins must dominate the errors they bound, and the share of undecided items must stay small on the bench-like scene;
  * the filtered kernel (emulated) is exercised with the filter on / off and its diagnostic counters are read back."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

import emu_lib
import oracle_lib
from niagara_b200 import host, scenes

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(HERE, "_build", "filter")


def _harness():
    os.makedirs(OUT, exist_ok=True)
    exe = os.path.join(OUT, "filter_harness")
    srcs = [os.path.join(HERE, "filter_harness.cpp"), os.path.join(ROOT, "niagara_b200", "csrc", "nvc_filter.cuh"), os.path.join(ROOT, "niagara_b200", "csrc", "nvc_math.cuh"), os.path.join(ROOT, "niagara_b200", "csrc", "nvc_internal.h")]
    if not os.path.exists(exe) or any(os.path.getmtime(s) > os.path.getmtime(exe) for s in srcs):
        cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-w", "-DNVF_PERTURB", "-DNVF_DEBUG", "-I", os.path.join(HERE, "cuda_emu", "include"), "-I", os.path.join(ROOT, "niagara_b200", "csrc"),
               "-o", exe, srcs[0], os.path.join(ROOT, "niagara_b200", "csrc", "nvc_host.cpp"), "-lpthread"]
        subprocess.run(cmd, check=True)
    return exe


@pytest.mark.parametrize("seed", [3, 4])
def test_filter_never_disagrees_with_the_exact_test(seed):
    res = subprocess.run([_harness(), "all", "3000000", str(seed), "4"], capture_output=True, text=True, timeout=600)
    lines = [json.loads(l) for l in res.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 6, res.stderr[-2000:]
    by = {l["scenario"]: l for l in lines}
    for name, l in by.items():
        assert l["wrong"] == 0, (name, l, res.stderr[-2000:])
        assert l["exact_centre_occlusion"]["wrong"] == 0 and l["exact_centre_occlusion"]["items"] > 100000, (name, l)  # the drawcull use
        assert l["max_center_err_over_E"] < 1.0 and l["max_uv_err_over_margin"] < 1.0, (name, l)
    assert res.returncode == 0
    # the bench-like scene: only a few per cent may need the exact path; hostile transforms are sent there wholesale
    assert by["c4"]["undecided"] < 0.08, by["c4"]
    assert by["biglocal"]["undecided"] < 0.08
    assert by["hostile"]["exact_only"] > 0.5
    # the flush range: most cone tests there are left to the exact path (|c|^2 < 2^-110), but the filter still decides the rest
    sub = by["subnormal"]
    print("subnormal scenario: undecided %.4f (frustum / cone %.4f, domain %.4f), exact-centre occlusion undecided %.4f" % (sub["undecided"], sub["undecided_by_stage"]["frustum_cone"], sub["undecided_by_stage"]["domain"], sub["exact_centre_occlusion"]["undecided"]))
    assert 0.05 < sub["undecided"] < 0.9 and sub["exact_centre_occlusion"]["undecided"] < 0.9, sub


def test_filter_on_off_same_results_and_counters(golden_dir):
    """the filtered kernel and the exact kernel (nvc_set_cluster_filter) write the same cluster sets and visibility bits;
    the diagnostic counters show that the filter really decided most meshlets"""
    s = scenes.config4_scene(draw_count=6000, screen=(1024, 1024))
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *s.screen, threads=4, cmd_capacity=12032)
    paths = []
    for on in (1, 0):
        e = emu_lib.EmuPath(s.meshes, s.meshlets, s.draws, *s.screen, cmd_capacity=12032)
        assert e.emu.nvc_set_cluster_filter(e.ctx, on) == 0
        e.set_visibility_bits(s.visibility_bits)
        paths.append(e)
    o.set_visibility_bits(s.visibility_bits)
    cams = [host.make_camera(), host.make_camera((0.5, 0.2, -0.3), host.quat_from_axis_angle((0, 1, 0), 0.02))]
    stats = (ctypes.c_uint64 * 2)()
    assert paths[0].emu.nvc_filter_stats(paths[0].ctx, stats, 1) == 0
    for f in range(2):
        s.camera = cams[f]
        cd = s.cull_data()
        for late in (False, True):
            for p in [o] + paths:
                if late:
                    p.pyramid(s.depth)
                p.cull(cd, late)
                p.render_clusters(cd, late, cluster_backface=True)
            for e in paths:
                assert np.array_equal(o.ccb, e.ccb), (f, late)
                n = int(o.ccb[0])
                oc = o.read_task_commands(int(o.dccb[1]) * 64)
                ec = e.read_task_commands(int(e.dccb[1]) * 64)
                assert np.array_equal(oracle_lib.cluster_pairs(o.read_cluster_indices(n), oc), oracle_lib.cluster_pairs(e.read_cluster_indices(n), ec)), (f, late)
                assert np.array_equal(o.mvb, e.mvb), (f, late)
    assert paths[0].emu.nvc_filter_stats(paths[0].ctx, stats, 0) == 0
    items, undecided = int(stats[0]), int(stats[1])
    assert items > 100000 and undecided < 0.1 * items, (items, undecided)
    off = (ctypes.c_uint64 * 2)()
    assert paths[1].emu.nvc_filter_stats(paths[1].ctx, off, 0) == 0 and int(off[0]) == 0  # the exact kernel does not count
    for e in paths:
        e.close()


def test_checker_host_helpers_match_the_product_helpers():
    """bench.py's CPU arms use the oracle's own host helpers: same CullData / pyramid layout / visibility offsets"""
    H = oracle_lib.CheckerHost
    cam = host.make_camera()
    a, b = host.cull_data(cam, 4096, 4096, 1000), H.cull_data(cam, 4096, 4096, 1000)
    assert bytes(a) == bytes(b)
    cam2 = host.make_camera((3, -2, 5), host.quat_from_axis_angle((0.2, 1, 0.1), 0.7))
    fa = np.frombuffer(bytes(host.cull_data(cam2, 1920, 1080, 10)), dtype=np.float32)[:27]
    fb = np.frombuffer(bytes(H.cull_data(cam2, 1920, 1080, 10)), dtype=np.float32)[:27]
    assert np.allclose(fa, fb, rtol=0, atol=4e-6)
    for w, h in [(4096, 4096), (1920, 1080), (1, 1), (2, 2), (5, 3), (1024, 768)]:
        x, y = host.hiz_layout(w, h), H.hiz_layout(w, h)
        assert (x.width, x.height, x.levels, list(x.level_offset), x.total_texels) == (y.width, y.height, y.levels, list(y.level_offset), y.total_texels)
    s1 = scenes.config4_scene(3000, 10, screen=(256, 256))
    s2 = scenes.config4_scene(3000, 10, screen=(256, 256), helpers=H)
    assert np.array_equal(s1.draws, s2.draws) and s1.visibility_bits == s2.visibility_bits
    pd1 = oracle_lib.OraclePath(s1.meshes, s1.meshlets, s1.draws, 256, 256)._pass_data(a, 1, 0)
    pd2 = H.pass_data(a, 1, 0)
    assert bytes(pd1) == bytes(pd2)
