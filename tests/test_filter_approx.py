"""The conservative cluster filter's approximate reciprocal and square root (nvc_filter.cuh: rcp.approx.ftz.f32 and
sqrt.approx.ftz.f32 on the device, FTZ-faithful stand-ins under NVC_EMU), and whole frames in the range where they flush.

  * nvc_filter_approx runs either instruction over an array of float bit patterns.  CPU tier: the emulated library's stand-ins on
    a fixed table of special values (every subnormal class, the edges of the normal range, +-0, +-inf, NaN, negative roots).
    -m gpu: the same table on the H100, and all 2^32 inputs of both instructions against float64: relative error <= 2^-22
    (the budget the filter's margins and tests/filter_harness.cpp assume) where argument and true result are normal, and
    bit-equal to the stand-ins everywhere else.
  * A frame of radius-0 and tiny meshlets within ~1e-20 .. 3e-16 of a camera with znear = 1e-21, where |c|^2 and c.z^2 - r^2 are
    subnormal or near the filter's domain threshold: filtered cluster passes (with and without the footprint image, and the
    filtered drawcull occlusion stage) against the oracle bit for bit, with the filter deciding some of the items.
  * Items the subnormal scenario of tests/filter_harness.cpp decided wrongly before the filter's domain check (8)."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

import boundary_scenes as bs
import emu_lib
import oracle_lib
import test_decision_boundaries as tdb
from niagara_b200 import host, layout, scenes

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(HERE, "_build", "filter")

RCP, SQRT = 0, 1
CANONICAL_NAN = 0x7FFFFFFF
BUDGET = 2.0**-22


def _standins():
    """The stand-ins as a host loop: nvf_standins(op, in, out, n)"""
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, "libnvf_standins.so")
    csrc = os.path.join(ROOT, "niagara_b200", "csrc")
    srcs = [os.path.join(HERE, "filter_standins.cpp"), os.path.join(csrc, "nvc_filter.cuh"), os.path.join(csrc, "nvc_math.cuh"), os.path.join(csrc, "nvc_internal.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-w", "-I", os.path.join(HERE, "cuda_emu", "include"), "-I", csrc, "-o", so, srcs[0]], check=True)
    lib = ctypes.CDLL(so)
    lib.nvf_standins.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64]
    lib.nvf_standins.restype = None
    return lib


def standins(op, bits):
    bits = np.ascontiguousarray(bits, np.uint32)
    out = np.empty_like(bits)
    _standins().nvf_standins(op, bits.ctypes.data, out.ctypes.data, len(bits))
    return out


def _f(b):
    return int(np.float32(b).view(np.uint32))


# (input bits, expected rcp bits or None = normal result checked against float64, expected sqrt bits or None)
INF, NINF, PZ, NZ = 0x7F800000, 0xFF800000, 0x00000000, 0x80000000
TABLE = [
    (PZ, INF, PZ),
    (NZ, NINF, NZ),
    (INF, PZ, INF),
    (NINF, NZ, CANONICAL_NAN),
    (0x7FC00000, CANONICAL_NAN, CANONICAL_NAN),  # quiet NaN
    (0x7F800001, CANONICAL_NAN, CANONICAL_NAN),  # signalling NaN
    (0xFFC00001, CANONICAL_NAN, CANONICAL_NAN),  # negative NaN with a payload
    (0x00000001, INF, PZ),  # smallest subnormal: read as +0
    (0x00400000, INF, PZ),
    (0x007FFFFF, INF, PZ),  # largest subnormal
    (0x80000001, NINF, NZ),
    (0x807FFFFF, NINF, NZ),
    (0x00800000, None, None),  # 2^-126: rcp 2^126, sqrt 2^-63
    (0x00800001, None, None),
    (0x80800000, None, CANONICAL_NAN),
    (0x7F7FFFFF, PZ, None),  # largest finite: its reciprocal (2.9e-39) is subnormal and written as 0
    (0xFF7FFFFF, NZ, CANONICAL_NAN),
    (0x7F000000, PZ, None),  # 2^127: reciprocal 2^-127, subnormal
    (0x7F400000, PZ, None),  # 1.5 * 2^127
    (0x7E800000, None, None),  # 2^126: reciprocal 2^-126, the smallest normal
    (_f(1.0), None, None),
    (_f(-1.0), None, CANONICAL_NAN),
    (_f(3.0), None, None),
    (_f(1e-21), None, None),
    (_f(-1e-30), None, CANONICAL_NAN),
    (_f(1.7e-21 * 1.7e-21), INF, PZ),  # |c|^2 of the cone's counterexample: subnormal
]


def _check_table(got_rcp, got_sqrt, who):
    for (x, want_r, want_s), gr, gs in zip(TABLE, got_rcp, got_sqrt):
        xf = float(np.uint32(x).view(np.float32))
        for op, want, got in ((RCP, want_r, gr), (SQRT, want_s, gs)):
            if want is not None:
                assert int(got) == want, (who, op, hex(x), hex(int(got)), hex(want))
            else:
                ref = 1.0 / xf if op == RCP else math.sqrt(xf)
                val = float(np.uint32(got).view(np.float32))
                assert abs(val - ref) <= BUDGET * abs(ref), (who, op, hex(x), val, ref)


def test_standins_on_special_values():
    """Emulated library (the SIMT-emulated kernel) and the host loop: the same bits, the device's special-value rules"""
    emu = emu_lib.load()
    ctx = ctypes.c_void_p()
    limits = layout.Limits(layout.TASK_WGLIMIT, layout.CLUSTER_LIMIT)
    assert emu.nvc_create(0, ctypes.byref(limits), ctypes.byref(ctx)) == 0
    x = np.array([t[0] for t in TABLE], np.uint32)
    got = []
    for op in (RCP, SQRT):
        out = np.zeros_like(x)
        assert emu.nvc_filter_approx(ctx, None, op, x.ctypes.data, out.ctypes.data, len(x)) == 0
        assert np.array_equal(out, standins(op, x)), op
        got.append(out)
    assert emu.nvc_filter_approx(ctx, None, 2, x.ctypes.data, x.ctypes.data, len(x)) != 0  # unknown op
    emu.nvc_destroy(ctx)
    _check_table(got[0], got[1], "emulated")


def _device_ctx(torch):
    from niagara_b200.lib import load_library

    lib = load_library()
    ctx = ctypes.c_void_p()
    limits = layout.Limits(layout.TASK_WGLIMIT, layout.CLUSTER_LIMIT)
    assert lib.nvc_create(0, ctypes.byref(limits), ctypes.byref(ctx)) == 0
    return lib, ctx


def _device_approx(torch, lib, ctx, op, bits):
    out = torch.empty_like(bits)
    assert lib.nvc_filter_approx(ctx, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream), op, ctypes.c_void_p(bits.data_ptr()), ctypes.c_void_p(out.data_ptr()), bits.numel()) == 0
    return out


@pytest.mark.gpu
def test_device_on_special_values():
    import torch

    lib, ctx = _device_ctx(torch)
    x = torch.from_numpy(np.array([t[0] for t in TABLE], np.uint32).view(np.int32)).cuda()
    got = [_device_approx(torch, lib, ctx, op, x).cpu().numpy().view(np.uint32) for op in (RCP, SQRT)]
    lib.nvc_destroy(ctx)
    _check_table(got[0], got[1], "H100")


@pytest.mark.gpu
def test_device_exhaustive_against_float64():
    """All 2^32 bit patterns through both instructions on the H100, in chunks of 2^28"""
    import torch

    lib, ctx = _device_ctx(torch)
    chunk = 1 << 28
    report = {}
    for op, name in ((RCP, "rcp.approx.ftz.f32"), (SQRT, "sqrt.approx.ftz.f32")):
        worst, worst_x, special = 0.0, 0, 0
        for k in range((1 << 32) // chunk):
            ids = torch.arange(k * chunk, (k + 1) * chunk, dtype=torch.int64, device="cuda")
            bits = torch.where(ids >= (1 << 31), ids - (1 << 32), ids).to(torch.int32)
            del ids
            out = _device_approx(torch, lib, ctx, op, bits)
            x = bits.view(torch.float32).double()
            ref = 1.0 / x if op == RCP else torch.sqrt(x)
            e = bits & 0x7F800000
            normal = (e != 0) & (e != 0x7F800000) & (ref.abs() >= 2.0**-126) & (ref.abs() < 2.0**128)
            if op == SQRT:
                normal &= x > 0
            y = out.view(torch.float32).double()
            rel = torch.where(normal, (y - ref).abs() / ref.abs(), torch.zeros_like(ref))
            m, i = torch.max(rel, 0)
            if float(m) > worst:
                worst, worst_x = float(m), int(bits[i]) & 0xFFFFFFFF
            del x, ref, y, rel, e
            # everywhere else: the stand-ins' bits
            sel = torch.nonzero(~normal).flatten()
            special += sel.numel()
            xs = bits[sel].cpu().numpy().view(np.uint32)
            dev = out[sel].cpu().numpy().view(np.uint32)
            want = standins(op, xs)
            bad = np.nonzero(dev != want)[0]
            assert len(bad) == 0, (name, len(bad), [(hex(int(xs[j])), hex(int(dev[j])), hex(int(want[j]))) for j in bad[:12]])
            del bits, out, normal, sel
        report[name] = (worst, worst_x, special)
        print("%s: max relative error %.4g (2^%.3f) at input 0x%08x over the normal range; %d special-value inputs, all equal to the stand-ins" % (name, worst, math.log2(worst), worst_x, special))
        assert worst <= BUDGET, (name, worst, hex(worst_x))
    lib.nvc_destroy(ctx)
    assert report["rcp.approx.ftz.f32"][2] > 0 and report["sqrt.approx.ftz.f32"][2] > (1 << 31)


# ---- whole frames in the flush range -----------------------------------------------------------------------------------

ZNEAR = 1e-21
# depth zones (u0, u1, v0, v1, reverse-Z depth): B occludes at view depth 2e-21, C at 1e-18, D at 1e-16
ZONES = [(0.55, 0.85, 0.2, 0.45, ZNEAR / 2e-21), (0.55, 0.85, 0.55, 0.8, ZNEAR / 1e-18), (0.15, 0.45, 0.55, 0.8, ZNEAR / 1e-16)]


def _cone_item(mk, rng, z, k8):
    """r = 0 at view depth ~z, cone axis 60 degrees from the centre direction, cutoff byte k8"""
    st = mk.st
    for _ in range(200):
        a8 = np.rint(rng.standard_normal(3) * 60).clip(-127, 127).astype(np.int8)
        q = bs._quat(rng, False)
        a = st.M @ bs._rotate64(a8.astype(np.float64) / 127.0, q)
        a /= np.linalg.norm(a)
        p = rng.standard_normal(3)
        p -= p.dot(a) * a
        p /= np.linalg.norm(p)
        d = 0.5 * a + math.sqrt(0.75) * p
        if d[2] < 0.6 or abs(d[0]) * st.P00 > 0.7 * d[2] or abs(d[1]) * st.P11 > 0.7 * d[2]:
            continue
        b = mk.base("cluster", "cone", d * z / d[2], 0.0, ("position", int(rng.integers(0, 3))), s=2.0**-39, lc_zero=True, cone=(a8, k8))
        b.draw["orientation"] = q
        b.p0 = float(b.draw["position"][0, b.sweep[1]])
        return b
    raise RuntimeError("no cone item")


def _zone_item(mk, rng, zone, z, r, kind="cluster", s=2.0**-39):
    st = mk.st
    u0, u1, v0, v1, _ = ZONES[zone]
    u, v = rng.uniform(u0 + 0.05, u1 - 0.05), rng.uniform(v0 + 0.05, v1 - 0.05)
    return mk.base(kind, "depth", st.view_point(u, v, z), r, ("position", int(rng.integers(0, 3))), s=s, lc_zero=True)


def subnormal_scene(seed=7):
    """radius-0 and tiny meshlets near a camera with znear = 1e-21 (boundary_scenes' ladders of +-2^24 ulps around each base
    position spread them over both sides of every outcome)"""
    st = bs.Setup("subnormal", (512, 512), host.make_camera(znear=ZNEAR), ZONES)
    rng = np.random.default_rng(seed)
    mk = bs._Maker(rng, st)
    r64 = 2.0**-64  # the smallest non-zero radius of a command the filter takes: fp16 2^-24 x scale 2^-40
    bases = []
    for _ in range(2):
        bases += [_cone_item(mk, rng, 1.5e-21, 115), _cone_item(mk, rng, 1.5e-21, 20), _cone_item(mk, rng, 3e-16, 115), _cone_item(mk, rng, 3e-16, 20)]
        bases += [_zone_item(mk, rng, 0, 1.5e-21, 0.0), _zone_item(mk, rng, 0, 4e-21, 0.0)]  # in front of / behind B
        bases += [_zone_item(mk, rng, 1, 5e-19, r64, s=2.0**-39.9), _zone_item(mk, rng, 1, 3e-18, r64, s=2.0**-39.9)]  # C
        bases += [_zone_item(mk, rng, 2, 5e-17, r64, s=2.0**-39.9), _zone_item(mk, rng, 2, 3e-16, r64, s=2.0**-39.9)]  # D
        bases += [_zone_item(mk, rng, 0, 1.5e-21, 1e-22, kind="draw"), _zone_item(mk, rng, 1, 3e-18, 1e-19, kind="draw")]  # drawcull spheres
    return bs.FamilyScene("subnormal", st, "cluster", bases, [int(bs.to_ord(np.float32(b.p0))) for b in bases])


CONFIGS = ["filtered", "filtered_no_footprint_image", "draw_filter"]


def _frame_check(config, make, monkeypatch, sync=lambda: None, zeros=None):
    cfg = tdb.CONFIGS[config]
    if cfg.get("draw_filter"):
        monkeypatch.setenv("NVC_DRAW_FILTER", "1")  # read by nvc_create
    s = subnormal_scene()
    items, undecided = tdb._run(s, cfg, make(s, cfg), sync=sync, zeros=zeros)
    print("%s: %d meshlets through the filter, %d undecided" % (config, items, undecided))
    assert 0 < undecided < items, (config, items, undecided)


@pytest.mark.parametrize("config", CONFIGS)
def test_emulated_frames_near_a_tiny_znear(config, monkeypatch):
    def make(s, cfg):
        def f(draws):
            e = emu_lib.EmuPath(s.meshes, s.meshlets, draws, *s.screen, prepare_hiz=cfg.get("prepare_hiz", True))
            e.depth_input = s.depth
            return e

        return f

    _frame_check(config, make, monkeypatch, zeros=lambda shape: np.zeros(shape, np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("config", CONFIGS)
def test_device_frames_near_a_tiny_znear(config, monkeypatch):
    import torch

    from niagara_b200.path import VisibilityPath

    def make(s, cfg):
        def f(draws):
            g = VisibilityPath(s.meshes, s.meshlets, draws, *s.screen, prepare_hiz=cfg.get("prepare_hiz", True))
            g.depth_input = torch.from_numpy(s.depth).cuda()
            return g

        return f

    _frame_check(config, make, monkeypatch, sync=torch.cuda.synchronize, zeros=lambda shape: torch.zeros(shape, dtype=torch.int32, device="cuda"))


# ---- the harness's counterexamples ---------------------------------------------------------------------------------------

# tests/filter_harness.cpp, scenario "subnormal", seed 3, with the FTZ-faithful stand-ins and without the domain check (8):
# decided not visible, visible on the exact path (the cone's root of a subnormal |c|^2 flushed to 0).  Float fields as bits:
# camera (position, orientation, fovY, znear), screen, draw distance, draws (position, scale, orientation), meshlets
# (centre / radius halves, cone bytes).
HARNESS_CASES = [
    dict(camera=[2629312546, 2628806088, 460680674, 1056695569, 3196052853, 3207217388, 1057018269, 1060307595, 466135362], screen=(512, 2048), draw_distance=1136080322,
         items=[([478168765, 2625284794, 2610954859, 764502221, 1050303746, 3208131064, 3198115339, 3205164586], [0, 0, 1163988655]),
                ([2625225578, 2628745744, 454674171, 746492852, 3200643457, 1061643381, 3198948543, 1052328579], [0, 0, 1004810126])]),
    dict(camera=[2450007020, 2457611010, 2427807212, 3196181177, 1030046428, 3199372285, 3211167850, 1059411901, 296184641], screen=(1920, 1080), draw_distance=1130190800,
         items=[([2614098386, 473160687, 2629729383, 756497615, 1057667314, 1057272394, 1052960410, 3205137546], [0, 0, 1842893480]),
                ([2614098386, 473160687, 2629729383, 756497615, 1057667314, 1057272394, 1052960410, 3205137546], [0, 32768, 1632657175])]),
]


class _CaseScene(scenes.Scene):
    def __init__(self, case):
        f = lambda b: np.uint32(b).view(np.float32)
        cb = case["camera"]
        cam = host.make_camera([f(b) for b in cb[0:3]], [f(b) for b in cb[3:7]], f(cb[7]), f(cb[8]))
        n = len(case["items"])
        meshes = np.zeros(n, layout.MESH_DTYPE)
        meshlets = np.zeros(n, layout.MESHLET_DTYPE)
        draws = np.zeros(n, layout.MESHDRAW_DTYPE)
        for i, (d, m) in enumerate(case["items"]):
            d = np.array(d, np.uint32).view(np.float32)
            draws["position"][i], draws["scale"][i], draws["orientation"][i], draws["meshIndex"][i] = d[0:3], d[3], d[4:8], i
            meshes["lodCount"][i] = 1
            meshes["lods"]["meshletOffset"][i, 0], meshes["lods"]["meshletCount"][i, 0], meshes["lods"]["indexCount"][i, 0] = i, 1, 3
            meshes["radius"][i] = np.float32(8.0 * (np.abs(d[0:3]).sum() + 1.0) / d[3])  # the draw's sphere contains the camera
            meshlets["center"][i] = [m[0] & 0xFFFF, m[0] >> 16, m[1] & 0xFFFF]
            meshlets["radius"][i] = m[1] >> 16
            meshlets["cone_axis"][i] = np.array([m[2] & 0xFF, (m[2] >> 8) & 0xFF, (m[2] >> 16) & 0xFF], np.uint8).view(np.int8)
            meshlets["cone_cutoff"][i] = np.uint8(m[2] >> 24).view(np.int8)
        meshlets["vertexCount"], meshlets["triangleCount"] = 3, 1
        bits, _ = host.visibility_offsets(draws, meshes)
        w, h = case["screen"]
        super().__init__("harness_case", meshes, meshlets, draws, np.zeros((h, w), np.float32), cam, (w, h), bits)
        self.draw_distance = float(f(case["draw_distance"]))
        self.backface, self.kind, self.family = True, "cluster", "harness_case"

    def cull_data(self, **toggles):
        return super().cull_data(draw_distance=self.draw_distance, **toggles)


@pytest.mark.parametrize("case", range(len(HARNESS_CASES)))
def test_emulated_harness_counterexamples(case):
    """The filtered kernel under the emulation against the oracle on the harness's items (empty depth: every sphere the
    frustum and cone keep is visible); the filter must now leave them to the exact path or agree"""
    s = _CaseScene(HARNESS_CASES[case])
    o = oracle_lib.OraclePath(s.meshes, s.meshlets, s.draws, *s.screen)
    o.set_visibility_bits(s.visibility_bits)
    cd = s.cull_data()
    o.pyramid(s.depth)
    o.cull(cd, True)
    o.render_clusters(cd, True, cluster_backface=True)
    assert int(o.ccb[0]) == len(s.draws)  # every item is visible on the exact path

    def make(draws):
        e = emu_lib.EmuPath(s.meshes, s.meshlets, draws, *s.screen)
        e.depth_input = s.depth
        return e

    tdb._run(s, tdb.CONFIGS["filtered"], make, zeros=lambda shape: np.zeros(shape, np.uint32))
