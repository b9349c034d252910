"""Boundary-ladder scenes: every cull decision placed on its rounding boundary — test infrastructure only.

Each *item* is one draw of its own mesh (one LOD, one meshlet; two LODs for the LOD families), so its decision is
isolated.  A *family* is one threshold comparison of the shaders; a *base* is one configuration (camera, screen, draw
orientation, scale, mesh / meshlet bounds) plus a 1-D float32 parameter of the item (a position component, the scale or a
LOD error) that moves the compared value through the threshold.  The generator locates the flip of the comparison with
the float32 restatement tests/numpy_ref.py by bisection over float32 ordinals (bits viewed as ordered integers), checks
that the item's verdict flips there too, and emits a *ladder*: the items at +-{0, 1, 2, 3, 4, 8, 16, ..., 2^24} ulps of the
flip.  The inner rungs test the strict path's exact rounding; the outer rungs cross any margin of the conservative filter.

Rung 0 is the last value on the first side of the flip, rung +1 the first on the other side; with a swept radius or LOD
error the compared values meet exactly (`>` against `>=` differ on one of these two rungs)."""
import ctypes
import math

import numpy as np

import numpy_ref as nr
from niagara_b200 import host, layout, scenes

F = np.float32
RUNGS = np.array(sorted({0} | {s * o for s in (1, -1) for o in [1, 2, 3, 4] + [1 << k for k in range(3, 25)]}), np.int64)
HOT = 4  # the verdicts of the rungs within +-HOT ulps must include both outcomes


def to_ord(x):
    """float32 -> int64 ordinal, monotone in the float order (-0.0 sits one below +0.0)"""
    i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
    return np.where(i >= 0, i, -(i & 0x7FFFFFFF) - 1)


def from_ord(o):
    o = np.asarray(o, np.int64)
    return np.where(o >= 0, o, (-o - 1) | 0x80000000).astype(np.uint32).view(np.float32)


def _pass_data(cd, for_drawcull, backface=None):
    from niagara_b200.lib import load_library

    pd = layout.CullData()
    load_library().nvc_host_pass_data(ctypes.byref(cd), for_drawcull, 0, ctypes.byref(pd))
    if backface is not None:
        pd.clusterBackfaceEnabled = int(backface)
    return pd.to_numpy()


class Setup:
    """Camera, screen, depth image (rectangles of constant reverse-Z depth on a far background) and CullData toggles."""

    def __init__(self, name, screen, camera, zones, toggles=None):
        self.name, self.screen, self.camera, self.zones, self.toggles = name, screen, camera, zones, dict(toggles or {})
        w, h = screen
        self.depth = np.zeros((h, w), np.float32)
        for u0, u1, v0, v1, value in zones:
            self.depth[int(v0 * h) : int(v1 * h), int(u0 * w) : int(u1 * w)] = value
        self.cd = host.cull_data(camera, w, h, 1, **self.toggles)
        self.hiz = host.hiz_layout(w, h)
        self.levels = nr.build_pyramid(self.depth, self.hiz.width, self.hiz.height, self.hiz.levels)
        v = np.array(self.cd.view, np.float64)
        self.M = np.array([[v[4 * j + i] for j in range(3)] for i in range(3)])  # view-space = M world + T
        self.T = v[12:15]
        self.P00, self.P11, self.znear, self.zfar = float(self.cd.P00), float(self.cd.P11), float(self.cd.znear), float(self.cd.zfar)
        self.frustum = [float(f) for f in self.cd.frustum]

    def pass_data(self, n, for_drawcull, backface=None):
        cd = self.cd.copy()
        cd.drawCount = n
        return _pass_data(cd, for_drawcull, backface)

    def zone(self, k):
        return self.zones[k]

    def view_point(self, u, v, z):
        """view-space point at screen coordinates (u, v) (aabb convention: v down) and depth z"""
        return np.array([(2 * u - 1) * z / self.P00, (1 - 2 * v) * z / self.P11, z])

    def world(self, c):
        return np.linalg.solve(self.M, np.asarray(c, np.float64) - self.T)


def _setups():
    D = 0.1 / 50.0  # occluder at view depth 50
    zones = [(0.15, 0.45, 0.3, 0.7, 1.0), (0.55, 0.8531, 0.2, 0.8, D)]  # A: at the near plane, B: at depth 50
    rot = host.quat_from_axis_angle((0.3, 1.0, 0.2), 0.6)
    return {
        "square": Setup("square", (1024, 1024), host.make_camera(), zones),
        "hd_rotated": Setup("hd_rotated", (1920, 1080), host.make_camera((3.0, -2.0, 5.0), rot), zones),
        "tiny": Setup("tiny", (512, 512), host.make_camera(znear=1e-21), [(0.15, 0.45, 0.3, 0.7, 1.0), (0.55, 0.8531, 0.2, 0.8, 0.5)]),
        "unculled": Setup("unculled", (640, 480), host.make_camera(), zones, dict(culling=False, occlusion=False)),
    }


def _rotate64(v, q):
    qv, w = np.asarray(q[:3], np.float64), float(q[3])
    t = np.cross(qv, v) + w * np.asarray(v, np.float64)
    return np.asarray(v, np.float64) + 2.0 * np.cross(qv, t)


class Base:
    """One configuration: item template + the swept parameter.  sweep: ('position', axis) | ('scale',) | ('error',)"""

    def __init__(self, setup, kind, indicator, sweep, p0, window, backface=True):
        self.setup, self.kind, self.indicator, self.sweep, self.p0, self.window, self.backface = setup, kind, indicator, sweep, p0, window, backface
        self.mesh = np.zeros(1, layout.MESH_DTYPE)
        self.meshlets = np.zeros(2, layout.MESHLET_DTYPE)
        self.draw = np.zeros(1, layout.MESHDRAW_DTYPE)

    def items(self, values):
        """n items with the swept parameter set to `values`: (meshes[n], meshlets[2n], draws[n]); item i owns meshlets 2i, 2i+1"""
        n = len(values)
        meshes = np.repeat(self.mesh, n)
        meshlets = np.tile(self.meshlets, n)
        draws = np.repeat(self.draw, n)
        meshes["lods"]["meshletOffset"] += (2 * np.arange(n, dtype=np.uint32))[:, None]
        meshes["lods"]["indexOffset"] += (6 * np.arange(n, dtype=np.uint32))[:, None]
        draws["meshIndex"] = np.arange(n, dtype=np.uint32)
        values = np.asarray(values, np.float32)
        if self.sweep[0] == "position":
            draws["position"][:, self.sweep[1]] = values
        elif self.sweep[0] == "scale":
            draws["scale"] = values
        else:
            meshes["lods"]["error"][:, 1] = values
        return meshes, meshlets, draws


def _probe(base, values):
    """(indicator, verdict) of every item per numpy_ref: the family's compared quantity and the late pass's outcome of the
    first frame (cluster kind: meshlet visible; draw kind: lod index or 255 when not emitted)."""
    st = base.setup
    meshes, meshlets, draws = base.items(values)
    n = len(draws)
    with np.errstate(all="ignore"):
        q = tuple(draws["orientation"][:, i] for i in range(4))
        if base.kind == "cluster":
            ml = meshlets[0::2]
            lc = tuple(nr.half_to_float(ml["center"][:, i]) for i in range(3))
            rl = nr.half_to_float(ml["radius"])
        else:
            lc = tuple(meshes["center"][:, i] for i in range(3))
            rl = meshes["radius"]
        s = draws["scale"]
        rc = nr.rotate_quat(lc, q)
        view = [F(x) for x in st.cd.view]
        c = nr.transform_point(view, tuple(rc[i] * s + draws["position"][:, i] for i in range(3)))
        r = rl * s
        f = [F(x) for x in st.frustum]
        znear, zfar, pw, ph = F(st.znear), F(st.zfar), F(st.cd.pyramidWidth), F(st.cd.pyramidHeight)
        key = base.indicator
        if key == "frustum_x":
            ind = c[2] * f[1] - np.abs(c[0]) * f[0] > -r
        elif key == "frustum_y":
            ind = c[2] * f[3] - np.abs(c[1]) * f[2] > -r
        elif key == "near":
            ind = c[2] + r > znear
        elif key == "far":
            ind = c[2] - r < zfar
        elif key == "cone":
            ml = meshlets[0::2]
            la = tuple(ml["cone_axis"][:, i].astype(np.float32) / F(127.0) for i in range(3))
            axis = nr.transform_vector(view, nr.rotate_quat(la, q))
            ind = nr.dot3(c, axis) >= (ml["cone_cutoff"].astype(np.float32) / F(127.0)) * nr.length3(c) + r
        elif key == "lod":
            ind = None
        else:
            ok, aabb = nr.project_sphere(c, r, znear, F(st.P00), F(st.P11))
            sx, sy = aabb[2] - aabb[0], aabb[3] - aabb[1]
            m = np.fmax(sx * pw, sy * ph)
            good = (m > 1) & np.isfinite(m)
            L = np.where(good, nr.ceil_log2_exact(np.where(good, m, F(1))), 0)
            if key == "ok":
                ind = ok
            elif key == "mip":
                # the selected level: ceil(log2 m) at the power-of-two crossings of m where the finer level's "fits" does not
                # take the level back (at most crossings it does: the box of 2^k texels nearly always fits 2 x 2 of mip k)
                ind = nr.occlusion_mip(aabb, pw, ph)
            elif key == "fits":
                scale = np.ldexp(F(1.0), (1 - np.maximum(L, 1)).astype(np.int32)).astype(np.float32)
                fmx, fmy = pw * scale, ph * scale
                px, py = aabb[0] * fmx, aabb[1] * fmy
                ind = good & (px - np.floor(px) + sx * fmx <= F(2.0)) & (py - np.floor(py) + sy * fmy <= F(2.0))
            elif key == "footprint":
                level = np.clip(nr.occlusion_mip(aabb, pw, ph), 0, len(st.levels) - 1).astype(np.int64)
                w = np.array([lv.shape[1] for lv in st.levels], np.float32)[level]
                x = ((aabb[0] + aabb[2]) * F(0.5)) * w - F(0.5)
                fl = np.floor(x)
                # (level, which texels count) as one number; locate() keeps only flips inside one level
                ind = np.where(np.isfinite(x), level * 1e6 + 2.0 * fl.astype(np.float64) + (x != fl), -1e300)
            elif key == "depth":
                u, v = (aabb[0] + aabb[2]) * F(0.5), (aabb[1] + aabb[3]) * F(0.5)
                safe = ok & np.isfinite(u) & np.isfinite(v)
                depth = np.zeros(n, np.float32)
                if safe.any():
                    depth[safe] = nr.sample_hiz(st.levels, u[safe], v[safe], nr.occlusion_mip(aabb, pw, ph)[safe])
                ind = ~ok | (znear / (c[2] - r) > depth)
            else:
                raise KeyError(key)
        if base.kind == "cluster":
            cmds = np.zeros(n, layout.MESHTASKCOMMAND_DTYPE)
            cmds["drawId"] = np.arange(n)
            cmds["taskOffset"] = 2 * np.arange(n)
            cmds["taskCount"] = 1
            cmds["meshletVisibilityOffset"] = np.arange(n)
            mvb = np.zeros((n + 31) // 32, np.uint32)
            verdict = nr.cluster_decisions(st.pass_data(n, 0, base.backface), True, cmds, draws, meshlets, mvb, st.levels)[4].astype(np.int64)
        else:
            _, _, emit, lod = nr.drawcull_decisions(st.pass_data(n, 1), True, draws, meshes, np.zeros(n, np.uint32), st.levels)
            verdict = np.where(emit, lod.astype(np.int64), 255)
    if ind is None:
        ind = verdict
    return np.asarray(ind, np.float64), verdict


def locate(base, max_candidates=24):
    """The ordinal of rung 0 (last item before the indicator changes, with a verdict change there), or None."""
    lo_v, hi_v = base.p0 - base.window, base.p0 + base.window
    grid = np.unique(np.linspace(lo_v, hi_v, 2049).astype(np.float32))
    grid = grid[np.isfinite(grid)]
    ind, _ = _probe(base, grid)
    ch = np.nonzero(ind[1:] != ind[:-1])[0]
    ch = ch[np.argsort(np.abs(grid[ch].astype(np.float64) - base.p0), kind="stable")]
    for c in ch[:max_candidates]:
        if base.indicator == "footprint" and ind[c] // 1e6 != ind[c + 1] // 1e6:
            continue  # a level change, not the sampler's footprint
        lo, hi = int(to_ord(grid[c])), int(to_ord(grid[c + 1]))
        want = ind[c]
        while hi - lo > 1:
            pts = np.unique(np.linspace(lo, hi, 65).astype(np.int64))
            pi, _ = _probe(base, from_ord(pts))
            k = int(np.argmax(pi != want))  # first point past the change (pi[-1] != want)
            if k == 0:
                break  # indicator not monotone inside the bracket
            lo, hi = int(pts[k - 1]), int(pts[k])
        if hi - lo != 1:
            continue
        i2, v = _probe(base, from_ord(np.array([lo, hi])))
        if base.indicator == "footprint" and i2[0] // 1e6 != i2[1] // 1e6:
            continue
        if v[0] != v[1]:
            return lo
    return None


# ---- families ---------------------------------------------------------------------------------------------------------


def _quat(rng, nonunit):
    q = rng.standard_normal(4)
    q /= np.linalg.norm(q)
    if nonunit:
        q *= math.sqrt(rng.uniform(0.995, 1.004))  # |q|^2 <= 1.01 keeps the filter on (nvc_filter.cuh, build_record)
    return q.astype(np.float32)


def _h(x):
    return np.float16(x).view(np.uint16)


def _pow2(x, lo=-24, hi=15):
    return float(2.0 ** min(max(round(math.log2(x)), lo), hi))


class _Maker:
    """Shared placement: a sphere of view radius ~r at view-space point c, scale s, orientation q."""

    def __init__(self, rng, setup):
        self.rng, self.st = rng, setup

    def base(self, kind, indicator, c, r, sweep, backface=True, lc_zero=None, s=None, window=None, cone=None):
        rng, st = self.rng, self.st
        s = float(np.float32(s if s is not None else 10.0 ** rng.uniform(-3, 3)))
        q = _quat(rng, rng.random() < 0.35)
        lc_zero = (sweep[0] == "scale") if lc_zero is None else lc_zero
        if kind == "cluster":
            rl = _pow2(r / s) if sweep[0] == "scale" else float(np.float16(r / s))
            lc = np.zeros(3) if lc_zero else np.float16(rng.uniform(-1, 1, 3) * rl).astype(np.float64)
        else:
            rl = float(np.float32(r / s)) if sweep[0] != "scale" else _pow2(r / s, -60, 60)
            lc = np.zeros(3) if lc_zero else np.float32(rng.uniform(-1, 1, 3) * rl).astype(np.float64)
        r = rl * s
        b = Base(st, kind, indicator, sweep, 0.0, 0.0, backface)
        c = np.asarray(c(r) if callable(c) else c, np.float64)
        pos = st.world(c) - _rotate64(lc, q) * s
        b.draw["position"] = pos.astype(np.float32)
        b.draw["scale"] = s
        b.draw["orientation"] = q
        m, ml = b.mesh, b.meshlets
        m["lodCount"] = 1
        m["lods"]["meshletCount"][0, :2] = 1
        m["lods"]["meshletOffset"][0, 1] = 1
        m["lods"]["indexCount"][0, :2] = 3
        m["lods"]["indexOffset"][0, 1] = 3
        ml["vertexCount"], ml["triangleCount"] = 3, 1
        if kind == "cluster":
            ml["center"][0] = [_h(x) for x in lc]
            ml["radius"][0] = _h(rl)
            # the draw's own sphere contains the camera: drawcull passes it on every rung
            m["radius"] = np.float32(8.0 * (np.linalg.norm(c) + r + 1.0) / s)
        else:
            m["center"] = lc.astype(np.float32)
            m["radius"] = np.float32(rl)
            ml["center"][:] = [_h(x) for x in lc]
            ml["radius"][:] = _h(min(rl, 60000.0))
        ax = rng.standard_normal(3)
        ml["cone_axis"][:] = np.rint(ax / np.linalg.norm(ax) * 127).astype(np.int8)
        ml["cone_cutoff"][:] = 127  # never back-facing: only the cone family tests the cone
        if cone is not None:
            ml["cone_axis"][0], ml["cone_cutoff"][0] = cone
        if sweep[0] == "position":
            b.p0 = float(b.draw["position"][0, sweep[1]])
            b.window = window if window is not None else 2.0 * r
        elif sweep[0] == "scale":
            b.p0, b.window = s, (window if window is not None else 0.45) * s
        return b

    def axis_for(self, i):
        """world axis that moves view-space component i the most"""
        return int(np.argmax(np.abs(self.st.M[i])))


def _frustum_base(mk, kind, rng):
    st = mk.st
    f = st.frustum
    plane = ["left", "right", "top", "bottom", "near", "far"][rng.integers(0, 6 if kind == "draw" else 4)]
    z0 = rng.uniform(2.0, 150.0)
    r = z0 * rng.uniform(0.005, 0.08)
    sweep_scale = rng.random() < 0.5
    if plane in ("left", "right"):
        sg = -1 if plane == "left" else 1
        c = lambda r: [sg * (z0 * f[1] + r) / f[0], (1 - 2 * rng.uniform(0.3, 0.7)) * z0 / st.P11, z0]
        ind, comp = "frustum_x", 0
    elif plane in ("top", "bottom"):
        sg = -1 if plane == "bottom" else 1
        c = lambda r: [(2 * rng.uniform(0.3, 0.7) - 1) * z0 / st.P00, sg * (z0 * f[3] + r) / f[2], z0]
        ind, comp = "frustum_y", 1
    elif plane == "near":
        r = rng.uniform(0.05, 5.0)
        c = lambda r: [0.0, 0.0, st.znear - r]
        ind, comp = "near", 2
    else:
        r = st.zfar * rng.uniform(0.002, 0.05)
        c = lambda r: [0.0, 0.35 * (st.zfar + r) / st.P11, st.zfar + r]
        ind, comp = "far", 2
    sweep = ("scale",) if sweep_scale else ("position", mk.axis_for(comp))
    return mk.base(kind, ind, c, r, sweep)


def _cone_base(mk, rng):
    st = mk.st
    for _ in range(100):
        axis = rng.standard_normal(3)
        a8 = np.rint(axis / np.linalg.norm(axis) * 127).astype(np.int8)
        k8 = int(rng.integers(-60, 115))
        q = _quat(rng, rng.random() < 0.35)
        a = st.M @ _rotate64(a8.astype(np.float64) / 127.0, q)  # view-space axis (approximately unit)
        a /= np.linalg.norm(a)
        kd = k8 / 127.0 + rng.uniform(0.02, 0.2)
        if kd >= 0.999:
            continue
        p = rng.standard_normal(3)
        p -= p.dot(a) * a
        p /= np.linalg.norm(p)
        d = kd * a + math.sqrt(1 - kd * kd) * p
        if d[2] < 0.6 or abs(d[0]) * st.P00 > 0.8 * d[2] or abs(d[1]) * st.P11 > 0.8 * d[2]:
            continue
        z = rng.uniform(3.0, 120.0)
        r = z * (kd - k8 / 127.0)
        b = mk.base("cluster", "cone", d * z, r, ("position", int(rng.integers(0, 3))), cone=(a8, k8))
        b.draw["orientation"] = q
        b.draw["position"] = (st.world(d * z) - _rotate64(_lc(b), q) * float(b.draw["scale"][0])).astype(np.float32)
        b.p0 = float(b.draw["position"][0, b.sweep[1]])
        return b
    raise RuntimeError("no cone base")


def _lc(b):
    return np.array([float(np.uint16(x).view(np.float16)) for x in b.meshlets["center"][0]])


def _occlusion_base(mk, kind, indicator, rng):
    st = mk.st
    if indicator in ("ok",):  # zone A: depth 1.0 (an occluder at the near plane)
        u0, u1, v0, v1, _ = st.zone(0)
        u, v = rng.uniform(u0 + 0.05, u1 - 0.05), rng.uniform(v0 + 0.05, v1 - 0.05)
        r = st.znear * rng.uniform(0.002, 0.05)
        c = lambda r: st.view_point(u, v, st.znear + r)
        comp = 2
    elif indicator == "depth":  # inside zone B, view depth around the occluder's
        u0, u1, v0, v1, dval = st.zone(1)
        u, v = rng.uniform(u0 + 0.05, u1 - 0.05), rng.uniform(v0 + 0.05, v1 - 0.05)
        zb = st.znear / dval
        r = zb * rng.uniform(0.001, 0.02)
        c = lambda r: st.view_point(u, v, zb + r)
        comp = 2
    else:  # mip / fits / footprint: across the right edge of zone B, behind its occluder
        u0, u1, v0, v1, dval = st.zone(1)
        zb = st.znear / dval
        z0 = zb * rng.uniform(1.2, 3.5)
        r = z0 * 10.0 ** rng.uniform(-3.0, -1.3)
        if indicator == "footprint":
            # mip 0 (m <= 1): above it the box of the selected level never centres on a texel (there the finer level would
            # fit), so only there do the sampler's texel pairs swap through the single-texel state fract(x) == 0
            r = z0 * 10.0 ** rng.uniform(-3.6, -2.8)
        # the zone's edge within a few projected radii of the centre: texels on both sides of it enter the footprints
        u, v = u1 + rng.uniform(-2.0, 2.0) * 0.5 * st.P00 * r / z0, rng.uniform(v0 + 0.1, v1 - 0.1)
        if indicator == "footprint":
            u = u1 + rng.uniform(-1.5, 1.5) / float(st.cd.pyramidWidth)
        c = lambda r: st.view_point(u, v, z0)
        comp = 0
    if indicator == "mip" or (indicator in ("ok", "depth") and rng.random() < 0.4):
        sweep = ("scale",)
    else:
        sweep = ("position", mk.axis_for(comp))
    b = mk.base(kind, indicator, c, r, sweep, lc_zero=None if indicator != "mip" else rng.random() < 0.5)
    if indicator == "footprint":  # +-3 mip-0 texels around the edge
        b.window = 6.0 * z0 / (st.P00 * float(st.cd.pyramidWidth)) / abs(st.M[0, sweep[1]])
    return b


def _tiny_base(mk, rng):
    st = mk.st
    indicator = ["ok", "depth", "near"][rng.integers(0, 3)]
    s = float(2.0 ** rng.choice([-39.5, -39.0, -38.0, -41.0]))  # 2^-41: below the filter's scale range (exact path only)
    rl = float(np.float16(2.0 ** rng.uniform(-24, -14)))
    r = rl * s
    if indicator == "ok":
        u0, u1, v0, v1, _ = st.zone(0)
        u, v = rng.uniform(u0 + 0.05, u1 - 0.05), rng.uniform(v0 + 0.05, v1 - 0.05)
        c = lambda r: st.view_point(u, v, st.znear + r)  # c.z^2 - r^2 ~ 2 r znear: subnormal
    elif indicator == "depth":
        u0, u1, v0, v1, dval = st.zone(1)
        u, v = rng.uniform(u0 + 0.05, u1 - 0.05), rng.uniform(v0 + 0.05, v1 - 0.05)
        c = lambda r: st.view_point(u, v, st.znear / dval + r)
    else:
        c = lambda r: [0.0, 0.0, st.znear - r]
    sweep = ("position", 2) if rng.random() < 0.6 else ("scale",)
    b = mk.base("cluster", indicator, c, r, sweep, s=s, lc_zero=True)
    if sweep[0] == "position":
        b.window = 4.0 * max(r, st.znear)
    return b


def _lod_base(mk, rng, edge):
    st = mk.st
    z0 = rng.uniform(3.0, 150.0)
    b = mk.base("draw", "lod", st.view_point(rng.uniform(0.1, 0.9), rng.uniform(0.02, 0.15), z0), z0 * rng.uniform(0.005, 0.05), ("error",))
    m = b.mesh
    m["lodCount"] = 2
    m["lods"]["meshletCount"][0, 1] = 1
    m["lods"]["meshletOffset"][0, 1] = 1
    m["lods"]["indexCount"][0, 1] = 3
    m["lods"]["indexOffset"][0, 1] = 3
    if edge:
        # NaN position: distance = max(NaN, 0) = 0 (IEEE maxNum), threshold 0, so a negative error selects the LOD
        comp = rng.integers(0, 3)
        b.draw["position"][0, comp] = np.nan
        b.p0, b.window = 0.0, 1e-3
        return b
    _, verdict = _probe(b, np.array([0.0], np.float32))
    c = st.M @ b.draw["position"][0].astype(np.float64) + st.T
    thr = (np.linalg.norm(c) - float(m["radius"][0]) * float(b.draw["scale"][0])) * st.cd.lodTarget / float(b.draw["scale"][0])
    b.p0, b.window = thr, 0.5 * abs(thr) + 1e-30
    return b


FAMILIES = {
    # name: (setups, kind, maker(mk, rng) -> Base)
    "frustum": (("square", "hd_rotated"), "cluster", lambda mk, rng: _frustum_base(mk, "cluster", rng)),
    "near_far": (("square", "hd_rotated"), "cluster", lambda mk, rng: _frustum_base_nf(mk, "cluster", rng)),
    "cone": (("square", "hd_rotated"), "cluster", _cone_base),
    "project_ok": (("square", "hd_rotated"), "cluster", lambda mk, rng: _occlusion_base(mk, "cluster", "ok", rng)),
    "mip_level": (("square", "hd_rotated"), "cluster", lambda mk, rng: _occlusion_base(mk, "cluster", "mip", rng)),
    "fits": (("square", "hd_rotated"), "cluster", lambda mk, rng: _occlusion_base(mk, "cluster", "fits", rng)),
    "footprint": (("square", "hd_rotated"), "cluster", lambda mk, rng: _occlusion_base(mk, "cluster", "footprint", rng)),
    "depth_compare": (("square", "hd_rotated"), "cluster", lambda mk, rng: _occlusion_base(mk, "cluster", "depth", rng)),
    "tiny": (("tiny",), "cluster", _tiny_base),
    "draw_frustum": (("square", "hd_rotated"), "draw", lambda mk, rng: _frustum_base(mk, "draw", rng)),
    "draw_occlusion": (("square", "hd_rotated"), "draw", lambda mk, rng: _occlusion_base(mk, "draw", ["depth", "footprint", "mip", "ok"][rng.integers(0, 4)], rng)),
    "lod_select": (("square", "hd_rotated"), "draw", lambda mk, rng: _lod_base(mk, rng, False)),
    "lod_edge": (("unculled",), "draw", lambda mk, rng: _lod_base(mk, rng, True)),
}


def _frustum_base_nf(mk, kind, rng):
    """near / far planes of the cluster pass"""
    st = mk.st
    if rng.random() < 0.5:
        r = rng.uniform(0.05, 5.0)
        c, ind = (lambda r: [0.0, 0.0, st.znear - r]), "near"
    else:
        r = st.zfar * rng.uniform(0.002, 0.05)
        c, ind = (lambda r: [0.0, 0.35 * (st.zfar + r) / st.P11, st.zfar + r]), "far"
    sweep = ("scale",) if rng.random() < 0.5 else ("position", mk.axis_for(2))
    return mk.base(kind, ind, c, r, sweep)


class FamilyScene(scenes.Scene):
    """All ladders of one family on one setup.  Per draw: base[i] (index into self.bases), rung[i] (ulps from the flip's
    rung 0).  kind 'cluster': the meshlet's visibility is the verdict; 'draw': the draw's (emitted, LOD index)."""

    def __init__(self, family, setup, kind, bases, flips):
        n = len(bases) * len(RUNGS)
        meshes, meshlets, draws = [], [], []
        for b, flip in zip(bases, flips):
            m, ml, d = b.items(from_ord(flip + RUNGS))
            meshes.append(m), meshlets.append(ml), draws.append(d)
        meshes, meshlets, draws = np.concatenate(meshes), np.concatenate(meshlets), np.concatenate(draws)
        k = len(RUNGS)
        meshes["lods"]["meshletOffset"] = (meshes["lods"]["meshletOffset"] % 2) + (2 * np.arange(n, dtype=np.uint32))[:, None]
        meshes["lods"]["meshletOffset"][:, 2:] = 0
        draws["meshIndex"] = np.arange(n, dtype=np.uint32)
        bits, _ = host.visibility_offsets(draws, meshes)
        super().__init__("%s/%s" % (family, setup.name), meshes, meshlets, draws, setup.depth, setup.camera, setup.screen, bits)
        self.family, self.setup, self.kind, self.bases, self.flips = family, setup, kind, bases, flips
        self.base = np.repeat(np.arange(len(bases)), k)
        self.rung = np.tile(RUNGS, len(bases))
        self.backface = bases[0].backface

    def cull_data(self, **toggles):
        return super().cull_data(**{**self.setup.toggles, **toggles})


def generate(bases_per_setup=4, seed=2024, families=None):
    """Deterministic: {family: [FamilyScene per setup]}.  Raises when a family cannot place its bases (a generator that
    drifts off the boundaries must not pass silently)."""
    setups = _setups()
    out = {}
    for fi, (name, (setup_names, kind, maker)) in enumerate(FAMILIES.items()):
        if families and name not in families:
            continue
        out[name] = []
        for si, sname in enumerate(setup_names):
            st = setups[sname]
            rng = np.random.default_rng([seed, fi, si])
            mk = _Maker(rng, st)
            bases, flips, tries = [], [], 0
            while len(bases) < bases_per_setup:
                tries += 1
                if tries > 40 * bases_per_setup:
                    raise RuntimeError("family %s on %s: only %d of %d bases found on a boundary" % (name, sname, len(bases), bases_per_setup))
                b = maker(mk, rng)
                flip = locate(b)
                if flip is not None:
                    bases.append(b)
                    flips.append(flip)
            out[name].append(FamilyScene(name, st, kind, bases, flips))
    return out
