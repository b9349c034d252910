"""Second, independent restatement of the reference GLSL in vectorised numpy float32 — test infrastructure.

Written separately from oracle/oracle.cpp (array-at-a-time instead of item-at-a-time, numpy's float32 kernels
instead of gcc scalar code) so that an interpretation slip in one of them shows up as a disagreement.  Every float32
numpy ufunc is a single correctly-rounded IEEE operation, which is exactly the arithmetic contract of DESIGN.md.
Cites: src/shaders/math.h:1-49, drawcull.comp.glsl:54-156, clustercull.comp.glsl:56-149."""
import numpy as np

F = np.float32


def half_to_float(bits):
    return np.asarray(bits, dtype=np.uint16).view(np.float16).astype(np.float32)


def cross(a, b):
    return (
        a[1] * b[2] - b[1] * a[2],
        a[2] * b[0] - b[2] * a[0],
        a[0] * b[1] - b[0] * a[1],
    )


def rotate_quat(v, q):  # math.h:46-49
    qv = (q[0], q[1], q[2])
    c1 = cross(qv, v)
    t = tuple(c1[i] + q[3] * v[i] for i in range(3))
    c2 = cross(qv, t)
    return tuple(v[i] + F(2.0) * c2[i] for i in range(3))


def transform_point(m, p):  # (view * vec4(p, 1)).xyz, column-major
    return tuple(((m[0 + i] * p[0] + m[4 + i] * p[1]) + m[8 + i] * p[2]) + m[12 + i] for i in range(3))


def transform_vector(m, v):
    return tuple((m[0 + i] * v[0] + m[4 + i] * v[1]) + m[8 + i] * v[2] for i in range(3))


def dot3(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def length3(a):
    return np.sqrt((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2])


def frustum_visible(cd, c, r):
    v = c[2] * F(cd["frustum"][1]) - np.abs(c[0]) * F(cd["frustum"][0]) > -r
    v &= c[2] * F(cd["frustum"][3]) - np.abs(c[1]) * F(cd["frustum"][2]) > -r
    v &= (c[2] + r > F(cd["znear"])) & (c[2] - r < F(cd["zfar"]))
    return v


def project_sphere(c, r, znear, P00, P11):  # math.h:1-22
    with np.errstate(all="ignore"):
        ok = ~(c[2] < r + znear)
        crx, cry, crz = c[0] * r, c[1] * r, c[2] * r
        czr2 = c[2] * c[2] - r * r
        vx = np.sqrt(c[0] * c[0] + czr2)
        minx = (vx * c[0] - crz) / (vx * c[2] + crx)
        maxx = (vx * c[0] + crz) / (vx * c[2] - crx)
        vy = np.sqrt(c[1] * c[1] + czr2)
        miny = (vy * c[1] - crz) / (vy * c[2] + cry)
        maxy = (vy * c[1] + crz) / (vy * c[2] - cry)
        ax = (minx * P00) * F(0.5) + F(0.5)
        ay = (maxy * P11) * F(-0.5) + F(0.5)
        az = (maxx * P00) * F(0.5) + F(0.5)
        aw = (miny * P11) * F(-0.5) + F(0.5)
    return ok, (ax, ay, az, aw)


def ceil_log2_exact(x):
    """smallest integer L with 2^L >= x, x > 0 finite (np.frexp is exact: x = m * 2^e, 0.5 <= m < 1)."""
    m, e = np.frexp(x.astype(np.float64))
    return np.where(m == 0.5, e - 1, e).astype(np.int64)


def occlusion_mip(aabb, pw, ph):  # math.h:24-39
    with np.errstate(all="ignore"):
        sx = aabb[2] - aabb[0]
        sy = aabb[3] - aabb[1]
        a, b = sx * pw, sy * ph
        # GLSL leaves max() with a NaN operand undefined; like GPU hardware (FMNMX / IEEE maxNum) and the oracle, the
        # defined operand wins
        m = np.fmax(a, b)
        pos = m > 0
        L = np.where(pos & np.isfinite(m), ceil_log2_exact(np.where(pos & np.isfinite(m), m, F(1.0))), 0)
        level = np.zeros(m.shape, dtype=np.float32)
        big = pos & np.isinf(m)
        use = pos & ~big & (L > 0)
        Lc = np.where(use, L, 1)
        scale = np.ldexp(F(1.0), (1 - Lc).astype(np.int32)).astype(np.float32)
        fmx, fmy = pw * scale, ph * scale
        px, py = aabb[0] * fmx, aabb[1] * fmy
        fx, fy = px - np.floor(px), py - np.floor(py)
        fits = (fx + sx * fmx <= F(2.0)) & (fy + sy * fmy <= F(2.0))
        lv = Lc.astype(np.float32) - fits.astype(np.float32)
        level = np.where(use, np.maximum(lv, F(0.0)), level)
        level = np.where(big, F(1e9), level)
    return level.astype(np.float32)


def sample_min_level(img, u, v):
    """MIN-reduction bilinear footprint (Appendix C.3) on one 2D float32 array, vectorised over u, v."""
    h, w = img.shape
    with np.errstate(all="ignore"):
        x = u * F(w) - F(0.5)
        y = v * F(h) - F(0.5)
        x0, y0 = np.floor(x), np.floor(y)
        fx, fy = x - x0, y - y0
        cx0 = np.clip(x0, 0, w - 1).astype(np.int64)
        cy0 = np.clip(y0, 0, h - 1).astype(np.int64)
        cx1 = np.clip(x0 + F(1), 0, w - 1).astype(np.int64)
        cy1 = np.clip(y0 + F(1), 0, h - 1).astype(np.int64)
    ux, uy = fx != 0, fy != 0
    inf = np.float32(np.inf)
    t00 = img[cy0, cx0]
    t01 = np.where(ux, img[cy0, cx1], inf)
    t10 = np.where(uy, img[cy1, cx0], inf)
    t11 = np.where(ux & uy, img[cy1, cx1], inf)
    return np.minimum(np.minimum(t00, t01), np.minimum(t10, t11))


def sample_hiz(levels, u, v, level):
    lc = np.clip(level, 0, len(levels) - 1).astype(np.int64)
    out = np.zeros(u.shape, dtype=np.float32)
    for l in np.unique(lc):
        sel = lc == l
        out[sel] = sample_min_level(levels[l], u[sel], v[sel])
    return out


def occlusion_visible(cd, levels, c, r):
    ok, aabb = project_sphere(c, r, F(cd["znear"]), F(cd["P00"]), F(cd["P11"]))
    level = occlusion_mip(aabb, F(cd["pyramidWidth"]), F(cd["pyramidHeight"]))
    u = (aabb[0] + aabb[2]) * F(0.5)
    v = (aabb[1] + aabb[3]) * F(0.5)
    safe = ok & np.isfinite(u) & np.isfinite(v)
    depth = np.zeros(u.shape, dtype=np.float32)
    if safe.any():
        depth[safe] = sample_hiz(levels, u[safe], v[safe], level[safe])
    with np.errstate(all="ignore"):
        ds = F(cd["znear"]) / (c[2] - r)
    return np.where(ok, ds > depth, True)


def build_pyramid(depth, pw, ph, nlevels):
    """depthreduce.comp.glsl:14-22 chain: level l = MIN-sample of level l-1 at (pos + 0.5) / size."""
    levels = []
    src = depth.astype(np.float32)
    for l in range(nlevels):
        w, h = max(1, pw >> l), max(1, ph >> l)
        xs = (np.arange(w, dtype=np.float32) + F(0.5)) / F(w)
        ys = (np.arange(h, dtype=np.float32) + F(0.5)) / F(h)
        u, v = np.meshgrid(xs, ys)
        dst = sample_min_level(src, u.astype(np.float32), v.astype(np.float32)).astype(np.float32)
        levels.append(dst)
        src = dst
    return levels


def drawcull_decisions(cd, late, draws, meshes, dvb, levels=None):
    """Returns (reached, visible, emit, lodIndex) per draw — drawcull.comp.glsl:54-127,154-155."""
    n = int(cd["drawCount"])
    d = draws[:n]
    mesh = meshes[d["meshIndex"]]
    reached = d["postPass"] == cd["postPass"]
    if not late:
        reached &= dvb[:n] != 0
    q = tuple(d["orientation"][:, i] for i in range(4))
    mc = tuple(mesh["center"][:, i] for i in range(3))
    rc = rotate_quat(mc, q)
    center = tuple(rc[i] * d["scale"] + d["position"][:, i] for i in range(3))
    m = [F(x) for x in cd["view"]]
    center = transform_point(m, center)
    radius = mesh["radius"] * d["scale"]
    visible = frustum_visible(cd, center, radius)
    if cd["cullingEnabled"] == 0:
        visible = np.ones(n, dtype=bool)
    if late and cd["occlusionEnabled"] == 1:
        visible = visible & occlusion_visible(cd, levels, center, radius)
    cond = np.ones(n, dtype=bool) if (not late or cd["clusterOcclusionEnabled"] == 1 or cd["postPass"] != 0) else (dvb[:n] == 0)
    emit = reached & visible & cond
    lod = np.zeros(n, dtype=np.uint32)
    if cd["lodEnabled"] == 1:
        # max(NaN, 0) = 0: IEEE maxNum, as GPU hardware, the kernels and the oracle take it (a NaN draw position selects by threshold 0)
        with np.errstate(invalid="ignore"):
            dist = np.fmax(length3(center) - radius, F(0.0))
        thr = dist * F(cd["lodTarget"]) / d["scale"]
        for i in range(1, layout_max_lods(meshes)):
            sel = (i < mesh["lodCount"]) & (mesh["lods"]["error"][:, i] < thr)
            lod = np.where(sel, np.uint32(i), lod)
    return reached, visible, emit, lod


def layout_max_lods(meshes):
    return meshes["lods"].shape[1]


def cluster_decisions(cd, late, cmds, draws, meshlets, mvb, levels=None):
    """Per (command, lane) decisions of clustercull.comp.glsl:56-149 against the mvb state BEFORE the pass.
    Returns (commandId, mgi, visible, emit) flattened over valid lanes."""
    ncmd = len(cmds)
    tc = np.minimum(cmds["taskCount"], 64).astype(np.int64)
    cid = np.repeat(np.arange(ncmd, dtype=np.int64), tc)
    start = np.cumsum(tc) - tc
    mgi = np.arange(int(tc.sum()), dtype=np.int64) - np.repeat(start, tc)
    c = cmds[cid]
    mi = (c["taskOffset"].astype(np.int64) + mgi).astype(np.int64)
    mvi = (c["meshletVisibilityOffset"].astype(np.int64) + mgi).astype(np.int64)
    d = draws[c["drawId"]]
    ml = meshlets[mi]
    q = tuple(d["orientation"][:, i] for i in range(4))
    lc = tuple(half_to_float(ml["center"][:, i]) for i in range(3))
    rc = rotate_quat(lc, q)
    center = tuple(rc[i] * d["scale"] + d["position"][:, i] for i in range(3))
    m = [F(x) for x in cd["view"]]
    center = transform_point(m, center)
    radius = half_to_float(ml["radius"]) * d["scale"]
    la = tuple(ml["cone_axis"][:, i].astype(np.float32) / F(127.0) for i in range(3))
    axis = transform_vector(m, rotate_quat(la, q))
    cutoff = ml["cone_cutoff"].astype(np.float32) / F(127.0)

    visible = np.ones(len(cid), dtype=bool)
    skip = np.zeros(len(cid), dtype=bool)
    if cd["clusterOcclusionEnabled"] == 1 and cd["postPass"] == 0:
        bit = (mvb[mvi >> 5] >> (mvi & 31).astype(np.uint32)) & 1
        if not late:
            visible &= bit != 0
        else:
            skip = (c["lateDrawVisibility"] == 1) & (bit != 0)
    if cd["clusterBackfaceEnabled"] != 0:
        visible &= ~(dot3(center, axis) >= cutoff * length3(center) + radius)
    visible &= frustum_visible(cd, center, radius)
    if late and cd["clusterOcclusionEnabled"] == 1:
        visible = visible & occlusion_visible(cd, levels, center, radius)
    return cid, mgi, mi, mvi, visible, visible & ~skip
