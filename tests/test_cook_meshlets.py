"""Widening N4 — meshlet building and packing on the device (csrc/nvc_meshlets.cuh / nvc_cook_meshlets).
The checker is the REFERENCE itself: what its cooker stored for kitten.obj, pirate.obj, pirate.glb and animated.gltf
(tests/golden/meshlet_cook.npz, kitten_cook.npz, pirate_cook.npz, kitten.nvcg, animated.raw.cache), and, for seeded
meshes, the reference's meshoptimizer (oracle/_ref/libmeshopt_cluster_ref.so: meshopt_buildMeshlets + meshopt_optimizeMeshletLevel +
meshopt_computeMeshletBounds) followed by appendMeshlet's packing.  The CPU tier runs the product's kernels under the SIMT
emulation (tests/emu_lib.py) through the C ABI; the -m gpu tier runs them on the device."""
import ctypes
import os

import numpy as np
import pytest

import emu_lib
from niagara_b200 import layout, scene_cache

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
MO_PATH = os.path.join(ROOT, "oracle", "_ref", "libmeshopt_cluster_ref.so")
needs_mo = pytest.mark.skipif(not os.path.exists(MO_PATH), reason="needs the reference's meshoptimizer (oracle/_ref/libmeshopt_cluster_ref.so)")


# ---- inputs ------------------------------------------------------------------------------------------------------------

def _vertices(positions):
    v = np.zeros((len(positions), 8), np.uint16)
    v[:, :3] = positions
    return v


def scene(name):
    """(vertices as (n, 8) uint16, indices, Mesh[], Meshlet[], meshletdata) as the reference's cooker left them"""
    if name == "animated":
        c = scene_cache.SceneCache(os.path.join(GOLDEN, "animated.raw.cache"))
        return (c.section("vertices").view(np.uint16).reshape(-1, 8).copy(), c.section("indices").astype(np.uint32), c.section("meshes").copy(),
                c.section("meshlets").copy(), c.section("meshletdata").view(np.uint32).copy())
    f = np.load(os.path.join(GOLDEN, "meshlet_cook.npz"))
    meshes = f[name + "_meshes"].reshape(-1).view(layout.MESH_DTYPE).copy()
    if name == "kitten":
        k = np.load(os.path.join(GOLDEN, "kitten_cook.npz"))
        return _vertices(k["positions"]), f["kitten_indices"], meshes, layout.load_nvcg(os.path.join(GOLDEN, "kitten.nvcg"))[1], k["meshletdata"]
    p = np.load(os.path.join(GOLDEN, "pirate_cook.npz"))
    return _vertices(p[name + "_positions"]), f[name + "_indices"], meshes, p[name + "_meshlets"].reshape(-1).view(layout.MESHLET_DTYPE).copy(), p[name + "_meshletdata"]


def scrub(meshes):
    """the LODs' meshlet fields overwritten: the call must fill them (those past lodCount are passed through)"""
    m = meshes.copy()
    for k in range(len(m)):
        m["lods"][k, : int(m[k]["lodCount"])]["meshletOffset"] = 0xDEAD
        m["lods"][k, : int(m[k]["lodCount"])]["meshletCount"] = 0xBEEF
    return m


def meaningful_words(meshlets, words):
    """uint32 mask of the meshletdata bits the cooker defines: all but the bytes past triangleCount * 3 in a last triangle word"""
    mask = np.full(words, 0xFFFFFFFF, np.uint32)
    for m in meshlets:
        refs = (int(m["vertexCount"]) + 1) // 2 if m["shortRefs"] else int(m["vertexCount"])
        tb = int(m["triangleCount"]) * 3
        if tb % 4:
            mask[int(m["dataOffset"]) + refs + tb // 4] = (1 << (8 * (tb % 4))) - 1
    return mask


def assert_same(got, want, what):
    gm, gl, gd, gt = got
    wm, wl, wd = want
    assert gt[0] == len(wl) and gt[1] == len(wd) and gt[2] == 0 and gt[3] == 0, (what, gt, len(wl), len(wd))
    assert gm.tobytes() == wm.tobytes(), (what, "meshes", gm["lods"], wm["lods"])
    g = gl.view(np.uint8).reshape(-1, 24)
    w = wl.view(np.uint8).reshape(-1, 24)
    bad = np.nonzero((g != w).any(1))[0]
    assert len(bad) == 0, (what, "meshlets", len(bad), bad[:5], gl[bad[:3]], wl[bad[:3]])
    mask = meaningful_words(wl, len(wd))
    bad = np.nonzero((gd & mask) != (wd & mask))[0]
    assert len(bad) == 0, (what, "meshletdata", len(bad), bad[:5])


# ---- the product, emulated (host pointers) or on the device ---------------------------------------------------------------

def capacity(lib, meshes):
    ml, words = ctypes.c_uint32(), ctypes.c_uint64()
    assert lib.nvc_cook_meshlets_capacity(meshes.ctypes.data, len(meshes), ctypes.byref(ml), ctypes.byref(words)) == 0
    return ml.value, words.value


class Emu:
    def __init__(self):
        self.lib = emu_lib.load()
        self.ctx = ctypes.c_void_p()
        assert self.lib.nvc_create(0, None, ctypes.byref(self.ctx)) == 0

    def close(self):
        self.lib.nvc_destroy(self.ctx)

    def cook(self, vertices, indices, meshes, cap=None, data_cap=None, index_count=None):
        """(meshes, Meshlet[], meshletdata, totals4); status != 0 raises"""
        if cap is None or data_cap is None:
            ml, words = capacity(self.lib, meshes)
            cap = ml if cap is None else cap
            data_cap = words if data_cap is None else data_cap
        out_meshes = np.zeros(len(meshes), layout.MESH_DTYPE)
        meshlets = np.full((cap + 4) * 24, 0xAB, np.uint8)
        data = np.full(data_cap + 4, 0xA5A5A5A5, np.uint32)
        totals = np.full(4, 0x77, np.uint32)
        vertices = np.ascontiguousarray(vertices)
        indices = np.ascontiguousarray(indices, np.uint32)
        status = self.lib.nvc_cook_meshlets(self.ctx, None, vertices.ctypes.data, len(vertices), indices.ctypes.data if len(indices) else None,
                                            len(indices) if index_count is None else index_count, meshes.ctypes.data, out_meshes.ctypes.data, len(meshes),
                                            meshlets.ctypes.data, cap, data.ctypes.data, data_cap, totals.ctypes.data)
        if status != 0:
            raise ValueError(status)
        assert (meshlets[cap * 24:] == 0xAB).all() and (data[data_cap:] == 0xA5A5A5A5).all(), "write past the capacity"
        n, w = int(totals[0]), int(totals[1])
        if totals[3]:
            return out_meshes, None, None, totals
        return out_meshes, meshlets[: n * 24].view(layout.MESHLET_DTYPE), data[:w], totals


class Gpu:
    def __init__(self):
        import torch

        from niagara_b200.lib import check, load_library

        self.torch, self.check = torch, check
        self.lib = load_library()
        self.ctx = ctypes.c_void_p()
        check(self.lib.nvc_create(0, None, ctypes.byref(self.ctx)), None, "nvc_create")

    def close(self):
        self.lib.nvc_destroy(self.ctx)

    def cook(self, vertices, indices, meshes):
        torch = self.torch
        ml, words = capacity(self.lib, meshes)
        dv = torch.from_numpy(np.ascontiguousarray(vertices).view(np.uint8).reshape(-1).copy()).cuda()
        di = torch.from_numpy(np.ascontiguousarray(indices, np.uint32).view(np.int32).copy()).cuda()
        dm = torch.zeros(len(meshes) * 208, dtype=torch.uint8, device="cuda")
        dl = torch.full((ml * 24 + 1,), 0xAB, dtype=torch.uint8, device="cuda")
        dd = torch.full((words + 1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        dt = torch.zeros(4, dtype=torch.int32, device="cuda")
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        self.check(self.lib.nvc_cook_meshlets(self.ctx, stream, dv.data_ptr(), len(vertices), di.data_ptr(), len(indices), meshes.ctypes.data, dm.data_ptr(), len(meshes),
                                              dl.data_ptr(), ml, dd.data_ptr(), words, dt.data_ptr()), self.ctx, "nvc_cook_meshlets")
        torch.cuda.synchronize()
        t = dt.cpu().numpy().view(np.uint32)
        n, w = int(t[0]), int(t[1])
        return (dm.cpu().numpy().view(layout.MESH_DTYPE), dl.cpu().numpy()[: n * 24].view(layout.MESHLET_DTYPE), dd.cpu().numpy().view(np.uint32)[:w], t)


# ---- the reference: its meshoptimizer + appendMeshlet's packing --------------------------------------------------------------

class MeshoptMeshlet(ctypes.Structure):
    _fields_ = [("vertex_offset", ctypes.c_uint), ("triangle_offset", ctypes.c_uint), ("vertex_count", ctypes.c_uint), ("triangle_count", ctypes.c_uint)]


class Bounds(ctypes.Structure):
    _fields_ = [("center", ctypes.c_float * 3), ("radius", ctypes.c_float), ("cone_apex", ctypes.c_float * 3), ("cone_axis", ctypes.c_float * 3),
                ("cone_cutoff", ctypes.c_float), ("cone_axis_s8", ctypes.c_byte * 3), ("cone_cutoff_s8", ctypes.c_byte)]


def meshopt():
    mo = ctypes.CDLL(MO_PATH)
    mo.meshopt_buildMeshletsBound.restype = ctypes.c_size_t
    mo.meshopt_buildMeshletsBound.argtypes = [ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t]
    mo.meshopt_buildMeshlets.restype = ctypes.c_size_t
    mo.meshopt_buildMeshlets.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t,
                                         ctypes.c_size_t, ctypes.c_size_t, ctypes.c_float]
    mo.meshopt_optimizeMeshletLevel.restype = None
    mo.meshopt_optimizeMeshletLevel.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
    mo.meshopt_computeMeshletBounds.restype = Bounds
    mo.meshopt_computeMeshletBounds.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t]
    mo.meshopt_quantizeHalf.restype = ctypes.c_ushort
    mo.meshopt_quantizeHalf.argtypes = [ctypes.c_float]
    return mo


def dequantize(h):
    """meshopt_dequantizeHalf: fp16 denormals flush to (signed) zero"""
    f = h.view(np.float16).astype(np.float32)
    small = (h & 0x7FFF) < 0x400
    f[small] = np.copysign(np.float32(0), f[small])
    return f


def reference_cook(mo, vertices, indices, meshes):
    """appendMesh's meshlet loop (scene.cpp:270-276 -> appendMeshlets -> appendMeshlet) with the reference's library"""
    out = meshes.copy()
    meshlets, data = [], []
    for mi, mesh in enumerate(meshes):
        vo, vc = int(mesh["vertexOffset"]), int(mesh["vertexCount"])
        pos = np.ascontiguousarray(dequantize(np.ascontiguousarray(vertices[vo: vo + vc, :3])))
        for li in range(int(mesh["lodCount"])):
            lod = mesh["lods"][li]
            idx = np.ascontiguousarray(indices[int(lod["indexOffset"]): int(lod["indexOffset"]) + int(lod["indexCount"])], np.uint32)
            n = len(idx)
            bound = mo.meshopt_buildMeshletsBound(n, 64, 24)
            ml = (MeshoptMeshlet * max(bound, 1))()
            mv = np.zeros(max(n, 1), np.uint32)
            mt = np.zeros(max(n, 1) + 4, np.uint8)
            count = mo.meshopt_buildMeshlets(ml, mv.ctypes.data, mt.ctypes.data, idx.ctypes.data, n, pos.ctypes.data, vc, 12, 64, 96, 0.25) if n else 0
            out["lods"][mi, li]["meshletOffset"] = len(meshlets)
            out["lods"][mi, li]["meshletCount"] = count
            for k in range(count):
                m = ml[k]
                mo.meshopt_optimizeMeshletLevel(mv.ctypes.data + 4 * m.vertex_offset, m.vertex_count, mt.ctypes.data + m.triangle_offset, m.triangle_count, 1)
                refs = mv[m.vertex_offset: m.vertex_offset + m.vertex_count].astype(np.int64)
                lo, hi = int(refs.min()), int(refs.max())
                short = hi - lo < (1 << 16)
                r = (refs - lo).astype(np.uint32)
                if short:
                    w = np.zeros((len(r) + 1) // 2, np.uint32)
                    w.view(np.uint16)[: len(r)] = r
                else:
                    w = r
                t = np.zeros((m.triangle_count * 3 + 3) // 4, np.uint32)
                t.view(np.uint8)[: m.triangle_count * 3] = mt[m.triangle_offset: m.triangle_offset + m.triangle_count * 3]
                b = mo.meshopt_computeMeshletBounds(mv.ctypes.data + 4 * m.vertex_offset, mt.ctypes.data + m.triangle_offset, m.triangle_count, pos.ctypes.data, vc, 12)
                rec = np.zeros(1, layout.MESHLET_DTYPE)
                rec["center"] = [mo.meshopt_quantizeHalf(b.center[q]) for q in range(3)]
                rec["radius"] = mo.meshopt_quantizeHalf(b.radius)
                rec["cone_axis"] = [b.cone_axis_s8[q] for q in range(3)]
                rec["cone_cutoff"] = b.cone_cutoff_s8
                rec["dataOffset"] = sum(len(d) for d in data)
                rec["baseVertex"] = vo + lo
                rec["vertexCount"], rec["triangleCount"], rec["shortRefs"] = m.vertex_count, m.triangle_count, int(short)
                meshlets.append(rec)
                data += [w, t]
    ml = np.concatenate(meshlets) if meshlets else np.zeros(0, layout.MESHLET_DTYPE)
    return out, ml, (np.concatenate(data) if data else np.zeros(0, np.uint32))


# ---- seeded meshes ----------------------------------------------------------------------------------------------------------

def half(x):
    return np.asarray(x, np.float32).astype(np.float16).view(np.uint16)


def grid(rng, gx, gy, scale=1.0):
    u, v = np.meshgrid(np.linspace(0, 1, gx), np.linspace(0, 1, gy))
    pos = np.stack([u.reshape(-1), v.reshape(-1), 0.1 * np.sin(3 * u.reshape(-1)) * np.cos(2 * v.reshape(-1))], 1) * scale
    pos += rng.uniform(-0.2, 0.2, pos.shape) * scale / max(gx, gy)
    q = np.arange((gx - 1) * (gy - 1))
    x, y = q % (gx - 1), q // (gx - 1)
    a, b, c, d = y * gx + x, y * gx + x + 1, (y + 1) * gx + x, (y + 1) * gx + x + 1
    return pos, np.stack([a, b, c, c, b, d], 1).reshape(-1)


def seeded_mesh(rng, kind):
    """(fp16 positions (n, 3), list of LOD index arrays)"""
    if kind == "grid":
        pos, idx = grid(rng, int(rng.integers(3, 30)), int(rng.integers(3, 30)), rng.uniform(0.1, 50))
        lods = [idx]
    elif kind == "pieces":  # disconnected patches: the kd-tree restarts the flow
        parts, base = [], 0
        ps = []
        for _ in range(int(rng.integers(2, 7))):
            p, i = grid(rng, int(rng.integers(2, 9)), int(rng.integers(2, 9)))
            ps.append(p + rng.uniform(-5, 5, (1, 3)))
            parts.append(i + base)
            base += len(p)
        pos, lods = np.concatenate(ps), [np.concatenate(parts)]
        perm = rng.permutation(len(lods[0]) // 3)
        lods = [lods[0].reshape(-1, 3)[perm].reshape(-1)]
    elif kind == "sparse":  # LODs that use a few of many vertices (vertex_count > index_count)
        pos, idx = grid(rng, 40, 40)
        tris = idx.reshape(-1, 3)
        lods = [tris[rng.choice(len(tris), int(rng.integers(1, 30)), replace=False)].reshape(-1), tris[:: int(rng.integers(7, 40))].reshape(-1)]
    elif kind == "long":  # vertices more than 65536 apart: shortRefs = 0
        p, idx = grid(rng, 12, 12)
        pos = np.concatenate([p[:72], rng.uniform(-1, 1, (70000, 3)), p[72:]])
        idx = np.where(idx >= 72, idx + 70000, idx)
        lods = [idx]
    elif kind == "degenerate":  # duplicated and zero-area triangles, a LOD of zero area only
        pos, idx = grid(rng, 8, 8)
        tris = idx.reshape(-1, 3)
        dup = tris[rng.integers(0, len(tris), 20)]
        flat = tris[rng.integers(0, len(tris), 10)][:, [0, 0, 1]]
        all_t = np.concatenate([tris, dup, flat])
        lods = [all_t[rng.permutation(len(all_t))].reshape(-1), np.tile(np.array([3, 3, 3, 5, 5, 7], np.int64), 4)]
    elif kind == "tiny":  # single-triangle and empty LODs
        pos, idx = grid(rng, 3, 3)
        lods = [idx[:3], np.zeros(0, np.int64), idx]
    elif kind == "vertexfull":  # a triangle soup over few shared vertices: meshlets fill to 64 vertices
        pos = rng.standard_normal((150, 3))
        lods = [rng.integers(0, 150, 1200)]
    elif kind == "trianglefull":  # a closed dense fan strip: meshlets fill to 96 triangles with few vertices
        n = 40
        a = np.linspace(0, 2 * np.pi, n, endpoint=False)
        ring = np.stack([np.cos(a), np.sin(a), np.zeros(n)], 1)
        pos = np.concatenate([ring, ring * 0.5 + [0, 0, 0.3], ring * 0.25 + [0, 0, 0.5]])
        t = []
        for r in range(2):
            for i in range(n):
                j = (i + 1) % n
                p, q, s, u = r * n + i, r * n + j, (r + 1) * n + i, (r + 1) * n + j
                t += [p, q, s, s, q, u]
        base = np.array(t).reshape(-1, 3)
        lods = [np.tile(base, (3, 1)).reshape(-1)]
    else:  # many LODs: decimated copies of a grid
        pos, idx = grid(rng, 20, 20)
        tris = idx.reshape(-1, 3)
        lods = [tris[:: k + 1].reshape(-1) for k in range(8)]
    return half(pos).reshape(-1, 3), [np.asarray(l, np.uint32) for l in lods]


KINDS = ["grid", "pieces", "sparse", "long", "degenerate", "tiny", "vertexfull", "trianglefull", "lods"]


def seeded_scene(seed, kinds=KINDS):
    """several meshes with up to 8 LODs each, as one call's vb / ib / Mesh[]"""
    rng = np.random.default_rng(seed)
    verts, idx, meshes = [], [], []
    vbase = ibase = 0
    for kind in kinds:
        pos, lods = seeded_mesh(rng, kind)
        m = np.zeros(1, layout.MESH_DTYPE)
        m["vertexOffset"], m["vertexCount"], m["lodCount"] = vbase, len(pos), len(lods)
        for li, l in enumerate(lods):
            m["lods"][0, li]["indexOffset"] = ibase
            m["lods"][0, li]["indexCount"] = len(l)
            idx.append(l)
            ibase += len(l)
        m["lods"]["meshletOffset"] = 0x1234
        verts.append(_vertices(pos))
        vbase += len(pos)
        meshes.append(m)
    return np.concatenate(verts), np.concatenate(idx).astype(np.uint32), np.concatenate(meshes)


# ---- CPU tier -------------------------------------------------------------------------------------------------------------

def test_emulated_cook_reproduces_reference_cooker():
    """animated.gltf, pirate.obj and pirate.glb cooked from their vertices, indices and Mesh[] (meshlet fields scrubbed):
    Mesh[], Meshlet[] and meshletdata equal the reference cooker's in every byte but the unread padding."""
    e = Emu()
    try:
        for name in ("animated", "pirate", "pirateglb"):
            v, i, meshes, ml, md = scene(name)
            got = e.cook(v, i, scrub(meshes))
            assert_same(got, (meshes, ml, md), name)
    finally:
        e.close()


@needs_mo
def test_emulated_cook_against_reference_library():
    """Seeded meshes (grid patches, disconnected pieces, sparse LODs, long references, duplicate and zero-area triangles,
    single-triangle and empty LODs, meshlets full by vertices and by triangles, 8 LODs) in one call: equal to the reference's
    meshopt_buildMeshlets + meshopt_optimizeMeshletLevel + appendMeshlet packing."""
    mo = meshopt()
    e = Emu()
    try:
        for seed in range(3):
            v, i, meshes = seeded_scene(seed)
            want = reference_cook(mo, v, i, meshes)
            got = e.cook(v, i, scrub(meshes))
            assert_same(got, want, seed)
            wl = want[1]
            assert (wl["shortRefs"] == 0).any() and (wl["vertexCount"] == 64).any() and (wl["triangleCount"] == 96).any(), seed
    finally:
        e.close()


def test_emulated_capacity_bounds_and_overflow():
    """The capacity helper bounds every LOD; a call short of either capacity writes nothing there and sets the flag."""
    e = Emu()
    try:
        for name in ("animated", "pirate"):
            v, i, meshes, ml, md = scene(name)
            cap, words = capacity(e.lib, meshes)
            assert len(ml) <= cap and len(md) <= words
            for c, w in ((len(ml) - 1, None), (None, len(md) - 1), (0, 0)):
                gm, gl, gd, t = e.cook(v, i, scrub(meshes), cap=c, data_cap=w)
                assert gl is None and t[3] == 1 and t[0] == len(ml) and t[1] == len(md)
                assert gm.tobytes() == meshes.tobytes()  # Mesh[] is still written
        for seed in range(2):
            v, i, meshes = seeded_scene(10 + seed)
            cap, words = capacity(e.lib, meshes)
            _, gl, gd, t = e.cook(v, i, meshes)
            assert t[3] == 0 and t[0] <= cap and t[1] <= words
    finally:
        e.close()


def test_emulated_rejects_bad_input():
    """Host checks: lodCount > 8, indexCount % 3, index and vertex ranges.  Device check: an index >= vertexCount rejects its
    LOD only (0 meshlets, counted), without reading past the vertices."""
    e = Emu()
    try:
        v, i, meshes = seeded_scene(20, ["grid", "tiny"])
        for field, value in (("lodCount", 9), ("vertexCount", len(v) + 1)):
            bad = meshes.copy()
            bad[0][field] = value
            with pytest.raises(ValueError):
                e.cook(v, i, bad, cap=0, data_cap=0)
        for field, value in (("indexCount", 4), ("indexOffset", len(i))):
            bad = meshes.copy()
            bad["lods"][0, 0][field] = value
            with pytest.raises(ValueError):
                e.cook(v, i, bad, cap=0, data_cap=0)
        with pytest.raises(ValueError):
            e.cook(v, i, meshes, index_count=len(i) - 3)
        bad = meshes.copy()
        bad[0]["lodCount"] = 9
        with pytest.raises(AssertionError):
            capacity(e.lib, bad)
        bad_i = i.copy()
        lod = meshes["lods"][1, 2]
        bad_i[int(lod["indexOffset"]) + 4] = meshes[1]["vertexCount"]
        gm, gl, gd, t = e.cook(v, bad_i, meshes)
        assert t[2] == 1 and gm["lods"][1, 2]["meshletCount"] == 0
        good = e.cook(v, i, meshes)
        assert gm["lods"][0].tobytes() == good[0]["lods"][0].tobytes()
        keep = good[0]["lods"][1, 2]["meshletCount"]
        assert t[0] == good[3][0] - keep
    finally:
        e.close()


# ---- GPU tier -------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_gpu_cook_reproduces_reference_cooker():
    """kitten.obj (792 meshlets over 8 LODs), pirate.obj, pirate.glb and animated.gltf cooked on the device: Mesh[],
    Meshlet[] and meshletdata equal the reference cooker's in every byte but the unread padding."""
    g = Gpu()
    try:
        for name in ("kitten", "pirate", "pirateglb", "animated"):
            v, i, meshes, ml, md = scene(name)
            assert_same(g.cook(v, i, scrub(meshes)), (meshes, ml, md), name)
        assert len(scene("kitten")[3]) == 792
    finally:
        g.close()


@pytest.mark.gpu
@needs_mo
def test_gpu_cook_against_reference_library():
    mo = meshopt()
    g = Gpu()
    try:
        for seed in range(6):
            v, i, meshes = seeded_scene(100 + seed)
            assert_same(g.cook(v, i, scrub(meshes)), reference_cook(mo, v, i, meshes), seed)
    finally:
        g.close()


@pytest.mark.gpu
def test_gpu_many_meshes_equal_single_mesh_calls():
    """One call over many meshes gives each mesh the bytes it gets alone, moved by its meshlet and data offsets."""
    g = Gpu()
    try:
        v, i, meshes = seeded_scene(7, KINDS * 3)
        gm, gl, gd, t = g.cook(v, i, meshes)
        for k in range(len(meshes)):
            one = meshes[k: k + 1].copy()
            sm, sl, sd, _ = g.cook(v, i, one)
            first = int(gm["lods"][k, 0]["meshletOffset"])
            n = len(sl)
            got = gl[first: first + n].copy()
            assert np.array_equal(gm["lods"][k]["meshletCount"], sm["lods"][0]["meshletCount"])
            if n:
                d0 = int(got["dataOffset"][0])
                assert np.array_equal(got["dataOffset"] - d0, sl["dataOffset"])
                got["dataOffset"] = sl["dataOffset"]
                assert got.tobytes() == sl.tobytes(), k
                assert np.array_equal(gd[d0: d0 + len(sd)], sd), k
    finally:
        g.close()


@pytest.mark.gpu
def test_gpu_frame_on_device_cooked_kitten():
    """A two-phase frame of the instanced kitten scene over device-cooked Mesh[] / Meshlet[] equals the same frame over
    kitten.nvcg (the reference cooker's)."""
    import torch

    from niagara_b200 import scenes
    from niagara_b200.path import VisibilityPath

    v, i, meshes, ml, md = scene("kitten")
    g = Gpu()
    try:
        gm, gl, gd, t = g.cook(v, i, scrub(meshes))
    finally:
        g.close()
    s = scenes.instanced_scene(os.path.join(GOLDEN, "kitten.nvcg"), 2048)
    outs = []
    for mesh_arr, meshlet_arr in ((s.meshes, s.meshlets), (gm.copy(), gl.copy())):
        mesh_arr = mesh_arr.copy()
        mesh_arr[["center", "radius"]] = s.meshes[["center", "radius"]]
        for k in range(len(mesh_arr)):
            mesh_arr["lods"][k]["error"] = s.meshes["lods"][k]["error"]
        p = VisibilityPath(mesh_arr, meshlet_arr, s.draws, *s.screen, device="cuda:0")
        p.set_visibility_bits(s.visibility_bits)
        depth = torch.from_numpy(s.depth).cuda()
        for _ in range(2):
            p.frame(s.cull_data(), depth, cluster_backface=True)
        torch.cuda.synchronize()
        d, c = p.read_counts()
        outs.append((d, c, p.dvb.cpu().numpy(), p.mvb.cpu().numpy(), p.depthPyramid.cpu().numpy()))
    for a, b in zip(*outs):
        assert np.array_equal(a, b)
