"""Meshlet cooking of clrt builds on the device (nvc_cook_meshlets_clrt): each mesh's lodRT built with
meshopt_buildMeshletsSpatial, meshletvtx0, every other LOD as nvc_cook_meshlets.  The checker is the REFERENCE itself: what
its cooker stored in a CLRT=1 run for kitten.obj, pirate.obj, pirate.glb and animated.gltf (tests/golden/meshlet_cook_clrt.npz,
animated_clrt.z.cache) and, for seeded meshes, the reference's meshoptimizer (oracle/_ref/libmeshopt_cluster_ref.so:
meshopt_buildMeshletsSpatial / meshopt_buildMeshlets + meshopt_optimizeMeshletLevel + meshopt_computeMeshletBounds) followed by
appendMeshlet's packing.  The CPU tier runs the product's kernels under the SIMT emulation; the -m gpu tier on the device."""
import ctypes
import os

import numpy as np
import pytest

import emu_lib
import test_cook_meshlets as base
from niagara_b200 import layout, scene_cache

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
needs_mo = base.needs_mo


# ---- inputs ------------------------------------------------------------------------------------------------------------

def scene(name):
    """(vertices as (n, 8) uint16, indices, Mesh[], Meshlet[], meshletdata, meshletvtx0, max_scale) of the reference's clrt cooker;
    vertices and indices are the default build's (the LOD chain does not depend on clrt)"""
    v, i = base.scene(name)[:2]
    f = np.load(os.path.join(GOLDEN, "meshlet_cook_clrt.npz"))
    return (v, i, f[name + "_meshes"].reshape(-1).view(layout.MESH_DTYPE).copy(), f[name + "_meshlets"].reshape(-1).view(layout.MESHLET_DTYPE).copy(),
            f[name + "_meshletdata"].copy(), f[name + "_meshletvtx0"].copy(), f[name + "_max_scale"].copy())


def scrub(meshes):
    """meshlet fields and lodRT overwritten: the call must fill them"""
    m = base.scrub(meshes)
    m["lodRT"] = 0xC0DE
    return m


def lod_rt(mesh, max_scale):
    """scene.cpp:266-268 in float32"""
    rt = 0
    for i in range(int(mesh["lodCount"])):
        if np.float32(mesh["lods"][i]["error"]) * np.float32(max_scale) < np.float32(3e-3):
            rt = i
    return rt


def assert_same(got, want, what, finite_bounds_only=False):
    """finite_bounds_only: the bounds (bytes 0-11) of a meshlet whose center or radius is not finite are not compared.  On the
    device, meshlet_bounds (nvc_cook.cuh) turns NaN into other snorm8 cone bits than x86 does; that is the bounds code's, not
    the builder's, and the CPU tier compares those bytes too."""
    gm, gl, gd, gx, gt = got
    wm, wl, wd, wx = want
    assert gt[4] == len(wx) and list(gt[5:]) == [0, 0, 0], (what, gt, len(wx))
    if finite_bounds_only and len(gl) == len(wl):
        nonfinite = lambda m: ((np.concatenate([m["center"], m["radius"][:, None]], 1) & 0x7C00) == 0x7C00).any(1)
        skip = nonfinite(gl) | nonfinite(wl)
        gl = gl.copy()
        gl.view(np.uint8).reshape(-1, 24)[skip, :12] = wl.view(np.uint8).reshape(-1, 24)[skip, :12]
    base.assert_same((gm, gl, gd, gt[:4]), (wm, wl, wd), what)
    assert gx.tobytes() == wx.tobytes(), (what, "meshletvtx0", np.nonzero(gx != wx)[0][:5])


# ---- the product, emulated (host pointers) or on the device ---------------------------------------------------------------

def capacity(lib, meshes, scale):
    ml, words, vtx = ctypes.c_uint32(), ctypes.c_uint64(), ctypes.c_uint64()
    sp = None if scale is None else np.ascontiguousarray(scale, np.float32)
    assert lib.nvc_cook_meshlets_clrt_capacity(meshes.ctypes.data, None if sp is None else sp.ctypes.data, len(meshes), ctypes.byref(ml), ctypes.byref(words),
                                               ctypes.byref(vtx)) == 0
    return ml.value, words.value, vtx.value


class Emu(base.Emu):
    def cook_clrt(self, vertices, indices, meshes, scale=None, cap=None, data_cap=None, vtx_cap=None, index_count=None, vtx_null=False):
        """(meshes, Meshlet[], meshletdata, meshletvtx0, totals8); status != 0 raises"""
        c = capacity(self.lib, meshes, scale) if None in (cap, data_cap, vtx_cap) else (cap, data_cap, vtx_cap)
        cap = c[0] if cap is None else cap
        data_cap = c[1] if data_cap is None else data_cap
        vtx_cap = c[2] if vtx_cap is None else vtx_cap
        out_meshes = np.zeros(len(meshes), layout.MESH_DTYPE)
        meshlets = np.full((cap + 4) * 24, 0xAB, np.uint8)
        data = np.full(data_cap + 4, 0xA5A5A5A5, np.uint32)
        vtx = np.full(vtx_cap + 8, 0x5A5A, np.uint16)
        totals = np.full(8, 0x77, np.uint32)
        vertices = np.ascontiguousarray(vertices)
        indices = np.ascontiguousarray(indices, np.uint32)
        sp = None if scale is None else np.ascontiguousarray(scale, np.float32)
        status = self.lib.nvc_cook_meshlets_clrt(self.ctx, None, vertices.ctypes.data, len(vertices), indices.ctypes.data if len(indices) else None,
                                                 len(indices) if index_count is None else index_count, meshes.ctypes.data, None if sp is None else sp.ctypes.data,
                                                 out_meshes.ctypes.data, len(meshes), meshlets.ctypes.data, cap, data.ctypes.data, data_cap,
                                                 None if vtx_null else vtx.ctypes.data, vtx_cap, totals.ctypes.data)
        if status != 0:
            raise ValueError(status)
        assert (meshlets[cap * 24:] == 0xAB).all() and (data[data_cap:] == 0xA5A5A5A5).all() and (vtx[vtx_cap:] == 0x5A5A).all(), "write past the capacity"
        n, w, x = int(totals[0]), int(totals[1]), int(totals[4])
        if totals[3]:
            assert (meshlets == 0xAB).all() and (data == 0xA5A5A5A5).all() and (vtx == 0x5A5A).all(), "written on overflow"
            return out_meshes, None, None, None, totals
        return out_meshes, meshlets[: n * 24].view(layout.MESHLET_DTYPE), data[:w], vtx[:x], totals


class Gpu(base.Gpu):
    def cook_clrt(self, vertices, indices, meshes, scale=None):
        torch = self.torch
        ml, words, vx = capacity(self.lib, meshes, scale)
        dv = torch.from_numpy(np.ascontiguousarray(vertices).view(np.uint8).reshape(-1).copy()).cuda()
        di = torch.from_numpy(np.ascontiguousarray(indices, np.uint32).view(np.int32).copy()).cuda()
        dm = torch.zeros(len(meshes) * 208, dtype=torch.uint8, device="cuda")
        dl = torch.full((ml * 24 + 1,), 0xAB, dtype=torch.uint8, device="cuda")
        dd = torch.full((words + 1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        dx = torch.full((vx + 1,), 0x5A5A, dtype=torch.int16, device="cuda")
        dt = torch.zeros(8, dtype=torch.int32, device="cuda")
        sp = None if scale is None else np.ascontiguousarray(scale, np.float32)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        self.check(self.lib.nvc_cook_meshlets_clrt(self.ctx, stream, dv.data_ptr(), len(vertices), di.data_ptr(), len(indices), meshes.ctypes.data,
                                                   None if sp is None else sp.ctypes.data, dm.data_ptr(), len(meshes), dl.data_ptr(), ml, dd.data_ptr(), words,
                                                   dx.data_ptr(), vx, dt.data_ptr()), self.ctx, "nvc_cook_meshlets_clrt")
        torch.cuda.synchronize()
        t = dt.cpu().numpy().view(np.uint32)
        n, w, x = int(t[0]), int(t[1]), int(t[4])
        return (dm.cpu().numpy().view(layout.MESH_DTYPE), dl.cpu().numpy()[: n * 24].view(layout.MESHLET_DTYPE), dd.cpu().numpy().view(np.uint32)[:w],
                dx.cpu().numpy().view(np.uint16)[:x], t)


# ---- the reference: its meshoptimizer + appendMeshlet's packing --------------------------------------------------------------

def meshopt():
    mo = base.meshopt()
    mo.meshopt_buildMeshletsSpatial.restype = ctypes.c_size_t
    mo.meshopt_buildMeshletsSpatial.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                                ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_float]
    return mo


def reference_cook(mo, vertices, indices, meshes, scale=None):
    """appendMesh's lodRT choice and meshlet loop with clrt on (scene.cpp:266-276 -> appendMeshlets -> appendMeshlet)"""
    out = meshes.copy()
    meshlets, data, vtx0 = [], [], []
    for mi, mesh in enumerate(meshes):
        vo, vc = int(mesh["vertexOffset"]), int(mesh["vertexCount"])
        pos = np.ascontiguousarray(base.dequantize(np.ascontiguousarray(vertices[vo: vo + vc, :3])))
        rt = lod_rt(mesh, 1.0 if scale is None else scale[mi])
        out[mi]["lodRT"] = rt
        for li in range(int(mesh["lodCount"])):
            lod = mesh["lods"][li]
            idx = np.ascontiguousarray(indices[int(lod["indexOffset"]): int(lod["indexOffset"]) + int(lod["indexCount"])], np.uint32)
            n = len(idx)
            bound = mo.meshopt_buildMeshletsBound(n, 64, 24)
            ml = (base.MeshoptMeshlet * max(bound, 1))()
            mv = np.zeros(max(n, 1), np.uint32)
            mt = np.zeros(max(n, 1) + 4, np.uint8)
            count = 0
            if n and (idx >= vc).any():
                count = 0  # the reference asserts; the product rejects the LOD
            elif n and li == rt:
                count = mo.meshopt_buildMeshletsSpatial(ml, mv.ctypes.data, mt.ctypes.data, idx.ctypes.data, n, pos.ctypes.data, vc, 12, 64, 24, 96, 0.5)
            elif n:
                count = mo.meshopt_buildMeshlets(ml, mv.ctypes.data, mt.ctypes.data, idx.ctypes.data, n, pos.ctypes.data, vc, 12, 64, 96, 0.25)
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
                if li == rt:
                    x = np.zeros((m.vertex_count, 4), np.uint16)
                    x[:, :3] = [[mo.meshopt_quantizeHalf(float(pos[v, q])) for q in range(3)] for v in refs]
                    vtx0.append(x.reshape(-1))
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
    return (out, ml, (np.concatenate(data) if data else np.zeros(0, np.uint32)), (np.concatenate(vtx0) if vtx0 else np.zeros(0, np.uint16)))


# ---- seeded meshes ----------------------------------------------------------------------------------------------------------

def set_errors(meshes, k, target):
    """LOD errors 1e-3 * 2^l for mesh k, and the max_scale that makes lodRT = target"""
    meshes["lods"][k]["error"] = [1e-3 * 2.0**l for l in range(8)]
    return np.float32(0.75 * 3.0 / 2.0**target)


def soup(rng, triangles, spread=1.0):
    """an unindexed triangle soup of small scattered triangles: every meshlet is vertex bound"""
    centers = rng.uniform(-spread, spread, (triangles, 1, 3))
    pos = (centers + rng.uniform(-0.02, 0.02, (triangles, 3, 3))).reshape(-1, 3)
    return base.half(pos).reshape(-1, 3), np.arange(3 * triangles, dtype=np.uint32)


def special_mesh(rng):
    """a grid with fp16 NaN, +-inf, denormal and +-0 positions"""
    pos, idx = base.grid(rng, 16, 16)
    h = base.half(pos).reshape(-1, 3)
    picks = rng.choice(len(h), 60, replace=False)
    specials = np.array([0x7E00, 0x7C01, 0xFE00, 0x7C00, 0xFC00, 0x0001, 0x83FF, 0x0000, 0x8000, 0x0200], np.uint16)
    for n, p in enumerate(picks):
        h[p, int(rng.integers(0, 3))] = specials[n % len(specials)]
    return h, [np.asarray(idx, np.uint32)]


def append(scene_parts, pos, lods, errors=None):
    scene_parts.append((pos, lods, errors))


def build_scene(parts):
    verts, idx, meshes = [], [], []
    vbase = ibase = 0
    for pos, lods, errors in parts:
        m = np.zeros(1, layout.MESH_DTYPE)
        m["vertexOffset"], m["vertexCount"], m["lodCount"] = vbase, len(pos), len(lods)
        for li, l in enumerate(lods):
            m["lods"][0, li]["indexOffset"] = ibase
            m["lods"][0, li]["indexCount"] = len(l)
            idx.append(l)
            ibase += len(l)
        if errors is not None:
            m["lods"][0, : len(errors)]["error"] = errors
        m["lods"]["meshletOffset"] = 0x1234
        verts.append(base._vertices(pos))
        vbase += len(pos)
        meshes.append(m)
    return np.concatenate(verts), np.concatenate(idx).astype(np.uint32), np.concatenate(meshes)


def clrt_scene(seed):
    """seeded_scene's meshes (lodRT = their last LOD: errors 0) plus: an 8-LOD mesh per lodRT 0..7 (by max_scale), triangle soups,
    fp16 specials, all-NaN geometry, single-triangle and empty lodRT; returns (vertices, indices, Mesh[], max_scale)"""
    rng = np.random.default_rng(seed)
    v, i, meshes = base.seeded_scene(seed)
    parts = []
    for k in range(len(meshes)):
        m = meshes[k]
        vo, vc = int(m["vertexOffset"]), int(m["vertexCount"])
        lods = [i[int(l["indexOffset"]): int(l["indexOffset"]) + int(l["indexCount"])] for l in m["lods"][: int(m["lodCount"])]]
        parts.append((v[vo: vo + vc, :3], lods, None))
    scale = [1.0] * len(parts)
    lod_pos, lod_idx = base.seeded_mesh(rng, "lods")
    for target in range(8):
        parts.append((lod_pos, lod_idx, [1e-3 * 2.0**l for l in range(8)]))
        scale.append(0.75 * 3.0 / 2.0**target)
    for n in (int(rng.integers(100, 400)), 1):
        p, x = soup(rng, n)
        parts.append((p, [x], None))
        scale.append(1.0)
    parts.append(special_mesh(rng) + (None,))
    scale.append(1.0)
    nan_pos = np.full((60, 3), 0x7E00, np.uint16)
    parts.append((nan_pos, [rng.integers(0, 60, 3 * 200).astype(np.uint32)], None))
    scale.append(1.0)
    tiny_pos, tiny_lods = base.seeded_mesh(rng, "tiny")  # LODs: one triangle, empty, a grid
    for target in (0, 1):
        parts.append((tiny_pos, tiny_lods, [1e-3 * 2.0**l for l in range(3)]))
        scale.append(0.75 * 3.0 / 2.0**target)
    parts.append((tiny_pos, tiny_lods, [np.nan, 1.0, 1.0]))  # no LOD passes: lodRT 0
    scale.append(1.0)
    v, i, meshes = build_scene(parts)
    return v, i, meshes, np.asarray(scale, np.float32)


# ---- CPU tier -------------------------------------------------------------------------------------------------------------

def test_emulated_clrt_reproduces_reference_cooker():
    """animated.gltf, pirate.obj and pirate.glb cooked with their max_scale from the default build's vertices and indices (meshlet
    fields and lodRT scrubbed): Mesh[], Meshlet[], meshletdata and meshletvtx0 equal the reference's clrt cooker's."""
    e = Emu()
    try:
        for name in ("animated", "pirate", "pirateglb"):
            v, i, meshes, ml, md, mx, scale = scene(name)
            assert_same(e.cook_clrt(v, i, scrub(meshes), scale), (meshes, ml, md, mx), name)
    finally:
        e.close()


@needs_mo
def test_emulated_clrt_against_reference_library():
    """Seeded multi-mesh scenes (see clrt_scene) in one call: equal to the reference's meshopt_buildMeshletsSpatial(64, 24, 96, 0.5) for
    each lodRT and meshopt_buildMeshlets for the other LODs, then meshopt_optimizeMeshletLevel, appendMeshlet's packing and meshletvtx0."""
    mo = meshopt()
    e = Emu()
    try:
        for seed in range(2):
            v, i, meshes, scale = clrt_scene(seed)
            want = reference_cook(mo, v, i, meshes, scale)
            got = e.cook_clrt(v, i, scrub(meshes), scale)
            assert_same(got, want, seed)
            assert sorted(set(int(x) for x in got[0]["lodRT"])) == list(range(8)), seed
            wl = want[1]
            assert (wl["shortRefs"] == 0).any() and (wl["vertexCount"] == 64).any() and (wl["triangleCount"] == 96).any(), seed
            assert (want[3] == 0x7E00).any() and len(want[3]) % 4 == 0, seed
    finally:
        e.close()


@needs_mo
def test_emulated_clrt_against_reference_library_unit_cases():
    """Single meshes that each reach one part of the spatial builder: a large soup (vertex-bound splits and the over-bound rule),
    all-NaN geometry (the NaN-cost fallback to bvhPackTail), a NaN-scattered grid (segmented box scans), shared-vertex soups
    (full meshlets) and a long thin strip (deep splits)."""
    mo = meshopt()
    e = Emu()
    try:
        rng = np.random.default_rng(5)
        cases = [soup(rng, 700, 3.0), soup(rng, 97, 0.01)]
        cases.append((np.full((30, 3), 0x7E00, np.uint16), rng.integers(0, 30, 3 * 300).astype(np.uint32)))
        h, lods = special_mesh(rng)
        cases.append((h, lods[0]))
        cases.append((base.half(rng.standard_normal((150, 3))).reshape(-1, 3), rng.integers(0, 150, 3 * 500).astype(np.uint32)))
        p, x = base.grid(rng, 300, 3)
        cases.append((base.half(p).reshape(-1, 3), np.asarray(x, np.uint32)))
        for k, (pos, idx) in enumerate(cases):
            v, i, meshes = build_scene([(pos, [idx], None)])
            assert_same(e.cook_clrt(v, i, scrub(meshes)), reference_cook(mo, v, i, meshes), k)
    finally:
        e.close()


def test_emulated_clrt_capacity_bounds_and_overflow():
    """The capacity helper bounds every LOD; a call short of any one of the three capacities writes none of the arrays and sets
    the flag, with the totals still counted."""
    e = Emu()
    try:
        v, i, meshes, ml, md, mx, scale = scene("animated")
        cap, words, vtx = capacity(e.lib, meshes, scale)
        assert len(ml) <= cap and len(md) <= words and len(mx) <= vtx
        assert vtx == sum(4 * int(m["lods"][int(m["lodRT"])]["indexCount"]) for m in meshes)
        for c, w, x in ((len(ml) - 1, None, None), (None, len(md) - 1, None), (None, None, len(mx) - 1), (0, 0, 0)):
            gm, gl, gd, gx, t = e.cook_clrt(v, i, scrub(meshes), scale, cap=c, data_cap=w, vtx_cap=x)
            assert gl is None and t[3] == 1 and t[0] == len(ml) and t[1] == len(md) and t[4] == len(mx)
            assert gm.tobytes() == meshes.tobytes()  # Mesh[] is still written
        v, i, meshes, scale = clrt_scene(10)
        cap, words, vtx = capacity(e.lib, meshes, scale)
        _, gl, gd, gx, t = e.cook_clrt(v, i, meshes, scale)
        assert t[3] == 0 and t[0] <= cap and t[1] <= words and t[4] <= vtx
    finally:
        e.close()


def test_emulated_clrt_rejects_bad_input():
    """nvc_cook_meshlets' host checks, a NULL meshletvtx0 with a capacity, and an index >= vertexCount in a lodRT (0 meshlets,
    counted, no meshletvtx0)."""
    e = Emu()
    try:
        v, i, meshes = base.seeded_scene(20, ["grid", "tiny"])
        for field, value in (("lodCount", 9), ("vertexCount", len(v) + 1)):
            bad = meshes.copy()
            bad[0][field] = value
            with pytest.raises(ValueError):
                e.cook_clrt(v, i, bad, cap=0, data_cap=0, vtx_cap=0)
        for field, value in (("indexCount", 4), ("indexOffset", len(i))):
            bad = meshes.copy()
            bad["lods"][0, 0][field] = value
            with pytest.raises(ValueError):
                e.cook_clrt(v, i, bad, cap=0, data_cap=0, vtx_cap=0)
        with pytest.raises(ValueError):
            e.cook_clrt(v, i, meshes, index_count=len(i) - 3)
        with pytest.raises(ValueError):
            e.cook_clrt(v, i, meshes, vtx_null=True)
        gm, gl, gd, gx, t = e.cook_clrt(v, i, meshes, vtx_cap=0, vtx_null=True, scale=np.array([np.inf, np.nan], np.float32))
        assert t[3] == 1 and list(gm["lodRT"]) == [0, 0]  # inf and NaN scales fail the test: lodRT 0
        bad = meshes.copy()
        bad[0]["lodCount"] = 9
        with pytest.raises(AssertionError):
            capacity(e.lib, bad, None)
        good = e.cook_clrt(v, i, meshes)
        rt = int(good[0][1]["lodRT"])
        assert rt == 2
        bad_i = i.copy()
        lod = meshes["lods"][1, rt]
        bad_i[int(lod["indexOffset"]) + 4] = meshes[1]["vertexCount"]
        gm, gl, gd, gx, t = e.cook_clrt(v, bad_i, meshes)
        assert t[2] == 1 and gm["lods"][1, rt]["meshletCount"] == 0
        assert gm["lods"][0].tobytes() == good[0]["lods"][0].tobytes()
        keep = int(good[0]["lods"][1, rt]["meshletCount"])
        assert t[0] == good[4][0] - keep
        first = int(good[0]["lods"][1, rt]["meshletOffset"])
        assert t[4] == good[4][4] - 4 * int(good[1][first: first + keep]["vertexCount"].sum())
    finally:
        e.close()


def test_emulated_clrt_cache_reader():
    """animated_clrt.z.cache, written by the reference with clrtMode = 1: the reader reports it, and its decoded meshletvtx0
    equals what the clrt cooker stored (the vertex codec is lossless)."""
    c = scene_cache.SceneCache(os.path.join(GOLDEN, "animated_clrt.z.cache"))
    assert c.header.compressed and c.header.clrtMode == 1
    f = np.load(os.path.join(GOLDEN, "meshlet_cook_clrt.npz"))
    assert np.array_equal(c.section("meshletvtx0"), f["animated_meshletvtx0"])
    assert c.section("meshes").tobytes() == f["animated_meshes"].tobytes()
    assert c.section("meshlets").tobytes() == f["animated_meshlets"].tobytes()
    assert len(f["animated_meshletvtx0"]) > 0


def test_clrt_fixture_lod_rt():
    """The fixtures' lodRT is the host rule over their max_scale; kitten's is LOD 3 with 118 spatial meshlets there."""
    for name in ("kitten", "pirate", "pirateglb", "animated"):
        _, _, meshes, ml, md, mx, scale = scene(name)
        assert [lod_rt(m, s) for m, s in zip(meshes, scale)] == [int(x) for x in meshes["lodRT"]], name
        rt_vertices = sum(int(ml[int(m["lods"][int(m["lodRT"])]["meshletOffset"]):][: int(m["lods"][int(m["lodRT"])]["meshletCount"])]["vertexCount"].sum()) for m in meshes)
        assert len(mx) == 4 * rt_vertices, name
    meshes = scene("kitten")[2]
    assert int(meshes[0]["lodRT"]) == 3 and int(meshes[0]["lods"][3]["meshletCount"]) == 118


# ---- GPU tier -------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_gpu_clrt_reproduces_reference_cooker():
    """kitten.obj (lodRT 3: 118 spatial meshlets), pirate.obj, pirate.glb and animated.gltf cooked on the device: Mesh[], Meshlet[],
    meshletdata and meshletvtx0 equal the reference's clrt cooker's."""
    g = Gpu()
    try:
        for name in ("kitten", "pirate", "pirateglb", "animated"):
            v, i, meshes, ml, md, mx, scale = scene(name)
            assert_same(g.cook_clrt(v, i, scrub(meshes), scale), (meshes, ml, md, mx), name)
    finally:
        g.close()


@pytest.mark.gpu
@needs_mo
def test_gpu_clrt_against_reference_library():
    """Kitten with a max_scale that makes lodRT = 0 (28 944 triangles), and seeded scenes (NaN and inf positions included: the
    builder's choices, meshletdata and meshletvtx0 are compared in full, the bounds of non-finite meshlets are not), against the
    reference's library."""
    mo = meshopt()
    g = Gpu()
    try:
        v, i, meshes, ml, md, mx, scale = scene("kitten")
        big = np.float32(1e9)
        assert lod_rt(meshes[0], big) == 0 and int(meshes[0]["lods"][0]["indexCount"]) == 3 * 28944
        got = g.cook_clrt(v, i, scrub(meshes), np.array([big], np.float32))
        assert_same(got, reference_cook(mo, v, i, meshes, [big]), "kitten lodRT 0")
        for seed in range(3):
            v, i, meshes, scale = clrt_scene(100 + seed)
            assert_same(g.cook_clrt(v, i, scrub(meshes), scale), reference_cook(mo, v, i, meshes, scale), seed, finite_bounds_only=True)
    finally:
        g.close()


@pytest.mark.gpu
def test_gpu_clrt_many_meshes_equal_single_mesh_calls():
    """One call over many meshes gives each mesh the bytes it gets alone, moved by its meshlet, data and meshletvtx0 offsets."""
    g = Gpu()
    try:
        v, i, meshes, scale = clrt_scene(7)
        gm, gl, gd, gx, t = g.cook_clrt(v, i, meshes, scale)
        xo = 0
        for k in range(len(meshes)):
            sm, sl, sd, sx, _ = g.cook_clrt(v, i, meshes[k: k + 1].copy(), scale[k: k + 1])
            first = int(gm["lods"][k, 0]["meshletOffset"])
            n = len(sl)
            got = gl[first: first + n].copy()
            assert np.array_equal(gm["lods"][k]["meshletCount"], sm["lods"][0]["meshletCount"]) and gm[k]["lodRT"] == sm[0]["lodRT"], k
            if n:
                d0 = int(got["dataOffset"][0])
                assert np.array_equal(got["dataOffset"] - d0, sl["dataOffset"])
                got["dataOffset"] = sl["dataOffset"]
                assert got.tobytes() == sl.tobytes(), k
                assert np.array_equal(gd[d0: d0 + len(sd)], sd), k
            assert np.array_equal(gx[xo: xo + len(sx)], sx), k
            xo += len(sx)
        assert xo == len(gx)
    finally:
        g.close()


@pytest.mark.gpu
def test_gpu_frame_on_clrt_cooked_kitten():
    """A two-phase frame of the instanced kitten scene in which every draw's LOD selection picks lodRT (LOD 3: the errors of LODs 4-7
    are set to infinity and the LOD target is huge, in both runs), over the device-cooked clrt Mesh[] / Meshlet[], equals the same
    frame over the reference clrt cooker's, and its task commands point into LOD 3's spatial meshlets."""
    import torch

    from niagara_b200 import scenes
    from niagara_b200.path import VisibilityPath

    v, i, meshes, ml, md, mx, scale = scene("kitten")
    g = Gpu()
    try:
        gm, gl, gd, gx, t = g.cook_clrt(v, i, scrub(meshes), scale)
    finally:
        g.close()
    s = scenes.instanced_scene(os.path.join(GOLDEN, "kitten.nvcg"), 2048)
    lod3 = meshes[0]["lods"][3]
    outs = []
    for mesh_arr, meshlet_arr in ((meshes, ml), (gm.copy(), gl.copy())):
        mesh_arr = mesh_arr.copy()
        mesh_arr["lods"][0, 4:]["error"] = np.inf
        p = VisibilityPath(mesh_arr, meshlet_arr, s.draws, *s.screen, device="cuda:0")
        p.set_visibility_bits(s.visibility_bits)
        depth = torch.from_numpy(s.depth).cuda()
        cd = s.cull_data()
        cd.lodTarget = 1e30
        for _ in range(2):
            p.frame(cd, depth, cluster_backface=True)
        torch.cuda.synchronize()
        d, c = p.read_counts()
        cmds = p.read_task_commands(int(d[1]) * 64)
        outs.append((d, c, p.dvb.cpu().numpy(), p.mvb.cpu().numpy(), p.depthPyramid.cpu().numpy()))
    for a, b in zip(*outs):
        assert np.array_equal(a, b)
    first, count = int(lod3["meshletOffset"]), int(lod3["meshletCount"])
    offsets = cmds["taskOffset"][cmds["taskCount"] > 0]
    assert len(offsets) and ((offsets >= first) & (offsets < first + count)).all(), "task commands outside LOD 3"
