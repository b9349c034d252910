"""N4 — appendMesh's vertex processing on the device (csrc/nvc_vertices.cuh / nvc_cook_mesh_vertices).
The checkers are the REFERENCE's stored outputs and its own library.  Given what loadObj / loadVertices leave (obj_vertices.npz
for kitten.obj and pirate.obj, nvc_gltf_primitive_data for the glTF files), the Vertex[] and LOD 0 must be those the reference's
cooker stored (scene_cache_write_raw.npz, meshlet_cook.npz / pirate_vertices.npz, animated.raw.cache, the importer fixtures);
end to end, nvc_cook_mesh_vertices -> nvc_cook_mesh_lods -> nvc_cook_meshlets(_clrt) -> nvc_scene_cache_write must give the
reference's .z.cache byte for byte.  For seeded meshes the checker is the reference's meshoptimizer (oracle/_ref/
libmeshopt_full_ref.so) driven by `ref_vertices`, a restatement of scene.cpp:172-184 that the fixtures check in turn.  The CPU
tier runs the product's kernels under the SIMT emulation (tests/emu_lib.py) through the C ABI; the -m gpu tier runs them on
the device."""
import ctypes
import glob
import mmap
import os

import numpy as np
import pytest

import emu_lib
import test_cook_lods as lods_tests
from niagara_b200 import gltf, layout

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
FULL_PATH = os.path.join(ROOT, "oracle", "_ref", "libmeshopt_full_ref.so")
needs_ref = pytest.mark.skipif(not os.path.exists(FULL_PATH), reason="needs the reference's meshoptimizer (oracle/_ref/libmeshopt_full_ref.so)")
INVALID = -1
# the glTF files whose reference run stored its cooked Vertex[]: (file, expected npz)
GLTF_VERTICES = [("hierarchy.glb", "hierarchy_expected.npz")] + [
    (os.path.join("meshopt", os.path.basename(p)[: -len("_expected.npz")] + ".glb"), os.path.join("meshopt", os.path.basename(p)))
    for p in sorted(glob.glob(os.path.join(GOLDEN, "meshopt", "*_expected.npz")))
    if len(np.load(p)["vertices"])
]


# ---- inputs ------------------------------------------------------------------------------------------------------------

def obj_input(name):
    """loadObj's Vertex[] of kitten.obj / pirate.obj as (n, 8) uint16, one record per corner; the indices are 0..n-1"""
    with np.load(os.path.join(GOLDEN, "obj_vertices.npz")) as z:
        v = z[name + "_records"][z[name + "_corners"]]
    return np.ascontiguousarray(v), np.arange(len(v), dtype=np.uint32)


def gltf_input(path):
    """loadVertices' output of every primitive, concatenated, and the meshes over it"""
    g = gltf.GltfScene(os.path.join(GOLDEN, path))
    parts = []
    for m in range(g.info.primitive_count):
        v, ix = g.primitive(m)
        parts.append((np.ascontiguousarray(v).view(np.uint16).reshape(-1, 8), ix.astype(np.uint32)))
    g.close()
    return lods_tests.scene_of(parts)


def cooked(name):
    """(Vertex[], LOD 0 of every mesh, concatenated, Mesh[]) as the reference's cooker stored them for a fixture of test_cook_lods"""
    v, ib, meshes, _ = lods_tests.fixture(name)
    lod0 = [ib[int(m["lods"][0]["indexOffset"]): int(m["lods"][0]["indexOffset"]) + int(m["lods"][0]["indexCount"])] for m in meshes]
    return v, np.concatenate(lod0).astype(np.uint32), meshes


# ---- the reference: scene.cpp:172-184 over the reference's meshoptimizer ---------------------------------------------------

_REF = None


def ref_lib():
    global _REF
    if _REF is None:
        lib = ctypes.CDLL(FULL_PATH)
        c_p, c_sz = ctypes.c_void_p, ctypes.c_size_t
        for name, restype, argtypes in (("meshopt_filterIndexBuffer", c_sz, [c_p, c_p, c_sz, c_p, c_sz, c_sz, c_sz]),
                                        ("meshopt_generateVertexRemap", c_sz, [c_p, c_p, c_sz, c_p, c_sz, c_sz]),
                                        ("meshopt_remapVertexBuffer", None, [c_p, c_p, c_sz, c_sz, c_p]),
                                        ("meshopt_remapIndexBuffer", None, [c_p, c_p, c_sz, c_p]),
                                        ("meshopt_optimizeVertexCache", None, [c_p, c_p, c_sz, c_sz]),
                                        ("meshopt_optimizeVertexFetch", c_sz, [c_p, c_p, c_sz, c_p, c_sz, c_sz])):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
        _REF = lib
    return _REF


def ref_vertices(vertices, indices):
    """(Vertex[] (n, 8) uint16, LOD 0) of scene.cpp:172-184 for one mesh, from loadObj / loadVertices' output"""
    lib = ref_lib()
    v = np.ascontiguousarray(vertices, np.uint16).reshape(-1, 8).copy()
    ix = np.ascontiguousarray(indices, np.uint32).copy()
    if len(ix) == 0:
        return np.zeros((0, 8), np.uint16), ix
    n = lib.meshopt_filterIndexBuffer(ix.ctypes.data, ix.ctypes.data, len(ix), v.ctypes.data, len(v), 6, 16)
    ix = ix[:n].copy()
    remap = np.zeros(len(v), np.uint32)
    unique = lib.meshopt_generateVertexRemap(remap.ctypes.data, ix.ctypes.data, n, v.ctypes.data, len(v), 16)
    lib.meshopt_remapVertexBuffer(v.ctypes.data, v.ctypes.data, len(v), 16, remap.ctypes.data)
    lib.meshopt_remapIndexBuffer(ix.ctypes.data, ix.ctypes.data, n, remap.ctypes.data)
    v = v[:unique].copy()
    lib.meshopt_optimizeVertexCache(ix.ctypes.data, ix.ctypes.data, n, unique)
    lib.meshopt_optimizeVertexFetch(v.ctypes.data, ix.ctypes.data, n, v.ctypes.data, unique, 16)
    return v, ix


def ref_scene(vertices, indices, host_meshes):
    """Mesh[], Vertex[] and LOD 0 buffer the call must give: ref_vertices per mesh, in mesh order"""
    out = np.zeros(len(host_meshes), layout.MESH_DTYPE)
    vs, ixs = [np.zeros((0, 8), np.uint16)], [np.zeros(0, np.uint32)]
    vb = ib = 0
    for k, hm in enumerate(host_meshes):
        vo, vc = int(hm["vertexOffset"]), int(hm["vertexCount"])
        io, ic = int(hm["lods"][0]["indexOffset"]), int(hm["lods"][0]["indexCount"])
        v, ix = ref_vertices(vertices[vo: vo + vc], indices[io: io + ic])
        out[k]["vertexOffset"], out[k]["vertexCount"], out[k]["lodCount"] = vb, len(v), 1
        out[k]["lods"][0]["indexOffset"], out[k]["lods"][0]["indexCount"] = ib, len(ix)
        vs.append(v)
        ixs.append(ix)
        vb += len(v)
        ib += len(ix)
    return out, np.concatenate(vs), np.concatenate(ixs).astype(np.uint32)


# ---- the product, emulated (host pointers) or on the device ---------------------------------------------------------------

class Emu:
    def __init__(self):
        self.lib = emu_lib.load()
        self.ctx = ctypes.c_void_p()
        assert self.lib.nvc_create(0, None, ctypes.byref(self.ctx)) == 0

    def close(self):
        self.lib.nvc_destroy(self.ctx)

    def cook(self, vertices, indices, meshes, vertex_capacity=None, index_capacity=None, vertex_count=None, index_count=None):
        """(Mesh[], Vertex[], LOD 0, totals4); status != 0 raises ValueError(status) after checking the outputs are untouched"""
        vertices = np.ascontiguousarray(vertices, np.uint16).reshape(-1, 8)
        indices = np.ascontiguousarray(indices, np.uint32)
        vcap = len(vertices) if vertex_capacity is None else vertex_capacity
        icap = len(indices) if index_capacity is None else index_capacity
        out_meshes = np.full(len(meshes) * 208, 0xCD, np.uint8)
        out_v = np.full((vcap + 1, 8), 0xA5A5, np.uint16)
        out_i = np.full(icap + 1, 0xA5A5A5A5, np.uint32)
        totals = np.full(4, 0x77, np.uint32)
        status = self.lib.nvc_cook_mesh_vertices(self.ctx, None, vertices.ctypes.data if len(vertices) else None, len(vertices) if vertex_count is None else vertex_count,
                                                 indices.ctypes.data if len(indices) else None, len(indices) if index_count is None else index_count, meshes.ctypes.data,
                                                 len(meshes), out_meshes.ctypes.data, out_v.ctypes.data, vcap, out_i.ctypes.data, icap, totals.ctypes.data)
        if status != 0:
            assert (out_meshes == 0xCD).all() and (out_v == 0xA5A5).all() and (out_i == 0xA5A5A5A5).all() and (totals == 0x77).all(), "a refused call wrote its outputs"
            raise ValueError(status)
        assert (out_v[int(totals[0]):] == 0xA5A5).all() and (out_i[int(totals[1]):] == 0xA5A5A5A5).all(), "write past the totals"
        return out_meshes.view(layout.MESH_DTYPE), out_v[: int(totals[0])], out_i[: int(totals[1])], totals


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

    def cook(self, vertices, indices, meshes, stream=None):
        torch = self.torch
        vertices = np.ascontiguousarray(vertices, np.uint16).reshape(-1, 8)
        indices = np.ascontiguousarray(indices, np.uint32)
        dv = torch.from_numpy(vertices.view(np.uint8).reshape(-1).copy()).cuda()
        di = torch.from_numpy(indices.view(np.int32).copy()).cuda()
        dm = torch.zeros(len(meshes) * 208, dtype=torch.uint8, device="cuda")
        dov = torch.zeros(max(len(vertices), 1) * 16, dtype=torch.uint8, device="cuda")
        doi = torch.zeros(max(len(indices), 1), dtype=torch.int32, device="cuda")
        dt = torch.zeros(4, dtype=torch.int32, device="cuda")
        s = stream.cuda_stream if stream is not None else None
        self.check(self.lib.nvc_cook_mesh_vertices(self.ctx, s, dv.data_ptr(), len(vertices), di.data_ptr(), len(indices), meshes.ctypes.data, len(meshes),
                                                   dm.data_ptr(), dov.data_ptr(), len(vertices), doi.data_ptr(), len(indices), dt.data_ptr()),
                   self.ctx, "nvc_cook_mesh_vertices")
        torch.cuda.synchronize()
        totals = dt.cpu().numpy().view(np.uint32)
        out_v = dov.cpu().numpy().view(np.uint16).reshape(-1, 8)[: int(totals[0])]
        return dm.cpu().numpy().view(layout.MESH_DTYPE), out_v, doi.cpu().numpy().view(np.uint32)[: int(totals[1])], totals


def assert_same(got, want, what):
    gm, gv, gi, gt = got
    wm, wv, wi = want
    assert gt[0] == len(wv) and gt[1] == len(wi) and gt[2] == 0 and gt[3] == 0, (what, gt, len(wv), len(wi))
    if gm.tobytes() != wm.tobytes():
        for k in range(len(wm)):
            assert gm[k].tobytes() == wm[k].tobytes(), (what, "mesh", k, gm[k], wm[k])
    bad = np.nonzero((gv != wv).any(axis=1))[0]
    assert len(bad) == 0, (what, "vertices", len(bad), bad[:8])
    bad = np.nonzero(gi != wi)[0]
    assert len(bad) == 0, (what, "indices", len(bad), bad[:8])


def expected_meshes(vertex_counts, index_counts):
    m = np.zeros(len(vertex_counts), layout.MESH_DTYPE)
    m["vertexCount"], m["lodCount"] = vertex_counts, 1
    m["vertexOffset"] = np.concatenate([[0], np.cumsum(vertex_counts)[:-1]])
    m["lods"][:, 0]["indexCount"] = index_counts
    m["lods"][:, 0]["indexOffset"] = np.concatenate([[0], np.cumsum(index_counts)[:-1]])
    return m


@pytest.fixture(scope="module")
def emu():
    e = Emu()
    yield e
    e.close()


# ---- reference outputs -------------------------------------------------------------------------------------------------------

def obj_case(name):
    v, ix = obj_input(name)
    wv, wi, stored = cooked(name)
    return (v, ix, lods_tests.scene_of([(v, ix)])[2]), (expected_meshes([len(wv)], [len(wi)]), wv, wi)


def animated_case():
    v, ix, m = gltf_input("animated.gltf")
    wv, wi, stored = cooked("animated")
    return (v, ix, m), (expected_meshes(stored["vertexCount"], stored["lods"][:, 0]["indexCount"]), wv, wi)


def test_obj_fixture_counts():
    (v, ix, m), (wm, wv, wi) = obj_case("kitten")
    assert len(wi) == 86832 and len(wv) == 14856 and len(v) == 86832


@pytest.mark.parametrize("name", ["kitten", "pirate"])
def test_obj_fixture_emulated(emu, name):
    """loadObj's Vertex[] -> the Vertex[] and LOD 0 the reference's cooker stored, bit for bit"""
    (v, ix, m), want = obj_case(name)
    assert_same(emu.cook(v, ix, m), want, name)


def test_animated_gltf_emulated(emu):
    """nvc_gltf_primitive_data's output of animated.gltf -> every mesh's Vertex[] and LOD 0 of animated.raw.cache"""
    (v, ix, m), want = animated_case()
    assert_same(emu.cook(v, ix, m), want, "animated.gltf")


@pytest.mark.parametrize("path,expected", GLTF_VERTICES)
def test_gltf_vertices_emulated(emu, path, expected):
    """the importer fixtures that hold the reference's cooked Vertex[]: equal, in order (no longer only as a set)"""
    v, ix, m = gltf_input(path)
    gm, gv, gi, gt = emu.cook(v, ix, m)
    ref = np.load(os.path.join(GOLDEN, expected))
    want = np.ascontiguousarray(ref["vertices"]).view(np.uint8).reshape(-1, 16)
    assert gt[2] == 0 and np.array_equal(gv.view(np.uint8).reshape(-1, 16), want), path
    assert np.array_equal(gm["vertexOffset"], ref["mesh_vertex_offset"]) and np.array_equal(gm["vertexCount"], ref["mesh_vertex_count"]), path


@needs_ref
@pytest.mark.parametrize("name", ["kitten", "pirate", "animated"])
def test_restatement_matches_fixtures(name):
    """ref_vertices, scene.cpp:172-184 restated over the reference's library, reproduces what the reference's cooker stored"""
    (v, ix, m), want = obj_case(name) if name != "animated" else animated_case()
    got = ref_scene(v, ix, m)
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2]), name


# ---- end to end ----------------------------------------------------------------------------------------------------------------

END_TO_END = [("kitten.z.cache", "kitten", False), ("animated.z.cache", "animated.raw.cache", False), ("animated_clrt.z.cache", "animated_clrt", True)]


def importer_output(raw):
    if raw == "kitten":
        v, ix = obj_input("kitten")
        return v, ix, lods_tests.scene_of([(v, ix)])[2]
    return gltf_input("animated.gltf")


def end_to_end_emulated(emu, raw, clrt):
    """nvc_cook_mesh_vertices -> nvc_cook_mesh_lods -> nvc_cook_meshlets(_clrt) -> nvc_scene_cache_write, all emulated on one
    context, from the importer's output; the non-geometry sections from the reference run's raw cache"""
    import test_scene_cache_write as write_tests

    lib, ctx = emu.lib, emu.ctx
    header, secs = lods_tests.raw_geometry(raw)
    header.clrtMode = int(clrt)
    v, ix, m = importer_output(raw)
    vm, vv, vi, vt = emu.cook(v, ix, m)
    assert vt[2] == 0
    scale = lods_tests.max_scale_of("animated_clrt" if clrt else raw, len(vm))
    cap = lods_tests.capacity(lib, vm)
    meshes = np.zeros(len(vm), layout.MESH_DTYPE)
    ib = np.zeros(cap + 1, np.uint32)
    totals = np.zeros(4, np.uint32)
    assert lib.nvc_cook_mesh_lods(ctx, None, vv.ctypes.data, len(vv), vi.ctypes.data, len(vi), vm.ctypes.data, scale.ctypes.data, len(vm),
                                  meshes.ctypes.data, ib.ctypes.data, cap, totals.ctypes.data) == 0
    assert totals[1] == 0 and totals[2] == 0
    ib = ib[: int(totals[0])]
    nm, nw, nv = ctypes.c_uint32(), ctypes.c_uint64(), ctypes.c_uint64()
    if clrt:
        assert lib.nvc_cook_meshlets_clrt_capacity(meshes.ctypes.data, scale.ctypes.data, len(meshes), ctypes.byref(nm), ctypes.byref(nw), ctypes.byref(nv)) == 0
    else:
        assert lib.nvc_cook_meshlets_capacity(meshes.ctypes.data, len(meshes), ctypes.byref(nm), ctypes.byref(nw)) == 0
    out_meshes = np.zeros(len(meshes), layout.MESH_DTYPE)
    ml = np.zeros(max(nm.value, 1) * 24, np.uint8)
    md = np.zeros(max(nw.value, 1), np.uint32)
    vtx0 = np.zeros(max(nv.value, 1), np.uint16)
    t = np.zeros(8, np.uint32)
    if clrt:
        st = lib.nvc_cook_meshlets_clrt(ctx, None, vv.ctypes.data, len(vv), ib.ctypes.data, len(ib), meshes.ctypes.data, scale.ctypes.data, out_meshes.ctypes.data, len(meshes),
                                        ml.ctypes.data, nm.value, md.ctypes.data, nw.value, vtx0.ctypes.data, nv.value, t.ctypes.data)
    else:
        st = lib.nvc_cook_meshlets(ctx, None, vv.ctypes.data, len(vv), ib.ctypes.data, len(ib), meshes.ctypes.data, out_meshes.ctypes.data, len(meshes),
                                   ml.ctypes.data, nm.value, md.ctypes.data, nw.value, t.ctypes.data)
    assert st == 0 and t[3] == 0
    s2 = dict(secs)
    s2.update(vertices=vv.view(np.uint8).reshape(-1), indices=ib, meshes=out_meshes.view(np.uint8), meshlets=ml[: int(t[0]) * 24], meshletdata=md[: int(t[1])])
    if clrt:
        s2["meshletvtx0"] = vtx0[: int(t[4])]
    status, got = write_tests.write(lib, ctx, write_tests.make_desc(header, s2, True))
    assert status == 0
    return got


@pytest.mark.parametrize("ref_file,raw,clrt", END_TO_END)
def test_end_to_end_emulated(emu, ref_file, raw, clrt):
    """importer output -> vertices -> LOD chains -> meshlets -> compressed cache: the reference's file, byte for byte"""
    want = np.fromfile(os.path.join(GOLDEN, ref_file), np.uint8)
    got = end_to_end_emulated(emu, raw, clrt)
    assert len(got) == len(want) and np.array_equal(got, want), ref_file


# ---- seeded meshes against the library -----------------------------------------------------------------------------------------

def soup(rng, tris):
    """an OBJ-style unindexed soup: the corners of `tris` triangles of a shared grid, one record each"""
    p, n, i = lods_tests.grid_mesh(rng, 8, 8)
    v = lods_tests.make_vertices(p, n)
    i = i[: 3 * tris]
    return v[i], np.arange(len(i), dtype=np.uint32)


def seeded_cases():
    rng = np.random.default_rng(17)
    out = {}
    out["soup"] = soup(rng, 128)
    p, n, i = lods_tests.grid_mesh(rng, 10, 9, seam=True)
    out["grid"] = (lods_tests.make_vertices(p, n), i)
    # a triangle, its duplicates in all three rotations, the reversed one (kept), a copy over other vertex records
    p, n, i = lods_tests.grid_mesh(rng, 4, 4)
    v = lods_tests.make_vertices(p, n)
    a, b, c = (int(x) for x in i[6:9])
    extra = v[[a, b, c]].copy()
    extra[:, 6] = 0x3C00  # other UVs, same positions
    k = len(v)
    out["duplicates"] = (np.concatenate([v, extra]), np.concatenate([i, [a, b, c, b, c, a, c, a, b, a, c, b, k, k + 1, k + 2, k + 1, k + 2, k]]).astype(np.uint32))
    # degenerate by position only: corners with the same position but other normals / UVs
    v2 = v.copy()
    twins = v2[[0, 1]].copy()
    twins[0, 4] ^= 0x155
    twins[1, 7] = 0x1234
    v2 = np.concatenate([v2, twins])
    k = len(v)
    out["degenerate"] = (v2, np.concatenate([[0, k, 5, 1, 6, k + 1, 0, 1, 2], i]).astype(np.uint32))
    # vertices that differ only in tp, np, tu or tv stay apart
    v3 = v.copy()
    variants = []
    for field in (3, 4, 6, 7):
        w = v3[[a, b, c]].copy()
        w[:, field] ^= 0x0101
        variants.append(w)
    v3 = np.concatenate([v3] + variants)
    ix = list(i)
    for f in range(4):  # each variant in triangles of their own, so that the filter keeps them
        base = len(v) + 3 * f
        ix += [base, 24 - f, 19 - f, base + 1, 19 - f, 24 - f]
    out["attributes"] = (v3, np.array(ix, np.uint32))
    # +-0, denormal, inf, NaN payloads
    sv, si = lods_tests.special_positions()
    sv = sv.copy()
    sv[8, :3] = sv[0, :3] ^ np.array([0x8000, 0, 0], np.uint16)  # vertex 0's position with +0 for its -0
    sv[10, :3] = [0x7E01, 0x7E02, 0]
    sv[11, :3] = [0x7E01, 0x7E03, 0]  # NaN payloads that differ
    out["special"] = (sv, si)
    # unreferenced vertices before, between and after
    p, n, i = lods_tests.grid_mesh(rng, 5, 5)
    v = lods_tests.make_vertices(p, n)
    junk = lods_tests.make_vertices(rng.normal(size=(7, 3)).astype(np.float32), np.tile([[0, 0, 1]], (7, 1)).astype(np.float32))
    out["unreferenced"] = (np.concatenate([junk[:3], v[:10], junk[3:5], v[10:], junk[5:]]), np.where(i < 10, i + 3, i + 5).astype(np.uint32))
    # everything filtered: degenerate triangles only
    out["all_filtered"] = (v[:4], np.array([0, 0, 1, 2, 3, 3, 1, 1, 1], np.uint32))
    out["empty"] = (v[:3], np.zeros(0, np.uint32))
    out["single"] = (v[:3], np.array([0, 1, 2], np.uint32))
    # more than one scan block (2048 flags) of triangles and of index positions
    p, n, i = lods_tests.sphere_mesh(rng, 30)
    out["multiblock"] = (lods_tests.make_vertices(p, n), i)
    return out


SEEDED = ["soup", "grid", "duplicates", "degenerate", "attributes", "special", "unreferenced", "all_filtered", "empty", "single", "multiblock"]


@needs_ref
@pytest.mark.parametrize("name", SEEDED)
def test_seeded_emulated(emu, name):
    v, i = seeded_cases()[name]
    v_all, i_all, m = lods_tests.scene_of([(v, i)])
    want = ref_scene(v_all, i_all, m)
    got = emu.cook(v_all, i_all, m)
    assert_same(got, want, name)
    again = emu.cook(v_all, i_all, m)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(got, again)), name
    if name == "all_filtered":
        assert int(got[0]["vertexCount"][0]) == 0 and int(got[0]["lods"][0, 0]["indexCount"]) == 0
    if name == "multiblock":
        assert len(i) // 3 > 2048


@needs_ref
def test_seeded_cases_reach_their_paths():
    """the seeded cases hold what they are named for, as the reference's library sees them"""
    cases = seeded_cases()
    v, i = cases["duplicates"]
    _, wi = ref_vertices(v, i)
    assert len(wi) == len(i) - 3 * 5  # the three rotations and the two over other records dropped, the reversed one kept
    v, i = cases["degenerate"]
    _, wi = ref_vertices(v, i)
    assert len(wi) == len(i) - 6
    v, i = cases["attributes"]
    wv, wi = ref_vertices(v, i)
    assert len(wi) == len(i) and len(wv) == len(np.unique(v[np.unique(i)].view(np.uint8).reshape(-1, 16), axis=0)) == len(np.unique(i))


@needs_ref
def test_many_meshes_equal_one_call_each(emu):
    cases = seeded_cases()
    parts = [cases[k] for k in SEEDED]
    v, i, m = lods_tests.scene_of(parts)
    gm, gv, gi, gt = emu.cook(v, i, m)
    vb = ib = 0
    for k, part in enumerate(parts):
        pv, pi, pm = lods_tests.scene_of([part])
        om, ov, oi, ot = emu.cook(pv, pi, pm)
        want = om.copy()
        want["vertexOffset"] += vb
        want["lods"]["indexOffset"][0, 0] += ib
        assert gm[k].tobytes() == want[0].tobytes(), k
        assert np.array_equal(gv[vb: vb + len(ov)], ov) and np.array_equal(gi[ib: ib + len(oi)], oi), k
        vb += len(ov)
        ib += len(oi)
    assert vb == gt[0] and ib == gt[1]


# ---- refusals and rejection ------------------------------------------------------------------------------------------------------

def test_argument_refusals(emu):
    rng = np.random.default_rng(9)
    p, n, i = lods_tests.grid_mesh(rng, 3, 3)
    v, idx, m = lods_tests.scene_of([(lods_tests.make_vertices(p, n), i)])
    for mutate in (lambda x: x["lods"][0, 0].__setitem__("indexCount", 5),
                   lambda x: x["lods"][0, 0].__setitem__("indexOffset", 3),
                   lambda x: x.__setitem__("vertexOffset", 1)):
        bad = m.copy()
        mutate(bad)
        with pytest.raises(ValueError, match=str(INVALID)):
            emu.cook(v, idx, bad)
    with pytest.raises(ValueError, match=str(INVALID)):
        emu.cook(v, idx, m, vertex_capacity=len(v) - 1)
    with pytest.raises(ValueError, match=str(INVALID)):
        emu.cook(v, idx, m, index_capacity=len(idx) - 1)
    # two meshes over the same ranges: the capacities cover both
    both = np.concatenate([m, m])
    with pytest.raises(ValueError, match=str(INVALID)):
        emu.cook(v, idx, both)
    gm, gv, gi, gt = emu.cook(v, idx, both, vertex_capacity=2 * len(v), index_capacity=2 * len(idx))
    assert np.array_equal(gv[: len(gv) // 2], gv[len(gv) // 2:]) and np.array_equal(gi[: len(gi) // 2], gi[len(gi) // 2:])


def test_rejected_mesh(emu):
    rng = np.random.default_rng(5)
    p, n, i = lods_tests.grid_mesh(rng, 4, 4)
    good = lods_tests.make_vertices(p, n)
    bad_i = i.copy()
    bad_i[7] = len(p)  # one past the mesh's vertices
    v, idx, m = lods_tests.scene_of([(good, i), (good, bad_i), (good, i)])
    gm, gv, gi, gt = emu.cook(v, idx, m)
    assert gt[2] == 1
    assert int(gm[1]["vertexCount"]) == 0 and int(gm[1]["lods"][0]["indexCount"]) == 0 and int(gm[1]["lodCount"]) == 1
    assert gm[1]["vertexOffset"] == gm[2]["vertexOffset"] == gm[0]["vertexCount"]
    assert gm[1]["lods"][0]["indexOffset"] == gm[2]["lods"][0]["indexOffset"] == gm[0]["lods"][0]["indexCount"] == gm[2]["lods"][0]["indexCount"]
    assert np.array_equal(gv[: int(gm[0]["vertexCount"])], gv[int(gm[2]["vertexOffset"]):])
    assert np.array_equal(gi[: int(gm[0]["lods"][0]["indexCount"])], gi[int(gm[2]["lods"][0]["indexOffset"]):])


def test_rejected_mesh_reads_no_vertex():
    """a rejected mesh's vertices lie past the end of an array that ends at an inaccessible page, and the call's device
    allocations end at one too: reading any of them, or past any scratch array, faults"""
    import test_scene_cache_device as dev_tests

    lib = emu_lib.load()
    rng = np.random.default_rng(13)
    p, n, i = lods_tests.grid_mesh(rng, 4, 4)
    good = lods_tests.make_vertices(p, n)
    bad_count = 200  # 3 200 bytes: inside the inaccessible page after `good`
    bad_i = (i % bad_count).astype(np.uint32)
    bad_i[4] = bad_count  # rejects the mesh
    vertices = dev_tests._guarded_zeros(good.nbytes).view(np.uint16).reshape(-1, 8)
    assert (vertices.ctypes.data + good.nbytes) % mmap.PAGESIZE == 0
    vertices[:] = good
    idx = np.concatenate([i, bad_i]).astype(np.uint32)
    m = np.zeros(2, layout.MESH_DTYPE)
    m["vertexOffset"] = [0, len(good)]
    m["vertexCount"] = [len(good), bad_count]
    m["lods"][:, 0]["indexOffset"] = [0, len(i)]
    m["lods"][:, 0]["indexCount"] = [len(i), len(bad_i)]
    vcap, icap = len(good) + bad_count, len(idx)
    meshes = np.zeros(2, layout.MESH_DTYPE)
    out_v = np.zeros((vcap, 8), np.uint16)
    out_i = np.zeros(icap, np.uint32)
    totals = np.zeros(4, np.uint32)
    ctx = ctypes.c_void_p()
    assert lib.nvc_create(0, None, ctypes.byref(ctx)) == 0
    lib.emu_guard_allocations(1)
    try:
        status = lib.nvc_cook_mesh_vertices(ctx, None, vertices.ctypes.data, vcap, idx.ctypes.data, len(idx), m.ctypes.data, 2, meshes.ctypes.data,
                                            out_v.ctypes.data, vcap, out_i.ctypes.data, icap, totals.ctypes.data)
    finally:
        lib.emu_guard_allocations(0)
        lib.nvc_destroy(ctx)
        assert lib.emu_guarded_live() == 0
    assert status == 0 and totals[2] == 1
    assert int(meshes[1]["vertexCount"]) == 0 and int(meshes[1]["lods"][0]["indexCount"]) == 0
    if os.path.exists(FULL_PATH):
        wv, wi = ref_vertices(good, i)
        assert np.array_equal(out_v[: int(totals[0])], wv) and np.array_equal(out_i[: int(totals[1])], wi)


# ---- GPU tier --------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def gpu():
    g = Gpu()
    yield g
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kitten", "pirate", "animated"])
def test_fixture_gpu(gpu, name):
    (v, ix, m), want = obj_case(name) if name != "animated" else animated_case()
    assert_same(gpu.cook(v, ix, m), want, name)


@pytest.mark.gpu
@pytest.mark.parametrize("ref_file,raw,clrt", END_TO_END)
def test_end_to_end_gpu(gpu, ref_file, raw, clrt):
    """the same chain on the device, the cache written from device memory: the reference's file"""
    import torch

    import test_scene_cache_write as write_tests

    want = np.fromfile(os.path.join(GOLDEN, ref_file), np.uint8)
    header, secs = lods_tests.raw_geometry(raw)
    header.clrtMode = int(clrt)
    v, ix, m = importer_output(raw)
    vm, vv, vi, vt = gpu.cook(v, ix, m)
    assert vt[2] == 0
    scale = lods_tests.max_scale_of("animated_clrt" if clrt else raw, len(vm))
    meshes, ib, totals = lods_tests.Gpu.cook(gpu, vv, vi, vm, scale)
    assert totals[1] == 0 and totals[2] == 0
    s2 = dict(secs)
    s2.update(vertices=vv.view(np.uint8).reshape(-1), indices=ib.view(np.uint8), meshes=meshes.view(np.uint8))
    s2.update(write_tests._cook(gpu.lib, gpu.ctx, s2, clrt, scale if clrt else None))
    torch.cuda.synchronize()
    got = write_tests._write_py(header, s2, True)
    assert len(got) == len(want) and np.array_equal(got, want), ref_file


def jittered_kitten(copies, seed=1):
    """`copies` copies of kitten's loadObj output, positions jittered (so that filtering and de-duplication still bite)"""
    rng = np.random.default_rng(seed)
    with np.load(os.path.join(GOLDEN, "obj_vertices.npz")) as z:
        records, corners = z["kitten_records"], z["kitten_corners"]
    parts = []
    for _ in range(copies):
        r = records.copy()
        pos = r[:, :3].view(np.float16).astype(np.float32)
        pos = pos * rng.uniform(0.5, 2.0) + rng.uniform(-100, 100, (1, 3)).astype(np.float32) + rng.normal(0, 1e-3, pos.shape).astype(np.float32)
        r[:, :3] = pos.astype(np.float16).view(np.uint16)
        v = r[corners]
        parts.append((v, np.arange(len(v), dtype=np.uint32)))
    return lods_tests.scene_of(parts)


@pytest.mark.gpu
@needs_ref
def test_jittered_kitten_copies_gpu(gpu):
    v, i, m = jittered_kitten(1000)
    assert_same(gpu.cook(v, i, m), ref_scene(v, i, m), "1000 jittered kitten copies")


@pytest.mark.gpu
def test_busy_nonblocking_stream_gpu(gpu):
    import torch

    (v, ix, m), want = animated_case()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a = torch.randn(4096, 4096, device="cuda")
        for _ in range(8):
            a = a @ a.T / 4096
    got = gpu.cook(v, ix, m, stream=s)
    torch.cuda.synchronize()
    assert_same(got, want, "non-blocking stream")
