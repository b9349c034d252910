"""N4 — the LOD chain on the device (csrc/nvc_lods.cuh / nvc_cook_mesh_lods).
The checker is the REFERENCE itself: given only the Vertex[] and LOD 0 of kitten.obj, pirate.obj, pirate.glb and animated.gltf
(and animated.gltf cooked with clrt on), the Mesh[] and index buffer must be those its cooker stored.  The inputs come from the
uncompressed caches of the reference's runs (scene_cache_write_raw.npz, animated.raw.cache) and meshlet_cook.npz /
pirate_vertices.npz: the index codec of a compressed cache rotates triangles, so only these hold the index order the cooker
saw.  End to end, nvc_cook_mesh_lods -> nvc_cook_meshlets(_clrt) -> nvc_scene_cache_write must give the reference's .z.cache
byte for byte.  For seeded meshes the checker is the reference's meshoptimizer (oracle/_ref/libmeshopt_simplify_ref.so)
driven by `ref_chain`, a restatement of appendMesh's LOD loop (scene.cpp:193-268) that the fixtures check in turn.  The CPU
tier runs the product's kernels under the SIMT emulation (tests/emu_lib.py) through the C ABI; the -m gpu tier runs them on
the device."""
import ctypes
import mmap
import os

import numpy as np
import pytest

import emu_lib
from niagara_b200 import layout

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
SIMPLIFY_PATH = os.path.join(ROOT, "oracle", "_ref", "libmeshopt_simplify_ref.so")
needs_ref = pytest.mark.skipif(not os.path.exists(SIMPLIFY_PATH), reason="needs the reference's meshoptimizer (oracle/_ref/libmeshopt_simplify_ref.so)")
FIXTURES = ["kitten", "pirate", "pirateglb", "animated", "animated_clrt"]
# the end-to-end files: (compressed reference file, raw geometry of the same run, clrt)
END_TO_END = [("kitten.z.cache", "kitten", False), ("animated.z.cache", "animated.raw.cache", False), ("animated_clrt.z.cache", "animated_clrt", True)]


# ---- inputs ------------------------------------------------------------------------------------------------------------

def raw_geometry(raw):
    """(header, {section: bytes}) of a reference run's uncompressed cache: a file under golden/ or a key of scene_cache_write_raw.npz"""
    import test_scene_cache_write as write_tests

    return write_tests.raw_sections(write_tests.raw_file(raw))


def max_scale_of(name, count):
    if name == "animated_clrt":
        with np.load(os.path.join(GOLDEN, "meshlet_cook_clrt.npz")) as z:
            return z["animated_max_scale"].astype(np.float32)
    return np.ones(count, np.float32)


def fixture(name):
    """(Vertex[] as (n, 8) uint16, ib, Mesh[] with the meshlet fields zeroed, max_scale) as the reference's cooker left them"""
    if name == "pirate":
        with np.load(os.path.join(GOLDEN, "meshlet_cook.npz")) as z:
            ib, meshes = z["pirate_indices"].astype(np.uint32), z["pirate_meshes"].reshape(-1).view(layout.MESH_DTYPE).copy()
        with np.load(os.path.join(GOLDEN, "pirate_vertices.npz")) as z:
            v = z["pirate_vertices"].copy()
    else:
        _, secs = raw_geometry("animated.raw.cache" if name == "animated" else name)
        v, ib, meshes = secs["vertices"].view(np.uint16).reshape(-1, 8).copy(), secs["indices"].view(np.uint32).copy(), secs["meshes"].view(layout.MESH_DTYPE).copy()
    meshes["lods"]["meshletOffset"] = 0
    meshes["lods"]["meshletCount"] = 0
    return v, ib, meshes, max_scale_of(name, len(meshes))


def lod0_input(meshes):
    """the call's host_meshes: only vertexOffset, vertexCount and lods[0]'s range survive"""
    m = np.zeros(len(meshes), layout.MESH_DTYPE)
    m["vertexOffset"] = meshes["vertexOffset"]
    m["vertexCount"] = meshes["vertexCount"]
    m["lods"][:, 0]["indexOffset"] = meshes["lods"][:, 0]["indexOffset"]
    m["lods"][:, 0]["indexCount"] = meshes["lods"][:, 0]["indexCount"]
    m["lodCount"] = 0x5A5A  # ignored
    return m


def dequantize(h):
    """meshopt_dequantizeHalf: fp16 denormals flush to 0, inf / NaN keep their payload"""
    h = h.astype(np.uint32)
    s = (h & 0x8000) << 16
    em = h & 0x7FFF
    r = (em + (112 << 10)) << 13
    r = np.where(em < (1 << 10), 0, r)
    r = r + np.where(em >= (31 << 10), 112 << 23, 0)
    return (s | r).astype(np.uint32).view(np.float32)


def make_vertices(positions, normals):
    """(n, 8) uint16 Vertex[]: fp16 positions, normals packed 10:10:10 as the reference's cooker does"""
    v = np.zeros((len(positions), 8), np.uint16)
    v[:, :3] = np.asarray(positions, np.float32).astype(np.float16).view(np.uint16) if np.asarray(positions).dtype != np.uint16 else positions
    n = np.clip(np.round((np.asarray(normals, np.float32) + 1.0) * 511.0), 0, 1023).astype(np.uint32)
    packed = n[:, 0] | (n[:, 1] << 10) | (n[:, 2] << 20)
    v[:, 4] = packed & 0xFFFF
    v[:, 5] = packed >> 16
    return v


# ---- the reference: appendMesh's LOD loop over the reference's meshoptimizer -------------------------------------------------

_REF = None


def ref_lib():
    global _REF
    if _REF is None:
        lib = ctypes.CDLL(SIMPLIFY_PATH)
        c_p, c_sz = ctypes.c_void_p, ctypes.c_size_t
        lib.meshopt_simplifyWithAttributes.restype = c_sz
        lib.meshopt_simplifyWithAttributes.argtypes = [c_p, c_p, c_sz, c_p, c_sz, c_sz, c_p, c_sz, c_p, c_sz, c_p, c_sz, ctypes.c_float, ctypes.c_uint, c_p]
        lib.meshopt_simplifyScale.restype = ctypes.c_float
        lib.meshopt_simplifyScale.argtypes = [c_p, c_sz, c_sz]
        lib.meshopt_optimizeVertexCache.restype = None
        lib.meshopt_optimizeVertexCache.argtypes = [c_p, c_p, c_sz, c_sz]
        _REF = lib
    return _REF


def ref_chain(vertices, lod0, max_scale=1.0):
    """(Mesh record fields, chain indices) of scene.cpp:193-268 for one mesh: vertices (n, 8) uint16, mesh-local lod0"""
    lib = ref_lib()
    f32 = np.float32
    n = len(vertices)
    pos = np.ascontiguousarray(dequantize(vertices[:, :3]).reshape(-1, 3))
    packed = vertices[:, 4].astype(np.uint32) | (vertices[:, 5].astype(np.uint32) << 16)
    nrm = np.ascontiguousarray(np.stack([((packed >> (10 * k)) & 1023).astype(f32) / f32(511) - f32(1) for k in range(3)], 1))
    with np.errstate(all="ignore"):
        # a sequential float sum (accumulate does not reorder), then the largest distance: NaN distances never win
        # `radius < d ? d : radius`, and fmax skips them too
        center = np.add.accumulate(pos, axis=0, dtype=f32)[-1] if n else np.zeros(3, f32)
        center = center / f32(n)
        d = pos - center
        dist = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
        radius = np.fmax.reduce(dist, initial=f32(0)) if n else f32(0)
    scale = f32(lib.meshopt_simplifyScale(pos.ctypes.data, n, 12))
    weights = np.ones(3, f32)
    cur = np.ascontiguousarray(lod0, np.uint32).copy()
    lod_error = f32(0)
    lods, chain = [], []
    while len(lods) < 8:
        with np.errstate(all="ignore"):
            lods.append((sum(len(c) for c in chain), len(cur), f32(lod_error * scale)))
        chain.append(cur.copy())
        if len(lods) == 8:
            break
        target = (int(float(len(cur)) * 0.6) // 3) * 3
        err = ctypes.c_float()
        nxt = lib.meshopt_simplifyWithAttributes(cur.ctypes.data, cur.ctypes.data, len(cur), pos.ctypes.data, n, 12, nrm.ctypes.data, 12, weights.ctypes.data, 3, None,
                                                 target, 1e-1, 2, ctypes.byref(err))
        if nxt == len(cur) or nxt == 0 or nxt >= int(float(len(cur)) * 0.85):
            break
        cur = cur[:nxt].copy()
        grown = f32(lod_error * f32(1.5))
        lod_error = f32(err.value) if grown < f32(err.value) else grown
        lib.meshopt_optimizeVertexCache(cur.ctypes.data, cur.ctypes.data, len(cur), n)
    rt = 0
    for i, (_, _, e) in enumerate(lods):
        with np.errstate(all="ignore"):
            if f32(e * f32(max_scale)) < f32(3e-3):
                rt = i
    return dict(center=np.array(center, f32), radius=f32(radius), lods=lods, lodRT=rt), np.concatenate(chain) if chain else np.zeros(0, np.uint32)


def ref_scene(vertices, indices, host_meshes, max_scale=None):
    """Mesh[] and ib the reference stores for these meshes, meshlet fields zeroed"""
    out = np.zeros(len(host_meshes), layout.MESH_DTYPE)
    ib = []
    total = 0
    for i, hm in enumerate(host_meshes):
        vo, vc = int(hm["vertexOffset"]), int(hm["vertexCount"])
        io, ic = int(hm["lods"][0]["indexOffset"]), int(hm["lods"][0]["indexCount"])
        rec, chain = ref_chain(vertices[vo: vo + vc], indices[io: io + ic], 1.0 if max_scale is None else max_scale[i])
        m = out[i: i + 1]
        m["center"] = rec["center"]
        m["radius"] = rec["radius"]
        m["vertexOffset"], m["vertexCount"] = vo, vc
        m["lodCount"] = len(rec["lods"])
        m["lodRT"] = rec["lodRT"]
        for l, (off, cnt, err) in enumerate(rec["lods"]):
            m["lods"][0, l]["indexOffset"] = total + off
            m["lods"][0, l]["indexCount"] = cnt
            m["lods"][0, l]["error"] = err
        total += len(chain)
        ib.append(chain)
    return out, (np.concatenate(ib).astype(np.uint32) if ib else np.zeros(0, np.uint32))


# ---- the product, emulated (host pointers) or on the device ---------------------------------------------------------------

def capacity(lib, meshes):
    n = ctypes.c_uint32()
    assert lib.nvc_cook_mesh_lods_capacity(meshes.ctypes.data, len(meshes), ctypes.byref(n)) == 0
    return n.value


class Emu:
    def __init__(self):
        self.lib = emu_lib.load()
        self.ctx = ctypes.c_void_p()
        assert self.lib.nvc_create(0, None, ctypes.byref(self.ctx)) == 0

    def close(self):
        self.lib.nvc_destroy(self.ctx)

    def cook(self, vertices, indices, meshes, max_scale=None, cap=None, vertex_count=None, index_count=None):
        """(Mesh[], ib, totals4); status != 0 raises ValueError(status) after checking the outputs are untouched"""
        cap = capacity(self.lib, meshes) if cap is None else cap
        out_meshes = np.full(len(meshes) * 208, 0xCD, np.uint8)
        ib = np.full(cap + 4, 0xA5A5A5A5, np.uint32)
        totals = np.full(4, 0x77, np.uint32)
        vertices = np.ascontiguousarray(vertices)
        indices = np.ascontiguousarray(indices, np.uint32)
        scale = None if max_scale is None else np.ascontiguousarray(max_scale, np.float32)
        status = self.lib.nvc_cook_mesh_lods(self.ctx, None, vertices.ctypes.data if len(vertices) else None, len(vertices) if vertex_count is None else vertex_count,
                                             indices.ctypes.data if len(indices) else None, len(indices) if index_count is None else index_count, meshes.ctypes.data,
                                             scale.ctypes.data if scale is not None else None, len(meshes), out_meshes.ctypes.data, ib.ctypes.data, cap, totals.ctypes.data)
        if status != 0:
            assert (out_meshes == 0xCD).all() and (ib == 0xA5A5A5A5).all() and (totals == 0x77).all(), "a refused call wrote its outputs"
            raise ValueError(status)
        assert (ib[cap:] == 0xA5A5A5A5).all(), "write past the capacity"
        m = out_meshes.view(layout.MESH_DTYPE)
        return m, (None if totals[2] else ib[: int(totals[0])]), totals


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

    def cook(self, vertices, indices, meshes, max_scale=None, stream=None):
        torch = self.torch
        cap = capacity(self.lib, meshes)
        dv = torch.from_numpy(np.ascontiguousarray(vertices).view(np.uint8).reshape(-1).copy()).cuda()
        di = torch.from_numpy(np.ascontiguousarray(indices, np.uint32).view(np.int32).copy()).cuda()
        dm = torch.zeros(len(meshes) * 208, dtype=torch.uint8, device="cuda")
        dib = torch.zeros(cap + 1, dtype=torch.int32, device="cuda")
        dt = torch.zeros(4, dtype=torch.int32, device="cuda")
        scale = None if max_scale is None else np.ascontiguousarray(max_scale, np.float32)
        s = stream.cuda_stream if stream is not None else None
        self.check(self.lib.nvc_cook_mesh_lods(self.ctx, s, dv.data_ptr(), len(vertices), di.data_ptr(), len(indices), meshes.ctypes.data,
                                               scale.ctypes.data if scale is not None else None, len(meshes), dm.data_ptr(), dib.data_ptr(), cap, dt.data_ptr()),
                   self.ctx, "nvc_cook_mesh_lods")
        torch.cuda.synchronize()
        totals = dt.cpu().numpy().view(np.uint32)
        return dm.cpu().numpy().view(layout.MESH_DTYPE), dib.cpu().numpy().view(np.uint32)[: int(totals[0])], totals


def assert_same(got, want, what):
    gm, gib, gt = got
    wm, wib = want
    assert gt[1] == 0 and gt[2] == 0 and gt[3] == 0 and gt[0] == len(wib), (what, gt, len(wib))
    if gm.tobytes() != wm.tobytes():
        for i in range(len(wm)):
            assert gm[i].tobytes() == wm[i].tobytes(), (what, "mesh", i, gm[i], wm[i])
    bad = np.nonzero(gib != wib)[0]
    assert len(bad) == 0, (what, "indices", len(bad), bad[:8])


@pytest.fixture(scope="module")
def emu():
    e = Emu()
    yield e
    e.close()


# ---- CPU tier --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_emulated(emu, name):
    """Vertex[] and LOD 0 of a reference run -> the Mesh[] (meshlet fields aside) and whole ib its cooker stored, bit for bit"""
    v, ib, meshes, scale = fixture(name)
    assert_same(emu.cook(v, ib, lod0_input(meshes), scale), (meshes, ib), name)


@needs_ref
@pytest.mark.parametrize("name", FIXTURES)
def test_restatement_matches_fixtures(name):
    """ref_chain, the LOD loop restated over the reference's library, reproduces what the reference's cooker stored"""
    v, ib, meshes, scale = fixture(name)
    wm, wib = ref_scene(v, ib, lod0_input(meshes), scale)
    assert wm.tobytes() == meshes.tobytes() and np.array_equal(wib, ib), name


def end_to_end_emulated(emu, ref_file, raw, clrt):
    """nvc_cook_mesh_lods -> nvc_cook_meshlets(_clrt) -> nvc_scene_cache_write, all emulated on one context, from the run's
    Vertex[] and LOD 0"""
    import test_scene_cache_write as write_tests

    lib, ctx = emu.lib, emu.ctx
    header, secs = raw_geometry(raw)
    header.clrtMode = int(clrt)
    v = secs["vertices"].view(np.uint16).reshape(-1, 8)
    stored = secs["meshes"].view(layout.MESH_DTYPE)
    scale = max_scale_of("animated_clrt" if clrt else raw, len(stored))
    cap = capacity(lib, lod0_input(stored))
    meshes = np.zeros(len(stored), layout.MESH_DTYPE)
    ib = np.zeros(cap + 1, np.uint32)
    totals = np.zeros(4, np.uint32)
    src_ib = secs["indices"].view(np.uint32)
    m0 = lod0_input(stored)
    assert lib.nvc_cook_mesh_lods(ctx, None, v.ctypes.data, len(v), src_ib.ctypes.data, len(src_ib), m0.ctypes.data, scale.ctypes.data, len(m0),
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
        st = lib.nvc_cook_meshlets_clrt(ctx, None, v.ctypes.data, len(v), ib.ctypes.data, len(ib), meshes.ctypes.data, scale.ctypes.data, out_meshes.ctypes.data, len(meshes),
                                        ml.ctypes.data, nm.value, md.ctypes.data, nw.value, vtx0.ctypes.data, nv.value, t.ctypes.data)
    else:
        st = lib.nvc_cook_meshlets(ctx, None, v.ctypes.data, len(v), ib.ctypes.data, len(ib), meshes.ctypes.data, out_meshes.ctypes.data, len(meshes),
                                   ml.ctypes.data, nm.value, md.ctypes.data, nw.value, t.ctypes.data)
    assert st == 0 and t[3] == 0
    s2 = dict(secs)
    s2.update(indices=ib, meshes=out_meshes.view(np.uint8), meshlets=ml[: int(t[0]) * 24], meshletdata=md[: int(t[1])])
    if clrt:
        s2["meshletvtx0"] = vtx0[: int(t[4])]
    status, got = write_tests.write(lib, ctx, write_tests.make_desc(header, s2, True))
    assert status == 0
    return got


@pytest.mark.parametrize("ref_file,raw,clrt", END_TO_END)
def test_end_to_end_emulated(emu, ref_file, raw, clrt):
    """Vertex[] and LOD 0 -> LOD chains -> meshlets -> compressed cache: the reference's file, byte for byte"""
    want = np.fromfile(os.path.join(GOLDEN, ref_file), np.uint8)
    got = end_to_end_emulated(emu, ref_file, raw, clrt)
    assert len(got) == len(want) and np.array_equal(got, want), ref_file


def grid_mesh(rng, nx, ny, seam=False, jitter=0.0):
    """an open nx * ny quad grid (borders), optionally with a UV-style seam: the middle column duplicated with other normals"""
    xs, ys = np.meshgrid(np.linspace(0, 1, nx + 1), np.linspace(0, 1, ny + 1))
    pos = np.stack([xs.ravel(), ys.ravel(), 0.1 * np.sin(3 * xs.ravel()) * np.cos(2 * ys.ravel())], 1).astype(np.float32)
    pos += rng.normal(0, jitter, pos.shape).astype(np.float32)
    nrm = np.tile(np.array([[0, 0, 1]], np.float32), (len(pos), 1))
    idx = []
    vid = lambda x, y: y * (nx + 1) + x  # noqa: E731
    extra = {}
    for y in range(ny):
        for x in range(nx):
            q = [vid(x, y), vid(x + 1, y), vid(x + 1, y + 1), vid(x, y + 1)]
            if seam and x >= nx // 2:
                for k, c in enumerate(q):
                    if c % (nx + 1) == nx // 2:
                        if c not in extra:
                            extra[c] = len(pos) + len(extra)
                        q[k] = extra[c]
            idx += [q[0], q[1], q[2], q[0], q[2], q[3]]
    if extra:
        keys = sorted(extra, key=extra.get)
        pos = np.concatenate([pos, pos[keys]])
        nrm = np.concatenate([nrm, np.tile(np.array([[1, 0, 0]], np.float32), (len(keys), 1))])
    return pos, nrm, np.array(idx, np.uint32)


def sphere_mesh(rng, n=12):
    """a closed UV sphere (manifold), normals = positions"""
    pos, idx = [], []
    for i in range(n + 1):
        for j in range(2 * n):
            t, p = np.pi * i / n, 2 * np.pi * j / (2 * n)
            pos.append([np.sin(t) * np.cos(p), np.sin(t) * np.sin(p), np.cos(t)])
    for i in range(n):
        for j in range(2 * n):
            a, b = i * 2 * n + j, i * 2 * n + (j + 1) % (2 * n)
            c, d = a + 2 * n, b + 2 * n
            idx += [a, c, b, b, c, d]
    pos = np.array(pos, np.float32) + rng.normal(0, 1e-3, (len(pos), 3)).astype(np.float32)
    return pos, pos / np.linalg.norm(pos, axis=1, keepdims=True), np.array(idx, np.uint32)


def seeded_meshes():
    rng = np.random.default_rng(7)
    out = {}
    out["border"] = grid_mesh(rng, 12, 10)
    out["seam"] = grid_mesh(rng, 12, 12, seam=True)
    out["sphere"] = sphere_mesh(rng)
    p, n, i = grid_mesh(rng, 8, 8, jitter=0.01)
    out["jitter"] = (p, n, i)
    # several components, with unreferenced vertices between them
    a, b = sphere_mesh(rng, 8), grid_mesh(rng, 6, 6)
    gap = np.zeros((5, 3), np.float32)
    out["components"] = (np.concatenate([a[0], gap, b[0] + 3]), np.concatenate([a[1], gap + [0, 0, 1], b[1]]), np.concatenate([a[2], b[2] + len(a[0]) + 5]))
    # non-manifold: a fin on a grid edge, a bowtie, degenerate and duplicate triangles
    p, n, i = grid_mesh(rng, 6, 6)
    fin = np.array([[0.5, 0.5, 0.5]], np.float32)
    v0 = len(p)
    p, n = np.concatenate([p, fin, fin + [0.2, 0, 0]]), np.concatenate([n, [[1, 0, 0], [1, 0, 0]]])
    e = i[:2]
    i = np.concatenate([i, [e[0], e[1], v0], [e[1], v0, v0 + 1], [i[3], i[3], i[4]], i[6:9], i[6:9]]).astype(np.uint32)
    out["nonmanifold"] = (p, n, i)
    out["single"] = (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32), np.tile([[0, 0, 1]], (3, 1)).astype(np.float32), np.array([0, 1, 2], np.uint32))
    out["empty"] = (np.array([[0, 0, 0], [1, 0, 0]], np.float32), np.tile([[0, 0, 1]], (2, 1)).astype(np.float32), np.zeros(0, np.uint32))
    out["big"] = sphere_mesh(rng, 40)  # 8 LODs
    return out


def special_positions():
    """fp16 +-0, denormals, +-inf and NaN in the positions of a small grid"""
    rng = np.random.default_rng(11)
    p, n, i = grid_mesh(rng, 6, 6)
    v = make_vertices(p, n)
    v[0, 0], v[1, 1] = 0x8000, 0x0000  # -0, +0
    v[2, 0], v[3, 2] = 0x0001, 0x83FF  # denormals (flush to 0)
    v[4, 1], v[5, 2] = 0x7C00, 0xFC00  # +inf, -inf
    v[6, 0], v[7, 1] = 0x7E01, 0xFD00  # NaN (quiet), NaN (signalling payload)
    return v, i


def scene_of(parts):
    verts, idx, meshes = [], [], []
    vb = ib = 0
    for v, i in parts:
        m = np.zeros(1, layout.MESH_DTYPE)
        m["vertexOffset"], m["vertexCount"] = vb, len(v)
        m["lods"][0, 0]["indexOffset"], m["lods"][0, 0]["indexCount"] = ib, len(i)
        verts.append(v)
        idx.append(i)
        vb += len(v)
        ib += len(i)
        meshes.append(m)
    return np.concatenate(verts), np.concatenate(idx).astype(np.uint32), np.concatenate(meshes)


@needs_ref
@pytest.mark.parametrize("name", ["border", "seam", "sphere", "jitter", "components", "nonmanifold", "single", "empty", "big", "special"])
def test_seeded_emulated(emu, name):
    if name == "special":
        v, i = special_positions()
    else:
        p, n, i = seeded_meshes()[name]
        v = make_vertices(p, n)
    v_all, i_all, m = scene_of([(v, i)])
    want = ref_scene(v_all, i_all, m)
    assert_same(emu.cook(v_all, i_all, m), want, name)
    if name == "big":
        assert int(want[0]["lodCount"][0]) == 8
    if name == "single":
        assert int(want[0]["lodCount"][0]) == 1


@needs_ref
def test_loop_exits_are_exercised():
    """the seeded meshes reach every exit of appendMesh's loop: 8 LODs, "no change", 0 indices, and the 85% rule"""
    exits = set()
    lib = ref_lib()
    for name, (p, n, i) in seeded_meshes().items():
        v = make_vertices(p, n)
        rec, _ = ref_chain(v, i)
        lods = rec["lods"]
        if len(lods) == 8:
            exits.add("eight")
            continue
        # replay the simplification after the last LOD to see which exit it took
        pos = np.ascontiguousarray(dequantize(v[:, :3]).reshape(-1, 3))
        cnt = lods[-1][1]
        if cnt == 0:
            exits.add("zero")
            continue
        _, chain = ref_chain(v, i)
        cur = np.ascontiguousarray(chain[lods[-1][0]:], np.uint32).copy()
        packed = v[:, 4].astype(np.uint32) | (v[:, 5].astype(np.uint32) << 16)
        nrm = np.ascontiguousarray(np.stack([((packed >> (10 * k)) & 1023).astype(np.float32) / np.float32(511) - np.float32(1) for k in range(3)], 1))
        err = ctypes.c_float()
        nxt = lib.meshopt_simplifyWithAttributes(cur.ctypes.data, cur.ctypes.data, cnt, pos.ctypes.data, len(v), 12, nrm.ctypes.data, 12, np.ones(3, np.float32).ctypes.data, 3, None,
                                                 (int(cnt * 0.6) // 3) * 3, 1e-1, 2, ctypes.byref(err))
        exits.add("zero" if nxt == 0 else ("same" if nxt == cnt else "85%"))
    assert {"eight", "same", "zero", "85%"} <= exits, exits


@needs_ref
def test_many_meshes_equal_one_call_each(emu):
    meshes = seeded_meshes()
    parts = [(make_vertices(p, n), i) for p, n, i in (meshes[k] for k in ("border", "seam", "sphere", "components", "nonmanifold", "single", "empty"))]
    parts.append(special_positions())
    v, i, m = scene_of(parts)
    gm, gib, gt = emu.cook(v, i, m)
    base = 0
    for k, part in enumerate(parts):
        pv, pi, pm = scene_of([part])
        om, oib, ot = emu.cook(pv, pi, pm)
        want = om.copy()
        want["vertexOffset"] = m["vertexOffset"][k]
        want["lods"]["indexOffset"][0, : int(om["lodCount"][0])] += base
        assert gm[k].tobytes() == want[0].tobytes(), k
        assert np.array_equal(gib[base: base + len(oib)], oib), k
        base += len(oib)
    assert base == len(gib) == gt[0]


def test_capacity_and_overflow(emu):
    rng = np.random.default_rng(3)
    p, n, i = sphere_mesh(rng, 16)
    v, i, m = scene_of([(make_vertices(p, n), i), (make_vertices(p, n), i)])
    cap = capacity(emu.lib, m)
    gm, gib, gt = emu.cook(v, i, m)
    assert gt[0] <= cap and gt[2] == 0
    # one index short: the flag, no index written (cook() checks the buffer beyond), Mesh[] written all the same
    om, oib, ot = emu.cook(v, i, m, cap=int(gt[0]) - 1)
    assert ot[2] == 1 and oib is None and ot[0] == gt[0]
    assert om.tobytes() == gm.tobytes()
    # the capacity is exact: c0 = n, c(l+1) = the largest multiple of 3 below c(l) * 0.85, at most 8 LODs
    def bound(n):
        total, c = 0, n
        for _ in range(8):
            total += c
            below = int(c * 0.85)
            c = (below - 1) // 3 * 3 if below else 0
            if c <= 0:
                break
        return total
    for n in (0, 3, 6, 9, 12, 300, 86832):
        one = np.zeros(1, layout.MESH_DTYPE)
        one["lods"][0, 0]["indexCount"] = n
        assert capacity(emu.lib, one) == bound(n), n


def test_rejected_mesh_reads_no_vertex():
    """a rejected mesh's vertices lie past the end of an array that ends at an inaccessible page, and the call's device
    allocations end at one too: reading any of them, or past any scratch array, faults"""
    import test_scene_cache_device as dev_tests

    lib = emu_lib.load()
    rng = np.random.default_rng(13)
    p, n, i = grid_mesh(rng, 4, 4)
    good = make_vertices(p, n)
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
    cap = capacity(lib, m)
    meshes = np.zeros(2, layout.MESH_DTYPE)
    ib = np.zeros(cap, np.uint32)
    totals = np.zeros(4, np.uint32)
    ctx = ctypes.c_void_p()
    assert lib.nvc_create(0, None, ctypes.byref(ctx)) == 0
    lib.emu_guard_allocations(1)
    try:
        status = lib.nvc_cook_mesh_lods(ctx, None, vertices.ctypes.data, len(good) + bad_count, idx.ctypes.data, len(idx), m.ctypes.data, None, 2,
                                        meshes.ctypes.data, ib.ctypes.data, cap, totals.ctypes.data)
    finally:
        lib.emu_guard_allocations(0)
        lib.nvc_destroy(ctx)
        assert lib.emu_guarded_live() == 0
    assert status == 0 and totals[1] == 1 and totals[2] == 0
    assert int(meshes[1]["lodCount"]) == 0 and int(meshes[0]["lodCount"]) >= 1
    want = ref_scene(good, i, m[:1]) if os.path.exists(SIMPLIFY_PATH) else None
    if want is not None:
        assert meshes[0].tobytes() == want[0][0].tobytes() and np.array_equal(ib[: int(totals[0])], want[1])


def test_rejected_mesh(emu):
    rng = np.random.default_rng(5)
    p, n, i = grid_mesh(rng, 4, 4)
    good = make_vertices(p, n)
    bad_i = i.copy()
    bad_i[7] = len(p)  # one past the mesh's vertices
    v, idx, m = scene_of([(good, i), (good, bad_i), (good, i)])
    gm, gib, gt = emu.cook(v, idx, m)
    assert gt[1] == 1
    assert int(gm[1]["lodCount"]) == 0 and gm[1]["radius"] == 0 and (gm[1]["center"] == 0).all()
    assert gm[1]["vertexOffset"] == m[1]["vertexOffset"] and gm[1]["vertexCount"] == m[1]["vertexCount"]
    assert gm[0]["lods"]["indexCount"][0] == len(i) and gm[2]["lods"]["indexOffset"][0] == int(gm[0]["lods"]["indexCount"][: int(gm[0]["lodCount"])].sum())


def test_argument_refusals(emu):
    rng = np.random.default_rng(9)
    p, n, i = grid_mesh(rng, 3, 3)
    v, idx, m = scene_of([(make_vertices(p, n), i)])
    for mutate in (lambda x: x["lods"][0, 0].__setitem__("indexCount", 5),
                   lambda x: x["lods"][0, 0].__setitem__("indexOffset", 3),
                   lambda x: x.__setitem__("vertexOffset", 1)):
        bad = m.copy()
        mutate(bad)
        with pytest.raises(ValueError, match=str(-1)):
            emu.cook(v, idx, bad)


# ---- GPU tier --------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def gpu():
    g = Gpu()
    yield g
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_gpu(gpu, name):
    v, ib, meshes, scale = fixture(name)
    assert_same(gpu.cook(v, ib, lod0_input(meshes), scale), (meshes, ib), name)


@pytest.mark.gpu
@pytest.mark.parametrize("ref_file,raw,clrt", END_TO_END)
def test_end_to_end_gpu(gpu, ref_file, raw, clrt):
    """the same chain on the device, the cache written from device memory: the reference's file"""
    import torch

    import test_scene_cache_write as write_tests

    want = np.fromfile(os.path.join(GOLDEN, ref_file), np.uint8)
    header, secs = raw_geometry(raw)
    header.clrtMode = int(clrt)
    stored = secs["meshes"].view(layout.MESH_DTYPE)
    scale = max_scale_of("animated_clrt" if clrt else raw, len(stored))
    v = secs["vertices"].view(np.uint16).reshape(-1, 8)
    meshes, ib, totals = gpu.cook(v, secs["indices"].view(np.uint32), lod0_input(stored), scale)
    assert totals[1] == 0 and totals[2] == 0
    s2 = dict(secs)
    s2.update(indices=ib.view(np.uint8), meshes=meshes.view(np.uint8))
    cooked = write_tests._cook(gpu.lib, gpu.ctx, s2, clrt, scale if clrt else None)
    s2.update(cooked)
    torch.cuda.synchronize()
    got = write_tests._write_py(header, s2, True)
    assert len(got) == len(want) and np.array_equal(got, want), ref_file


def jittered_fixture_scene(copies, seed=1):
    """`copies` copies of the fixture meshes (kitten, pirate.obj, pirate.glb, animated's two), positions jittered"""
    rng = np.random.default_rng(seed)
    sources = []
    for name in ("kitten", "pirate", "pirateglb", "animated"):
        v, ib, meshes, _ = fixture(name)
        for mesh in meshes:
            vo, vc = int(mesh["vertexOffset"]), int(mesh["vertexCount"])
            io, ic = int(mesh["lods"][0]["indexOffset"]), int(mesh["lods"][0]["indexCount"])
            sources.append((v[vo: vo + vc], ib[io: io + ic]))
    parts = []
    for k in range(copies):
        sv, si = sources[k % len(sources)]
        part = sv.copy()
        pos = part[:, :3].view(np.float16).astype(np.float32)
        pos = pos * rng.uniform(0.5, 2.0) + rng.uniform(-100, 100, (1, 3)).astype(np.float32) + rng.normal(0, 1e-3, pos.shape).astype(np.float32)
        part[:, :3] = pos.astype(np.float16).view(np.uint16)
        parts.append((part, si))
    return scene_of(parts)


@pytest.mark.gpu
@needs_ref
def test_jittered_scene_gpu(gpu):
    v, i, m = jittered_fixture_scene(300)
    assert_same(gpu.cook(v, i, m), ref_scene(v, i, m), "300 jittered copies")


@pytest.mark.gpu
def test_busy_nonblocking_stream_gpu(gpu):
    import torch

    v, ib, meshes, scale = fixture("animated")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a = torch.randn(4096, 4096, device="cuda")
        for _ in range(8):
            a = a @ a.T / 4096
    m0 = lod0_input(meshes)
    got = gpu.cook(v, ib, m0, scale, stream=s)
    torch.cuda.synchronize()
    want = gpu.cook(v, ib, m0, scale)
    assert_same(got, want[:2], "non-blocking stream")
