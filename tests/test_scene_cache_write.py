"""nvc_scene_cache_write: the file saveSceneCache writes, byte for byte.  The CPU tier runs the product's encoder kernels under
the SIMT emulation (tests/emu_lib.py), some writes with allocations that end at an inaccessible page; the GPU tier writes through scene_cache.write_scene_cache.  The reference files are
tests/golden/*.z.cache with the raw geometry of the same runs (scene_cache_write_raw.npz, animated.raw.cache); the codec
streams are compared against the reference's own encoders (oracle/_ref/libmeshopt_ref.so), skipped where that library was not
built."""
import ctypes
import os

import numpy as np
import pytest

import test_scene_cache_device as dev_tests
from niagara_b200 import layout
from niagara_b200.scene_cache import _ELEMENT_SIZE
from niagara_b200.lib import load_library

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
SECTIONS = layout.CACHE_SECTIONS
OK, INVALID = 0, -1
# (compressed reference file, raw geometry of the same run): the raw fixture is a file, or a key of the npz
REFERENCE_FILES = [("animated.z.cache", "animated.raw.cache"), ("kitten.z.cache", "kitten"), ("pirateglb.z.cache", "pirateglb"), ("animated_clrt.z.cache", "animated_clrt")]
RAW_NPZ = os.path.join(GOLDEN, "scene_cache_write_raw.npz")
needs_ref = dev_tests.needs_ref
vp, sz = ctypes.c_void_p, ctypes.c_size_t


def raw_file(name):
    if name.endswith(".cache"):
        return np.fromfile(os.path.join(GOLDEN, name), np.uint8)
    with np.load(RAW_NPZ) as z:
        return z[name]


def raw_sections(data):
    """the header and every section's bytes of an uncompressed cache"""
    info = layout.SceneCacheInfo()
    assert load_library().nvc_scene_cache_parse(data.ctypes.data, len(data), ctypes.byref(info)) == OK
    assert not info.header.compressed
    secs = {}
    for s, name in enumerate(SECTIONS):
        sec = info.sections[s]
        secs[name] = data[int(sec.offset) : int(sec.offset + sec.stored_bytes)].copy()
    return info.header, secs


def make_desc(header, secs, compressed, device_mask=0):
    desc = layout.SceneCacheWriteDesc()
    desc.hashMeta, desc.clrtMode, desc.compressed, desc.ommStates = header.hashMeta, header.clrtMode, int(compressed), header.ommStates
    desc.camera = header.camera
    desc.sunDirection[:] = list(header.sunDirection)
    desc.device_sections = device_mask
    keep = []
    for s, name in enumerate(SECTIONS):
        a = np.ascontiguousarray(secs.get(name, np.zeros(0, np.uint8)))
        keep.append(a)
        desc.data[s] = a.ctypes.data if a.nbytes else None
        desc.count[s] = a.nbytes // _ELEMENT_SIZE[name]
    desc._keep = keep
    return desc


def write(lib, ctx, desc, capacity=None, fill=0xEE):
    bound = ctypes.c_size_t()
    assert lib.nvc_scene_cache_write_bound(ctypes.byref(desc), ctypes.byref(bound)) == OK
    cap = int(bound.value) if capacity is None else capacity
    out = np.full(max(cap, 1), fill, np.uint8)
    size = ctypes.c_size_t()
    status = lib.nvc_scene_cache_write(ctx, None, ctypes.byref(desc), out.ctypes.data, cap, ctypes.byref(size))
    return status, out[: size.value] if status == OK else out


# ---- CPU tier ---------------------------------------------------------------------------------------------------------
def emu():
    """the emulated library and a context of it (test_scene_cache_device's)"""
    return dev_tests._emu()


def ref_lib():
    lib = dev_tests._ref()
    lib.meshopt_encodeIndexBufferBound.restype = sz
    lib.meshopt_encodeIndexBufferBound.argtypes = [sz, sz]
    lib.meshopt_encodeIndexBuffer.restype = sz
    lib.meshopt_encodeIndexBuffer.argtypes = [vp, sz, vp, sz]
    return lib


def ref_index_stream(ref, idx):
    idx = np.ascontiguousarray(idx, np.uint32)
    buf = np.zeros(ref.meshopt_encodeIndexBufferBound(len(idx), 0xFFFFFFFF), np.uint8)
    n = ref.meshopt_encodeIndexBuffer(buf.ctypes.data, len(buf), idx.ctypes.data, len(idx))
    assert n > 0
    return buf[:n].copy()


def ref_meshlet_section(ref, meshlets, meshletdata):
    """MESHLETDATA as writeMeshletDataCompressed builds it: per meshlet a uint16 size and meshopt_encodeMeshlet's block"""
    words = np.ascontiguousarray(meshletdata, np.uint32)
    out = []
    for m in meshlets:
        vc, tc, off = int(m["vertexCount"]), int(m["triangleCount"]), int(m["dataOffset"])
        if m["shortRefs"]:
            refs = words[off:].view(np.uint16)[:vc].astype(np.uint32)
            vw = (vc + 1) // 2
        else:
            refs = words[off : off + vc]
            vw = vc
        tris = words[off + vw :].view(np.uint8)[: tc * 3]
        block = dev_tests.encode_meshlet(ref, refs, tris) if vc or tc else encode_empty(ref)
        out.append(np.uint16(len(block)).tobytes() + block.tobytes())
    return np.frombuffer(b"".join(out), np.uint8)


def encode_empty(ref):
    buf = np.zeros(ref.meshopt_encodeMeshletBound(256, 256), np.uint8)
    n = ref.meshopt_encodeMeshlet(buf.ctypes.data, len(buf), None, 0, None, 0)
    return buf[:n].copy()


def compressed_sections(data):
    """(info, {name: stored bytes}) of a compressed file"""
    info = layout.SceneCacheInfo()
    assert load_library().nvc_scene_cache_parse(data.ctypes.data, len(data), ctypes.byref(info)) == OK
    return info, {name: data[int(info.sections[s].offset) : int(info.sections[s].offset + info.sections[s].stored_bytes)] for s, name in enumerate(SECTIONS)}


def only(secs_or_streams, compressed, ctx_lib, **fields):
    """write a cache holding the given sections and return (status, file)"""
    lib, ctx = ctx_lib
    h = layout.SceneCacheHeader()
    return write(lib, ctx, make_desc(h, secs_or_streams, compressed, **fields))


def written_stream(ctx_lib, name, array):
    status, out = only({name: array}, True, ctx_lib)
    assert status == OK, status
    info, streams = compressed_sections(out)
    return streams[name]


@pytest.mark.parametrize("raw", ["animated.raw.cache", "kitten", "pirateglb", "animated_clrt"])
def test_raw_round_trip(raw):
    data = raw_file(raw)
    header, secs = raw_sections(data)
    lib, ctx = emu()
    for c in (ctx, None):  # an uncompressed write of host arrays needs no context
        status, out = write(lib, c, make_desc(header, secs, False))
        assert status == OK
        assert np.array_equal(out, data)


@pytest.mark.parametrize("ref_file,raw", REFERENCE_FILES)
def test_reference_files(ref_file, raw):
    want = np.fromfile(os.path.join(GOLDEN, ref_file), np.uint8)
    header, secs = raw_sections(raw_file(raw))
    header.clrtMode = np.frombuffer(want[:160].tobytes(), np.uint8)[24]
    lib, ctx = emu()
    status, out = write(lib, ctx, make_desc(header, secs, True))
    assert status == OK
    assert len(out) == len(want) and np.array_equal(out, want), (ref_file, int(np.flatnonzero(out[: len(want)] != want[: len(out)])[0]) if min(len(out), len(want)) else -1)


VERTEX_COUNTS = (0, 1, 2, 15, 16, 17, 255, 256, 257, 767, 768, 769)


@needs_ref
@pytest.mark.parametrize("stride", [16, 8])
def test_vertex_streams_against_reference(stride):
    ref = ref_lib()
    rng = np.random.default_rng(1000 + stride)
    name = "vertices" if stride == 16 else "meshletvtx0"
    cases = 0
    for count in VERTEX_COUNTS:
        for kind in ("random", "zeros", "smooth16", "floats", "sparse", "channel1", "tie"):
            values = vertex_values(rng, count, stride, kind)
            want = dev_tests.encode_vertices(ref, values, 2, 1)
            got = written_stream(emu(), name, values.reshape(-1))
            assert np.array_equal(got, want), (stride, count, kind)
            cases += 1
    assert cases == len(VERTEX_COUNTS) * 7


def vertex_values(rng, count, stride, kind):
    if kind == "channel1":  # slowly varying 16-bit fields whose low bytes wrap: the 16-bit delta channel wins
        base = np.cumsum(rng.integers(-300, 301, (count, stride // 2)), axis=0).astype(np.int64) + 30000
        return (base & 0xFFFF).astype("<u2").view(np.uint8).reshape(count, stride)
    if kind == "tie":  # a constant first column: both channels measure the same there, and channel 0 is kept
        v = np.zeros((count, stride), np.uint8)
        v[:, :4] = rng.integers(0, 256, 4)
        v[:, 4:] = np.arange(count)[:, None] % 7 * (np.arange(stride - 4)[None, :] % 2)
        return v
    return dev_tests.vertex_data(rng, count, stride, kind)


@needs_ref
def test_vertex_stream_of_more_than_1024_blocks():
    ref = ref_lib()
    rng = np.random.default_rng(1100)
    for stride, kind in ((16, "smooth16"), (8, "channel1")):
        values = vertex_values(rng, 1030 * 256 + 77, stride, kind)
        want = dev_tests.encode_vertices(ref, values, 2, 1)
        got = written_stream(emu(), "vertices" if stride == 16 else "meshletvtx0", values.reshape(-1))
        assert np.array_equal(got, want), stride


def meshlet_inputs(rng, cases):
    """Meshlet[] and meshletdata for (vertexCount, triangleCount, style, shortRefs) cases, packed as appendMeshlet packs
    them, with garbage in the padding bytes (the encoder must not read them)"""
    meshlets = np.zeros(len(cases), layout.MESHLET_DTYPE)
    words = []
    at = 0
    for i, (vc, tc, style, short) in enumerate(cases):
        refs, tris = meshlet_refs_tris(rng, vc, tc, style)
        short = short and (vc == 0 or int(refs.max()) < 65536)
        rb = refs.astype("<u2").tobytes() if short else refs.astype("<u4").tobytes()
        rb += b"\xab" * (-len(rb) % 4)
        tb = tris.astype(np.uint8).tobytes()
        tb += bytes(rng.integers(0, 256, -len(tb) % 4, dtype=np.uint8))
        w = np.frombuffer(rb + tb, "<u4")
        meshlets[i]["dataOffset"], meshlets[i]["vertexCount"], meshlets[i]["triangleCount"], meshlets[i]["shortRefs"] = at, vc, tc, int(short)
        words.append(w)
        at += len(w)
    return meshlets, (np.concatenate(words) if words else np.zeros(0, np.uint32)).astype(np.uint32)


def meshlet_refs_tris(rng, vc, tc, style):
    if style == "chain":  # strips: edge reuse of the last triangles
        i = np.arange(tc) % max(1, vc - 2)
        tris = np.stack([i, i + 1, i + 2], 1)
        if tc:
            tris[1::2] = tris[1::2][:, [1, 0, 2]]
    elif style == "restart":  # fresh triangles: each fea / feb / fec pattern, next-vertex runs and explicit bytes
        tris = np.zeros((tc, 3), np.int64)
        nxt = 0
        for t in range(tc):
            p = t % 4
            if p == 0 and nxt + 3 <= vc:
                tris[t] = (nxt, nxt + 1, nxt + 2)
                nxt += 3
            elif p == 1 and nxt + 2 <= vc:
                tris[t] = (rng.integers(0, max(1, nxt)), nxt, nxt + 1)
                nxt += 2
            elif p == 2 and nxt + 1 <= vc:
                tris[t] = (rng.integers(0, max(1, nxt)), rng.integers(0, max(1, nxt)), nxt)
                nxt += 1
            else:
                tris[t] = rng.integers(0, max(vc, 1), 3)
    else:
        tris = rng.integers(0, max(vc, 1), (tc, 3))
    deltas = {"d1": (1, 60), "d2": (200, 30000), "d3": (70000, 8000000), "d4": (1 << 25, 1 << 30)}.get(style, (1, 3))
    if style == "all3":  # every group of four needs 3 bytes: 4-byte coding
        refs = np.cumsum(rng.integers(70000, 8000000, vc)) % (1 << 32)
    elif style in deltas or style in ("d1", "d2", "d3", "d4"):
        refs = np.cumsum(rng.integers(deltas[0], deltas[1], vc) * rng.choice([-1, 1], vc)) % (1 << 32)
    else:
        refs = rng.integers(0, 1 << 16 if rng.random() < 0.5 else 1 << 32, vc, dtype=np.uint64)
    return refs.astype(np.uint32), tris.astype(np.uint8)


def meshlet_cases(rng, n):
    fixed = [(0, 0, "random", False), (0, 0, "random", True), (1, 1, "random", False), (3, 1, "restart", True), (64, 96, "random", False), (64, 96, "chain", True),
             (64, 96, "restart", False), (64, 96, "restart", True), (40, 60, "chain", False), (17, 9, "d1", False), (17, 9, "d2", False), (17, 9, "d3", False),
             (17, 9, "d4", False), (16, 5, "all3", False), (12, 0, "d2", True), (0, 5, "random", False)]
    out = list(fixed)
    styles = ("random", "chain", "restart", "d1", "d2", "d3", "d4", "all3")
    while len(out) < n:
        out.append((int(rng.integers(0, 65)), int(rng.integers(0, 97)), styles[int(rng.integers(0, len(styles)))], bool(rng.random() < 0.5)))
    return out


@needs_ref
def test_meshlet_records_against_reference():
    ref = ref_lib()
    rng = np.random.default_rng(1200)
    meshlets, words = meshlet_inputs(rng, meshlet_cases(rng, 300))
    want = ref_meshlet_section(ref, meshlets, words)
    status, out = only({"meshlets": meshlets, "meshletdata": words}, True, emu())
    assert status == OK
    got = compressed_sections(out)[1]["meshletdata"]
    assert np.array_equal(got, want)


def index_cases(rng):
    yield "empty", np.zeros(0, np.uint32)
    for t in (1, 2, 17, 1000):
        i = np.arange(t, dtype=np.uint32)
        yield "strip%d" % t, np.stack([i, i + 1, i + 2], 1).reshape(-1)
        w = 17
        q = np.arange(t // 2 + 1, dtype=np.uint32)
        x, y = q % (w - 1), q // (w - 1)
        a, b, c, d = y * w + x, y * w + x + 1, (y + 1) * w + x, (y + 1) * w + x + 1
        yield "grid%d" % t, np.stack([a, b, c, c, b, d], 1).reshape(-1)[: t * 3].astype(np.uint32)
        yield "soup%d" % t, rng.integers(0, max(3, t), t * 3).astype(np.uint32)
        base = rng.integers(0, 1 << 31, t, dtype=np.int64)
        yield "jumps%d" % t, np.stack([base, base + rng.integers(-1, 2, t), base ^ 0x40000000], 1).reshape(-1).astype(np.uint32)
    # restarts: a second mesh starting at 0, 1, 2 after the counter moved
    i = np.arange(50, dtype=np.uint32)
    yield "restart", np.concatenate([np.stack([i, i + 1, i + 2], 1).reshape(-1), np.stack([i, i + 2, i + 1], 1).reshape(-1)])


@needs_ref
def test_index_streams_against_reference():
    ref = ref_lib()
    rng = np.random.default_rng(1300)
    cases = list(index_cases(rng))
    header, secs = raw_sections(raw_file("kitten"))
    cases.append(("kitten LOD chain", secs["indices"].view(np.uint32)))
    for label, idx in cases:
        got = written_stream((load_library(), None), "indices", idx)  # an index-only compressed write needs no context
        assert np.array_equal(got, ref_index_stream(ref, idx)), label



@needs_ref
def test_index_streams_fuzz_against_reference():
    """short random index buffers over few vertices: edge and vertex FIFO hits at every slot, restarts at 0, 1, 2 after the
    counter moved, and indices equal to the FIFOs' empty value ~0"""
    ref = ref_lib()
    rng = np.random.default_rng(1350)
    for case in range(3000):
        tris, kind = int(rng.integers(0, 50)), case % 4
        if kind == 0:
            idx = rng.integers(0, 8, 3 * tris)
        elif kind == 1:
            idx = rng.integers(0, 40, 3 * tris)
        elif kind == 2:  # restarts: meshes starting at 0, 1, 2 after others
            idx = np.concatenate([np.arange(6), [0, 1, 2], rng.integers(0, 10, 3 * tris), [0, 1, 2]])
        else:
            idx = rng.choice([0, 1, 2, 3, 5, 0xFFFFFFFE, 0xFFFFFFFF], 3 * tris)
        idx = np.ascontiguousarray(idx, np.uint32)
        got = written_stream((load_library(), None), "indices", idx)
        assert np.array_equal(got, ref_index_stream(ref, idx)), (case, idx.tolist())

def _guarded(a):
    """a copy of `a` whose last byte ends at an inaccessible page"""
    g = dev_tests._guarded_zeros(a.nbytes)
    g[:] = a.view(np.uint8).reshape(-1)
    return g


def test_rejections_leave_the_output_untouched():
    lib, ctx = emu()
    header, secs = raw_sections(raw_file("kitten"))
    md = secs["meshletdata"].view(np.uint32)
    m = secs["meshlets"].view(layout.MESHLET_DTYPE).copy()
    mask_md = 1 << SECTIONS.index("meshletdata")
    cases = []
    past = m.copy()
    past[-1]["dataOffset"] = len(md) - 1  # its words run past meshletdata
    cases.append(("range past meshletdata", {"meshlets": past}, mask_md, None, INVALID))
    for field, n in (("vertexCount", 65), ("triangleCount", 97)):
        big = m.copy()
        big[len(big) // 2][field] = n
        big[len(big) // 2]["dataOffset"] = 0
        cases.append((field + " above the limit", {"meshlets": big}, mask_md, None, INVALID))
    cases.append(("indices not a multiple of 3", {"indices": secs["indices"][:-4]}, 0, None, INVALID))
    cases.append(("meshletvtx0 not a multiple of 4", {"meshletvtx0": np.zeros(6, np.uint16)}, 0, None, INVALID))
    cases.append(("capacity below the bound", {}, 0, -1, INVALID))
    for label, edit, mask, cap_delta, want in cases:
        s2 = dict(secs)
        s2.update(edit)
        s2["meshletdata"] = _guarded(md)  # read by the kernels where it lies: a read past its end faults
        desc = make_desc(header, s2, True, device_mask=mask)
        bound = ctypes.c_size_t()
        assert lib.nvc_scene_cache_write_bound(ctypes.byref(desc), ctypes.byref(bound)) == OK
        cap = int(bound.value) + (cap_delta or 0)
        out = np.full(cap, 0xEE, np.uint8)
        size = ctypes.c_size_t(12345)
        c2 = ctypes.c_void_p()
        assert lib.nvc_create(0, None, ctypes.byref(c2)) == 0
        lib.emu_guard_allocations(1)
        try:
            status = lib.nvc_scene_cache_write(c2, None, ctypes.byref(desc), out.ctypes.data, cap, ctypes.byref(size))
        finally:
            lib.emu_guard_allocations(0)
            lib.nvc_destroy(c2)
            assert lib.emu_guarded_live() == 0
        assert status == want, (label, status)
        assert (out == 0xEE).all() and size.value == 12345, label
    # a device pointer, or compressed vertex / meshlet data, without a context
    for mask, compressed in ((1 << SECTIONS.index("draws"), False), (0, True)):
        desc = make_desc(header, secs, compressed, device_mask=mask)
        status, out = write(lib, None, desc)
        assert status == INVALID and (out == 0xEE).all()


def test_written_files_read_back():
    """what the writer makes parses, and every section reads back, on the host and into (emulated) device memory, to the
    bytes the reference's decoder gives for the reference's encoding"""
    lib, ctx = emu()
    host = load_library()
    for ref_file, raw in REFERENCE_FILES:
        header, secs = raw_sections(raw_file(raw))
        for compressed in (False, True):
            status, out = write(lib, ctx, make_desc(header, secs, compressed))
            assert status == OK
            info = layout.SceneCacheInfo()
            assert host.nvc_scene_cache_parse(out.ctypes.data, len(out), ctypes.byref(info)) == OK
            ref_data = np.fromfile(os.path.join(GOLDEN, ref_file), np.uint8) if compressed else raw_file(raw)
            ref_info = layout.SceneCacheInfo()
            assert host.nvc_scene_cache_parse(ref_data.ctypes.data, len(ref_data), ctypes.byref(ref_info)) == OK
            for s in range(len(SECTIONS)):
                hs, want = dev_tests._host_read(ref_data, ref_info, s)
                assert hs == OK
                hs, got = dev_tests._host_read(out, info, s)
                assert hs == OK and np.array_equal(got, want), (ref_file, compressed, SECTIONS[s])
                n = int(info.sections[s].decoded_bytes)
                dev = np.full(n, 0xEE, np.uint8)
                assert lib.nvc_scene_cache_read_device(ctx, None, out.ctypes.data, len(out), ctypes.byref(info), s, dev.ctypes.data if n else None, n) == OK
                assert np.array_equal(dev, want), (ref_file, compressed, SECTIONS[s])


def test_texture_paths_are_normalised():
    lib, ctx = emu()
    rec = np.zeros((3, 256), np.uint8)
    rec[0, :5] = np.frombuffer(b"a.png", np.uint8)
    rec[0, 6:9] = 7  # bytes after the first NUL
    rec[1, :] = ord("x")  # no NUL: byte 255 becomes 0
    rec[2, 0] = 0
    rec[2, 1:] = 9
    status, out = only({"texture_paths": rec.reshape(-1)}, False, (lib, None))
    assert status == OK
    got = compressed_sections(out)[1]["texture_paths"].reshape(3, 256)
    want = np.zeros((3, 256), np.uint8)
    want[0, :5] = rec[0, :5]
    want[1, :255] = ord("x")
    assert np.array_equal(got, want)


# ---- GPU tier ---------------------------------------------------------------------------------------------------------
def _torch_sections(secs, on_gpu):
    import torch

    return {k: (torch.from_numpy(v.copy()).cuda() if on_gpu and k in on_gpu else v) for k, v in secs.items()}


def _write_py(header, secs, compressed, **kw):
    from niagara_b200.scene_cache import write_scene_cache

    return np.frombuffer(write_scene_cache(secs, compressed=compressed, hash_meta=header.hashMeta, clrt_mode=header.clrtMode, omm_states=header.ommStates,
                                           camera=header.camera, sun_direction=list(header.sunDirection), **kw), np.uint8)


GEOMETRY = ("vertices", "indices", "meshlets", "meshletdata", "meshletvtx0")


@pytest.mark.gpu
@pytest.mark.parametrize("ref_file,raw", REFERENCE_FILES)
def test_gpu_reference_files(ref_file, raw):
    want = np.fromfile(os.path.join(GOLDEN, ref_file), np.uint8)
    header, secs = raw_sections(raw_file(raw))
    header.clrtMode = want[24]
    for on_gpu in (GEOMETRY, tuple(SECTIONS), ()):
        got = _write_py(header, _torch_sections(secs, on_gpu), True)
        assert np.array_equal(got, want), (ref_file, on_gpu)
    assert np.array_equal(_write_py(header, _torch_sections(secs, GEOMETRY), False), raw_file(raw))


@pytest.mark.gpu
@needs_ref
def test_gpu_codecs_against_reference():
    ref = ref_lib()
    rng = np.random.default_rng(1400)
    import torch

    for stride in (16, 8):
        name = "vertices" if stride == 16 else "meshletvtx0"
        for count in VERTEX_COUNTS + (100 * 256 + 3, 2000 * 256 + 255):
            for kind in ("random", "smooth16", "floats", "sparse", "channel1", "tie"):
                values = vertex_values(rng, count, stride, kind)
                out = _write_py(layout.SceneCacheHeader(), {name: torch.from_numpy(values.reshape(-1).copy()).cuda()}, True)
                assert np.array_equal(compressed_sections(out)[1][name], dev_tests.encode_vertices(ref, values, 2, 1)), (stride, count, kind)
    meshlets, words = meshlet_inputs(rng, meshlet_cases(rng, 20000))
    out = _write_py(layout.SceneCacheHeader(), {"meshlets": torch.from_numpy(meshlets.view(np.uint8).copy()).cuda(), "meshletdata": torch.from_numpy(words.view(np.uint8).copy()).cuda()}, True)
    assert np.array_equal(compressed_sections(out)[1]["meshletdata"], ref_meshlet_section(ref, meshlets, words))
    big = 1_000_000  # triangles
    w = 1001
    q = np.arange(big // 2, dtype=np.int64)
    x, y = q % (w - 1), q // (w - 1)
    grid = np.stack([y * w + x, y * w + x + 1, (y + 1) * w + x, (y + 1) * w + x, y * w + x + 1, (y + 1) * w + x + 1], 1).reshape(-1).astype(np.uint32)
    large = [("soup 10^6", rng.integers(0, 1 << 20, 3 * big).astype(np.uint32)), ("grid 10^6", grid)]
    for label, idx in list(index_cases(rng)) + large:
        out = _write_py(layout.SceneCacheHeader(), {"indices": torch.from_numpy(idx.copy()).cuda()}, True)
        assert np.array_equal(compressed_sections(out)[1]["indices"], ref_index_stream(ref, idx)), label


def _cook(lib, ctx, secs, clrt, max_scale=None):
    """Meshlet[], meshletdata (and meshletvtx0) cooked on the device from the raw fixture's Vertex[], LOD indices and Mesh[]"""
    import torch

    meshes = secs["meshes"].view(layout.MESH_DTYPE).copy()
    vb = torch.from_numpy(secs["vertices"].copy()).cuda()
    ib = torch.from_numpy(secs["indices"].copy()).cuda()
    dmeshes = torch.zeros(meshes.nbytes, dtype=torch.uint8, device="cuda")
    nm = ctypes.c_uint32()
    nw = ctypes.c_uint64()
    nv = ctypes.c_uint64()
    mp = meshes.ctypes.data
    if clrt:
        assert lib.nvc_cook_meshlets_clrt_capacity(mp, max_scale.ctypes.data, len(meshes), ctypes.byref(nm), ctypes.byref(nw), ctypes.byref(nv)) == OK
    else:
        assert lib.nvc_cook_meshlets_capacity(mp, len(meshes), ctypes.byref(nm), ctypes.byref(nw)) == OK
    ml = torch.zeros(nm.value * 24, dtype=torch.uint8, device="cuda")
    md = torch.zeros(nw.value, dtype=torch.int32, device="cuda")
    vtx0 = torch.zeros(max(int(nv.value), 1), dtype=torch.int16, device="cuda")
    totals = torch.zeros(8, dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    if clrt:
        st = lib.nvc_cook_meshlets_clrt(ctx, s, vb.data_ptr(), len(secs["vertices"]) // 16, ib.data_ptr(), len(secs["indices"]) // 4, mp, max_scale.ctypes.data, dmeshes.data_ptr(), len(meshes),
                                        ml.data_ptr(), nm.value, md.data_ptr(), nw.value, vtx0.data_ptr(), int(nv.value), totals.data_ptr())
    else:
        st = lib.nvc_cook_meshlets(ctx, s, vb.data_ptr(), len(secs["vertices"]) // 16, ib.data_ptr(), len(secs["indices"]) // 4, mp, dmeshes.data_ptr(), len(meshes),
                                   ml.data_ptr(), nm.value, md.data_ptr(), nw.value, totals.data_ptr())
    assert st == OK
    t = totals.cpu().numpy().view(np.uint32)
    assert t[3] == 0
    out = {"meshes": dmeshes, "meshlets": ml[: int(t[0]) * 24], "meshletdata": md[: int(t[1])], "vertices": vb, "indices": ib}
    if clrt:
        out["meshletvtx0"] = vtx0[: int(t[4])]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("ref_file,raw,clrt", [("kitten.z.cache", "kitten", False), ("animated_clrt.z.cache", "animated_clrt", True)])
def test_gpu_end_to_end_cook_then_write(ref_file, raw, clrt):
    """the cooker's inputs (Vertex[], LOD index buffers, Mesh[] LOD ranges) from the raw fixture, meshlets cooked on the
    device, the cache written from device memory: the reference's file"""
    import torch

    from niagara_b200.scene_cache import _write_context

    lib = load_library()
    want = np.fromfile(os.path.join(GOLDEN, ref_file), np.uint8)
    header, secs = raw_sections(raw_file(raw))
    header.clrtMode = int(clrt)
    ctx = _write_context(lib, torch.cuda.current_device())
    max_scale = None
    if clrt:
        with np.load(os.path.join(GOLDEN, "meshlet_cook_clrt.npz")) as z:
            max_scale = np.ascontiguousarray(z["animated_max_scale"], np.float32)
    cooked = _cook(lib, ctx, secs, clrt, max_scale)
    s2 = dict(secs)
    s2.update(cooked)
    got = _write_py(header, s2, True)
    assert np.array_equal(got, want)


@pytest.mark.gpu
@needs_ref
def test_gpu_large_write_on_a_busy_non_blocking_stream():
    import sys

    import torch

    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import scene_cache_write_bench as bench

    secs = bench.geometry(copies=1000, seed=11)
    want, _ = bench.reference_file(secs)
    side = torch.cuda.Stream()
    gpu = _torch_sections(secs, GEOMETRY)
    with torch.cuda.stream(side):
        torch.cuda._sleep(1_000_000)  # work already queued on the stream the write is issued on
        got = np.frombuffer(bench.write(gpu), np.uint8)
    assert np.array_equal(got, want)
