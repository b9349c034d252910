"""nvc_scene_cache_read_device: every section of a scene cache read into device memory equals nvc_scene_cache_read's bytes and
status.  The CPU tier runs the product's kernels under the SIMT emulation (tests/emu_lib.py), some reads with allocations that
end at an inaccessible page; the GPU tier reads the same caches
through SceneCache.section_device.  Synthetic caches are built here from streams of the reference's encoders
(oracle/_ref/libmeshopt_ref.so) and skip where that library was not built."""
import ctypes
import mmap
import os

import numpy as np
import pytest

import emu_lib
from niagara_b200 import layout
from niagara_b200.lib import load_library

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libmeshopt_ref.so")
CACHES = ["kitten.z.cache", "pirateglb.z.cache", "animated.z.cache", "animated_clrt.z.cache", "animated.raw.cache"]
SECTIONS = layout.CACHE_SECTIONS
OK, INVALID, UNSUPPORTED, CORRUPT = 0, -1, -6, -7
vp, sz = ctypes.c_void_p, ctypes.c_size_t

needs_ref = pytest.mark.skipif(not os.path.exists(REF_SO), reason="needs the reference's codecs (oracle/_ref/libmeshopt_ref.so)")


# ---- the emulated library and a context of it -----------------------------------------------------------------------------
_CTX = []


def _emu():
    lib = emu_lib.load()
    if not _CTX:
        ctx = ctypes.c_void_p()
        assert lib.nvc_create(0, None, ctypes.byref(ctx)) == 0
        _CTX.append(ctx)
    return lib, _CTX[0]


_KEEP = []


def _guarded_zeros(n):
    """n bytes that end at an inaccessible page: exactly, or up to 3 bytes before it to keep dst 4-byte aligned"""
    page = mmap.PAGESIZE
    n1 = max(n, 1)
    span = (n1 + page - 1) // page * page
    m = mmap.mmap(-1, span + page, flags=mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS, prot=mmap.PROT_READ | mmap.PROT_WRITE)
    libc = ctypes.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
    base = ctypes.addressof(ctypes.c_char.from_buffer(m))
    assert libc.mprotect(base + span, page, 0) == 0, ctypes.get_errno()
    _KEEP.append(m)
    return np.frombuffer(m, dtype=np.uint8, count=n, offset=(span - n) & ~3)


def _parse(data):
    info = layout.SceneCacheInfo()
    return load_library().nvc_scene_cache_parse(data.ctypes.data, len(data), ctypes.byref(info)), info


def _host_read(data, info, s):
    out = np.zeros(int(info.sections[s].decoded_bytes), np.uint8)
    status = load_library().nvc_scene_cache_read(data.ctypes.data, len(data), ctypes.byref(info), s, out.ctypes.data if out.size else None, out.size)
    return status, out


def _device_read(data, info, s, guard=False, fill=0xEE):
    """Guarded: a fresh context, so that its scratch is allocated for this read alone and ends where the staged stream's
    last word does, against an inaccessible page, as `dst` does; a read or write past either faults."""
    lib, ctx = _emu()
    n = int(info.sections[s].decoded_bytes)
    out = _guarded_zeros(n) if guard else np.zeros(n, np.uint8)
    out[:] = fill
    if guard:
        ctx = ctypes.c_void_p()
        assert lib.nvc_create(0, None, ctypes.byref(ctx)) == 0
        lib.emu_guard_allocations(1)
    try:
        status = lib.nvc_scene_cache_read_device(ctx, None, data.ctypes.data, len(data), ctypes.byref(info), s, out.ctypes.data if n else None, n)
    finally:
        if guard:
            lib.emu_guard_allocations(0)
            lib.nvc_destroy(ctx)
            assert lib.emu_guarded_live() == 0
    return status, np.array(out)


def _check_file(data, sections=range(len(SECTIONS)), guard=False, what=""):
    status, info = _parse(data)
    assert status == OK, what
    for s in sections:
        hs, host = _host_read(data, info, s)
        ds, dev = _device_read(data, info, s, guard)
        assert ds == hs, (what, SECTIONS[s], ds, hs)
        if hs == OK:
            assert np.array_equal(dev, host), (what, SECTIONS[s], int(np.flatnonzero(dev != host)[0]))


# ---- synthetic caches ------------------------------------------------------------------------------------------------------
def _ref():
    lib = ctypes.CDLL(REF_SO)
    lib.meshopt_encodeVertexBufferBound.restype = sz
    lib.meshopt_encodeVertexBufferBound.argtypes = [sz, sz]
    lib.meshopt_encodeVertexBufferLevel.restype = sz
    lib.meshopt_encodeVertexBufferLevel.argtypes = [vp, sz, vp, sz, sz, ctypes.c_int, ctypes.c_int]
    lib.meshopt_encodeMeshletBound.restype = sz
    lib.meshopt_encodeMeshletBound.argtypes = [sz, sz]
    lib.meshopt_encodeMeshlet.restype = sz
    lib.meshopt_encodeMeshlet.argtypes = [vp, sz, vp, sz, vp, sz]
    return lib


def encode_vertices(ref, data, level, version):
    data = np.ascontiguousarray(data)
    count, stride = data.shape
    buf = np.zeros(ref.meshopt_encodeVertexBufferBound(count, stride), np.uint8)
    n = ref.meshopt_encodeVertexBufferLevel(buf.ctypes.data, len(buf), data.ctypes.data, count, stride, level, version)
    assert n > 0
    return buf[:n].copy()


def encode_meshlet(ref, refs, tris):
    refs, tris = np.ascontiguousarray(refs, np.uint32), np.ascontiguousarray(tris, np.uint8)
    buf = np.zeros(ref.meshopt_encodeMeshletBound(256, 256), np.uint8)
    n = ref.meshopt_encodeMeshlet(buf.ctypes.data, len(buf), refs.ctypes.data, len(refs), tris.ctypes.data, len(tris) // 3 if tris.ndim == 1 else len(tris))
    assert n > 0 and n < 65536
    return buf[:n].copy()


def make_cache(vertices=None, vtx0=None, meshlets=None, blocks=None, meshletdata_count=0, vertex_count=0, vtx0_count=0):
    """A compressed cache with the given streams: `vertices` (vertex codec, stride 16, vertex_count vertices), `vtx0`
    (vertex codec, stride 8, vtx0_count uint16), `meshlets` (Meshlet records) with `blocks` (one meshlet codec block each)."""
    h = layout.SceneCacheHeader()
    h.magic, h.version, h.compressed = 0x434E4353, 7, 1
    vertices = np.zeros(0, np.uint8) if vertices is None else vertices
    vtx0 = np.zeros(0, np.uint8) if vtx0 is None else vtx0
    meshlets = np.zeros(0, layout.MESHLET_DTYPE) if meshlets is None else meshlets
    chain = b"".join(np.uint16(len(b)).tobytes() + b.tobytes() for b in (blocks or []))
    h.vertexCount, h.compressedVertexBytes = vertex_count, len(vertices)
    h.meshletCount, h.meshletdataCount, h.compressedMeshletDataBytes = len(meshlets), meshletdata_count, len(chain)
    h.meshletvtx0Count, h.compressedMeshletVtx0Bytes = vtx0_count, len(vtx0)
    body = bytes(h) + vertices.tobytes() + meshlets.tobytes() + chain + vtx0.tobytes()
    return np.frombuffer(body, np.uint8).copy()


def vertex_data(rng, count, stride, kind):
    if count == 0:
        return np.zeros((0, stride), np.uint8)
    if kind == "random":
        return rng.integers(0, 256, (count, stride), dtype=np.uint8)
    if kind == "zeros":
        return np.zeros((count, stride), np.uint8)
    if kind == "smooth16":
        base = np.cumsum(rng.integers(-40, 41, (count, stride // 2)), axis=0).astype(np.int64) + 30000
        return (base & 0xFFFF).astype("<u2").view(np.uint8).reshape(count, stride)
    if kind == "floats":
        f = (rng.standard_normal((count, stride // 4)) * 0.01 + np.linspace(1, 2, stride // 4)).astype("<f4")
        return f.view(np.uint8).reshape(count, stride)
    if kind == "sparse":
        d = np.full((count, stride), 7, np.uint8)
        idx = rng.integers(0, count, max(1, count // 9))
        d[idx, rng.integers(0, stride, len(idx))] = rng.integers(0, 256, len(idx))
        return np.cumsum(d, axis=0).astype(np.uint8)
    raise ValueError(kind)


def vertex_cache(ref, rng, count, stride, kind, version, level):
    data = vertex_data(rng, count, stride, kind)
    stream = encode_vertices(ref, data, level, version)
    if stride == 16:
        return make_cache(vertices=stream, vertex_count=count), data
    return make_cache(vtx0=stream, vtx0_count=4 * count), data


def meshlet_case(rng, vc, tc, style):
    if style == 0:  # arbitrary references, arbitrary triangles
        refs = rng.integers(0, 1 << 32, vc, dtype=np.uint64).astype(np.uint32)
        tris = rng.integers(0, max(vc, 1), (tc, 3)).astype(np.uint8)
    elif style == 1:  # ascending references with small gaps, strip-like triangles
        refs = (np.cumsum(rng.integers(1, 4, vc)) + 1000).astype(np.uint32)
        i = np.arange(tc) % max(1, vc - 2)
        tris = np.stack([i, i + 1, i + 2], 1).astype(np.uint8)
    elif style == 2:  # 16-bit references, fans
        refs = rng.integers(0, 1 << 16, vc).astype(np.uint32)
        i = 1 + np.arange(tc) % max(1, vc - 2)
        tris = np.stack([np.zeros(tc, np.int64), i, i + 1], 1).astype(np.uint8)
    else:  # large deltas: 3- and 4-byte groups
        refs = (rng.integers(0, 1 << 24, vc) * rng.integers(1, 200, vc)).astype(np.uint32)
        tris = rng.integers(0, max(vc, 1), (tc, 3)).astype(np.uint8)
    return refs, tris


def meshlet_cache(ref, rng, count, big=False, empty_every=0, gaps=False):
    """A cache of `count` meshlets of the four styles (up to 255 / 255 when `big`), shortRefs both ways where the
    references fit 16 bits, every `empty_every`-th meshlet empty, word gaps between meshlets when `gaps`"""
    meshlets = np.zeros(count, layout.MESHLET_DTYPE)
    blocks = []
    at = 0
    for i in range(count):
        if empty_every and i % empty_every == 0:
            vc = tc = 0
        elif big and rng.random() < 0.5:
            vc, tc = int(rng.integers(1, 256)), int(rng.integers(1, 256))
        else:
            vc, tc = int(rng.integers(3, 65)), int(rng.integers(1, 97))
        refs, tris = meshlet_case(rng, vc, tc, int(rng.integers(0, 4)))
        short = bool(vc and int(refs.max()) < (1 << 16) and rng.random() < 0.7)
        blocks.append(encode_meshlet(ref, refs, tris))
        at += int(rng.integers(0, 3)) if gaps else 0
        meshlets[i]["dataOffset"] = at
        meshlets[i]["vertexCount"], meshlets[i]["triangleCount"], meshlets[i]["shortRefs"] = vc, tc, int(short)
        at += ((vc + 1) // 2 if short else vc) + (3 * tc + 3) // 4
    return make_cache(meshlets=meshlets, blocks=blocks, meshletdata_count=at + (2 if gaps else 0))


# ---- CPU tier -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CACHES)
def test_reference_written_caches(name):
    data = np.fromfile(os.path.join(GOLDEN, name), np.uint8)
    _check_file(data, what=name)


@needs_ref
@pytest.mark.parametrize("stride", [16, 8])
def test_synthetic_vertex_streams(stride):
    ref = _ref()
    rng = np.random.default_rng(400 + stride)
    s = SECTIONS.index("vertices" if stride == 16 else "meshletvtx0")
    cases = 0
    for count in (0, 1, 15, 16, 17, 255, 256, 257, 1000, 3000, 40 * 256 + 77):
        for kind in ("random", "zeros", "smooth16", "floats", "sparse"):
            for version, level in ((0, 2), (1, 0), (1, 1), (1, 2), (1, 3)):
                if count > 3000 and (kind, level) not in (("random", 2), ("smooth16", 3), ("floats", 1), ("sparse", 2)):
                    continue  # the many-block count: a selection keeps the emulated run short
                data, values = vertex_cache(ref, rng, count, stride, kind, version, level)
                status, info = _parse(data)
                assert status == OK
                ds, dev = _device_read(data, info, s)
                assert ds == OK, (count, kind, version, level)
                assert np.array_equal(dev, values.reshape(-1)), (count, kind, version, level)
                cases += 1
    assert cases >= 220


@needs_ref
def test_vertex_stream_longer_than_one_carry_pass():
    """more blocks than the carry kernel's CTA has threads (1024): the scan carries its running total between passes"""
    ref = _ref()
    rng = np.random.default_rng(450)
    for stride, kind, version, level in ((8, "sparse", 1, 2), (16, "smooth16", 0, 2)):
        count = 1030 * 256 + 77
        data, values = vertex_cache(ref, rng, count, stride, kind, version, level)
        status, info = _parse(data)
        assert status == OK
        ds, dev = _device_read(data, info, SECTIONS.index("vertices" if stride == 16 else "meshletvtx0"))
        assert ds == OK and np.array_equal(dev, values.reshape(-1)), (stride, kind)


@needs_ref
@pytest.mark.parametrize("count", [1, 31, 32, 33, 1000])
def test_synthetic_meshlet_streams(count):
    ref = _ref()
    rng = np.random.default_rng(500 + count)
    s = SECTIONS.index("meshletdata")
    for big, empty_every, gaps in ((False, 0, False), (True, 7, True)):
        data = meshlet_cache(ref, rng, count, big, empty_every, gaps)
        status, info = _parse(data)
        assert status == OK
        hs, host = _host_read(data, info, s)
        ds, dev = _device_read(data, info, s)
        assert hs == OK and ds == OK
        assert np.array_equal(dev, host), (count, big, int(np.flatnonzero(dev != host)[0]))


def hostile_files(seed, per_section=6):
    """Variants of reference-written caches: bytes flipped in each compressed section, meshlet blocks truncated with the size
    chain kept consistent, and edited counts.  Yields (label, bytes)."""
    rng = np.random.default_rng(seed)
    for name in ("kitten.z.cache", "animated.z.cache", "animated_clrt.z.cache"):
        base = np.fromfile(os.path.join(GOLDEN, name), np.uint8)
        _, info = _parse(base)
        for s in ("vertices", "meshletdata", "meshletvtx0"):
            sec = info.sections[SECTIONS.index(s)]
            if not sec.stored_bytes:
                continue
            for k in range(per_section):
                d = base.copy()
                pos = int(sec.offset) + int(rng.integers(0, int(sec.stored_bytes)))
                d[pos] ^= np.uint8(1 << int(rng.integers(0, 8))) if k % 2 else np.uint8(rng.integers(1, 256))
                yield "%s %s flip@%d" % (name, s, pos), d
        md = info.sections[SECTIONS.index("meshletdata")]
        chain = base[int(md.offset) : int(md.offset + md.stored_bytes)]
        starts, at = [], 0
        while at < len(chain):
            starts.append(at)
            at += 2 + int(chain[at : at + 2].view(np.uint16)[0])
        for k in range(per_section):
            i = int(rng.integers(0, len(starts)))
            at = starts[i]
            n = int(chain[at : at + 2].view(np.uint16)[0])
            cut = int(rng.integers(1, min(n, 8) + 1))
            drop = at + 2 + int(rng.integers(0, n - cut + 1))  # bytes [drop, drop + cut) of the block go
            c = np.concatenate([chain[:drop], chain[drop + cut :]])
            c[at : at + 2] = np.frombuffer(np.uint16(n - cut).tobytes(), np.uint8)
            h = layout.SceneCacheHeader.from_buffer_copy(base[: ctypes.sizeof(layout.SceneCacheHeader)].tobytes())
            h.compressedMeshletDataBytes -= cut
            d = np.concatenate([np.frombuffer(bytes(h), np.uint8), base[ctypes.sizeof(h) : int(md.offset)], c, base[int(md.offset + md.stored_bytes) :]])
            yield "%s meshlet %d truncated by %d" % (name, i, cut), d
        ms = info.sections[SECTIONS.index("meshlets")]
        for k in range(per_section):
            d = base.copy()
            h = layout.SceneCacheHeader.from_buffer_copy(d[: ctypes.sizeof(layout.SceneCacheHeader)].tobytes())
            if k % 3 == 0:
                h.vertexCount = max(0, h.vertexCount + int(rng.integers(-300, 300)))
                d[: ctypes.sizeof(h)] = np.frombuffer(bytes(h), np.uint8)
                yield "%s vertexCount %d" % (name, h.vertexCount), d
            elif k % 3 == 1 and h.meshletvtx0Count:
                h.meshletvtx0Count = max(0, h.meshletvtx0Count + int(rng.integers(-9, 9)))
                d[: ctypes.sizeof(h)] = np.frombuffer(bytes(h), np.uint8)
                yield "%s meshletvtx0Count %d" % (name, h.meshletvtx0Count), d
            else:
                i = int(rng.integers(0, h.meshletCount))
                rec = int(ms.offset) + 24 * i
                field = 20 + int(rng.integers(0, 2))  # vertexCount or triangleCount
                d[rec + field] = max(0, int(d[rec + field]) - int(rng.integers(1, 4)))
                yield "%s meshlet %d count byte %d" % (name, i, field), d


def _ordered(data, info):
    m = np.frombuffer(data[int(info.sections[2].offset) :][: 24 * info.header.meshletCount].tobytes(), layout.MESHLET_DTYPE)
    refw = np.where(m["shortRefs"] != 0, (m["vertexCount"].astype(np.int64) + 1) // 2, m["vertexCount"])
    end = m["dataOffset"].astype(np.int64) + refw + (m["triangleCount"].astype(np.int64) * 3 + 3) // 4
    return bool(np.all(m["dataOffset"][1:] >= end[:-1]))


def _check_hostile(label, d, guard, sections=("vertices", "meshletdata", "meshletvtx0")):
    status, info = _parse(d)
    if status != OK:
        return None
    outcomes = []
    for name in sections:
        s = SECTIONS.index(name)
        hs, host = _host_read(d, info, s)
        ds, dev = _device_read(d, info, s, guard)
        want = UNSUPPORTED if name == "meshletdata" and not _ordered(d, info) else hs
        assert ds == want, (label, name, ds, hs)
        if hs == OK and ds == OK:
            assert np.array_equal(dev, host), (label, name)
        outcomes.append(ds)
    return outcomes


def test_hostile_files_in_the_guarded_build():
    outcomes = []
    for label, d in hostile_files(600):
        o = _check_hostile(label, d, guard=True)
        if o:
            outcomes += o
    assert CORRUPT in outcomes and OK in outcomes and len(outcomes) > 60


@needs_ref
def test_out_of_order_and_overlapping_meshlets_are_refused():
    ref = _ref()
    rng = np.random.default_rng(700)
    s = SECTIONS.index("meshletdata")
    data = meshlet_cache(ref, rng, 40)
    hsize = ctypes.sizeof(layout.SceneCacheHeader)
    m = data[hsize : hsize + 24 * 40].view(layout.MESHLET_DTYPE)
    for edit in ("overlap", "reverse"):
        d = data.copy()
        mm = d[hsize : hsize + 24 * 40].view(layout.MESHLET_DTYPE)
        if edit == "overlap":
            mm[5]["dataOffset"] = m[4]["dataOffset"] + 1
        else:
            mm[3]["dataOffset"], mm[4]["dataOffset"] = m[4]["dataOffset"], m[3]["dataOffset"]
        status, info = _parse(d)
        assert status == OK
        ds, dev = _device_read(d, info, s, fill=0xEE)
        assert ds == UNSUPPORTED, edit
        assert (dev == 0xEE).all()  # nothing was written
        assert _host_read(d, info, s)[0] in (OK, CORRUPT)  # the host decoder still reads it


def test_bad_arguments_are_rejected():
    lib, ctx = _emu()
    data = np.fromfile(os.path.join(GOLDEN, "animated.z.cache"), np.uint8)
    status, info = _parse(data)
    assert status == OK
    s = SECTIONS.index("vertices")
    n = int(info.sections[s].decoded_bytes)
    out = np.zeros(n + 8, np.uint8)
    p, f = out.ctypes.data, data.ctypes.data
    call = lib.nvc_scene_cache_read_device
    assert call(None, None, f, len(data), ctypes.byref(info), s, p, n) == INVALID
    assert call(ctx, None, None, len(data), ctypes.byref(info), s, p, n) == INVALID
    assert call(ctx, None, f, len(data), None, s, p, n) == INVALID
    assert call(ctx, None, f, len(data), ctypes.byref(info), s, None, n) == INVALID
    assert call(ctx, None, f, len(data), ctypes.byref(info), s, p, n - 1) == INVALID
    assert call(ctx, None, f, len(data), ctypes.byref(info), -1, p, n) == INVALID
    assert call(ctx, None, f, len(data), ctypes.byref(info), len(SECTIONS), p, n) == INVALID
    assert call(ctx, None, f, len(data), ctypes.byref(info), s, p + 1, n) == INVALID  # dst must be 4-byte aligned
    # an info that does not fit the file: a shorter file, or meshlet records the info places past its end
    assert call(ctx, None, f, int(info.sections[s].offset + info.sections[s].stored_bytes) - 1, ctypes.byref(info), s, p, n) == INVALID
    md = SECTIONS.index("meshletdata")
    forged = layout.SceneCacheInfo.from_buffer_copy(info)
    forged.header.meshletCount += 1
    assert call(ctx, None, f, len(data), ctypes.byref(forged), md, p, len(out)) == INVALID
    assert call(ctx, None, f, len(data), ctypes.byref(info), s, p, n) == OK


# ---- GPU tier -------------------------------------------------------------------------------------------------------------
def _gpu_read(data, s, tmp_path, label):
    """(host status, host bytes, device status, device bytes) through SceneCache over a file holding `data`"""
    from niagara_b200.lib import NvcError
    from niagara_b200.scene_cache import SceneCache

    path = os.path.join(str(tmp_path), "case.cache")
    data.tofile(path)
    c = SceneCache(path)
    try:
        hs, host = _host_read(data, c.info, s)
        try:
            dev, ds = c.section_device(SECTIONS[s]).cpu().numpy(), OK
        except NvcError as e:
            dev, ds = None, next(code for code, word in ((CORRUPT, "corrupt"), (UNSUPPORTED, "unsupported"), (INVALID, "invalid")) if word in str(e).lower())
        return hs, host, ds, dev
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", CACHES)
def test_gpu_reference_written_caches(name, tmp_path):
    data = np.fromfile(os.path.join(GOLDEN, name), np.uint8)
    for s in range(len(SECTIONS)):
        hs, host, ds, dev = _gpu_read(data, s, tmp_path, name)
        assert hs == OK and ds == OK, (name, SECTIONS[s], hs, ds)
        assert np.array_equal(dev, host), (name, SECTIONS[s])


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("stride", [16, 8])
def test_gpu_synthetic_vertex_streams(stride, tmp_path):
    ref = _ref()
    rng = np.random.default_rng(800 + stride)
    s = SECTIONS.index("vertices" if stride == 16 else "meshletvtx0")
    for count in (0, 1, 15, 16, 17, 255, 256, 257, 1000, 3000, 60 * 256 + 77):
        for kind in ("random", "zeros", "smooth16", "floats", "sparse"):
            for version, level in ((0, 2), (1, 0), (1, 1), (1, 2), (1, 3)):
                data, values = vertex_cache(ref, rng, count, stride, kind, version, level)
                hs, host, ds, dev = _gpu_read(data, s, tmp_path, "")
                assert hs == OK and ds == OK and np.array_equal(dev, values.reshape(-1)), (count, kind, version, level)


@pytest.mark.gpu
@needs_ref
def test_gpu_synthetic_meshlet_streams(tmp_path):
    ref = _ref()
    rng = np.random.default_rng(900)
    s = SECTIONS.index("meshletdata")
    for count in (1, 31, 32, 33, 1000):
        for big, empty_every, gaps in ((False, 0, False), (True, 7, True)):
            data = meshlet_cache(ref, rng, count, big, empty_every, gaps)
            hs, host, ds, dev = _gpu_read(data, s, tmp_path, "")
            assert hs == OK and ds == OK and np.array_equal(dev, host), (count, big)


@pytest.mark.gpu
def test_gpu_hostile_files(tmp_path):
    """a few of the hostile files the guarded emulated build reads (test_hostile_files_in_the_guarded_build)"""
    seen = 0
    for label, d in hostile_files(600, per_section=2):
        status, info = _parse(d)
        if status != OK:
            continue
        for name in ("vertices", "meshletdata", "meshletvtx0"):
            s = SECTIONS.index(name)
            hs, host, ds, dev = _gpu_read(d, s, tmp_path, label)
            want = UNSUPPORTED if name == "meshletdata" and not _ordered(d, info) else hs
            assert ds == want, (label, name, ds, hs)
            if hs == OK:
                assert np.array_equal(dev, host), (label, name)
            seen += 1
    assert seen > 20


@pytest.mark.gpu
@needs_ref
def test_gpu_read_on_a_non_blocking_stream(tmp_path):
    """On a stream that is not ordered with the legacy default stream (torch's side streams are created non-blocking),
    the call's uploads have landed before its kernels read them, and its result is in place when it returns."""
    import sys

    import torch

    from niagara_b200.scene_cache import SceneCache

    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import scene_cache_device_bench as bench

    path = os.path.join(str(tmp_path), "large.cache")
    bench.generate(copies=40, seed=5).tofile(path)  # its compressed sections: vertices and meshlet data
    side = torch.cuda.Stream()
    for cache, names in ((path, ("vertices", "meshletdata", "meshlets")), (os.path.join(GOLDEN, "kitten.z.cache"), SECTIONS)):
        c = SceneCache(cache)
        try:
            for name in names:
                s = SECTIONS.index(name)
                host = _host_read(np.fromfile(cache, np.uint8), c.info, s)[1]
                with torch.cuda.stream(side):
                    for _ in range(3):
                        # work already queued on the side stream must finish before the call's copies
                        torch.cuda._sleep(1_000_000)
                        got = c.section_device(name).cpu().numpy()  # a copy on the side stream, after the call returned
                        assert np.array_equal(got, host), (cache, name)
        finally:
            c.close()


@pytest.mark.gpu
@needs_ref
def test_gpu_large_generated_cache(tmp_path):
    import sys

    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import scene_cache_device_bench as bench

    data = bench.generate(copies=40, seed=3)
    for name in ("vertices", "meshletdata"):
        hs, host, ds, dev = _gpu_read(data, SECTIONS.index(name), tmp_path, name)
        assert hs == OK and ds == OK and np.array_equal(dev, host), name
