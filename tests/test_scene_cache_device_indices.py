"""nvc_scene_cache_read_device on INDICES: the index codec decoded by kernels (a symbolic pass per chunk, a scan of the
chunks' state substitutions, a concrete pass per chunk) equals nvc_scene_cache_read byte for byte, with the same status,
and writes nothing to `dst` when the stream is refused.  The CPU tier runs the kernels under the SIMT emulation
(tests/emu_lib.py); the GPU tier reads through SceneCache.section_device.  Streams come from the reference's encoder
(oracle/_ref/libmeshopt_ref.so; those cases skip where it was not built) and from a generator here that writes any code
the format allows, so that chunk boundaries land on resets, deep lookups and never-written slots."""
import ctypes
import os

import numpy as np
import pytest

from niagara_b200 import layout
from test_scene_cache_device import CORRUPT, GOLDEN, INVALID, OK, REF_SO, ROOT, SECTIONS, UNSUPPORTED, _device_read, _gpu_read, _host_read, _parse, needs_ref

IDX = SECTIONS.index("indices")
CHUNK, RUN = 256, 256  # kIndexChunk, kIndexRun (nvc_internal.h)
vp, sz = ctypes.c_void_p, ctypes.c_size_t


def index_cache(stream, index_count):
    """a compressed cache whose only section is INDICES holding `stream`"""
    h = layout.SceneCacheHeader()
    h.magic, h.version, h.compressed = 0x434E4353, 7, 1
    stream = np.asarray(stream, np.uint8)
    h.indexCount, h.compressedIndexBytes = index_count, len(stream)
    return np.frombuffer(bytes(h) + stream.tobytes(), np.uint8).copy()


def _ref():
    lib = ctypes.CDLL(REF_SO)
    lib.meshopt_encodeIndexVersion.argtypes = [ctypes.c_int]
    lib.meshopt_encodeIndexBufferBound.restype = sz
    lib.meshopt_encodeIndexBufferBound.argtypes = [sz, sz]
    lib.meshopt_encodeIndexBuffer.restype = sz
    lib.meshopt_encodeIndexBuffer.argtypes = [vp, sz, vp, sz]
    return lib


def encode(ref, indices, version):
    indices = np.ascontiguousarray(indices, np.uint32)
    ref.meshopt_encodeIndexVersion(version)
    vertex_count = int(indices.max()) + 1 if len(indices) else 1
    buf = np.zeros(ref.meshopt_encodeIndexBufferBound(len(indices), min(vertex_count, 1 << 32)), np.uint8)
    n = ref.meshopt_encodeIndexBuffer(buf.ctypes.data, len(buf), indices.ctypes.data, len(indices))
    assert n > 0 and buf[0] == 0xE0 | version
    return buf[:n].copy()


def _check(stream, index_count, guard=False, what="", want=None):
    data = index_cache(stream, index_count)
    status, info = _parse(data)
    assert status == OK, what
    hs, host = _host_read(data, info, IDX)
    ds, dev = _device_read(data, info, IDX, guard)
    assert ds == hs, (what, ds, hs)
    assert hs == want if want is not None else hs != OK, (what, hs, want)
    if hs == OK:
        assert np.array_equal(dev, host), (what, int(np.flatnonzero(dev != host)[0]) // 4)
    else:
        assert (dev == 0xEE).all(), what  # a refused stream is found before any launch: dst untouched
    return hs


# ---- meshes ----------------------------------------------------------------------------------------------------------------
def strip(n):
    i = np.arange(n)
    tris = np.stack([i, i + 1 + (i & 1), i + 2 - (i & 1)], 1)
    return tris.ravel()


def grid(w, h):
    q = (np.arange(h)[:, None] * (w + 1) + np.arange(w)[None, :]).ravel()
    return np.stack([q, q + 1, q + w + 1, q + 1, q + w + 2, q + w + 1], 1).ravel()


def fan(n):
    i = np.arange(n)
    return np.stack([np.zeros(n, np.int64), i + 1, i + 2], 1).ravel()


def kitten_chain():
    data = np.fromfile(os.path.join(GOLDEN, "kitten.z.cache"), np.uint8)
    status, info = _parse(data)
    assert status == OK
    return _host_read(data, info, IDX)[1].view(np.uint32)


# ---- streams any code of the format writes ---------------------------------------------------------------------------------
def varint(v):
    out = []
    while True:
        if v < 128:
            return out + [v]
        out.append((v & 127) | 128)
        v >>= 7


def zigzag(d):
    d &= 0xFFFFFFFF
    s = d - (1 << 32) if d >= 1 << 31 else d
    return ((s << 1) ^ (s >> 31)) & 0xFFFFFFFF


def synthetic_stream(rng, triangles, version, resets_at=(), deep_at=(), jumps=False):
    """a valid stream of `triangles` codes drawn over the whole code space: edge lookups 1..15 back, FIFO lookups up to 15
    back, last -/+ 1 (v1), explicit varints (31-bit jumps and 5-byte encodings when `jumps`), restarts from the aux table
    and explicit restarts; `resets_at` triangles are 0xfe restarts with aux 0 (next = 0), `deep_at` triangles look 15 back
    in the edge ring and the vertex ring"""
    direct = 13 if version else 15
    aux = rng.integers(0, 256, 16).astype(np.uint8)
    aux[aux >> 4 == 15] &= 0xEF  # aux-table restarts with explicit corners are legal but rare; keep most table entries lookups
    codes, data = [], []

    def delta():
        if jumps and rng.random() < 0.3:
            return int(rng.choice([0x7FFFFFFF, 0x80000000, 0xFFFFFFFF, 1 << 31 | 5, int(rng.integers(0, 1 << 32))]))
        return int(rng.integers(-40, 41))

    def explicit():
        z = zigzag(delta())
        if jumps and rng.random() < 0.1 and z < (1 << 28):
            # the same value in 5 bytes, the fifth with its top bit set (a varint ends after 5 bytes whatever that
            # byte says) and bits past 32 that the decoder drops
            b = [(z >> (7 * i)) & 127 | 128 for i in range(4)] + [(z >> 28) | int(rng.integers(0, 8)) << 4 | 128]
            return b
        return varint(z)

    for t in range(triangles):
        if t in resets_at:
            codes.append(0xFE)
            data.append(0)
            continue
        if t in deep_at:
            codes.append(0xE0 | (14 if direct == 15 else 12))  # edge 15 back; vertex back(15) in v0, back(13) in v1
            continue
        r = rng.random()
        if r < 0.55:
            sel = int(rng.integers(0, 16))
            codes.append(int(rng.integers(0, 15)) << 4 | sel)
            if sel == 15:
                data += explicit()
        elif r < 0.75:
            codes.append(0xF0 | int(rng.integers(0, 14)))
            x = int(aux[codes[-1] & 15])
            for sel in (x >> 4, x & 15):
                if sel == 15:
                    data += explicit()
        else:
            code = 0xFE if rng.random() < 0.5 else 0xFF
            x = int(rng.integers(0, 256)) if rng.random() < 0.9 else 0
            codes.append(code)
            data.append(x)
            if code == 0xFF:
                data += explicit()
            for sel in (x >> 4, x & 15):
                if sel == 15:
                    data += explicit()
    return np.array([0xE0 | version] + codes + data + list(aux), np.uint8)


# ---- CPU tier ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["kitten.z.cache", "pirateglb.z.cache", "animated.z.cache", "animated_clrt.z.cache"])
def test_reference_written_caches(name):
    data = np.fromfile(os.path.join(GOLDEN, name), np.uint8)
    status, info = _parse(data)
    assert status == OK and info.sections[IDX].compressed
    hs, host = _host_read(data, info, IDX)
    ds, dev = _device_read(data, info, IDX)
    assert hs == OK and ds == OK and np.array_equal(dev, host), name


@needs_ref
@pytest.mark.parametrize("version", [0, 1])
def test_encoder_streams_at_chunk_boundaries(version):
    ref = _ref()
    rng = np.random.default_rng(10 + version)
    for triangles in (0, 1, CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 5):
        tris = rng.integers(0, max(3, triangles // 2), (triangles, 3))
        _check(encode(ref, tris.ravel(), version), 3 * triangles, what=("random", triangles), want=OK)
    for name, idx in (("strip", strip(5 * CHUNK + 7)), ("grid", grid(40, 30)), ("fan", fan(4 * CHUNK + 3))):
        _check(encode(ref, idx, version), len(idx), what=name, want=OK)


@needs_ref
def test_encoder_stream_over_several_runs():
    """more than RUN chunks: the combine step's run totals, their scan and the per-run prefixes all take part"""
    ref = _ref()
    idx = grid(260, 2 * RUN * CHUNK // 520 + 3)
    assert len(idx) // 3 > 2 * RUN * CHUNK
    _check(encode(ref, idx, 1), len(idx), what="grid", want=OK)


@needs_ref
@pytest.mark.parametrize("version", [0, 1])
def test_kitten_chain_reencoded(version):
    ref = _ref()
    chain = kitten_chain()
    _check(encode(ref, chain, version), len(chain), what="kitten", want=OK)


@needs_ref
def test_short_random_encoder_streams():
    """a few thousand short buffers: random triangles over few and over 2^32 vertices (31-bit jumps, `last` wrapping),
    with repeated and restarted runs"""
    ref = _ref()
    rng = np.random.default_rng(77)
    for k in range(2000):
        triangles = int(rng.integers(0, 3 * CHUNK))
        kind = k % 4
        if kind == 0:
            tris = rng.integers(0, 12, (triangles, 3))
        elif kind == 1:
            tris = rng.integers(0, 1 << 32, (triangles, 3), dtype=np.uint64)
        elif kind == 2:
            tris = strip(triangles).reshape(-1, 3) if triangles else np.zeros((0, 3), np.int64)
            tris = np.where(rng.random(tris.shape) < 0.05, rng.integers(0, 1 << 32, tris.shape, dtype=np.uint64), tris)
        else:
            tris = np.concatenate([grid(4, 4).reshape(-1, 3)] * (triangles // 32 + 1))[:triangles]
        _check(encode(ref, np.asarray(tris, np.uint64).astype(np.uint32).ravel(), int(rng.integers(0, 2))), 3 * triangles, what=("short", k), want=OK)


@pytest.mark.parametrize("version", [0, 1])
def test_synthetic_streams_cross_chunks(version):
    """every code kind, resets on a chunk's first triangle, lookups 15 back at a chunk's start, never-written slots read
    near the stream's start, 31-bit jumps, `last` wrapping and 5-byte varints"""
    rng = np.random.default_rng(30 + version)
    cases = [
        dict(triangles=1, deep_at={0}),
        dict(triangles=20, deep_at={0, 1, 2, 3}),
        dict(triangles=3 * CHUNK + 1, resets_at={CHUNK, 2 * CHUNK}, deep_at={CHUNK + 1, 2 * CHUNK + 1, 3 * CHUNK}),
        dict(triangles=4 * CHUNK, deep_at={CHUNK, 2 * CHUNK, 3 * CHUNK}, jumps=True),
        dict(triangles=2 * CHUNK + 17, resets_at={0, CHUNK, CHUNK + 1}, jumps=True),
    ]
    for k, case in enumerate(cases):
        triangles = case.pop("triangles")
        _check(synthetic_stream(rng, triangles, version, **case), 3 * triangles, what=(k, triangles), want=OK)
    for k in range(300):
        triangles = int(rng.integers(0, 2 * CHUNK + 40))
        resets = set(rng.integers(0, max(triangles, 1), 3).tolist())
        _check(synthetic_stream(rng, triangles, version, resets_at=resets, jumps=k % 2 == 1), 3 * triangles, what=("random", k), want=OK)


def hostile_streams():
    """(label, stream, index_count, status the host read gives; None: some refusal)"""
    rng = np.random.default_rng(5)
    good = synthetic_stream(rng, CHUNK + 3, 1, jumps=True)
    tri = CHUNK + 3
    # a stream whose last data token is a 5-byte varint with a set top bit in its fifth byte: legal
    five = np.array([0xE1, 0x0F, 0x81, 0x82, 0x83, 0x84, 0xF5] + [0] * 16, np.uint8)
    out = [("five-byte varint", five, 3, OK)]
    n_data = len(good) - 16 - 1 - tri
    assert n_data > 2
    out.append(("one data byte short", np.concatenate([good[: len(good) - 17], good[-16:]]), 3 * tri, None))
    out.append(("trailing data byte", np.concatenate([good[:-16], [0], good[-16:]]).astype(np.uint8), 3 * tri, CORRUPT))
    out.append(("truncated", good[: 1 + tri + 15], 3 * tri, CORRUPT))
    bad = good.copy()
    bad[0] = 0xD1
    out.append(("bad header", bad, 3 * tri, CORRUPT))
    v2 = good.copy()
    v2[0] = 0xE2
    out.append(("version 2", v2, 3 * tri, UNSUPPORTED))
    out.append(("count not a multiple of 3", good, 3 * tri - 1, INVALID))
    # a varint cut by the aux table in the first chunk, with valid chunks after it
    cut = np.array([0xE1, 0x0F] + [0xE0] * (CHUNK + 2) + [0x80, 0x80] + [0] * 16, np.uint8)
    out.append(("data runs into the aux table", cut, 3 * (CHUNK + 3), CORRUPT))
    return out


@pytest.mark.parametrize("guard", [False, True])
def test_hostile_streams(guard):
    """the same status as the host read; a refused stream leaves dst untouched.  Guarded: a fresh context whose scratch,
    like dst, ends at an inaccessible page"""
    for label, stream, count, want in hostile_streams():
        _check(stream, count, guard=guard, what=label, want=want)


@needs_ref
def test_valid_streams_in_the_guarded_build():
    ref = _ref()
    rng = np.random.default_rng(9)
    for triangles in (1, CHUNK, 2 * CHUNK + 1):
        _check(encode(ref, rng.integers(0, 1 << 32, 3 * triangles, dtype=np.uint64).astype(np.uint32), 1), 3 * triangles, guard=True, want=OK)
    _check(synthetic_stream(rng, 3 * CHUNK + 2, 0, resets_at={CHUNK}, jumps=True), 3 * (3 * CHUNK + 2), guard=True, want=OK)


# ---- GPU tier ----------------------------------------------------------------------------------------------------------------
def _gpu_check(stream, count, tmp_path, what, want=OK):
    hs, host, ds, dev = _gpu_read(index_cache(stream, count), IDX, tmp_path, what)
    assert ds == hs and (hs == want if want is not None else hs != OK), (what, hs, ds)
    if want == OK:
        assert np.array_equal(dev, host), (what, int(np.flatnonzero(dev != host)[0]) // 4)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kitten.z.cache", "pirateglb.z.cache", "animated.z.cache", "animated_clrt.z.cache"])
def test_gpu_reference_written_caches(name, tmp_path):
    data = np.fromfile(os.path.join(GOLDEN, name), np.uint8)
    hs, host, ds, dev = _gpu_read(data, IDX, tmp_path, name)
    assert hs == OK and ds == OK and np.array_equal(dev, host), name


@pytest.mark.gpu
@needs_ref
def test_gpu_thousand_kitten_chains(tmp_path):
    ref = _ref()
    chain = np.tile(kitten_chain(), 1000)
    _gpu_check(encode(ref, chain, 1), len(chain), tmp_path, "1000 kittens")


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("version", [0, 1])
def test_gpu_random_encoder_streams(version, tmp_path):
    ref = _ref()
    rng = np.random.default_rng(60 + version)
    for triangles, span in ((1, 3), (CHUNK * RUN + 1, 1 << 32), (3_000_000, 2000), (10_000_000, 1 << 20)):
        if span < 1 << 20:
            idx = rng.integers(0, span, 3 * triangles, dtype=np.uint64).astype(np.uint32)
        else:
            # a strip whose corners now and then jump anywhere: long edge chains, explicit varints of every length
            idx = strip(triangles).astype(np.uint64)
            jumps = rng.random(len(idx)) < 0.02
            idx[jumps] = rng.integers(0, span, int(jumps.sum()), dtype=np.uint64)
            idx = idx.astype(np.uint32)
        _gpu_check(encode(ref, idx, version), len(idx), tmp_path, (version, triangles))


@pytest.mark.gpu
def test_gpu_synthetic_and_hostile_streams(tmp_path):
    rng = np.random.default_rng(70)
    for version in (0, 1):
        triangles = 40 * CHUNK + 9
        resets = {CHUNK * k for k in range(0, 40, 3)}
        _gpu_check(synthetic_stream(rng, triangles, version, resets_at=resets, deep_at={CHUNK * k + 1 for k in range(40)}, jumps=True), 3 * triangles, tmp_path, version)
    for label, stream, count, want in hostile_streams():
        if want != INVALID:  # SceneCache parses the file; a count that is not a multiple of 3 is checked on the CPU tier
            _gpu_check(stream, count, tmp_path, label, want)


@pytest.mark.gpu
@needs_ref
def test_gpu_read_on_a_busy_non_blocking_stream(tmp_path):
    """work already queued on a non-blocking stream finishes before the call's uploads; the result is in place on return"""
    import torch

    from niagara_b200.scene_cache import SceneCache

    ref = _ref()
    chain = np.tile(kitten_chain(), 20)
    path = os.path.join(str(tmp_path), "indices.cache")
    data = index_cache(encode(ref, chain, 1), len(chain))
    data.tofile(path)
    side = torch.cuda.Stream()
    c = SceneCache(path)
    try:
        want = chain.view(np.uint8)
        with torch.cuda.stream(side):
            for _ in range(3):
                torch.cuda._sleep(1_000_000)
                got = c.section_device("indices").cpu().numpy()
                assert np.array_equal(got, want)
    finally:
        c.close()
