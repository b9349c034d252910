"""CPU-only: meshopt-compressed glTF import (EXT_meshopt_compression / KHR_meshopt_compression, row N3).

* the decoders the extension adds to the vertex and index codecs — the index codec into 16-bit indices, the index-sequence codec,
  the four vertex filters — against the REFERENCE's own meshoptimizer (oracle/_ref/libmeshopt_full_ref.so, all of
  extern/meshoptimizer/src compiled where it lies), byte for byte; the 8-bit OCTAHEDRAL and COLOR filters over every input,
  because their results depend on the CPU's rsqrtps / rcpps;
* the importer on gltfpack's output (tests/golden/meshopt/, written by make_meshopt_gltf_fixtures.py with the reference's
  gltfpack) against what the reference's loadScene produced from the same files, and on a lossless pair (the same scene with
  and without compression);
* the refusals, each against the reference loader's verdict on the same hostile edit;
* the importer built with ASan + UBSan over mutations of the compressed fixtures."""
import ctypes
import importlib.util
import json
import os
import subprocess

import numpy as np
import pytest

from niagara_b200 import gltf
from niagara_b200.lib import load_library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
MESHOPT = os.path.join(GOLDEN, "meshopt")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libmeshopt_full_ref.so")

vp, sz = ctypes.c_void_p, ctypes.c_size_t
OK, INVALID, UNSUPPORTED, CORRUPT = 0, -1, -6, -7
NONE, OCTAHEDRAL, QUATERNION, EXPONENTIAL, COLOR = range(5)

needs_ref = pytest.mark.skipif(not os.path.exists(REF_SO), reason="needs the reference's codecs (oracle/_ref/libmeshopt_full_ref.so, built by build())")


def _fixtures():
    spec = importlib.util.spec_from_file_location("make_meshopt_gltf_fixtures", os.path.join(GOLDEN, "make_meshopt_gltf_fixtures.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def ref():
    lib = ctypes.CDLL(REF_SO)
    lib.meshopt_encodeIndexVersion.argtypes = [ctypes.c_int]
    lib.meshopt_encodeIndexBufferBound.restype = sz
    lib.meshopt_encodeIndexBufferBound.argtypes = [sz, sz]
    lib.meshopt_encodeIndexBuffer.restype = sz
    lib.meshopt_encodeIndexBuffer.argtypes = [vp, sz, vp, sz]
    lib.meshopt_decodeIndexBuffer.restype = ctypes.c_int
    lib.meshopt_decodeIndexBuffer.argtypes = [vp, sz, sz, vp, sz]
    lib.meshopt_encodeIndexSequenceBound.restype = sz
    lib.meshopt_encodeIndexSequenceBound.argtypes = [sz, sz]
    lib.meshopt_encodeIndexSequence.restype = sz
    lib.meshopt_encodeIndexSequence.argtypes = [vp, sz, vp, sz]
    lib.meshopt_decodeIndexSequence.restype = ctypes.c_int
    lib.meshopt_decodeIndexSequence.argtypes = [vp, sz, sz, vp, sz]
    for name in ("Oct", "Quat", "Exp", "Color"):
        getattr(lib, "meshopt_decodeFilter" + name).argtypes = [vp, sz, sz]
    for name in ("Oct", "Quat", "Color"):
        getattr(lib, "meshopt_encodeFilter" + name).argtypes = [vp, sz, sz, ctypes.c_int, vp]
    lib.meshopt_encodeFilterExp.argtypes = [vp, sz, sz, ctypes.c_int, vp, ctypes.c_int]
    return lib


def _p(a):
    return a.ctypes.data_as(vp)


# ---- decoders against the reference's --------------------------------------------------------------------------------------
def _sequences(rng):
    yield "empty", np.zeros(0, np.uint32)
    yield "monotonic", np.arange(3000, dtype=np.uint32)
    yield "random", rng.integers(0, 70000, 3001, dtype=np.uint32)
    yield "restarts", np.concatenate([np.arange(k * 1000, k * 1000 + 200, dtype=np.uint32) for k in range(5)] + [np.full(7, 0xFFFFFFFF, np.uint32)])
    yield "jumps31", (rng.integers(0, 1 << 31, 999, dtype=np.int64) ^ np.where(np.arange(999) % 2, 0x7FFFFFFF, 0)).astype(np.uint32)
    yield "short", np.array([5], np.uint32)


@needs_ref
@pytest.mark.parametrize("version", [0, 1])
def test_index_sequence_against_reference(ref, version):
    ours = load_library()
    rng = np.random.default_rng(40 + version)
    ref.meshopt_encodeIndexVersion(version)
    try:
        for name, seq in _sequences(rng):
            seq = np.ascontiguousarray(seq)
            buf = np.zeros(ref.meshopt_encodeIndexSequenceBound(len(seq), 1 << 32 if len(seq) else 1), np.uint8)
            n = ref.meshopt_encodeIndexSequence(_p(buf), len(buf), _p(seq), len(seq))
            assert n > 0 and buf[0] == 0xD0 | version
            stream = np.ascontiguousarray(buf[:n])
            for size, dtype in ((2, np.uint16), (4, np.uint32)):
                want = np.zeros(len(seq) + 1, dtype)
                got = np.full(len(seq) + 1, 0xEEEE, dtype)
                assert ref.meshopt_decodeIndexSequence(_p(want), len(seq), size, _p(stream), n) == 0
                assert ours.nvc_decode_index_sequence(_p(got), len(seq), size, _p(stream), n) == OK, (name, size)
                assert np.array_equal(got[: len(seq)], want[: len(seq)]), (name, size)
                assert got[len(seq)] == dtype(0xEEEE)
                if name != "jumps31":  # deltas of 2^30 and more do not survive the encoder (its varint has 32 bits for 33)
                    assert np.array_equal(want[: len(seq)], seq.astype(dtype))
                # truncated, extended and re-headered streams: refused by both
                for bad, bad_n in ((stream, n - 1), (np.concatenate([stream[:-4], [0x10], stream[-4:]]).astype(np.uint8), n + 1)):
                    bad = np.ascontiguousarray(bad)
                    assert (ref.meshopt_decodeIndexSequence(_p(want), len(seq), size, _p(bad), bad_n) != 0) == (ours.nvc_decode_index_sequence(_p(got), len(seq), size, _p(bad), bad_n) != 0)
                    assert ours.nvc_decode_index_sequence(_p(got), len(seq), size, _p(bad), bad_n) == CORRUPT
                wrong = stream.copy()
                wrong[0] = 0xE0 | version
                assert ours.nvc_decode_index_sequence(_p(got), len(seq), size, _p(wrong), n) == CORRUPT
                wrong[0] = 0xD2
                assert ours.nvc_decode_index_sequence(_p(got), len(seq), size, _p(wrong), n) == UNSUPPORTED
            assert ours.nvc_decode_index_sequence(_p(got), len(seq), 3, _p(stream), n) == INVALID
    finally:
        ref.meshopt_encodeIndexVersion(1)


@needs_ref
@pytest.mark.parametrize("version", [0, 1])
def test_index_codec_into_16_bits_against_reference(ref, version):
    ours = load_library()
    rng = np.random.default_rng(60 + version)
    ref.meshopt_encodeIndexVersion(version)
    try:
        for triangles in (0, 1, 7, 500, 4000):
            for kind in ("strip", "random", "wide"):
                if kind == "strip":
                    t = np.arange(triangles, dtype=np.uint32)
                    idx = np.stack([t, t + 1, t + 2], 1).reshape(-1)
                elif kind == "random":
                    idx = rng.integers(0, max(3, triangles), triangles * 3, dtype=np.uint32)
                else:  # indices past 16 bits: the 16-bit output keeps the low half, as the reference's does
                    idx = rng.integers(0, 1 << 20, triangles * 3, dtype=np.uint32)
                idx = np.ascontiguousarray(idx.astype(np.uint32))
                buf = np.zeros(ref.meshopt_encodeIndexBufferBound(len(idx), 1 << 20), np.uint8)
                n = ref.meshopt_encodeIndexBuffer(_p(buf), len(buf), _p(idx), len(idx))
                assert n > 0
                stream = np.ascontiguousarray(buf[:n])
                for size, dtype in ((2, np.uint16), (4, np.uint32)):
                    want = np.zeros(len(idx) + 1, dtype)
                    got = np.full(len(idx) + 1, 0xEEEE, dtype)
                    assert ref.meshopt_decodeIndexBuffer(_p(want), len(idx), size, _p(stream), n) == 0
                    assert ours.nvc_decode_index_buffer(_p(got), len(idx), size, _p(stream), n) == OK
                    assert np.array_equal(got[: len(idx)], want[: len(idx)]) and got[len(idx)] == dtype(0xEEEE), (triangles, kind, size)
                    assert ours.nvc_decode_index_buffer(_p(got), len(idx), size, _p(stream), n - 1) != OK
                wide = np.zeros(len(idx), np.uint32)
                assert ours.nvc_decode_index_stream(_p(wide), len(idx), _p(stream), n) == OK
                assert np.array_equal(wide, want[: len(idx)])  # 4-byte output == the 32-bit decoder's
    finally:
        ref.meshopt_encodeIndexVersion(1)
    assert load_library().nvc_decode_index_buffer(None, 4, 2, _p(np.zeros(32, np.uint8)), 32) == INVALID


def _filter_inputs(rng, filt, count, stride, bits, mode):
    """(encoded bytes, via the reference's encoder) for count elements of `stride` bytes"""
    if filt == EXPONENTIAL:
        data = (rng.standard_normal(count * stride // 4) * np.exp2(rng.integers(-30, 30, count * stride // 4))).astype(np.float32)
        return data, (stride, bits, mode)
    data = rng.standard_normal((count, 4)).astype(np.float32)
    if filt in (OCTAHEDRAL, QUATERNION):
        data /= np.linalg.norm(data if filt == QUATERNION else np.concatenate([data[:, :3], np.zeros((count, 1), np.float32)], 1), axis=1, keepdims=True)
        if filt == OCTAHEDRAL:
            data[:, 3] = rng.uniform(-1, 1, count)
    else:
        data = rng.uniform(0, 1, (count, 4)).astype(np.float32)
    return np.ascontiguousarray(data, np.float32), (stride, bits)


_LEGAL = [(OCTAHEDRAL, 4, range(2, 9)), (OCTAHEDRAL, 8, range(2, 17)), (QUATERNION, 8, range(4, 17)), (COLOR, 4, range(2, 9)), (COLOR, 8, range(2, 17))]
_LEGAL += [(EXPONENTIAL, s, range(1, 25)) for s in (4, 8, 12, 16, 64, 256)]


@needs_ref
def test_vertex_filters_against_reference(ref):
    ours = load_library()
    rng = np.random.default_rng(77)
    names = {OCTAHEDRAL: "Oct", QUATERNION: "Quat", EXPONENTIAL: "Exp", COLOR: "Color"}
    cases = 0
    for filt, stride, bit_range in _LEGAL:
        for bits in bit_range:
            for mode in (range(4) if filt == EXPONENTIAL else (None,)):
                if filt == EXPONENTIAL and stride > 16 and bits not in (1, 8, 15, 24):
                    continue
                for count in list(range(10)) + [97, 1000]:
                    data, _ = _filter_inputs(rng, filt, count, stride, bits, mode)
                    enc = np.zeros(count * stride + 16, np.uint8)
                    if count:
                        if filt == EXPONENTIAL:
                            ref.meshopt_encodeFilterExp(_p(enc), count, stride, bits, _p(data), mode)
                        else:
                            getattr(ref, "meshopt_encodeFilter" + names[filt])(_p(enc), count, stride, bits, _p(data))
                    # raw bytes too: every bit pattern of the stored fields, not only what the encoder emits
                    raw = rng.integers(0, 256, count * stride + 16, dtype=np.uint8)
                    for src in (enc, raw):
                        want, got = src.copy(), src.copy()
                        getattr(ref, "meshopt_decodeFilter" + names[filt])(_p(want), count, stride)
                        assert ours.nvc_decode_vertex_filter(filt, _p(got), count, stride) == OK
                        assert got.tobytes() == want.tobytes(), (filt, stride, bits, mode, count)
                        cases += 1
    assert cases > 3000


@needs_ref
@pytest.mark.parametrize("filt", [OCTAHEDRAL, COLOR])
def test_8bit_octahedral_and_color_filters_over_every_input(ref, filt):
    """the three bytes these filters scale through rsqrtps / rcpps (x, y, z / Y, Co, Cg), all 2^24 of them, under four alpha / w
    values (the COLOR filter's bit count comes from alpha)"""
    ours = load_library()
    names = {OCTAHEDRAL: "Oct", COLOR: "Color"}
    low = np.arange(1 << 24, dtype=np.uint32)
    for top in (0x00, 0x01, 0x7F, 0xFF):
        x = low | np.uint32(top << 24)
        want, got = x.copy(), x.copy()
        getattr(ref, "meshopt_decodeFilter" + names[filt])(_p(want), len(x), 4)
        assert ours.nvc_decode_vertex_filter(filt, _p(got), len(x), 4) == OK
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (top, [hex(int(x[i])) for i in bad[:5]])


def test_vertex_filter_strides_follow_the_extension():
    ours = load_library()
    buf = np.zeros(4096, np.uint8)
    legal = {NONE: set(range(4, 257, 4)), OCTAHEDRAL: {4, 8}, QUATERNION: {8}, EXPONENTIAL: set(range(4, 257, 4)), COLOR: {4, 8}}
    for filt, ok in legal.items():
        for stride in range(0, 264):
            assert (ours.nvc_decode_vertex_filter(filt, _p(buf), 3, stride) == OK) == (stride in ok), (filt, stride)
    assert ours.nvc_decode_vertex_filter(5, _p(buf), 3, 8) == INVALID
    assert ours.nvc_decode_vertex_filter(OCTAHEDRAL, None, 3, 8) == INVALID
    assert ours.nvc_decode_vertex_filter(OCTAHEDRAL, None, 0, 8) == OK


# ---- the importer against the reference's loader ----------------------------------------------------------------------------
def _names():
    return _fixtures().fixture_names()


def _same_draws(mine, ref):
    mine = mine.copy()
    mine["meshletVisibilityOffset"] = ref["meshletVisibilityOffset"]  # assigned later by the application (niagara.cpp:1002-1020)
    return mine.tobytes() == ref.tobytes()


@pytest.mark.parametrize("name", _names())
def test_compressed_scene_matches_the_reference_loader(name):
    g = gltf.GltfScene(os.path.join(MESHOPT, name + ".glb"))
    ref = np.load(os.path.join(MESHOPT, name + "_expected.npz"))
    assert g.info.draw_count == len(ref["draws"]) > 0
    assert _same_draws(g.draws, ref["draws"])
    assert g.animations.tobytes() == ref["animations"].tobytes()
    assert g.keyframes.tobytes() == ref["keyframes"].tobytes()
    if g.info.has_camera:
        cam = np.array(list(g.info.camera.position) + list(g.info.camera.orientation) + [g.info.camera.fovY], np.float32)
        assert cam.tobytes() == ref["camera"].tobytes()
    if g.info.has_sun:
        assert np.array(list(g.info.sun_direction), np.float32).tobytes() == ref["sun"].tobytes()
    assert g.info.primitive_count == len(ref["mesh_vertex_offset"])
    verts = ref["vertices"].view(gltf.VERTEX_DTYPE) if ref["vertices"].dtype != gltf.VERTEX_DTYPE else ref["vertices"]
    for m in range(g.info.primitive_count):
        v, ix = g.primitive(m)
        assert len(ix) % 3 == 0 and ix.max() < len(v)
        if len(verts):  # loadVertices output == the reference's cooked vertices as a set (it de-duplicates and reorders)
            used = np.unique(v[np.unique(ix)].view(np.uint8).reshape(-1, 16), axis=0)
            lo, n = int(ref["mesh_vertex_offset"][m]), int(ref["mesh_vertex_count"][m])
            assert np.array_equal(used, np.unique(np.ascontiguousarray(verts[lo : lo + n]).view(np.uint8).reshape(-1, 16), axis=0)), m
    g.close()


def _canonical_triangles(ix):
    """each triangle rotated to start at its smallest index: the index codec keeps a triangle's winding, not its first corner"""
    t = ix.reshape(-1, 3)
    r = np.argmin(t, axis=1)
    return np.stack([t[np.arange(len(t)), (r + k) % 3] for k in range(3)], 1)


@pytest.mark.parametrize("scene", ["animated", "hierarchy"])
def test_lossless_compression_imports_identically(scene):
    """gltfpack -noq with and without -c: the same data; everything the importer returns is equal"""
    a = gltf.GltfScene(os.path.join(MESHOPT, scene + "_noq.glb"))
    b = gltf.GltfScene(os.path.join(MESHOPT, scene + "_noqc.glb"))
    assert b"meshopt_compression" in open(os.path.join(MESHOPT, scene + "_noqc.glb"), "rb").read()
    assert a.draws.tobytes() == b.draws.tobytes() and a.animations.tobytes() == b.animations.tobytes() and a.keyframes.tobytes() == b.keyframes.tobytes()
    assert a.mesh_scale.tobytes() == b.mesh_scale.tobytes()
    assert a.info.primitive_count == b.info.primitive_count > 0
    for m in range(a.info.primitive_count):
        va, ia = a.primitive(m)
        vb, ib = b.primitive(m)
        assert va.tobytes() == vb.tobytes()
        assert np.array_equal(_canonical_triangles(ia), _canonical_triangles(ib))


def test_kitten_cc_loads_through_the_package():
    g = gltf.GltfScene(os.path.join(MESHOPT, "kitten_cc.glb"))
    ref = np.load(os.path.join(MESHOPT, "kitten_cc_expected.npz"))
    assert g.info.primitive_count == 1 and _same_draws(g.draws, ref["draws"]) and g.keyframes.tobytes() == ref["keyframes"].tobytes()
    v, ix = g.primitive(0)
    assert len(ix) > 10000 and len(v) > 1000
    g.close()


# ---- refusals -----------------------------------------------------------------------------------------------------------------
def _import(data):
    lib = load_library()
    scene = ctypes.c_void_p(0x1234)
    status = lib.nvc_gltf_import(data, len(data), b".", 0, 1, ctypes.byref(scene))
    ok = scene.value is not None
    if status == OK:
        lib.nvc_gltf_free(scene)
    return status, ok


def test_hostile_edits_are_refused_where_the_reference_refuses():
    fx = _fixtures()
    verdicts = json.load(open(os.path.join(MESHOPT, "hostile_verdicts.json")))
    assert set(verdicts) == {e[0] for e in fx.HOSTILE_EDITS}
    for name, base, _, status in fx.HOSTILE_EDITS:
        data = fx.apply_edit(name)
        got, has_scene = _import(data)
        if name == "fallback buffer read by an uncompressed view":
            # the reference's loader accepts this file: cgltf reads nothing from a buffer without data and the attribute stays
            # zero.  The importer refuses it instead of inventing the attribute's values.
            assert verdicts[name] is True and got == CORRUPT and not has_scene
            continue
        assert (got == OK) == verdicts[name], (name, got)
        if got != OK:
            assert not has_scene, name  # a refusal hands back no scene
            assert got == status if status is not None else got in (CORRUPT, UNSUPPORTED), (name, got)
        elif status is not None:
            assert status == OK, name


def test_fallback_buffer_without_the_flag_is_still_a_buffer_without_data():
    fx = _fixtures()
    doc, blob = fx.read_glb(open(os.path.join(MESHOPT, "hierarchy_cc.glb"), "rb").read())
    del doc["buffers"][1]["extensions"]
    assert _import(fx.write_glb(doc, blob))[0] == CORRUPT


# ---- sanitizers ---------------------------------------------------------------------------------------------------------------
def test_importer_under_address_and_ub_sanitizers_on_compressed_files(tmp_path):
    """tests/fuzz_gltf.cpp + the importer with ASan + UBSan (the command line of test_gltf_import.py) over mutations of every
    compressed fixture: the importer's decoders link from its own translation unit"""
    exe = str(tmp_path / "fuzz_gltf")
    srcs = [os.path.join(ROOT, "tests", "fuzz_gltf.cpp"), os.path.join(ROOT, "niagara_b200", "csrc", "nvc_gltf.cpp")]
    build = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-o", exe] + srcs, capture_output=True, text=True)
    if build.returncode != 0 and "sanitize" in build.stderr:
        pytest.skip("this toolchain has no sanitizer runtime: " + build.stderr.splitlines()[0])
    assert build.returncode == 0, build.stderr
    for name in ("hierarchy_cc", "animated_cz", "kitten_ccvpf", "synthetic", "hierarchy_noqc"):
        run = subprocess.run([exe, os.path.join(MESHOPT, name + ".glb"), "3000"], capture_output=True, text=True)
        assert run.returncode == 0, (name, run.stdout[-500:], run.stderr[-3000:])
        assert "mutations 3000" in run.stdout
