#!/usr/bin/env python3
"""Writes tests/golden/meshopt/: meshopt-compressed glTF files and what the REFERENCE's loader makes of them.

* gltfpack (the reference's vendored packer, built into oracle/_ref/gltfpack by oracle/refgltfpack) run on our own animated.gltf
  and hierarchy.glb and on the reference's kitten.obj with -c, -cc, -cc -vpf and -cz (EXT_meshopt_compression; -cz writes
  KHR_meshopt_compression), and with -noq / -noq -c on the two scenes: the same data uncompressed and compressed (lossless pair);
* synthetic.glb, assembled here, for the combinations gltfpack does not write: 16-bit OCTAHEDRAL, 8- and 16-bit COLOR, TRIANGLES
  with 4-byte indices, INDICES (index sequences, 2- and 4-byte) and vertex codec v0 — its views encoded by the reference's own
  encoders (meshopt_encode*, meshopt_encodeFilter* in oracle/_ref/libmeshopt_full_ref.so);
* <name>_expected.npz per file: the reference's loadScene output through oracle/_ref/write_cache (MeshDraw[], Animation[],
  Keyframe[], camera, sun, per-mesh vertex ranges and cooked Vertex[] — empty for three of the four kitten files, to keep
  the fixtures small), in the form of hierarchy_expected.npz;
* hostile_verdicts.json: whether the reference's loader accepts each edit of HOSTILE_EDITS (defined here, applied to
  hierarchy_cc.glb / synthetic.glb by tests/test_gltf_meshopt.py as well).

Only runs where the reference checkout exists.  Run: python tests/golden/make_meshopt_gltf_fixtures.py"""
import copy
import ctypes
import json
import os
import struct
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "meshopt")
REF_BIN = os.path.join(ROOT, "oracle", "_ref")
REFERENCE = os.environ.get("NIAGARA_REFERENCE", "/root/reference")

PACKED = {"c": ["-c"], "cc": ["-cc"], "ccvpf": ["-cc", "-vpf"], "cz": ["-cz"]}
LOSSLESS = {"noq": ["-noq"], "noqc": ["-noq", "-c"]}
EXTENSIONS = ("EXT_meshopt_compression", "KHR_meshopt_compression")


def sources():
    return {"animated": os.path.join(HERE, "animated.gltf"), "hierarchy": os.path.join(HERE, "hierarchy.glb"), "kitten": os.path.join(REFERENCE, "data", "kitten.obj")}


def fixture_names():
    names = [f"{s}_{m}" for s in ("animated", "hierarchy", "kitten") for m in PACKED]
    names += [f"{s}_{m}" for s in ("animated", "hierarchy") for m in LOSSLESS]
    return names + ["synthetic"]


# ---- GLB ----------------------------------------------------------------------------------------------------------------------
def read_glb(data):
    jlen = struct.unpack_from("<I", data, 12)[0]
    doc = json.loads(data[20 : 20 + jlen])
    rest = data[20 + jlen :]
    blob = rest[8 : 8 + struct.unpack_from("<I", rest, 0)[0]] if len(rest) >= 8 else b""
    return doc, bytearray(blob)


def write_glb(doc, blob):
    js = json.dumps(doc, separators=(",", ":")).encode()
    js += b" " * (-len(js) % 4)
    blob = bytes(blob) + b"\0" * (-len(blob) % 4)
    return struct.pack("<4sII", b"glTF", 2, 12 + 8 + len(js) + 8 + len(blob)) + struct.pack("<II", len(js), 0x4E4F534A) + js + struct.pack("<II", len(blob), 0x004E4942) + blob


def meshopt_ext(view):
    ext = view.get("extensions", {})
    for name in EXTENSIONS:
        if name in ext:
            return ext[name]
    return None


def combinations(doc):
    """{(extension, mode, filter, stride)} of the file's compressed views"""
    out = set()
    for v in doc.get("bufferViews", []):
        for name in EXTENSIONS:
            e = v.get("extensions", {}).get(name)
            if e:
                out.add((name, e["mode"], e.get("filter", "NONE"), e["byteStride"]))
    return out


# ---- the synthetic file ----------------------------------------------------------------------------------------------------
def _ref_codecs():
    lib = ctypes.CDLL(os.path.join(REF_BIN, "libmeshopt_full_ref.so"))
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    lib.meshopt_encodeVertexBufferBound.restype = sz
    lib.meshopt_encodeVertexBufferBound.argtypes = [sz, sz]
    lib.meshopt_encodeVertexBufferLevel.restype = sz
    lib.meshopt_encodeVertexBufferLevel.argtypes = [vp, sz, vp, sz, sz, ctypes.c_int, ctypes.c_int]
    lib.meshopt_encodeIndexVersion.argtypes = [ctypes.c_int]
    lib.meshopt_encodeIndexBufferBound.restype = sz
    lib.meshopt_encodeIndexBufferBound.argtypes = [sz, sz]
    lib.meshopt_encodeIndexBuffer.restype = sz
    lib.meshopt_encodeIndexBuffer.argtypes = [vp, sz, vp, sz]
    lib.meshopt_encodeIndexSequenceBound.restype = sz
    lib.meshopt_encodeIndexSequenceBound.argtypes = [sz, sz]
    lib.meshopt_encodeIndexSequence.restype = sz
    lib.meshopt_encodeIndexSequence.argtypes = [vp, sz, vp, sz]
    for name in ("Oct", "Quat", "Color"):
        getattr(lib, "meshopt_encodeFilter" + name).argtypes = [vp, sz, sz, ctypes.c_int, vp]
    lib.meshopt_encodeFilterExp.argtypes = [vp, sz, sz, ctypes.c_int, vp, ctypes.c_int]
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def synthetic_glb():
    sys.path.insert(0, HERE)
    from make_animated_gltf import icosphere

    lib = _ref_codecs()
    pos, tri = icosphere(2)  # 162 vertices, 320 triangles
    n = len(pos)
    rng = np.random.default_rng(31)
    blob, views, accessors = bytearray(), [], []
    fallback_at = [0]

    def add(raw, count, stride, mode, comp, typ, acount=None, filt=None, normalized=False, version=1):
        """one compressed view of `count` elements of `stride` bytes (raw: their decoded bytes, already filtered)"""
        raw = np.ascontiguousarray(np.frombuffer(bytes(raw), np.uint8))
        assert len(raw) == count * stride
        if mode == "ATTRIBUTES":
            buf = np.zeros(lib.meshopt_encodeVertexBufferBound(count, stride), np.uint8)
            size = lib.meshopt_encodeVertexBufferLevel(_p(buf), len(buf), _p(raw), count, stride, 2, version)
        else:
            idx = np.ascontiguousarray(raw.view("<u2" if stride == 2 else "<u4").astype(np.uint32))
            lib.meshopt_encodeIndexVersion(version)
            if mode == "TRIANGLES":
                buf = np.zeros(lib.meshopt_encodeIndexBufferBound(count, n), np.uint8)
                size = lib.meshopt_encodeIndexBuffer(_p(buf), len(buf), _p(idx), count)
            else:
                buf = np.zeros(lib.meshopt_encodeIndexSequenceBound(count, n), np.uint8)
                size = lib.meshopt_encodeIndexSequence(_p(buf), len(buf), _p(idx), count)
            lib.meshopt_encodeIndexVersion(1)
        assert size > 0
        while len(blob) % 4:
            blob.append(0)
        ext = {"buffer": 0, "byteOffset": len(blob), "byteLength": int(size), "byteStride": stride, "count": count, "mode": mode}
        if filt:
            ext["filter"] = filt
        blob.extend(buf[:size].tobytes())
        view = {"buffer": 1, "byteOffset": fallback_at[0], "byteLength": count * stride, "extensions": {"EXT_meshopt_compression": ext}}
        if mode == "ATTRIBUTES":
            view["byteStride"] = stride
        fallback_at[0] += count * stride
        views.append(view)
        acc = {"bufferView": len(views) - 1, "componentType": comp, "count": acount or count, "type": typ}
        if normalized:
            acc["normalized"] = True
        accessors.append(acc)
        return len(accessors) - 1

    def filtered(fn, count, stride, bits, data, *mode):
        out = np.zeros(count * stride, np.uint8)
        getattr(lib, "meshopt_encodeFilter" + fn)(_p(out), count, stride, bits, _p(np.ascontiguousarray(data, np.float32)), *mode)
        return out

    a_pos = add(pos.astype("<f4").tobytes(), n, 12, "ATTRIBUTES", 5126, "VEC3", version=0)
    accessors[a_pos]["min"], accessors[a_pos]["max"] = pos.min(0).tolist(), pos.max(0).tolist()
    nrm4 = np.concatenate([pos, np.zeros((n, 1), np.float32)], 1)
    a_nrm16 = add(filtered("Oct", n, 8, 12, nrm4), n, 8, "ATTRIBUTES", 5122, "VEC3", filt="OCTAHEDRAL", normalized=True)
    uv = np.stack([pos[:, 0] * 0.5 + 0.5, pos[:, 1] * 0.5 + 0.5], 1)
    a_uv = add((np.clip(uv, 0, 1) * 65535 + 0.5).astype("<u2").tobytes(), n, 4, "ATTRIBUTES", 5123, "VEC2", normalized=True, version=0)
    rgba = np.concatenate([rng.uniform(0, 1, (n, 3)), rng.uniform(0.2, 1, (n, 1))], 1)
    a_col8 = add(filtered("Color", n, 4, 7, rgba), n, 4, "ATTRIBUTES", 5121, "VEC4", filt="COLOR", normalized=True)
    a_col16 = add(filtered("Color", n, 8, 13, rgba), n, 8, "ATTRIBUTES", 5123, "VEC4", filt="COLOR", normalized=True)
    third = len(tri) // 3
    tris = [tri[:third], tri[third : 2 * third], tri[2 * third :]]
    a_i32 = add(tris[0].astype("<u4").tobytes(), len(tris[0]) * 3, 4, "TRIANGLES", 5125, "SCALAR")
    a_seq16 = add(tris[1].astype("<u2").tobytes(), len(tris[1]) * 3, 2, "INDICES", 5123, "SCALAR")
    a_seq32 = add(tris[2].astype("<u4").tobytes(), len(tris[2]) * 3, 4, "INDICES", 5125, "SCALAR", version=0)

    times = np.linspace(0, 2, 7).astype(np.float32)
    a_time = add(times.tobytes(), len(times), 4, "ATTRIBUTES", 5126, "SCALAR")
    accessors[a_time]["min"], accessors[a_time]["max"] = [0.0], [2.0]
    tr = rng.uniform(-3, 3, (len(times), 3)).astype(np.float32)
    a_tr = add(filtered("Exp", len(times), 12, 15, tr, 1), len(times), 12, "ATTRIBUTES", 5126, "VEC3", filt="EXPONENTIAL")
    q = rng.standard_normal((len(times), 4)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    a_rot = add(filtered("Quat", len(times), 8, 14, q), len(times), 8, "ATTRIBUTES", 5122, "VEC4", filt="QUATERNION", normalized=True)
    sc = rng.uniform(0.5, 2, (len(times), 4)).astype(np.float32)
    a_sc = add(filtered("Exp", len(times), 16, 12, sc, 0), len(times), 16, "ATTRIBUTES", 5126, "VEC3", filt="EXPONENTIAL")
    accessors[a_sc]["byteOffset"] = 0  # VEC3 read from a 16-byte stride

    doc = {
        "asset": {"version": "2.0", "generator": "niagara_b200 tests/golden/make_meshopt_gltf_fixtures.py"},
        "extensionsUsed": ["EXT_meshopt_compression", "KHR_mesh_quantization"],
        "extensionsRequired": ["EXT_meshopt_compression", "KHR_mesh_quantization"],
        "scene": 0,
        "scenes": [{"nodes": [0, 2]}],
        "nodes": [
            {"name": "parent", "children": [1], "translation": [0.5, -1.0, 2.0], "scale": [1.5, 1.5, 1.5]},
            {"name": "ball", "mesh": 0},
            {"name": "camera", "camera": 0, "translation": [0.0, 1.0, 6.0]},
        ],
        "cameras": [{"type": "perspective", "perspective": {"yfov": 0.9, "znear": 0.1}}],
        "meshes": [{"primitives": [
            {"attributes": {"POSITION": a_pos, "NORMAL": a_nrm16, "TEXCOORD_0": a_uv, "COLOR_0": a_col8}, "indices": a_i32},
            {"attributes": {"POSITION": a_pos, "NORMAL": a_nrm16, "COLOR_0": a_col16}, "indices": a_seq16},
            {"attributes": {"POSITION": a_pos, "TEXCOORD_0": a_uv}, "indices": a_seq32},
        ]}],
        "animations": [{"samplers": [{"input": a_time, "output": a_tr}, {"input": a_time, "output": a_rot}, {"input": a_time, "output": a_sc}],
                        "channels": [{"sampler": 0, "target": {"node": 1, "path": "translation"}}, {"sampler": 1, "target": {"node": 1, "path": "rotation"}},
                                     {"sampler": 2, "target": {"node": 1, "path": "scale"}}]}],
        "accessors": accessors,
        "bufferViews": views,
        "buffers": [{"byteLength": len(blob)}, {"byteLength": fallback_at[0], "extensions": {"EXT_meshopt_compression": {"fallback": True}}}],
    }
    return write_glb(doc, blob)


# ---- hostile edits: (name, file, edit(doc, blob), our status) -----------------------------------------------------------------
def _find(doc, mode, filt=None, stride=None):
    for i, v in enumerate(doc["bufferViews"]):
        e = meshopt_ext(v)
        if e and e["mode"] == mode and (filt is None or e.get("filter", "NONE") == filt) and (stride is None or e["byteStride"] == stride):
            return i, v, e
    raise LookupError((mode, filt, stride))


def _set(mode, key, value, filt=None, stride=None):
    def edit(doc, blob):
        _find(doc, mode, filt, stride)[2][key] = value

    return edit


def _outer(mode, key, fn, filt=None, stride=None):
    def edit(doc, blob):
        i, v, e = _find(doc, mode, filt, stride)
        v[key] = fn(v, e)

    return edit


def _restride(new_stride, count_fn, mode, filt=None, stride=None):
    def edit(doc, blob):
        i, v, e = _find(doc, mode, filt, stride)
        e["byteStride"], e["count"] = new_stride, count_fn(e["count"])
        v["byteLength"] = new_stride * e["count"]
        if "byteStride" in v:
            v["byteStride"] = new_stride

    return edit


def _stream_byte(mode, at, value, filt=None):
    def edit(doc, blob):
        e = _find(doc, mode, filt)[2]
        blob[e["byteOffset"] + at] = value

    return edit


def _flips(seed):
    def edit(doc, blob):
        rng = np.random.default_rng(seed)
        comp = [meshopt_ext(v) for v in doc["bufferViews"] if meshopt_ext(v)]
        e = comp[int(rng.integers(0, len(comp)))]
        for _ in range(3):
            k = e["byteOffset"] + int(rng.integers(0, e["byteLength"]))
            blob[k] ^= 1 << int(rng.integers(0, 8))

    return edit


def _uncompress(mode, filt):
    def edit(doc, blob):
        v = _find(doc, mode, filt)[1]
        del v["extensions"]

    return edit


def _unused_view(truncate):
    def edit(doc, blob):
        v = copy.deepcopy(_find(doc, "ATTRIBUTES", "OCTAHEDRAL")[1])
        meshopt_ext(v)["byteLength"] -= truncate
        doc["bufferViews"].append(v)

    return edit


def _rename_khr(doc, blob):
    for v in doc["bufferViews"] + doc["buffers"]:
        if "EXT_meshopt_compression" in v.get("extensions", {}):
            v["extensions"]["KHR_meshopt_compression"] = v["extensions"].pop("EXT_meshopt_compression")
    for key in ("extensionsUsed", "extensionsRequired"):
        if key in doc:
            doc[key] = ["KHR_meshopt_compression" if x == "EXT_meshopt_compression" else x for x in doc[key]]


def _source_outside(doc, blob):
    e = _find(doc, "ATTRIBUTES", "OCTAHEDRAL")[2]
    e["byteOffset"] = doc["buffers"][e["buffer"]]["byteLength"] - e["byteLength"] + 1


CORRUPT, UNSUPPORTED = -7, -6
BASE = "hierarchy_cc"
HOSTILE_EDITS = [
    ("source outside its buffer", BASE, _source_outside, CORRUPT),
    ("outer byteStride differs", BASE, _outer("ATTRIBUTES", "byteStride", lambda v, e: e["byteStride"] + 4, "NONE", 8), CORRUPT),
    ("outer byteLength is not stride * count", BASE, _outer("ATTRIBUTES", "byteLength", lambda v, e: v["byteLength"] - e["byteStride"], "NONE", 8), CORRUPT),
    ("invalid mode", BASE, _set("TRIANGLES", "mode", "POINTS"), CORRUPT),
    ("missing mode", BASE, lambda d, b: _find(d, "TRIANGLES")[2].pop("mode"), CORRUPT),
    ("ATTRIBUTES stride not a multiple of 4", BASE, _restride(6, lambda c: c, "ATTRIBUTES", "NONE", 8), CORRUPT),
    ("ATTRIBUTES stride above 256", BASE, _restride(260, lambda c: 1, "ATTRIBUTES", "NONE", 8), CORRUPT),
    ("TRIANGLES count not a multiple of 3", BASE, _restride(2, lambda c: c - 1, "TRIANGLES"), CORRUPT),
    ("index stride 8", BASE, _restride(8, lambda c: c // 12 * 3, "TRIANGLES"), CORRUPT),
    ("filter on an index view", BASE, _set("TRIANGLES", "filter", "OCTAHEDRAL"), CORRUPT),
    ("QUATERNION on stride 4", BASE, _set("ATTRIBUTES", "filter", "QUATERNION", "OCTAHEDRAL"), CORRUPT),
    ("COLOR on stride 12", BASE, _set("ATTRIBUTES", "filter", "COLOR", "EXPONENTIAL"), CORRUPT),
    ("OCTAHEDRAL on stride 12", BASE, _set("ATTRIBUTES", "filter", "OCTAHEDRAL", "EXPONENTIAL"), CORRUPT),
    ("truncated vertex stream", BASE, _outer("ATTRIBUTES", "extensions", lambda v, e: {"EXT_meshopt_compression": dict(e, byteLength=e["byteLength"] - 1)}, "OCTAHEDRAL"), CORRUPT),
    ("truncated index stream", BASE, _outer("TRIANGLES", "extensions", lambda v, e: {"EXT_meshopt_compression": dict(e, byteLength=e["byteLength"] - 1)}), CORRUPT),
    ("newer vertex codec version", BASE, _stream_byte("ATTRIBUTES", 0, 0xA2, "OCTAHEDRAL"), UNSUPPORTED),
    ("newer index codec version", BASE, _stream_byte("TRIANGLES", 0, 0xE2), UNSUPPORTED),
    ("fallback buffer read by an uncompressed view", BASE, _uncompress("ATTRIBUTES", "OCTAHEDRAL"), CORRUPT),
    ("corrupt stream in a view no primitive uses", BASE, _unused_view(1), CORRUPT),
    ("valid stream in a view no primitive uses", BASE, _unused_view(0), 0),
    ("KHR_meshopt_compression names", BASE, _rename_khr, 0),
    ("truncated index sequence", "synthetic", _outer("INDICES", "extensions", lambda v, e: {"EXT_meshopt_compression": dict(e, byteLength=e["byteLength"] - 5)}), CORRUPT),
    ("index sequence count too large", "synthetic", _restride(2, lambda c: c + 3, "INDICES"), CORRUPT),
] + [("bit flips %d" % k, BASE if k % 2 == 0 else "synthetic", _flips(k), None) for k in range(12)]


def apply_edit(name):
    """the bytes of HOSTILE_EDITS[name] applied to its committed base file"""
    for n, base, edit, _ in HOSTILE_EDITS:
        if n == name:
            doc, blob = read_glb(open(os.path.join(OUT, base + ".glb"), "rb").read())
            edit(doc, blob)
            return write_glb(doc, blob)
    raise KeyError(name)


# ---- the reference's loader -----------------------------------------------------------------------------------------------------
def reference_load(path, tmp):
    """(accepted, SceneCache of the raw cache or None) from the reference's loadScene via write_cache"""
    from niagara_b200 import scene_cache

    prefix = os.path.join(tmp, os.path.basename(path) + ".out")
    run = subprocess.run([os.path.join(REF_BIN, "write_cache"), prefix, path], capture_output=True, text=True)
    if run.returncode != 0:
        return False, None
    return True, scene_cache.SceneCache(prefix + ".raw.cache")


# the cooked Vertex[] of kitten is 150 KB per file: kept for kitten_cc only, the other three compare draws, animations and camera
WITHOUT_VERTICES = ("kitten_c", "kitten_ccvpf", "kitten_cz")


def expected_npz(path, out, tmp):
    ok, c = reference_load(path, tmp)
    assert ok, path
    cam, h = c.header.camera, c.header
    vertices = c.section("vertices")
    if os.path.basename(path)[:-4] in WITHOUT_VERTICES:
        vertices = vertices[:0]
    np.savez_compressed(
        out, draws=c.section("draws"), animations=c.section("animations"), keyframes=c.section("keyframes"),
        camera=np.array(list(cam.position) + list(cam.orientation) + [cam.fovY], np.float32), sun=np.array(list(h.sunDirection), np.float32),
        mesh_vertex_offset=c.section("meshes")["vertexOffset"], mesh_vertex_count=c.section("meshes")["vertexCount"], vertices=vertices,
    )
    c.close()


REQUIRED = {
    ("ATTRIBUTES", "NONE", 4), ("ATTRIBUTES", "NONE", 8), ("ATTRIBUTES", "NONE", 12), ("ATTRIBUTES", "OCTAHEDRAL", 4), ("ATTRIBUTES", "OCTAHEDRAL", 8),
    ("ATTRIBUTES", "QUATERNION", 8), ("ATTRIBUTES", "EXPONENTIAL", 12), ("ATTRIBUTES", "EXPONENTIAL", 16), ("ATTRIBUTES", "COLOR", 4), ("ATTRIBUTES", "COLOR", 8),
    ("TRIANGLES", "NONE", 2), ("TRIANGLES", "NONE", 4), ("INDICES", "NONE", 2), ("INDICES", "NONE", 4),
}


def main():
    sys.path.insert(0, ROOT)
    for d in ("", "refgltfpack"):
        subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle", d), "ref" if not d else "all"], check=True)
    os.makedirs(OUT, exist_ok=True)
    gltfpack = os.path.join(REF_BIN, "gltfpack")
    for name in fixture_names()[:-1]:
        src, mode = name.split("_", 1)
        flags = PACKED.get(mode) or LOSSLESS[mode]
        subprocess.run([gltfpack, "-i", sources()[src], "-o", os.path.join(OUT, name + ".glb")] + flags, check=True, capture_output=True)
    open(os.path.join(OUT, "synthetic.glb"), "wb").write(synthetic_glb())

    seen, total = set(), 0
    for name in fixture_names():
        data = open(os.path.join(OUT, name + ".glb"), "rb").read()
        total += len(data)
        seen |= combinations(read_glb(data)[0])
    assert {c[1:] for c in seen} >= REQUIRED, REQUIRED - {c[1:] for c in seen}
    assert {c[0] for c in seen} == set(EXTENSIONS)
    assert total < 1 << 20, total

    tmp = tempfile.mkdtemp()
    for name in fixture_names():
        expected_npz(os.path.join(OUT, name + ".glb"), os.path.join(OUT, name + "_expected.npz"), tmp)
    verdicts = {}
    for name, _, _, _ in HOSTILE_EDITS:
        path = os.path.join(tmp, "hostile.glb")
        open(path, "wb").write(apply_edit(name))
        verdicts[name] = reference_load(path, tmp)[0]
    with open(os.path.join(OUT, "hostile_verdicts.json"), "w") as f:
        json.dump(verdicts, f, indent=1, sort_keys=True)
        f.write("\n")
    print(len(fixture_names()), "files,", total, "bytes;", sorted(seen))
    print(verdicts)


if __name__ == "__main__":
    main()
