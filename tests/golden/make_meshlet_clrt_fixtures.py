#!/usr/bin/env python3
"""Regenerates meshlet_cook_clrt.npz and animated_clrt.z.cache: what the REFERENCE's cooker stores in a clrt build (CLRT=1),
with its own importer and cooker (oracle/_ref/write_cache_clrt, built by `make -C oracle/refscene_clrt` from the reference
checkout named by NIAGARA_REFERENCE; see oracle/refscene_clrt/write_cache_clrt.cpp).  For kitten (data/kitten.obj), pirate (the meshoptimizer
demo's pirate.obj), pirateglb (its pirate.glb) and animated (animated.gltf), from the uncompressed caches:

  <name>_meshes       Mesh[] as bytes (208 per mesh), lodRT included
  <name>_meshlets     Meshlet[] as bytes (24 per meshlet)
  <name>_meshletdata  uint32
  <name>_meshletvtx0  uint16, 4 per vertex of every meshlet of each mesh's lodRT
  <name>_max_scale    float32 per mesh: the maxScale appendMesh received (1 for .obj; for glTF loadScene's meshScale,
                      scene.cpp:502-519: nvc_gltf_scene_arrays' mesh_scale, or, for pirate.glb, whose EXT_meshopt_compression
                      the importer does not read, recomputed from its node transform in float32), checked to give the
                      reference's lodRT

The vertices, indices and LOD errors do not depend on clrt: they are checked equal to the default build's fixtures
(kitten_cook.npz, pirate_cook.npz, meshlet_cook.npz, animated.raw.cache), which the tests read them from.

animated_clrt.z.cache is the compressed cache of animated.gltf written with clrtMode = 1, for the scene-cache reader.

Run: NIAGARA_REFERENCE=/path/to/niagara python tests/golden/make_meshlet_clrt_fixtures.py"""
import json
import os
import shutil
import struct
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def lod_rt(mesh, max_scale):
    """scene.cpp:266-268 with float32 arithmetic"""
    rt = 0
    for i in range(int(mesh["lodCount"])):
        if np.float32(mesh["lods"][i]["error"]) * np.float32(max_scale) < np.float32(3e-3):
            rt = i
    return rt


def gltf_json(path):
    data = open(path, "rb").read()
    if data[:4] == b"glTF":
        return json.loads(data[20: 20 + struct.unpack("<I", data[12:16])[0]])
    return json.loads(data)


def node_matrix(node):
    """the node's local transform, column-major as cgltf (translation * rotation * scale)"""
    if "matrix" in node:
        return np.asarray(node["matrix"], np.float32).reshape(4, 4).T
    x, y, z, w = (np.float32(c) for c in node.get("rotation", [0, 0, 0, 1]))
    r = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], np.float32)
    m = np.eye(4, dtype=np.float32)
    m[:3, :3] = r * np.asarray(node.get("scale", [1, 1, 1]), np.float32)[None, :]
    m[:3, 3] = node.get("translation", [0, 0, 0])
    return m


def gltf_mesh_scale(path):
    """meshScale per reference mesh (one per triangle primitive, in mesh then primitive order)"""
    j = gltf_json(path)
    nodes = j.get("nodes", [])
    parent = {c: i for i, n in enumerate(nodes) for c in n.get("children", [])}
    scale = np.ones(len(j["meshes"]), np.float32)
    for i, n in enumerate(nodes):
        if "mesh" not in n:
            continue
        m, k = node_matrix(n), i
        while k in parent:
            k = parent[k]
            m = node_matrix(nodes[k]) @ m
        xf = m.T.reshape(-1)  # cgltf's column-major array
        det = xf[0] * (xf[5] * xf[10] - xf[9] * xf[6]) - xf[1] * (xf[4] * xf[10] - xf[6] * xf[8]) + xf[2] * (xf[4] * xf[9] - xf[5] * xf[8])
        scale[n["mesh"]] = max(scale[n["mesh"]], abs(np.cbrt(np.float32(det))))
    return np.concatenate([np.full(sum(p.get("mode", 4) == 4 for p in mesh["primitives"]), s, np.float32) for mesh, s in zip(j["meshes"], scale)])


def main():
    from niagara_b200 import gltf, layout, scene_cache

    ref_dir = os.environ["NIAGARA_REFERENCE"]
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle", "refscene_clrt"), "REF=" + os.path.abspath(ref_dir)], check=True)
    tool = os.path.join(ROOT, "oracle", "_ref", "write_cache_clrt")
    demo = os.path.join(ref_dir, "extern", "meshoptimizer", "demo")
    sources = {"kitten": os.path.join(ref_dir, "data", "kitten.obj"), "pirate": os.path.join(demo, "pirate.obj"), "pirateglb": os.path.join(demo, "pirate.glb"),
               "animated": os.path.join(HERE, "animated.gltf")}
    default = np.load(os.path.join(HERE, "meshlet_cook.npz"))
    kitten = np.load(os.path.join(HERE, "kitten_cook.npz"))
    pirate = np.load(os.path.join(HERE, "pirate_cook.npz"))
    animated = scene_cache.SceneCache(os.path.join(HERE, "animated.raw.cache"))
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, src in sources.items():
            subprocess.run([tool, os.path.join(tmp, name), src], check=True, stdout=subprocess.DEVNULL)
            c = scene_cache.SceneCache(os.path.join(tmp, name + ".raw.cache"))
            assert not c.header.compressed and c.header.clrtMode == 1
            positions = c.section("vertices").view(np.uint16).reshape(-1, 8)[:, :3]
            indices = c.section("indices").astype(np.uint32)
            meshes = c.section("meshes").copy()
            if name == "animated":
                want_pos, want_idx, want_meshes = animated.section("vertices").view(np.uint16).reshape(-1, 8)[:, :3], animated.section("indices"), animated.section("meshes")
            else:
                want_pos = kitten["positions"] if name == "kitten" else pirate[name + "_positions"]
                want_idx = default[name + "_indices"]
                want_meshes = default[name + "_meshes"].reshape(-1).view(layout.MESH_DTYPE)
            # the LOD chain does not depend on clrt
            assert np.array_equal(positions, want_pos) and np.array_equal(indices, want_idx), name
            for field in ("center", "radius", "vertexOffset", "vertexCount", "lodCount"):
                assert np.array_equal(meshes[field], want_meshes[field]), (name, field)
            for field in ("indexOffset", "indexCount", "error"):
                assert np.array_equal(meshes["lods"][field], want_meshes["lods"][field]), (name, field)
            if src.endswith((".gltf", ".glb")):
                if name == "animated":
                    g = gltf.GltfScene(src)
                    scale = g.mesh_scale.copy()
                    g.close()
                else:
                    scale = gltf_mesh_scale(src)
            else:
                scale = np.ones(len(meshes), np.float32)
            assert len(scale) == len(meshes), name
            assert [lod_rt(m, s) for m, s in zip(meshes, scale)] == [int(x) for x in meshes["lodRT"]], name
            out[name + "_meshes"] = meshes.view(np.uint8).reshape(-1, 208)
            out[name + "_meshlets"] = c.section("meshlets").view(np.uint8).reshape(-1, 24)
            out[name + "_meshletdata"] = c.section("meshletdata").view(np.uint32)
            out[name + "_meshletvtx0"] = c.section("meshletvtx0").view(np.uint16)
            out[name + "_max_scale"] = scale
            print(name, "lodRT", [int(x) for x in meshes["lodRT"]], len(out[name + "_meshlets"]), "meshlets", len(out[name + "_meshletvtx0"]), "meshletvtx0")
            if name == "animated":
                shutil.copyfile(os.path.join(tmp, name + ".z.cache"), os.path.join(HERE, "animated_clrt.z.cache"))
    np.savez_compressed(os.path.join(HERE, "meshlet_cook_clrt.npz"), **out)


if __name__ == "__main__":
    main()
