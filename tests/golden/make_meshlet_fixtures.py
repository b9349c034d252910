#!/usr/bin/env python3
"""Regenerates meshlet_cook.npz, the inputs of the reference's meshlet cooker that nvc_cook_meshlets needs, with the
REFERENCE's own importer and cooker (oracle/_ref/write_cache, built by `make -C oracle ref` from the reference checkout named
by NIAGARA_REFERENCE; see oracle/refscene/write_cache.cpp).  For kitten (data/kitten.obj), pirate (the meshoptimizer demo's
pirate.obj) and pirateglb (its pirate.glb), taken from the uncompressed caches (the index codec of a compressed cache rotates
triangles, so only the raw cache holds the index order the cooker saw):

  <name>_indices      uint32, the cooked index buffer (mesh-local indices of every LOD)
  <name>_meshes       Mesh[] as bytes (208 per mesh)

What the other fixtures already hold is not repeated; it is checked against the same caches here: the fp16 positions and
meshletdata (kitten_cook.npz, pirate_cook.npz), and Meshlet[] (kitten.nvcg, pirate_cook.npz).

Run: NIAGARA_REFERENCE=/path/to/niagara python tests/golden/make_meshlet_fixtures.py"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def main():
    from niagara_b200 import layout, scene_cache

    ref_dir = os.environ["NIAGARA_REFERENCE"]
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "ref", "REF=" + os.path.abspath(ref_dir)], check=True)
    tool = os.path.join(ROOT, "oracle", "_ref", "write_cache")
    demo = os.path.join(ref_dir, "extern", "meshoptimizer", "demo")
    sources = {"kitten": os.path.join(ref_dir, "data", "kitten.obj"), "pirate": os.path.join(demo, "pirate.obj"), "pirateglb": os.path.join(demo, "pirate.glb")}
    kitten = np.load(os.path.join(HERE, "kitten_cook.npz"))
    pirate = np.load(os.path.join(HERE, "pirate_cook.npz"))
    positions = {"kitten": kitten["positions"], "pirate": pirate["pirate_positions"], "pirateglb": pirate["pirateglb_positions"]}
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, src in sources.items():
            subprocess.run([tool, os.path.join(tmp, name), src], check=True, stdout=subprocess.DEVNULL)
            c = scene_cache.SceneCache(os.path.join(tmp, name + ".raw.cache"))
            assert not c.header.compressed
            vertices = c.section("vertices").view(np.uint16).reshape(-1, 8)
            assert np.array_equal(vertices[:, :3], positions[name]), name
            out[name + "_indices"] = c.section("indices").astype(np.uint32)
            out[name + "_meshes"] = c.section("meshes").view(np.uint8).reshape(-1, 208)
            meshlets = c.section("meshlets").view(np.uint8).reshape(-1, 24)
            assert np.array_equal(c.section("meshletdata").view(np.uint32), kitten["meshletdata"] if name == "kitten" else pirate[name + "_meshletdata"]), name
            want = layout.load_nvcg(os.path.join(HERE, "kitten.nvcg"))[1].view(np.uint8).reshape(-1, 24) if name == "kitten" else pirate[name + "_meshlets"]
            assert np.array_equal(meshlets, want), name
            print(name, len(out[name + "_indices"]), "indices", len(out[name + "_meshes"]), "meshes", len(meshlets), "meshlets")
    np.savez_compressed(os.path.join(HERE, "meshlet_cook.npz"), **out)


if __name__ == "__main__":
    main()
