#!/usr/bin/env python3
"""Regenerates pirate_vertices.npz, the one input of the reference's LOD chain for pirate.obj (the meshoptimizer demo's) that
no other fixture holds: its processed Vertex[] with normals (meshlet_cook.npz keeps the index buffer and Mesh[], pirate_cook.npz
only the fp16 positions).  Taken from the uncompressed cache the REFERENCE's own importer and cooker write
(oracle/_ref/write_cache, built by `make -C oracle ref` from the reference checkout named by NIAGARA_REFERENCE), and checked
against the fixtures above:

  pirate_vertices     uint16 (n, 8), the Vertex[] (vx, vy, vz, tp, np low, np high, tu, tv)

Run: NIAGARA_REFERENCE=/path/to/niagara python tests/golden/make_lod_fixtures.py"""
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
    cook = np.load(os.path.join(HERE, "meshlet_cook.npz"))
    positions = np.load(os.path.join(HERE, "pirate_cook.npz"))["pirate_positions"]
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run([tool, os.path.join(tmp, "pirate"), os.path.join(ref_dir, "extern", "meshoptimizer", "demo", "pirate.obj")], check=True, stdout=subprocess.DEVNULL)
        c = scene_cache.SceneCache(os.path.join(tmp, "pirate.raw.cache"))
        assert not c.header.compressed
        vertices = c.section("vertices").view(np.uint16).reshape(-1, 8).copy()
        assert np.array_equal(vertices[:, :3], positions)
        assert np.array_equal(c.section("indices").astype(np.uint32), cook["pirate_indices"])
        assert np.array_equal(c.section("meshes").view(np.uint8).reshape(-1, 208), cook["pirate_meshes"])
        assert (c.section("meshes").view(layout.MESH_DTYPE)["vertexCount"] == len(vertices)).all()
    np.savez_compressed(os.path.join(HERE, "pirate_vertices.npz"), pirate_vertices=vertices)
    print("pirate", len(vertices), "vertices")


if __name__ == "__main__":
    main()
