#!/usr/bin/env python3
"""Regenerates obj_vertices.npz: the Vertex[] the REFERENCE's loadObj makes of data/kitten.obj and of the meshoptimizer demo's
pirate.obj, the input of appendMesh's vertex processing (oracle/_ref/load_obj, built by oracle/refobj's Makefile from the
reference checkout named by NIAGARA_REFERENCE).  loadObj writes one record per triangle corner; each file is stored as its
distinct 16-byte records and one record index per corner:

  <name>_records   uint16 (r, 8), the distinct Vertex records (vx, vy, vz, tp, np low, np high, tu, tv), sorted by bytes
  <name>_corners   uint32 (n,), per corner its record: records[corners] is loadObj's array

The generator checks that the expansion is exact, and that the reference's own meshoptimizer (oracle/_ref/
libmeshopt_full_ref.so) running scene.cpp:172-184 on it (tests/test_cook_vertices.py's ref_vertices) gives the Vertex[] and LOD 0
the reference's cooker stored for the same file (scene_cache_write_raw.npz's kitten, meshlet_cook.npz / pirate_vertices.npz).

Run: NIAGARA_REFERENCE=/path/to/niagara python tests/golden/make_vertex_fixtures.py"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))


def main():
    import test_cook_lods as lods_tests
    import test_cook_vertices as vertex_tests

    ref_dir = os.path.abspath(os.environ["NIAGARA_REFERENCE"])
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle", "refobj"), "REF=" + ref_dir], check=True)
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle", "refgltfpack"), "REF=" + ref_dir], check=True)
    tool = os.path.join(ROOT, "oracle", "_ref", "load_obj")
    sources = {"kitten": os.path.join(ref_dir, "data", "kitten.obj"), "pirate": os.path.join(ref_dir, "extern", "meshoptimizer", "demo", "pirate.obj")}
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, path in sources.items():
            raw = os.path.join(tmp, name + ".bin")
            subprocess.run([tool, path, raw], check=True)
            loaded = np.fromfile(raw, np.uint16).reshape(-1, 8)
            records, corners = np.unique(loaded.view(np.uint8).reshape(-1, 16), axis=0, return_inverse=True)
            records = np.ascontiguousarray(records).view(np.uint16).reshape(-1, 8)
            corners = corners.reshape(-1).astype(np.uint32)
            assert np.array_equal(records[corners], loaded), name
            # the reference's steps 1-5 on it give what its cooker stored
            v, ib, meshes, _ = lods_tests.fixture(name)
            lod = meshes[0]["lods"][0]
            want_lod0 = ib[int(lod["indexOffset"]): int(lod["indexOffset"]) + int(lod["indexCount"])]
            got_v, got_i = vertex_tests.ref_vertices(loaded, np.arange(len(loaded), dtype=np.uint32))
            assert np.array_equal(got_v, v) and np.array_equal(got_i, want_lod0), name
            out[name + "_records"], out[name + "_corners"] = records, corners
            print(name, len(loaded), "corners,", len(records), "records ->", len(got_v), "vertices,", len(got_i), "LOD 0 indices")
    np.savez_compressed(os.path.join(HERE, "obj_vertices.npz"), **out)


if __name__ == "__main__":
    main()
