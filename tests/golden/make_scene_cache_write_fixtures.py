#!/usr/bin/env python3
"""Regenerates scene_cache_write_raw.npz: the uncompressed caches the REFERENCE's writer makes in the same runs that wrote the
committed compressed caches, so that nvc_scene_cache_write can be checked to turn the one into the other byte for byte
(tests/test_scene_cache_write.py).  The reference's own importer, cooker and saveSceneCache run through oracle/_ref/write_cache
and oracle/_ref/write_cache_clrt (built by `make -C oracle ref` and `make -C oracle/refscene_clrt` from the reference checkout
named by NIAGARA_REFERENCE):

  kitten         data/kitten.obj                           -> kitten.raw.cache          (same run: kitten.z.cache)
  pirateglb      extern/meshoptimizer/demo/pirate.glb      -> pirateglb.raw.cache       (same run: pirateglb.z.cache)
  animated_clrt  tests/golden/animated.gltf, clrtMode = 1  -> animated_clrt.raw.cache   (same run: animated_clrt.z.cache)

each stored whole as one uint8 array (the npz is deflated).  animated.raw.cache is already committed.  Every compressed cache
of these runs must equal its committed counterpart byte for byte; the script stops otherwise, and changes no committed cache.

Run: NIAGARA_REFERENCE=/path/to/niagara python tests/golden/make_scene_cache_write_fixtures.py"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def main():
    ref_dir = os.path.abspath(os.environ["NIAGARA_REFERENCE"])
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "ref", "REF=" + ref_dir], check=True)
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle", "refscene_clrt"), "REF=" + ref_dir], check=True)
    tools = os.path.join(ROOT, "oracle", "_ref")
    demo = os.path.join(ref_dir, "extern", "meshoptimizer", "demo")
    runs = [
        ("kitten", "write_cache", os.path.join(ref_dir, "data", "kitten.obj"), "kitten.z.cache"),
        ("pirateglb", "write_cache", os.path.join(demo, "pirate.glb"), "pirateglb.z.cache"),
        ("animated_clrt", "write_cache_clrt", os.path.join(HERE, "animated.gltf"), "animated_clrt.z.cache"),
        ("animated", "write_cache", os.path.join(HERE, "animated.gltf"), "animated.z.cache"),
    ]
    raw = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, tool, src, committed in runs:
            prefix = os.path.join(tmp, name)
            subprocess.run([os.path.join(tools, tool), prefix, src], check=True, stdout=subprocess.DEVNULL)
            z = open(prefix + ".z.cache", "rb").read()
            if z != open(os.path.join(HERE, committed), "rb").read():
                sys.exit("%s: the reference's compressed cache differs from the committed %s" % (name, committed))
            r = open(prefix + ".raw.cache", "rb").read()
            if name == "animated":
                if r != open(os.path.join(HERE, "animated.raw.cache"), "rb").read():
                    sys.exit("animated: the reference's raw cache differs from the committed animated.raw.cache")
                continue
            raw[name] = np.frombuffer(r, np.uint8)
    np.savez_compressed(os.path.join(HERE, "scene_cache_write_raw.npz"), **raw)
    print({k: len(v) for k, v in raw.items()})


if __name__ == "__main__":
    main()
