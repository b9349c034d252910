#!/usr/bin/env python3
"""Times nvc_cook_mesh_lods (appendMesh's LOD chain: simplification and vertex cache optimisation per LOD) on the GPU against
the reference's meshoptimizer (oracle/_ref/libmeshopt_simplify_ref.so, driven by tests/test_cook_lods.py's ref_chain) on one
and on 8 host threads, on two workloads:

  kitten    the Vertex[] and LOD 0 the reference's cooker started from: one mesh, 86 832 LOD 0 indices; one sequential CTA
  scene     300 copies of the fixture meshes (kitten, pirate.obj, pirate.glb, animated.gltf's two), positions jittered: throughput

Every GPU output is checked against the reference's in the same run.  GPU times: CUDA events around the call (its
synchronisations included), median of --iters calls after --warmup.  The reference's time covers its whole chain per mesh:
the library calls (which release the GIL, so the 8 threads run them side by side) and ref_chain's numpy work around them
(dequantisation, normal decoding, center and radius as whole-array operations).  Prints the card, its power limit and max SM
clock.

Usage: python tools/cook_lods_bench.py [--iters 20] [--warmup 2] [--copies 300]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--copies", type=int, default=300)
    ap.add_argument("--out", help="also write the results as JSON here")
    args = ap.parse_args()

    import torch

    import test_cook_lods as t

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", card)
    gpu = t.Gpu()
    v, ib, meshes, _ = t.fixture("kitten")
    workloads = {"kitten": (v, ib, t.lod0_input(meshes)), "scene": t.jittered_fixture_scene(args.copies)}
    results = {"card": card}
    for name, (v, i, m) in workloads.items():
        lib = gpu.lib
        cap = t.capacity(lib, m)
        dv = torch.from_numpy(np.ascontiguousarray(v).view(np.uint8).reshape(-1).copy()).cuda()
        di = torch.from_numpy(np.ascontiguousarray(i, np.uint32).view(np.int32).copy()).cuda()
        dm = torch.zeros(len(m) * 208, dtype=torch.uint8, device="cuda")
        dib = torch.zeros(cap + 1, dtype=torch.int32, device="cuda")
        dt = torch.zeros(4, dtype=torch.int32, device="cuda")

        def call():
            gpu.check(lib.nvc_cook_mesh_lods(gpu.ctx, None, dv.data_ptr(), len(v), di.data_ptr(), len(i), m.ctypes.data, None, len(m), dm.data_ptr(), dib.data_ptr(), cap, dt.data_ptr()),
                      gpu.ctx, "nvc_cook_mesh_lods")

        for _ in range(args.warmup):
            call()
        times = []
        for _ in range(args.iters):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            call()
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        totals = dt.cpu().numpy().view(np.uint32)
        got = (dm.cpu().numpy().view(t.layout.MESH_DTYPE), dib.cpu().numpy().view(np.uint32)[: int(totals[0])], totals)

        def ref(threads):
            def one(k):
                return t.ref_scene(v, i, m[k: k + 1])
            t0 = time.perf_counter()
            with ThreadPoolExecutor(threads) as ex:
                parts = list(ex.map(one, range(len(m))))
            return time.perf_counter() - t0, parts

        ref1, _ = ref(1)
        ref8, _ = ref(8)
        want = t.ref_scene(v, i, m)
        t.assert_same(got, want, name)
        row = dict(meshes=len(m), lod0_indices=int(m["lods"]["indexCount"][:, 0].sum()), chain_indices=int(totals[0]), gpu_ms=float(np.median(times)),
                   gpu_ms_min=float(np.min(times)), ref_1_thread_ms=ref1 * 1e3, ref_8_threads_ms=ref8 * 1e3, equal=True)
        results[name] = row
        print(name, json.dumps(row))
    gpu.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
