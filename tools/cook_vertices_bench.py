#!/usr/bin/env python3
"""Times nvc_cook_mesh_vertices (appendMesh's vertex processing: index filtering, vertex de-duplication, vertex cache and fetch
ordering) on the GPU against the reference's meshoptimizer (oracle/_ref/libmeshopt_full_ref.so, driven by
tests/test_cook_vertices.py's ref_vertices) on one and on 8 host threads, on two workloads:

  kitten    loadObj's output for kitten.obj: one mesh, 86 832 corners; the vertex cache pass is one sequential CTA
  scene     --copies meshes cycling through kitten.obj, pirate.obj and animated.gltf's primitives, positions jittered

Every GPU output is checked against the reference's in the same run.  GPU times: CUDA events around the call (its
synchronisations included), median of --iters calls after --warmup.  Then, in a pass of its own after the timed one,
torch.profiler gives each kernel's share over --iters calls.  The reference's time covers ref_vertices per mesh: the library
calls (which release the GIL, so the 8 threads run them side by side) and the numpy copies around them.  Prints the card, its
power limit and max SM clock.

Usage: python tools/cook_vertices_bench.py [--iters 20] [--warmup 2] [--copies 300] [--out results.json]"""
import argparse
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


def jittered_scene(t, copies, seed=1):
    import test_cook_lods as lods_tests

    rng = np.random.default_rng(seed)
    v, ix, m = t.gltf_input("animated.gltf")
    sources = [t.obj_input("kitten"), t.obj_input("pirate")]
    for mesh in m:
        vo, vc = int(mesh["vertexOffset"]), int(mesh["vertexCount"])
        io, ic = int(mesh["lods"][0]["indexOffset"]), int(mesh["lods"][0]["indexCount"])
        sources.append((v[vo: vo + vc], ix[io: io + ic]))
    parts = []
    for k in range(copies):
        sv, si = sources[k % len(sources)]
        part = sv.copy()
        pos = part[:, :3].view(np.float16).astype(np.float32)
        pos = pos * rng.uniform(0.5, 2.0) + rng.uniform(-100, 100, (1, 3)).astype(np.float32) + rng.normal(0, 1e-3, pos.shape).astype(np.float32)
        part[:, :3] = pos.astype(np.float16).view(np.uint16)
        parts.append((part, si))
    return lods_tests.scene_of(parts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--copies", type=int, default=300)
    ap.add_argument("--out", help="also write the results as JSON here")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import test_cook_vertices as t

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", card)
    gpu = t.Gpu()
    v, ix = t.obj_input("kitten")
    workloads = {"kitten": t.lods_tests.scene_of([(v, ix)]), "scene": jittered_scene(t, args.copies)}
    results = {"card": card}
    for name, (v, i, m) in workloads.items():
        lib = gpu.lib
        dv = torch.from_numpy(np.ascontiguousarray(v).view(np.uint8).reshape(-1).copy()).cuda()
        di = torch.from_numpy(np.ascontiguousarray(i, np.uint32).view(np.int32).copy()).cuda()
        dm = torch.zeros(len(m) * 208, dtype=torch.uint8, device="cuda")
        dov = torch.zeros(len(v) * 16, dtype=torch.uint8, device="cuda")
        doi = torch.zeros(len(i), dtype=torch.int32, device="cuda")
        dt = torch.zeros(4, dtype=torch.int32, device="cuda")

        def call():
            gpu.check(lib.nvc_cook_mesh_vertices(gpu.ctx, None, dv.data_ptr(), len(v), di.data_ptr(), len(i), m.ctypes.data, len(m), dm.data_ptr(), dov.data_ptr(), len(v),
                                                 doi.data_ptr(), len(i), dt.data_ptr()), gpu.ctx, "nvc_cook_mesh_vertices")

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
        got = (dm.cpu().numpy().view(t.layout.MESH_DTYPE), dov.cpu().numpy().view(np.uint16).reshape(-1, 8)[: int(totals[0])],
               doi.cpu().numpy().view(np.uint32)[: int(totals[1])], totals)

        # per-kernel split, profiler on, in a pass of its own
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                call()
            torch.cuda.synchronize()
        split = {}
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            if us > 0:
                split[e.key] = round(us / 1e3 / args.iters, 4)
        split = dict(sorted(split.items(), key=lambda kv: -kv[1]))

        def ref(threads):
            def one(k):
                return t.ref_scene(v, i, m[k: k + 1])
            t0 = time.perf_counter()
            with ThreadPoolExecutor(threads) as ex:
                list(ex.map(one, range(len(m))))
            return time.perf_counter() - t0

        ref1, ref8 = ref(1), ref(8)
        t.assert_same(got, t.ref_scene(v, i, m), name)
        row = dict(meshes=len(m), input_indices=len(i), vertices_out=int(totals[0]), lod0_indices=int(totals[1]), gpu_ms=float(np.median(times)),
                   gpu_ms_min=float(np.min(times)), ref_1_thread_ms=ref1 * 1e3, ref_8_threads_ms=ref8 * 1e3, equal=True, kernel_ms_per_call=split)
        results[name] = row
        print(name, json.dumps(row))
    gpu.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
