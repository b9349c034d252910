#!/usr/bin/env python3
"""Times nvc_cook_meshlets_clrt (the clrt cooker: each mesh's lodRT built with meshopt_buildMeshletsSpatial, meshletvtx0, the
other LODs as nvc_cook_meshlets) on the GPU against the reference's meshoptimizer (oracle/_ref/libmeshopt_cluster_ref.so) on
1 and 8 host threads, on three workloads:

  kitten        data/kitten.obj at max_scale 1: lodRT = LOD 3 (118 spatial meshlets), the other 7 LODs greedy
  kitten_rt0    the same with a max_scale that makes lodRT = LOD 0 (28 944 triangles built spatially)
  scene         a seeded scene of --meshes copies of the four fixture meshes with jittered positions, max_scale 1

Every GPU output (Mesh[], Meshlet[], meshletdata, meshletvtx0) is checked against the reference's in the same run.  GPU
times: CUDA events around the call (its synchronisations included), median of --iters calls after --warmup.  The reference's
time covers meshopt_buildMeshletsSpatial / meshopt_buildMeshlets and meshopt_optimizeMeshletLevel per LOD (through ctypes, one
LOD per task; ctypes releases the GIL), not its packing and bounds; the spatial builds alone are timed as well.  Prints the
card, its power limit and max SM clock.

Usage: python tools/cook_meshlets_clrt_bench.py [--iters 20] [--warmup 3] [--meshes 300] [--out results.json]"""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))


def ref_build(mo, job):
    """one LOD: the reference's builder for it, then meshopt_optimizeMeshletLevel per meshlet"""
    import test_cook_meshlets as base

    pos, idx, vertex_count, spatial = job
    n = len(idx)
    ml = (base.MeshoptMeshlet * max(mo.meshopt_buildMeshletsBound(n, 64, 24), 1))()
    mv = np.zeros(max(n, 1), np.uint32)
    mt = np.zeros(max(n, 1) + 4, np.uint8)
    if not n:
        return 0
    if spatial:
        count = mo.meshopt_buildMeshletsSpatial(ml, mv.ctypes.data, mt.ctypes.data, idx.ctypes.data, n, pos.ctypes.data, vertex_count, 12, 64, 24, 96, 0.5)
    else:
        count = mo.meshopt_buildMeshlets(ml, mv.ctypes.data, mt.ctypes.data, idx.ctypes.data, n, pos.ctypes.data, vertex_count, 12, 64, 96, 0.25)
    for k in range(count):
        m = ml[k]
        mo.meshopt_optimizeMeshletLevel(mv.ctypes.data + 4 * m.vertex_offset, m.vertex_count, mt.ctypes.data + m.triangle_offset, m.triangle_count, 1)
    return count


def ref_time(mo, jobs, threads):
    jobs = sorted(jobs, key=lambda j: -len(j[1]))
    t0 = time.perf_counter()
    if threads == 1:
        for job in jobs:
            ref_build(mo, job)
    else:
        with ThreadPoolExecutor(threads) as ex:
            list(ex.map(lambda job: ref_build(mo, job), jobs))
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--meshes", type=int, default=300)
    ap.add_argument("--out", help="also write the results as JSON here")
    args = ap.parse_args()

    import torch

    import cook_meshlets_bench
    import test_cook_meshlets as base
    import test_cook_meshlets_clrt as t

    assert torch.cuda.is_available(), "needs a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", smi)
    mo = t.meshopt()
    g = t.Gpu()
    rng = np.random.default_rng(2024)
    kv, ki, km = t.scene("kitten")[:3]
    sources = [base.scene(n)[:3] for n in ("kitten", "pirate", "pirateglb", "animated")]
    sv, si, sm = cook_meshlets_bench.jittered_scene(rng, sources, args.meshes)
    workloads = {"kitten": (kv, ki, km, np.ones(1, np.float32)), "kitten_rt0": (kv, ki, km, np.full(1, 1e9, np.float32)),
                 "scene": (sv, si, sm, np.ones(len(sm), np.float32))}
    results = {"card": smi}
    for name, (v, i, meshes, scale) in workloads.items():
        jobs = []
        for m, s in zip(meshes, scale):
            rt = t.lod_rt(m, s)
            vo, vc = int(m["vertexOffset"]), int(m["vertexCount"])
            pos = np.ascontiguousarray(base.dequantize(np.ascontiguousarray(v[vo: vo + vc, :3])))
            for l in range(int(m["lodCount"])):
                o, c = int(m["lods"][l]["indexOffset"]), int(m["lods"][l]["indexCount"])
                jobs.append((pos, np.ascontiguousarray(i[o: o + c], np.uint32), vc, l == rt))
        spatial = [j for j in jobs if j[3]]
        ref = {"ref_build_1thread_ms": ref_time(mo, jobs, 1), "ref_build_8threads_ms": ref_time(mo, jobs, 8),
               "ref_spatial_1thread_ms": ref_time(mo, spatial, 1), "ref_spatial_8threads_ms": ref_time(mo, spatial, 8)}
        want = t.reference_cook(mo, v, i, meshes, scale)
        got = g.cook_clrt(v, i, t.scrub(meshes), scale)
        t.assert_same(got, want, name)
        ml, words, vx = t.capacity(g.lib, meshes, scale)
        dv = torch.from_numpy(np.ascontiguousarray(v).view(np.uint8).reshape(-1).copy()).cuda()
        di = torch.from_numpy(np.ascontiguousarray(i, np.uint32).view(np.int32).copy()).cuda()
        dm = torch.zeros(len(meshes) * 208, dtype=torch.uint8, device="cuda")
        dl = torch.zeros(ml * 24, dtype=torch.uint8, device="cuda")
        dd = torch.zeros(words, dtype=torch.int32, device="cuda")
        dx = torch.zeros(vx, dtype=torch.int16, device="cuda")
        dt = torch.zeros(8, dtype=torch.int32, device="cuda")
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        times = []
        for it in range(args.warmup + args.iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.check(g.lib.nvc_cook_meshlets_clrt(g.ctx, stream, dv.data_ptr(), len(v), di.data_ptr(), len(i), meshes.ctypes.data, scale.ctypes.data, dm.data_ptr(),
                                                 len(meshes), dl.data_ptr(), ml, dd.data_ptr(), words, dx.data_ptr(), vx, dt.data_ptr()), g.ctx, "nvc_cook_meshlets_clrt")
            e1.record()
            torch.cuda.synchronize()
            if it >= args.warmup:
                times.append(e0.elapsed_time(e1))
        tt = dt.cpu().numpy().view(np.uint32)
        n, x = int(tt[0]), int(tt[4])
        assert dl.cpu().numpy()[: n * 24].tobytes() == got[1].tobytes() and dx.cpu().numpy().view(np.uint16)[:x].tobytes() == got[3].tobytes()
        rt_meshlets = sum(int(m["lods"][int(m["lodRT"])]["meshletCount"]) for m in got[0])
        r = {"meshes": len(meshes), "lods": int(meshes["lodCount"].sum()), "indices": int(meshes["lods"]["indexCount"].sum()),
             "rt_indices": int(sum(len(j[1]) for j in spatial)), "meshlets": n, "rt_meshlets": rt_meshlets, "gpu_ms_median": float(np.median(times)),
             "gpu_ms_min": float(np.min(times)), **ref, "identical": True}
        print(name, json.dumps(r))
        results[name] = r
    g.close()
    if args.out:
        json.dump(results, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
