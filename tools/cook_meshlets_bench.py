#!/usr/bin/env python3
"""Times nvc_cook_meshlets (meshlet building, optimisation, packing and bounds) on the GPU against the reference's
meshoptimizer (oracle/_ref/libmeshopt_cluster_ref.so: meshopt_buildMeshlets + meshopt_optimizeMeshletLevel +
meshopt_computeMeshletBounds and appendMeshlet's packing) on one host thread and on all host cores, on two workloads:

  kitten    data/kitten.obj as the reference cooked it: one mesh, 8 LODs, 213 414 indices; the longest job decides
  scene     a seeded scene of ~2000 meshes, copies of the four fixture meshes with jittered positions: throughput

Every GPU output is checked against the reference's in the same run.  GPU times: CUDA events around the call (its
synchronisations included), median of --iters calls after --warmup.  The reference's time covers meshopt_buildMeshlets
and meshopt_optimizeMeshletLevel only (called through ctypes), not its packing and bounds.  Prints the card, its power limit and max SM clock.

Usage: python tools/cook_meshlets_bench.py [--iters 20] [--warmup 3] [--meshes 2000]"""
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


def jittered_scene(rng, sources, count):
    verts, idx, meshes = [], [], []
    vbase = ibase = 0
    for k in range(count):
        v, i, m = sources[k % len(sources)]
        for mi in range(len(m)):
            mesh = m[mi: mi + 1].copy()
            vo, vc = int(mesh["vertexOffset"][0]), int(mesh["vertexCount"][0])
            part = v[vo: vo + vc].copy()
            pos = part[:, :3].view(np.float16).astype(np.float32)
            pos = pos * rng.uniform(0.5, 2.0) + rng.uniform(-100, 100, (1, 3)).astype(np.float32) + rng.normal(0, 1e-3, pos.shape).astype(np.float32)
            part[:, :3] = pos.astype(np.float16).view(np.uint16)
            lo = int(mesh["lods"][0, : int(mesh["lodCount"][0])]["indexOffset"].min())
            hi = int((mesh["lods"][0]["indexOffset"] + mesh["lods"][0]["indexCount"])[: int(mesh["lodCount"][0])].max())
            mesh["vertexOffset"] = vbase
            mesh["lods"]["indexOffset"] += np.uint32(ibase - lo)
            verts.append(part)
            idx.append(i[lo:hi])
            vbase += vc
            ibase += hi - lo
            meshes.append(mesh)
            if len(meshes) >= count:
                return np.concatenate(verts), np.concatenate(idx), np.concatenate(meshes)
    return np.concatenate(verts), np.concatenate(idx), np.concatenate(meshes)


def ref_build(mo, pos, idx, vertex_count):
    n = len(idx)
    ml = (t_module().MeshoptMeshlet * max(mo.meshopt_buildMeshletsBound(n, 64, 96), 1))()
    mv = np.zeros(max(n, 1), np.uint32)
    mt = np.zeros(max(n, 1) + 4, np.uint8)
    count = mo.meshopt_buildMeshlets(ml, mv.ctypes.data, mt.ctypes.data, idx.ctypes.data, n, pos.ctypes.data, vertex_count, 12, 64, 96, 0.25) if n else 0
    for k in range(count):
        m = ml[k]
        mo.meshopt_optimizeMeshletLevel(mv.ctypes.data + 4 * m.vertex_offset, m.vertex_count, mt.ctypes.data + m.triangle_offset, m.triangle_count, 1)
    return count


def t_module():
    import test_cook_meshlets

    return test_cook_meshlets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--meshes", type=int, default=2000)
    ap.add_argument("--out", help="also write the results as JSON here")
    args = ap.parse_args()

    import torch

    import test_cook_meshlets as t

    assert torch.cuda.is_available(), "needs a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", smi)
    mo = t.meshopt()
    g = t.Gpu()
    rng = np.random.default_rng(2024)
    kitten = t.scene("kitten")[:3]
    sources = [t.scene(n)[:3] for n in ("kitten", "pirate", "pirateglb", "animated")]
    workloads = {"kitten": kitten, "scene": jittered_scene(rng, sources, args.meshes)}
    results = {"card": smi}
    for name, (v, i, meshes) in workloads.items():
        lods = int(meshes["lodCount"].sum())
        # reference: meshopt_buildMeshlets + meshopt_optimizeMeshletLevel per LOD (the packing and bounds are left out of
        # its time), on one thread and on all cores (one LOD per task; ctypes releases the GIL)
        jobs = []
        for m in meshes:
            vo, vc = int(m["vertexOffset"]), int(m["vertexCount"])
            pos = np.ascontiguousarray(t.dequantize(np.ascontiguousarray(v[vo: vo + vc, :3])))
            for l in range(int(m["lodCount"])):
                o, c = int(m["lods"][l]["indexOffset"]), int(m["lods"][l]["indexCount"])
                jobs.append((pos, np.ascontiguousarray(i[o: o + c], np.uint32), vc))
        t0 = time.perf_counter()
        for job in jobs:
            ref_build(mo, *job)
        ref1 = time.perf_counter() - t0
        cores = os.cpu_count()
        with ThreadPoolExecutor(cores) as ex:
            t0 = time.perf_counter()
            list(ex.map(lambda job: ref_build(mo, *job), sorted(jobs, key=lambda j: -len(j[1]))))
            refn = time.perf_counter() - t0
        want = t.reference_cook(mo, v, i, meshes)
        # GPU
        got = g.cook(v, i, t.scrub(meshes))
        t.assert_same(got, want, name)
        ml, words = t.capacity(g.lib, meshes)
        dv = torch.from_numpy(np.ascontiguousarray(v).view(np.uint8).reshape(-1).copy()).cuda()
        di = torch.from_numpy(np.ascontiguousarray(i, np.uint32).view(np.int32).copy()).cuda()
        dm = torch.zeros(len(meshes) * 208, dtype=torch.uint8, device="cuda")
        dl = torch.zeros(ml * 24, dtype=torch.uint8, device="cuda")
        dd = torch.zeros(words, dtype=torch.int32, device="cuda")
        dt = torch.zeros(4, dtype=torch.int32, device="cuda")
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        times = []
        for it in range(args.warmup + args.iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.check(g.lib.nvc_cook_meshlets(g.ctx, stream, dv.data_ptr(), len(v), di.data_ptr(), len(i), meshes.ctypes.data, dm.data_ptr(), len(meshes), dl.data_ptr(), ml,
                                            dd.data_ptr(), words, dt.data_ptr()), g.ctx, "nvc_cook_meshlets")
            e1.record()
            torch.cuda.synchronize()
            if it >= args.warmup:
                times.append(e0.elapsed_time(e1))
        n = int(dt.cpu()[0])
        assert dl.cpu().numpy()[: n * 24].tobytes() == got[1].tobytes()
        r = {"meshes": len(meshes), "lods": lods, "indices": int(meshes["lods"]["indexCount"].sum()), "meshlets": n, "gpu_ms_median": float(np.median(times)),
             "gpu_ms_min": float(np.min(times)), "ref_build_1thread_ms": ref1 * 1e3, "ref_build_%dthreads_ms" % cores: refn * 1e3, "identical": True}
        print(name, json.dumps(r))
        results[name] = r
    g.close()
    if args.out:
        json.dump(results, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
