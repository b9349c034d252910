#!/usr/bin/env python3
"""Times the two-phase loop on depth PRODUCED on the device in each of the reference's three submission modes (niagara.cpp:1524-1525,
1582-1694) on the C3 stand-in (scenes.config3_scene: kitten draws, 4096^2 depth by default):

    cluster   nvc_drawcull(task=1) + nvc_clustercull -> nvc_raster_depth
    tasks     nvc_drawcull(task=1) + nvc_taskcull    -> nvc_raster_depth_tasks
    indexed   nvc_drawcull(task=0)                   -> nvc_raster_depth_indexed (vertices / indices of tests/golden/kitten.z.cache)

Every pass is timed with CUDA events over --steps frames after --warmup frames; one JSON line per mode with the median and minimum of
every pass, the frame time, the triangles rasterised, the visible draws / clusters and the card (name, power limit, max SM clock from
nvidia-smi).  The last frame is run twice from the same visibility state and must give the same depth bits.  Needs a CUDA device;
writes nothing.

--mesh-cull: the cluster and task modes only, each run with the mesh shader's per-triangle cull stage (nvc_set_mesh_cull) off and on,
alternating, --rounds times in one process; every line then also carries "mesh_cull" and the triangles the stage culled per pass.

--task-cull: the cluster and task modes only, each run with the reference's TASK_CULL switch (nvc_set_task_cull) off and on,
alternating, --rounds times in one process; every line then also carries "task_cull".  After them, one "passthrough" line per pass
times the TASK_CULL 0 cluster and task passes alone on the C4 scene (1 M draws, early pass) and gives the bytes they must move
over kernel time as a share of the H100 SXM's 3.35 TB/s."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from niagara_b200 import host, scene_cache, scenes  # noqa: E402
from niagara_b200.path import VisibilityPath  # noqa: E402

PASSES = ["cull_early", "clusters_early", "raster_early", "pyramid", "cull_late", "clusters_late", "raster_late"]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    first = out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else ""
    name, power, clock = (first.split(", ") + ["?", "?", "?"])[:3] if first else ("?", "?", "?")
    return {"device": name or torch.cuda.get_device_name(0), "power_limit": power, "sm_clock_max": clock}


def run_mode(mode, s, geometry, args, mesh_cull=None, task_cull=None):
    dev = torch.device("cuda:0")
    mesh_shading = mode != "indexed"
    kw = {}
    if mode == "tasks":
        # payload storage for every command drawcull can write: ceil(meshlets / 64) per draw at its largest LOD
        per_draw = (s.meshes["lods"]["meshletCount"].max(axis=1)[s.draws["meshIndex"]].astype(np.int64) + 63) // 64
        kw["task_wglimit"] = int((per_draw.sum() + 63) // 64 * 64)
    path = VisibilityPath(s.meshes, s.meshlets, s.draws, *s.screen, mesh_shading=mesh_shading, **kw)
    path.set_visibility_bits(s.visibility_bits)
    if mesh_cull is not None:
        path.set_mesh_cull(mesh_cull)
    if task_cull is not None:
        path.set_task_cull(task_cull)
    cd = s.cull_data(**({} if mesh_shading else dict(mesh_shading=False, cluster_occlusion=False)))
    proj = host.projection(s.camera, *s.screen)
    vb = torch.from_numpy(np.ascontiguousarray(geometry["vertices"])).to(dev)
    md = torch.from_numpy(np.ascontiguousarray(s.meshletdata).view(np.int32)).to(dev)
    ib = torch.from_numpy(np.ascontiguousarray(geometry["indices"], dtype=np.uint32).view(np.int32)).to(dev)
    depth = torch.zeros((s.screen[1], s.screen[0]), dtype=torch.float32, device=dev)
    stats = [torch.zeros(4, dtype=torch.int32, device=dev) for _ in range(2)]
    if mode == "tasks":
        payloads = torch.zeros((path.task_wglimit, 64), dtype=torch.int32, device=dev)
        emit = torch.zeros(path.task_wglimit, dtype=torch.int32, device=dev)
    counts = {}

    def clusters(late, k):
        if mode == "cluster":
            path.render_clusters(cd, late, cluster_backface=True)
        elif mode == "tasks":
            path.task_shading(cd, late, payloads, emit, cluster_backface=True)

    def raster(k):
        if mode == "cluster":
            path.raster_depth(cd, proj, vb, md, depth, stats[k])
        elif mode == "tasks":
            path.raster_depth_tasks(cd, proj, payloads, emit, vb, md, depth, stats[k])
        else:
            path.raster_depth_indexed(cd, proj, vb, ib, depth, stats[k])

    def frame(ev=None, probe=False):
        def mark(i):
            if ev is not None:
                ev[i].record()

        mark(0)
        path.cull(cd, late=False)
        mark(1)
        clusters(False, 0)
        if probe:
            torch.cuda.synchronize()
            counts["clusters_early"] = int(path.ccb[0].item()) if mode == "cluster" else int(emit[: int(path.dccb[1].item()) * 64].clamp(max=64).sum().item()) if mode == "tasks" else None
        mark(2)
        depth.zero_()
        raster(0)
        if probe and mesh_cull is not None:
            counts["culled_early"] = path.mesh_cull_stats(reset=True)[1]
        mark(3)
        path.pyramid(depth)
        mark(4)
        path.cull(cd, late=True)
        mark(5)
        clusters(True, 1)
        if probe:
            torch.cuda.synchronize()
            counts["clusters_late"] = int(path.ccb[0].item()) if mode == "cluster" else int(emit[: int(path.dccb[1].item()) * 64].clamp(max=64).sum().item()) if mode == "tasks" else None
        mark(6)
        raster(1)
        if probe and mesh_cull is not None:
            counts["culled_late"] = path.mesh_cull_stats(reset=True)[1]
        mark(7)

    for _ in range(max(3, args.warmup)):
        frame()
    torch.cuda.synchronize()
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(8)] for _ in range(args.steps)]
    for k in range(args.steps):
        frame(evs[k])
    torch.cuda.synchronize()
    ms = np.array([[e[i].elapsed_time(e[i + 1]) for i in range(7)] + [e[0].elapsed_time(e[7])] for e in evs])

    # determinism: the last frame again from the same visibility state, twice
    dvb, mvb = path.dvb.clone(), path.mvb.clone()
    if mesh_cull is not None:
        path.mesh_cull_stats(reset=True)
    frame(probe=True)
    torch.cuda.synchronize()
    first = depth.clone()
    st = [t.cpu().numpy().astype(np.uint32) for t in stats]
    path.dvb.copy_(dvb)
    path.mvb.copy_(mvb)
    frame()
    torch.cuda.synchronize()
    if not torch.equal(first.view(torch.int32), depth.view(torch.int32)):
        raise SystemExit("raster_modes_bench.py: %s: repeating the last frame changed the depth image" % mode)

    def summary(col):
        return {"median": float(np.median(ms[:, col])), "min": float(ms[:, col].min())}

    passes = {name: summary(i) for i, name in enumerate(PASSES) if mesh_shading or not name.startswith("clusters")}
    out = {
        "mode": mode,
        "workload": "C3 stand-in: %s" % s.note,
        "steps": args.steps,
        "warmup": args.warmup,
        "passes_ms": passes,
        "frame_ms": summary(7),
        "triangles_rasterised": {"early": int(st[0][1]), "late": int(st[1][1])},
        "visible_draws": int((dvb != 0).sum().item()),
        "drawn": {"early": int(st[0][0]), "late": int(st[1][0]), "what": "draw commands" if mode == "indexed" else "clusters"},
        "clusters": None if mode == "indexed" else {"early": counts["clusters_early"], "late": counts["clusters_late"]},
        "rejected": {"early": int(st[0][2]), "late": int(st[1][2])},
    }
    if mesh_cull is not None:
        out["mesh_cull"] = bool(mesh_cull)
        out["triangles_culled"] = {"early": counts["culled_early"], "late": counts["culled_late"]}
    if task_cull is not None:
        out["task_cull"] = bool(task_cull)
    out.update(card())
    path.close()
    return out


def passthrough_c4(args):
    """the TASK_CULL 0 cluster and task passes alone on the C4 scene's early commands: CUDA events around --steps launches each"""
    s = scenes.config4_scene()
    path = VisibilityPath(s.meshes, s.meshlets, s.draws, *s.screen)
    path.set_visibility_bits(s.visibility_bits)
    path.set_task_cull(False)
    path.dvb.fill_(1)
    cd = s.cull_data()
    path.cull(cd, late=False)
    torch.cuda.synchronize()
    ncmd = int(path.dccb[1].item()) * 64
    payloads = torch.empty((ncmd, 64), dtype=torch.int32, device="cuda:0")
    emit = torch.empty(ncmd, dtype=torch.int32, device="cuda:0")
    runs = {"clusters": lambda: path.render_clusters(cd, False), "tasks": lambda: path.task_shading(cd, False, payloads, emit)}
    out = []
    for name, run in runs.items():
        for _ in range(max(3, args.warmup)):
            run()
        torch.cuda.synchronize()
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
        for a, b in evs:
            a.record()
            run()
            b.record()
        torch.cuda.synchronize()
        ms = np.array([a.elapsed_time(b) for a, b in evs])
        clusters = int(path.ccb[0].item())
        # every 32-byte sector of the 20-byte command records holds a taskCount that is read; output as written
        moved = ncmd * 20 + (clusters + 255) // 256 * 256 * 4 if name == "clusters" else ncmd * 20 + ncmd * (256 + 4)
        med = float(np.median(ms))
        out.append({"passthrough": name, "workload": "C4: %d draws, early pass, %d task commands" % (len(s.draws), ncmd), "steps": args.steps,
                    "kernel_ms": {"median": med, "min": float(ms.min())}, "clusters": clusters if name == "clusters" else None, "bytes": moved,
                    "share_of_3.35TBps": moved / (med * 1e-3) / 3.35e12})
    path.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--draws", type=int, default=10000)
    ap.add_argument("--depth", type=int, default=4096, help="depth target size (square)")
    ap.add_argument("--modes", default="cluster,tasks,indexed")
    ap.add_argument("--mesh-cull", action="store_true", help="cluster / task modes with the mesh-cull stage off and on, alternating")
    ap.add_argument("--rounds", type=int, default=3, help="off / on pairs per mode with --mesh-cull / --task-cull")
    ap.add_argument("--task-cull", action="store_true", help="cluster / task modes with the TASK_CULL switch off and on, alternating, then the pass-through kernels on C4")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("raster_modes_bench.py needs a CUDA device")
    if args.steps < 1:
        sys.exit("--steps must be >= 1")
    golden = os.path.join(ROOT, "tests", "golden")
    s = scenes.config3_scene(golden, draw_count=args.draws, screen=(args.depth, args.depth))
    cache = scene_cache.SceneCache(os.path.join(golden, "kitten.z.cache"))
    if not np.array_equal(cache.section("meshes"), s.meshes):
        sys.exit("kitten.z.cache does not hold the meshes of kitten.nvcg")
    if args.task_cull:
        modes = [m for m in args.modes.split(",") if m != "indexed"]  # the draw path has no cluster pass
        geometry = {"vertices": s.vertices, "indices": cache.section("indices")}
        for r in range(args.rounds):
            for mode in modes:
                for on in ((False, True) if r % 2 == 0 else (True, False)):
                    print(json.dumps(run_mode(mode, s, geometry, args, task_cull=on)), flush=True)
        card_info = card()
        for line in passthrough_c4(args):
            line.update(card_info)
            print(json.dumps(line), flush=True)
        return
    if args.mesh_cull:
        modes = [m for m in args.modes.split(",") if m != "indexed"]  # mesh.vert has no per-triangle stage
        geometry = {"vertices": s.vertices, "indices": cache.section("indices")}
        for r in range(args.rounds):
            for mode in modes:
                for on in ((False, True) if r % 2 == 0 else (True, False)):
                    print(json.dumps(run_mode(mode, s, geometry, args, mesh_cull=on)), flush=True)
        return
    for mode in args.modes.split(","):
        geometry = {"vertices": s.vertices if mode != "indexed" else cache.section("vertices"), "indices": cache.section("indices")}
        print(json.dumps(run_mode(mode, s, geometry, args)), flush=True)


if __name__ == "__main__":
    main()
