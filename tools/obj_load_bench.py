#!/usr/bin/env python3
"""Times nvc_obj_load on the GPU against the reference's loadObj on one host thread (the whole oracle/_ref/load_obj process,
wall clock, writing its output to /dev/null: process start and file read included), on a generated
OBJ file of a few hundred MB (positions, texcoords, normals, quads and triangles, relative indices), and checks that both give
the same Vertex[].  The device time covers the whole call, upload included, between CUDA events (median of --runs after one
warm-up call); the kernel split comes from torch.profiler.  Prints one JSON line.

    python tools/obj_load_bench.py [--mb 300] [--runs 5]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def generate(size, seed=0):
    """about `size` bytes of OBJ text: a grid of positions with texcoords and normals, then quads and triangles over it by
    relative indices, repeated"""
    rng = np.random.default_rng(seed)
    parts, total = [], 0
    while total < size:
        n = 64
        p = rng.normal(0, 50, (n * n, 3)).astype(np.float32)
        t = rng.uniform(0, 1, (n * n, 2)).astype(np.float32)
        nm = rng.normal(0, 1, (n * n, 3)).astype(np.float32)
        nm /= np.linalg.norm(nm, axis=1, keepdims=True)
        lines = ["v %.6f %.6f %.6f" % tuple(x) for x in p]
        lines += ["vt %.5f %.5f" % tuple(x) for x in t]
        lines += ["vn %.6f %.6f %.6f" % tuple(x) for x in nm]
        base = n * n
        for y in range(n - 1):
            for x in range(n - 1):
                a, b, c, d = y * n + x, y * n + x + 1, (y + 1) * n + x + 1, (y + 1) * n + x
                r = [k - base for k in (a, b, c, d)]  # relative: -base .. -1
                if (x + y) % 3:
                    lines.append("f " + " ".join("%d/%d/%d" % (k, k, k) for k in r))
                else:
                    lines.append("f " + " ".join("%d/%d/%d" % (k, k, k) for k in r[:3]))
                    lines.append("f " + " ".join("%d//%d" % (k, k) for k in (r[0], r[2], r[3])))
        chunk = ("\n".join(lines) + "\n").encode()
        parts.append(chunk)
        total += len(chunk)
    return b"".join(parts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=300)
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()

    import torch

    from niagara_b200.lib import check, load_library
    from niagara_b200.obj import ObjInfo, file_table

    blob = generate(args.mb << 20)
    lib = load_library()
    ctx = ctypes.c_void_p()
    check(lib.nvc_create(0, None, ctypes.byref(ctx)), None, "nvc_create")
    table, keep = file_table([blob])
    infos = (ObjInfo * 1)()
    check(lib.nvc_obj_load(ctx, None, table, 1, None, 0, infos), ctx, "nvc_obj_load")
    n = int(infos[0].corner_count)
    out = torch.empty((n, 16), dtype=torch.uint8, device="cuda")

    def call():
        check(lib.nvc_obj_load(ctx, None, table, 1, out.data_ptr(), n, infos), ctx, "nvc_obj_load")

    call()  # warm-up: the scratch grows to its size here
    times = []
    for _ in range(args.runs):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        call()
        end.record()
        torch.cuda.synchronize()
        times.append(start.elapsed_time(end))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            key = e.key if "obj_" in e.key or "scan" in e.key else ("memcpy" if "Memcpy" in e.key else e.key[:40])
            split[key] = round(split.get(key, 0.0) + e.device_time_total / 1000.0, 3)
    got = out.cpu().numpy().view(np.uint16).reshape(-1, 8)

    result = {"bytes": len(blob), "corners": n, "faces": int(infos[0].face_count), "device_ms_median": float(np.median(times)), "device_ms": times,
              "kernel_ms": split, "gpu": torch.cuda.get_device_name(0)}
    ref = os.path.join(ROOT, "oracle", "_ref", "load_obj")
    if os.path.exists(ref):
        with tempfile.TemporaryDirectory() as d:
            src, dst = os.path.join(d, "in.obj"), os.path.join(d, "out.bin")
            with open(src, "wb") as f:
                f.write(blob)
            ms = []
            for _ in range(3):
                t0 = time.perf_counter()
                subprocess.run([ref, src, os.devnull], check=True)
                ms.append((time.perf_counter() - t0) * 1000.0)
            subprocess.run([ref, src, dst], check=True)
            want = np.fromfile(dst, np.uint16).reshape(-1, 8)
        result["reference_ms_median"] = float(np.median(ms))
        result["reference_ms"] = ms
        result["equal"] = bool(want.shape == got.shape and np.array_equal(want, got))
    lib.nvc_destroy(ctx)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
