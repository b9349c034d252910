#!/usr/bin/env python3
"""Times writing a compressed scene cache with nvc_scene_cache_write from device memory, against the reference's encoders.

Workload: --copies copies of kitten's raw geometry (tests/golden/scene_cache_write_raw.npz, the uncompressed cache of the run
that wrote kitten.z.cache) in one cache, from --seed: the vertices with seeded jitter in the fp16 positions (as
tools/scene_cache_device_bench.py builds its workload), the LOD index buffers repeated, Meshlet[] with per-copy data offsets and
meshletdata repeated; the other sections once.  The geometry sections are CUDA tensors.

Measured:
  write          the whole nvc_scene_cache_write call (host clock; the call ends in a device synchronise)
  per section    a write of that section alone through the Python wrapper (its output buffer and copy included); for the
                 vertex and meshlet streams also their encode kernels' device time (torch.profiler); for INDICES also the
                 host index encode alone (nvc::encode_index_stream on the same indices, timed by the C++ timer below)
  reference      the reference's encoders on one host thread (tools/scene_cache_ref_encode_timer.cpp over
                 oracle/_ref/libmeshopt_ref.so, required), per section
The file written from device memory is compared with the reference encoders' file in the same run.  Median of --iters calls
after --warmup.  Prints the card, its power limit and max SM clock, and one JSON line.

Usage: python tools/scene_cache_write_bench.py [--copies 1000] [--iters 10] [--warmup 2] [--seed 1] [--ref-iters 3]"""
import argparse
import functools
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libmeshopt_ref.so")
GEOMETRY = ("vertices", "indices", "meshlets", "meshletdata", "meshletvtx0")


@functools.lru_cache(maxsize=1)
def kitten():
    """(header, sections) of kitten's uncompressed cache (not to be modified)"""
    import ctypes

    from niagara_b200 import layout
    from niagara_b200.lib import load_library

    with np.load(os.path.join(ROOT, "tests", "golden", "scene_cache_write_raw.npz")) as z:
        data = z["kitten"]
    info = layout.SceneCacheInfo()
    assert load_library().nvc_scene_cache_parse(data.ctypes.data, len(data), ctypes.byref(info)) == 0
    secs = {name: data[int(info.sections[s].offset) : int(info.sections[s].offset + info.sections[s].stored_bytes)].copy() for s, name in enumerate(layout.CACHE_SECTIONS)}
    return info.header, secs


def geometry(copies=1000, seed=1):
    """the workload's sections as numpy uint8 arrays"""
    from niagara_b200 import layout

    header, secs = kitten()
    rng = np.random.default_rng(seed)
    many = np.tile(secs["vertices"].reshape(-1, 16), (copies, 1))
    pos = many[:, :6].copy().view(np.uint16)
    pos += rng.integers(-2, 3, pos.shape).astype(np.uint16)  # a few ulps of fp16 jitter per coordinate
    many[:, :6] = pos.view(np.uint8)
    meshlets = np.tile(secs["meshlets"].view(layout.MESHLET_DTYPE), copies)
    words = len(secs["meshletdata"]) // 4
    meshlets["dataOffset"] += (np.arange(copies, dtype=np.uint32) * words).repeat(len(meshlets) // copies)
    out = dict(secs)
    out["vertices"] = many.reshape(-1)
    out["indices"] = np.tile(secs["indices"], copies)
    out["meshlets"] = meshlets.view(np.uint8)
    out["meshletdata"] = np.tile(secs["meshletdata"], copies)
    return out


def write(sections, compressed=True):
    """the file's bytes (scene_cache.write_scene_cache with kitten's header fields)"""
    from niagara_b200.scene_cache import write_scene_cache

    h = kitten()[0]
    return write_scene_cache(sections, compressed=compressed, hash_meta=h.hashMeta, camera=h.camera, sun_direction=list(h.sunDirection))



def _timer(tmp):
    exe = os.path.join(tmp, "scene_cache_ref_encode_timer")
    if not os.path.exists(exe):
        csrc = os.path.join(ROOT, "niagara_b200", "csrc")
        subprocess.run(["g++", "-O2", "-std=c++17", "-I", csrc, "-o", exe, os.path.join(ROOT, "tools", "scene_cache_ref_encode_timer.cpp"),
                        os.path.join(csrc, "nvc_scene_cache.cpp"), os.path.join(csrc, "nvc_meshopt_decode.cpp"), os.path.join(csrc, "nvc_meshopt_encode.cpp"), "-ldl"],
                       check=True)
    return exe


def reference_file(sections, iters=1, tmp=None):
    """(the compressed file the reference's encoders make from `sections`, their per-section medians in ms, plus the median of
    this library's host index encode alone and whether its stream equals the reference's)"""
    if not os.path.exists(REF_SO):
        raise SystemExit("needs the reference's encoders: %s (built by __graft_entry__.build() where the reference is present)" % REF_SO)
    with tempfile.TemporaryDirectory() as own:
        tmp = tmp or own
        raw = os.path.join(tmp, "in.raw.cache")
        with open(raw, "wb") as f:
            f.write(write(sections, compressed=False))
        out = os.path.join(tmp, "ref.z.cache")
        times = json.loads(subprocess.run([_timer(tmp), REF_SO, raw, out, str(iters)], capture_output=True, text=True, check=True).stdout)
        return np.fromfile(out, np.uint8), times


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return out.splitlines()[0] if out else "unknown"


def median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def kernel_ms(fn):
    """device kernel time of one call, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total = 0.0
    for k in prof.key_averages():
        if "encode" in k.key:
            total += getattr(k, "device_time_total", None) or getattr(k, "cuda_time_total", 0.0)
    return total / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--copies", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--ref-iters", type=int, default=3, help="calls of the reference's encoders (seconds each at 1000 copies)")
    args = ap.parse_args()

    import torch

    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    t0 = time.perf_counter()
    secs = geometry(args.copies, args.seed)
    gpu = {k: (torch.from_numpy(v).cuda() if k in GEOMETRY else v) for k, v in secs.items()}
    torch.cuda.synchronize()
    print("generated %d copies in %.1f s" % (args.copies, time.perf_counter() - t0), flush=True)
    results = {"card": card(), "copies": args.copies, "seed": args.seed, "iters": args.iters,
               "vertices": len(secs["vertices"]) // 16, "indices": len(secs["indices"]) // 4, "meshlets": len(secs["meshlets"]) // 24}
    with tempfile.TemporaryDirectory() as tmp:
        want, ref_times = reference_file(secs, args.ref_iters, tmp)
    got = np.frombuffer(write(gpu), np.uint8)
    results["equal"] = bool(len(got) == len(want) and np.array_equal(got, want))
    results["file_bytes"] = len(got)
    results["write_ms"] = round(median_ms(lambda: write(gpu), args.iters, args.warmup), 3)
    own_index_ms, own_index_equal = ref_times.pop("own_index_encode_ms"), ref_times.pop("own_index_equal")
    results["reference_ms"] = {k: round(v, 3) for k, v in ref_times.items()}
    results["reference_total_ms"] = round(sum(ref_times.values()), 3)
    sections = {}
    for name, keys in (("vertices", ("vertices",)), ("meshletdata", ("meshlets", "meshletdata")), ("indices", ("indices",))):
        alone = {k: gpu[k] for k in keys}
        sections[name] = {"write_alone_ms": round(median_ms(lambda: write(alone), args.iters, args.warmup), 3)}
        if name != "indices":
            sections[name]["device_kernels_ms"] = round(kernel_ms(lambda: write(alone)), 3)
    sections["indices"]["host_encode_ms"] = round(own_index_ms, 3)  # the index codec alone, from host memory, one thread
    sections["indices"]["host_encode_equal"] = own_index_equal
    results["sections"] = sections
    print(json.dumps(results), flush=True)
    assert results["equal"], "the device-written file differs from the reference encoders' file"
    assert own_index_equal, "the host index encoder's stream differs from the reference's"


if __name__ == "__main__":
    main()
