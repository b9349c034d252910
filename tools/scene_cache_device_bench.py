#!/usr/bin/env python3
"""Times reading a compressed scene cache's VERTICES, INDICES and MESHLETDATA sections into device memory two ways:

  (a) host   nvc_scene_cache_read into pinned host memory, then one copy up, ending in a synchronise
  (b) device nvc_scene_cache_read_device: the stream goes up as stored and is decoded by kernels; its host walk (the
             serial part) is also timed on its own, by tools/scene_cache_walk_timer.cpp built from the library's sources

Workload: --copies copies of tests/golden/kitten.z.cache's geometry in one cache, from --seed: the vertices with seeded
jitter in the fp16 positions, re-encoded with the reference's vertex encoder at level 2 (as writeVertexCompressed does;
oracle/_ref/libmeshopt_ref.so, required); Meshlet[] with per-copy data offsets; the meshlet blocks copied verbatim
(references are mesh-local); kitten's index chain (every LOD) repeated per copy, re-encoded with the reference's index
encoder at the stream's own version (as saveSceneCache writes it).  Both outputs are compared in the same run.  Times: host clock around each call (every
call ends in a device synchronise), median of --iters calls after --warmup.  Prints the card, its power limit and max SM
clock, and one JSON line.

Usage: python tools/scene_cache_device_bench.py [--copies 1000] [--iters 10] [--warmup 2] [--seed 1]"""
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
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libmeshopt_ref.so")
HEADER = 160


def generate(copies=1000, seed=1, indices=False):
    """the workload cache as a uint8 array; with `indices`, an INDICES section too"""
    from niagara_b200 import layout
    from niagara_b200.lib import load_library

    if not os.path.exists(REF_SO):
        raise SystemExit("needs the reference's vertex encoder: %s (built by __graft_entry__.build() where the reference is present)" % REF_SO)
    lib = load_library()
    src = np.fromfile(os.path.join(ROOT, "tests", "golden", "kitten.z.cache"), np.uint8)
    info = layout.SceneCacheInfo()
    assert lib.nvc_scene_cache_parse(src.ctypes.data, len(src), ctypes.byref(info)) == 0

    def read(name):
        s = layout.CACHE_SECTIONS.index(name)
        out = np.zeros(int(info.sections[s].decoded_bytes), np.uint8)
        assert lib.nvc_scene_cache_read(src.ctypes.data, len(src), ctypes.byref(info), s, out.ctypes.data, out.size) == 0
        return out

    def stored(name):
        sec = info.sections[layout.CACHE_SECTIONS.index(name)]
        return src[int(sec.offset) : int(sec.offset + sec.stored_bytes)]

    rng = np.random.default_rng(seed)
    verts = read("vertices").reshape(-1, 16)
    many = np.tile(verts, (copies, 1))
    pos = many[:, :6].copy().view(np.uint16)
    pos += rng.integers(-2, 3, pos.shape).astype(np.uint16)  # a few ulps of fp16 jitter per coordinate
    many[:, :6] = pos.view(np.uint8)
    ref = ctypes.CDLL(REF_SO)
    ref.meshopt_encodeVertexBufferBound.restype = ctypes.c_size_t
    ref.meshopt_encodeVertexBufferBound.argtypes = [ctypes.c_size_t, ctypes.c_size_t]
    ref.meshopt_encodeVertexBufferLevel.restype = ctypes.c_size_t
    ref.meshopt_encodeVertexBufferLevel.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int, ctypes.c_int]
    many = np.ascontiguousarray(many)
    buf = np.zeros(ref.meshopt_encodeVertexBufferBound(len(many), 16), np.uint8)
    version = int(stored("vertices")[0]) & 15
    n = ref.meshopt_encodeVertexBufferLevel(buf.ctypes.data, len(buf), many.ctypes.data, len(many), 16, 2, version)
    assert n > 0
    vstream = buf[:n]

    meshlets = read("meshlets").view(layout.MESHLET_DTYPE)
    words = int(info.header.meshletdataCount)
    all_meshlets = np.tile(meshlets, copies)
    all_meshlets["dataOffset"] += (np.arange(copies, dtype=np.uint32) * words).repeat(len(meshlets))
    chain = np.tile(stored("meshletdata"), copies)

    istream = np.zeros(0, np.uint8)
    index_count = 0
    if indices:
        ichain = np.ascontiguousarray(np.tile(read("indices").view(np.uint32), copies))
        ref.meshopt_encodeIndexVersion.argtypes = [ctypes.c_int]
        ref.meshopt_encodeIndexBufferBound.restype = ctypes.c_size_t
        ref.meshopt_encodeIndexBufferBound.argtypes = [ctypes.c_size_t, ctypes.c_size_t]
        ref.meshopt_encodeIndexBuffer.restype = ctypes.c_size_t
        ref.meshopt_encodeIndexBuffer.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t]
        ref.meshopt_encodeIndexVersion(int(stored("indices")[0]) & 15)
        ibuf = np.zeros(ref.meshopt_encodeIndexBufferBound(len(ichain), int(ichain.max()) + 1), np.uint8)
        m = ref.meshopt_encodeIndexBuffer(ibuf.ctypes.data, len(ibuf), ichain.ctypes.data, len(ichain))
        assert m > 0
        istream, index_count = ibuf[:m], len(ichain)

    h = layout.SceneCacheHeader.from_buffer_copy(src[:HEADER].tobytes())
    h.compressed = 1
    h.vertexCount, h.compressedVertexBytes = len(many), n
    h.indexCount, h.compressedIndexBytes = index_count, len(istream)
    h.meshletCount, h.meshletdataCount, h.compressedMeshletDataBytes = len(all_meshlets), words * copies, len(chain)
    for field in ("meshletvtx0Count", "compressedMeshletVtx0Bytes", "meshCount", "materialCount", "drawCount", "texturePathCount", "lightCount",
                  "animationCount", "keyframeCount", "ommArrayDataSize", "ommIndexDataSize", "ommDescCount"):
        setattr(h, field, 0)
    return np.concatenate([np.frombuffer(bytes(h), np.uint8), vstream, istream, all_meshlets.view(np.uint8), chain])


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return out.splitlines()[0] if out else "unknown"


def walk_times(path, iters):
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "scene_cache_walk_timer")
        csrc = os.path.join(ROOT, "niagara_b200", "csrc")
        subprocess.run(["g++", "-O3", "-std=c++17", "-I", csrc, "-o", exe, os.path.join(ROOT, "tools", "scene_cache_walk_timer.cpp"),
                        os.path.join(csrc, "nvc_meshopt_decode.cpp"), os.path.join(csrc, "nvc_scene_cache.cpp")], check=True)
        return json.loads(subprocess.run([exe, path, str(iters)], capture_output=True, text=True, check=True).stdout)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--copies", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()

    import torch

    from niagara_b200 import layout
    from niagara_b200.lib import check, load_library

    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    lib = load_library()
    t0 = time.perf_counter()
    data = generate(args.copies, args.seed, indices=True)
    print("generated %d copies in %.1f s" % (args.copies, time.perf_counter() - t0), flush=True)
    info = layout.SceneCacheInfo()
    assert lib.nvc_scene_cache_parse(data.ctypes.data, len(data), ctypes.byref(info)) == 0
    ctx = ctypes.c_void_p()
    check(lib.nvc_create(0, None, ctypes.byref(ctx)), None, "nvc_create")
    stream = torch.cuda.current_stream().cuda_stream
    results = {"card": card(), "copies": args.copies, "seed": args.seed, "iters": args.iters}
    for name in ("vertices", "indices", "meshletdata"):
        s = layout.CACHE_SECTIONS.index(name)
        sec = info.sections[s]
        n = int(sec.decoded_bytes)
        pinned = torch.empty(n, dtype=torch.uint8, pin_memory=True)
        host_dst = torch.empty(n, dtype=torch.uint8, device="cuda")
        dev_dst = torch.empty(n, dtype=torch.uint8, device="cuda")

        def host_path():
            assert lib.nvc_scene_cache_read(data.ctypes.data, len(data), ctypes.byref(info), s, pinned.data_ptr(), n) == 0
            host_dst.copy_(pinned)
            torch.cuda.synchronize()

        def device_path():
            check(lib.nvc_scene_cache_read_device(ctx, stream, data.ctypes.data, len(data), ctypes.byref(info), s, dev_dst.data_ptr(), n), ctx, "nvc_scene_cache_read_device")

        times = {}
        for label, fn in (("host", host_path), ("device", device_path)):
            for _ in range(args.warmup):
                fn()
            t = []
            for _ in range(args.iters):
                t0 = time.perf_counter()
                fn()
                t.append((time.perf_counter() - t0) * 1e3)
            times[label] = float(np.median(t))
        equal = bool(torch.equal(host_dst, dev_dst))
        results[name] = {"stored_bytes": int(sec.stored_bytes), "decoded_bytes": n, "host_read_and_copy_ms": round(times["host"], 3),
                         "device_read_ms": round(times["device"], 3), "equal": equal}
        print(name, results[name], flush=True)
        assert equal, name
    lib.nvc_destroy(ctx)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "bench.cache")
        data.tofile(path)
        walks = walk_times(path, args.iters)
    results["vertices"]["host_walk_ms"] = walks["vertices_walk_ms"]
    results["meshletdata"]["host_walk_ms"] = walks["meshletdata_walk_ms"]
    results["indices"]["host_walk_ms"] = walks["indices_walk_ms"]
    print(json.dumps(results))


if __name__ == "__main__":
    main()
