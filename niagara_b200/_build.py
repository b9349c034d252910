"""In-tree build of the sm_90a shared library (libniagara_cull.so) with nvcc.

The built .so is git-ignored: build() makes it in every checkout."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB_PATH = os.path.join(HERE, "libniagara_cull.so")

SOURCES = ["nvc_kernels.cu", "nvc_api.cu", "nvc_peer.cu", "nvc_host.cpp", "nvc_scene_cache.cpp", "nvc_scene_cache_device.cpp", "nvc_scene_cache_write.cpp", "nvc_meshopt_decode.cpp", "nvc_meshopt_encode.cpp", "nvc_gltf.cpp", "nvc_nccl.cpp"]
HEADERS = ["nvc_internal.h", "nvc_math.cuh", "nvc_filter.cuh", "nvc_cook.cuh", "nvc_meshlets.cuh", "nvc_lods.cuh", "nvc_vertices.cuh", "nvc_obj.cuh", "nvc_scan.cuh", "nvc_cache_decode.cuh", "nvc_cache_encode.cuh", "nvc_meshopt_format.h", "nvc_meshopt_host.h", "nvc_tma.cuh", os.path.join(ROOT, "include", "niagara_cull.h")]

NVCC_FLAGS = [
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-O3",
    "-lineinfo",
    "-std=c++17",
    "-fmad=false",  # arithmetic contract: no FMA contraction (see csrc/nvc_math.cuh)
    "-Xcompiler",
    "-fPIC,-fvisibility=hidden,-ffp-contract=off",
    "-shared",
]


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; cannot build libniagara_cull.so")
    return nvcc


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, out=None):
    """Compiles every CUDA source for sm_90a into niagara_b200/libniagara_cull.so (or `out`, e.g. a build of another
    revision for an A/B, selected at run time with NVC_LIB_PATH)."""
    out = out or LIB_PATH
    if not force and out == LIB_PATH and not needs_build():
        return LIB_PATH
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", out] + srcs + ["-ldl"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return out


if __name__ == "__main__":
    print(build(force=True, verbose=True))
