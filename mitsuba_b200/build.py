"""Builds libb2mts.so (CUDA kernels for sm_90a + the C-ABI) in-tree with nvcc.

    python -m mitsuba_b200.build [--force]

nvcc cross-compiles without a GPU.  The kernel translation unit is compiled twice: kernels_parity.cu with
-fmad=false and kernels_fast.cu with FMA contraction on.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
HOST = os.path.join(HERE, "host")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libb2mts.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-ffp-contract=off,-fno-fast-math", "-I", os.path.join(HERE, "..", "include")]

UNITS = [
    # (source, extra flags)
    (os.path.join(CSRC, "kernels_parity.cu"), ["-fmad=false"]),
    # throughput build: FMA contraction + fast intrinsics (approximate div/sqrt/sincos/exp, flush-to-zero); the image
    # parity tests hold it to the same 1e-3 relative-L2 tolerance as the parity build
    (os.path.join(CSRC, "kernels_fast.cu"), ["--use_fast_math"]),
    (os.path.join(CSRC, "b2_host.cpp"), ["-x", "cu"]),
    (os.path.join(CSRC, "b2_commit.cpp"), ["-x", "cu"]),
    (os.path.join(CSRC, "bvh_builder.cpp"), []),
    # device BVH build: byte-identical to bvh_builder.cpp, so IEEE arithmetic without contraction (division and sqrt stay IEEE)
    (os.path.join(CSRC, "bvh_device.cu"), ["-fmad=false"]),
    (os.path.join(HOST, "scene_xml.cpp"), []),
    (os.path.join(HOST, "mipmap.cpp"), []),
    (os.path.join(HOST, "spectrum.cpp"), []),
]
HEADERS = [os.path.join(CSRC, f) for f in ("b2_math.cuh", "b2_types.h", "b2_sampler.cuh", "b2_bsdf.cuh", "b2_trace.cuh",
                                           "b2_kernels.inl", "b2_launch.h", "b2_host.h", "bvh_builder.h", "bvh_device.h", "b2_medium.cuh", "b2_texture.cuh", "b2_envmap.cuh")] + \
          [os.path.join(HOST, "mipmap.h"), os.path.join(HOST, "spectrum.h")] + \
          [os.path.join(HERE, "..", "include", "b2mts.h")]


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    units = [(s, f) for s, f in UNITS if os.path.exists(s)]
    jobs = []
    objs = []
    for src, extra in units:
        obj = os.path.join(OBJ, os.path.basename(src) + ".o")
        objs.append(obj)
        if force or _newer(obj, [src] + HEADERS):
            cmd = [NVCC] + ARCH + COMMON + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        return r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=len(jobs)) as ex:
            outs = list(ex.map(run, jobs))
        if verbose:
            print("\n".join(outs))
    if force or jobs or _newer(LIB, objs):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-lexpat", "-lz", "-ldl", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    # stand-alone CLI driver over the C-ABI (mirrors `mitsuba -o out -D k=v scene.xml`)
    exe = os.path.join(HERE, "mtsb200")
    main_src = os.path.join(HOST, "mtsb200_main.cpp")
    if os.path.exists(main_src) and (force or _newer(exe, [main_src, LIB])):
        cmd = ["g++", "-O2", "-std=c++17", "-o", exe, main_src, "-L", HERE, "-lb2mts", "-Wl,-rpath,$ORIGIN"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("mtsb200 link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
