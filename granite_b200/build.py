"""Builds libgranite_b200.so in-tree with nvcc for sm_90a (no torch extension machinery:
the product is a plain C-ABI shared library)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libgranite_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr"]
# diagnostics only, e.g. GRB_EXTRA_NVCC_FLAGS=-DGRB_LIGHTING_DEBUG for tools/lighting_timeline.py
COMMON += os.environ.get("GRB_EXTRA_NVCC_FLAGS", "").split()

# (source, extra flags).  -fmad=false: bit-exact contract with the oracle (see file headers).
UNITS = [
    ("grb_api.cu", []),
    ("grb_cluster.cu", ["-fmad=false"]),
    ("grb_light_prep.cu", ["-fmad=false"]),
    ("grb_post.cu", ["-fmad=false"]),
    ("grb_post_tiles.cu", ["-fmad=false"]),
    ("grb_post_fast.cu", []),
    ("grb_smaa.cu", ["-fmad=false"]),
    ("grb_fsr.cu", ["-fmad=false"]),
    ("grb_decal.cu", ["-fmad=false"]),
    ("grb_fog.cu", ["-fmad=false"]),
    ("grb_lighting.cu", []),
    ("grb_gbuffer.cu", []),
]


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    hdrs = [os.path.join(CSRC, "grb_common.cuh"), os.path.join(HERE, "..", "include", "granite_b200.h"),
            os.path.abspath(__file__)]
    hdrs += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".inc"))]
    objs = []
    for src, extra in UNITS:
        s = os.path.join(CSRC, src)
        o = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            cmd = [NVCC, *ARCH, *COMMON, *extra, "-c", s, "-o", o]
            r = subprocess.run(cmd, capture_output=True, text=True)
            log = os.path.join(HERE, "build", src + ".log")
            with open(log, "w") as f:
                f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
            if verbose or r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed on {src}")
    if force or _stale(OUT, objs):
        cmd = [NVCC, *ARCH, "-shared", "-o", OUT, *objs, "-lcudart", "-Xlinker", f"-rpath={os.environ.get('CUDA_HOME', '/usr/local/cuda')}/lib64"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return OUT


HOST_DIR = os.path.join(HERE, "host")
HOST_OUT = os.path.join(HERE, "libgranite_b200_host.so")
HOST_SRCS = ["math.cpp", "frustum.cpp", "cuda_backend.cpp", "render_graph.cpp", "shard_plan.cpp", "render_context.cpp", "lights.cpp", "clusterer.cpp",
             "renderer.cpp", "nccl_collectives.cpp", "scene_viewer.cpp", "post/hdr.cpp", "post/fxaa.cpp",
             "post/temporal.cpp", "post/aa.cpp", "post/smaa.cpp"]
CXX = os.environ.get("CXX", "g++")
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def build_host(force: bool = False, verbose: bool = False) -> str:
    """C++ host layer (RenderGraph surface, pass builders, viewer harness) -> libgranite_b200_host.so.
    -ffp-contract=off: host light prep is compared bit-for-bit with the oracle."""
    build(force=force, verbose=verbose)
    odir = os.path.join(HERE, "build", "host")
    os.makedirs(os.path.join(odir, "post"), exist_ok=True)
    hdrs = []
    for root, _, files in os.walk(HOST_DIR):
        hdrs += [os.path.join(root, f) for f in files if f.endswith(".hpp")]
    hdrs += [os.path.join(HERE, "..", "include", "granite_b200.h"), os.path.join(HERE, "..", "include", "granite_b200_host.h"),
             os.path.abspath(__file__)]
    objs = []
    for src in HOST_SRCS:
        s = os.path.join(HOST_DIR, src)
        o = os.path.join(odir, src.replace(".cpp", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            cmd = [CXX, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-Wno-unused-parameter",
                   f"-I{CUDA_HOME}/include", "-c", s, "-o", o]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if verbose or r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
            if r.returncode != 0:
                raise RuntimeError(f"{CXX} failed on host/{src}")
    if force or _stale(HOST_OUT, objs + [OUT]):
        cmd = [CXX, "-shared", "-o", HOST_OUT, *objs, f"-L{HERE}", "-lgranite_b200", f"-L{CUDA_HOME}/lib64", "-lcudart", "-ldl",
               "-Wl,-rpath,$ORIGIN", f"-Wl,-rpath,{CUDA_HOME}/lib64"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("host link failed")
    return HOST_OUT


def build_all(force: bool = False, verbose: bool = False):
    return build(force, verbose), build_host(force, verbose)


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose="-v" in sys.argv))
