"""Builds libfuelgpu.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libfuelgpu.so")
SOURCES = ["api.cu", "esdf.cu", "esdf_tile.cu", "sharded.cu", "frontier.cu", "bspline.cu", "bspline_solve.cu", "bspline_solve_long.cu",
           "fusion.cu", "viewpoints.cu"]
FMAD_OK = {"bspline_solve.cu", "bspline_solve_long.cu", "esdf.cu", "esdf_tile.cu", "sharded.cu"}  # files whose arithmetic need not follow the host rounding sequence
HEADERS = [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "bspline_eval.cuh"),
           os.path.join(ROOT, "include", "fuelgpu.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    # the B-spline cost and the PCA follow the reference's fp64 rounding sequence: no FMA contraction
    "-fmad=false",
    "-I", os.path.join(ROOT, "include"), "-I", CSRC,
] + (["-DFUEL_PROF"] if os.environ.get("FUEL_PROF") else [])


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + HEADERS + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for s in SOURCES:
        o = os.path.join(HERE, "build", s.replace(".cu", ".o"))
        flags = [f for f in NVCC_FLAGS if not (s in FMAD_OK and f == "-fmad=false")]
        cmd = [_nvcc()] + flags + (["-Xptxas", "-v"] if verbose else []) + [
            "-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(o)
    failed = False
    for s, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0 or verbose:
            sys.stderr.write("== %s ==\n%s\n" % (s, out))
        failed = failed or p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    cmd = [_nvcc(), "-shared", "-o", SO] + objs + ["-gencode", "arch=compute_90a,code=sm_90a",
                                                   "-Xcompiler", "-fPIC", "-cudart", "static"]
    subprocess.check_call(cmd)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
