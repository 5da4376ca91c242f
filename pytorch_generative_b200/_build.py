"""In-tree build of libpg_b200.so (nvcc, sm_90a only).

The library is plain CUDA C++ behind a C ABI (include/pg_b200.h): no torch headers, no pybind, so a
full rebuild is a few nvcc invocations run in parallel.  Object files are cached under csrc/_obj and
rebuilt when their source (or a shared header) is newer.
"""

import concurrent.futures
import os
import shutil
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")
LIB_PATH = os.path.join(_HERE, "libpg_b200.so")

SOURCES = ["pg_host.cu", "pg_gemm.cu", "pg_elementwise.cu", "pg_attention.cu", "pg_conv.cu", "pg_optim.cu", "pg_linear_attn.cu",
           "pg_made.cu", "pg_nade.cu", "pg_fvbn.cu", "pg_nice.cu",
           "pg_vae.cu", "pg_vq.cu", "pg_density.cu", "pg_vd_vae.cu", "pg_gp.cu", "pg_categorical.cu",
           "pg_logistic_mixture.cu"]
import glob

HEADERS = sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + [os.path.join(INCLUDE, "pg_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; cannot build libpg_b200.so")
    return nvcc


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _compile_one(src, obj, verbose):
    cmd = [_nvcc(), *NVCC_FLAGS, "-c", src, "-o", obj]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    log = proc.stdout + proc.stderr
    with open(obj + ".log", "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed on {src}:\n{log}")
    if verbose:
        print(f"[pg build] compiled {os.path.basename(src)}", file=sys.stderr)
    return log


def build(force=False, verbose=True):
    """Compiles every CUDA source for sm_90a and links libpg_b200.so next to this file."""
    obj_dir = os.path.join(CSRC, "_obj")
    os.makedirs(obj_dir, exist_ok=True)
    jobs = []
    objs = []
    for name in SOURCES:
        src = os.path.join(CSRC, name)
        if not os.path.exists(src):
            raise RuntimeError(f"missing source {src}")
        obj = os.path.join(obj_dir, name.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [src, *HEADERS]):
            jobs.append((src, obj))
    if jobs:
        with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(lambda j: _compile_one(j[0], j[1], verbose), jobs))
    if jobs or force or _stale(LIB_PATH, objs):
        cmd = [_nvcc(), "-shared", "-o", LIB_PATH, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError("link failed:\n" + proc.stdout + proc.stderr)
        if verbose:
            print(f"[pg build] linked {LIB_PATH}", file=sys.stderr)
    return LIB_PATH


if __name__ == "__main__":
    build(force="--force" in sys.argv)
