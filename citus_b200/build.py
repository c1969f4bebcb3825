"""Builds citus_b200/lib/libcitus_gpu.so with nvcc for sm_90a (H100) only.

    python -m citus_b200.build [--force]

The .so and the object files under citus_b200/lib/ are build products and stay out of git.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libcitus_gpu.so")
STAMP = LIB + ".flags"          # the compile flags the library was built with: other flags (another GPU target) rebuild it
SOURCES = ["cg_scan.cu", "cg_decompress.cu", "cg_scan_fast.cu", "cg_scan_small.cu", "cg_scan_rows.cu", "cg_partition.cu", "cg_join.cu", "cg_comm.cu", "cg_values.cu", "cg_varlena.cu", "cg_narrow.cu", "cg_host.cpp", "cg_plan.cpp", "cg_numeric.cpp", "cg_gen.cpp", "cg_jit.cpp"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-fopenmp,-Wall,-Wno-unused-function", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
    "-x", "cu",
]


def flags_stamp() -> str:
    return " ".join(f for f in FLAGS if f != "-I" and not os.path.isabs(f))     # no include paths: a moved tree keeps its build


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    try:
        with open(STAMP) as f:
            if f.read() != flags_stamp():
                return True
    except OSError:
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "citus_gpu.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    objs = []
    procs = []
    objdir = os.path.join(HERE, "lib", "obj")
    os.makedirs(objdir, exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(objdir, src + ".o")
        objs.append(obj)
        cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd += ["-Xptxas", "-v"]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- {src}\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    subprocess.check_call([NVCC, "-shared", "-o", LIB] + objs + ["-Xcompiler", "-fopenmp", "-lgomp", "-ldl"])
    with open(STAMP, "w") as f:
        f.write(flags_stamp())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
