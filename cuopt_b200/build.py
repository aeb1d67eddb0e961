"""Builds cuopt_b200/lib/libcuopt.so (sm_90a) with nvcc.  No JIT, no torch: the library is a plain C-ABI .so."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libcuopt.so")

CU_SOURCES = ["pdlp_solver.cu", "csr_transpose.cu"]
CPP_SOURCES = ["c_api.cpp", "mps_reader.cpp", "solver_settings.cpp", "dist_comm.cpp", "file_writers.cpp"]


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise FileNotFoundError("nvcc not found")


def sources():
    return [os.path.join(CSRC, s) for s in CU_SOURCES + CPP_SOURCES]


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps += [os.path.join(ROOT, "include", "cuopt", "linear_programming", f) for f in ("cuopt_c.h", "constants.h")]
    deps += [os.path.join(ROOT, "include", "cuopt_b200", "cuopt_b200_ext.h"), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    os.makedirs(LIB_DIR, exist_ok=True)
    host_cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else None
    cmd = [nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
           "-Xcompiler", "-fPIC", "-shared", "-x", "cu",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]
    if host_cxx:
        cmd += ["-ccbin", host_cxx]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    tmp = LIB + ".tmp"  # link next to the target, then rename: a reader never sees a half-written library
    cmd += sources() + ["-o", tmp, "-Xlinker", "-soname,libcuopt.so", "-ldl"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed")
    os.replace(tmp, LIB)
    if verbose:
        sys.stderr.write(res.stderr)
    return LIB


CLI = os.path.join(HERE, "bin", "cuopt_cli")


def build_cli(force: bool = False) -> str:
    """cuopt_b200/bin/cuopt_cli: the command-line runner over the C ABI (csrc/cuopt_cli.cpp), linked against lib/libcuopt.so."""
    lib = build()
    src = os.path.join(CSRC, "cuopt_cli.cpp")
    if not force and os.path.exists(CLI) and os.path.getmtime(CLI) >= max(os.path.getmtime(src), os.path.getmtime(lib)):
        return CLI
    os.makedirs(os.path.dirname(CLI), exist_ok=True)
    cmd = [nvcc_path(), "-O2", "-std=c++17", "-x", "cu", "-gencode", "arch=compute_90a,code=sm_90a",
           "-I" + os.path.join(ROOT, "include"), src, "-o", CLI, "-L" + LIB_DIR, "-lcuopt",
           "-Xlinker", "-rpath,$ORIGIN/../lib", "-Xcompiler", "-pthread"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed (cuopt_cli)")
    return CLI


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_cli(force="--force" in sys.argv))
