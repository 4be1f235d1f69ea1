"""Build libian_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python neural-photo-editor_b200/build.py [--force]

Every .cu is compiled to its own object (in parallel, only when stale) and the objects are linked into the shared
library; objects live under csrc/_obj/ (git-ignored), so a rebuild only recompiles what changed.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = ["ian_api.cu", "tapgemm_simt.cu", "tapgemm_tc.cu", "decout_tc.cu", "conv1_tc.cu", "edge_kernels.cu",
       "head_tc.cu", "train_kernels.cu", "enc_vjp.cu", "wgrad_tc.cu", "param_vjp.cu",
       "gn_kernels.cu", "feat_kernels.cu", "disc_kernels.cu"]
HDR = ["tapgemm.h", "edge.h", "tc_ptx.cuh", "../../include/ian_b200.h"]
LIB = os.path.join(HERE, "libian_b200.so")
OBJ_DIR = os.path.join(HERE, "csrc", "_obj")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17"] + ARCH + ["-lineinfo",
              "-Xcompiler", "-fPIC"]


def _sources():
    return [f for f in SRC if os.path.exists(os.path.join(HERE, "csrc", f))]


def _stale_objects(force: bool):
    os.makedirs(OBJ_DIR, exist_ok=True)
    newest_hdr = max([os.path.getmtime(os.path.join(HERE, "csrc", f)) for f in HDR] + [os.path.getmtime(os.path.abspath(__file__))])
    out = []
    for f in _sources():
        src, obj = os.path.join(HERE, "csrc", f), os.path.join(OBJ_DIR, f[:-3] + ".o")
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), newest_hdr):
            out.append((src, obj))
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    todo = _stale_objects(force)
    objs = [os.path.join(OBJ_DIR, f[:-3] + ".o") for f in _sources()]
    if not todo and os.path.exists(LIB) and all(os.path.getmtime(o) <= os.path.getmtime(LIB) for o in objs):
        return LIB

    def cc(job):
        cmd = [nvcc] + NVCC_FLAGS + ["-c", job[0], "-o", job[1]]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.run(cmd, check=True)

    with ThreadPoolExecutor(max_workers=max(1, min(len(todo), os.cpu_count() or 1))) as ex:
        list(ex.map(cc, todo))
    cmd = [nvcc, "-shared"] + ARCH + ["-o", LIB] + objs
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)
    return LIB


C_HOST_SRC = os.path.join(HERE, "..", "examples", "c_host", "ian_cli.c")
C_HOST_BIN = os.path.join(HERE, "..", "examples", "c_host", "ian_cli")


def build_c_host(force: bool = False) -> str:
    """the plain-C host program over the C-ABI (examples/c_host): strict C99 against include/ian_b200.h, linked to
    the in-tree library with an $ORIGIN-relative rpath so it runs from wherever the tree is copied."""
    lib = build()
    deps = [C_HOST_SRC, os.path.join(HERE, "..", "include", "ian_b200.h"), lib]
    if not force and os.path.exists(C_HOST_BIN) and all(os.path.getmtime(d) <= os.path.getmtime(C_HOST_BIN) for d in deps):
        return C_HOST_BIN
    cmd = [os.environ.get("CC", "gcc"), "-std=c99", "-O2", "-Wall", "-Wextra", "-Werror", "-pedantic",
           "-I", os.path.join(HERE, "..", "include"), C_HOST_SRC, "-o", C_HOST_BIN,
           "-L", HERE, "-lian_b200", "-Wl,-rpath,$ORIGIN/../../" + os.path.basename(HERE)]
    subprocess.run(cmd, check=True)
    return C_HOST_BIN


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
    print(build_c_host(force="--force" in sys.argv))
