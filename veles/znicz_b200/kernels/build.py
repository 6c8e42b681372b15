"""Ahead-of-time build of the sm_90a extension, in-tree.

``python -m veles.znicz_b200.kernels.build`` compiles every ``csrc/*.cu`` with
``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` (cross-compiles without a GPU),
``csrc/ext.cpp`` against the torch headers, and links ``_znicz_b200_C.so`` next to this
file so the binary travels with the source tree (no JIT cache, no site-packages install).
"""
from __future__ import annotations

import concurrent.futures
import hashlib
import os
import shutil
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
SO_NAME = "_znicz_b200_C.so"
SO_PATH = os.path.join(HERE, SO_NAME)
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr"]


def _nvcc():
    for cand in (os.environ.get("CUDA_HOME", ""), "/usr/local/cuda"):
        p = os.path.join(cand, "bin", "nvcc")
        if cand and os.path.exists(p):
            return p
    p = shutil.which("nvcc")
    if not p:
        raise RuntimeError("nvcc not found")
    return p


def _sources():
    cu = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdr = sorted(f for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    return cu, hdr


def source_digest():
    # the flags are part of the digest: an extension built for another architecture is stale
    h = hashlib.sha1(" ".join(ARCH_FLAGS + NVCC_FLAGS).encode())
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".cpp", ".h")):
            with open(os.path.join(CSRC, f), "rb") as fin:
                h.update(f.encode())
                h.update(fin.read())
    return h.hexdigest()


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("command failed:\n  %s\n%s" % (" ".join(cmd), r.stdout))
    return r.stdout


def is_fresh():
    stamp = os.path.join(BUILD, "digest")
    return os.path.exists(SO_PATH) and os.path.exists(stamp) and \
        open(stamp).read().strip() == source_digest()


def build(force=False, verbose=True):
    if not force and is_fresh():
        if verbose:
            print("znicz_b200 kernels: up to date (%s)" % SO_PATH)
        return SO_PATH
    import torch
    from torch.utils import cpp_extension as ce
    os.makedirs(BUILD, exist_ok=True)
    nvcc = _nvcc()
    cuda_home = os.path.dirname(os.path.dirname(nvcc))
    cu, _ = _sources()
    objs = []
    jobs = []
    for f in cu:
        obj = os.path.join(BUILD, f[:-3] + ".o")
        objs.append(obj)
        jobs.append([nvcc] + ARCH_FLAGS + NVCC_FLAGS + ["-I", CSRC, "-c",
                                                        os.path.join(CSRC, f), "-o", obj])
    inc = []
    for p in ce.include_paths():
        inc += ["-I", p]
    inc += ["-I", os.path.join(cuda_home, "include"), "-I", sysconfig.get_paths()["include"]]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    ext_obj = os.path.join(BUILD, "ext.o")
    objs.append(ext_obj)
    jobs.append(["g++", "-O3", "-std=c++17", "-fPIC", "-D_GLIBCXX_USE_CXX11_ABI=%d" % abi,
                 "-DTORCH_EXTENSION_NAME=_znicz_b200_C", "-DTORCH_API_INCLUDE_EXTENSION_H",
                 "-w"] + inc + ["-c", os.path.join(CSRC, "ext.cpp"), "-o", ext_obj])
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
        for out in ex.map(_run, jobs):
            if verbose and out.strip():
                print(out)
    libs = []
    for p in ce.library_paths():
        libs += ["-L", p, "-Wl,-rpath," + p]
    libs += ["-L", os.path.join(cuda_home, "lib64")]
    _run(["g++", "-shared"] + objs + libs +
         ["-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda",
          "-lcudart", "-o", SO_PATH])
    with open(os.path.join(BUILD, "digest"), "w") as fout:
        fout.write(source_digest())
    if verbose:
        print("znicz_b200 kernels: built %s (%d bytes)" % (SO_PATH, os.path.getsize(SO_PATH)))
    return SO_PATH


if __name__ == "__main__":
    build(force="--force" in sys.argv)
