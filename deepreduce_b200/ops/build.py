"""In-tree native build: ``python -m deepreduce_b200.ops.build``.

Two shared objects next to this file (git-ignored build products):

* ``_dr_cpu.so``  — host ops (g++ + pybind11, no CUDA/torch dependency)
* ``_dr_cuda.so`` — sm_90a (H100) kernels (nvcc ``-gencode arch=compute_90a,code=sm_90a
  -lineinfo``) + ATen/pybind bindings and the C++ runtime (engine ctx, launch thread)

nvcc cross-compiles without a GPU, so this also runs on a machine without one.  The
rebuild stamp hashes the sources, the compiler flags and the torch version, so a
change of target architecture or flags always rebuilds.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")

CUDA_SOURCES = ["engine.cu", "ops.cu", "p2p.cu", "bn.cu", "p2.cu", "repack.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "--expt-relaxed-constexpr", "--expt-extended-lambda", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _run(cmd, log=None):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if log is not None:
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + r.stdout)
    if r.returncode != 0:
        raise RuntimeError("command failed:\n" + " ".join(cmd) + "\n" + r.stdout[-6000:])
    return r.stdout


def _stale(target, sources, extra=""):
    stamp = target + ".stamp"
    h = hashlib.sha256(extra.encode())
    for s in sources:
        with open(s, "rb") as f:
            h.update(f.read())
    digest = h.hexdigest()
    if os.path.exists(target) and os.path.exists(stamp) and open(stamp).read() == digest:
        return False, digest, stamp
    return True, digest, stamp


def _headers():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]


def build_cpu(verbose=True):
    import pybind11
    src = os.path.join(CSRC, "cpu", "native_cpu.cpp")
    out = os.path.join(HERE, "_dr_cpu.so")
    stale, digest, stamp = _stale(out, [src])
    if not stale:
        return out
    os.makedirs(OBJ, exist_ok=True)
    cmd = ["g++", "-O3", "-std=c++17", "-shared", "-fPIC", "-fvisibility=hidden",
           "-I", pybind11.get_include(), "-I", sysconfig.get_paths()["include"], src, "-o", out]
    _run(cmd, os.path.join(OBJ, "cpu.log"))
    open(stamp, "w").write(digest)
    if verbose:
        print(f"[build] {out}")
    return out


def build_cuda(verbose=True):
    import torch
    from torch.utils import cpp_extension as ce
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    out = os.path.join(HERE, "_dr_cuda.so")
    srcs = [os.path.join(CSRC, s) for s in CUDA_SOURCES] + [os.path.join(CSRC, "binding.cpp")]
    stale, digest, stamp = _stale(out, srcs + _headers(), extra=torch.__version__ + " ".join(NVCC_FLAGS))
    if not stale:
        return out
    os.makedirs(OBJ, exist_ok=True)
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)

    def cu(src):
        o = os.path.join(OBJ, os.path.basename(src) + ".o")
        _run([nvcc] + NVCC_FLAGS + ["-I", CSRC, "-c", src, "-o", o], os.path.join(OBJ, os.path.basename(src) + ".log"))
        return o

    def cpp(src):
        o = os.path.join(OBJ, "binding.o")
        inc = []
        for p in ce.include_paths("cuda"):
            inc += ["-isystem", p]
        cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-c", src, "-o", o, "-I", CSRC,
               "-I", sysconfig.get_paths()["include"], f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
               "-DTORCH_EXTENSION_NAME=_dr_cuda", "-DTORCH_API_INCLUDE_EXTENSION_H", "-w"] + inc
        _run(cmd, os.path.join(OBJ, "binding.log"))
        return o

    with ThreadPoolExecutor(max_workers=4) as ex:
        futs = [ex.submit(cu, s) for s in srcs[:-1]] + [ex.submit(cpp, srcs[-1])]
        objs = [f.result() for f in futs]
    libdirs = ce.library_paths("cuda")
    link = ["g++", "-shared", "-o", out] + objs
    for d in libdirs:
        link += ["-L", d, f"-Wl,-rpath,{d}"]
    link += ["-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python", "-lcudart"]
    _run(link, os.path.join(OBJ, "link.log"))
    open(stamp, "w").write(digest)
    if verbose:
        print(f"[build] {out}")
    return out


def build_all(verbose=True):
    return build_cpu(verbose), build_cuda(verbose)


if __name__ == "__main__":
    build_all()
    for f in sorted(os.listdir(OBJ)):
        if f.endswith(".cu.log"):
            txt = open(os.path.join(OBJ, f)).read()
            for line in txt.splitlines():
                if "registers" in line or "Compiling entry" in line or "spill" in line:
                    print(line)
