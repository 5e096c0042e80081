"""Build libtb200.so (sm_90a) in-tree with nvcc.

Used by ``__graft_entry__.build()`` and by developers; the Python modules never
build implicitly and never fall back to host code when the library is missing.
"""

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libtb200.so")
BUILD = os.path.join(ROOT, "build")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CUFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC"] + ARCH
SOURCES = ["kernels.cu", "deflate.cu", "runtime.cu", "loadgen.cc", "mock_server.cu"]


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; cannot build libtb200.so")
    return nvcc


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build_native(force=False, verbose=False):
    """Compile every CUDA/C++ source for sm_90a and link libtb200.so."""
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(BUILD, exist_ok=True)
    nvcc = _nvcc()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(ROOT, "include", "tb200.h"))
    headers.append(os.path.join(ROOT, "include", "tb200_loadgen.h"))
    objs = []
    for src in SOURCES:
        path = os.path.join(CSRC, src)
        if not os.path.exists(path):
            continue
        obj = os.path.join(BUILD, os.path.splitext(src)[0] + ".o")
        objs.append(obj)
        if force or _newer(obj, [path] + headers):
            cmd = [nvcc] + CUFLAGS + (["-x", "cu"] if src.endswith(".cc") else []) + ["-c", path, "-o", obj]
            if verbose:
                print(" ".join(cmd))
            subprocess.run(cmd, check=True)
    if force or _newer(LIB, objs):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + ARCH + ["-lpthread"]
        if verbose:
            print(" ".join(cmd))
        subprocess.run(cmd, check=True)
    return LIB


CLIENT_LIB = os.path.join(LIBDIR, "libtb200client.so")


def build_cpp_client(force=False, verbose=False):
    """The C++ front end (client_b200/cpp): plain g++, linked against libtb200.so."""
    cpp = os.path.join(HERE, "cpp")
    srcs = [os.path.join(cpp, "tb200_client.cc"), os.path.join(cpp, "tb200_grpc_client.cc")]
    deps = srcs + [os.path.join(cpp, h) for h in ("tb200_client.h", "tb200_grpc_client.h", "json.h", "pb.h", "grpc_service.pb.h")]
    deps += [os.path.join(HERE, "csrc", "h2.h"), os.path.join(ROOT, "include", "tb200.h"), LIB]
    if force or _newer(CLIENT_LIB, deps):
        gxx = shutil.which("g++") or "g++"
        cmd = [gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + os.path.join(ROOT, "include"), "-o", CLIENT_LIB] + srcs + [
               "-L" + LIBDIR, "-ltb200", "-Wl,-rpath,$ORIGIN", "-lpthread", "-lz"]
        if verbose:
            print(" ".join(cmd))
        subprocess.run(cmd, check=True)
    return CLIENT_LIB


if __name__ == "__main__":
    print(build_native(force="--force" in sys.argv, verbose=True))
    print(build_cpp_client(force="--force" in sys.argv, verbose=True))
