"""Compile the reference's own C++ example programs, UNMODIFIED and from where they lie under
/root/reference/src/c++/examples, against this repo's C++ front end (client_b200/cpp/compat
headers + libtb200client.so).  Outputs go to oracle/_ref/cc_examples/ (git-ignored; they travel
to the GPU box with the snapshot).  Test infrastructure: the binaries end with the examples' own
value checks ("PASS : ..."), so running them against the stand-in servers shows that code
written for the reference C++ HTTP / gRPC clients builds and behaves the same on the front end.

Not built: examples that need json_utils.h (RapidJSON, absent) or OpenCV (image clients).
"""

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = "/root/reference/src/c++/examples"
OUT = os.path.join(HERE, "_ref", "cc_examples")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
EXAMPLES = ["simple_http_infer_client", "simple_http_async_infer_client", "simple_http_string_infer_client",
            "simple_http_shm_client", "simple_http_sequence_sync_infer_client", "reuse_infer_objects_client"]
GRPC_EXAMPLES = ["simple_grpc_infer_client", "simple_grpc_async_infer_client", "simple_grpc_string_infer_client",
                 "simple_grpc_shm_client", "simple_grpc_health_metadata", "simple_grpc_sequence_sync_infer_client",
                 "simple_grpc_sequence_stream_infer_client", "simple_grpc_keepalive_client", "simple_grpc_custom_args_client",
                 "simple_grpc_custom_repeat", "simple_grpc_model_control"]
CUDA_EXAMPLES = ["simple_http_cudashm_client", "simple_grpc_cudashm_client"]
# the reference's own client test programs that need no gtest (src/c++/tests); they use
# cudaIpcMemHandle_t through the client headers, hence the CUDA include path and cudart
TESTS = ["client_timeout_test", "memory_leak_test"]  # cudaMalloc + cudaIpcGetMemHandle by hand, needs cudart


def build_ref_examples(force=False):
    """Returns {name: path}.  Without the reference tree or g++: the programs built earlier that are
    still in OUT (they travel with the working tree to machines that have no reference tree)."""
    if not os.path.isdir(REF) or shutil.which("g++") is None:
        found = {n: os.path.join(OUT, n) for n in EXAMPLES + GRPC_EXAMPLES + CUDA_EXAMPLES + TESTS}
        return {n: p for n, p in found.items() if os.access(p, os.X_OK)}
    from client_b200.build import build_cpp_client, build_native

    build_native()
    build_cpp_client()
    os.makedirs(OUT, exist_ok=True)
    cpp = os.path.join(ROOT, "client_b200", "cpp")
    libdir = os.path.join(ROOT, "client_b200", "lib")
    built = {}
    for name in EXAMPLES + GRPC_EXAMPLES + CUDA_EXAMPLES + TESTS:
        src = os.path.join(REF if name not in TESTS else os.path.join(os.path.dirname(REF), "tests"), name + ".cc")
        exe = os.path.join(OUT, name)
        deps = [src, os.path.join(libdir, "libtb200client.so"), os.path.join(cpp, "tb200_client.h"), os.path.join(cpp, "tb200_grpc_client.h")]
        if force or not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
            cmd = ["g++", "-O1", "-std=c++17", "-I" + os.path.join(cpp, "compat"), "-I" + cpp, src, "-o", exe,
                   "-L" + libdir, "-ltb200client", "-ltb200", "-Wl,-rpath,$ORIGIN/../../../client_b200/lib", "-lpthread", "-lrt"]
            if name in CUDA_EXAMPLES or name in TESTS:
                cmd += ["-I/usr/local/cuda/include", "-L/usr/local/cuda/lib64", "-lcudart"]
            subprocess.run(cmd, check=True)
        built[name] = exe
    return built


if __name__ == "__main__":
    for k, v in build_ref_examples(force=True).items():
        print(k, "->", v)
