"""client_b200 -- a GPU-native (H100, sm_90a), tritonclient-compatible client data plane.

The package mirrors the module layout of the reference Python client
(``tritonclient.http``, ``tritonclient.grpc``, ``tritonclient.utils``,
``tritonclient.utils.shared_memory``, ``tritonclient.utils.cuda_shared_memory``;
reference: src/python/library/tritonclient) and adds ``client_b200.perf``, the
device-side load generator.  Tensor marshalling that the reference does with
numpy + cudaMemcpy runs as sm_90a CUDA kernels behind the C ABI in
``include/tb200.h`` (``client_b200/lib/libtb200.so``).

``install_as_tritonclient()`` registers the modules under the ``tritonclient``
name so existing ``import tritonclient.http as httpclient`` code runs unchanged.
"""

import importlib
import sys

__version__ = "0.1.0"

_ALIASES = (
    "utils",
    "utils.shared_memory",
    "utils.cuda_shared_memory",
    "http",
    "grpc",
)


def install_as_tritonclient(include_cuda=True):
    """Expose this package as ``tritonclient`` in ``sys.modules``.

    Returns the list of module names that were registered.  The CUDA shared
    memory module needs libtb200.so; with ``include_cuda=False`` it is skipped
    (useful on hosts without the native build).
    """
    registered = []
    sys.modules["tritonclient"] = sys.modules[__name__]
    registered.append("tritonclient")
    for sub in _ALIASES:
        if sub.endswith("cuda_shared_memory") and not include_cuda:
            continue
        mod = importlib.import_module(__name__ + "." + sub)
        sys.modules["tritonclient." + sub] = mod
        registered.append("tritonclient." + sub)
    # the protobuf modules the gRPC package builds at import time (reference: generated
    # service_pb2 / service_pb2_grpc / model_config_pb2, tritonclient/grpc/__init__.py:29-73)
    for name in ("service_pb2", "service_pb2_grpc", "model_config_pb2"):
        mod = sys.modules.get(__name__ + ".grpc." + name)
        if mod is not None:
            sys.modules["tritonclient.grpc." + name] = mod
            registered.append("tritonclient.grpc." + name)
    return registered
