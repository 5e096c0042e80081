"""CUDA shared memory (CUDA IPC) regions.

Drop-in for ``tritonclient.utils.cuda_shared_memory`` (reference:
src/python/library/tritonclient/utils/cuda_shared_memory/__init__.py:107-429):
same functions, arguments, handle attributes and exception texts.  The data
plane is libtb200 (include/tb200.h): regions, pinned multi-threaded staging for
host arrays, and -- beyond the reference -- device-side producers that write
straight into a region (``fill_shared_memory_region``,
``set_shared_memory_region_from_image``) and device-side validation
(``check_shared_memory_region``), so no numpy serialise or per-request H2D sits
on the request path.
"""

import base64
import ctypes

import numpy as np

from ... import _native
from .. import _dlpack
from .._shared_memory_tensor import SharedMemoryTensor
from ._utils import (
    CudaSharedMemoryException,
    CudaSharedMemoryRegion,
    CudaStream,
    IpcMemHandle,
    maybe_set_device,
)

allocated_shm_regions = []
_dlpack_stream = {}


def _get_or_create_global_cuda_stream(device_id):
    if device_id not in _dlpack_stream:
        _dlpack_stream[device_id] = CudaStream(device_id)
    return _dlpack_stream[device_id]


def _ctx(device_id):
    return _native.default_context(device_id)


_device_ops = {}


def _ops(device_id):
    """One DeviceOps per device (it caches its pinned scratch buffers)."""
    ops = _device_ops.get(device_id)
    if ops is None:
        from ...device import DeviceOps

        ops = _device_ops[device_id] = DeviceOps(_ctx(device_id))
    return ops


def _is_device_supported(device):
    return int(device[0]) in (
        _dlpack.DLDeviceType.kDLCPU,
        _dlpack.DLDeviceType.kDLCUDA,
        _dlpack.DLDeviceType.kDLCUDAHost,
    )


def create_shared_memory_region(triton_shm_name, byte_size, device_id):
    """Create a CUDA shared memory region of ``byte_size`` bytes on GPU
    ``device_id`` and export its IPC handle (reference :107-149).

    Raises
    ------
    CudaSharedMemoryException
        If unable to create the cuda shared memory region on the device.
    """
    try:
        lib = _native.load()
        region = ctypes.c_void_p()
        _native.check(
            lib.tb200_region_create(
                str(triton_shm_name).encode("utf-8"), int(byte_size), int(device_id), ctypes.byref(region)
            )
        )
        raw = (ctypes.c_uint8 * _native.IPC_HANDLE_BYTES)()
        _native.check(lib.tb200_region_ipc_handle(region, raw))
        handle = CudaSharedMemoryRegion(
            triton_shm_name,
            IpcMemHandle(bytes(raw)),
            int(lib.tb200_region_base(region)),
            int(byte_size),
            int(device_id),
            native_region=region,
        )
        allocated_shm_regions.append(handle)
    except Exception as ex:
        if isinstance(ex, CudaSharedMemoryException):
            raise
        raise CudaSharedMemoryException("unable to create cuda shared memory handle") from ex
    return handle


def get_raw_handle(cuda_shm_handle):
    """base64 of the 64-byte cudaIpcMemHandle_t -- the value
    ``register_cuda_shared_memory`` sends (reference :152-170)."""
    return base64.b64encode(cuda_shm_handle._cuda_shm_handle.reserved)


def _host_chunks(input_values):
    """(keepalive objects, pointers, sizes) of the arrays laid out back to back
    (reference :203-230)."""
    keep, ptrs, sizes = [], [], []
    for input_value in input_values:
        flat = np.ascontiguousarray(input_value).reshape(-1)
        if flat.dtype == np.object_:
            # serialised BYTES tensor (tritonclient.utils.serialize_byte_tensor)
            payload = flat.item()
            buf = (ctypes.c_char * len(payload)).from_buffer_copy(payload) if len(payload) else None
            keep.append(buf)
            ptrs.append(ctypes.addressof(buf) if buf is not None else 0)
            sizes.append(len(payload))
        else:
            keep.append(flat)
            ptrs.append(flat.ctypes.data)
            sizes.append(flat.size * flat.itemsize)
    return keep, ptrs, sizes


def set_shared_memory_region(cuda_shm_handle, input_values):
    """Copy numpy arrays back to back into the region, from offset 0; returns
    when the bytes are visible on the device (reference :173-239).

    Raises
    ------
    CudaSharedMemoryException
        If unable to set values in the cuda shared memory region.
    """
    if not isinstance(input_values, (list, tuple)):
        raise CudaSharedMemoryException("input_values must be specified as a numpy array")
    for input_value in input_values:
        if not isinstance(input_value, (np.ndarray,)):
            raise CudaSharedMemoryException(
                "input_values must be specified as a list/tuple of numpy arrays"
            )
    try:
        if len(input_values) == 1 and input_values[0].dtype != np.object_ and input_values[0].flags.c_contiguous:
            # one plain array: no gather table
            arr = input_values[0]
            _native.check(
                _native.load().tb200_region_write_host(
                    _ctx(cuda_shm_handle._device_id).handle, cuda_shm_handle._native, 0, arr.ctypes.data, arr.nbytes
                )
            )
            return
        keep, ptrs, sizes = _host_chunks(input_values)
        n = len(ptrs)
        c_ptrs = (ctypes.c_void_p * max(n, 1))(*ptrs)
        c_sizes = (ctypes.c_uint64 * max(n, 1))(*sizes)
        _native.check(
            _native.load().tb200_region_write_host_gather(
                _ctx(cuda_shm_handle._device_id).handle, cuda_shm_handle._native, 0, n, c_ptrs, c_sizes
            )
        )
        del keep
    except Exception as ex:
        if isinstance(ex, CudaSharedMemoryException):
            raise
        raise CudaSharedMemoryException("unable to set values in cuda shared memory") from ex
    return


def _read_region(cuda_shm_handle, offset, nbytes):
    host = np.empty(nbytes, dtype=np.uint8)
    _native.check(
        _native.load().tb200_region_read_host(
            _ctx(cuda_shm_handle._device_id).handle,
            cuda_shm_handle._native,
            int(offset),
            host.ctypes.data,
            int(nbytes),
        )
    )
    return host


def get_contents_as_numpy(cuda_shm_handle, datatype, shape):
    """numpy array holding the first ``prod(shape)`` elements of the region.
    Only the requested bytes cross PCIe (the reference copies the whole region,
    :266-276) (reference :242-325).
    """
    fixed = (datatype != np.object_) and (datatype != np.bytes_)
    if fixed:
        requested = int(np.prod(shape)) * np.dtype(datatype).itemsize
        if cuda_shm_handle._byte_size < requested:
            raise CudaSharedMemoryException(
                "The size of the shared memory region is insufficient to provide numpy array with requested size"
            )
        nbytes = requested
    else:
        # BYTES: the <u32 length><payload> chain is walked on the device (tb200_bytes_decode_async);
        # offsets + packed payloads come back instead of the whole region (reference :306-323
        # copies the region and walks it with struct.unpack_from)
        count = max(int(np.prod(shape)), 1)
        try:
            offsets, packed, _ = _ops(cuda_shm_handle._device_id).bytes_decode(
                cuda_shm_handle._base_addr, cuda_shm_handle._byte_size, count)
        except Exception as ex:
            raise CudaSharedMemoryException("failed to read cuda shared memory results") from ex
        strs = [packed[offsets[i]:offsets[i + 1]] for i in range(count)]
        return np.reshape(np.array(strs, dtype=object), shape)
    try:
        host = _read_region(cuda_shm_handle, 0, nbytes)
    except Exception as ex:
        if isinstance(ex, CudaSharedMemoryException):
            raise
        raise CudaSharedMemoryException("failed to read cuda shared memory results") from ex

    if nbytes == 0:
        return np.empty(shape, dtype=datatype)
    return host.view(np.dtype(datatype)).reshape(shape)


def set_shared_memory_region_from_dlpack(cuda_shm_handle, input_values):
    """Copy DLPack tensors (CPU, CUDA or pinned host; contiguous C order) back to
    back into the region (reference :328-388)."""
    offset_current = 0
    for input_value in input_values:
        dl_device = _dlpack.get_dlpack_device(input_value)
        stream = _get_or_create_global_cuda_stream(cuda_shm_handle._device_id)
        if dl_device is not None and not _is_device_supported(dl_device):
            raise CudaSharedMemoryException(
                "DLPack device type {} is not supported".format(dl_device[0])
            )
        # the producer orders its pending work before our stream (DLPack protocol)
        dlcapsule = _dlpack.get_dlpack_capsule(input_value, stream.getPtr())
        dmt = _dlpack.get_managed_tensor(dlcapsule)
        if not _dlpack.is_contiguous_data(
            dmt.dl_tensor.ndim, dmt.dl_tensor.shape, dmt.dl_tensor.strides
        ):
            raise CudaSharedMemoryException(
                "DLPack tensor is not contiguous. Only contiguous DLPack tensors that are stored in C-Order are supported."
            )
        byte_size = _dlpack.get_byte_size(dmt.dl_tensor.dtype, dmt.dl_tensor.ndim, dmt.dl_tensor.shape)
        data_ptr = (dmt.dl_tensor.data or 0) + dmt.dl_tensor.byte_offset
        try:
            _native.check(
                _native.load().tb200_region_write_ptr(
                    _ctx(cuda_shm_handle._device_id).handle,
                    cuda_shm_handle._native,
                    offset_current,
                    data_ptr,
                    byte_size,
                )
            )
        except Exception as ex:
            raise CudaSharedMemoryException("unable to set values in cuda shared memory") from ex
        offset_current += byte_size
    return


def as_shared_memory_tensor(cuda_shm_handle, datatype, shape):
    """DLPack-exportable view of the region (reference :391-399)."""
    return SharedMemoryTensor(
        datatype,
        shape,
        cuda_shm_handle._base_addr,
        0,
        cuda_shm_handle._byte_size,
        cuda_shm_handle._device_id,
    )


def allocated_shared_memory_regions():
    """All regions allocated through this module and not destroyed (reference :402-411)."""
    return allocated_shm_regions


def destroy_shared_memory_region(cuda_shm_handle):
    """Forget the region; its device memory is released with the handle object
    (reference :414-429)."""
    allocated_shm_regions.remove(cuda_shm_handle)
    del cuda_shm_handle
    return


# ---------------------------------------------------------------------------
# GPU-native producers / consumers (no counterpart in the reference: there the
# data always starts in a numpy array and is copied with cudaMemcpy).
# ---------------------------------------------------------------------------
def fill_shared_memory_region(
    cuda_shm_handle, datatype, shape=None, offset=0, seed=0, stream_id=0, mode="random",
    low=0.0, high=None, byte_size=None, sync=True,
):
    """Generate a synthetic tensor directly inside the region (Philox4x32-10,
    see DESIGN.md "fill contract").

    ``mode``: "random" (floats uniform in [low, high), default the unit
    interval; integers uniform in [low, high), default raw bits) or "zero".
    """
    from ...device import make_fill_job

    es = _native.DTYPE_SIZES.get(datatype)
    if es is None:
        raise CudaSharedMemoryException("datatype '{}' cannot be generated on the device".format(datatype))
    nbytes = int(byte_size) if byte_size is not None else int(np.prod(shape)) * es
    if offset < 0 or offset + nbytes > cuda_shm_handle._byte_size:
        raise CudaSharedMemoryException(
            "The size of the shared memory region is insufficient for the generated tensor"
        )
    job = make_fill_job(cuda_shm_handle._base_addr + offset, nbytes, datatype, stream_id, mode, low, high)
    ops = _ops(cuda_shm_handle._device_id)
    ops.fill([job], seed=seed)
    if sync:
        ops.sync()


def set_shared_memory_region_from_image(
    cuda_shm_handle, images_u8_nhwc, datatype="FP32", scaling="NONE", layout="NCHW", offset=0, resize=None
):
    """uint8 NHWC host images -> scaled ``datatype`` tensor in ``layout`` inside
    the region.  Only the uint8 bytes cross PCIe; resize, cast, scaling and the HWC->CHW
    transpose run in one kernel — the whole of ``image_client.preprocess``
    (src/python/examples/image_client.py:154-193) after the decode.

    ``resize=(h, w)``: ``Image.resize((w, h), Image.BILINEAR)`` first, bit-identical to
    Pillow (antialiased triangle filter, horizontal pass first, 8-bit intermediate)."""
    arr = np.ascontiguousarray(images_u8_nhwc)
    if arr.dtype != np.uint8 or arr.ndim not in (3, 4):
        raise CudaSharedMemoryException("images must be a uint8 array of shape [N,]H,W,C")
    if arr.ndim == 3:
        arr = arr[None]
    n, h, w, c = arr.shape
    out_h, out_w = (int(resize[0]), int(resize[1])) if resize is not None else (h, w)
    es = _native.DTYPE_SIZES[datatype]
    if offset + n * out_h * out_w * c * es > cuda_shm_handle._byte_size:
        raise CudaSharedMemoryException(
            "The size of the shared memory region is insufficient for the packed images"
        )
    ops = _ops(cuda_shm_handle._device_id)
    try:
        if resize is not None:
            ops.resize_pack_image_from_host(cuda_shm_handle._base_addr + offset, datatype, layout, arr, out_h, out_w, scaling)
        else:
            ops.pack_image_from_host(cuda_shm_handle._base_addr + offset, datatype, layout, arr, scaling)
    except _native.NativeError as ex:
        raise CudaSharedMemoryException(str(ex)) from ex
    ops.sync()


def check_shared_memory_region(cuda_shm_handle, kind="sum", byte_size=None, offset=0, expected=None, defer=False):
    """Validate / checksum region contents on the device; returns a dict with
    ``mismatches``, ``sum``, ``xor32``, ``argmax``, ``max_value``.  ``expected``
    (another region handle) is compared byte-wise for ``kind='equal'``.

    ``defer=True`` only launches the check and returns a callable giving that dict: device work queued
    before it is called (``fill_shared_memory_region(..., sync=False)`` for the next request) is waited
    for in the same synchronisation.  One deferred check at a time per device."""
    nbytes = int(byte_size) if byte_size is not None else cuda_shm_handle._byte_size - offset
    ops = _ops(cuda_shm_handle._device_id)
    b = expected._base_addr if expected is not None else 0
    if defer:
        return ops.check_one_deferred(kind, cuda_shm_handle._base_addr + offset, nbytes, b=b)
    return ops.check_one(kind, cuda_shm_handle._base_addr + offset, nbytes, b=b)


def classify_shared_memory_region(cuda_shm_handle, datatype, shape, class_count, offset=0, labels=None):
    """Top-``class_count`` classification of an output that stayed in CUDA shared memory.

    The server refuses ``class_count`` on shared-memory outputs
    (http/_requested_output.py:84-85), so this does on the device what the server's
    classification extension does for inline outputs: the last axis of ``shape`` is the
    class axis, every leading index is one batch item.  Returns a ``np.object_`` array of
    shape ``shape[:-1] + [class_count]`` holding ``b"<value>:<index>[:<label>]"`` — the
    form ``InferResult.as_numpy`` gives for a classification output and
    src/python/examples/image_client.py:196-216 parses.  Only 8 bytes per class leave the GPU.
    """
    from ... import _native as nat

    if datatype not in ("FP32", "FP16", "BF16"):
        raise CudaSharedMemoryException("classification needs an FP32, FP16 or BF16 tensor")
    shape = [int(d) for d in shape]
    classes = shape[-1]
    batch = int(np.prod(shape[:-1])) if len(shape) > 1 else 1
    es = nat.DTYPE_SIZES[datatype]
    if offset + batch * classes * es > cuda_shm_handle._byte_size:
        raise CudaSharedMemoryException(
            "The size of the shared memory region is insufficient to provide numpy array with requested size"
        )
    ops = _ops(cuda_shm_handle._device_id)
    base = cuda_shm_handle._base_addr + offset
    values, indices = ops.topk([(base + i * classes * es, classes, datatype) for i in range(batch)], class_count)
    out = np.empty((batch, class_count), dtype=np.object_)
    for i in range(batch):
        for j in range(class_count):
            idx = int(indices[i, j])
            if idx == 0xFFFFFFFF:
                out[i, j] = b""
                continue
            text = "%f:%d" % (float(values[i, j]), idx)
            if labels is not None:
                text += ":" + str(labels[idx])
            out[i, j] = text.encode()
    return out.reshape(shape[:-1] + [class_count])

