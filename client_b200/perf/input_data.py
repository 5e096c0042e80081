"""User-supplied request data for the load generator: ``--input-data FILE|DIR``.

perf_analyzer accepts a path for ``--input-data`` (SURVEY.md section 10, "Data"); this module
restates the part of that format the device loop replays.  Parity with perf_analyzer is
unpinned.

JSON file: ``{"data": [entry, ...], "validation_data": [entry, ...]}`` (``validation_data``
optional, one entry per data entry).  An entry maps tensor names to

* a flat or nested list of values (row-major),
* ``{"content": <list>, "shape": [...]}``, or
* ``{"b64": "<base64 of the raw little-endian bytes>"}``.

Values are cast by numpy to the tensor's datatype; BF16 is truncated like
``utils.serialize_bf16_tensor``, BYTES strings are serialised like
``utils.serialize_byte_tensor``.  Directory: one entry, one file of raw bytes per input,
named after the input.

The parsed entries become one ``[entries, nbytes]`` uint8 array per tensor.  ``upload``
copies them once into device memory; from there the copy kernel writes each request's
entry into the slot's inputs and the check kernel compares its outputs with the expected
entry, so no tensor bytes cross PCIe per request.
"""

import base64
import binascii
import json
import os

import numpy as np

from ..utils import deserialize_bytes_tensor, serialize_bf16_tensor, serialize_byte_tensor, triton_to_np_dtype

SYNTHETIC = ("random", "zero")


class InputDataError(ValueError):
    """A data file or directory that does not fit the model or the run."""


def replay_entry(slot, request, lookahead, once, entries):
    """The entry request ``request`` (counted from 0) of slot ``slot`` carries: (slot + r) mod
    entries, with r = request mod lookahead when the inputs are written only once.  With
    look-ahead L, image g of generation k is request k * L + g.  The native device loop uses
    the same rule (tb200_loadgen_replay_entry)."""
    r = request % max(1, int(lookahead)) if once else request
    return (int(slot) + int(r)) % int(entries)


class InputData:
    """Parsed entries: ``inputs[name]`` and ``expected[name]`` are uint8 arrays
    [entries, nbytes], one row per entry."""

    def __init__(self, inputs, expected):
        self.inputs, self.expected = inputs, expected
        self.entries = next((len(a) for a in inputs.values()), 0)
        self._pool = {}

    def nbytes(self, name):
        arr = self.inputs.get(name)
        return int((arr if arr is not None else self.expected[name]).shape[1])

    def upload(self, ops):
        """Copy every tensor's entries into device memory once (tb200_device_alloc + copy +
        sync); later calls are no-ops."""
        if self._pool:
            return
        for kind, table in (("in", self.inputs), ("out", self.expected)):
            for name, arr in table.items():
                self._pool[(kind, name)] = ops.upload(arr)

    def input_ptr(self, name):
        """Device address of entry 0 of input ``name`` (entry e at + e * nbytes)."""
        return self._pool[("in", name)].ptr

    def expected_ptr(self, name):
        return self._pool[("out", name)].ptr

    def close(self):
        for buf in self._pool.values():
            buf.close()
        self._pool = {}


def load(path, inputs, outputs):
    """Parse a JSON file or a directory for the given input / output TensorSpecs."""
    if os.path.isdir(path):
        return read_directory(path, inputs)
    if not os.path.isfile(path):
        raise InputDataError("--input-data: '%s' is neither random, zero, a JSON file nor a directory" % path)
    try:
        with open(path, "rb") as fh:
            doc = json.loads(fh.read().decode("utf-8"))
    except (ValueError, UnicodeDecodeError) as ex:
        raise InputDataError("%s: not a JSON document (%s)" % (path, ex)) from None
    return parse_json(doc, inputs, outputs)


def read_directory(path, inputs):
    """One entry: the file named after each input holds its raw bytes."""
    table = {}
    for t in inputs:
        if t.datatype == "BYTES":
            raise InputDataError("directory %s: input '%s' is BYTES, which a raw file cannot size; pass BYTES data in a JSON file" % (path, t.name))
        f = os.path.join(path, t.name)
        if not os.path.isfile(f):
            raise InputDataError("directory %s: no file for input '%s'" % (path, t.name))
        raw = np.fromfile(f, dtype=np.uint8)
        if raw.size != t.nbytes:
            raise InputDataError("directory %s: file '%s' holds %d bytes, input '%s' of shape %s needs %d" % (path, t.name, raw.size, t.name, t.shape, t.nbytes))
        table[t.name] = raw.reshape(1, -1)
    return InputData(table, {})


def parse_json(doc, inputs, outputs):
    if not isinstance(doc, dict) or not isinstance(doc.get("data"), list):
        raise InputDataError("input data: expected an object with a 'data' list")
    data = doc["data"]
    if not data:
        raise InputDataError("input data: 'data' holds no entries")
    ins = _entries(data, {t.name: t for t in inputs}, "entry", "input", require_all=True)
    expected = {}
    if "validation_data" in doc:
        vd = doc["validation_data"]
        if not isinstance(vd, list) or len(vd) != len(data):
            raise InputDataError("input data: 'validation_data' has %s entries, 'data' has %d; they must pair up" % (
                len(vd) if isinstance(vd, list) else "no list of", len(data)))
        expected = _entries(vd, {t.name: t for t in outputs}, "validation entry", "output", require_all=False)
    return InputData(ins, expected)


def _entries(entries, specs, what, role, require_all):
    """[entries] of {name: value} -> {name: uint8 [entries, nbytes]}"""
    rows = {}
    names0 = None
    for e, entry in enumerate(entries):
        if isinstance(entry, list):
            raise InputDataError("%s %d is a list: 'data' made of lists of entries (perf_analyzer's multi-stream / sequence form) is not supported" % (what, e))
        if not isinstance(entry, dict):
            raise InputDataError("%s %d: expected an object mapping tensor names to values" % (what, e))
        for name in entry:
            if name not in specs:
                raise InputDataError("%s %d: '%s' is not an %s of the model" % (what, e, name, role))
        if require_all:
            for name in specs:
                if name not in entry:
                    raise InputDataError("%s %d: input '%s' is missing (every entry names every input)" % (what, e, name))
        elif names0 is None:
            names0 = sorted(entry)
        elif sorted(entry) != names0:
            raise InputDataError("%s %d names the outputs %s, %s 0 names %s; every entry must name the same outputs" % (what, e, sorted(entry), what, names0))
        for name, value in entry.items():
            raw = _encode(value, specs[name], "%s %d, tensor '%s'" % (what, e, name))
            prev = rows.get(name)
            if prev and len(raw) != len(prev[0]):
                raise InputDataError("%s %d, tensor '%s': BYTES serialise to %d bytes, %s 0 to %d; every entry must have the same byte size" % (
                    what, e, name, len(raw), what, len(prev[0])))
            rows.setdefault(name, []).append(raw)
    return {name: np.frombuffer(b"".join(r), dtype=np.uint8).reshape(len(r), -1) for name, r in rows.items()}


def _encode(value, t, where):
    """One tensor value of an entry -> its wire bytes."""
    count = int(np.prod(t.shape)) if t.shape else 1
    if isinstance(value, dict):
        if "b64" in value:
            try:
                raw = base64.b64decode(value["b64"], validate=True)
            except (binascii.Error, TypeError, ValueError) as ex:
                raise InputDataError("%s: 'b64' is not base64 (%s)" % (where, ex)) from None
            if t.datatype == "BYTES":
                try:
                    n = deserialize_bytes_tensor(raw).size
                except Exception as ex:  # noqa: BLE001 -- the codec raises its own exception type
                    raise InputDataError("%s: 'b64' is not a serialised BYTES tensor (%s)" % (where, ex)) from None
                if n != count:
                    raise InputDataError("%s: %d elements, the shape %s holds %d" % (where, n, t.shape, count))
            elif len(raw) != t.nbytes:
                raise InputDataError("%s: 'b64' decodes to %d bytes, %s of shape %s needs %d" % (where, len(raw), t.datatype, t.shape, t.nbytes))
            return raw
        if "content" not in value:
            raise InputDataError("%s: an object value needs 'content' or 'b64'" % where)
        if "shape" in value and [int(d) for d in value["shape"]] != t.shape:
            raise InputDataError("%s: shape %s differs from the run's shape %s" % (where, list(value["shape"]), t.shape))
        value = value["content"]
    try:
        if t.datatype == "BYTES":
            arr = np.array(value, dtype=np.object_).reshape(-1)
        else:
            arr = np.asarray(value, dtype=np.float32 if t.datatype == "BF16" else triton_to_np_dtype(t.datatype)).reshape(-1)
    except (ValueError, TypeError, OverflowError) as ex:
        raise InputDataError("%s: cannot convert the values to %s (%s)" % (where, t.datatype, ex)) from None
    if arr.size != count:
        raise InputDataError("%s: %d elements, the shape %s holds %d" % (where, arr.size, t.shape, count))
    if t.datatype == "BYTES":
        return serialize_byte_tensor(arr).item()
    if t.datatype == "BF16":
        return serialize_bf16_tensor(arr).item()
    return arr.astype(arr.dtype.newbyteorder("<"), copy=False).tobytes()
