"""--input-data FILE|DIR on the CPU: parsing of every value form against the utils serialisers,
every rejection with its message, and the entry rule (which entry request r of slot s carries)
pinned for the native device loop and the Python engine's SlotSet against one table."""

import base64
import json

import numpy as np
import pytest

from client_b200.perf import cli
from client_b200.perf import input_data as idata
from client_b200.perf.loadgen import SlotSet, TensorSpec
from client_b200.utils import serialize_bf16_tensor, serialize_byte_tensor


def _spec(name, dtype, shape=(2, 3)):
    return TensorSpec(name, dtype, list(shape))


VALUES = {
    "INT32": [[1, -2, 3], [4, 5, -6]],
    "INT64": [[1, -(2 ** 40), 3], [4, 5, 2 ** 62]],
    "FP16": [[0.5, -1.25, 3.0], [65504.0, 0.0, -0.001]],
    "FP32": [[0.1, -2.5, 3.25], [1e30, -0.0, 7.0]],
    "BF16": [[0.1, -2.5, 3.3], [1e30, -0.0, 7.7]],
    "BOOL": [[True, False, True], [False, False, True]],
    "BYTES": [["a", "bc", ""], ["dé", "xyz", "0"]],
}


def _expected(dtype, nested):
    if dtype == "BYTES":
        return serialize_byte_tensor(np.array(nested, dtype=np.object_)).item()
    if dtype == "BF16":
        return serialize_bf16_tensor(np.array(nested, dtype=np.float32)).item()
    npt = {"INT32": np.int32, "INT64": np.int64, "FP16": np.float16, "FP32": np.float32, "BOOL": np.bool_}[dtype]
    return np.array(nested, dtype=npt).tobytes()


@pytest.mark.parametrize("dtype", sorted(VALUES))
def test_every_value_form_matches_the_serialisers(dtype):
    t = _spec("X", dtype)
    nested = VALUES[dtype]
    want = _expected(dtype, nested)
    flat = [v for row in nested for v in row]
    forms = [nested, flat, {"content": flat, "shape": [2, 3]}, {"content": nested}, {"b64": base64.b64encode(want).decode()}]
    data = idata.parse_json({"data": [{"X": f} for f in forms]}, [t], [])
    assert data.entries == len(forms)
    for e in range(len(forms)):
        assert data.inputs["X"][e].tobytes() == want, (dtype, forms[e])


def test_validation_data_and_entry_count():
    ins, outs = [_spec("A", "INT32", [4])], [_spec("Y", "INT32", [4]), _spec("Z", "FP32", [4])]
    doc = {"data": [{"A": [i, i, i, i]} for i in range(3)], "validation_data": [{"Y": [2 * i] * 4} for i in range(3)]}
    data = idata.parse_json(doc, ins, outs)
    assert data.entries == 3 and set(data.expected) == {"Y"}
    assert data.expected["Y"].shape == (3, 16) and data.expected["Y"][2].view(np.int32).tolist() == [4, 4, 4, 4]
    assert data.nbytes("A") == 16 and data.nbytes("Y") == 16


def test_json_file_and_directory(tmp_path):
    ins = [_spec("A", "INT32", [4]), _spec("B", "FP32", [2])]
    f = tmp_path / "data.json"
    f.write_text(json.dumps({"data": [{"A": [1, 2, 3, 4], "B": [0.5, 1.5]}]}))
    data = idata.load(str(f), ins, [])
    assert data.entries == 1 and data.inputs["B"][0].view(np.float32).tolist() == [0.5, 1.5]
    d = tmp_path / "dir"
    d.mkdir()
    (d / "A").write_bytes(np.arange(4, dtype=np.int32).tobytes())
    (d / "B").write_bytes(np.ones(2, np.float32).tobytes())
    data = idata.load(str(d), ins, [])
    assert data.entries == 1 and data.expected == {}
    assert data.inputs["A"][0].view(np.int32).tolist() == [0, 1, 2, 3]


REJECTIONS = [
    ({"entries": []}, "expected an object with a 'data' list"),
    ({"data": []}, "'data' holds no entries"),
    ({"data": [[{"A": [1, 2, 3, 4]}]]}, "entry 0 is a list: .*multi-stream / sequence form"),
    ({"data": [{"A": [1, 2, 3, 4], "S": ["x"]}, 3]}, "entry 1: expected an object"),
    ({"data": [{"A": [1, 2, 3, 4]}]}, "entry 0: input 'S' is missing"),
    ({"data": [{"A": [1, 2, 3, 4], "S": ["x"], "Q": [1]}]}, "entry 0: 'Q' is not an input of the model"),
    ({"data": [{"A": {"content": [1, 2, 3, 4], "shape": [2, 2]}, "S": ["x"]}]}, r"entry 0, tensor 'A': shape \[2, 2\] differs from the run's shape \[4\]"),
    ({"data": [{"A": [1, 2, 3], "S": ["x"]}]}, r"entry 0, tensor 'A': 3 elements, the shape \[4\] holds 4"),
    ({"data": [{"A": {"b64": base64.b64encode(b"123").decode()}, "S": ["x"]}]}, "entry 0, tensor 'A': 'b64' decodes to 3 bytes, INT32 of shape \\[4\\] needs 16"),
    ({"data": [{"A": {"b64": "not base64!"}, "S": ["x"]}]}, "entry 0, tensor 'A': 'b64' is not base64"),
    ({"data": [{"A": {"shape": [4]}, "S": ["x"]}]}, "entry 0, tensor 'A': an object value needs 'content' or 'b64'"),
    ({"data": [{"A": ["x", 1, 2, 3], "S": ["x"]}]}, "entry 0, tensor 'A': cannot convert the values to INT32"),
    ({"data": [{"A": [1, 2, 3, 4], "S": ["x"]}, {"A": [1, 2, 3, 4], "S": ["xy"]}]},
     "entry 1, tensor 'S': BYTES serialise to 6 bytes, entry 0 to 5"),
    ({"data": [{"A": [1, 2, 3, 4], "S": ["x"]}], "validation_data": []}, "'validation_data' has 0 entries, 'data' has 1"),
    ({"data": [{"A": [1, 2, 3, 4], "S": ["x"]}] * 2, "validation_data": [{"Y": [1]}, {"Z": [1]}]},
     r"validation entry 1 names the outputs \['Z'\], validation entry 0 names \['Y'\]"),
    ({"data": [{"A": [1, 2, 3, 4], "S": ["x"]}], "validation_data": [{"W": [1]}]}, "validation entry 0: 'W' is not an output of the model"),
]


@pytest.mark.parametrize("doc,message", REJECTIONS, ids=[m.split(":")[0][:40] for _, m in REJECTIONS])
def test_every_rejection_names_entry_and_tensor(doc, message):
    ins = [_spec("A", "INT32", [4]), _spec("S", "BYTES", [1])]
    outs = [_spec("Y", "INT32", [1]), _spec("Z", "INT32", [1])]
    with pytest.raises(idata.InputDataError, match=message):
        idata.parse_json(doc, ins, outs)


def test_directory_rejections(tmp_path):
    (tmp_path / "A").write_bytes(b"\0" * 12)
    with pytest.raises(idata.InputDataError, match="file 'A' holds 12 bytes, input 'A' of shape \\[4\\] needs 16"):
        idata.read_directory(str(tmp_path), [_spec("A", "INT32", [4])])
    with pytest.raises(idata.InputDataError, match="no file for input 'B'"):
        idata.read_directory(str(tmp_path), [_spec("B", "INT32", [3])])
    with pytest.raises(idata.InputDataError, match="input 'S' is BYTES.*JSON file"):
        idata.read_directory(str(tmp_path), [_spec("S", "BYTES", [1])])
    with pytest.raises(idata.InputDataError, match="neither random, zero, a JSON file nor a directory"):
        idata.load(str(tmp_path / "missing.json"), [], [])
    (tmp_path / "bad.json").write_text("{not json")
    with pytest.raises(idata.InputDataError, match="not a JSON document"):
        idata.load(str(tmp_path / "bad.json"), [], [])


def test_validation_needs_cuda_shared_memory():
    data = idata.parse_json({"data": [{"A": [1]}], "validation_data": [{"Y": [1]}]}, [_spec("A", "INT32", [1])], [_spec("Y", "INT32", [1])])
    for shm in ("none", "system"):
        with pytest.raises(idata.InputDataError, match="only with --shared-memory cuda"):
            SlotSet([_spec("A", "INT32", [1])], [_spec("Y", "INT32", [1])], 2, shm, 0, "random", 0, replay=data)


# The entry rule: request r of slot s carries entry (s + r) mod N; with the inputs written once,
# r is taken mod the look-ahead L.  N = 5 entries, slots 0..2, requests 0..7.
N = 5
TABLE = {
    (1, False): {0: [0, 1, 2, 3, 4, 0, 1, 2], 1: [1, 2, 3, 4, 0, 1, 2, 3], 2: [2, 3, 4, 0, 1, 2, 3, 4]},
    (4, False): {0: [0, 1, 2, 3, 4, 0, 1, 2], 1: [1, 2, 3, 4, 0, 1, 2, 3], 2: [2, 3, 4, 0, 1, 2, 3, 4]},
    (1, True): {0: [0] * 8, 1: [1] * 8, 2: [2] * 8},
    (4, True): {0: [0, 1, 2, 3, 0, 1, 2, 3], 1: [1, 2, 3, 4, 1, 2, 3, 4], 2: [2, 3, 4, 0, 2, 3, 4, 0]},
}


@pytest.mark.parametrize("lookahead,once", sorted(TABLE))
def test_entry_rule_of_the_native_loop(lookahead, once):
    from client_b200 import _native

    lib = _native.load()
    for s, want in TABLE[(lookahead, once)].items():
        assert [idata.replay_entry(s, r, lookahead, once, N) for r in range(8)] == want
        assert [int(lib.tb200_loadgen_replay_entry(s, r, lookahead, 1 if once else 0, N)) for r in range(8)] == want


class HostStaging:
    """Test double for the pinned staging buffer (the CPU box has no device)."""

    def allocate(self, nbytes):
        self.buf = np.zeros(nbytes, np.uint8)

    def view(self, off, n):
        return memoryview(self.buf)[off:off + n]


@pytest.mark.parametrize("lookahead,once", sorted(TABLE))
def test_entry_rule_of_slotset(lookahead, once):
    """SlotSet (the Python engine, and the layout the native loop copies into): every generation
    writes image g of slot s from entry (s + kL + g) mod N; the transport sends the images in order."""
    ins = [_spec("A", "INT32", [2]), _spec("B", "INT64", [1])]
    data = idata.parse_json({"data": [{"A": [e, -e], "B": [100 + e]} for e in range(N)]}, ins, [])
    ss = SlotSet(ins, [], 3, "none", 0, "random", 0, staging=HostStaging(), lookahead=lookahead, replay=data)
    sent = {s: [] for s in range(3)}
    ss.generate([0, 1, 2])
    for _ in range(8 // lookahead):
        for s in range(3):
            for g in range(lookahead):
                a = np.frombuffer(bytes(ss._staging.view(ss.input_offset(s, 0, g), 8)), np.int32)
                b = np.frombuffer(bytes(ss._staging.view(ss.input_offset(s, 1, g), 8)), np.int64)
                assert a.tolist() == [a[0], -a[0]] and b[0] == 100 + a[0]
                sent[s].append(int(a[0]))
        if not once:
            ss.generate([0, 1, 2])
    assert sent == TABLE[(lookahead, once)]


def test_input_data_flag_keeps_random_and_zero():
    ap = cli.build_parser()
    assert ap.parse_args(["-m", "m"]).input_data == "random"
    assert ap.parse_args(["-m", "m", "--input-data", "zero"]).input_data == "zero"
    assert ap.parse_args(["-m", "m", "--input-data", "random"]).input_data == "random"
    assert ap.parse_args(["-m", "m", "--input-data", "/tmp/x.json"]).input_data == "/tmp/x.json"
    assert idata.SYNTHETIC == ("random", "zero")


def test_exit_status():
    assert cli.exit_status([{"validation_mismatches": 0}, {}]) == 0
    assert cli.exit_status([{"validation_mismatches": 0}, {"validation_mismatches": 3}]) == 1
