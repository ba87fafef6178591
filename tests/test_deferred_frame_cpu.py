"""Deferred framing (b200tfs_encode_requests_async): the tables the host writes for a request and the framing code
frame_requests_kernel runs over them, executed on the HOST (b200tfs_request_frame_deferred - the same inline source), against the
golden PredictRequests of the unmodified reference - including the ones with packed-varint inputs, whose length prefixes
depend on lengths only the counting kernel knows (here supplied by numpy)."""
import ctypes as C

import numpy as np
import pytest

import golden_util as G
from min_tfs_client import _native as N
from min_tfs_client.codec import _Prepared
from oracle import wire_oracle

REQ = G.load("requests.json")
_FIXED = (np.float32, np.float64, np.bool_, np.complex64, np.complex128)


def _varint(v):
    v &= (1 << 64) - 1
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def payload_bytes(arr, wire_dtype=None):
    """What the kernels put on the wire for one input (numpy restatement, test side)."""
    a = np.ascontiguousarray(arr)
    if wire_dtype is not None:
        a = a.astype(np.float32)
    if a.dtype == np.float32:
        u = a.view(np.uint32).copy()
        u[(u & 0x7FFFFFFF) > 0x7F800000] |= 0x00400000
        return u.tobytes()
    if a.dtype == np.bool_:
        return (a.view(np.uint8) != 0).astype(np.uint8).tobytes()
    if a.dtype.type in _FIXED:
        return a.tobytes()
    if a.dtype.kind == "U":
        return None                                     # pre-serialised TensorProto: the struct carries it
    return b"".join(_varint(int(v)) for v in a.ravel().tolist())    # sign-extended to 64 bits by the & in _varint


def deferred_wire(model, version, inputs, wire_dtype=None, grpc=False):
    lib = N.load()
    preps = [_Prepared(a, k.encode(), wire_dtype, False, False) for k, a in inputs]
    arr = (N.Tensor * max(len(preps), 1))(*[p.struct for p in preps])
    name = model.encode()
    req = N.Request(model_name=name, model_name_len=len(name), has_version=int(version is not None), order=N.ORDER_UPB, version=version or 0,
                    n_inputs=len(preps), flags=N.RF_GRPC_FRAME if grpc else 0, inputs=arr)
    pay = []
    for p, (k, a) in zip(preps, inputs):
        if p.struct.flags & N.F_PRESERIALIZED:
            pay.append(p.array.tobytes())
        else:
            pay.append(payload_bytes(a, wire_dtype))
    n = max(len(preps), 1)
    packed = (C.c_uint64 * n)(*[len(b) for b in pay] + [0] * (n - len(pay)))
    need = C.c_uint64()
    N.check(lib.b200tfs_request_arena_size(1, C.byref(req), C.byref(need)))      # sizes worst-case slots when an input is unmeasured
    cap = need.value + 4096
    buf = (C.c_uint8 * cap)()
    off, ln = C.c_uint64(), C.c_uint64()
    poff, plen = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    N.check(lib.b200tfs_request_frame_deferred(C.byref(req), packed, buf, cap, C.byref(off), C.byref(ln), poff, plen))
    raw = bytearray(bytes(buf))
    for i, b in enumerate(pay):
        assert plen[i] == len(b), (inputs[i][0], plen[i], len(b))
        a = np.asarray(inputs[i][1])
        if a.dtype.kind in "iu" and 0 < a.size <= 32:
            # a tiny packed-varint input (a label, an id): the framing code counted AND wrote it itself - nothing to lay in
            assert bytes(raw[poff[i]: poff[i] + len(b)]) == b, inputs[i][0]
        else:
            raw[poff[i]: poff[i] + len(b)] = b
    return bytes(raw[off.value: off.value + ln.value]), off.value, [poff[i] for i in range(len(pay))], [plen[i] for i in range(len(pay))]


@pytest.mark.parametrize("name", list(REQ))
def test_deferred_frame_matches_golden(name):
    case = REQ[name]
    inputs = [(k, G.make_array(r)) for k, r in case["inputs"]]
    wd = "DT_FLOAT" if case.get("wire_dtype") == "DT_FLOAT" else None
    if any(int(np.prod(a.shape)) > (1 << 21) for _, a in inputs):
        pytest.skip("full-size case: covered on the GPU")
    wire, off, poff, plen = deferred_wire(case["model_name"], case["model_version"], inputs, wd)
    G.check_wire(wire, case["wire"], name)
    fixed = [i for i in range(len(plen)) if inputs[i][1].dtype.type in _FIXED and plen[i]]
    if fixed:      # the record is placed so that a largest fixed-width payload starts 128-byte aligned (like the host planner's place_record)
        top = max(plen[i] for i in fixed)
        assert any(poff[i] % 128 == 0 for i in fixed if plen[i] == top)


def test_deferred_frame_lengths_and_layout_across_varint_boundaries():
    """The dependent varints (payload length, TensorProto length, entry length, gRPC length) each change size as the packed length
    crosses 127 / 128, 16383 / 16384, ...: every side of those edges, against the oracle, with the payloads placed as the encoder
    places them."""
    for n in (1, 100, 127, 128, 129, 5000, 16380, 16383, 16384, 16390, 70000):
        ids = (np.arange(n, dtype=np.int64) % 100)              # one byte each: packed length == n
        x = np.arange(6, dtype=np.float32).reshape(2, 3)
        inputs = [("ids", ids), ("x", x), ("neg", np.array([-1, 5, -300], dtype=np.int32))]
        want = wire_oracle.encode_predict_request("m", 7, inputs)
        wire, off, poff, plen = deferred_wire("m", 7, inputs)
        assert wire == want, n
        wire5, *_ = deferred_wire("m", 7, inputs, grpc=True)
        assert wire5 == b"\x00" + len(want).to_bytes(4, "big") + want
        # the varint input LAST on the wire: the fixed-width payload in front of it starts 128-byte aligned, the varint payload
        # ends the record
        last = [("img", x), ("z_ids", ids)]
        want = wire_oracle.encode_predict_request("m", 7, last)
        wire, off, poff, plen = deferred_wire("m", 7, last)
        assert wire == want, n
        assert poff[0] % 128 == 0 and off + len(want) == poff[1] + plen[1], (n, off, poff)
        assert deferred_wire("m", 7, last, grpc=True)[0] == b"\x00" + len(want).to_bytes(4, "big") + want
        # a varint input alone: with no fixed-width payload, its own payload starts 128-byte aligned
        want = wire_oracle.encode_predict_request("", None, [("only", ids)])
        wire, off, poff, plen = deferred_wire("", None, [("only", ids)])
        assert wire == want and poff[0] % 128 == 0 and off + len(want) == poff[0] + plen[0], (n, off, poff)
    # a request whose only inputs are empty or zero-element tensors, and one with no inputs at all
    assert deferred_wire("m", None, [("e", np.zeros((0, 3), np.int64))])[0] == wire_oracle.encode_predict_request("m", None, [("e", np.zeros((0, 3), np.int64))])
    assert deferred_wire("", 0, [])[0] == wire_oracle.encode_predict_request("", 0, [])
