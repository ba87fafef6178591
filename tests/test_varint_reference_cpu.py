"""Pins tests/varint_ref.py - the packed-varint reference the edge tests compare the device kernels with - against the protobuf
runtime and the reference's algorithm (oracle/ref_port.py), pins the kernel geometry it mirrors against the sources, and checks
the CPU oracle's error order for one output against ref_port."""
import os
import re

import numpy as np
import pytest
from google.protobuf.message import DecodeError

import golden_util as G
import varint_ref as V
from oracle import ref_port, wire_oracle
from tensorflow.core.framework import tensor_pb2

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "min-tfs-client_b200", "csrc")
FIELD_NAME = {7: "int_val", 10: "int64_val", 16: "uint32_val", 17: "uint64_val", 11: "bool_val", 13: "half_val"}


def edge_values(dtype):
    """0, 1, -1, min, max and 2^(7k) +- 1 inside the dtype's range, as the tensor's numpy type."""
    np_type = V.DTYPES[dtype][1]
    if dtype == 10:
        return np.array([False, True, True, False], dtype=np.bool_)
    if dtype == 19:
        return np.array([0, 1, 0x3C00, 0x7BFF, 0x7C00, 0x7E00, 0x8000, 0xFBFF, 0xFFFF, 127, 128, 16383, 16384], np.uint16).view(np.float16)
    info = np.iinfo(np_type)
    cand = [0, 1, -1, info.min, info.max, info.min + 1, info.max - 1]
    for k in range(1, 10):
        cand += [(1 << (7 * k)) - 1, 1 << (7 * k), (1 << (7 * k)) + 1, -(1 << (7 * k)), -(1 << (7 * k)) - 1]
    return np.array([v for v in cand if info.min <= v <= info.max], dtype=np_type)


def protobuf_tensor(values, dtype):
    tp = tensor_pb2.TensorProto(dtype=dtype)
    tp.tensor_shape.dim.add(size=values.size)
    src = values.view(np.uint16) if dtype == 19 else values
    getattr(tp, FIELD_NAME[V.DTYPES[dtype][0]]).extend([v.item() for v in src.reshape(-1)])
    return tp


@pytest.mark.parametrize("dtype", sorted(V.DTYPES), ids=[V.NAMES[d] for d in sorted(V.DTYPES)])
def test_encode_matches_the_protobuf_runtime(dtype):
    vals = edge_values(dtype)
    rng = np.random.default_rng(dtype)
    more = rng.permutation(np.concatenate([vals] * 5))
    for x in (vals, more, vals[:1], vals[:0]):
        want = protobuf_tensor(x, dtype).SerializeToString()
        assert V.tensor_proto(x, dtype) == want
        assert len(want) == len(V.tensor_header(dtype, [x.size], V.packed_len(x, dtype))) + V.packed_len(x, dtype)
        if dtype not in (19, 10):      # ref_port's own element loop (half_val: the quirk; bool: .item() is the same)
            assert ref_port.encode_tensor_proto(x) == want
        # and back: FromString + the reference's ndarray conversion, and the runtime's own field for half_val
        got, st = V.decode(want[len(V.tensor_header(dtype, [x.size], V.packed_len(x, dtype))):], dtype, x.size)
        assert st == V.OK and got.tobytes() == x.tobytes()
        if dtype != 19:
            assert ref_port.decode_tensor_proto(want).tobytes() == x.tobytes()


def _outcome_protobuf(wire, dtype):
    """What FromString + the reference's conversion make of a bare TensorProto: ('ok', bytes) or ('raise', exception name)."""
    try:
        tp = tensor_pb2.TensorProto.FromString(wire)
        if dtype == 19:       # half_val as bit patterns (the strict DT_HALF value quirk is not this reference's business)
            bits = np.array([v & 0xFFFF for v in tp.half_val], dtype=np.uint16)
            if bits.size != int(np.prod([d.size for d in tp.tensor_shape.dim])):
                raise ValueError("count")
            return "ok", bits.tobytes()
        return "ok", ref_port.from_tensor_proto(tp).tobytes()
    except (DecodeError, OverflowError, ValueError) as e:
        return "raise", type(e).__name__


def _outcome_ref(chunks, dtype, n):
    vals, st = V.decode(chunks, dtype, n)
    return ("ok", vals.tobytes()) if st == V.OK else ("raise", V.EXCEPTION[st])


def wire_cases():
    """(name, value chunks, element count): hand-made wires - 10-byte negatives, 11-byte varints, bits above 32 in int_val,
    unterminated runs, out-of-range values, wrong counts and their combinations."""
    vi = G.vi
    eleven = b"\xac\x82" + b"\x80" * 8 + b"\x00"        # eleven bytes whose first ten read 300
    return [
        ("neg10", [vi(-1) + vi(-(1 << 63)) + vi(-2)], 3),
        ("above32", [vi((1 << 40) + 5) + vi((1 << 35) - 1) + vi(0xFFFFFFFF) + vi(1 << 32)], 4),
        ("ten_nonminimal", [b"\x81" + b"\x80" * 8 + b"\x00" + b"\x05"], 2),
        ("eleven", [vi(1) + b"\xff" * 10 + b"\x01"], 2),
        ("eleven_300", [vi(1) + eleven], 2),
        ("unterminated", [vi(1) + vi(2) + b"\x80"], 3),
        ("range_last", [vi(1) + vi(2) + vi(300)], 3),
        ("range_first", [vi(-129) + vi(2)], 2),
        ("range_and_count", [vi(1) + vi(2) + vi(300)], 4),
        ("parse_and_range", [vi(300) + vi(1) + b"\xff" * 10 + b"\x01"], 3),
        ("parse_range_count", [vi(300) + eleven], 5),
        ("count", [vi(1) + vi(2) + vi(3)], 4),
        ("split", [vi(1) + vi(300), vi(-5) + vi(1 << 33), vi(7)], 5),
    ]


@pytest.mark.parametrize("dtype", sorted(V.DTYPES), ids=[V.NAMES[d] for d in sorted(V.DTYPES)])
def test_decode_matches_the_protobuf_runtime_and_ref_port(dtype):
    for name, chunks, n in wire_cases():
        wire = G.tproto(dtype, [n], V.field(dtype, chunks))
        assert _outcome_ref(chunks, dtype, n) == _outcome_protobuf(wire, dtype), name


def test_error_order_in_one_output():
    """The three errors of one output in the reference's order, as the issue of this order was found: an int8 output holding
    an 11-byte varint whose first ten bytes read 300 is a DecodeError, and int8 [4] holding [1, 2, 300] an OverflowError."""
    eleven = b"\xac\x82" + b"\x80" * 8 + b"\x00"
    assert V.decode([G.vi(1) + eleven], 6, 2)[1] == V.E_PARSE
    assert V.decode([G.vi(1) + G.vi(2) + G.vi(300)], 6, 4)[1] == V.E_RANGE
    assert V.decode([G.vi(1) + G.vi(2) + G.vi(3)], 6, 4, tolerant=True)[0].tolist() == [1, 2, 3, 3]


def precedence_responses():
    """Small PredictResponses, one output each, that combine a malformed varint, an out-of-range value and a wrong count."""
    vi = G.vi
    eleven = b"\xac\x82" + b"\x80" * 8 + b"\x00"
    cases = []
    for dtype in (6, 5, 4, 17):
        lo, hi = V.RANGE[dtype]
        cases += [
            (dtype, [vi(1) + eleven], 2),                                  # parse + range (first ten bytes read 300)
            (dtype, [vi(1) + vi(2) + vi(hi + 1)], 4),                       # range + count
            (dtype, [vi(lo - 1) + vi(1) + b"\xff" * 10 + b"\x01"], 7),      # all three
            (dtype, [vi(hi + 1), vi(1)], 3),                                # range + count over two occurrences
        ]
    return [(dt, G.entry("x", G.tproto(dt, [n], V.field(dt, chunks))) + G.mspec(), chunks, n)
            for dt, chunks, n in cases]


def _outcome(fn):
    try:
        got = fn()
        return "ok", {k: v.tobytes() for k, v in got.items()}
    except (DecodeError, wire_oracle.ParseError) as e:
        del e
        return "raise", "DecodeError"
    except (OverflowError, ValueError) as e:
        return "raise", type(e).__name__


def test_oracle_error_order_agrees_with_ref_port():
    for dt, wire, chunks, n in precedence_responses():
        want = _outcome(lambda: ref_port.decode_predict_response(wire))
        assert want[0] == "raise" and want == _outcome_ref(chunks, dt, n), (dt, chunks)
        assert _outcome(lambda: wire_oracle.decode_predict_response(wire, strict=True)) == want, (dt, chunks, n)
        # TF's MakeNdarray reads the typed values with np.fromiter(values, dtype) before it pads: range before count there too
        assert _outcome(lambda: wire_oracle.decode_predict_response(wire, strict=False)) == want, (dt, chunks, n)


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _const(text, name):
    m = re.search(r"\b%s\s*=\s*([^;,]+)[;,]" % name, text)
    assert m, name
    return m.group(1).strip()


def test_the_mirrored_geometry_matches_the_sources():
    plan, kern, host = _read("plan.h"), _read("kernels.cu"), _read("codec_host.cpp")
    threads = int(_const(plan, "kVarThreads"))
    per = int(_const(plan, "kVarPerThread"))
    assert _const(plan, "kVarTileElems") == "kVarThreads * kVarPerThread" and threads * per == V.ENC_TILE
    assert re.fullmatch(r"kVarThreads \* (\d+)", _const(plan, "kVarTileBytes")).group(1) == str(V.DEC_TILE // threads)
    assert _const(plan, "kVarGroupTiles") == "kVarThreads" and threads == V.GROUP_TILES
    assert int(_const(plan, "kTinyVarElems")) == V.TINY
    body = host[host.index("bool host_measurable_varint("):]
    body = body[: body.index("\n}\n")]
    assert re.findall(r"> (\d+)\)", body) == [str(V.HOST_MEASURE)] * 2
    assert V.ENC_GROUP_ELEMS == 524288 and V.DEC_GROUP_BYTES == 2 << 20
