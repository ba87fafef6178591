"""GPU parity against the golden vectors the unmodified reference produced (tests/golden/*.json).

Every comparison is bit-exact: encoded wire bytes == the reference's SerializeToString output,
decoded arrays == the reference's tensor_proto_to_ndarray output (or the same exception type).
"""
import hashlib

import numpy as np
import pytest
from google.protobuf.message import DecodeError

import golden_util as G

pytestmark = pytest.mark.gpu

ENC = G.load("encode.json")
REQ = G.load("requests.json")
DEC = G.load("decode.json")


@pytest.mark.parametrize("name", [k for k in ENC if not k.startswith("_")])
def test_encode_tensor_proto(codec, name):
    case = ENC[name]
    x = G.apply_transform(G.make_array(case["input"]), case.get("transform"))
    wire = codec.encode_tensor_protos([x])[0]
    G.check_wire(wire, case["wire"], name)


def test_encode_refused_dtypes(codec):
    """bytes_/object_/datetime64 raise ValueError like DataType() does; float16/complex, which the
    reference cannot encode (TypeError), follow TF's convention here instead."""
    refused = ENC["_refused"]
    for label, arr in (("bytes_", np.array([b"ab"])), ("object_", np.array([None], dtype=object)),
                       ("datetime64", np.array(["2020-01-01"], dtype="datetime64[D]"))):
        assert refused[label] == "ValueError"
        with pytest.raises(ValueError):
            codec.encode_tensor_protos([arr])
    # KAT-8 (TF convention, equals vendored tensor_util_test.py:224-259 goldens)
    assert codec.encode_tensor_protos([np.array([10, 20], dtype=np.float16)])[0].hex() == "08131204120208026a06809201809a01"
    import ml_dtypes
    assert codec.encode_tensor_protos([np.array([10, 20], dtype=ml_dtypes.bfloat16)])[0].hex() == "080e1204120208026a06a08201a08301"
    assert codec.encode_tensor_protos([np.array([10, 20, 30], dtype=np.float32)], tensor_content=True)[0].hex() == \
        "0801120412020803220c000020410000a0410000f041"


@pytest.mark.parametrize("name", list(REQ))
def test_encode_predict_request(codec, name):
    case = REQ[name]
    inputs = [(k, G.make_array(r)) for k, r in case["inputs"]]
    wd = "DT_FLOAT" if case.get("wire_dtype") == "DT_FLOAT" else None
    wire = codec.encode_predict_requests([(case["model_name"], case["model_version"], inputs)], wire_dtype=wd)[0]
    G.check_wire(wire, case["wire"], name)


def test_grpc_length_prefixed_message(codec):
    """RF_GRPC_FRAME: 00 + big-endian uint32 length in front of the same PredictRequest bytes (single request, batch of
    requests, a varint input whose length the device measures)."""
    from oracle import wire_oracle

    rng = np.random.default_rng(8)
    reqs = [("default", 1, [("x", rng.standard_normal((64, 257)).astype(np.float32))]),
            ("m", None, [("ids", rng.integers(0, 50000, size=(4, 300), dtype=np.int64)), ("mask", np.ones((4, 300), dtype=np.bool_))]),
            ("", 0, [])]
    plain = codec.encode_predict_requests(reqs)
    framed = codec.encode_predict_requests(reqs, grpc_frame=True)
    for (name, version, inputs), p, f in zip(reqs, plain, framed):
        assert p == wire_oracle.encode_predict_request(name, version, inputs)
        assert f == b"\x00" + len(p).to_bytes(4, "big") + p
    assert codec.encode_predict_request("default", dict(reqs[0][2]), 1, grpc_frame=True) == framed[0]


def test_encode_request_batch_matches_singles(codec):
    names = ["kat2_c1", "no_version", "mixed_dtypes", "c3_req7", "order_quirk", "no_inputs"]
    batch = [(REQ[n]["model_name"], REQ[n]["model_version"], [(k, G.make_array(r)) for k, r in REQ[n]["inputs"]]) for n in names]
    wires = codec.encode_predict_requests(batch)
    for n, w in zip(names, wires):
        G.check_wire(w, REQ[n]["wire"], n)


@pytest.mark.parametrize("name", list(DEC))
def test_decode_predict_response(codec, name):
    rec = DEC[name]
    wire = G.decode_case_wire(name, rec)
    if "parse_raises" in rec:
        with pytest.raises(DecodeError):
            codec.decode_predict_response(wire, strict=True)
        return
    expected = rec["outputs"]
    raising = {k: v for k, v in expected.items() if "raises" in v}
    if raising:
        # the reference decodes output by output; here one call decodes all, so check each on its own
        for k, v in raising.items():
            exc = {"ValueError": ValueError, "KeyError": KeyError, "TypeError": TypeError, "OverflowError": OverflowError,
                   "UnicodeDecodeError": UnicodeDecodeError}[v["raises"]]
            with pytest.raises(exc):
                codec.decode_predict_response(wire, strict=True)
        return
    outs, spec = codec.decode_predict_response(wire, strict=True)
    assert set(outs) == set(expected)
    for k, v in expected.items():
        got = outs[k]
        if v["dtype"] == "str":
            assert got.dtype.kind == "U" and list(got.shape) == v["shape"] and got.ravel().tolist() == v["strings"]
            continue
        assert got.dtype.str == v["dtype"], (k, got.dtype)
        assert list(got.shape) == v["shape"]
        if "data" in v:
            assert got.tobytes().hex() == v["data"], k
        else:
            assert hashlib.sha256(got.tobytes()).hexdigest() == v["sha256"], k
    ms = rec["model_spec"]
    assert (spec.name, spec.version, spec.has_version, spec.version_label, spec.signature_name) == \
        (ms["name"], ms["version"], ms["has_version"], ms["version_label"], ms["signature_name"])


def test_round_trip_all_numeric_dtypes(codec):
    """encode -> decode is the identity (reference tensors_test.py:111-117), every dtype of the table."""
    rng = np.random.default_rng(123)
    for dt in (np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.bool_):
        if dt is np.bool_:
            x = rng.integers(0, 2, size=(7, 13)).astype(np.bool_)
        elif np.dtype(dt).kind == "f":
            x = rng.standard_normal((7, 13)).astype(dt)
        else:
            info = np.iinfo(dt)
            x = rng.integers(info.min, info.max, size=(7, 13), dtype=dt, endpoint=True)
        wire = codec.encode_tensor_protos([x])[0]
        back = codec.decode_tensor_protos([wire], strict=True)[0]
        assert back.dtype == x.dtype and back.shape == x.shape and back.tobytes() == x.tobytes(), dt


def test_alignment_sweep_against_oracle(codec):
    """Every relative alignment of payload vs wire: key lengths 0..17 shift the payload offset byte by byte;
    sizes straddle the small-item / one-tile / multi-tile / ragged-tail boundaries; float32 (quieting path),
    float64 and bool; on encode the second large input of a request lands misaligned."""
    from oracle import wire_oracle

    rng = np.random.default_rng(99)
    sizes = [1, 3, 4, 5, 127, 511, 512, 513, 2047, 4097, 8191, 8192, 8193, 16385, 40001, 262147]
    for klen in range(0, 18):
        key = "k" * klen
        n = sizes[klen % len(sizes)]
        for dt in (np.float32, np.float64):
            x = rng.integers(0, 256, size=n * np.dtype(dt).itemsize, dtype=np.uint8).view(dt)   # random bits: NaNs of every kind
            resp = wire_oracle.build_predict_response([(key, x)], keep_snan=True)
            got = codec.decode_predict_response(resp, strict=True)[0][key]
            ref = wire_oracle.decode_predict_response(resp)[key]
            assert got.tobytes() == ref.tobytes(), (klen, n, dt)
    for n in sizes:
        a = rng.integers(0, 256, size=n * 4, dtype=np.uint8).view(np.float32)
        b = rng.integers(0, 256, size=(n + 7) * 4, dtype=np.uint8).view(np.float32)
        c = rng.integers(0, 2, size=n + 3).astype(np.bool_)
        d = rng.standard_normal(n + 1)
        inputs = [("a", a), ("bb", b), ("ccc", c), ("dddd", d)]
        wire = codec.encode_predict_requests([("m", 3, inputs)])[0]
        assert wire == wire_oracle.encode_predict_request("m", 3, inputs), n
        resp = wire_oracle.build_predict_response(inputs, keep_snan=True)
        outs = codec.decode_predict_response(resp, strict=True)[0]
        ref = wire_oracle.decode_predict_response(resp)
        for k in ref:
            assert outs[k].tobytes() == ref[k].tobytes(), (n, k)


def test_varint_multi_tile_against_oracle(codec):
    """Packed-varint dtypes across many encode tiles (2048 elements) and decode tiles (8 KB windows of wire):
    varints straddling tile edges, 10-byte negatives, every dtype of the int_val / int64_val / uint32_val /
    uint64_val / half_val / bool_val family, odd element counts."""
    import ml_dtypes
    from oracle import wire_oracle

    rng = np.random.default_rng(5)
    for dt, n in ((np.int64, 100003), (np.int32, 70001), (np.uint64, 50021), (np.uint32, 33333), (np.int16, 20011), (np.uint16, 20480),
                  (np.int8, 12289), (np.uint8, 4097), (np.float16, 30011), (ml_dtypes.bfloat16, 8193), (np.bool_, 10007)):
        if dt is np.bool_:
            x = rng.integers(0, 2, size=n).astype(np.bool_)
        elif np.dtype(dt).kind == "f" or dt is ml_dtypes.bfloat16:
            x = rng.standard_normal(n).astype(dt)
        else:
            info = np.iinfo(dt)
            mag = rng.integers(0, info.bits + 1, size=n)
            raw = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64) & ((np.uint64(1) << mag.astype(np.uint64)) - np.uint64(1))
            x = raw.astype(np.uint64).view(np.int64).astype(dt) if info.min < 0 else raw.astype(dt)
            if info.min < 0:
                x[::3] = -np.abs(x[::3])
        wire = codec.encode_tensor_protos([x])[0]
        assert wire == wire_oracle.encode_tensor_proto(x), dt
        back = codec.decode_tensor_protos([wire], strict=False)[0]
        assert back.dtype == x.dtype and back.tobytes() == x.tobytes(), dt
    # element count that disagrees with the shape -> ValueError, like reshape()
    good = wire_oracle.encode_tensor_proto(np.arange(5000, dtype=np.int64))
    bad = good.replace(b"\x08\x09\x12\x05\x12\x03\x08\x88\x27", b"\x08\x09\x12\x05\x12\x03\x08\x89\x27")
    assert bad != good
    with pytest.raises(ValueError):
        codec.decode_tensor_protos([bad], strict=True)
    padded = codec.decode_tensor_protos([bad], strict=False)[0]          # TF's convention: the last value repeats
    assert padded.shape == (5001,) and padded[:5000].tolist() == list(range(5000)) and padded[5000] == 4999


def _varint(v):
    out = bytearray()
    v &= (1 << 64) - 1
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def test_varint_tile_geometry_chunks_and_malformed(codec):
    """Decode tiles are aligned 8 KB windows of each chunk: sweep the chunk's start alignment (key lengths shift it byte by
    byte) with wire lengths around one and two tiles, split one tensor's values over several packed occurrences (chunks)
    with varints straddling tile edges, run many small tensors as one multi-job launch, and feed the malformed tails the
    protobuf runtime rejects (a last varint that never terminates, an eleven-byte varint)."""
    from oracle import wire_oracle

    rng = np.random.default_rng(17)
    # (a) alignment sweep, ~1 and ~2 tiles of wire, ten-byte negatives sprinkled in so varints straddle every edge
    for klen in range(0, 18):
        n = (1500, 2731, 2740, 5461, 5470, 9000)[klen % 6]
        x = rng.integers(0, 2 ** 21, size=n, dtype=np.int64)
        x[:: 5 + klen] = -x[:: 5 + klen] - 1
        resp = wire_oracle.build_predict_response([("k" * klen, x), ("z", x[::-1].astype(np.int32))])
        got = codec.decode_predict_response(resp, strict=True)[0]
        ref = wire_oracle.decode_predict_response(resp)
        for k in ref:
            assert got[k].dtype == ref[k].dtype and got[k].tobytes() == ref[k].tobytes(), (klen, k)
    # (b) one tensor, values spread over 5 packed int64_val occurrences of ragged lengths (field 10, wire type 2)
    vals = rng.integers(-2 ** 40, 2 ** 40, size=30011, dtype=np.int64)
    cuts = [0, 1, 4099, 4100, 20000, 30011]
    body = b"\x08\x09" + b"\x12\x06\x12\x04\x08" + _varint(30011)      # dtype DT_INT64, shape [30011] (dim submessage of 4 bytes)
    assert len(_varint(30011)) == 3
    for a, b in zip(cuts[:-1], cuts[1:]):
        chunk = b"".join(_varint(int(v)) for v in vals[a:b])
        body += b"\x52" + _varint(len(chunk)) + chunk
    ref = wire_oracle.decode_tensor_proto(body)
    assert ref.tobytes() == vals.tobytes()
    got = codec.decode_tensor_protos([body], strict=True)[0]
    assert got.dtype == np.int64 and got.tobytes() == vals.tobytes()
    # (c) many small tensors in one call: the multi-job tables (not the inline single-job path), both directions
    smalls = [rng.integers(-5, 70000, size=int(rng.integers(1, 700)), dtype=np.int64).astype(dt)
              for dt in (np.int64, np.int32, np.uint16, np.int8) for _ in range(13)]
    smalls = [np.abs(a) if a.dtype.kind == "u" else a for a in smalls]
    wires = codec.encode_tensor_protos(smalls)
    for a, w in zip(smalls, wires):
        assert w == wire_oracle.encode_tensor_proto(a)
    backs = codec.decode_tensor_protos(wires, strict=True)
    for a, b in zip(smalls, backs):
        assert b.dtype == a.dtype and b.tobytes() == a.tobytes()
    # (d) malformed tails
    good = wire_oracle.encode_tensor_proto(np.arange(3000, 3005, dtype=np.int64))
    assert good.endswith(_varint(3004))
    never_ends = good[:-1] + bytes([good[-1] | 0x80])                      # last byte keeps the continuation bit
    with pytest.raises(DecodeError):
        codec.decode_tensor_protos([never_ends])
    eleven = b"\x08\x09\x12\x04\x12\x02\x08\x01" + b"\x52\x0b" + b"\xff" * 10 + b"\x01"
    with pytest.raises(DecodeError):
        codec.decode_tensor_protos([eleven])
    ten = b"\x08\x09\x12\x04\x12\x02\x08\x01" + b"\x52\x0a" + b"\xff" * 9 + b"\x01"
    assert codec.decode_tensor_protos([ten], strict=True)[0].tolist() == [-1] == wire_oracle.decode_tensor_proto(ten).tolist()


def test_varint_randomised_magnitudes_and_sizes(codec):
    """40 random varint tensors: dtype of the int_val / int64_val / uint32_val / uint64_val family, 1 to ~400k elements,
    value magnitudes drawn per tensor (all one byte, token-id-like, mixed bit lengths, full range with negatives), random
    key length (alignment of the chunk on the wire).  Encode byte for byte and decode element for element vs the oracle."""
    from oracle import wire_oracle

    rng = np.random.default_rng(77)
    dts = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64]
    for it in range(40):
        dt = dts[int(rng.integers(len(dts)))]
        info = np.iinfo(dt)
        n = int(np.exp(rng.uniform(0, np.log(400000))))
        kind = int(rng.integers(4))
        if kind == 0:
            x = rng.integers(0, 128, size=n, dtype=np.int64)
        elif kind == 1:
            x = rng.integers(0, 50000, size=n, dtype=np.int64)
        elif kind == 2:
            x = (rng.integers(0, 2 ** 62, size=n, dtype=np.int64) >> rng.integers(0, 62, size=n))
        else:
            x = rng.integers(-2 ** 62, 2 ** 62, size=n, dtype=np.int64)
        if info.min < 0 and kind >= 2:
            x[:: 3] = -x[:: 3]
        x = (x.view(np.uint64) & np.uint64(info.max)).astype(dt) if info.min == 0 else np.clip(x, info.min, info.max).astype(dt)
        key = "k" * int(rng.integers(0, 20))
        wire = codec.encode_predict_requests([("m", 1, [(key, x)])])[0]
        assert wire == wire_oracle.encode_predict_request("m", 1, [(key, x)]), (it, dt, n, kind)
        resp = wire_oracle.build_predict_response([(key, x)])
        got = codec.decode_predict_response(resp, strict=True)[0][key]
        assert got.dtype == x.dtype and got.tobytes() == x.tobytes(), (it, dt, n, kind)


def test_tolerant_padding_follows_tensorflow(codec):
    """strict=False on fewer typed values than the shape holds - how TF writes constants - follows TensorFlow's MakeNdarray:
    no values -> zeros, else the last value repeats (B200TFS_OF_PAD_EDGE: a fill kernel behind the unpack); as bare
    TensorProtos, as outputs of one PredictResponse next to a full-size output, and strict=True keeps the ValueError."""
    from oracle import ref_port
    from test_oracle import _padding_cases

    cases = _padding_cases()
    for name, w in cases.items():
        want = ref_port.make_ndarray_tf(w)
        got = codec.decode_tensor_protos([w], strict=False)[0]
        assert got.dtype == want.dtype and got.shape == want.shape and got.tobytes() == want.tobytes(), name
        with pytest.raises(ValueError):
            codec.decode_tensor_protos([w], strict=True)
    from tensorflow.core.framework import tensor_pb2
    from tensorflow_serving.apis import predict_pb2

    resp = predict_pb2.PredictResponse()
    full = np.arange(600, dtype=np.float32).reshape(20, 30)
    resp.outputs["full"].CopyFrom(ref_port.to_tensor_proto(full))
    for name in ("f32_broadcast", "i64_broadcast", "f32_none", "bool_one", "i64_large"):
        resp.outputs[name].CopyFrom(tensor_pb2.TensorProto.FromString(cases[name]))
    outs = codec.decode_predict_response(resp.SerializeToString(), strict=False)[0]
    assert outs["full"].tobytes() == full.tobytes()
    for name in ("f32_broadcast", "i64_broadcast", "f32_none", "bool_one", "i64_large"):
        want = ref_port.make_ndarray_tf(cases[name])
        assert outs[name].dtype == want.dtype and outs[name].shape == want.shape and outs[name].tobytes() == want.tobytes(), name
    # more values than the shape holds: an error either way
    m = tensor_pb2.TensorProto(dtype=9, int64_val=[1, 2, 3])
    m.tensor_shape.dim.add().size = 2
    for strict in (True, False):
        with pytest.raises(ValueError):
            codec.decode_tensor_protos([m.SerializeToString()], strict=strict)


def test_modes_tensor_content_and_keep_snan(codec):
    """The two non-default encode modes against the oracle: tensor_content (TF's own layout, raw little-endian
    memory for every numeric dtype) and KEEP_SNAN (typed field, float32 bits untouched); and the tolerant decoder
    reading tensor_content back."""
    import ml_dtypes
    from oracle import wire_oracle

    rng = np.random.default_rng(8)
    bits = rng.integers(0, 2 ** 32, size=5003, dtype=np.uint32).view(np.float32)     # NaNs of every kind
    assert codec.encode_tensor_protos([bits], keep_snan=True)[0] == wire_oracle.encode_tensor_proto(bits, keep_snan=True)
    assert codec.encode_tensor_protos([bits], keep_snan=True)[0] != codec.encode_tensor_protos([bits])[0]
    for x in (bits.reshape(5003, 1), rng.standard_normal((33, 65)), rng.integers(-2 ** 62, 2 ** 62, size=(9, 11), dtype=np.int64),
              rng.integers(0, 2, size=77).astype(np.bool_), rng.standard_normal(4099).astype(np.float16),
              rng.standard_normal(130).astype(ml_dtypes.bfloat16), (rng.standard_normal(50) + 1j * rng.standard_normal(50)).astype(np.complex64)):
        wire = codec.encode_tensor_protos([x], tensor_content=True)[0]
        assert wire == wire_oracle.encode_tensor_proto(x, tensor_content=True), x.dtype
        back = codec.decode_tensor_protos([wire], strict=False)[0]                    # tolerant: raw bytes, TF convention
        assert back.dtype == x.dtype and back.shape == x.shape and back.tobytes() == x.tobytes(), x.dtype
        if x.size:
            with pytest.raises((ValueError, KeyError)):                               # the reference reads only the typed field (and has no bfloat16 row)
                codec.decode_tensor_protos([wire], strict=True)
    pair = [("a", bits), ("b", rng.standard_normal(7))]
    assert codec.encode_predict_requests([("m", None, pair)], tensor_content=True)[0] == wire_oracle.encode_predict_request("m", None, pair, tensor_content=True)


def test_randomised_requests_and_responses_against_oracle(codec):
    """150 random PredictRequests / PredictResponses: 1-4 tensors each, every numeric dtype of the table,
    sizes from 0 to ~70k elements (small-item, single-tile, multi-tile, multi-job varint paths), random key
    lengths (all relative alignments).  Encode must equal the oracle byte for byte, decode element for element."""
    import ml_dtypes
    from oracle import wire_oracle

    rng = np.random.default_rng(2026)
    dts = [np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.bool_,
           np.float16, ml_dtypes.bfloat16, np.complex64, np.complex128]
    alphabet = "abcdefghijklmnopqrstuvwxyz_0123456789"

    def rand_array():
        dt = dts[rng.integers(len(dts))]
        size_class = rng.integers(4)
        n = int([rng.integers(0, 8), rng.integers(8, 600), rng.integers(600, 9000), rng.integers(9000, 70000)][size_class])
        rank = int(rng.integers(1, 4))
        shape = [n] if rank == 1 else ([1, n] if rank == 2 else [n, 1, 1])
        raw = rng.integers(0, 256, size=n * np.dtype(dt).itemsize, dtype=np.uint8)
        a = raw.view(dt).reshape(shape)
        if dt is np.bool_:
            a = (raw & 1).astype(np.bool_).reshape(shape)
        return a

    for it in range(150):
        k = int(rng.integers(1, 5))
        keys = set()
        while len(keys) < k:
            keys.add("".join(alphabet[i] for i in rng.integers(0, len(alphabet), size=int(rng.integers(0, 24)))))
        tensors = [(key, rand_array()) for key in sorted(keys)]
        model = "m" * int(rng.integers(0, 40))
        version = None if rng.integers(3) == 0 else int(rng.integers(0, 2 ** 40))
        wire = codec.encode_predict_requests([(model, version, tensors)])[0]
        assert wire == wire_oracle.encode_predict_request(model, version, tensors), (it, [(k2, a.dtype, a.shape) for k2, a in tensors])
        resp = wire_oracle.build_predict_response(tensors, model_name=model or "x", version=version or 0, keep_snan=True)
        got = codec.decode_predict_response(resp, strict=False)[0]
        ref = wire_oracle.decode_predict_response(resp, strict=False)
        assert set(got) == set(ref), it
        for key in ref:
            assert got[key].dtype == ref[key].dtype and got[key].shape == ref[key].shape and got[key].tobytes() == ref[key].tobytes(), (it, key, ref[key].dtype)
