"""Device-resident C-ABI paths: batched encode, fused single-launch decode, CUDA-graph replay.

The checker is the CPU oracle (oracle/wire_oracle.py), itself pinned to the reference's goldens.
"""
import ctypes as C

import numpy as np
import pytest

from devutil import Dev, tensor_struct
from min_tfs_client import _native as N
from oracle import wire_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture()
def dev():
    d = Dev(0)
    yield d
    d.close()


def _encode_requests_device(dev, batch, order=N.ORDER_UPB):
    """batch: list of (model, version, [(key, ndarray)]); tensors uploaded first.  Returns list of wires."""
    keep, reqs = [], []
    for model, version, inputs in batch:
        ts = []
        for k, a in inputs:
            t, dims = tensor_struct(dev.upload(a), a, key=k.encode())
            keep.append((t, dims))
            ts.append(t)
        arr = (N.Tensor * max(len(ts), 1))(*ts)
        keep.append(arr)
        name = model.encode()
        reqs.append(N.Request(model_name=name, model_name_len=len(name), has_version=int(version is not None), order=order,
                              version=version or 0, n_inputs=len(ts), flags=0, inputs=arr))
    n = len(reqs)
    rq = (N.Request * n)(*reqs)
    flat = []
    for r in reqs:
        flat += [r.inputs[i] for i in range(r.n_inputs)]
    need = C.c_uint64()
    m = (N.Tensor * max(len(flat), 1))(*flat)
    N.check(dev.lib.b200tfs_measure(dev.ctx, len(flat), m))
    k = 0
    for r in reqs:  # copy packed_len back into the request structs
        for i in range(r.n_inputs):
            r.inputs[i].packed_len = m[k].packed_len
            k += 1
    rq = (N.Request * n)(*reqs)
    N.check(dev.lib.b200tfs_request_arena_size(n, rq, C.byref(need)))
    arena = dev.malloc(need.value)
    off = (C.c_uint64 * n)()
    ln = (C.c_uint64 * n)()
    N.check(dev.lib.b200tfs_encode_requests(dev.ctx, n, rq, arena, need.value, off, ln))
    dev.sync()
    whole = dev.download(arena, need.value)
    return [whole[off[i]: off[i] + ln[i]].tobytes() for i in range(n)], (arena, off, ln)


def test_c3_batch_encode_device(dev):
    """256 requests {image fp32[3,224,224], label int64[1]} (BASELINE configs[2]) in one launch set."""
    rng = np.random.default_rng(0)
    base = rng.standard_normal((3, 224, 224), dtype=np.float32)
    batch = []
    for i in range(256):
        img = base + np.float32(i)
        batch.append(("default", 1, [("image", img), ("label", np.array([i % 1000], dtype=np.int64))]))
    wires, _ = _encode_requests_device(dev, batch)
    for i in (0, 1, 7, 128, 255):
        expect = wire_oracle.encode_predict_request("default", 1, batch[i][2])
        assert wires[i] == expect, i
    assert len(wires[0]) == 602186  # SURVEY KAT-4


def _decode_fused(dev, wires, dst_stride):
    n = len(wires)
    off = (C.c_uint64 * n)()
    ln = (C.c_uint64 * n)()
    cur = 0
    for i, w in enumerate(wires):
        off[i], ln[i] = cur, len(w)
        cur += (len(w) + 255) & ~255
    buf = np.zeros(cur + 256, dtype=np.uint8)
    for i, w in enumerate(wires):
        buf[off[i]: off[i] + len(w)] = np.frombuffer(w, dtype=np.uint8)
    arena = dev.upload(buf)
    dst = dev.malloc(dst_stride * n)
    N.check(dev.lib.b200tfs_memset(dev.ctx, dst, 0xEE, dst_stride * n))
    N.check(dev.lib.b200tfs_decode_responses(dev.ctx, arena, n, off, ln, dst, dst_stride))
    outs = (N.Output * (n * N.FUSED_MAX_OUTPUTS))()
    n_outs = (C.c_int32 * n)()
    specs = (N.ModelSpec * n)()
    status = (C.c_int32 * n)()
    N.check(dev.lib.b200tfs_decode_results(dev.ctx, n, outs, n_outs, specs, status))
    return buf, dst, outs, n_outs, specs, status


def test_fused_decode_c2(dev):
    x = np.random.default_rng(0).standard_normal((1024, 1024), dtype=np.float32)
    x.reshape(-1)[:3] = np.array([0x7F800001, 0xFF800001, 0x7FC00001], dtype=np.uint32).view(np.float32)
    wire = wire_oracle.build_predict_response([("y", x)], keep_snan=True)
    buf, dst, outs, n_outs, specs, status = _decode_fused(dev, [wire], 4 << 20)
    assert status[0] == 0 and n_outs[0] == 1
    o = outs[0]
    assert o.dtype == 1 and o.rank == 2 and o.dims[0] == 1024 and o.dims[1] == 1024 and o.status == 0
    got = dev.download(dst + o.dst_off, o.dst_bytes).view(np.float32).reshape(1024, 1024)
    assert o.runs[0].off == len(wire) - 4 * 1024 * 1024 - 32 and o.key_off == 7  # offsets are record-relative
    ref = wire_oracle.decode_predict_response(wire)["y"]
    assert got.tobytes() == ref.tobytes()
    assert buf[specs[0].name_off: specs[0].name_off + specs[0].name_len].tobytes() == b"default" and specs[0].version == 1
    # the second launch takes the framing-template fast path: same answer, fresh destination
    x2 = np.random.default_rng(5).standard_normal((1024, 1024), dtype=np.float32)
    wire2 = wire_oracle.build_predict_response([("y", x2)])
    assert len(wire2) == len(wire)
    N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, dev.allocs[0], np.frombuffer(wire2, dtype=np.uint8).ctypes.data, len(wire2)))
    off1, ln1 = (C.c_uint64 * 1)(0), (C.c_uint64 * 1)(len(wire2))
    for _ in range(2):
        N.check(dev.lib.b200tfs_memset(dev.ctx, dst, 0x11, 4 << 20))
        N.check(dev.lib.b200tfs_decode_responses(dev.ctx, dev.allocs[0], 1, off1, ln1, dst, 4 << 20))
        N.check(dev.lib.b200tfs_decode_results(dev.ctx, 1, outs, n_outs, specs, status))
        assert status[0] == 0 and n_outs[0] == 1 and outs[0].dst_bytes == 4 << 20 and outs[0].dims[1] == 1024
        assert dev.download(dst + outs[0].dst_off, 4 << 20).tobytes() == x2.tobytes()
    # a response with different framing (other key) after a template was learnt: falls back to the walk
    wire3 = wire_oracle.build_predict_response([("z", x2[:512])])
    N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, dev.allocs[0], np.frombuffer(wire3, dtype=np.uint8).ctypes.data, len(wire3)))
    ln1[0] = len(wire3)
    N.check(dev.lib.b200tfs_decode_responses(dev.ctx, dev.allocs[0], 1, off1, ln1, dst, 4 << 20))
    N.check(dev.lib.b200tfs_decode_results(dev.ctx, 1, outs, n_outs, specs, status))
    assert status[0] == 0 and outs[0].dims[0] == 512 and outs[0].key_len == 1
    assert dev.download(dst + outs[0].dst_off, 2 << 20).tobytes() == x2[:512].tobytes()


def _vi(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _response_with_chunks(key, x, cuts):
    """PredictResponse bytes whose float_val values lie in several packed occurrences (cuts = element indices)."""
    raw = x.tobytes()
    tp = b"\x08\x01" + b"\x12" + _vi(2 + len(_vi(x.size)) + 1) + b"\x12" + _vi(1 + len(_vi(x.size))) + b"\x08" + _vi(x.size)
    for a, b in zip([0] + cuts, cuts + [x.size]):
        tp += b"\x2a" + _vi(4 * (b - a)) + raw[4 * a: 4 * b]
    entry = b"\x0a" + _vi(len(key)) + key + b"\x12" + _vi(len(tp)) + tp
    spec = b"\x0a\x07default\x12\x02\x08\x01\x1a\x0fserving_default"
    return b"\x0a" + _vi(len(entry)) + entry + b"\x12" + _vi(len(spec)) + spec


def test_fused_decode_same_length_other_framing_needs_more_tiles(dev, codec):
    """The launch budgets slack CTAs per record; when a record has the template's length they leave before the verdict.
    A record of the SAME length whose framing differs and whose values need MORE tiles than the template's then cannot be
    covered: it must say so (B200TFS_E_NONCANONICAL), never decode wrongly; the two-phase path and the Python codec (which
    falls back to it) decode it; and the next fused launch, with no valid template, covers it again."""
    rng = np.random.default_rng(21)
    a = rng.standard_normal(20000).astype(np.float32)            # 80000 B in one chunk: 3 tiles of 32 KB
    b = rng.standard_normal(19999).astype(np.float32)            # 40000 + 39996 B in two chunks: 2 + 2 tiles
    wa = _response_with_chunks(b"k", a, [])
    wb = _response_with_chunks(b"k", b, [10000])
    assert wa == wire_oracle.build_predict_response([("k", a)]) and len(wa) == len(wb)
    assert wire_oracle.decode_predict_response(wb)["k"].tobytes() == b.tobytes()
    stride = 1 << 17
    for _ in range(2):                                           # learn the template, then take the fast path
        buf, dst, outs, n_outs, specs, status = _decode_fused(dev, [wa], stride)
        assert status[0] == 0 and dev.download(dst + outs[0].dst_off, a.nbytes).tobytes() == a.tobytes()
    buf, dst, outs, n_outs, specs, status = _decode_fused(dev, [wb], stride)
    assert status[0] == N.E_NONCANONICAL
    buf, dst, outs, n_outs, specs, status = _decode_fused(dev, [wb], stride)   # that launch left no valid template
    assert status[0] == 0 and n_outs[0] == 1 and outs[0].n_runs == 2
    assert dev.download(dst + outs[0].dst_off, b.nbytes).tobytes() == b.tobytes()
    # the Python codec: same sequence, the second message comes out right (two-phase fallback)
    assert codec.decode_predict_response(wa)[0]["k"].tobytes() == a.tobytes()
    assert codec.decode_predict_response(wa)[0]["k"].tobytes() == a.tobytes()
    assert codec.decode_predict_response(wb)[0]["k"].tobytes() == b.tobytes()


def test_fused_decode_staged_batch_variety(dev):
    """Batches above ~38 MB of wire get tiles of several 32 KB chunks and the TMA-staged kernel: every source alignment (key
    lengths 0..15 shift the payload byte by byte), float32 (quieting) and float64, two outputs per record, values split over
    two chunks (destination head not 16-aligned: the register path inside the staged kernel), a record of another length and
    a malformed one (the walk inside the staged kernel).  Twice: the second launch takes the template path for record 0's
    look-alikes."""
    rng = np.random.default_rng(31)
    wires, refs = [], []
    for i in range(72):
        key = b"k" * (i % 16)
        if i % 9 == 4:
            x = rng.standard_normal(75000)                                   # float64, 600 KB
        else:
            x = rng.integers(0, 2 ** 32, size=150000, dtype=np.uint64).astype(np.uint32).view(np.float32)   # every kind of NaN
        if i % 9 == 7:
            y = rng.standard_normal(1000).astype(np.float32)
            w = wire_oracle.build_predict_response([(key.decode() or "x", x), ("second", y)], keep_snan=True)
        elif i % 9 == 2 and x.dtype == np.float32:
            w = _response_with_chunks(key or b"x", x, [50001])
        elif i == 40:
            w = wire_oracle.build_predict_response([("short", x[:1234])], keep_snan=True)
        else:
            w = wire_oracle.build_predict_response([(key.decode() or "x", x)], keep_snan=True)
        if i == 41:
            w = w[:-2]
        wires.append(w)
        refs.append(None if i == 41 else wire_oracle.decode_predict_response(w))
    assert sum(len(w) for w in wires) > 40 << 20
    stride = 1 << 20
    for _ in range(2):
        buf, dst, outs, n_outs, specs, status = _decode_fused(dev, wires, stride)
        whole = dev.download(dst, stride * len(wires))
        off = 0
        for i, w in enumerate(wires):
            if refs[i] is None:
                assert status[i] == N.E_PARSE
            else:
                assert status[i] == 0 and n_outs[i] == len(refs[i]), i
                for q in range(n_outs[i]):
                    o = outs[i * N.FUSED_MAX_OUTPUTS + q]
                    key = buf[off + o.key_off: off + o.key_off + o.key_len].tobytes().decode()
                    want = refs[i][key]
                    got = whole[i * stride + o.dst_off: i * stride + o.dst_off + o.dst_bytes]
                    assert o.dst_bytes == want.nbytes and got.tobytes() == want.tobytes(), (i, key)
            off += (len(w) + 255) & ~255


def test_fused_decode_batch_256(dev):
    """256 responses {scores fp32[1000]} (BASELINE configs[2] outputs): the n > 16 table path."""
    wires, refs = [], []
    for i in range(256):
        s = np.random.default_rng(10000 + i).standard_normal(1000, dtype=np.float32)
        wires.append(wire_oracle.build_predict_response([("scores", s)]))
        refs.append(s)
    buf, dst, outs, n_outs, specs, status = _decode_fused(dev, wires, 4096)
    whole = dev.download(dst, 4096 * 256)
    for i in range(256):
        assert status[i] == 0 and n_outs[i] == 1
        o = outs[i * N.FUSED_MAX_OUTPUTS]
        assert o.dst_off == 0 and o.dst_bytes == 4000
        assert whole[i * 4096: i * 4096 + 4000].tobytes() == refs[i].tobytes(), i


def test_fused_decode_mixed_and_errors(dev):
    a = np.arange(12, dtype=np.float32).reshape(3, 4)
    b = np.array([5, -6, 7], dtype=np.int64)
    d = np.linspace(0, 1, 33)
    good = wire_oracle.build_predict_response([("a", a), ("b", b), ("d", d)])
    bad = good[:-3]
    buf, dst, outs, n_outs, specs, status = _decode_fused(dev, [good, bad, b""], 1 << 16)
    assert status[0] == 0 and n_outs[0] == 3
    assert status[1] == N.E_PARSE
    assert status[2] == 0 and n_outs[2] == 0
    by_key = {}
    for k in range(n_outs[0]):
        o = outs[k]
        by_key[buf[o.key_off: o.key_off + o.key_len].tobytes().decode()] = o   # record 0 starts at arena offset 0
    assert dev.download(dst + by_key["a"].dst_off, 48).tobytes() == a.tobytes()
    assert dev.download(dst + by_key["d"].dst_off, 33 * 8).tobytes() == d.tobytes()
    ob = by_key["b"]  # varint output: tabulated, not moved by the fused kernel
    assert ob.flags & N.OF_VARINT and ob.n_elems == 3 and ob.dtype == 9
    # ... and finished by the two-phase unpack
    dptr = (C.c_void_p * 1)(dev.malloc(64))
    st = (C.c_int32 * 1)()
    o_arr = (N.Output * 1)(ob)
    N.check(dev.lib.b200tfs_unpack_outputs(dev.ctx, _arena_of(dev, buf), 1, o_arr, None, dptr, None, st))
    assert st[0] == 0 and dev.download(dptr[0], 24).view(np.int64).tolist() == [5, -6, 7]


def _arena_of(dev, buf):
    return dev.upload(buf)


def test_graph_replay_encode_decode(dev):
    """Capture encode + fused decode into a CUDA graph, refill the inputs, replay."""
    lib = dev.lib
    x = np.random.default_rng(1).standard_normal((256, 1024), dtype=np.float32)
    src = dev.upload(x)
    t, dims = tensor_struct(src, x, key=b"x")
    ts = (N.Tensor * 1)(t)
    rq = (N.Request * 1)(N.Request(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_inputs=1,
                                   flags=0, inputs=ts))
    need = C.c_uint64()
    N.check(lib.b200tfs_request_arena_size(1, rq, C.byref(need)))
    arena = dev.malloc(need.value)
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    resp = wire_oracle.build_predict_response([("y", x)])
    resp_dev = dev.upload(np.frombuffer(resp, dtype=np.uint8))
    dst = dev.malloc(1 << 20)
    p_off, p_len = (C.c_uint64 * 1)(0), (C.c_uint64 * 1)(len(resp))

    def both():
        N.check(lib.b200tfs_encode_requests(dev.ctx, 1, rq, arena, need.value, off, ln))
        N.check(lib.b200tfs_decode_responses(dev.ctx, resp_dev, 1, p_off, p_len, dst, 1 << 20))

    both()  # warm: sizes every scratch buffer
    dev.sync()
    N.check(lib.b200tfs_capture_begin(dev.ctx))
    both()
    g = C.c_void_p()
    N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
    # new data in the same buffers, then replay
    x2 = np.random.default_rng(2).standard_normal((256, 1024), dtype=np.float32)
    N.check(lib.b200tfs_memcpy_h2d(dev.ctx, src, x2.ctypes.data, x2.nbytes))
    resp2 = wire_oracle.build_predict_response([("y", x2)])
    assert len(resp2) == len(resp)
    r2 = np.frombuffer(resp2, dtype=np.uint8)
    N.check(lib.b200tfs_memcpy_h2d(dev.ctx, resp_dev, r2.ctypes.data, r2.nbytes))
    N.check(lib.b200tfs_memset(dev.ctx, arena, 0, need.value))
    for _ in range(3):
        N.check(lib.b200tfs_graph_launch(dev.ctx, g))
    dev.sync()
    wire = dev.download(arena + off[0], ln[0]).tobytes()
    assert wire == wire_oracle.encode_predict_request("m", 3, [("x", x2)])
    assert dev.download(dst, x2.nbytes).tobytes() == x2.tobytes()
    lib.b200tfs_graph_destroy(g)


def test_c5_full_size_batch_1024(dev):
    """BASELINE configs[4] per-GPU share: 1024 PredictRequests of fp32 [3,224,224] in ONE encode call,
    then 1024 PredictResponses of the same size through the fused decode (table path, n > 16).

    Size-independent checks: every record length equals the closed form (602164, SURVEY 8d), a stride-64
    sample is compared byte for byte with the oracle, the XOR-fold of all payload words on the wire equals
    the XOR-fold of all input words (no byte lost, duplicated or altered anywhere in 617 MB), and
    decode(encode-side payloads) returns the inputs exactly."""
    n = 1024
    base = np.random.default_rng(42).standard_normal((3, 224, 224), dtype=np.float32)
    big = np.empty((n, 3, 224, 224), dtype=np.float32)
    for i in range(n):
        np.add(base, np.float32(i) * np.float32(0.001), out=big[i])
    src = dev.upload(big)
    P = 3 * 224 * 224 * 4
    dims = (C.c_int64 * 3)(3, 224, 224)
    ts = (N.Tensor * n)()
    rq = (N.Request * n)()
    for i in range(n):
        ts[i] = N.Tensor(data=src + i * P, src_dtype=1, wire_dtype=1, rank=3, flags=0, dims=dims, key=b"image", key_len=5, packed_len=0)
        rq[i] = N.Request(model_name=b"default", model_name_len=7, has_version=1, order=N.ORDER_UPB, version=1, n_inputs=1, flags=0,
                          inputs=C.cast(C.byref(ts, i * C.sizeof(N.Tensor)), C.POINTER(N.Tensor)))
    need = C.c_uint64()
    N.check(dev.lib.b200tfs_request_arena_size(n, rq, C.byref(need)))
    arena = dev.malloc(need.value)
    off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    N.check(dev.lib.b200tfs_encode_requests(dev.ctx, n, rq, arena, need.value, off, ln))
    dev.sync()
    assert all(ln[i] == 602164 for i in range(n))
    whole = dev.download(arena, need.value)
    for i in range(0, n, 64):
        expect = wire_oracle.encode_predict_request("default", 1, [("image", big[i])])
        assert whole[off[i]: off[i] + ln[i]].tobytes() == expect, i
    fold_in = np.bitwise_xor.reduce(big.view(np.uint32).reshape(-1))
    fold_wire = np.uint32(0)
    H = 602164 - P
    for i in range(n):
        fold_wire ^= np.bitwise_xor.reduce(whole[off[i] + H: off[i] + H + P].view(np.uint32))
    assert fold_wire == fold_in
    # responses of the same payloads, canonical server layout, decoded in one fused launch
    prefix = wire_oracle.build_predict_response([("image", big[0])])
    hdr_len = len(prefix) - P - 32      # bytes before the payload (32 = trailing model_spec field)
    head, tail = prefix[:hdr_len], prefix[hdr_len + P:]
    stride = (len(prefix) + 255) & ~255
    buf = np.zeros(stride * n, dtype=np.uint8)
    hb, tb = np.frombuffer(head, np.uint8), np.frombuffer(tail, np.uint8)
    roff, rlen = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    flat = big.view(np.uint8).reshape(n, P)
    for i in range(n):
        o = i * stride
        buf[o: o + hdr_len] = hb
        buf[o + hdr_len: o + hdr_len + P] = flat[i]
        buf[o + hdr_len + P: o + len(prefix)] = tb
        roff[i], rlen[i] = o, len(prefix)
    assert buf[: len(prefix)].tobytes() == prefix
    wire_dev = dev.upload(buf)
    dst_stride = (P + 255) & ~255
    dst = dev.malloc(dst_stride * n)
    for _ in range(2):   # second pass: framing-template fast path for all 1024 records
        N.check(dev.lib.b200tfs_memset(dev.ctx, dst, 0, dst_stride * n))
        N.check(dev.lib.b200tfs_decode_responses(dev.ctx, wire_dev, n, roff, rlen, dst, dst_stride))
        outs = (N.Output * (n * N.FUSED_MAX_OUTPUTS))()
        n_outs, status = (C.c_int32 * n)(), (C.c_int32 * n)()
        N.check(dev.lib.b200tfs_decode_results(dev.ctx, n, outs, n_outs, None, status))
        assert all(status[i] == 0 and n_outs[i] == 1 for i in range(n))
        got = dev.download(dst, dst_stride * n).reshape(n, dst_stride)[:, :P]
        assert np.array_equal(got, flat)


def test_c4_cast_round_trip(dev, codec):
    """BASELINE configs[3]: fp16 / bf16 [8,512,1024] cast to DT_FLOAT on encode (wire bit-exact vs the oracle on
    x.astype(float32)) and cast back on decode (round-to-nearest-even: exact for values that came from 16 bits)."""
    import ml_dtypes

    rng = np.random.default_rng(4)
    for np_dt in (np.float16, ml_dtypes.bfloat16):
        x = rng.standard_normal((8, 512, 1024)).astype(np_dt)
        x.reshape(-1)[:4] = np.array([np.inf, -np.inf, 0.0, -0.0]).astype(np_dt)
        wire = codec.encode_predict_request("default", {"x": x}, 1, wire_dtype="DT_FLOAT")
        assert wire == wire_oracle.encode_predict_request("default", 1, [("x", x.astype(np.float32))])
        resp = wire_oracle.build_predict_response([("y", x.astype(np.float32))])
        back = codec.decode_predict_response(resp, out_dtypes={"y": np_dt})[0]["y"]
        assert back.dtype == np.dtype(np_dt) and back.tobytes() == x.tobytes()
        # a float32 payload that is NOT representable in 16 bits rounds to nearest even, like numpy's astype
        f = rng.standard_normal((1000, 37)).astype(np.float32)
        resp = wire_oracle.build_predict_response([("y", f)])
        back = codec.decode_predict_response(resp, out_dtypes={"y": np_dt})[0]["y"]
        assert np.array_equal(back.view(np.uint16), f.astype(np_dt).view(np.uint16))


def test_varint_measure_then_encode_contract(dev):
    """b200tfs_measure leaves its counters for the next encode of the same buffer: (a) that encode (one kernel fewer) and a
    second encode of the unchanged tensor (which counts again) produce the same bytes; (b) refill the buffer, measure again,
    encode: the new contents; (c) two tensors measured in separate calls, encoded together; (d) the same buffer as two
    inputs of one request."""
    from oracle import wire_oracle

    lib = dev.lib
    rng = np.random.default_rng(3)

    keep = []

    def tensor(ptr, n, key=b""):
        dims = (C.c_int64 * 1)(n)
        keep.append(dims)                                 # the struct only holds a pointer to it
        return N.Tensor(data=ptr, src_dtype=9, wire_dtype=9, rank=1, flags=0, dims=dims, key=key, key_len=len(key), packed_len=0)

    def launches():
        v = C.c_uint64()
        N.check(lib.b200tfs_kernel_launches(dev.ctx, C.byref(v)))
        return v.value

    def encode(ts):
        arr = (N.Tensor * len(ts))(*ts)
        need = C.c_uint64()
        N.check(lib.b200tfs_tensor_arena_size(len(ts), arr, C.byref(need)))
        arena = dev.malloc(need.value)
        off, ln = (C.c_uint64 * len(ts))(), (C.c_uint64 * len(ts))()
        before = launches()
        N.check(lib.b200tfs_encode_tensor_protos(dev.ctx, len(ts), arr, arena, need.value, off, ln))
        used = launches() - before
        raw = dev.download(arena, need.value)
        return [bytes(raw[off[i]: off[i] + ln[i]]) for i in range(len(ts))], used

    n = 70001
    a = (rng.integers(0, 2 ** 62, size=n, dtype=np.int64) >> rng.integers(0, 62, size=n)).astype(np.int64)
    pa = dev.upload(a)
    ta = (N.Tensor * 1)(tensor(pa, n))
    N.check(lib.b200tfs_measure(dev.ctx, 1, ta))
    first, l1 = encode([ta[0]])
    second, l2 = encode([ta[0]])
    assert first[0] == second[0] == wire_oracle.encode_tensor_proto(a)
    assert l2 == l1 + 1                                   # the second encode ran the counting kernel again
    # (b) new contents in the same buffer
    b = rng.integers(-50, 50, size=n, dtype=np.int64)
    N.check(lib.b200tfs_memcpy_h2d(dev.ctx, pa, b.ctypes.data, b.nbytes))
    dev.sync()
    N.check(lib.b200tfs_measure(dev.ctx, 1, ta))
    assert encode([ta[0]])[0][0] == wire_oracle.encode_tensor_proto(b)
    # (c) measured separately, encoded together
    c2 = rng.integers(0, 300, size=5000, dtype=np.int64)
    pc = dev.upload(c2)
    tc = (N.Tensor * 1)(tensor(pc, 5000))
    N.check(lib.b200tfs_measure(dev.ctx, 1, ta))
    N.check(lib.b200tfs_measure(dev.ctx, 1, tc))
    both, _ = encode([ta[0], tc[0]])
    assert both == [wire_oracle.encode_tensor_proto(b), wire_oracle.encode_tensor_proto(c2)]
    # (d) one buffer, two inputs of a request
    two = (N.Tensor * 2)(tensor(pc, 5000, b"x"), tensor(pc, 5000, b"yy"))
    N.check(lib.b200tfs_measure(dev.ctx, 2, two))
    rq = (N.Request * 1)(N.Request(model_name=b"m", model_name_len=1, has_version=0, order=N.ORDER_UPB, version=0, n_inputs=2, flags=0,
                                   inputs=C.cast(two, C.POINTER(N.Tensor))))
    need = C.c_uint64()
    N.check(lib.b200tfs_request_arena_size(1, rq, C.byref(need)))
    arena = dev.malloc(need.value)
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    N.check(lib.b200tfs_encode_requests(dev.ctx, 1, rq, arena, need.value, off, ln))
    raw = dev.download(arena, need.value)
    assert bytes(raw[off[0]: off[0] + ln[0]]) == wire_oracle.encode_predict_request("m", None, [("x", c2), ("yy", c2)])


def test_one_gib_tensor(dev):
    """Largest practical single message: fp32 [16384, 16384] = 1 GiB payload (protobuf's limit is 2 GiB; the
    E_TOOBIG side of that limit is a CPU test).  The whole 1 GiB wire is compared with the C oracle's."""
    n = 16384
    P = n * n * 4
    row = np.random.default_rng(3).integers(0, 2 ** 32, size=n, dtype=np.uint32)
    full = np.empty((n, n), dtype=np.uint32)
    for r in range(n):                                             # every row a different rotation: no two blocks equal
        full[r, : n - (r % n)] = row[r % n:]
        full[r, n - (r % n):] = row[: r % n]
    x = full.view(np.float32)                                      # random bits: includes NaNs of every kind (quieting path)
    src = dev.upload(x)
    dims = (C.c_int64 * 2)(n, n)
    ts = (N.Tensor * 1)(N.Tensor(data=src, src_dtype=1, wire_dtype=1, rank=2, flags=0, dims=dims, key=b"x", key_len=1, packed_len=0))
    rq = (N.Request * 1)(N.Request(model_name=b"default", model_name_len=7, has_version=1, order=N.ORDER_UPB, version=1, n_inputs=1, flags=0,
                                   inputs=ts))
    need, total = C.c_uint64(), C.c_uint64()
    N.check(dev.lib.b200tfs_request_size(rq, C.byref(total)))
    N.check(dev.lib.b200tfs_request_arena_size(1, rq, C.byref(need)))
    arena = dev.malloc(need.value)
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    N.check(dev.lib.b200tfs_encode_requests(dev.ctx, 1, rq, arena, need.value, off, ln))
    dev.sync()
    expect = wire_oracle.encode_predict_request("default", 1, [("x", x)])
    assert ln[0] == total.value == len(expect)
    got = dev.download(arena + off[0], ln[0])
    assert got.tobytes() == expect


BEYOND_THE_INLINE_TABLE = {"outputs_x40": N.E_SIZE, "split_packed_x20": N.E_NONCANONICAL, "split_packed_ints_x20": N.E_NONCANONICAL,
                           "all_unpacked_ints_300": N.E_NONCANONICAL, "unpacked_between_foreign_runs": N.E_NONCANONICAL,
                           "rank_20": N.E_NONCANONICAL, "rank_20_ints_dim_minus_one": N.E_NONCANONICAL}


def test_fused_decode_replays_every_golden_case_twice(dev):
    """All golden PredictResponses through the single-launch decode, each TWICE in a row: the first launch walks
    the tags, the second takes the framing-template fast path; both must tabulate the same thing and both must
    agree with the reference for every fixed-width output (varint / string outputs are tabulated only)."""
    import hashlib

    import golden_util as G
    from min_tfs_client.constants import numpy_for_enum

    cases = G.load("decode.json")
    for name, rec in cases.items():
        wire = G.decode_case_wire(name, rec)
        if not wire:
            continue
        stride = max(256, (len(wire) + 255) & ~255)
        snap = []
        for rep in range(2):
            buf, dst, outs, n_outs, specs, status = _decode_fused(dev, [wire], stride)
            if "parse_raises" in rec:
                assert status[0] == N.E_PARSE, (name, rep)
                snap.append(None)
                continue
            if name in BEYOND_THE_INLINE_TABLE:
                # more outputs / value runs / dims than the single-launch table holds: it says so and the two-phase calls decode
                # the record (test_golden_gpu.py::test_decode_predict_response runs these through the Python codec, which falls back)
                assert status[0] == BEYOND_THE_INLINE_TABLE[name], (name, rep, status[0])
                snap.append(None)
                continue
            assert status[0] == N.OK, (name, rep, status[0])
            table = {}
            for k in range(n_outs[0]):
                o = outs[k]
                key = buf[o.key_off: o.key_off + o.key_len].tobytes().decode()
                vals = None
                if o.status == N.OK and not (o.flags & N.OF_VARINT) and o.dtype != 7 and o.n_elems:
                    vals = dev.download(dst + o.dst_off, o.dst_bytes).tobytes()
                table[key] = (o.dtype, o.rank, tuple(o.dims[i] for i in range(o.rank)), o.status, o.flags, o.n_runs, o.n_elems, vals)
            snap.append(table)
            expected = rec["outputs"]
            assert set(table) == set(expected), (name, rep)
            for key, exp in expected.items():
                dtype, rank, dims, st, flags, n_chunks, n_elems, vals = table[key]
                if "raises" in exp or exp.get("dtype") == "str" or vals is None:
                    continue
                np_t = numpy_for_enum(dtype)
                if np_t in (np.complex64, np.complex128) or (name == "dtype_half_ref_quirk"):
                    continue
                assert np.dtype(np_t).str == exp["dtype"] and list(dims) == exp["shape"], (name, key)
                if "data" in exp:
                    assert vals.hex() == exp["data"], (name, key, rep)
                else:
                    assert hashlib.sha256(vals).hexdigest() == exp["sha256"], (name, key, rep)
        assert snap[0] == snap[1], name      # walk and template fast path tabulate identically


def _stats(dev):
    a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
    N.check(dev.lib.b200tfs_decode_stats(dev.ctx, C.byref(a), C.byref(b), C.byref(c)))
    return a.value, b.value, c.value


def _decode_host(dev, wires, dst_stride, pinned):
    """b200tfs_decode_responses_host_async + b200tfs_decode_results on a host-resident wire."""
    n = len(wires)
    off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    cur = 0
    for i, w in enumerate(wires):
        off[i], ln[i] = cur, len(w)
        cur += (len(w) + 255) & ~255
    wire_buf, out_buf = pinned(cur + 256), pinned(dst_stride * n)
    for i, w in enumerate(wires):
        wire_buf.array[off[i]: off[i] + len(w)] = np.frombuffer(w, dtype=np.uint8)
    out_buf.array[:] = 0xEE
    N.check(dev.lib.b200tfs_decode_responses_host_async(dev.ctx, wire_buf.ptr, n, off, ln, out_buf.ptr, dst_stride))
    outs = (N.Output * (n * N.FUSED_MAX_OUTPUTS))()
    n_outs, specs, status = (C.c_int32 * n)(), (N.ModelSpec * n)(), (C.c_int32 * n)()
    N.check(dev.lib.b200tfs_decode_results(dev.ctx, n, outs, n_outs, specs, status))
    return out_buf.array, outs, n_outs, status


def test_template_rides_in_the_parameters_when_the_host_has_it(dev):
    """Host-resident wire: the library walks record 0 itself, so the FIRST launch already takes the template path (no serial
    tag walk on the device), whatever the payload's alignment inside the record; a device-resident wire adopts the template
    the previous launch left in pinned memory once the stream has gone idle; a stale template costs a walk, never a wrong
    answer."""
    keep = []

    def pinned(nbytes):
        b = N.PinnedBuffer(nbytes)
        keep.append(b)
        return b
    rng = np.random.default_rng(77)
    x = rng.standard_normal((1000,)).astype(np.float32)
    x[:3] = np.array([0x7F800001, 0xFF800001, 0x7FC00001], dtype=np.uint32).view(np.float32)
    want = wire_oracle.decode_predict_response(wire_oracle.build_predict_response([("scores", x)]))["scores"].tobytes()
    for key in ("scores", "s", "a_rather_longer_output_name"):           # the payload offset (mod 16) changes with the key length
        wire = wire_oracle.build_predict_response([(key, x)], "default", 1, "serving_default")
        s0 = _stats(dev)
        out, outs, n_outs, status = _decode_host(dev, [wire], 4096, pinned)
        s1 = _stats(dev)
        assert status[0] == 0 and n_outs[0] == 1 and outs[0].dims[0] == 1000 and outs[0].key_len == len(key)
        assert out[outs[0].dst_off: outs[0].dst_off + 4000].tobytes() == want
        assert (s1[0] - s0[0], s1[2] - s0[2]) == (1, 0), "first launch on a host-resident wire must not walk on the device"
    # a batch of 5 responses in host memory, record 3 with another key of the same length: four by template, one walked
    ws = [wire_oracle.build_predict_response([("scores", x + i)]) for i in range(5)]
    ws[3] = wire_oracle.build_predict_response([("scorez", x + 3)])
    s0 = _stats(dev)
    out, outs, n_outs, status = _decode_host(dev, ws, 4096, pinned)
    s1 = _stats(dev)
    assert all(v == 0 for v in status) and (s1[0] - s0[0], s1[2] - s0[2]) == (4, 1)
    for i in range(5):
        o = outs[i * N.FUSED_MAX_OUTPUTS]
        assert out[i * 4096 + o.dst_off: i * 4096 + o.dst_off + 4000].tobytes() == (x + i).astype(np.float32).tobytes()
    # device-resident wire on a fresh context: walk, then (stream idle after decode_results) the pinned template in the parameters
    d2 = Dev(0)
    try:
        wire = wire_oracle.build_predict_response([("scores", x)])
        for rep, expect in enumerate([(0, 0, 1), (1, 0, 0), (1, 0, 0)]):
            s0 = _stats(d2)
            buf, dst, outs, n_outs, specs, status = _decode_fused(d2, [wire], 4096)
            s1 = _stats(d2)
            assert status[0] == 0 and tuple(b - a for a, b in zip(s0, s1)) == expect, (rep, s0, s1)
            assert d2.download(dst + outs[0].dst_off, 4000).tobytes() == want
        # two launches back to back without the stream going idle in between: the second cannot adopt anything new, it uses what
        # the host knows (still valid here)
        arena = d2.upload(np.frombuffer(wire, dtype=np.uint8))
        dst = d2.malloc(8192)
        off, ln = (C.c_uint64 * 1)(0), (C.c_uint64 * 1)(len(wire))
        N.check(d2.lib.b200tfs_decode_responses(d2.ctx, arena, 1, off, ln, dst, 4096))
        N.check(d2.lib.b200tfs_decode_responses(d2.ctx, arena, 1, off, ln, dst + 4096, 4096))
        d2.sync()
        assert d2.download(dst, 4000).tobytes() == want and d2.download(dst + 4096, 4000).tobytes() == want
        # stale: another response of the SAME length but other framing - the parameters' template misses, the record is walked
        other = wire_oracle.build_predict_response([("scorez", x)])
        s0 = _stats(d2)
        buf, dst, outs, n_outs, specs, status = _decode_fused(d2, [other], 4096)
        s1 = _stats(d2)
        assert status[0] == 0 and s1[2] - s0[2] == 1 and buf[outs[0].key_off: outs[0].key_off + 6].tobytes() == b"scorez"
        assert d2.download(dst + outs[0].dst_off, 4000).tobytes() == want
        buf, dst, outs, n_outs, specs, status = _decode_fused(d2, [other], 4096)      # ... and is the template from then on
        s2 = _stats(d2)
        assert status[0] == 0 and s2[0] - s1[0] == 1 and s2[2] == s1[2]
    finally:
        d2.close()


def test_two_phase_decode_beyond_the_inline_table(dev):
    """Through the C ABI: a response whose values lie in 20 packed occurrences of different lengths (12 runs spill), a rank-20
    output (4 dims spill) and a row of 1000 unpacked elements (one strided run), parsed by b200tfs_parse_responses (which
    re-runs itself with a larger spill area), listed by b200tfs_output_runs / _dims, unpacked by b200tfs_unpack_outputs."""
    import golden_util as G

    rng = np.random.default_rng(5)
    parts = [rng.standard_normal(1 + 3 * (k % 5)).astype(np.float32) for k in range(20)]
    many = np.concatenate(parts)
    dims20 = [1, 2, 1, 1, 3, 1, 1, 1, 1, 2, 1, 1, 1, 1, 1, 1, 1, 1, 5, 1]
    deep = np.arange(60, dtype=np.float32)
    row = (np.arange(1000, dtype=np.float32) * 0.5 - 7)
    ints = np.array([(i * 7919) % 100000 - 500 for i in range(300)], dtype=np.int64)
    wire = (G.entry("many", G.tproto(1, [many.size], b"".join(G.ld(0x2A, p.tobytes()) for p in parts)))
            + G.entry("deep", G.tproto(1, dims20, G.ld(0x2A, deep.tobytes())))
            + G.entry("row", G.tproto(1, [1000], b"".join(b"\x2D" + v.tobytes() for v in row)))
            + G.entry("ints", G.tproto(9, [300], b"".join(b"\x50" + G.vi(int(v)) for v in ints))) + G.mspec())
    arena = dev.upload(np.frombuffer(wire, dtype=np.uint8))
    off, ln = (C.c_uint64 * 1)(0), (C.c_uint64 * 1)(len(wire))
    outs = (N.Output * 8)()
    n_outs, specs, status = (C.c_int32 * 1)(), (N.ModelSpec * 1)(), (C.c_int32 * 1)()
    N.check(dev.lib.b200tfs_parse_responses(dev.ctx, arena, 1, off, ln, 8, outs, n_outs, specs, status))
    assert status[0] == 0 and n_outs[0] == 4
    by = {wire[outs[k].key_off: outs[k].key_off + outs[k].key_len].decode(): outs[k] for k in range(4)}
    o = by["many"]
    assert o.status == 0 and (o.n_runs, o.n_inline) == (20, 8) and o.flags & N.OF_SPILLED
    runs = (N.Run * 20)()
    N.check(dev.lib.b200tfs_output_runs(dev.ctx, C.byref(o), runs, 20))
    assert b"".join(wire[r.off: r.off + r.len] for r in runs) == many.tobytes()
    o = by["deep"]
    assert o.status == 0 and o.rank == 20 and o.flags & N.OF_SPILLED
    dims = (C.c_int64 * 20)()
    N.check(dev.lib.b200tfs_output_dims(dev.ctx, C.byref(o), dims, 20))
    assert list(dims) == dims20
    o = by["row"]
    assert o.status == 0 and o.n_runs == 1 and (o.runs[0].len, o.runs[0].count, o.runs[0].stride) == (4, 1000, 5)
    assert by["ints"].status == 0 and by["ints"].n_runs > N.MAX_RUNS
    order = ["many", "deep", "row", "ints"]
    want = [many, deep, row, ints]
    sel = (N.Output * 4)(*[by[k] for k in order])
    dsts = [dev.malloc(a.nbytes) for a in want]
    st = (C.c_int32 * 4)()
    N.check(dev.lib.b200tfs_unpack_outputs(dev.ctx, arena, 4, sel, None, (C.c_void_p * 4)(*dsts), None, st))
    assert list(st) == [0, 0, 0, 0]
    for d, a in zip(dsts, want):
        assert dev.download(d, a.nbytes).tobytes() == a.tobytes()
    # float32 -> float16 while gathering a strided row
    half = dev.malloc(2000)
    codes = (C.c_int32 * 1)(19)
    N.check(dev.lib.b200tfs_unpack_outputs(dev.ctx, arena, 1, (N.Output * 1)(by["row"]), None, (C.c_void_p * 1)(half), codes, st))
    assert dev.download(half, 2000).tobytes() == row.astype(np.float16).tobytes()


def test_scratch_buffers_are_pinned_once_a_graph_exists(dev):
    """A captured graph carries the addresses of the context's scratch buffers: a later, larger call that would have to
    reallocate them is refused (B200TFS_E_ARG) instead of leaving the graph with dangling addresses; same-size calls go on."""
    x = np.random.default_rng(1).standard_normal((64, 64)).astype(np.float32)
    wire = wire_oracle.build_predict_response([("y", x)])
    arena = dev.upload(np.frombuffer(wire, dtype=np.uint8))
    dst = dev.malloc(1 << 16)
    off, ln = (C.c_uint64 * 1)(0), (C.c_uint64 * 1)(len(wire))
    N.check(dev.lib.b200tfs_decode_responses(dev.ctx, arena, 1, off, ln, dst, 1 << 15))
    dev.sync()
    N.check(dev.lib.b200tfs_capture_begin(dev.ctx))
    N.check(dev.lib.b200tfs_decode_responses(dev.ctx, arena, 1, off, ln, dst, 1 << 15))
    g = C.c_void_p()
    N.check(dev.lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
    N.check(dev.lib.b200tfs_graph_launch(dev.ctx, g))
    dev.sync()
    assert dev.download(dst, x.nbytes).tobytes() == x.tobytes()
    n = 4096                                                     # the result table of 4096 records does not fit the pinned buffer sized for one
    big = dev.upload(np.zeros(n * 256, dtype=np.uint8))
    offs, lens = (C.c_uint64 * n)(*[i * 256 for i in range(n)]), (C.c_uint64 * n)(*[0] * n)
    bigdst = dev.malloc(n * 256)
    rc = dev.lib.b200tfs_decode_responses(dev.ctx, big, n, offs, lens, bigdst, 256)
    assert rc == N.E_ARG and b"graph" in dev.lib.b200tfs_last_error()
    N.check(dev.lib.b200tfs_graph_launch(dev.ctx, g))            # the graph still runs and still lands in live memory
    N.check(dev.lib.b200tfs_decode_responses(dev.ctx, arena, 1, off, ln, dst, 1 << 15))
    dev.sync()
    dev.lib.b200tfs_graph_destroy(g)


def _requests_on_device(dev, batch, grpc=False):
    """request structs over uploaded tensors, packed_len left at 0 (nothing measured)"""
    keep, reqs, ptrs = [], [], []
    for model, version, inputs in batch:
        ts = []
        for k, a in inputs:
            p = dev.upload(a)
            ptrs.append((p, a))
            t, dims = tensor_struct(p, a, key=k.encode())
            keep.append((t, dims))
            ts.append(t)
        arr = (N.Tensor * max(len(ts), 1))(*ts)
        keep.append(arr)
        name = model.encode()
        reqs.append(N.Request(model_name=name, model_name_len=len(name), has_version=int(version is not None), order=N.ORDER_UPB,
                              version=version or 0, n_inputs=len(ts), flags=N.RF_GRPC_FRAME if grpc else 0, inputs=arr))
    return (N.Request * len(reqs))(*reqs), keep, ptrs


def _deferred_batch(rng, scale):
    """requests with fixed-width, tiny and large packed-varint inputs, zero-element tensors, and one request without inputs;
    `scale` changes the values (and with them the varint lengths) but not the shapes"""
    out = []
    for i in range(9):
        img = rng.standard_normal((3, 16, 16)).astype(np.float32)
        img.reshape(-1)[:2] = np.array([0x7F800001, 0xFF800001], dtype=np.uint32).view(np.float32)
        label = np.array([[(i * 37) % 1000 * scale]], dtype=np.int64)
        toks = (rng.integers(0, 50000, size=(2, 40 + i)) * scale - (i % 3)).astype(np.int32)      # some negatives: ten-byte varints
        out.append(("default", 1 if i % 2 else None, [("image", img), ("label", label), ("tokens", toks), ("mask", toks > 100),
                                                       ("empty", np.zeros((0, 4), np.int64))]))
    out.append(("m", 3, [("big", (rng.integers(0, 2 ** 62, size=70000, dtype=np.int64) >> rng.integers(0, 62, size=70000)))]))
    out.append(("two", 2, [("a_ids", (rng.integers(0, 50000, size=5000) * scale).astype(np.int64)),                                 # two large varint inputs
                           ("b_ids", (rng.integers(-9, 300, size=4097) * scale).astype(np.int16)), ("x", rng.standard_normal(9).astype(np.float32))]))
    out.append(("", None, []))
    return out


def test_deferred_encode_no_host_round_trip(dev):
    """b200tfs_encode_requests_async: packed-varint inputs are measured, framed and emitted by kernels alone (count -> frame ->
    move + emit), bit-exact against the oracle; the whole call is captured in a CUDA graph and the replay re-measures: new label
    values of other varint lengths give other record lengths, again bit-exact."""
    rng = np.random.default_rng(31)
    batch = _deferred_batch(rng, 1)
    for grpc in (False, True):
        rq, keep, ptrs = _requests_on_device(dev, batch, grpc)
        n = len(batch)
        need = C.c_uint64()
        N.check(dev.lib.b200tfs_request_arena_size(n, rq, C.byref(need)))
        arena = dev.malloc(need.value)
        N.check(dev.lib.b200tfs_memset(dev.ctx, arena, 0xCD, need.value))
        N.check(dev.lib.b200tfs_encode_requests_async(dev.ctx, n, rq, arena, need.value))
        off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
        N.check(dev.lib.b200tfs_encode_results(dev.ctx, n, off, ln))
        whole = dev.download(arena, need.value)
        for i, (model, version, inputs) in enumerate(batch):
            want = wire_oracle.encode_predict_request(model, version, inputs)
            if grpc:
                want = b"\x00" + len(want).to_bytes(4, "big") + want
            assert whole[off[i]: off[i] + ln[i]].tobytes() == want, (i, grpc)
            assert i == 0 or off[i] >= off[i - 1] + ln[i - 1]
    # captured: the same call as a graph; then other VALUES in the same buffers (other varint lengths) and a replay
    rq, keep, ptrs = _requests_on_device(dev, batch)
    n = len(batch)
    N.check(dev.lib.b200tfs_request_arena_size(n, rq, C.byref(need)))
    arena = dev.malloc(need.value)
    N.check(dev.lib.b200tfs_encode_requests_async(dev.ctx, n, rq, arena, need.value))     # sizes the scratch buffers
    dev.sync()
    N.check(dev.lib.b200tfs_capture_begin(dev.ctx))
    N.check(dev.lib.b200tfs_encode_requests_async(dev.ctx, n, rq, arena, need.value))
    g = C.c_void_p()
    N.check(dev.lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
    batch2 = _deferred_batch(rng, 977)
    k = 0
    for model, version, inputs in batch2:
        for key, a in inputs:
            p, old = ptrs[k]
            k += 1
            assert old.shape == a.shape and old.dtype == a.dtype
            if a.nbytes:
                N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, p, np.ascontiguousarray(a).ctypes.data, a.nbytes))
    dev.sync()
    N.check(dev.lib.b200tfs_graph_launch(dev.ctx, g))
    off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    N.check(dev.lib.b200tfs_encode_results(dev.ctx, n, off, ln))
    whole = dev.download(arena, need.value)
    lens1 = [len(wire_oracle.encode_predict_request(m, v, i)) for m, v, i in batch]
    for i, (model, version, inputs) in enumerate(batch2):
        want = wire_oracle.encode_predict_request(model, version, inputs)
        assert whole[off[i]: off[i] + ln[i]].tobytes() == want, i
    assert [int(x) for x in ln] != lens1            # the replay really produced other lengths
    dev.lib.b200tfs_graph_destroy(g)


def test_deferred_frame_on_the_host_lays_records_out_like_the_device(dev):
    """b200tfs_request_frame_deferred runs the framing code on the host, with packed lengths the caller supplies (here: numpy's).
    For a request encoded alone by b200tfs_encode_requests_async it must give the device's rec_off / rec_len, and every
    payload_off must point at the bytes the device wrote for that input."""
    from test_deferred_frame_cpu import deferred_wire, payload_bytes
    rng = np.random.default_rng(53)
    x = np.arange(6, dtype=np.float32).reshape(2, 3)
    batch = []
    for n in (100, 5000, 70000):
        ids = rng.integers(0, 2 ** 40, size=n, dtype=np.int64) >> rng.integers(0, 40, size=n)
        batch += [("m", 7, [("img", x), ("z_ids", ids)]), ("m", 7, [("z_ids", ids)])]
    batch.append(("two", 2, [("a_ids", rng.integers(0, 50000, size=5000).astype(np.int64)),
                             ("b_ids", rng.integers(-9, 300, size=4097).astype(np.int16))]))
    batch += _deferred_batch(rng, 1)
    for model, version, inputs in batch:
        rq, keep, ptrs = _requests_on_device(dev, [(model, version, inputs)])
        need = C.c_uint64()
        N.check(dev.lib.b200tfs_request_arena_size(1, rq, C.byref(need)))
        arena = dev.malloc(need.value)
        N.check(dev.lib.b200tfs_memset(dev.ctx, arena, 0xCD, need.value))
        N.check(dev.lib.b200tfs_encode_requests_async(dev.ctx, 1, rq, arena, need.value))
        off, ln = C.c_uint64(), C.c_uint64()
        N.check(dev.lib.b200tfs_encode_results(dev.ctx, 1, C.byref(off), C.byref(ln)))
        whole = dev.download(arena, need.value)
        what = (model, [(k, a.dtype.name, a.shape) for k, a in inputs])
        wire, host_off, poff, plen = deferred_wire(model, version, inputs)
        assert (off.value, ln.value) == (host_off, len(wire)), what
        assert whole[off.value: off.value + ln.value].tobytes() == wire, what
        for (key, a), p, length in zip(inputs, poff, plen):
            assert whole[p: p + length].tobytes() == payload_bytes(a), (what, key)


def _decode_cast(dev, wires, dst_stride, cast):
    """b200tfs_set_decode_cast + b200tfs_decode_responses on device-resident wires; returns (slots, outs, n_outs, status)."""
    n = len(wires)
    off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    cur = 0
    for i, w in enumerate(wires):
        off[i], ln[i] = cur, len(w)
        cur += (len(w) + 255) & ~255
    buf = np.zeros(cur + 256, dtype=np.uint8)
    for i, w in enumerate(wires):
        buf[off[i]: off[i] + len(w)] = np.frombuffer(w, dtype=np.uint8)
    wire_dev = dev.upload(buf)
    dst = dev.malloc(dst_stride * n + 256)
    N.check(dev.lib.b200tfs_memset(dev.ctx, dst, 0xEE, dst_stride * n))
    N.check(dev.lib.b200tfs_set_decode_cast(dev.ctx, cast))
    N.check(dev.lib.b200tfs_decode_responses(dev.ctx, wire_dev, n, off, ln, dst, dst_stride))
    outs = (N.Output * (n * N.FUSED_MAX_OUTPUTS))()
    n_outs, status = (C.c_int32 * n)(), (C.c_int32 * n)()
    N.check(dev.lib.b200tfs_decode_results(dev.ctx, n, outs, n_outs, None, status))
    return dev.download(dst, dst_stride * n).reshape(n, dst_stride), outs, n_outs, status


@pytest.mark.parametrize("cast", [19, 14])
def test_fused_decode_narrows_float_outputs(dev, cast):
    """b200tfs_set_decode_cast: DT_FLOAT outputs leave the single-launch decode as fp16 / bf16 (numpy's astype rounding, bit for
    bit), other dtypes untouched; walk path (first launch), template path (second), a record the template does not fit (third),
    odd sizes and a payload that starts at an odd destination phase; then a batch large enough for the TMA-staged kernel."""
    import ml_dtypes

    np_dt = np.float16 if cast == 19 else ml_dtypes.bfloat16
    rng = np.random.default_rng(cast)
    f = (rng.standard_normal(100003) * 100).astype(np.float32)
    f[:6] = np.array([np.inf, -np.inf, 0.0, -0.0, 65504.0, 1e-8], dtype=np.float32)
    d = rng.standard_normal(777)
    small = rng.standard_normal(5).astype(np.float32)
    wires = [wire_oracle.build_predict_response([("scores", f), ("aux", d), ("s", small)]),
             wire_oracle.build_predict_response([("scores", f[::-1].copy()), ("aux", d), ("s", small)]),
             wire_oracle.build_predict_response([("other", f[:4099])])]
    for rep in range(2):
        for w in wires:
            slot, outs, n_outs, status = _decode_cast(dev, [w], 1 << 20, cast)
            assert status[0] == 0, (rep, status[0])
            ref = wire_oracle.decode_predict_response(w)
            buf = np.frombuffer(w, dtype=np.uint8)
            for k in range(n_outs[0]):
                o = outs[k]
                name = bytes(buf[o.key_off: o.key_off + o.key_len]).decode()
                want = ref[name].astype(np_dt) if ref[name].dtype == np.float32 else ref[name]
                assert o.status == 0 and o.dst_bytes == want.nbytes, (name, o.dst_bytes)
                assert slot[0, o.dst_off: o.dst_off + o.dst_bytes].tobytes() == want.tobytes(), (rep, name)
    # switching the cast off again: the template learnt for the cast must not serve the uncast launch
    slot, outs, n_outs, status = _decode_cast(dev, [wires[0]], 1 << 20, 1)
    ref = wire_oracle.decode_predict_response(wires[0])
    for k in range(n_outs[0]):
        name = bytes(np.frombuffer(wires[0], dtype=np.uint8)[outs[k].key_off: outs[k].key_off + outs[k].key_len]).decode()
        assert slot[0, outs[k].dst_off: outs[k].dst_off + outs[k].dst_bytes].tobytes() == ref[name].tobytes()
    # a batch for the staged kernel: 96 responses x 602 KB of float32
    imgs = [rng.standard_normal(150528).astype(np.float32) for _ in range(4)]
    batch = [wire_oracle.build_predict_response([("image", imgs[i % 4])]) for i in range(96)]
    for rep in range(2):
        slot, outs, n_outs, status = _decode_cast(dev, batch, (150528 * 2 + 255) & ~255, cast)
        assert all(status[i] == 0 and n_outs[i] == 1 for i in range(96))
        for i in range(96):
            o = outs[i * N.FUSED_MAX_OUTPUTS]
            assert slot[i, o.dst_off: o.dst_off + o.dst_bytes].tobytes() == imgs[i % 4].astype(np_dt).tobytes(), (rep, i)
    assert dev.lib.b200tfs_set_decode_cast(dev.ctx, 9) == N.E_DTYPE


@pytest.mark.parametrize("cast", [19, 14])
def test_narrowing_batch_decode_in_three_launches(dev, cast):
    """A batch whose record length the host knows a template for: verify launch (guard words + table), guarded move over a
    host-built plan, fallback launch for the records the verify launch did not vouch for.  Record 5 has the same LENGTH but
    another key (same key length): its guard stays 0 and the third launch walks it; records of a batch with two outputs each."""
    import ml_dtypes

    np_dt = np.float16 if cast == 19 else ml_dtypes.bfloat16
    rng = np.random.default_rng(100 + cast)
    imgs = [rng.standard_normal(150528).astype(np.float32) * 50 for _ in range(3)]
    aux = rng.standard_normal(4099).astype(np.float32)
    def wire(i, key="image"):
        return wire_oracle.build_predict_response([(key, imgs[i % 3]), ("aux", aux + i)])
    batch = [wire(i) for i in range(24)]
    stride = (150528 * 2 + 4099 * 2 + 1024 + 255) & ~255
    l0 = C.c_uint64(); N.check(dev.lib.b200tfs_kernel_launches(dev.ctx, C.byref(l0)))
    for rep in range(3):
        if rep == 2:
            batch[5] = wire(5, key="imagf")          # same length, other framing
        slot, outs, n_outs, status = _decode_cast(dev, batch, stride, cast)
        for i in range(24):
            assert status[i] == 0 and n_outs[i] == 2, (rep, i, status[i])
            ref = wire_oracle.decode_predict_response(batch[i])
            buf = np.frombuffer(batch[i], dtype=np.uint8)
            for k in range(2):
                o = outs[i * N.FUSED_MAX_OUTPUTS + k]
                name = bytes(buf[o.key_off: o.key_off + o.key_len]).decode()
                want = ref[name].astype(np_dt)
                assert o.dst_bytes == want.nbytes and slot[i, o.dst_off: o.dst_off + o.dst_bytes].tobytes() == want.tobytes(), (rep, i, name)
    l1 = C.c_uint64(); N.check(dev.lib.b200tfs_kernel_launches(dev.ctx, C.byref(l1)))
    assert l1.value - l0.value >= 1 + 3 + 3, "the second and third call run as three launches each"


def test_python_out_dtypes_take_the_narrowing_launch(codec):
    """decode_predict_response(out_dtypes={key: float16}) on float32 outputs is one launch (no parse + synchronise + unpack);
    a request that does not cover every float32 output, or asks a non-float output to change, falls back and is still right."""
    import ml_dtypes

    rng = np.random.default_rng(77)
    f, g = rng.standard_normal((300, 70)).astype(np.float32), rng.standard_normal(999).astype(np.float32)
    ids = rng.integers(0, 1000, 50)
    resp = wire_oracle.build_predict_response([("f", f), ("g", g), ("ids", ids)])
    for np_dt in (np.float16, ml_dtypes.bfloat16):
        def fused_records():
            a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
            N.check(codec._lib.b200tfs_decode_stats(codec._ctx, C.byref(a), C.byref(b), C.byref(c)))
            return a.value + b.value + c.value
        r0 = fused_records()
        got = codec.decode_predict_response(resp, out_dtypes={"f": np_dt, "g": np_dt})[0]
        assert got["f"].dtype == np.dtype(np_dt) and got["f"].tobytes() == f.astype(np_dt).tobytes()
        assert got["g"].tobytes() == g.astype(np_dt).tobytes() and got["ids"].tobytes() == ids.tobytes()
        assert fused_records() == r0 + 1                   # served by the single-launch decode, not by parse + unpack
        part = codec.decode_predict_response(resp, out_dtypes={"f": np_dt})[0]      # g stays float32: the two-phase route
        assert part["f"].tobytes() == f.astype(np_dt).tobytes() and part["g"].tobytes() == g.tobytes()


def test_randomised_batches_through_the_fused_decode(codec):
    """Seeded fuzz of the single-launch decode's bookkeeping (framing templates kept across launches, per-record CTA budgets from
    a known template, batches mixing records that match the template with records of the same or another length that do not):
    random responses of 1-4 outputs of random fixed-width / varint dtypes, decoded in random groupings, repeatedly, against
    the oracle."""
    rng = np.random.default_rng(20260921)
    dtypes = [np.float32, np.float64, np.int32, np.int64, np.uint8, np.bool_, np.float32, np.float32]
    def tensor():
        dt = dtypes[rng.integers(len(dtypes))]
        shape = tuple(int(v) for v in rng.integers(1, 40, size=rng.integers(1, 4)))
        if dt in (np.float32, np.float64):
            return rng.standard_normal(shape).astype(dt)
        if dt == np.bool_:
            return rng.integers(0, 2, size=shape).astype(np.bool_)
        return rng.integers(-1000 if dt != np.uint8 else 0, 100000 if dt not in (np.uint8,) else 256, size=shape).astype(dt)
    shapes = []       # a pool of "models": fixed keys / dtypes / shapes, fresh values per response
    for _ in range(6):
        keys = ["out%d" % k for k in range(rng.integers(1, 5))]
        shapes.append([(k, tensor()) for k in keys])
    def response(m):
        outs = []
        for k, proto in shapes[m]:
            if proto.dtype.kind == "f":
                v = rng.standard_normal(proto.shape).astype(proto.dtype)
            elif proto.dtype == np.bool_:
                v = rng.integers(0, 2, size=proto.shape).astype(np.bool_)
            else:
                v = rng.integers(0, 100, size=proto.shape).astype(proto.dtype)      # same varint lengths: same record length
            outs.append((k, v))
        return wire_oracle.build_predict_response(outs)
    for round_ in range(40):
        n = int(rng.integers(1, 20))
        favourite = int(rng.integers(len(shapes)))
        wires = [response(favourite if rng.random() < 0.7 else int(rng.integers(len(shapes)))) for _ in range(n)]
        got = codec.decode_predict_responses(wires)
        assert len(got) == n
        for w, (arrays, spec) in zip(wires, got):
            ref = wire_oracle.decode_predict_response(w)
            assert set(arrays) == set(ref), round_
            for k in ref:
                assert arrays[k].dtype == ref[k].dtype and arrays[k].shape == ref[k].shape and arrays[k].tobytes() == ref[k].tobytes(), (round_, k)
