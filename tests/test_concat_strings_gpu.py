"""DT_STRING outputs of the concatenated batch decode as offset-indexed byte columns (Codec.decode_predict_responses_concat with
string_columns=True, b200tfs_decode_concat_strings), against the definition in tests/string_responses.py."""
import ctypes as C

import numpy as np
import pytest
from google.protobuf.message import DecodeError

import decode_mutants as D
import golden_util as G
import string_responses as SR
from min_tfs_client import _native as N
from min_tfs_client import device as DV
from min_tfs_client.codec import BytesColumn

pytestmark = pytest.mark.gpu


def host(a):
    return a.copy_to_host() if hasattr(a, "copy_to_host") else np.asarray(a)


def same_column(col, ref):
    data, offsets, shape = ref
    assert isinstance(col, BytesColumn) and col.shape == shape
    assert host(col.offsets).dtype == np.int64 and host(col.offsets).tolist() == offsets.tolist()
    assert host(col.data).tobytes() == data.tobytes()


def concat(codec, wires, keys, **kw):
    return codec.decode_predict_responses_concat(wires, keys, string_columns=True, **kw)[0]


def launches(codec):
    c = C.c_uint64()
    N.check(codec._lib.b200tfs_kernel_launches(codec._ctx, C.byref(c)))
    return c.value


EDGE = [b"", b"\x00", b"\x00\xff\x80\x7f", b"a" * 127, b"b" * 128, b"c" * 16383, b"d" * 16384, b"\xee" * 70000]


def test_edges_beside_numeric_keys_on_the_device_route(codec):
    rng = np.random.default_rng(1)
    s = SR.random_strings(rng, 30, 0, 20)
    x, ids = rng.standard_normal((3, 4)).astype(np.float32), np.arange(-6, 6, dtype=np.int64).reshape(3, 4)
    wires = [
        SR.response(("f", SR.float_tensor(x)), ("s", SR.string_tensor(EDGE, [len(EDGE)])), ("i", SR.int64_tensor(ids))),
        SR.response(("s", SR.string_tensor([], [0])), ("f", SR.float_tensor(x[:0])), ("i", SR.int64_tensor(ids[:0]))),
        SR.response(("i", SR.int64_tensor(ids)), ("s", SR.string_tensor(s[:12], [-1], unknown=True)), ("f", SR.float_tensor(x))),
        SR.response(("f", SR.float_tensor(x)), ("s", SR.string_tensor(s[12:], [18], dtype_last=True)), ("i", SR.int64_tensor(ids))),
    ]
    for device in (False, True):
        before, l0 = codec.concat_device_calls, launches(codec)
        got = concat(codec, wires, ["s", "f", "i"], device=device)
        assert codec.concat_device_calls == before + 1 and launches(codec) == l0 + 10
        same_column(got["s"], SR.reference(wires, "s"))
        plain = codec.decode_predict_responses_concat(wires, ["f", "i"])[0]
        for k in ("f", "i"):
            assert host(got[k]).tobytes() == plain[k].tobytes() and host(got[k]).shape == plain[k].shape


def test_no_string_key_keeps_six_launches(codec):
    wires = [SR.response(("f", SR.float_tensor(np.ones((2, 3), np.float32))))] * 3
    l0 = launches(codec)
    got = concat(codec, wires, ["f"])
    assert launches(codec) == l0 + 6 and got["f"].shape == (6, 3)


def test_merged_value_takes_the_host_route(codec):
    s = SR.random_strings(np.random.default_rng(2), 8, 0, 9)
    merged = G.ld(0x0A, G.ld(0x0A, b"s") + G.ld(0x12, SR.string_tensor(s[:4], [8])) + G.ld(0x12, SR.strings_body(s[4:]))) + G.mspec()
    wires = [SR.response(("s", SR.string_tensor(s[:3], [3]))), merged]
    before = codec.concat_device_calls
    got = concat(codec, wires, ["s"])
    assert codec.concat_device_calls == before
    same_column(got["s"], SR.reference(wires, "s"))
    same_column(concat(codec, wires, ["s"], device=True)["s"], SR.reference(wires, "s"))


@pytest.mark.parametrize("n,shape,lo,hi", [(4096, (3,), 0, 12), (64, (64, 1000), 3, 10)], ids=["4096_records", "64_labels"])
def test_large_batches(codec, n, shape, lo, hi):
    rng = np.random.default_rng(3)
    m = int(np.prod(shape))
    wires = [SR.response(("s", SR.string_tensor(SR.random_strings(rng, m, lo, hi), list(shape)))) for _ in range(n)]
    before = codec.concat_device_calls
    got = concat(codec, wires, ["s"], device=True)
    assert codec.concat_device_calls == before + 1
    same_column(got["s"], SR.reference(wires, "s"))


def test_every_error_class(codec):
    s = [b"a", b"\x00b"]
    good = SR.response(("s", SR.string_tensor(s, [2])))
    bad = {
        "key": SR.response(("t", SR.string_tensor(s, [2]))),
        "dtype": SR.response(("s", SR.float_tensor(np.ones(2, np.float32)))),
        "rank": SR.response(("s", SR.string_tensor(s, [1, 2]))),
        "rank0": SR.response(("s", SR.string_tensor(s[:1], []))),
        "count": SR.response(("s", SR.string_tensor(s, [3]))),
        "parse": good[:-4],
    }
    for name, w in bad.items():
        want = SR.outcome(lambda: SR.reference([good, w], "s"))
        assert isinstance(want, type) and issubclass(want, Exception), name
        for device in (False, True):
            got = SR.outcome(lambda: concat(codec, [good, w], ["s"], device=device))
            assert got is want, (name, device, got, want)
    trailing = [SR.response(("s", SR.string_tensor([b"x"] * 4, [2, 2]))), SR.response(("s", SR.string_tensor([b"x"] * 3, [1, 3])))]
    assert SR.outcome(lambda: concat(codec, trailing, ["s"])) is ValueError
    with pytest.raises(ValueError):
        concat(codec, [good], ["s"], out={"s": np.zeros(3, np.int64)})


def test_every_mutant_of_the_string_seed(codec):
    (seed, ms), = [(s, m) for s, m in D.corpus() if s.name == "multi"]
    assert b"\x42\x02ab" in seed.wire
    checked = 0
    for m in [D.Mutant(seed.name, "seed", seed.wire, len(seed.wire))] + ms:
        rec = m.record
        want = SR.outcome(lambda: SR.reference([rec], "s"))
        got = SR.outcome(lambda: concat(codec, [rec], ["s"]))
        if isinstance(got, dict) and not isinstance(got["s"], BytesColumn):   # a flip made "s" numeric: today's result
            plain = codec.decode_predict_responses_concat([rec], ["s"])[0]["s"]
            assert got["s"].dtype == plain.dtype and got["s"].tobytes() == plain.tobytes(), (m.kind, m.rec_len)
            continue
        if want is DecodeError and isinstance(got, dict):
            # malformed varints inside the unrequested "ids" payload: like today's route, only the requested output is decoded
            plain = codec.decode_predict_responses_concat([rec], ["s"])[0]["s"]
            col = got["s"]
            assert [x.encode() for x in plain.ravel().tolist()] == [bytes(col.data[a:b]) for a, b in zip(col.offsets[:-1], col.offsets[1:])]
            assert col.shape == plain.shape, (m.kind, m.rec_len)
            continue
        if isinstance(want, tuple):
            assert not isinstance(got, type), (m.kind, m.rec_len, got)
            same_column(got["s"], want)
            checked += 1
        else:
            assert got is want, (m.kind, m.rec_len, got, want)
    assert checked > 10


def test_device_columns_feed_the_example_encode(codec):
    rng = np.random.default_rng(4)
    wires = [SR.response(("s", SR.string_tensor(SR.random_strings(rng, 2 * r, 0, 30), [r, 2]))) for r in (3, 0, 5)]
    dev = concat(codec, wires, ["s"], device=True)["s"]
    hst = concat(codec, wires, ["s"])["s"]
    assert DV.is_device_object(dev.data) and DV.is_device_object(dev.offsets)
    data, offsets, shape = SR.reference(wires, "s")          # the host round trip: FromString, then the column of its strings
    ids = np.arange(8, dtype=np.int64)
    a = codec.encode_example_requests([("m", 1, {"s": dev, "id": ids})])
    b = codec.encode_example_requests([("m", 1, {"s": BytesColumn(data, offsets, shape), "id": ids})])
    assert a == b and a == codec.encode_example_requests([("m", 1, {"s": hst, "id": ids})])


def _c_call(codec, wires, keys, caps=None, data_caps=None, guard=64):
    """The C ABI over a device arena: (lib, ctx, off, ln, ck, sc, arena, offsets buffers, data buffers, kept alive)."""
    lib, ctx = codec._lib, codec._ctx
    buf, off, ln = codec._pack_wires(wires)
    n, nk = len(wires), len(keys)
    ck, sc = (N.ConcatKey * nk)(), (N.ConcatStrings * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        ck[i].key, ck[i].key_len = k, len(k)
    N.check(lib.b200tfs_concat_strings_layout(buf.ctypes.data, n, off, ln, nk, ck, sc, 0))
    arena = DV.DeviceArray(codec, (len(buf),), np.uint8).copy_from_host(buf)
    offs, datas = [], []
    for i in range(nk):
        oc = caps[i] if caps else int(ck[i].bytes)
        dc = data_caps[i] if data_caps else int(sc[i].data_bytes)
        offs.append(DV.DeviceArray(codec, (oc + guard,), np.uint8).copy_from_host(np.full(oc + guard, 0xEE, np.uint8)))
        datas.append(DV.DeviceArray(codec, (dc + guard,), np.uint8).copy_from_host(np.full(dc + guard, 0xEE, np.uint8)))
        ck[i].dst, ck[i].dst_cap = offs[i].ptr, oc
        sc[i].data, sc[i].data_cap = datas[i].ptr, dc
    return lib, ctx, off, ln, ck, sc, arena, offs, datas, kb


def _results(codec, n, nk):
    outs, st = (N.Output * (n * nk))(), (C.c_int32 * n)()
    N.check(codec._lib.b200tfs_concat_results(codec._ctx, n, nk, outs, None, st))
    return outs


def _column(offs, datas, i, m):
    o = offs[i].copy_to_host()[: 8 * (m + 1)].view(np.int64)
    return datas[i].copy_to_host()[: int(o[-1])], o


@pytest.mark.parametrize("short", ["offsets", "data"])
def test_capacity_short_by_one(codec, short):
    rng = np.random.default_rng(5)
    wires = [SR.response(("s", SR.string_tensor(SR.random_strings(rng, 4, 1, 9), [4]))) for _ in range(3)]
    data, offsets, _ = SR.reference(wires, "s")
    oc, dc = 8 * len(offsets), len(data)
    if short == "offsets":
        oc -= 8
    else:
        dc -= 1
    lib, ctx, off, ln, ck, sc, arena, offs, datas, kb = _c_call(codec, wires, ["s"], [oc], [dc])
    N.check(lib.b200tfs_decode_concat_strings(ctx, arena.ptr, 3, off, ln, 1, ck, sc))
    outs = _results(codec, 3, 1)
    assert [outs[r].status for r in range(3)] == [N.OK, N.OK, N.E_SIZE]
    assert [outs[r].dst_off for r in range(3)] == [0, 32, 64]
    assert (offs[0].copy_to_host()[oc:] == 0xEE).all() and (datas[0].copy_to_host()[dc:] == 0xEE).all()
    o = offs[0].copy_to_host()[:64].view(np.int64)
    assert o.tolist() == offsets[:8].tolist()
    assert datas[0].copy_to_host()[: offsets[8]].tobytes() == data[: offsets[8]].tobytes()


def test_c_graph_with_closed_form_caps_replays_over_new_records(codec):
    from min_tfs_client.codec import Codec

    def rec(strs, pad_to):
        w = SR.response(("s", SR.string_tensor(strs, [len(strs)])), ("f", SR.float_tensor(np.full(2, len(strs), np.float32))))
        pad = pad_to - len(w)
        assert 0 <= pad
        return w + (b"\xAA\x06" + G.vi(pad - 3) + b"z" * (pad - 3) if pad else b"")
    a = [rec([b"ab"] * 10, 160), rec([b"\x00" * 30], 160), rec([b""] * 3, 160)]
    b = [rec([b"q" * 7] * 3, 160), rec([b""] * 40, 160), rec([b"\xff" * 50, b"r"], 160)]
    assert [len(w) for w in a] == [len(w) for w in b] == [160] * 3
    gc = Codec(0)            # a captured graph pins the context's scratch buffers
    ms, mb = C.c_uint64(), C.c_uint64()
    N.check(gc._lib.b200tfs_concat_strings_bound(3, (C.c_uint64 * 3)(160, 160, 160), C.byref(ms), C.byref(mb)))
    lib, ctx, off, ln, ck, sc, arena, offs, datas, kb = _c_call(gc, a, ["s", "f"], [8 * (ms.value + 1), 64], [mb.value, 0])
    N.check(lib.b200tfs_decode_concat_strings(ctx, arena.ptr, 3, off, ln, 2, ck, sc))
    _results(gc, 3, 2)
    N.check(lib.b200tfs_capture_begin(ctx))
    N.check(lib.b200tfs_decode_concat_strings(ctx, arena.ptr, 3, off, ln, 2, ck, sc))
    g = C.c_void_p()
    N.check(lib.b200tfs_capture_end(ctx, C.byref(g)))
    for wires in (b, a, b):
        buf, _, _ = gc._pack_wires(wires)
        N.check(lib.b200tfs_memcpy_h2d(ctx, arena.ptr, buf.ctypes.data, buf.nbytes))
        N.check(lib.b200tfs_graph_launch(ctx, g))
        outs = _results(gc, 3, 2)
        assert all(outs[j].status == N.OK for j in range(6))
        data, offsets, _ = SR.reference(wires, "s")
        got_d, got_o = _column(offs, datas, 0, len(offsets) - 1)
        assert got_o.tolist() == offsets.tolist() and got_d.tobytes() == data.tobytes()
        assert offs[1].copy_to_host()[:24].view(np.float32).tolist() == [x for w in wires for x in floats(w)]
    N.check(lib.b200tfs_graph_destroy(g))
    del arena, offs, datas
    gc.close()


def floats(w):
    from tensorflow_serving.apis import predict_pb2

    return list(predict_pb2.PredictResponse.FromString(w).outputs["f"].float_val)


def test_host_wire_form(codec):
    rng = np.random.default_rng(6)
    wires = [SR.response(("s", SR.string_tensor(SR.random_strings(rng, r, 0, 300), [r]))) for r in (2, 7, 0, 1)]
    lib, ctx, off, ln, ck, sc, arena, offs, datas, kb = _c_call(codec, wires, ["s"])
    buf, _, _ = codec._pack_wires(wires)
    N.check(lib.b200tfs_decode_concat_strings_host_async(ctx, buf.ctypes.data, 4, off, ln, 1, ck, sc))
    _results(codec, 4, 1)
    data, offsets, _ = SR.reference(wires, "s")
    got_d, got_o = _column(offs, datas, 0, len(offsets) - 1)
    assert got_o.tolist() == offsets.tolist() and got_d.tobytes() == data.tobytes()
