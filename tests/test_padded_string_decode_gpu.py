"""DT_STRING outputs of the padded batch decode as padded byte columns (Codec.decode_predict_responses_padded with
string_columns=True, b200tfs_decode_padded_strings), byte for byte against the definition in tests/padded_string_decode_ref.py."""
import ctypes as C

import numpy as np
import pytest
from google.protobuf.message import DecodeError

import golden_util as G
import padded_string_decode_ref as PR
import string_responses as SR
from min_tfs_client import _native as N
from min_tfs_client import device as DV
from min_tfs_client.codec import BytesColumn
from tensorflow_serving.apis import predict_pb2

pytestmark = pytest.mark.gpu

EDGE = [b"", b"\x00", b"\x00\xff\x80\x7f", b"a" * 127, b"b" * 128, b"c" * 16383, b"d" * 16384, b"\xee" * 70000]


def host(a):
    return a.copy_to_host() if hasattr(a, "copy_to_host") else np.asarray(a)


def same_column(col, ref, shapes=None):
    data, offsets, shape, want_shapes = ref
    assert isinstance(col, BytesColumn) and col.shape == shape
    assert host(col.offsets).dtype == np.int64 and host(col.offsets).tolist() == offsets.tolist()
    assert host(col.data).tobytes() == data.tobytes()
    if shapes is not None:
        assert shapes.dtype == np.int64 and shapes.tolist() == want_shapes.tolist()


def padded(codec, wires, keys, **kw):
    return codec.decode_predict_responses_padded(wires, keys, string_columns=True, **kw)


def launches(codec):
    c = C.c_uint64()
    N.check(codec._lib.b200tfs_kernel_launches(codec._ctx, C.byref(c)))
    return c.value


def ragged(rng, n, rank, lo, hi, max_t=6):
    """n responses of a string key "s" of the given rank, trailing dims differing per response, beside float32 "f" [1, T, 3] and
    packed int64 "i" [T]."""
    wires = []
    for _ in range(n):
        dims = [int(rng.integers(0, 4))] + [int(rng.integers(0, max_t)) for _ in range(rank - 1)]
        t = int(rng.integers(0, max_t))
        wires.append(SR.response(("f", SR.float_tensor(rng.standard_normal((1, t, 3)).astype(np.float32))),
                                 ("s", SR.string_tensor(SR.random_strings(rng, int(np.prod(dims)), lo, hi), dims)),
                                 ("i", SR.int64_tensor(rng.integers(-2**40, 2**40, t)))))
    return wires


@pytest.mark.parametrize("pad", [b"", b"[PAD]"], ids=["empty_pad", "PAD"])
@pytest.mark.parametrize("rank", [1, 2, 3])
def test_ranks_beside_numeric_keys(codec, rank, pad):
    rng = np.random.default_rng(rank)
    wires = ragged(rng, 17, rank, 0, 30)
    plain = codec.decode_predict_responses_padded(wires, ["f", "i"], pad_value=-1)
    for device in (False, True):
        before, l0 = codec.padded_device_calls, launches(codec)
        got, shapes, _ = padded(codec, wires, ["s", "f", "i"], device=device, string_pad=pad, pad_value=-1)
        assert codec.padded_device_calls == before + 1 and launches(codec) == l0 + 10
        same_column(got["s"], PR.reference(wires, "s", pad), shapes["s"])
        if device:
            assert DV.is_device_object(got["s"].data) and DV.is_device_object(got["s"].offsets)
        for k in ("f", "i"):
            assert host(got[k]).tobytes() == plain[0][k].tobytes() and host(got[k]).shape == plain[0][k].shape
            assert shapes[k].tolist() == plain[1][k].tolist()


def test_pad_to_zero_rows_and_zero_trailing_dim(codec):
    rng = np.random.default_rng(5)
    s = SR.random_strings(rng, 40, 0, 12)
    wires = [SR.response(("s", SR.string_tensor(s[:6], [1, 2, 3]))), SR.response(("s", SR.string_tensor([], [0, 4, 1]))),
             SR.response(("s", SR.string_tensor(s[6:14], [2, 1, 4]))), SR.response(("s", SR.string_tensor([], [3, 0, 2])))]
    for pad_to in (None, (6, 7)):
        kw = {"pad_to": {"s": pad_to}} if pad_to else {}
        before = codec.padded_device_calls
        got, shapes, _ = padded(codec, wires, ["s"], string_pad=b"<p>", **kw)
        assert codec.padded_device_calls == before + 1
        same_column(got["s"], PR.reference(wires, "s", b"<p>", pad_to), shapes["s"])
    zero = [SR.response(("s", SR.string_tensor([], [2, 0]))), SR.response(("s", SR.string_tensor([], [1, 0])))]
    got, shapes, _ = padded(codec, zero, ["s"], string_pad=b"x")
    same_column(got["s"], PR.reference(zero, "s", b"x"), shapes["s"])
    assert got["s"].shape == (3, 0)


def test_edge_strings(codec):
    rng = np.random.default_rng(6)
    s = SR.random_strings(rng, 12, 0, 20)
    wires = [SR.response(("s", SR.string_tensor(EDGE, [1, len(EDGE)]))), SR.response(("s", SR.string_tensor(s[:3], [1, 3], unknown=True))),
             SR.response(("s", SR.string_tensor(s[3:], [-1, 9], dtype_last=True)))]
    for pad in (b"", b"[PAD]", b"\x00" * 200):
        for device in (False, True):
            before = codec.padded_device_calls
            got, shapes, _ = padded(codec, wires, ["s"], string_pad=pad, device=device)
            assert codec.padded_device_calls == before + 1
            same_column(got["s"], PR.reference(wires, "s", pad), shapes["s"])


def test_4096_records(codec):
    rng = np.random.default_rng(7)
    wires = [SR.response(("s", SR.string_tensor(SR.random_strings(rng, t, 0, 12), [1, t]))) for t in rng.integers(0, 9, 4096).tolist()]
    before = codec.padded_device_calls
    got, shapes, _ = padded(codec, wires, ["s"], device=True, string_pad=b"[PAD]")
    assert codec.padded_device_calls == before + 1
    same_column(got["s"], PR.reference(wires, "s", b"[PAD]"), shapes["s"])


def test_64_by_t_by_1000(codec):
    rng = np.random.default_rng(8)
    wires = []
    for t in rng.integers(1, 9, 64):
        lens = rng.integers(3, 11, int(t) * 1000)
        strs = [bytes([65 + int(x) % 26]) * int(x) for x in lens]
        wires.append(SR.response(("s", SR.string_tensor(strs, [int(t), 1000]))))
    got, shapes, _ = padded(codec, wires, ["s"], device=True)
    data, offsets, shape, want_shapes = PR.reference(wires, "s")
    assert got["s"].shape == shape and shapes["s"].tolist() == want_shapes.tolist()
    assert host(got["s"].offsets).tolist() == offsets.tolist() and host(got["s"].data).tobytes() == data.tobytes()


def merged_response(s):
    return G.ld(0x0A, G.ld(0x0A, b"s") + G.ld(0x12, SR.string_tensor(s[:4], [1, 8])) + G.ld(0x12, SR.strings_body(s[4:8]))) + G.mspec()


def test_refusals_take_the_host_route(codec):
    rng = np.random.default_rng(9)
    s = SR.random_strings(rng, 8, 0, 9)
    good = SR.response(("s", SR.string_tensor(s[:3], [1, 3])))
    cases = {"merged": [good, merged_response(s)]}
    many = [SR.response(*[(f"k{j}", SR.string_tensor(s[:j % 4], [1, j % 4])) for j in range(9)]) for _ in range(3)]
    cases["nine_keys"] = many
    for name, wires in cases.items():
        keys = [f"k{j}" for j in range(9)] if name == "nine_keys" else ["s"]
        for device in (False, True):
            before = codec.padded_device_calls
            got, shapes, _ = padded(codec, wires, keys, string_pad=b"~", device=device)
            assert codec.padded_device_calls == before, name
            for k in keys:
                same_column(got[k], PR.reference(wires, k, b"~"), shapes[k])


def test_every_error_class(codec):
    s = [b"a", b"\x00b"]
    good = SR.response(("s", SR.string_tensor(s, [1, 2])))
    bad = {
        "key": SR.response(("t", SR.string_tensor(s, [1, 2]))),
        "dtype": SR.response(("s", SR.float_tensor(np.ones((1, 2), np.float32)))),
        "rank": SR.response(("s", SR.string_tensor(s, [2]))),
        "rank0": SR.response(("s", SR.string_tensor(s[:1], []))),
        "count": SR.response(("s", SR.string_tensor(s, [1, 3]))),
        "parse": good[:-4],
    }
    for name, w in bad.items():
        want = SR.outcome(lambda: PR.reference([good, w], "s"))
        assert isinstance(want, type) and issubclass(want, Exception), name
        for device in (False, True):
            got = SR.outcome(lambda: padded(codec, [good, w], ["s"], device=device))
            assert got is want, (name, device, got, want)
    big = [good, SR.response(("s", SR.string_tensor([b"x"] * 3, [1, 3])))]
    assert SR.outcome(lambda: PR.reference(big, "s", pad_to=(2,))) is ValueError
    assert SR.outcome(lambda: padded(codec, big, ["s"], pad_to={"s": (2,)})) is ValueError
    assert SR.outcome(lambda: padded(codec, [good, good[:-4]], ["s"])) is DecodeError
    with pytest.raises(ValueError):
        padded(codec, [good], ["s"], out={"s": np.zeros(3, np.int64)})


def test_without_string_columns_nothing_changes(codec):
    wires = [SR.response(("f", SR.float_tensor(np.ones((1, t, 2), np.float32)))) for t in (1, 3)]
    l0 = launches(codec)
    got, _, _ = codec.decode_predict_responses_padded(wires, ["f"])
    assert launches(codec) == l0 + 6 and got["f"].shape == (2, 3, 2)
    l0 = launches(codec)
    padded(codec, wires, ["f"])            # no string key: the same call
    assert launches(codec) == l0 + 6


def test_round_trip_into_the_padded_encode(codec):
    rng = np.random.default_rng(10)
    outs = [SR.random_strings(rng, 1 * t, 0, 16) for t in (3, 0, 7, 1)]
    wires = [SR.response(("s", SR.string_tensor(o, [1, len(o)]))) for o in outs]
    got, shapes, _ = padded(codec, wires, ["s"], device=True)
    reqs = codec.encode_predict_requests_padded("m", {"s": got["s"]}, {"s": shapes["s"]})
    assert len(reqs) == len(wires)
    for q, o in zip(reqs, outs):
        assert list(predict_pb2.PredictRequest.FromString(q).inputs["s"].string_val) == o


# ---- the C ABI ------------------------------------------------------------------------------------------------------------
def _c_call(codec, wires, keys, tail, pad=b"", caps=None, data_caps=None, guard=64):
    """b200tfs_decode_padded_strings over a device arena, destinations with guard bytes of 0xEE behind their capacities."""
    lib, ctx = codec._lib, codec._ctx
    buf, off, ln = codec._pack_wires(wires)
    n, nk = len(wires), len(keys)
    pk, ps = (N.PadKey * nk)(), (N.PaddedStrings * nk)()
    kb = [k.encode() for k in keys]
    for i, k in enumerate(kb):
        pk[i].key, pk[i].key_len = k, len(k)
    N.check(lib.b200tfs_padded_strings_layout(buf.ctypes.data, n, off, ln, nk, pk, ps, 0))
    arena = DV.DeviceArray(codec, (len(buf),), np.uint8).copy_from_host(buf)
    offs, datas = [], []
    for i in range(nk):
        m = int(pk[i].dims[0]) * int(np.prod(tail[i], dtype=np.int64))
        oc = caps[i] if caps else 8 * (m + 1)
        dc = data_caps[i] if data_caps else int(ps[i].data_bytes) + (m - int(ps[i].strings)) * len(pad)
        offs.append(DV.DeviceArray(codec, (oc + guard,), np.uint8).copy_from_host(np.full(oc + guard, 0xEE, np.uint8)))
        datas.append(DV.DeviceArray(codec, (dc + guard,), np.uint8).copy_from_host(np.full(dc + guard, 0xEE, np.uint8)))
        pk[i].dst, pk[i].dst_cap, pk[i].rank = offs[i].ptr, oc, len(tail[i]) + 1
        for d, x in enumerate(tail[i]):
            pk[i].dims[d + 1] = x
        ps[i].data, ps[i].data_cap, ps[i].pad, ps[i].pad_len = datas[i].ptr, dc, C.cast(C.c_char_p(pad), C.c_void_p), len(pad)
    return lib, ctx, off, ln, pk, ps, arena, offs, datas, (kb, pad)


def _results(codec, n, nk):
    outs, st = (N.Output * (n * nk))(), (C.c_int32 * n)()
    N.check(codec._lib.b200tfs_padded_results(codec._ctx, n, nk, outs, None, st))
    return outs


@pytest.mark.parametrize("short", ["offsets", "data"])
def test_capacity_short_by_one(codec, short):
    rng = np.random.default_rng(11)
    wires = [SR.response(("s", SR.string_tensor(SR.random_strings(rng, t, 1, 9), [1, t]))) for t in (2, 4, 3)]
    data, offsets, _, _ = PR.reference(wires, "s", b"PAD", (4,))
    oc, dc = 8 * len(offsets), len(data)
    if short == "offsets":
        oc -= 8
    else:
        dc -= 1
    lib, ctx, off, ln, pk, ps, arena, offs, datas, keep = _c_call(codec, wires, ["s"], [(4,)], b"PAD", [oc], [dc])
    l0 = launches(codec)
    N.check(lib.b200tfs_decode_padded_strings(ctx, arena.ptr, 3, off, ln, 1, pk, ps))
    assert launches(codec) == l0 + 10
    outs = _results(codec, 3, 1)
    assert [outs[r].status for r in range(3)] == [N.OK, N.OK, N.E_SIZE]
    assert [outs[r].dst_off for r in range(3)] == [0, 32, 64]
    assert (offs[0].copy_to_host()[oc:] == 0xEE).all() and (datas[0].copy_to_host()[dc:] == 0xEE).all()
    o = offs[0].copy_to_host()[:8 * 9].view(np.int64)        # the first two records' rows, and the entry behind them
    assert o.tolist() == offsets[:9].tolist()
    assert datas[0].copy_to_host()[: offsets[8]].tobytes() == data[: offsets[8]].tobytes()


def test_launches_without_entries_match_the_numeric_decode(codec):
    wires = [SR.response(("f", SR.float_tensor(np.ones((1, 2), np.float32))))] * 2
    buf, off, ln = codec._pack_wires(wires)
    arena = DV.DeviceArray(codec, (len(buf),), np.uint8).copy_from_host(buf)
    dst = DV.DeviceArray(codec, (64,), np.uint8)
    pk = (N.PadKey * 1)()
    pk[0].key, pk[0].key_len, pk[0].dst, pk[0].dst_cap, pk[0].rank, pk[0].dims[1] = b"f", 1, dst.ptr, 64, 2, 2
    counts = []
    for call in (lambda: codec._lib.b200tfs_decode_padded(codec._ctx, arena.ptr, 2, off, ln, 1, pk),
                 lambda: codec._lib.b200tfs_decode_padded_strings(codec._ctx, arena.ptr, 2, off, ln, 1, pk, None)):
        l0 = launches(codec)
        N.check(call())
        _results(codec, 2, 1)
        counts.append(launches(codec) - l0)
    assert counts == [6, 6]


def test_c_graph_replays_over_new_records(codec):
    from min_tfs_client.codec import Codec

    def rec(strs, size):
        w = SR.response(("s", SR.string_tensor(strs, [1, len(strs)])), ("f", SR.float_tensor(np.full((1, 2), len(strs), np.float32))))
        pad = size - len(w)
        assert pad >= 3
        return w + b"\xAA\x06" + G.vi(pad - 3) + b"z" * (pad - 3)
    a = [rec([b"ab"] * 10, 200), rec([b"\x00" * 30], 200), rec([b""] * 3, 200)]
    b = [rec([b"q" * 7] * 3, 200), rec([b""] * 12, 200), rec([b"\xff" * 50, b"r"], 200)]
    assert [len(w) for w in a] == [len(w) for w in b] == [200] * 3
    gc = Codec(0)            # a captured graph pins the context's scratch buffers
    ms, mb = C.c_uint64(), C.c_uint64()
    N.check(gc._lib.b200tfs_concat_strings_bound(3, (C.c_uint64 * 3)(200, 200, 200), C.byref(ms), C.byref(mb)))
    T, R = 16, 3            # trailing dims fixed at the longest sequence, at most R rows
    lib, ctx, off, ln, pk, ps, arena, offs, datas, keep = _c_call(gc, a, ["s", "f"], [(T,), (2,)], b"[PAD]",
                                                                  [8 * (R * T + 1), 64], [mb.value + R * T * 5, 0])
    N.check(lib.b200tfs_decode_padded_strings(ctx, arena.ptr, 3, off, ln, 2, pk, ps))
    _results(gc, 3, 2)
    N.check(lib.b200tfs_capture_begin(ctx))
    N.check(lib.b200tfs_decode_padded_strings(ctx, arena.ptr, 3, off, ln, 2, pk, ps))
    g = C.c_void_p()
    N.check(lib.b200tfs_capture_end(ctx, C.byref(g)))
    for wires in (b, a, b):
        buf, _, _ = gc._pack_wires(wires)
        N.check(lib.b200tfs_memcpy_h2d(ctx, arena.ptr, buf.ctypes.data, buf.nbytes))
        N.check(lib.b200tfs_graph_launch(ctx, g))
        outs = _results(gc, 3, 2)
        assert all(outs[j].status == N.OK for j in range(6))
        data, offsets, _, _ = PR.reference(wires, "s", b"[PAD]", (T,))
        got_o = offs[0].copy_to_host()[: 8 * len(offsets)].view(np.int64)
        assert got_o.tolist() == offsets.tolist()
        assert datas[0].copy_to_host()[: len(data)].tobytes() == data.tobytes()
        assert offs[1].copy_to_host()[:24].view(np.float32).tolist() == [x for w in wires for x in floats(w)]
    N.check(lib.b200tfs_graph_destroy(g))
    del arena, offs, datas
    gc.close()


def floats(w):
    return list(predict_pb2.PredictResponse.FromString(w).outputs["f"].float_val)


def test_host_wire_form(codec):
    rng = np.random.default_rng(12)
    wires = [SR.response(("s", SR.string_tensor(SR.random_strings(rng, 2 * r, 0, 300), [r, 2]))) for r in (2, 3, 0, 1)]
    lib, ctx, off, ln, pk, ps, arena, offs, datas, keep = _c_call(codec, wires, ["s"], [(2,)], b"-")
    buf, _, _ = codec._pack_wires(wires)
    N.check(lib.b200tfs_decode_padded_strings_host_async(ctx, buf.ctypes.data, 4, off, ln, 1, pk, ps))
    _results(codec, 4, 1)
    data, offsets, _, _ = PR.reference(wires, "s", b"-")
    assert offs[0].copy_to_host()[: 8 * len(offsets)].view(np.int64).tolist() == offsets.tolist()
    assert datas[0].copy_to_host()[: len(data)].tobytes() == data.tobytes()
