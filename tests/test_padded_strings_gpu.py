"""DT_STRING inputs of the padded batch encode (Codec.encode_predict_requests_padded with BytesColumn inputs,
b200tfs_encode_padded_requests_columns_async), byte for byte against the protobuf runtime's requests (tests/padded_strings_ref.py)."""
import ctypes as C

import numpy as np
import pytest

import padded_strings_ref as R
from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn

pytestmark = pytest.mark.gpu

EDGE = [b"", b"\x00", b"ab\x00\x00", b"\x00\xff\x80\x7f", b"a" * 127, b"b" * 128, b"c" * 16383, b"d" * 16384,
        b"\xe9" * ((1 << 21) - 1), b"\x01" * (1 << 21), bytes(range(256)) * 4096]   # the last one: 1 MiB


def column(strings, dims, start=0):
    """A BytesColumn of host arrays; `start`: junk bytes in front (offsets[0] != 0)."""
    lens = np.array([len(s) for s in strings], np.int64)
    off = np.zeros(len(strings) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    data = np.concatenate([np.full(start, 0x5A, np.uint8)] + [np.frombuffer(s, np.uint8) for s in strings] + [np.zeros(0, np.uint8)])
    return BytesColumn(data, off + start, tuple(dims))


def rand_strings(rng, m, lo=0, hi=40):
    return [rng.integers(0, 256, int(k)).astype(np.uint8).tobytes() for k in rng.integers(lo, hi + 1, m)]


def launches(codec):
    return codec.kernel_launches()


def check(codec, padded, shapes, broadcast=None, strings=None, **kw):
    """padded / broadcast: codec inputs; strings: {key: (strings, dims)} of every string column (the reference's view)."""
    broadcast = broadcast or {}
    strings = strings or {}
    calls = codec.padded_encode_device_calls
    got = codec.encode_predict_requests_padded("model", padded, shapes, broadcast=broadcast, model_version=5, **kw)
    assert codec.padded_encode_device_calls == calls + 1
    host = lambda v: v.copy_to_host() if hasattr(v, "copy_to_host") else v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)
    ref = R.reference_requests("model", 5, {k: strings.get(k, None) or host(v) for k, v in padded.items()},
                               {k: host(s) for k, s in shapes.items()}, {k: strings.get(k, None) or host(v) for k, v in broadcast.items()},
                               order=kw.get("order", "deterministic"), grpc=kw.get("grpc_frame", False))
    assert len(got) == len(ref)
    for r, (g, w) in enumerate(zip(got, ref)):
        assert bytes(g) == w, r
    return got


def test_edge_strings_host_and_device_shapes(codec):
    n = len(EDGE)
    col = column(EDGE, (n,))
    rows = np.array([1, 1, 1, 1, 0, 2, 2, 2, n - 10], np.int64)   # a zero-row request too
    assert rows.sum() == n
    for s in (rows, codec.device_array(rows), rows.reshape(-1, 1), codec.device_array(rows.reshape(-1, 1))):
        check(codec, {"text": col}, {"text": s}, strings={"text": (EDGE, (n,))})


@pytest.mark.parametrize("rank", [2, 3])
def test_trimmed_trailing_dims(codec, rank):
    rng = np.random.default_rng(rank)
    n = 40
    dims = (3 * n,) + ((5,) if rank == 2 else (4, 6))
    strs = rand_strings(rng, int(np.prod(dims)), 0, 30)
    col = column(strs, dims, start=7)
    S = np.stack([rng.integers(0, 4, n)] + [rng.integers(0, d + 1, n) for d in dims[1:]], axis=1).astype(np.int64)
    S[rng.integers(0, n, 5), 0] = 0
    ids = rng.integers(-(1 << 40), 1 << 40, (3 * n, 9))
    check(codec, {"text": col, "ids": ids}, {"text": S, "ids": S[:, 0].copy()}, strings={"text": (strs, dims)})
    check(codec, {"text": col}, {"text": codec.device_array(S)}, strings={"text": (strs, dims)}, order="given", grpc_frame=True)


@pytest.mark.parametrize("rank", [0, 2])
def test_broadcast_strings(codec, rank):
    rng = np.random.default_rng(30 + rank)
    dims = () if rank == 0 else (3, 2)
    strs = rand_strings(rng, int(np.prod(dims, dtype=np.int64)), 0, 300)
    x = rng.standard_normal((20, 4)).astype(np.float32)
    check(codec, {"x": x}, {"x": np.array([3, 0, 7, 10], np.int64)}, {"image_bytes": column(strs, dims, start=3)},
          strings={"image_bytes": (strs, dims)})


def test_beside_numeric_inputs_all_options(codec):
    rng = np.random.default_rng(4)
    n, Rr = 64, 300
    strs = rand_strings(rng, Rr * 2, 0, 200)
    col = column(strs, (Rr, 2))
    rows = rng.multinomial(Rr, np.ones(n) / n).astype(np.int64)
    padded = {"text": col, "f": rng.standard_normal((Rr, 3)).astype(np.float32), "ids": rng.integers(-(1 << 62), 1 << 62, (Rr,)),
              "mask": rng.integers(0, 2, (Rr, 2)).astype(np.bool_)}
    shapes = {"text": rows, "f": rows, "ids": rows, "mask": rows}
    for kw in ({}, {"order": "given"}, {"grpc_frame": True}, {"out": "pinned"}):
        check(codec, padded, shapes, {"label": column([b"\x00q\x00"], ())}, strings={"text": (strs, (Rr, 2)), "label": ([b"\x00q\x00"], ())},
              **kw)


def test_sliced_pinned_torch_dlpack(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(5)
    strs = rand_strings(rng, 90, 0, 70)
    base = column(strs, (30, 3), start=11)
    rows = np.array([4, 0, 16, 10], np.int64)
    ref = {"s": (strs, (30, 3))}
    check(codec, {"s": base}, {"s": rows}, strings=ref)
    data = codec.pinned_empty((base.data_len,), np.uint8)
    data[:] = base.data
    offs = codec.pinned_empty((base.offsets.size,), np.int64)
    offs[:] = base.offsets
    check(codec, {"s": BytesColumn(data, offs, (30, 3))}, {"s": rows}, strings=ref)
    td, to = torch.from_numpy(base.data).cuda(), torch.from_numpy(base.offsets).cuda()
    check(codec, {"s": BytesColumn(td, to, (30, 3))}, {"s": torch.from_numpy(rows).cuda()}, strings=ref)
    dl = torch.utils.dlpack.from_dlpack(torch.utils.dlpack.to_dlpack(to))
    check(codec, {"s": BytesColumn(td, dl, (30, 3))}, {"s": rows}, strings=ref)
    # a slice of a longer device offsets vector: offsets[0] != 0 and the column's end before the buffer's
    big = torch.cat([torch.zeros(5, dtype=torch.int64, device="cuda"), to])
    check(codec, {"s": BytesColumn(td, big[5:], (30, 3))}, {"s": rows}, strings=ref)


def test_scale(codec):
    rng = np.random.default_rng(6)
    n = 4096
    rows = rng.integers(0, 4, n).astype(np.int64)
    strs = rand_strings(rng, int(rows.sum()), 0, 60)
    check(codec, {"q": column(strs, (len(strs),))}, {"q": rows}, strings={"q": (strs, (len(strs),))})
    m = 100_000
    strs = rand_strings(rng, m, 0, 30)
    rows = np.array([m // 2, 0, m - m // 2], np.int64)
    check(codec, {"q": column(strs, (m,)), "w": np.ones((m,), np.float32)}, {"q": rows, "w": rows}, strings={"q": (strs, (m,))})


def test_round_trip_from_string_decode(codec):
    from tensorflow_serving.apis import predict_pb2
    rng = np.random.default_rng(7)
    wires, allstr = [], []
    for r in range(12):
        k = int(rng.integers(0, 5))
        s = rand_strings(rng, k * 2, 0, 50)
        allstr += s
        resp = predict_pb2.PredictResponse()
        resp.outputs["tokens"].CopyFrom(R.string_proto(s, (k, 2)))
        wires.append(resp.SerializeToString())
    out = codec.decode_predict_responses_concat(wires, ["tokens"], string_columns=True, device=True)[0]["tokens"]
    assert out.data_on_device and out.offsets_on_device
    rows = np.array([len(allstr) // 2 - 3, 3], np.int64)
    check(codec, {"tokens": out}, {"tokens": rows}, strings={"tokens": (allstr, (len(allstr) // 2, 2))})


def test_fallback_and_per_request_route(codec):
    rng = np.random.default_rng(8)
    strs = rand_strings(rng, 20, 0, 9)
    strs[3] = b"tail\x00\x00"
    col = column(strs, (20,))
    padded = {f"k{i}": np.arange(20, dtype=np.float32) * i for i in range(8)}
    padded["s"] = col
    rows = np.array([5, 0, 15], np.int64)
    shapes = {k: rows for k in padded}
    calls = codec.padded_encode_device_calls
    got = codec.encode_predict_requests_padded("model", padded, shapes, model_version=5)
    assert codec.padded_encode_device_calls == calls
    ref = R.reference_requests("model", 5, {**{k: v for k, v in padded.items() if k != "s"}, "s": (strs, (20,))}, shapes, {})
    assert got == ref
    # the per-request encode of a host column; a device one is refused
    one = codec.encode_predict_requests([("model", 5, {"s": column(strs[:4], (2, 2))})])[0]
    assert one == R.request_wire("model", 5, {"s": R.string_proto(strs[:4], (2, 2))})
    with pytest.raises(ValueError, match="encode_predict_requests_padded"):
        codec.encode_predict_requests([("model", 5, {"s": BytesColumn(codec.device_array(col.data), col.offsets, (20,))})])
    # numpy str / bytes inputs keep their host route
    a = np.array(["x", "yy", "", "zzz"] * 5)
    got = codec.encode_predict_requests_padded("model", {"a": a}, {"a": rows}, model_version=5)
    assert codec.padded_encode_device_calls == calls
    assert got == codec.encode_predict_requests([("model", 5, {"a": a[0:5]}), ("model", 5, {"a": a[5:5]}), ("model", 5, {"a": a[5:]})])


def test_wire_dtype_and_host_offsets_refused_before_launch(codec):
    col = column([b"ab", b"c"], (2,))
    before = launches(codec)
    with pytest.raises(ValueError):
        codec.encode_predict_requests_padded("m", {"s": col}, {"s": np.array([2])}, wire_dtype="DT_FLOAT")
    bad = BytesColumn(col.data, np.array([0, 2, 1], np.int64), (2,))
    with pytest.raises(ValueError):
        codec.encode_predict_requests_padded("m", {"s": bad}, {"s": np.array([1, 1])})
    with pytest.raises(ValueError):
        codec.encode_predict_requests_padded("m", {"x": np.zeros((2,), np.float32)}, {"x": np.array([1, 1])}, broadcast={"s": bad})
    assert launches(codec) == before


def test_launch_counts(codec):
    x = np.zeros((6, 2), np.float32)
    rows = np.array([2, 4], np.int64)
    a = launches(codec)
    codec.encode_predict_requests_padded("m", {"x": x}, {"x": rows})
    b = launches(codec)
    codec.encode_predict_requests_padded("m", {"x": x, "s": column([b"a"] * 6, (6,))}, {"x": rows, "s": rows})
    c = launches(codec)
    assert b - a == 4                       # plan, layout, frame, move
    assert c - b == (b - a) + 2             # string count and string emit


def _raw_call(dev, col_data, col_off, dims, shapes_dev, cols, n):
    """One padded string input through the C ABI: (req, pins, bytes, keep)."""
    d = (C.c_int64 * len(dims))(*dims)
    t = N.Tensor(data=col_data, src_dtype=7, wire_dtype=7, rank=len(dims), flags=N.F_DEVICE_DATA, dims=d, key=b"s", key_len=1, packed_len=0)
    ts = (N.Tensor * 1)(t)
    pins = (N.PadInput * 1)(N.PadInput(shapes=shapes_dev, cols=cols))
    bs = (N.Bytes * 1)(N.Bytes(offsets=col_off, data_len=0, flags=N.F_DEVICE_DATA))
    req = N.Request(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_inputs=1, flags=0, inputs=ts)
    return req, pins, bs, (d, ts)


def test_bad_device_offsets_ahead_of_good_requests(codec):
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(9)
        n, per = 4, 50
        strs = rand_strings(rng, n * per * 2, 0, 40)
        col = column(strs, (n * per, 2), start=16)
        o = col.offsets.copy()
        o[20] = o[19] - 1                                   # request 0 reads offsets 0..100: a decrease there
        rows = np.full(n, per, np.int64)
        dd, do, ds = dev.upload(col.data), dev.upload(o), dev.upload(rows)
        req, pins, bs, keep = _raw_call(dev, dd, do, (n * per, 2), ds, 1, n)
        bs[0].data_len = col.data_len
        cap = C.c_uint64()
        N.check(lib.b200tfs_padded_request_columns_arena_size(n, C.byref(req), bs, C.byref(cap)))
        slack = 1 << 16
        arena0 = dev.malloc(cap.value + 2 * slack + 256)
        arena = (arena0 + slack + 255) & ~255
        fill = np.full(cap.value + 2 * slack + 256, 0xC3, np.uint8)
        N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena0, fill.ctypes.data, fill.nbytes))
        N.check(lib.b200tfs_encode_padded_requests_columns_async(dev.ctx, n, C.byref(req), pins, bs, arena, cap.value))
        off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
        assert lib.b200tfs_encode_results(dev.ctx, n, off, ln) == N.E_SHAPE
        assert off[0] == 0 and ln[0] == 0
        ref = R.reference_requests("m", 3, {"s": (strs, (n * per, 2))}, {"s": rows}, {})
        for r in range(1, n):
            assert dev.download(arena + off[r], ln[r]).tobytes() == ref[r], r
        mem = dev.download(arena0, fill.nbytes)
        inside = np.zeros(fill.nbytes, bool)
        for r in range(1, n):
            inside[arena - arena0 + off[r]: arena - arena0 + off[r] + ln[r]] = True
        assert (mem[~inside] == 0xC3).all()                # nothing written outside the good records
        torch = pytest.importorskip("torch")
        with pytest.raises(ValueError):
            codec.encode_predict_requests_padded("m", {"s": BytesColumn(col.data, torch.from_numpy(o).cuda(), (n * per, 2))}, {"s": rows})
    finally:
        dev.close()


def test_graph_replay_follows_shapes_data_and_offsets():
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(10)
        n, Rr, W, data_len = 8, 64, 3, 40_000

        def make():
            strs = rand_strings(rng, Rr * W, 0, 50)
            c = column(strs, (Rr, W), start=int(rng.integers(0, 30)))
            data = np.zeros(data_len, np.uint8)
            data[: c.data_len] = c.data
            S = np.stack([rng.multinomial(Rr - 5, np.ones(n) / n), rng.integers(0, W + 1, n)], axis=1).astype(np.int64)
            return strs, data, c.offsets, S
        strs, data, offs, S = make()
        dd, do, ds = dev.upload(data), dev.upload(offs), dev.upload(S)
        req, pins, bs, keep = _raw_call(dev, dd, do, (Rr, W), ds, 2, n)
        bs[0].data_len = data_len
        cap = C.c_uint64()
        N.check(lib.b200tfs_padded_request_columns_arena_size(n, C.byref(req), bs, C.byref(cap)))
        slack = 4096
        arena0 = dev.malloc(cap.value + 2 * slack + 256)
        arena = (arena0 + slack + 255) & ~255
        N.check(lib.b200tfs_encode_padded_requests_columns_async(dev.ctx, n, C.byref(req), pins, bs, arena, cap.value))
        N.check(lib.b200tfs_encode_results(dev.ctx, n, None, None))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_encode_padded_requests_columns_async(dev.ctx, n, C.byref(req), pins, bs, arena, cap.value))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
        for rep in range(4):
            strs, data, offs, S = make()
            fill = np.full(cap.value + 2 * slack + 256, 0x3C, np.uint8)
            for ptr, a in ((arena0, fill), (dd, data), (do, offs), (ds, S)):
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, ptr, a.ctypes.data, a.nbytes))
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_encode_results(dev.ctx, n, off, ln))
            ref = R.reference_requests("m", 3, {"s": (strs, (Rr, W))}, {"s": S}, {})
            mem = dev.download(arena0, fill.nbytes)
            inside = np.zeros(fill.nbytes, bool)
            for r in range(n):
                a = arena - arena0 + off[r]
                assert mem[a: a + ln[r]].tobytes() == ref[r], (rep, r)
                inside[a: a + ln[r]] = True
            assert (mem[~inside] == 0x3C).all()
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


@pytest.mark.parametrize("empty", [(0,), (3, 0), (0, 2)])
def test_empty_broadcast_beside_string_inputs(codec, empty):
    """A broadcast column of no strings still takes a string tile per request, next to other string inputs."""
    rng = np.random.default_rng(11)
    strs = rand_strings(rng, 4, 0, 20)
    tag = rand_strings(rng, 3, 1, 9)
    for n, rows in ((4, np.ones(4, np.int64)), (300, np.r_[np.zeros(296, np.int64), np.ones(4, np.int64)])):
        check(codec, {"text": column(strs, (4,))}, {"text": rows},
              {"none": column([], empty), "none2": column([], (0,)), "tag": column(tag, (3,))},
              strings={"text": (strs, (4,)), "none": ([], empty), "none2": ([], (0,)), "tag": (tag, (3,))})


def test_offsets_no_box_reads_are_ignored_on_both_routes(codec):
    """Device offsets that are wrong only where no box reads them: the device route and the host route (9 inputs) agree."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(12)
    strs = rand_strings(rng, 18, 0, 9)
    col = column(strs, (6, 3))
    o = col.offsets.copy()
    o[15] = -5                                  # rows 4 and 5 belong to no request
    dev = BytesColumn(torch.from_numpy(col.data).cuda(), torch.from_numpy(o).cuda(), (6, 3))
    S = np.array([[2, 2], [2, 3]], np.int64)
    ref = R.reference_requests("model", 5, {"s": (strs, (6, 3))}, {"s": S}, {})
    assert codec.encode_predict_requests_padded("model", {"s": dev}, {"s": S}, model_version=5) == ref
    padded = {f"k{i}": np.arange(6, dtype=np.float32) * i for i in range(8)}
    calls = codec.padded_encode_device_calls
    got = codec.encode_predict_requests_padded("model", {**padded, "s": dev}, {**{k: S[:, 0] for k in padded}, "s": S}, model_version=5)
    assert codec.padded_encode_device_calls == calls
    assert got == R.reference_requests("model", 5, {**padded, "s": (strs, (6, 3))}, {**{k: S[:, 0] for k in padded}, "s": S}, {})
    o[4] = o[3] - 1                             # now inside request 0's box: both routes refuse
    bad = BytesColumn(dev.data, torch.from_numpy(o).cuda(), (6, 3))
    with pytest.raises(ValueError):
        codec.encode_predict_requests_padded("model", {"s": bad}, {"s": S})
    with pytest.raises(ValueError):
        codec.encode_predict_requests_padded("model", {**padded, "s": bad}, {**{k: S[:, 0] for k in padded}, "s": S})
