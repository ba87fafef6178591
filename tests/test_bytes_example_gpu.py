"""String (bytes_list) tf.Example columns encoded on the GPU: every case compares bytes with the protobuf runtime's serialization
of the request examples_from_input_dict builds from host copies of the same columns (and, where numpy can hold the strings, from
the equivalent numpy str / bytes arrays)."""
import ctypes as C

import numpy as np
import pytest

from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn, _example_columns
from min_tfs_client.requests import TensorServingClient, examples_from_input_dict
from tensorflow.core.framework import types_pb2
from tensorflow_serving.apis.classification_pb2 import ClassificationRequest
from tensorflow_serving.apis.predict_pb2 import PredictRequest

pytestmark = pytest.mark.gpu


def _host(v):
    if isinstance(v, RaggedColumn):
        return RaggedColumn(_host(v.values), _host(v.lengths))
    if isinstance(v, BytesColumn):
        return BytesColumn(_host(v.data), _host(v.offsets), v.shape)
    return v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)


def _frame(wire, grpc_frame):
    return (b"\x00" + len(wire).to_bytes(4, "big") + wire) if grpc_frame else wire


def ref(name, version, d, grpc_frame=False):
    h = {k: _host(v) for k, v in d.items()}
    req = TensorServingClient._make_example_request(None, ClassificationRequest, name, h, version)
    return _frame(req.SerializeToString(deterministic=True), grpc_frame)


def pref(name, version, d, key="examples", grpc_frame=False):
    req = PredictRequest()
    req.model_spec.name = name
    if version is not None:
        req.model_spec.version.value = version
    ex = examples_from_input_dict({k: _host(v) for k, v in d.items()}).example_list.examples
    t = req.inputs[key]
    t.dtype = types_pb2.DT_STRING
    t.tensor_shape.dim.add().size = len(ex)
    t.string_val.extend(e.SerializeToString(deterministic=True) for e in ex)
    return _frame(req.SerializeToString(deterministic=True), grpc_frame)


def _strings(rng, m, lo=0, hi=12):
    alphabet = np.frombuffer(bytes(range(256)), np.uint8)
    return [rng.choice(alphabet, int(rng.integers(lo, hi + 1))).tobytes() for _ in range(m)]


def _column(strs, shape=None, start=0, tail=3):
    """a BytesColumn of these strings, `start` bytes into its buffer (offsets[0] == start), `tail` bytes of slack behind"""
    lens = np.array([len(s) for s in strs], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64) + start
    data = np.frombuffer(b"\xEE" * start + b"".join(strs) + b"\xEE" * tail, np.uint8).copy()
    return BytesColumn(data, offsets, shape)


def _lengths(rng, n, L):
    x = rng.integers(0, L + 1, n)
    x[: min(n, 2)] = [0, L][: min(n, 2)]
    return x


def _check(codec, d, name="m", version=1, **kw):
    got = codec.encode_example_requests([(name, version, d)], **kw)[0]
    if kw.get("predict_input") is None:
        assert got == ref(name, version, d, grpc_frame=kw.get("grpc_frame", False))
    else:
        assert got == pref(name, version, d, kw["predict_input"], grpc_frame=kw.get("grpc_frame", False))
    return got


def test_edge_strings(codec):
    rng = np.random.default_rng(1)
    n = 50
    edge = [b"", b"\x00", b"a\x00", b"\x00b", b"\xff\xfe\x80", bytes(range(256)), b"x" * 127, b"y" * 128]
    strs = [edge[i % len(edge)] for i in range(n * 3)]
    d = {"s": _column(strs, (n, 3), start=5), "empty": _column([], (n, 0)), "one": _column([b"\x00\xff"], ()),
         "blank": _column([b""], ()), "col": _column([b""] * n)}
    for grpc_frame in (False, True):
        _check(codec, d, grpc_frame=grpc_frame)
        _check(codec, d, version=None, grpc_frame=grpc_frame)
    got = codec.encode_example_requests([("m", 1, d)], order="given")[0]
    assert ClassificationRequest.FromString(got) == ClassificationRequest.FromString(ref("m", 1, d))
    assert got.find(b"\x01s") < got.find(b"\x05empty")
    # a row of no strings still writes its empty list; an empty string is 0A 00 inside it
    assert b"\x0a\x05empty\x12\x02\x0a\x00" in got and b"\x0a\x05blank\x12\x04\x0a\x02\x0a\x00" in got


def test_equivalent_numpy_strings(codec):
    rng = np.random.default_rng(2)
    n = 300
    words = np.array(["", "us", "de", "été", "中文", "a\x00b", "longer text " * 5])
    u = rng.choice(words, (n, 4))
    s = np.array([b"", b"\x01\xff", b"q\x00r", b"zz" * 30])[rng.integers(0, 4, n)]
    d_np = {"u": u, "s": s, "c": np.array("country"), "f": rng.standard_normal((n, 2)).astype(np.float32), "i": rng.integers(-9, 9, n)}
    d = {k: BytesColumn.from_array(v) if v.dtype.kind in "US" else v for k, v in d_np.items()}
    wire = TensorServingClient._make_example_request(None, ClassificationRequest, "m", d_np, 1).SerializeToString(deterministic=True)
    assert codec.encode_example_requests([("m", 1, d)])[0] == wire
    assert codec.encode_example_requests([("m", 1, d_np)])[0] == wire          # the numpy route is unchanged (host)


def test_ragged_and_mixed_columns(codec):
    rng = np.random.default_rng(3)
    n, L = 400, 6
    tags = _column(_strings(rng, n * L * 2, 0, 20), (n, L, 2), start=11)
    d = {"tags": RaggedColumn(tags, _lengths(rng, n, L)), "country": _column(_strings(rng, n, 2, 2)),
         "dense": rng.standard_normal((n, 16)).astype(np.float32), "bias": np.float64(0.5), "ids": rng.integers(-(1 << 40), 1 << 40, (n, 3)),
         "hist": RaggedColumn(rng.integers(0, 1000, (n, 9)), _lengths(rng, n, 9)), "z": _column([b"zero-d"], ())}
    _check(codec, d)
    _check(codec, d, version=None, grpc_frame=True)
    _check(codec, d, predict_input="examples")
    _check(codec, d, predict_input=b"in", grpc_frame=True)
    _check(codec, {"one": RaggedColumn(_column([b"a", b"b"], (1, 2)), [1])})
    _check(codec, {"none": RaggedColumn(_column([], (0, 3)), np.zeros(0, np.int64)), "x": np.zeros((0, 2), np.float32)})


def test_ragged_with_device_lengths(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(4)
    n, L = 200, 5
    col = _column(_strings(rng, n * L, 0, 30), (n, L))
    lengths = _lengths(rng, n, L)
    got = codec.encode_example_requests([("m", 1, {"r": RaggedColumn(col, torch.from_numpy(lengths).cuda())})])[0]
    assert got == ref("m", 1, {"r": RaggedColumn(col, lengths)})


def test_examples_larger_than_the_emit_image(codec):
    rng = np.random.default_rng(5)
    n = 12
    strs = [b"s" * 3] * n
    strs[4] = bytes(rng.integers(0, 256, 40_000, dtype=np.uint8))                     # a 40 KB string: an example larger than 16 KB
    strs[9] = bytes(rng.integers(0, 256, 17_000, dtype=np.uint8))
    _check(codec, {"big": _column(strs), "x": rng.standard_normal((n, 2)).astype(np.float32)})
    _check(codec, {"big": _column(strs)}, predict_input="examples")
    m = 40                                                                              # ~3 KB strings: some straddle an image window
    mid = _strings(rng, m, 2500, 3500)
    _check(codec, {"mid": _column(mid), "tags": _column(_strings(rng, m * 3, 0, 9), (m, 3))})
    _check(codec, {"b": _column([bytes(rng.integers(0, 256, 60_000, dtype=np.uint8))], ())} | {"x": np.zeros((3, 1), np.int8)})


def test_100k_examples(codec):
    rng = np.random.default_rng(6)
    n = 100_000
    pool = _strings(rng, 97, 0, 14)
    idx = rng.integers(0, 97, n * 2)
    _check(codec, {"t": _column([pool[i] for i in idx], (n, 2)), "c": _column([b"us"], ()), "f": rng.standard_normal((n, 4)).astype(np.float32)})


def _structs(items):
    """ExampleRequests, Ragged, Bytes and targets of [(name, version, d, predict key or None)]"""
    keep, structs, rg, bs, tg = [], [], [], [], []
    for name, version, d, key in items:
        n, preps = _example_columns(d)
        feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
        nb = name.encode()
        keep.append((preps, feats, nb, key))
        structs.append(N.ExampleRequest(model_name=nb, model_name_len=len(nb), has_version=int(version is not None), order=N.ORDER_UPB,
                                        version=version or 0, n_examples=n, n_features=len(preps), flags=0, features=feats))
        rg += [p[3] or N.Ragged() for p in preps]
        bs += [p.bytes_entry or N.Bytes() for p in preps]
        tg.append(N.ExampleTarget(kind=N.EXAMPLES_PREDICT_STRING, key=key, key_len=len(key)) if key else N.ExampleTarget())
    return ((N.ExampleRequest * len(structs))(*structs), (N.Ragged * max(len(rg), 1))(*rg), (N.Bytes * max(len(bs), 1))(*bs),
            (N.ExampleTarget * len(tg))(*tg), keep)


def test_forty_requests_mixing_classify_and_predict(codec):
    rng = np.random.default_rng(7)
    items = []
    for i in range(40):
        n = int(rng.integers(0, 120))
        d = {"dense": rng.standard_normal((n, i % 3)).astype(np.float32)}
        if i % 2:
            d["s"] = _column(_strings(rng, n * (i % 4), 0, 40), (n, i % 4), start=i)
        if i % 3 == 0:
            L = 1 + i % 5
            d["r"] = RaggedColumn(_column(_strings(rng, n * L, 0, 9), (n, L)), _lengths(rng, n, L))
        if i % 5 == 1:
            d["c"] = _column([b"const"], ())
        if i % 7 == 2:
            d["i"] = rng.integers(-5, 1 << 35, (n, 2))
        items.append((f"model{i}", i if i % 4 else None, d, b"examples" if i % 3 == 1 else None))
    reqs, rg, bs, tg, keep = _structs(items)
    lib = codec._lib
    cap = C.c_uint64()
    N.check(lib.b200tfs_example_columns_arena_size(40, reqs, bs, tg, C.byref(cap)))
    wire = np.empty(cap.value, np.uint8)
    off, ln = (C.c_uint64 * 40)(), (C.c_uint64 * 40)()
    N.check(lib.b200tfs_encode_example_columns_host(codec._ctx, 40, reqs, rg, bs, tg, wire.ctypes.data, cap.value, off, ln))
    for j, (name, version, d, key) in enumerate(items):
        want = pref(name, version, d, key.decode()) if key else ref(name, version, d)
        assert wire[off[j]: off[j] + ln[j]].tobytes() == want, j


def test_torch_and_pinned_columns(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(8)
    n = 256
    col = _column(_strings(rng, n * 3, 0, 25), (n, 3), start=7)
    dev = BytesColumn(torch.from_numpy(col.data).cuda(), torch.from_numpy(col.offsets).cuda(), (n, 3))
    d = {"s": dev, "x": torch.from_numpy(rng.standard_normal((n, 2)).astype(np.float32)).cuda()}
    _check(codec, d)
    _check(codec, d, predict_input="examples")
    mixed = {"s": BytesColumn(torch.from_numpy(col.data).cuda(), col.offsets, (n, 3))}     # device data, host offsets
    _check(codec, mixed)
    mixed = {"s": BytesColumn(col.data, torch.from_numpy(col.offsets).cuda(), (n, 3))}     # host data, device offsets
    _check(codec, mixed)
    # DLPack of a slice: offsets that start off their 16-byte grid and at a string other than the first
    big = torch.from_numpy(np.concatenate([[0], col.offsets])).cuda()
    sliced = BytesColumn(torch.from_numpy(col.data).cuda(), torch.utils.dlpack.from_dlpack(torch.utils.dlpack.to_dlpack(big[4:])),
                         (n - 1, 3))
    _check(codec, {"s": sliced})
    with pytest.raises(ValueError, match="int64"):
        BytesColumn(torch.from_numpy(col.data).cuda(), torch.from_numpy(col.offsets.astype(np.int32)).cuda())
    data = codec.pinned_empty((col.data_len,), np.uint8)
    data[:] = col.data
    offsets = codec.pinned_empty((col.offsets.size,), np.int64)
    offsets[:] = col.offsets
    _check(codec, {"s": BytesColumn(data, offsets, (n, 3)), "n": np.arange(n, dtype=np.uint16)})


def _raw(dev, items):
    """device ExampleRequests: items = [(n, [(key, BytesColumn, lengths ptr or None, L)])], data and offsets uploaded"""
    keep, structs, rg, bs = [], [], [], []
    for n, cols in items:
        feats = []
        for key, col, lptr, L in cols:
            dp, op = dev.upload(col.data), dev.upload(col.offsets)
            row = int(np.prod(col.shape[1:]))
            feats.append(N.Feature(data=dp, src_dtype=7, flags=0, row_elems=row, key=key, key_len=len(key)))
            bs.append(N.Bytes(offsets=op, data_len=col.data_len, flags=N.F_DEVICE_DATA))
            rg.append(N.Ragged(lengths=lptr, max_len=L, unit=row // L, flags=N.F_DEVICE_DATA) if lptr else N.Ragged())
        fa = (N.Feature * len(feats))(*feats)
        keep.append(fa)
        structs.append(N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_examples=n,
                                        n_features=len(feats), flags=0, features=fa))
    return (N.ExampleRequest * len(structs))(*structs), (N.Ragged * len(rg))(*rg), (N.Bytes * len(bs))(*bs), keep


def test_graph_replay_with_new_data_offsets_and_lengths():
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(9)
        n, L, cap_bytes = 2000, 4, 200_000
        def make(rep):
            strs = _strings(rng, n * L, 0, 3 + 6 * rep)
            c = _column(strs, (n, L), start=int(rng.integers(0, 50)), tail=0)
            data = np.zeros(cap_bytes, np.uint8)
            data[: c.data_len] = c.data
            return BytesColumn(data, c.offsets, (n, L)), _lengths(rng, n, L) // (1 + rep % 2)
        col, li = make(0)
        dli = dev.upload(li)
        reqs, rg, bs, keep = _raw(dev, [(n, [(b"tags", col, dli, L)])])
        ddata, doff = keep[0][0].data, bs[0].offsets
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_columns_arena_size(1, reqs, bs, None, C.byref(cap)))
        arena = (dev.malloc(cap.value + 256) + 255) & ~255
        N.check(lib.b200tfs_encode_example_columns_async(dev.ctx, 1, reqs, rg, bs, None, arena, cap.value))   # sizes every buffer
        N.check(lib.b200tfs_encode_results(dev.ctx, 1, None, None))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_encode_example_columns_async(dev.ctx, 1, reqs, rg, bs, None, arena, cap.value))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        for rep in range(4):
            col, li = make(rep)
            for ptr, a in ((ddata, col.data), (doff, col.offsets), (dli, li)):
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, ptr, a.ctypes.data, a.nbytes))
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            if rep == 3:        # offsets out of order in a replay: E_SHAPE, and the next replay is clean again
                bad = np.array([-1], np.int64)                  # the end of example 1's first string (it has two)
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, doff + 8 * (L + 1), bad.ctypes.data, 8))
                N.check(lib.b200tfs_graph_launch(dev.ctx, g))
                assert lib.b200tfs_encode_results(dev.ctx, 1, off, ln) == N.E_SHAPE
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, doff, col.offsets.ctypes.data, col.offsets.nbytes))
                N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_encode_results(dev.ctx, 1, off, ln))
            wire = dev.download(arena + off[0], ln[0]).tobytes()
            assert wire == ref("m", 3, {"tags": RaggedColumn(col, li)}), rep
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


@pytest.mark.parametrize("case", ["decreasing", "negative", "past_data_len", "row_start_past_next", "zigzag"])
def test_bad_device_offsets(codec, case):
    """The bad request sits in front of good ones, its buffer inside a larger allocation, and the arena has a zeroed tail: a
    missing check or clamp shows as a wrong status or wrong bytes."""
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(10)
        n, R = 300, 3
        items, dicts = [], []
        for r in range(4):
            col = _column(_strings(rng, n * R, 0, 30), (n, R), start=16, tail=4096)
            dicts.append({"s": col, "x": rng.standard_normal((n, 2)).astype(np.float32)})
        o = dicts[0]["s"].offsets.copy()
        if case == "decreasing":
            o[40] = o[39] - 1
        elif case == "negative":
            o[n * R // 2] = -(1 << 40)
        elif case == "past_data_len":
            o[n * R] = dicts[0]["s"].data_len + 1
        elif case == "row_start_past_next":
            o[R * 10] = o[R * 11] + 5
        else:                                   # every other row starts back at 0: rows overlap, each passes its own order check
            o[R * np.arange(0, n, 2)] = 0
            o[R * np.arange(1, n, 2)] = o[-1] - 1 - 4096
        bad_col = BytesColumn(dicts[0]["s"].data, o, (n, R))
        items = [(n, [(b"s", bad_col, None, 1)])] + [(n, [(b"s", d["s"], None, 1)]) for d in dicts[1:]]
        reqs, rg, bs, keep = _raw(dev, items)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_columns_arena_size(4, reqs, bs, None, C.byref(cap)))
        slack = 1 << 20
        arena = (dev.malloc(cap.value + slack + 256) + 255) & ~255
        zeros = np.zeros(cap.value + slack, np.uint8)
        N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena, zeros.ctypes.data, zeros.nbytes))
        N.check(lib.b200tfs_encode_example_columns_async(dev.ctx, 4, reqs, None, bs, None, arena, cap.value))
        off, ln = (C.c_uint64 * 4)(), (C.c_uint64 * 4)()
        assert lib.b200tfs_encode_results(dev.ctx, 4, off, ln) == N.E_SHAPE
        assert off[0] == 0 and ln[0] == 0
        for r in range(1, 4):
            assert dev.download(arena + off[r], ln[r]).tobytes() == ref("m", 3, {"s": dicts[r]["s"]}), r
        assert not dev.download(arena + cap.value, slack).any()
        torch = pytest.importorskip("torch")
        with pytest.raises(ValueError):
            codec.encode_example_requests([("m", 1, dicts[1]),
                                           ("m", 1, {"s": BytesColumn(bad_col.data, torch.from_numpy(o).cuda(), (n, R)), "x": dicts[0]["x"]})])
        with pytest.raises(ValueError):                      # the same offsets from the host: refused before any launch
            codec.encode_example_requests([("m", 1, {"s": bad_col})])
        _check(codec, dicts[2])
    finally:
        dev.close()


def test_classify_end_to_end():
    import grpc
    from fake_server import IdentityServer
    from min_tfs_client.requests import CLASSIFY_METHOD, gpu_example_request_serializer
    from tensorflow_serving.apis.classification_pb2 import ClassificationResponse

    srv = IdentityServer()
    try:
        client = TensorServingClient("127.0.0.1", srv.port)
        rng = np.random.default_rng(11)
        d = {"q": BytesColumn.from_array(np.array(["hello", "", "wörld"] * 7)), "x": rng.standard_normal((21, 3)).astype(np.float32)}
        ch = grpc.insecure_channel(f"127.0.0.1:{srv.port}")
        cls = ch.unary_unary(CLASSIFY_METHOD, request_serializer=gpu_example_request_serializer,
                             response_deserializer=ClassificationResponse.FromString)(("m", 4, d), timeout=30)
        assert cls == client.classification_request("m", d, model_version=4)
        assert srv.received[0] == ref("m", 4, d) and len(cls.result.classifications) == 21
        ch.close()
    finally:
        srv.stop()
