"""Ragged (variable-length) tf.Example columns encoded on the GPU: every case compares bytes with ragged_ref, the request built
one example at a time by the unchanged examples_from_input_dict."""
import ctypes as C

import numpy as np
import pytest

from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import RaggedColumn, _example_columns
from ragged_ref import ragged_ref

pytestmark = pytest.mark.gpu

ALL = [np.float16, np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.bool_]


def _values(rng, dt, shape):
    if np.dtype(dt).kind == "f":
        return rng.standard_normal(shape).astype(dt)
    if dt is np.bool_:
        return rng.integers(0, 2, shape).astype(np.bool_)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, shape, dtype=dt, endpoint=True)


def _lengths(rng, n, L):
    x = rng.integers(0, L + 1, n)
    x[: min(n, 2)] = [0, L][: min(n, 2)]
    return x


def _check(codec, d, name="m", version=1, **kw):
    got = codec.encode_example_requests([(name, version, d)], **kw)[0]
    assert got == ragged_ref(name, version, d, grpc_frame=kw.get("grpc_frame", False))
    return got


@pytest.mark.parametrize("dt", ALL, ids=lambda t: np.dtype(t).name)
def test_every_dtype(codec, dt):
    rng = np.random.default_rng(1)
    _check(codec, {"v": RaggedColumn(_values(rng, dt, (60, 9)), _lengths(rng, 60, 9)),
                   "w": RaggedColumn(_values(rng, dt, (60, 5, 3)), _lengths(rng, 60, 5).astype(np.int32)),      # unit 3
                   "z": RaggedColumn(_values(rng, dt, (60, 4, 0)), _lengths(rng, 60, 4))})                    # unit 0


def test_quirks_match_dense_rows(codec):
    rng = np.random.default_rng(3)
    f32 = np.array([np.nan, -0.0, np.inf], np.float32)
    f32 = np.concatenate([f32, np.array([0x7F800001, 0xFF800002], np.uint32).view(np.float32)])          # signalling NaNs
    f64 = np.array([0x7FF0000020000001, 0x3690000000000001, 0x47EFFFFFF0000000, 0], np.uint64).view(np.float64)
    u64 = np.array([0, (1 << 64) - 1, 1 << 63, 127], np.uint64)
    b = np.frombuffer(bytes([0, 2, 255, 1]), np.bool_)
    with np.errstate(all="ignore"):
        for col in (f32, f64, u64, b):
            v = np.tile(col, (7, 1))
            _check(codec, {"q": RaggedColumn(v, _lengths(rng, 7, v.shape[1])), "d": v})


def test_mixed_with_dense_and_zero_d(codec):
    rng = np.random.default_rng(5)
    n = 500
    d = {"hist": RaggedColumn(rng.integers(0, 50_000, (n, 64)), _lengths(rng, n, 64)),
         "emb": RaggedColumn(rng.standard_normal((n, 16, 4)).astype(np.float32), _lengths(rng, n, 16)),
         "dense": rng.standard_normal((n, 8)).astype(np.float32), "ids": rng.integers(-9, 9, (n, 2)), "bias": np.float64(0.25),
         "été": RaggedColumn(rng.integers(0, 2, (n, 3)).astype(np.bool_), _lengths(rng, n, 3))}
    _check(codec, d)
    _check(codec, d, version=None, grpc_frame=True)
    _check(codec, {"one": RaggedColumn(np.ones((1, 3), np.float16), [2])})
    _check(codec, {"none": RaggedColumn(np.ones((0, 3), np.int8), np.zeros(0, np.int64)), "x": np.zeros((0, 2), np.float32)})


def test_float_only_100k_examples(codec):
    rng = np.random.default_rng(7)
    n = 100_000
    _check(codec, {"emb": RaggedColumn(rng.standard_normal((n, 12)).astype(np.float32), rng.integers(1, 13, n))})


def test_example_larger_than_the_emit_image(codec):
    rng = np.random.default_rng(9)
    n, L = 40, 5000
    v = rng.integers(-(1 << 62), -1, (n, L))                    # negative: ten bytes per varint, 50 000 bytes at full length
    lengths = rng.integers(0, 3, n)
    lengths[[5, 6, 20]] = [L, L - 1, L]
    _check(codec, {"big": RaggedColumn(v, lengths), "x": rng.standard_normal((n, 2)).astype(np.float32)})


def test_forty_requests_in_one_call(codec):
    rng = np.random.default_rng(11)
    items = []
    for i in range(40):
        n = int(rng.integers(0, 200))
        d = {"dense": rng.standard_normal((n, i % 4)).astype(np.float32)}
        if i % 2:
            d["r"] = RaggedColumn(rng.integers(-1000, 1 << 33, (n, 1 + i % 9)), _lengths(rng, n, 1 + i % 9))
        if i % 3 == 0:
            d["f"] = RaggedColumn(rng.standard_normal((n, 6, 2)).astype(np.float64), _lengths(rng, n, 6))
        if i % 7 == 3:
            d["s"] = RaggedColumn(np.array([["a", "bb", "ccc"]] * n).reshape(n, 3), _lengths(rng, n, 3))     # the host route
        items.append((f"model{i}", i if i % 4 else None, d))
    for grpc_frame in (False, True):
        got = codec.encode_example_requests(items, grpc_frame=grpc_frame)
        assert got == [ragged_ref(*it, grpc_frame=grpc_frame) for it in items]
    from tensorflow_serving.apis.classification_pb2 import ClassificationRequest as CR

    d = {"zz": RaggedColumn(np.arange(12, dtype=np.float32).reshape(3, 4), [1, 0, 4]), "a": np.arange(3)}
    got = codec.encode_example_requests([("m", 2, d)], order="given")[0]
    det = ragged_ref("m", 2, d)
    assert got != det and CR.FromString(got) == CR.FromString(det)
    assert got.find(b"zz") < got.find(b"\x01a")


def test_torch_values_and_lengths(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(13)
    v = rng.integers(-5, 1 << 40, (64, 10))
    x = rng.standard_normal((64, 6, 2)).astype(np.float32)
    lv, lx = _lengths(rng, 64, 10), _lengths(rng, 64, 6)
    d = {"v": RaggedColumn(torch.from_numpy(v).cuda(), torch.from_numpy(lv).cuda()), "x": RaggedColumn(torch.from_numpy(x).cuda(), lx)}
    assert codec.encode_example_requests([("m", 1, d)])[0] == ragged_ref("m", 1, {"v": RaggedColumn(v, lv), "x": RaggedColumn(x, lx)})
    # slices that start off their 16-byte grid, values and lengths alike
    bigv = torch.from_numpy(np.concatenate([v.ravel(), v.ravel()])).cuda()[3: 3 + 63 * 10].reshape(63, 10)
    bigl = torch.from_numpy(np.concatenate([lv, lv])).cuda()[1: 64]
    ref = {"v": RaggedColumn(bigv.cpu().numpy(), bigl.cpu().numpy())}
    assert codec.encode_example_requests([("m", None, {"v": RaggedColumn(bigv, bigl)})])[0] == ragged_ref("m", None, ref)
    with pytest.raises(ValueError):
        RaggedColumn(torch.from_numpy(v).cuda(), torch.from_numpy(lv.astype(np.int32)).cuda())
    bad = torch.from_numpy(lv).cuda().clone()
    bad[9] = 11
    with pytest.raises(ValueError):
        codec.encode_example_requests([("m", 1, {"v": RaggedColumn(torch.from_numpy(v).cuda(), bad)})])
    assert codec.encode_example_requests([("m", 1, d)])[0] == ragged_ref("m", 1, {"v": RaggedColumn(v, lv), "x": RaggedColumn(x, lx)})


def test_pinned_inputs(codec):
    rng = np.random.default_rng(15)
    v = codec.pinned_empty((300, 7), np.float32)
    v[:] = rng.standard_normal((300, 7))
    lengths = codec.pinned_empty((300,), np.int64)
    lengths[:] = _lengths(rng, 300, 7)
    _check(codec, {"v": RaggedColumn(v, lengths), "n": np.arange(300, dtype=np.uint16)})


def _raw(dev, items):
    """ExampleRequests with device columns: items = [(n, [(key, array, lengths or None, device lengths ptr or None)])]"""
    keep, structs, rg = [], [], []
    for n, cols in items:
        feats = []
        for key, a, lengths, lptr in cols:
            p = dev.upload(a)
            dt = {np.dtype(np.float32): 1, np.dtype(np.int64): 9}[a.dtype]
            row = int(np.prod(a.shape[1:]))
            feats.append(N.Feature(data=p, src_dtype=dt, flags=0, row_elems=row, key=key, key_len=len(key)))
            rg.append(N.Ragged(lengths=lptr, max_len=a.shape[1], unit=row // a.shape[1], flags=N.F_DEVICE_DATA) if lptr else N.Ragged())
        fa = (N.Feature * len(feats))(*feats)
        keep.append(fa)
        structs.append(N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_examples=n,
                                        n_features=len(feats), flags=0, features=fa))
    return (N.ExampleRequest * len(structs))(*structs), (N.Ragged * len(rg))(*rg), keep


def test_graph_replay_with_new_values_and_lengths():
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(17)
        n, L = 3000, 48
        ids, emb = rng.integers(0, 1000, (n, L)), rng.standard_normal((n, 8, 2)).astype(np.float32)
        li, le = _lengths(rng, n, L), _lengths(rng, n, 8)
        dli, dle = dev.upload(li), dev.upload(le)
        reqs, rg, keep = _raw(dev, [(n, [(b"ids", ids, li, dli), (b"emb", emb, le, dle)])])
        dids, demb = keep[0][0].data, keep[0][1].data
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_arena_size(1, reqs, C.byref(cap)))
        arena = (dev.malloc(cap.value + 256) + 255) & ~255
        N.check(lib.b200tfs_encode_example_requests_ragged_async(dev.ctx, 1, reqs, rg, arena, cap.value))   # sizes every buffer
        N.check(lib.b200tfs_encode_results(dev.ctx, 1, None, None))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_encode_example_requests_ragged_async(dev.ctx, 1, reqs, rg, arena, cap.value))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        for rep in range(4):
            ids = rng.integers(-(1 << (20 * rep)), 1 << min(20 * rep + 5, 62), (n, L))
            emb = rng.standard_normal((n, 8, 2)).astype(np.float32)
            li, le = rng.integers(0, L + 1, n) // (rep + 1), rng.integers(0, 9, n)
            if rep == 2:
                li[:] = L
            for ptr, a in ((dids, ids), (demb, emb), (dli, li), (dle, le)):
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, ptr, a.ctypes.data, a.nbytes))
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            if rep == 3:        # a length out of range in a replay: E_SHAPE, and the next replay is clean again
                bad = np.array([L + 1], np.int64)
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, dli + 8 * 17, bad.ctypes.data, 8))
                N.check(lib.b200tfs_graph_launch(dev.ctx, g))
                assert lib.b200tfs_encode_results(dev.ctx, 1, off, ln) == N.E_SHAPE
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, dli + 8 * 17, li[17:18].ctypes.data, 8))
                N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_encode_results(dev.ctx, 1, off, ln))
            wire = dev.download(arena + off[0], ln[0]).tobytes()
            assert wire == ragged_ref("m", 3, {"ids": RaggedColumn(ids, li), "emb": RaggedColumn(emb, le)}), rep
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


@pytest.mark.parametrize("bad_len", [-1, "L+1", 1 << 62])
def test_out_of_range_device_lengths(codec, bad_len):
    """The bad request sits in front of good ones, its padded column inside a larger allocation and the arena has slack behind
    it: a missing check shows as a wrong status or wrong bytes."""
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(19)
        n, L = 300, 20
        items, dicts = [], []
        for r in range(4):
            ids = rng.integers(-(1 << 40), 1 << 40, (n, L))
            x = rng.standard_normal((n, L)).astype(np.float32)
            li, lx = _lengths(rng, n, L), _lengths(rng, n, L)
            dicts.append({"ids": RaggedColumn(ids, li), "x": RaggedColumn(x, lx)})
            host = np.concatenate([ids, ids])                  # the padded column is the first half of a larger allocation
            items.append((n, [(b"ids", host, li, None), (b"x", x, lx, None)]))
        lens = []
        for r, (n_, cols) in enumerate(items):
            li = cols[0][2].copy()
            if r == 0:
                li[n // 2] = L + 1 if bad_len == "L+1" else bad_len
            lens.append((dev.upload(li), dev.upload(cols[1][2])))
        items = [(n_, [(k, a, l, lens[r][j]) for j, (k, a, l, _) in enumerate(cols)]) for r, (n_, cols) in enumerate(items)]
        reqs, rg, keep = _raw(dev, items)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_arena_size(4, reqs, C.byref(cap)))
        slack = 1 << 20
        arena = (dev.malloc(cap.value + slack + 256) + 255) & ~255
        zeros = np.zeros(cap.value + slack, np.uint8)
        N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena, zeros.ctypes.data, zeros.nbytes))
        N.check(lib.b200tfs_encode_example_requests_ragged_async(dev.ctx, 4, reqs, rg, arena, cap.value))
        off, ln = (C.c_uint64 * 4)(), (C.c_uint64 * 4)()
        assert lib.b200tfs_encode_results(dev.ctx, 4, off, ln) == N.E_SHAPE
        assert off[0] == 0 and ln[0] == 0
        for r in range(1, 4):
            assert dev.download(arena + off[r], ln[r]).tobytes() == ragged_ref("m", 3, dicts[r]), r
        tail = dev.download(arena + cap.value, slack)
        assert not tail.any()
        bad = dict(dicts[0])
        li = bad["ids"].lengths.copy()
        li[n // 2] = L + 1 if bad_len == "L+1" else bad_len
        torch = pytest.importorskip("torch")
        with pytest.raises(ValueError):
            codec.encode_example_requests([("m", 1, dicts[1]), ("m", 1, {"ids": RaggedColumn(bad["ids"].values, torch.from_numpy(li).cuda()),
                                                                       "x": bad["x"]})])
        assert codec.encode_example_requests([("m", 3, dicts[2])])[0] == ragged_ref("m", 3, dicts[2])
    finally:
        dev.close()


def test_classify_and_regress_end_to_end():
    import grpc
    from fake_server import IdentityServer
    from min_tfs_client.requests import CLASSIFY_METHOD, REGRESS_METHOD, TensorServingClient, gpu_example_request_serializer
    from tensorflow_serving.apis.classification_pb2 import ClassificationResponse
    from tensorflow_serving.apis.regression_pb2 import RegressionResponse

    srv = IdentityServer()
    try:
        client = TensorServingClient("127.0.0.1", srv.port)
        rng = np.random.default_rng(21)
        d = {"hist": RaggedColumn(rng.integers(0, 500, (20, 16)), _lengths(rng, 20, 16)), "x": rng.standard_normal((20, 3)).astype(np.float32),
             "bias": np.float64(0.5)}
        ch = grpc.insecure_channel(f"127.0.0.1:{srv.port}")
        cls = ch.unary_unary(CLASSIFY_METHOD, request_serializer=gpu_example_request_serializer,
                             response_deserializer=ClassificationResponse.FromString)(("m", 4, d), timeout=30)
        reg = ch.unary_unary(REGRESS_METHOD, request_serializer=gpu_example_request_serializer,
                             response_deserializer=RegressionResponse.FromString)(("m", 4, d), timeout=30)
        assert cls == client.classification_request("m", d, model_version=4)
        assert reg == client.regression_request("m", d, model_version=4)
        assert srv.received[0] == ragged_ref("m", 4, d) and len(cls.result.classifications) == 20
        ch.close()
    finally:
        srv.stop()


def test_example_columns_with_device_lengths():
    torch = pytest.importorskip("torch")
    lengths = torch.tensor([0, 3, 1], dtype=torch.int64, device="cuda")
    n, preps = _example_columns({"r": RaggedColumn(np.zeros((3, 3), np.int32), lengths)})
    g = preps[0][3]
    assert g.lengths == lengths.data_ptr() and g.flags == N.F_DEVICE_DATA and g.max_len == 3 and g.unit == 1
