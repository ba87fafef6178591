"""tf.Example requests (Classify / Regress) encoded on the GPU: every case compares bytes against
``_make_example_request(...).SerializeToString(deterministic=True)``, the request examples_from_input_dict builds."""
import ctypes as C

import numpy as np
import pytest

import cast_sweep as CS
from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import _example_columns
from min_tfs_client.requests import TensorServingClient
from tensorflow_serving.apis.classification_pb2 import ClassificationRequest

pytestmark = pytest.mark.gpu


def _ref(name, version, d):
    return TensorServingClient._make_example_request(None, ClassificationRequest, name, d, version).SerializeToString(deterministic=True)


def _check(codec, d, name="m", version=1, **kw):
    got = codec.encode_example_requests([(name, version, d)], **kw)[0]
    assert got == _ref(name, version, d)
    return got


ALL = [np.float16, np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.bool_]


@pytest.mark.parametrize("dt", ALL, ids=lambda t: np.dtype(t).name)
def test_every_dtype(codec, dt):
    rng = np.random.default_rng(1)
    if np.dtype(dt).kind == "f":
        x = rng.standard_normal((50, 3)).astype(dt)
    elif dt is np.bool_:
        x = rng.integers(0, 2, (50, 3)).astype(np.bool_)
    else:
        info = np.iinfo(dt)
        x = rng.integers(info.min, info.max, (50, 3), dtype=dt, endpoint=True)
    _check(codec, {"v": x, "w": x[:, 0].copy(), "s": x[0, 0]})


def test_float_sweeps(codec):
    f32 = CS.f32_patterns()
    pad = (-len(f32)) % 1024
    x = np.concatenate([f32, np.zeros(pad, np.uint32)]).view(np.float32).reshape(-1, 1024)
    _check(codec, {"f": x})
    _check(codec, {"h": CS.all_f16().reshape(-1, 256)})


def test_f64_sweep(codec):
    rng = np.random.default_rng(5)
    vals = []
    for e in range(1, 2047):        # every exponent: ties and their neighbours at float32's rounding cut (29 dropped bits)
        for m in (0x10000000, 0x10000001, 0x0FFFFFFF, 0x30000000, 0x20000000, 0xFFFFFFFFFFFFF, 0):
            vals.append((e << 52) | m)
        vals += [(e << 52) | int(v) for v in rng.integers(0, 1 << 52, 4, dtype=np.uint64)]
    # overflow to +-inf, float32 subnormal results, infinities, NaNs with payloads (signalling and quiet)
    vals += [0x47EFFFFFE0000000, 0x47EFFFFFF0000000, 0x47F0000000000000, 0x36A0000000000000, 0x3690000000000000, 0x3690000000000001,
             0x380FFFFFFFFFFFFF, 0x3800000000000000, 0x7FF0000000000000, 0x7FF0000000000001, 0x7FF4000020000000, 0x7FF8000000000000,
             0x7FFFFFFFFFFFFFFF, 0x7FF0000020000000, 0x7FF000001FFFFFFF, 0]
    vals += [(0x7FF << 52) | int(v) for v in rng.integers(1, 1 << 52, 300, dtype=np.uint64)]
    bits = np.array(vals, dtype=np.uint64)
    bits = np.concatenate([bits, bits | np.uint64(1 << 63)])
    bits = np.concatenate([bits, np.zeros((-len(bits)) % 64, np.uint64)])
    with np.errstate(all="ignore"):
        _check(codec, {"d": bits.view(np.float64).reshape(-1, 64)})


def test_integer_extremes_and_varint_lengths(codec):
    lengths = np.array([(1 << (7 * k)) - 1 for k in range(1, 10)] + [1 << 63 - 1, -1, -(1 << 63), (1 << 63) - 1, 0], dtype=np.int64)
    _check(codec, {"i": lengths.reshape(1, -1), "j": lengths[::-1].reshape(1, -1)})
    u = np.array([0, 1, 1 << 63, (1 << 63) + 5, (1 << 64) - 1, 127, 128], dtype=np.uint64)
    _check(codec, {"u": u.reshape(-1, 1)})
    b = np.frombuffer(bytes([2, 0, 1, 255, 0, 7]), dtype=np.bool_).reshape(3, 2)
    _check(codec, {"b": b})


def test_shapes(codec):
    rng = np.random.default_rng(7)
    _check(codec, {})
    _check(codec, {"a": np.float32(3.0), "b": np.int64(-4)})                         # all 0-d: one example
    _check(codec, {"a": np.zeros((0, 4), np.float32), "b": np.zeros((0,), np.int64)})    # n = 0
    _check(codec, {"a": np.zeros((5, 0), np.float32), "b": np.zeros((5, 0), np.int32), "c": np.ones(5, np.int8)})   # zero-width rows
    _check(codec, {"a": rng.standard_normal((1, 3, 2)).astype(np.float32)}, name="", version=None)
    for w in (1, 33, 5000):
        _check(codec, {"ids": rng.integers(-1 << 40, 1 << 40, (7, w)), "x": rng.standard_normal((7, 2)).astype(np.float32),
                       "k": np.float64(1.5)}, version=0)
    n = 100_000
    _check(codec, {"dense": rng.standard_normal((n, 16)).astype(np.float32), "ids": rng.integers(0, 50_000, (n, 8)),
                   "age": rng.standard_normal(n).astype(np.float32)})
    _check(codec, {"dense": rng.standard_normal((n, 5)).astype(np.float32)}, version=7)


def test_several_requests_in_one_call(codec):
    rng = np.random.default_rng(9)
    items = []
    for i in range(40):
        n = int(rng.integers(0, 300))
        d = {"dense": rng.standard_normal((n, i % 5)).astype(np.float32)}
        if i % 2:
            d["ids"] = rng.integers(-1000, 1 << 33, (n, i % 7))
        if i % 3 == 0:
            d[f"k{i}"] = np.int16(i)
        items.append((f"model{i}", i if i % 4 else None, d))
    items.append(("s", None, {"s": np.array(["x", "yy"]), "v": np.arange(2)}))          # a string column: the host assembles it
    got = codec.encode_example_requests(items)
    assert got == [_ref(*it) for it in items]
    framed = codec.encode_example_requests(items, grpc_frame=True)
    assert framed == [b"\x00" + len(w).to_bytes(4, "big") + w for w in got]


def test_given_order(codec):
    from tensorflow_serving.apis.classification_pb2 import ClassificationRequest as CR

    d = {"zz": np.arange(6, dtype=np.float32).reshape(3, 2), "a": np.arange(3), "ab": np.ones(3, np.float64)}
    got = codec.encode_example_requests([("m", 2, d)], order="given")[0]
    det = _ref("m", 2, d)
    assert got != det and CR.FromString(got) == CR.FromString(det)
    pos = [got.find(k.encode()) for k in d]
    assert pos == sorted(pos)


def test_device_inputs(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(11)
    x = rng.standard_normal((64, 8)).astype(np.float32)
    ids = rng.integers(-5, 1 << 40, (64, 3))
    h = rng.standard_normal((64,)).astype(np.float16)
    d = {"x": torch.from_numpy(x).cuda(), "ids": torch.from_numpy(ids).cuda(), "h": torch.from_numpy(h).cuda()}
    assert codec.encode_example_requests([("m", 1, d)])[0] == _ref("m", 1, {"x": x, "ids": ids, "h": h})
    big = codec.device_array(np.concatenate([ids.ravel(), ids.ravel()]))
    xs = codec.device_array(x.ravel())
    # slices of DeviceArrays that start off their 16-byte (and, for ids, 8-element) grid, viewed through torch
    sl = {"ids": torch.as_tensor(big, device="cuda")[3: 3 + 63 * 3].reshape(63, 3),
          "x": torch.as_tensor(xs, device="cuda")[1: 1 + 63 * 8].reshape(63, 8)}
    ref = {"ids": np.concatenate([ids.ravel(), ids.ravel()])[3: 3 + 63 * 3].reshape(63, 3), "x": x.ravel()[1: 1 + 63 * 8].reshape(63, 8)}
    assert codec.encode_example_requests([("m", None, sl)])[0] == _ref("m", None, ref)
    with pytest.raises(ValueError):
        codec.encode_example_requests([("m", 1, {"c": torch.zeros(3, 2, dtype=torch.complex64, device="cuda")})])


def test_pinned_inputs(codec):
    x = codec.pinned_empty((300, 7), np.float32)
    x[:] = np.random.default_rng(2).standard_normal((300, 7))
    _check(codec, {"x": x, "n": np.arange(300, dtype=np.uint16)})


def test_value_errors_match(codec):
    from min_tfs_client.requests import examples_from_input_dict

    for bad in ({"a": np.zeros((2, 3), np.float32), "b": np.zeros(3, np.int64)}, {"c": np.zeros((2,), np.complex64)}):
        with pytest.raises(ValueError) as ref:
            examples_from_input_dict(bad)
        with pytest.raises(ValueError) as ours:
            codec.encode_example_requests([("m", 1, bad)])
        assert str(ours.value) == str(ref.value)


def test_graph_replay_with_new_lengths():
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(13)
        n = 2000
        x = rng.standard_normal((n, 4)).astype(np.float32)
        ids = rng.integers(0, 100, (n, 5))
        dx, dids = dev.upload(x), dev.upload(ids)
        keep = []
        feats = (N.Feature * 2)(N.Feature(data=dx, src_dtype=1, flags=0, row_elems=4, key=b"x", key_len=1),
                                N.Feature(data=dids, src_dtype=9, flags=0, row_elems=5, key=b"ids", key_len=3))
        req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_examples=n,
                               n_features=2, flags=0, features=feats)
        keep.append(feats)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_arena_size(1, C.byref(req), C.byref(cap)))
        arena = dev.malloc(cap.value + 256)
        arena = (arena + 255) & ~255
        N.check(lib.b200tfs_encode_example_requests_async(dev.ctx, 1, C.byref(req), arena, cap.value))   # sizes every buffer
        N.check(lib.b200tfs_encode_results(dev.ctx, 1, None, None))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_encode_example_requests_async(dev.ctx, 1, C.byref(req), arena, cap.value))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        for rep in range(3):
            x = rng.standard_normal((n, 4)).astype(np.float32)
            ids = rng.integers(-(1 << (20 * rep)), 1 << (20 * rep + 5), (n, 5))      # other lengths, other offsets
            N.check(lib.b200tfs_memcpy_h2d(dev.ctx, dx, x.ctypes.data, x.nbytes))
            N.check(lib.b200tfs_memcpy_h2d(dev.ctx, dids, ids.ctypes.data, ids.nbytes))
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_encode_results(dev.ctx, 1, off, ln))
            wire = dev.download(arena + off[0], ln[0]).tobytes()
            assert wire == _ref("m", 3, {"x": x, "ids": ids}), rep
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


def test_classify_and_regress_end_to_end():
    import grpc
    from fake_server import IdentityServer
    from min_tfs_client.requests import CLASSIFY_METHOD, REGRESS_METHOD, gpu_example_request_serializer
    from tensorflow_serving.apis.classification_pb2 import ClassificationResponse
    from tensorflow_serving.apis.regression_pb2 import RegressionResponse

    srv = IdentityServer()
    try:
        client = TensorServingClient("127.0.0.1", srv.port)
        rng = np.random.default_rng(17)
        d = {"x": rng.standard_normal((20, 3)).astype(np.float32), "id": np.arange(20), "bias": np.float64(0.5)}
        ch = grpc.insecure_channel(f"127.0.0.1:{srv.port}")
        cls = ch.unary_unary(CLASSIFY_METHOD, request_serializer=gpu_example_request_serializer,
                             response_deserializer=ClassificationResponse.FromString)(("m", 4, d), timeout=30)
        reg = ch.unary_unary(REGRESS_METHOD, request_serializer=gpu_example_request_serializer,
                             response_deserializer=RegressionResponse.FromString)(("m", 4, d), timeout=30)
        assert cls == client.classification_request("m", d, model_version=4)
        assert reg == client.regression_request("m", d, model_version=4)
        assert srv.received[0] == _ref("m", 4, d) and len(cls.result.classifications) == 20
        ch.close()
    finally:
        srv.stop()
