"""PredictRequests carrying serialized tf.Examples (a DT_STRING [n] input) encoded on the GPU: every case compares bytes with
predict_examples_ref, the request the protobuf runtime builds from the examples examples_from_input_dict makes."""
import ctypes as C

import numpy as np
import pytest

import cast_sweep as CS
from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import RaggedColumn, _example_columns
from predict_examples_ref import examples, predict_examples_ref
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


def _check(codec, d, name="m", version=1, key="examples", **kw):
    got = codec.encode_example_requests([(name, version, d)], predict_input=key, **kw)[0]
    assert got == predict_examples_ref(name, version, d, key, grpc_frame=kw.get("grpc_frame", False))
    return got


@pytest.mark.parametrize("dt", ALL, ids=lambda t: np.dtype(t).name)
def test_every_dtype(codec, dt):
    rng = np.random.default_rng(1)
    x = _values(rng, dt, (50, 3))
    _check(codec, {"v": x, "w": x[:, 0].copy(), "s": x[0, 0]})


def test_float_sweeps(codec):
    f32 = CS.f32_patterns()
    x = np.concatenate([f32, np.zeros((-len(f32)) % 1024, np.uint32)]).view(np.float32).reshape(-1, 1024)
    _check(codec, {"f": x})
    _check(codec, {"h": CS.all_f16().reshape(-1, 256)})
    rng = np.random.default_rng(5)
    bits = np.array([(e << 52) | m for e in range(0, 2048, 3) for m in (0x10000000, 0x10000001, 0x0FFFFFFF, 0xFFFFFFFFFFFFF, 0)]
                    + [int(v) for v in rng.integers(0, 1 << 63, 500, dtype=np.uint64)], dtype=np.uint64)
    bits = np.concatenate([bits, bits | np.uint64(1 << 63)])
    bits = np.concatenate([bits, np.zeros((-len(bits)) % 64, np.uint64)])
    with np.errstate(all="ignore"):
        _check(codec, {"d": bits.view(np.float64).reshape(-1, 64)})


def test_integer_extremes_and_varint_lengths(codec):
    v = np.array([(1 << (7 * k)) - 1 for k in range(1, 10)] + [1 << 62, -1, -(1 << 63), (1 << 63) - 1, 0], dtype=np.int64)
    _check(codec, {"i": v.reshape(1, -1), "j": v[::-1].reshape(1, -1)})
    _check(codec, {"u": np.array([0, 1, 1 << 63, (1 << 63) + 5, (1 << 64) - 1, 127, 128], dtype=np.uint64).reshape(-1, 1)})
    _check(codec, {"b": np.frombuffer(bytes([2, 0, 1, 255, 0, 7]), dtype=np.bool_).reshape(3, 2)})


def test_zero_d_and_zero_examples(codec):
    _check(codec, {"a": np.float32(3.0), "b": np.int64(-4)})                          # all 0-d: one example
    _check(codec, {"a": np.zeros((0, 4), np.float32), "b": np.zeros((0,), np.int64)})   # n = 0: an empty string_val
    _check(codec, {})
    _check(codec, {"a": np.zeros((5, 0), np.float32), "c": np.ones(5, np.int8), "k": np.float64(1.5)}, name="", version=None, key="")


@pytest.mark.parametrize("n", [1, 127, 128, 16383, 16384, 2_097_151, 2_097_152])
def test_example_counts_at_varint_edges(codec, n):
    rng = np.random.default_rng(n)
    d = {"x": rng.standard_normal((n, 1)).astype(np.float32)}
    if n < 20_000:
        d["id"] = rng.integers(-3, 300, n)
        _check(codec, d, key="中文")
        _check(codec, d, version=None, key="k" * 200, grpc_frame=True)
        return
    # millions of examples: the reference is the dense Classify encode of the same columns, whose examples are the same bytes
    got = codec.encode_example_requests([("m", 1, d)], predict_input="examples")[0]
    lst = codec.encode_example_requests([("m", 1, d)])[0]
    from tensorflow_serving.apis.predict_pb2 import PredictRequest

    req = PredictRequest.FromString(got)
    t = req.inputs["examples"]
    assert t.dtype == 7 and [x.size for x in t.tensor_shape.dim] == [n] and len(t.string_val) == n
    assert req.ByteSize() == len(got) and req.SerializeToString(deterministic=True) == got
    assert b"".join(b"\x0a" + _vi(len(s)) + s for s in t.string_val) == lst[len(lst) - sum(len(s) + 1 + len(_vi(len(s))) for s in t.string_val):]


def _vi(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def test_examples_larger_than_the_emit_image(codec):
    rng = np.random.default_rng(9)
    _check(codec, {"ids": rng.integers(-(1 << 62), -1, (6, 5000)), "x": rng.standard_normal((6, 2)).astype(np.float32)})
    _check(codec, {"big": rng.standard_normal((3, 9000)).astype(np.float32)}, key="a")


def test_ragged_columns_host_and_device_lengths(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(11)
    n = 300
    hist, emb = rng.integers(0, 50_000, (n, 64)), rng.standard_normal((n, 16, 4)).astype(np.float32)
    lh, le = _lengths(rng, n, 64), _lengths(rng, n, 16)
    d = {"hist": RaggedColumn(hist, lh), "emb": RaggedColumn(emb, le), "dense": rng.standard_normal((n, 8)).astype(np.float32),
         "bias": np.float64(0.25), "b": RaggedColumn(rng.integers(0, 2, (n, 3)).astype(np.bool_), _lengths(rng, n, 3))}
    _check(codec, d)
    _check(codec, d, version=None, grpc_frame=True, key="été")
    dd = dict(d, hist=RaggedColumn(torch.from_numpy(hist).cuda(), torch.from_numpy(lh).cuda()),
              emb=RaggedColumn(torch.from_numpy(emb).cuda(), le))
    got = codec.encode_example_requests([("m", 1, dd)], predict_input="examples")[0]
    assert got == predict_examples_ref("m", 1, d, "examples")
    # a ragged str column: the host route, one example at a time in the reference
    s = {"s": RaggedColumn(np.array([["a", "bb", "ccc"]] * 4), [0, 3, 1, 2]), "v": np.arange(4)}
    _check(codec, s)


def test_given_order(codec):
    from tensorflow_serving.apis.predict_pb2 import PredictRequest

    d = {"zz": np.arange(6, dtype=np.float32).reshape(3, 2), "a": np.arange(3), "ab": np.ones(3, np.float64)}
    got = codec.encode_example_requests([("m", 2, d)], order="given", predict_input="examples")[0]
    det = predict_examples_ref("m", 2, d)
    assert got != det and len(got) == len(det)
    from tensorflow.core.example.example_pb2 import Example

    g = PredictRequest.FromString(got).inputs["examples"].string_val
    assert [Example.FromString(x) for x in g] == examples(d)
    pos = [g[0].find(k.encode()) for k in d]
    assert pos == sorted(pos)


def test_device_and_pinned_columns(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(13)
    x, ids, h = rng.standard_normal((64, 8)).astype(np.float32), rng.integers(-5, 1 << 40, (64, 3)), rng.standard_normal(64).astype(np.float16)
    d = {"x": torch.from_numpy(x).cuda(), "ids": torch.from_numpy(ids).cuda(), "h": torch.from_numpy(h).cuda()}
    got = codec.encode_example_requests([("m", 1, d)], predict_input="examples")[0]
    assert got == predict_examples_ref("m", 1, {"x": x, "ids": ids, "h": h})
    p = codec.pinned_empty((300, 7), np.float32)
    p[:] = rng.standard_normal((300, 7))
    q = codec.pinned_empty((300,), np.int64)
    q[:] = _lengths(rng, 300, 7)
    _check(codec, {"x": p, "n": np.arange(300, dtype=np.uint16), "r": RaggedColumn(p, q)})


def _structs(items):
    """host-column ExampleRequests, ragged entries and targets: items = [(name, version, input_dict, key or None)]"""
    keep, structs, rg, tg = [], [], [], []
    for name, version, d, key in items:
        n, preps = _example_columns(d)
        feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
        nb = name.encode()
        structs.append(N.ExampleRequest(model_name=nb, model_name_len=len(nb), has_version=int(version is not None), order=N.ORDER_UPB,
                                        version=version or 0, n_examples=n, n_features=len(preps), flags=0, features=feats))
        rg += [p[3] or N.Ragged() for p in preps]
        kb = key.encode() if key is not None else None
        tg.append(N.ExampleTarget(kind=N.EXAMPLES_PREDICT_STRING, key=kb, key_len=len(kb)) if key is not None else N.ExampleTarget())
        keep.append((preps, feats, nb, kb))
    return (N.ExampleRequest * len(structs))(*structs), (N.Ragged * max(len(rg), 1))(*rg), (N.ExampleTarget * len(tg))(*tg), keep


def test_forty_requests_mixing_classify_and_predict(codec):
    rng = np.random.default_rng(15)
    items = []
    for i in range(40):
        n = int(rng.integers(0, 200))
        d = {"dense": rng.standard_normal((n, i % 4)).astype(np.float32)}
        if i % 2:
            d["r"] = RaggedColumn(rng.integers(-1000, 1 << 33, (n, 1 + i % 9)), _lengths(rng, n, 1 + i % 9))
        if i % 3 == 0:
            d["ids"] = rng.integers(-1000, 1 << 33, (n, i % 5))
        if i % 5 == 2:
            d["k"] = np.float64(i)
        key = None if i % 3 == 1 else ["examples", "", "a", "ab", "été", "k" * 200][i % 6]
        items.append((f"model{i}", i if i % 4 else None, d, key))
    reqs, rg, tg, keep = _structs(items)
    cap = C.c_uint64()
    N.check(codec._lib.b200tfs_example_target_arena_size(40, reqs, tg, C.byref(cap)))
    wire = np.empty(cap.value, np.uint8)
    off, ln = (C.c_uint64 * 40)(), (C.c_uint64 * 40)()
    N.check(codec._lib.b200tfs_encode_example_targets_host(codec.ctx, 40, reqs, rg, tg, wire.ctypes.data, cap.value, off, ln))
    for i, (name, version, d, key) in enumerate(items):
        ref = ragged_ref(name, version, d) if key is None else predict_examples_ref(name, version, d, key)
        assert wire[off[i]: off[i] + ln[i]].tobytes() == ref, i
    # every request Predict, through the Python call, framed
    got = codec.encode_example_requests([it[:3] for it in items], predict_input="x", grpc_frame=True)
    assert got == [predict_examples_ref(*it[:3], "x", grpc_frame=True) for it in items]


def test_graph_replay_with_new_values_and_lengths():
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(17)
        n, L = 3000, 48
        ids, x = rng.integers(0, 1000, (n, L)), rng.standard_normal((n, 4)).astype(np.float32)
        li = _lengths(rng, n, L)
        dids, dx, dli = dev.upload(ids), dev.upload(x), dev.upload(li)
        feats = (N.Feature * 2)(N.Feature(data=dids, src_dtype=9, flags=0, row_elems=L, key=b"ids", key_len=3),
                                N.Feature(data=dx, src_dtype=1, flags=0, row_elems=4, key=b"x", key_len=1))
        rg = (N.Ragged * 2)(N.Ragged(lengths=dli, max_len=L, unit=1, flags=N.F_DEVICE_DATA), N.Ragged())
        reqs = (N.ExampleRequest * 2)(*[N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3,
                                                         n_examples=n, n_features=2, flags=0, features=feats)] * 2)
        rg2 = (N.Ragged * 4)(*(list(rg) * 2))
        tg = (N.ExampleTarget * 2)(N.ExampleTarget(kind=N.EXAMPLES_PREDICT_STRING, key=b"examples", key_len=8), N.ExampleTarget())
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_target_arena_size(2, reqs, tg, C.byref(cap)))
        arena = (dev.malloc(cap.value + 256) + 255) & ~255
        N.check(lib.b200tfs_encode_example_targets_async(dev.ctx, 2, reqs, rg2, tg, arena, cap.value))   # sizes every buffer
        N.check(lib.b200tfs_encode_results(dev.ctx, 2, None, None))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_encode_example_targets_async(dev.ctx, 2, reqs, rg2, tg, arena, cap.value))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        off, ln = (C.c_uint64 * 2)(), (C.c_uint64 * 2)()
        for rep in range(3):
            ids = rng.integers(-(1 << (20 * rep)), 1 << min(20 * rep + 5, 62), (n, L))
            x = rng.standard_normal((n, 4)).astype(np.float32)
            li = rng.integers(0, L + 1, n) // (rep + 1)
            for ptr, a in ((dids, ids), (dx, x), (dli, li)):
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, ptr, a.ctypes.data, a.nbytes))
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_encode_results(dev.ctx, 2, off, ln))
            d = {"ids": RaggedColumn(ids, li), "x": x}
            assert dev.download(arena + off[0], ln[0]).tobytes() == predict_examples_ref("m", 3, d), rep
            assert dev.download(arena + off[1], ln[1]).tobytes() == ragged_ref("m", 3, d), rep
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


def test_out_of_range_device_length():
    """The bad request sits in front of good ones inside a zeroed arena with slack behind it: a missing check shows as a wrong
    status, wrong neighbours or bytes past the arena."""
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(19)
        n, L = 300, 20
        items, dicts, keep = [], [], []
        for r in range(4):
            ids, x = rng.integers(-(1 << 40), 1 << 40, (n, L)), rng.standard_normal((n, L)).astype(np.float32)
            li, lx = _lengths(rng, n, L), _lengths(rng, n, L)
            dicts.append({"ids": RaggedColumn(ids, li), "x": RaggedColumn(x, lx)})
            bad_li = li.copy()
            if r == 0:
                bad_li[n // 2] = L + 1
            dids = dev.upload(np.concatenate([ids, ids]))      # the padded column is the first half of a larger allocation
            feats = (N.Feature * 2)(N.Feature(data=dids, src_dtype=9, flags=0, row_elems=L, key=b"ids", key_len=3),
                                    N.Feature(data=dev.upload(x), src_dtype=1, flags=0, row_elems=L, key=b"x", key_len=1))
            keep.append(feats)
            items.append((N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_examples=n,
                                           n_features=2, flags=0, features=feats),
                          [N.Ragged(lengths=dev.upload(bad_li), max_len=L, unit=1, flags=N.F_DEVICE_DATA),
                           N.Ragged(lengths=dev.upload(lx), max_len=L, unit=1, flags=N.F_DEVICE_DATA)]))
        reqs = (N.ExampleRequest * 4)(*[it[0] for it in items])
        rg = (N.Ragged * 8)(*[g for it in items for g in it[1]])
        keys = [b"examples", b"a", b"ab", b""]
        tg = (N.ExampleTarget * 4)(*[N.ExampleTarget(kind=N.EXAMPLES_PREDICT_STRING, key=k, key_len=len(k)) for k in keys])
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_target_arena_size(4, reqs, tg, C.byref(cap)))
        slack = 1 << 20
        arena = (dev.malloc(cap.value + slack + 256) + 255) & ~255
        zeros = np.zeros(cap.value + slack, np.uint8)
        N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena, zeros.ctypes.data, zeros.nbytes))
        N.check(lib.b200tfs_encode_example_targets_async(dev.ctx, 4, reqs, rg, tg, arena, cap.value))
        off, ln = (C.c_uint64 * 4)(), (C.c_uint64 * 4)()
        assert lib.b200tfs_encode_results(dev.ctx, 4, off, ln) == N.E_SHAPE
        assert off[0] == 0 and ln[0] == 0
        for r in range(1, 4):
            assert dev.download(arena + off[r], ln[r]).tobytes() == predict_examples_ref("m", 3, dicts[r], keys[r]), r
        assert not dev.download(arena + cap.value, slack).any()
    finally:
        dev.close()


def test_predict_examples_end_to_end():
    import grpc
    from fake_server import IdentityServer
    from min_tfs_client.requests import PREDICT_METHOD, TensorServingClient, gpu_predict_examples_serializer, gpu_response_deserializer
    from tensorflow.core.example.example_pb2 import Example

    srv = IdentityServer()
    try:
        client = TensorServingClient("127.0.0.1", srv.port)
        rng = np.random.default_rng(21)
        d = {"hist": RaggedColumn(rng.integers(0, 500, (20, 16)), _lengths(rng, 20, 16)), "x": rng.standard_normal((20, 3)).astype(np.float32),
             "bias": np.float64(0.5)}
        resp = client.predict_examples_request("m", d, model_version=4)
        assert srv.received[-1] == predict_examples_ref("m", 4, d)
        out = resp.to_proto().outputs["examples"]
        assert out.dtype == 7 and [x.size for x in out.tensor_shape.dim] == [20]
        assert [Example.FromString(s) for s in out.string_val] == examples(d)
        assert resp.model_spec.name == "m" and resp.model_spec.version.value == 4
        ch = grpc.insecure_channel(f"127.0.0.1:{srv.port}")
        call = ch.unary_unary(PREDICT_METHOD, request_serializer=gpu_predict_examples_serializer, response_deserializer=gpu_response_deserializer)
        call(("m", None, d, "inputs"), timeout=30)
        assert srv.received[-1] == predict_examples_ref("m", None, d, "inputs")
        ch.close()
    finally:
        srv.stop()
