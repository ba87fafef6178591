"""tf.Example requests with a shared context (ExampleListWithContext) encoded on the GPU: every case compares bytes with the
protobuf runtime's serialization of the request examples_with_context_from_input_dict builds from host copies of the same
columns, in the Classify form and the Predict-ELWC form."""
import ctypes as C

import numpy as np
import pytest

from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn
from min_tfs_client.requests import TensorServingClient, examples_from_input_dict, examples_with_context_from_input_dict
from tensorflow.core.framework import types_pb2
from tensorflow_serving.apis.classification_pb2 import ClassificationRequest
from tensorflow_serving.apis.input_pb2 import ExampleListWithContext
from tensorflow_serving.apis.predict_pb2 import PredictRequest

pytestmark = pytest.mark.gpu


def _host(v):
    if isinstance(v, RaggedColumn):
        return RaggedColumn(_host(v.values), _host(v.lengths))
    if isinstance(v, BytesColumn):
        return BytesColumn(_host(v.data), _host(v.offsets), v.shape)
    return v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)


def ref(name, version, d, ctx=None, key=None, grpc_frame=False):
    """the wire of one request: Classify (key None) or Predict, with a context (ctx not None) or without"""
    h = {k: _host(v) for k, v in d.items()}
    hc = None if ctx is None else {k: _host(v) for k, v in ctx.items()}
    if key is None:
        msg = TensorServingClient._make_example_request(None, ClassificationRequest, name, h, version, hc)
    else:
        msg = PredictRequest()
        msg.model_spec.name = name
        if version is not None:
            msg.model_spec.version.value = version
        if hc is None:
            values = examples_from_input_dict(h).example_list.examples
        else:
            values = [examples_with_context_from_input_dict(h, hc).example_list_with_context]
        t = msg.inputs[key.decode() if isinstance(key, bytes) else key]
        t.dtype = types_pb2.DT_STRING
        t.tensor_shape.dim.add().size = len(values)
        t.string_val.extend(v.SerializeToString(deterministic=True) for v in values)
    wire = msg.SerializeToString(deterministic=True)
    return (b"\x00" + len(wire).to_bytes(4, "big") + wire) if grpc_frame else wire


def _strings(rng, m, lo=0, hi=12):
    return [bytes(rng.integers(0, 256, int(rng.integers(lo, hi + 1)), dtype=np.uint8)) for _ in range(m)]


def _column(strs, shape=None, start=0, tail=3):
    lens = np.array([len(s) for s in strs], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64) + start
    data = np.frombuffer(b"\xEE" * start + b"".join(strs) + b"\xEE" * tail, np.uint8).copy()
    return BytesColumn(data, offsets, shape)


def _check(codec, d, ctx, name="m", version=1, **kw):
    got = codec.encode_example_requests([(name, version, d, ctx)], **kw)[0]
    want = ref(name, version, d, ctx, kw.get("predict_input"), kw.get("grpc_frame", False))
    assert got == want
    return got


def _every_dtype(rng):
    ctx = {f"f{np.dtype(t).name}": rng.standard_normal(7).astype(t) for t in (np.float32, np.float64, np.float16)}
    for t in (np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64):
        info = np.iinfo(t)
        ctx[f"i{np.dtype(t).name}"] = np.array([info.min, info.max, 0, 1, -1 if info.min else 2], t).reshape(5, 1)
    ctx["bool"] = np.array([[True, False], [False, True]])
    ctx["nan"] = np.array([np.nan, -np.inf, np.float32(np.uint32(0x7F800001).view(np.float32))], np.float32)
    ctx["scalar"] = np.float64(0.25)
    ctx["i0"] = np.int64(-(1 << 63))
    ctx["s"] = _column([b"", b"\x00", b"\xff\xfe", b"x" * 64])
    ctx["none"] = np.zeros((3, 0), np.float32)
    return ctx


@pytest.mark.parametrize("key", [None, "elwc"])
def test_every_context_dtype(codec, key):
    rng = np.random.default_rng(1)
    d = {"item": rng.standard_normal((20, 4)).astype(np.float32), "item_id": rng.integers(-5, 1 << 40, 20)}
    ctx = _every_dtype(rng)
    for grpc_frame in (False, True):
        _check(codec, d, ctx, predict_input=key, grpc_frame=grpc_frame)
        _check(codec, d, ctx, version=None, predict_input=key, grpc_frame=grpc_frame)
    _check(codec, d, {}, predict_input=key)                                    # an empty context: 12 00
    _check(codec, {}, ctx, predict_input=key)                                  # no examples
    _check(codec, {}, {}, predict_input=key)
    _check(codec, {"x": np.zeros((0, 3), np.float32)}, {"c": np.ones(2, np.float32)}, predict_input=key)
    got = _check(codec, d, {}, predict_input=key)
    assert got.endswith(b"\x12\x00")


def test_empty_context_wire(codec):
    got = _check(codec, {"a": np.ones((2, 1), np.float32)}, {})
    assert got.endswith(b"\x12\x00") and not got.endswith(b"\x12\x02\x0a\x00")


@pytest.mark.parametrize("key", [None, "elwc"])
def test_context_only_columns_and_large_contexts(codec, key):
    rng = np.random.default_rng(2)
    d = {"item": rng.standard_normal((50, 8)).astype(np.float32)}                 # dense examples: a closed-form size
    _check(codec, d, {"hist": rng.integers(-(1 << 62), 1 << 62, 50)}, predict_input=key)
    _check(codec, d, {"q": _column(_strings(rng, 3, 0, 40))}, predict_input=key)
    # a context larger than the 16 KB emit image, dense and integer
    _check(codec, d, {"user": rng.standard_normal(6000).astype(np.float32)}, predict_input=key)
    _check(codec, d, {"ids": rng.integers(-(1 << 63), -1, 3000, dtype=np.int64), "f": rng.standard_normal(10).astype(np.float32)},
           predict_input=key)
    # strings of 0 B, 64 B and over 16 KiB, with NULs and high bytes
    strs = [b"", bytes(range(64)), bytes(rng.integers(0, 256, 20_000, dtype=np.uint8)), b"\x00" * 5, b"\xff" * 65]
    _check(codec, d, {"s": _column(strs, start=13), "t": _column([b"q\x00"], ())}, predict_input=key)
    _check(codec, {"s": _column(_strings(rng, 30, 0, 20), (10, 3))}, {"s": _column(strs)}, predict_input=key)


def test_order_given_and_grpc_frame(codec):
    rng = np.random.default_rng(3)
    d = {"zz": rng.standard_normal((5, 2)).astype(np.float32), "aa": rng.integers(0, 9, 5)}
    ctx = {"cz": np.arange(3), "cb": np.ones(2, np.float32), "cm": _column([b"mm"])}
    for key in (None, b"in"):
        for grpc_frame in (False, True):
            got = codec.encode_example_requests([("m", 1, d, ctx)], order="given", grpc_frame=grpc_frame, predict_input=key)[0]
            want = ref("m", 1, d, ctx, key, grpc_frame)
            assert len(got) == len(want) and got != want
            body, wbody = (got[5:], want[5:]) if grpc_frame else (got, want)
            if key is None:
                assert ClassificationRequest.FromString(body).SerializeToString(deterministic=True) == wbody
            else:                               # the ELWC is opaque bytes to the PredictRequest: compare it as a message
                elwc = [ExampleListWithContext.FromString(PredictRequest.FromString(b).inputs["in"].string_val[0]) for b in (body, wbody)]
                assert elwc[0] == elwc[1]
            assert got.find(b"\x02cz") < got.find(b"\x02cb") < got.find(b"\x02cm")       # insertion order in the context too
    _check(codec, d, ctx, grpc_frame=True)


def test_forty_requests_mixing_forms(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(4)
    items, wants = [], []
    for i in range(40):
        n = int(rng.integers(0, 60))
        d = {"dense": rng.standard_normal((n, i % 3)).astype(np.float32)}
        if i % 2:
            d["s"] = _column(_strings(rng, n * 2, 0, 30), (n, 2), start=i)
        if i % 7 == 2:
            d["i"] = rng.integers(-5, 1 << 35, (n, 2))
        ctx = None
        if i % 4:
            ctx = {"u": rng.standard_normal(i).astype(np.float32)}
            if i % 3 == 0:
                ctx["h"] = torch.from_numpy(rng.integers(-(1 << 40), 1 << 40, 5)).cuda()
            if i % 5 == 1:
                p = codec.pinned_empty((4,), np.int32)
                p[:] = rng.integers(-9, 9, 4)
                ctx["p"] = p
            if i % 6 == 1:
                c = _column(_strings(rng, 4, 0, 100))
                ctx["q"] = BytesColumn(torch.from_numpy(c.data).cuda(), torch.from_numpy(c.offsets).cuda()) if i % 12 == 1 else c
            if i % 8 == 3:
                ctx = {}
        items.append((f"model{i}", i if i % 5 else None, d, ctx))
    for key in (None, "ex"):
        got = codec.encode_example_requests(items, predict_input=key)
        for j, (name, version, d, ctx) in enumerate(items):
            assert got[j] == ref(name, version, d, ctx, key), (key, j)
    # 3-tuples and 4-tuples in one call
    got = codec.encode_example_requests([items[1][:3], items[2], items[0][:3] + (None,)], predict_input="ex")
    assert got == [ref(*items[1][:3], None, "ex"), ref(*items[2], "ex"), ref(*items[0][:3], None, "ex")]


def test_numpy_str_context_takes_the_host_route(codec):
    rng = np.random.default_rng(5)
    d = {"x": rng.standard_normal((4, 2)).astype(np.float32)}
    ctx = {"query": np.array(["été", "a\x00b"]), "id": np.arange(3)}
    before = codec.kernel_launches()
    for key in (None, "elwc"):
        want = ref("m", 1, d, ctx, key)
        assert codec.encode_example_requests([("m", 1, d, ctx)], predict_input=key)[0] == want
    assert codec.kernel_launches() == before
    with pytest.raises(ValueError, match="context"):
        codec.encode_example_requests([("m", 1, d, {"r": RaggedColumn(np.zeros((2, 3), np.float32), [1, 2])})])


def test_graph_replay_with_new_context_values():
    """a captured encode replayed over new context integers and string offsets that change the context's and the request's
    length (the varints of both move across a byte edge)"""
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(6)
        n, m, cap_bytes = 100, 40, 8192
        items = rng.standard_normal((n, 4)).astype(np.float32)
        def make(rep):
            ints = rng.integers(-(1 << 62), 1 << 62, m) if rep % 2 else rng.integers(0, 100, m)
            strs = _strings(rng, 3, 0, 10 + 1000 * (rep % 2))
            c = _column(strs, tail=0)
            data = np.zeros(cap_bytes, np.uint8)
            data[: c.data_len] = c.data
            return ints.astype(np.int64), data, c.offsets, c
        ints, data, offs, col = make(0)
        di, dd, do = dev.upload(ints), dev.upload(data), dev.upload(offs)
        dx = dev.upload(items)
        fa = (N.Feature * 1)(N.Feature(data=dx, src_dtype=1, flags=0, row_elems=4, key=b"item", key_len=4))
        cfa = (N.Feature * 2)(N.Feature(data=di, src_dtype=9, flags=0, row_elems=m, key=b"hist", key_len=4),
                              N.Feature(data=dd, src_dtype=7, flags=0, row_elems=3, key=b"q", key_len=1))
        cba = (N.Bytes * 2)(N.Bytes(), N.Bytes(offsets=do, data_len=cap_bytes, flags=N.F_DEVICE_DATA))
        req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_examples=n,
                               n_features=1, flags=0, features=fa)
        cx = N.ExampleContext(features=cfa, n_features=2, present=1)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_context_arena_size(1, C.byref(req), None, None, C.byref(cx), cba, C.byref(cap)))
        arena = (dev.malloc(cap.value + 256) + 255) & ~255
        N.check(lib.b200tfs_encode_example_contexts_async(dev.ctx, 1, C.byref(req), None, None, None, C.byref(cx), cba, arena, cap.value))
        N.check(lib.b200tfs_encode_results(dev.ctx, 1, None, None))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_encode_example_contexts_async(dev.ctx, 1, C.byref(req), None, None, None, C.byref(cx), cba, arena, cap.value))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        lens = set()
        for rep in range(4):
            ints, data, offs, col = make(rep)
            for ptr, a in ((di, ints), (dd, data), (do, offs)):
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, ptr, a.ctypes.data, a.nbytes))
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_encode_results(dev.ctx, 1, off, ln))
            wire = dev.download(arena + off[0], ln[0]).tobytes()
            assert wire == ref("m", 3, {"item": items}, {"hist": ints, "q": col}), rep
            lens.add(ln[0])
        assert len(lens) > 1
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


@pytest.mark.parametrize("case", ["decreasing", "negative", "past_data_len"])
def test_bad_device_context_offsets(codec, case):
    """The request whose context has bad device offsets sits in front of good ones, its buffer inside a larger allocation, and
    the arena has a zeroed tail: E_SHAPE for it, the others byte-exact, nothing written past the arena."""
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(7)
        n, m = 50, 20
        cols = [_column(_strings(rng, m, 0, 30), start=16, tail=4096) for _ in range(4)]
        o = cols[0].offsets.copy()
        if case == "decreasing":
            o[7] = o[6] - 1
        elif case == "negative":
            o[m // 2] = -(1 << 40)
        else:
            o[m] = cols[0].data_len + 1
        x = rng.standard_normal((n, 3)).astype(np.float32)
        dx = dev.upload(x)
        keep, reqs, cxs, cbs = [], [], [], []
        for r in range(4):
            offs = o if r == 0 else cols[r].offsets
            fa = (N.Feature * 1)(N.Feature(data=dx, src_dtype=1, flags=0, row_elems=3, key=b"x", key_len=1))
            cfa = (N.Feature * 1)(N.Feature(data=dev.upload(cols[r].data), src_dtype=7, flags=0, row_elems=m, key=b"q", key_len=1))
            keep += [fa, cfa]
            reqs.append(N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_examples=n,
                                         n_features=1, flags=0, features=fa))
            cxs.append(N.ExampleContext(features=cfa, n_features=1, present=1))
            cbs.append(N.Bytes(offsets=dev.upload(offs), data_len=cols[r].data_len, flags=N.F_DEVICE_DATA))
        ra, ca, ba = (N.ExampleRequest * 4)(*reqs), (N.ExampleContext * 4)(*cxs), (N.Bytes * 4)(*cbs)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_context_arena_size(4, ra, None, None, ca, ba, C.byref(cap)))
        slack = 1 << 20
        arena = (dev.malloc(cap.value + slack + 256) + 255) & ~255
        zeros = np.zeros(cap.value + slack, np.uint8)
        N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena, zeros.ctypes.data, zeros.nbytes))
        N.check(lib.b200tfs_encode_example_contexts_async(dev.ctx, 4, ra, None, None, None, ca, ba, arena, cap.value))
        off, ln = (C.c_uint64 * 4)(), (C.c_uint64 * 4)()
        assert lib.b200tfs_encode_results(dev.ctx, 4, off, ln) == N.E_SHAPE
        assert off[0] == 0 and ln[0] == 0
        for r in range(1, 4):
            assert dev.download(arena + off[r], ln[r]).tobytes() == ref("m", 3, {"x": x}, {"q": cols[r]}), r
        assert not dev.download(arena + cap.value, slack).any()
        torch = pytest.importorskip("torch")
        bad = BytesColumn(torch.from_numpy(cols[0].data).cuda(), torch.from_numpy(o).cuda())
        with pytest.raises(ValueError):
            codec.encode_example_requests([("m", 1, {"x": x}, {"q": cols[1]}), ("m", 1, {"x": x}, {"q": bad})])
        with pytest.raises(ValueError):                      # the same offsets from the host: refused before any launch
            codec.encode_example_requests([("m", 1, {"x": x}, {"q": BytesColumn(cols[0].data, o)})])
        _check(codec, {"x": x}, {"q": cols[2]})
    finally:
        dev.close()


def _context_server():
    """the fake server's toy model for ExampleListWithContext requests: an example's score is the sum of its float features and
    of the context's"""
    from fake_server import IdentityServer
    from tensorflow_serving.apis import classification_pb2, regression_pb2

    class ContextServer(IdentityServer):
        def _scores(self, req):
            elwc = req.input.example_list_with_context
            return [self._score(ex) + self._score(elwc.context) for ex in elwc.examples]

        def _classify(self, request_bytes, context):
            self.received.append(request_bytes)
            req = classification_pb2.ClassificationRequest.FromString(request_bytes)
            resp = classification_pb2.ClassificationResponse()
            resp.model_spec.CopyFrom(req.model_spec)
            resp.result.SetInParent()
            for s in self._scores(req):
                cls = resp.result.classifications.add()
                cls.classes.add(label="positive", score=s)
                cls.classes.add(label="negative", score=-s)
            return resp.SerializeToString()

        def _regress(self, request_bytes, context):
            self.received.append(request_bytes)
            req = regression_pb2.RegressionRequest.FromString(request_bytes)
            resp = regression_pb2.RegressionResponse()
            resp.model_spec.CopyFrom(req.model_spec)
            resp.result.SetInParent()
            for s in self._scores(req):
                resp.result.regressions.add(value=s)
            return resp.SerializeToString()

    return ContextServer()


def test_classify_and_regress_end_to_end():
    import grpc
    from min_tfs_client.requests import CLASSIFY_METHOD, REGRESS_METHOD, gpu_example_request_serializer
    from tensorflow_serving.apis.classification_pb2 import ClassificationResponse
    from tensorflow_serving.apis.regression_pb2 import RegressionResponse

    srv = _context_server()
    try:
        client = TensorServingClient("127.0.0.1", srv.port)
        rng = np.random.default_rng(8)
        d = {"item": rng.standard_normal((12, 3)).astype(np.float32), "item_id": rng.integers(0, 1 << 40, 12)}
        ctx = {"user": rng.standard_normal(16).astype(np.float32), "query": BytesColumn.from_array(np.array(["wörld"]))}
        ch = grpc.insecure_channel(f"127.0.0.1:{srv.port}")
        cls = ch.unary_unary(CLASSIFY_METHOD, request_serializer=gpu_example_request_serializer,
                             response_deserializer=ClassificationResponse.FromString)(("m", 4, d, ctx), timeout=30)
        assert cls == client.classification_request("m", d, model_version=4, context_dict=ctx)
        assert srv.received[0] == ref("m", 4, d, ctx)
        assert ClassificationRequest.FromString(srv.received[1]) == ClassificationRequest.FromString(srv.received[0])   # host protobuf
        assert len(cls.result.classifications) == 12
        assert cls.result.classifications[0].classes[0].score == pytest.approx(float(d["item"][0].sum() + ctx["user"].sum()), rel=1e-5)
        reg = ch.unary_unary(REGRESS_METHOD, request_serializer=gpu_example_request_serializer,
                             response_deserializer=RegressionResponse.FromString)(("m", 4, d, ctx), timeout=30)
        assert reg == client.regression_request("m", d, model_version=4, context_dict=ctx)
        assert len(reg.result.regressions) == 12
        ch.close()
    finally:
        srv.stop()
