"""tf.Example requests with a shared context (ExampleListWithContext) without a GPU: the b200tfs_example_context mirror, the
refusals of the *_example_context* entry points (checked before the context is looked at), the closed-form size against the
protobuf ByteSize() in the Classify and the Predict-ELWC form, and the arena bound against the protobuf size of random integer
and bytes contexts at their worst case."""
import ctypes as C

import numpy as np
import pytest

from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn, _example_columns
from min_tfs_client.requests import TensorServingClient, examples_with_context_from_input_dict
from tensorflow_serving.apis.classification_pb2 import ClassificationRequest
from tensorflow_serving.apis.predict_pb2 import PredictRequest

DT_STRING = 7


def _ref(d, ctx, key=None, grpc_frame=False):
    """the Classify form, or with `key` the Predict-ELWC form, as the protobuf runtime serializes it"""
    if key is None:
        msg = TensorServingClient._make_example_request(None, ClassificationRequest, "m", d, 2, ctx)
    else:
        msg = PredictRequest()
        msg.model_spec.name = "m"
        msg.model_spec.version.value = 2
        t = msg.inputs[key]
        t.dtype = DT_STRING
        t.tensor_shape.dim.add().size = 1
        t.string_val.append(examples_with_context_from_input_dict(d, ctx).example_list_with_context.SerializeToString(deterministic=True))
    wire = msg.SerializeToString(deterministic=True)
    return (b"\x00" + len(wire).to_bytes(4, "big") + wire) if grpc_frame else wire


def _struct(d, ctx, key=None, grpc_frame=False):
    """(request, target or None, context, bytes entries, context bytes entries, keep-alive) of the device route's structs"""
    n, preps = _example_columns(d)
    feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
    bs = (N.Bytes * max(len(preps), 1))(*[p.bytes_entry or N.Bytes() for p in preps])
    _, cpreps = _example_columns(ctx, context=True)
    cfeats = (N.Feature * max(len(cpreps), 1))(*[p[0] for p in cpreps])
    cbs = (N.Bytes * max(len(cpreps), 1))(*[p.bytes_entry or N.Bytes() for p in cpreps])
    req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=2, n_examples=n,
                           n_features=len(preps), flags=N.RF_GRPC_FRAME if grpc_frame else 0, features=feats)
    cx = N.ExampleContext(features=cfeats, n_features=len(cpreps), present=1)
    tg = None
    if key is not None:
        kb = key.encode()
        tg = N.ExampleTarget(kind=N.EXAMPLES_PREDICT_ELWC, key=kb, key_len=len(kb))
    return req, tg, cx, bs, cbs, (preps, feats, cpreps, cfeats)


def _rcs(req, tg, cx, bs, cbs):
    """arena size, _host and _async with no device context: their argument checks, or E_ARG for the missing context"""
    lib = N.load()
    out = C.c_uint64()
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    buf = C.create_string_buffer(256)
    t = C.byref(tg) if tg is not None else None
    return [lib.b200tfs_example_context_arena_size(1, C.byref(req), bs, t, C.byref(cx), cbs, C.byref(out)),
            lib.b200tfs_encode_example_contexts_host(None, 1, C.byref(req), None, bs, t, C.byref(cx), cbs, buf, 16, off, ln),
            lib.b200tfs_encode_example_contexts_async(None, 1, C.byref(req), None, bs, t, C.byref(cx), cbs, buf, 16)]


def _size(req, tg, cx):
    out = C.c_uint64()
    rc = N.load().b200tfs_example_context_request_size(C.byref(req), C.byref(tg) if tg is not None else None,
                                                       C.byref(cx) if cx is not None else None, C.byref(out))
    return rc, out.value


def _column(strs, shape=None):
    lens = np.array([len(s) for s in strs], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return BytesColumn(np.frombuffer(b"".join(strs) + b"\xEE", np.uint8), offsets, shape)


def test_context_mirror():
    assert C.sizeof(N.ExampleContext) == 16
    assert [f[0] for f in N.ExampleContext._fields_] == ["features", "n_features", "present"]
    assert N.ExampleContext.n_features.offset == 8 and N.ExampleContext.present.offset == 12
    assert N.EXAMPLES_PREDICT_ELWC == 2


def test_context_refusals():
    d = {"x": np.zeros((4, 3), np.float32)}
    ctx = {"u": np.zeros(5, np.float32), "s": _column([b"ab", b"c"])}
    req, tg, cx, bs, cbs, keep = _struct(d, ctx)
    assert _rcs(req, tg, cx, bs, cbs) == [N.OK, N.E_ARG, N.E_ARG]        # well-formed: only the device context is missing
    assert "context" in N.last_error() or "bad arguments" in N.last_error()
    for present in (2, -1):
        cx.present = present
        assert _rcs(req, tg, cx, bs, cbs) == [N.E_ARG] * 3 and "present" in N.last_error()
    cx.present = 1
    cx.n_features = -1
    assert _rcs(req, tg, cx, bs, cbs) == [N.E_ARG] * 3
    cx.n_features = 2
    cx.features = None
    assert _rcs(req, tg, cx, bs, cbs) == [N.E_ARG] * 3
    cx.features = keep[3]
    keep[3][1].flags |= N.F_BROADCAST
    assert _rcs(req, tg, cx, bs, cbs) == [N.E_ARG] * 3 and "broadcast" in N.last_error()
    keep[3][1].flags &= ~N.F_BROADCAST
    # the targets: PREDICT_STRING carries no context, PREDICT_ELWC needs one
    kb = b"examples"
    ps = N.ExampleTarget(kind=N.EXAMPLES_PREDICT_STRING, key=kb, key_len=len(kb))
    assert _rcs(req, ps, cx, bs, cbs) == [N.E_ARG] * 3 and "PREDICT_STRING" in N.last_error()
    pe = N.ExampleTarget(kind=N.EXAMPLES_PREDICT_ELWC, key=kb, key_len=len(kb))
    assert _rcs(req, pe, cx, bs, cbs) == [N.OK, N.E_ARG, N.E_ARG]
    cx.present = 0
    assert _rcs(req, pe, cx, bs, cbs) == [N.E_ARG] * 3 and "kind" in N.last_error()
    cx.present = 1
    assert _size(req, pe, None)[0] == N.E_ARG and "kind" in N.last_error()
    # a DT_STRING context feature without its bytes entry
    assert _rcs(req, tg, cx, bs, None) == [N.E_DTYPE] * 3
    # host offsets that break the rule: refused by the _host entry point before anything is looked up on a device
    o = np.array([0, 3, 1], np.int64)
    cbs[1].offsets = o.ctypes.data
    assert _rcs(req, tg, cx, bs, cbs)[:2] == [N.OK, N.E_SHAPE]
    # a ragged context and a device dtype the device route does not take
    with pytest.raises(ValueError, match="context"):
        _example_columns({"r": RaggedColumn(np.zeros((2, 3), np.float32), [1, 2])}, context=True)
    with pytest.raises(ValueError, match="context"):
        examples_with_context_from_input_dict(d, {"r": RaggedColumn(np.zeros((2, 3), np.float32), [1, 2])})


@pytest.mark.parametrize("key", [None, "elwc"])
@pytest.mark.parametrize("grpc_frame", [False, True])
def test_context_request_size(key, grpc_frame):
    """float-only contexts whose sizes cross the one / two / three byte varint edges, in both forms, and the empty context"""
    d = {"a": np.arange(6, dtype=np.float32).reshape(2, 3), "b": np.float64(0.5)}
    sizes = set()
    for m in list(range(20, 36)) + list(range(4083, 4099)) + [None]:
        ctx = {} if m is None else {"ctx": np.linspace(-1, 1, m, dtype=np.float32), "z": np.float16(2)}
        req, tg, cx, bs, cbs, keep = _struct(d, ctx, key, grpc_frame)
        rc, size = _size(req, tg, cx)
        assert rc == N.OK, N.last_error()
        ref = _ref(d, ctx, key, grpc_frame)
        assert size == len(ref), m
        ctx_len = len(examples_with_context_from_input_dict(d, ctx).example_list_with_context.context.SerializeToString())
        sizes.add(ctx_len)
    assert min(sizes) <= 127 and max(s for s in sizes if s < 1000) >= 128
    assert min(s for s in sizes if s > 1000) <= 16383 and max(sizes) >= 16384
    # no examples at all
    req, tg, cx, bs, cbs, keep = _struct({}, {"c": np.ones(3, np.float32)}, key, grpc_frame)
    assert _size(req, tg, cx) == (N.OK, len(_ref({}, {"c": np.ones(3, np.float32)}, key, grpc_frame)))
    # an integer context has a length that depends on its values
    req, tg, cx, bs, cbs, keep = _struct(d, {"i": np.arange(3)}, key, grpc_frame)
    assert _size(req, tg, cx)[0] == N.E_ARG


@pytest.mark.parametrize("key", [None, "elwc"])
def test_context_arena_bound(key):
    """the arena slot holds every request at its worst case: negative int64s (ten bytes each) and long strings"""
    rng = np.random.default_rng(7)
    lib = N.load()
    for trial in range(40):
        n = int(rng.integers(0, 5))
        d = {"f": rng.standard_normal((n, 3)).astype(np.float32), "i": rng.integers(-2 ** 63, 0, (n, 2), dtype=np.int64)}
        ctx = {}
        for k in range(int(rng.integers(0, 4))):
            kind = rng.integers(0, 3)
            m = int(rng.integers(0, 40))
            if kind == 0:
                ctx[f"i{k}"] = rng.integers(-2 ** 63, -2 ** 62, m, dtype=np.int64)
            elif kind == 1:
                ctx[f"s{k}"] = _column([bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)) for _ in range(m)])
            else:
                ctx[f"b{k}"] = rng.integers(0, 2, m).astype(bool)
        req, tg, cx, bs, cbs, keep = _struct(d, ctx, key)
        out = C.c_uint64()
        assert lib.b200tfs_example_context_arena_size(1, C.byref(req), bs, C.byref(tg) if tg is not None else None, C.byref(cx),
                                                      cbs, C.byref(out)) == N.OK, N.last_error()
        # the slot starts at 0; the record ends at most at its end
        assert out.value >= len(_ref(d, ctx, key)), trial
