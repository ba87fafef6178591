"""ModelSpec.signature_name, ModelSpec.version_label and PredictRequest.output_filter on every PredictRequest route the GPU encodes,
bit for bit against the protobuf runtime: the route's bytes without the fields (checked elsewhere against the reference), parsed,
given the fields and serialised with deterministic=True."""
import ctypes as C

import numpy as np
import pytest

from devutil import Dev, tensor_struct
from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, _RequestSpec
from oracle import wire_oracle
from tensorflow_serving.apis import predict_pb2

pytestmark = pytest.mark.gpu

SPECS = [dict(signature_name="predict"), dict(version_label="canary"), dict(output_filter=["scores", "ids", "scores"]),
         dict(signature_name="sigé" * 40, version_label="", output_filter=[""] + ["out%d" % i for i in range(300)])]


def with_fields(base, grpc=False, signature_name=None, version_label=None, output_filter=None):
    body = bytes(base)[5:] if grpc else bytes(base)
    m = predict_pb2.PredictRequest.FromString(body)
    assert m.SerializeToString(deterministic=True) == body
    if signature_name is not None:
        m.model_spec.signature_name = signature_name
    if version_label is not None:
        m.model_spec.version_label = version_label
    if output_filter is not None:
        m.output_filter.extend(output_filter)
    out = m.SerializeToString(deterministic=True)
    return b"\x00" + len(out).to_bytes(4, "big") + out if grpc else out


def _batch(rng, n, version=3):
    return [("model", version if i % 2 else None, {"image": rng.standard_normal((3, 8, 8)).astype(np.float32),
                                                   "ids": rng.integers(-50, 2 ** 40, 5 + i),
                                                   "words": np.array(["a", "bé"][: 1 + i % 2])}) for i in range(n)]


@pytest.mark.parametrize("kw", SPECS)
@pytest.mark.parametrize("grpc", [False, True])
def test_encode_predict_requests(codec, kw, grpc):
    rng = np.random.default_rng(1)
    one = [("model", None, {"x": rng.standard_normal(100).astype(np.float32)})]      # the single-request closed-form path
    batch = _batch(rng, 9, None if "version_label" in kw else 3)
    for reqs in (one, batch):
        base = codec.encode_predict_requests(reqs, grpc_frame=grpc)
        got = codec.encode_predict_requests(reqs, grpc_frame=grpc, **kw)
        assert got == [with_fields(b, grpc, **kw) for b in base]
        pinned = codec.encode_predict_requests(reqs, grpc_frame=grpc, out="pinned", **kw)
        assert [bytes(p) for p in pinned] == got
    assert codec.encode_predict_request("model", one[0][2], None, **kw) == with_fields(codec.encode_predict_request("model", one[0][2]), **kw)


def test_pipelined_request(codec):
    """a request above the pipelining threshold: the output_filter run is framing, written with slice 0, behind the last slice"""
    rng = np.random.default_rng(2)
    inputs = {"a": rng.standard_normal(1 << 20).astype(np.float32), "b": rng.standard_normal(300000).astype(np.float32)}
    kw = dict(signature_name="serving_default", output_filter=["y", "x"])
    N.check(codec._lib.b200tfs_set_pipeline(codec._ctx, 1 << 18, 4))
    try:
        before = C.c_uint64()
        N.check(codec._lib.b200tfs_pipelined_calls(codec._ctx, C.byref(before)))
        for out in (None, "pinned"):
            got = codec.encode_predict_requests([("m", 1, inputs)], out=out, **kw)
            assert bytes(got[0]) == with_fields(wire_oracle.encode_predict_request("m", 1, list(inputs.items())), **kw)
        after = C.c_uint64()
        N.check(codec._lib.b200tfs_pipelined_calls(codec._ctx, C.byref(after)))
        assert after.value > before.value
    finally:
        N.check(codec._lib.b200tfs_set_pipeline(codec._ctx, 1 << 20, 8))


def _device_requests(dev, batch):
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
                              version=version or 0, n_inputs=len(ts), flags=0, inputs=arr))
    return (N.Request * len(reqs))(*reqs), keep, ptrs


def _deferred_batch(rng, scale):
    return [("m", None, [("label", np.array([7 * scale], np.int64)), ("toks", rng.integers(0, 5000, 40 + i) * scale),
                         ("big", rng.integers(0, 2 ** 40, 6000) // scale), ("x", rng.standard_normal(9).astype(np.float32))])
            for i in range(6)]


def test_deferred_encode_and_graph_replay():
    """b200tfs_encode_requests_async_spec: frame_requests_kernel places the output_filter run behind payloads whose lengths the
    device counts; a replay with values of other varint lengths moves it and the bytes still match"""
    dev = Dev()
    try:
        rng = np.random.default_rng(4)
        batch = _deferred_batch(rng, 1)
        rq, keep, ptrs = _device_requests(dev, batch)
        n = len(batch)
        kws = [dict(signature_name="sig%d" % i, version_label="canary" if i % 2 else None, output_filter=["o"] * i) for i in range(n)]
        specs_py = [_RequestSpec.of([None], **kw) for kw in kws]
        specs = (N.RequestSpec * n)(*[s.struct for s in specs_py])
        need = C.c_uint64()
        N.check(dev.lib.b200tfs_request_arena_size_spec(n, rq, specs, C.byref(need)))
        arena = dev.malloc(need.value)

        def check(b):
            off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
            N.check(dev.lib.b200tfs_encode_results(dev.ctx, n, off, ln))
            whole = dev.download(arena, need.value)
            for i, (model, version, inputs) in enumerate(b):
                want = with_fields(wire_oracle.encode_predict_request(model, version, inputs), **kws[i])
                assert whole[off[i]: off[i] + ln[i]].tobytes() == want, i
            return [int(x) for x in ln]

        N.check(dev.lib.b200tfs_encode_requests_async_spec(dev.ctx, n, rq, specs, arena, need.value))
        lens1 = check(batch)
        N.check(dev.lib.b200tfs_capture_begin(dev.ctx))
        N.check(dev.lib.b200tfs_encode_requests_async_spec(dev.ctx, n, rq, specs, arena, need.value))
        g = C.c_void_p()
        N.check(dev.lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        batch2 = _deferred_batch(rng, 300)
        k = 0
        for _, _, inputs in batch2:
            for _, a in inputs:
                p, old = ptrs[k]
                k += 1
                assert old.shape == a.shape and old.dtype == a.dtype
                N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, p, np.ascontiguousarray(a).ctypes.data, a.nbytes))
        dev.sync()
        N.check(dev.lib.b200tfs_graph_launch(dev.ctx, g))
        lens2 = check(batch2)
        assert lens1 != lens2
        N.check(dev.lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


@pytest.mark.parametrize("kw", SPECS)
def test_padded_encode(codec, kw):
    rng = np.random.default_rng(6)
    n, R = 12, 64
    P = rng.standard_normal((R, 8)).astype(np.float32)
    ids = rng.integers(-9, 2 ** 35, (R, 5))
    rows = rng.multinomial(R - 5, np.ones(n) / n)
    S = np.stack([rows, rng.integers(0, 9, n)], 1).astype(np.int64)
    strs = np.array(["w%d" % (i * 7) for i in range(R * 2)]).reshape(R, 2)
    col = BytesColumn.from_array(strs)
    version = None if "version_label" in kw else 3
    inputs = {"p": P, "ids": ids, "s": col}
    shapes = {"p": S, "ids": S[:, 0].copy(), "s": S[:, 0].copy()}
    base = codec.encode_predict_requests_padded("model", inputs, shapes, model_version=version)
    calls = codec.padded_encode_device_calls
    got = codec.encode_predict_requests_padded("model", inputs, shapes, model_version=version, **kw)
    assert codec.padded_encode_device_calls == calls + 1
    assert got == [with_fields(b, **kw) for b in base]
    # device shapes and device tensors
    import torch

    dev_in = {"p": torch.from_numpy(P).cuda(), "ids": torch.from_numpy(ids).cuda(), "s": col}
    dev_sh = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in shapes.items()}
    assert codec.encode_predict_requests_padded("model", dev_in, dev_sh, model_version=version, **kw) == got


def test_padded_graph_replay_moves_the_filter(codec):
    """b200tfs_encode_padded_requests_columns_async_spec captured once, replayed with new shapes: each record's output_filter
    run follows its new last payload"""
    dev = Dev()
    try:
        rng = np.random.default_rng(8)
        n, R = 16, 128
        P = rng.standard_normal((R, 4, 3)).astype(np.float32)
        ids = rng.integers(0, 2 ** 30, (R, 6))

        def shapes():
            rows = rng.multinomial(R - 3, np.ones(n) / n)
            return np.stack([rows, rng.integers(0, 5, n), rng.integers(0, 4, n)], 1).astype(np.int64)

        S = shapes()
        pP, pI, pS, pS2 = dev.upload(P), dev.upload(ids), dev.upload(S), dev.upload(np.ascontiguousarray(S[:, :1]))
        ts, keep = [], []
        for k, p, a in (("x", pP, P), ("ids", pI, ids)):
            t, dims = tensor_struct(p, a, key=k.encode())
            ts.append(t)
            keep.append(dims)
        arr = (N.Tensor * 2)(*ts)
        pins = (N.PadInput * 2)(N.PadInput(shapes=pS, cols=3), N.PadInput(shapes=pS2, cols=1))
        req = N.Request(model_name=b"model", model_name_len=5, has_version=0, order=N.ORDER_UPB, version=0, n_inputs=2, flags=0,
                        inputs=arr)
        kw = dict(signature_name="classify", version_label="stable", output_filter=["probs", "classes"])
        spec = _RequestSpec.of([None], **kw)
        cap = C.c_uint64()
        N.check(dev.lib.b200tfs_padded_request_columns_arena_size_spec(n, C.byref(req), None, C.byref(spec.struct), C.byref(cap)))
        arena = (dev.malloc(cap.value + 256) + 255) & ~255

        def run(graph=None):
            if graph is None:
                N.check(dev.lib.b200tfs_encode_padded_requests_columns_async_spec(dev.ctx, n, C.byref(req), pins, None,
                                                                                   C.byref(spec.struct), arena, cap.value))
            else:
                N.check(dev.lib.b200tfs_graph_launch(dev.ctx, graph))
            off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
            N.check(dev.lib.b200tfs_encode_results(dev.ctx, n, off, ln))
            wire = dev.download(arena, cap.value)
            return [wire[off[r]: off[r] + ln[r]].tobytes() for r in range(n)]

        def want(P, ids, S):
            base = codec.encode_predict_requests_padded("model", {"x": P, "ids": ids}, {"x": S, "ids": S[:, 0].copy()})
            return [with_fields(b, **kw) for b in base]

        assert run() == want(P, ids, S)
        N.check(dev.lib.b200tfs_capture_begin(dev.ctx))
        run_capture = dev.lib.b200tfs_encode_padded_requests_columns_async_spec(dev.ctx, n, C.byref(req), pins, None,
                                                                                C.byref(spec.struct), arena, cap.value)
        g = C.c_void_p()
        N.check(dev.lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        N.check(run_capture)
        S2 = shapes()
        ids2 = rng.integers(-2 ** 40, 2 ** 40, ids.shape)
        for ptr, a in ((pS, S2), (pS2, np.ascontiguousarray(S2[:, :1])), (pI, ids2)):
            N.check(dev.lib.b200tfs_memcpy_h2d(dev.ctx, ptr, a.ctypes.data, a.nbytes))
        dev.sync()
        assert run(g.value) == want(P, ids2, S2)
        N.check(dev.lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


def test_host_assembled_padded_route(codec):
    """numpy str inputs make the padded encode cut boxes on the host: the fields ride along"""
    strs = np.array([["a", "b"], ["cé", "d"], ["e", "f"]])
    kw = dict(signature_name="s", output_filter=["z"])
    base = codec.encode_predict_requests_padded("m", {"w": strs}, {"w": np.array([1, 2])})
    calls = codec.padded_encode_device_calls
    got = codec.encode_predict_requests_padded("m", {"w": strs}, {"w": np.array([1, 2])}, **kw)
    assert codec.padded_encode_device_calls == calls
    assert got == [with_fields(b, **kw) for b in base]


def test_errors(codec):
    x = {"x": np.zeros(3, np.float32)}
    with pytest.raises(ValueError, match="oneof"):
        codec.encode_predict_requests([("m", 1, x)], version_label="canary")
    with pytest.raises(ValueError, match="oneof"):
        codec.encode_predict_requests_padded("m", {"x": np.zeros((2, 3), np.float32)}, {"x": np.array([1, 1])}, model_version=0,
                                             version_label="")
    with pytest.raises(ValueError, match="UTF-8"):
        codec.encode_predict_request("m", x, signature_name=b"\xff")
    with pytest.raises(ValueError, match="UTF-8"):
        codec.encode_predict_request("m", x, output_filter=[b"\xc3\x28"])


def test_client_round_trip():
    """TensorServingClient.predict_request with the fields, against a servicer that honours output_filter and echoes the
    signature: the bytes it received, and the spec the GPU decode returns"""
    import grpc  # noqa: F401

    from fake_server import IdentityServer
    from min_tfs_client.codec import get_codec
    from min_tfs_client.requests import TensorServingClient

    class FilteringServer(IdentityServer):
        def _predict(self, request_bytes, context):
            self.received.append(request_bytes)
            req = predict_pb2.PredictRequest.FromString(request_bytes)
            resp = predict_pb2.PredictResponse()
            for key, proto in req.inputs.items():
                out = key[: -len("_input")] + "_output" if key.endswith("_input") else key
                if not req.output_filter or out in req.output_filter:
                    resp.outputs[out].CopyFrom(proto)
            resp.model_spec.name = req.model_spec.name
            resp.model_spec.version.value = 7
            resp.model_spec.signature_name = req.model_spec.signature_name or "serving_default"
            return resp.SerializeToString()

    srv = FilteringServer()
    try:
        client = TensorServingClient("127.0.0.1", srv.port)
        rng = np.random.default_rng(9)
        inputs = {"a_input": rng.standard_normal(16).astype(np.float32), "b_input": np.arange(5, dtype=np.int64)}
        resp = client.predict_request("m", inputs, signature_name="embed", version_label="canary", output_filter=["b_output"])
        base = get_codec().encode_predict_request("m", inputs)
        assert srv.received[-1] == with_fields(base, signature_name="embed", version_label="canary", output_filter=["b_output"])
        outs, spec = get_codec().decode_predict_response(resp.SerializeToString())
        assert list(outs) == ["b_output"] and (outs["b_output"] == inputs["b_input"]).all()
        assert spec.signature_name == "embed" and spec.version == 7
        plain = client.predict_request("m", inputs)
        assert srv.received[-1] == base and set(plain.outputs) == {"a_output", "b_output"}
    finally:
        srv.server.stop(0)


def test_sharded_codec_forwards_the_keywords():
    from min_tfs_client.sharding import ShardedCodec

    rng = np.random.default_rng(10)
    reqs = _batch(rng, 7, None)
    kw = dict(signature_name="score", version_label="stable", output_filter=["y"])
    with ShardedCodec([0, 0]) as sc:     # two shards on one GPU: the keywords must reach both
        got = sc.encode_predict_requests(reqs, **kw)
    from min_tfs_client.codec import get_codec

    assert got == [with_fields(b, **kw) for b in get_codec().encode_predict_requests(reqs)]


# ---- the tf.Example family ---------------------------------------------------------------------------------------------------
def msg_with_fields(base, cls, grpc=False, signature_name=None, version_label=None, output_filter=None):
    """protobuf's bytes of `base` (a message of class `cls`) with the fields set; a MultiInferenceRequest's label goes into every
    task's model_spec"""
    body = bytes(base)[5:] if grpc else bytes(base)
    m = cls.FromString(body)
    assert m.SerializeToString(deterministic=True) == body
    specs = [t.model_spec for t in m.tasks] if cls.DESCRIPTOR.name == "MultiInferenceRequest" else [m.model_spec]
    for s in specs:
        if signature_name is not None:
            s.signature_name = signature_name
        if version_label is not None:
            s.version_label = version_label
    if output_filter is not None:
        m.output_filter.extend(output_filter)
    out = m.SerializeToString(deterministic=True)
    return b"\x00" + len(out).to_bytes(4, "big") + out if grpc else out


def _columns(rng, n):
    from min_tfs_client.codec import RaggedColumn

    return {"dense": rng.standard_normal((n, 3)).astype(np.float32), "ids": rng.integers(-5, 2 ** 40, (n, 4)),
            "rag": RaggedColumn(rng.standard_normal((n, 5)).astype(np.float32), rng.integers(0, 6, n)),
            "words": BytesColumn.from_array(np.array([["w%d" % i, "é" * (i % 4)] for i in range(n)]))}


@pytest.mark.parametrize("grpc", [False, True])
def test_classify_and_regress(codec, grpc):
    from tensorflow_serving.apis import classification_pb2

    rng = np.random.default_rng(11)
    reqs = [("model", None, _columns(rng, 7)), ("model", None, {"x": rng.standard_normal((4, 2)).astype(np.float32)})]
    for kw in (dict(signature_name="classification"), dict(version_label="canary"), dict(signature_name="regression", version_label="")):
        base = codec.encode_example_requests(reqs, grpc_frame=grpc)
        got = codec.encode_example_requests(reqs, grpc_frame=grpc, **kw)
        assert got == [msg_with_fields(b, classification_pb2.ClassificationRequest, grpc, **kw) for b in base]


@pytest.mark.parametrize("grpc", [False, True])
def test_predict_examples_and_elwc_with_a_filter(codec, grpc):
    rng = np.random.default_rng(12)
    ctx = {"user": rng.standard_normal(4).astype(np.float32), "uid": np.array([123456789])}
    reqs = [("model", None, _columns(rng, 9)), ("model", None, _columns(rng, 3), ctx),
            ("model", None, {"x": np.zeros((0, 3), np.float32)})]
    for kw in (dict(output_filter=["scores", "", "scores"]), dict(signature_name="predict", version_label="stable", output_filter=["p"] * 200)):
        base = codec.encode_example_requests(reqs, grpc_frame=grpc, predict_input="examples")
        got = codec.encode_example_requests(reqs, grpc_frame=grpc, predict_input="examples", **kw)
        assert got == [with_fields(b, grpc, **kw) for b in base]


def test_sequence_examples_with_a_filter(codec):
    from min_tfs_client.codec import RaggedColumn

    rng = np.random.default_rng(13)
    n = 6
    ctx = {"user": rng.standard_normal((n, 2)).astype(np.float32)}
    fl = {"clicks": RaggedColumn(rng.integers(0, 2 ** 33, (n, 5, 2)), rng.integers(0, 6, n)),
          "dwell": rng.standard_normal((n, 5)).astype(np.float32)}
    kw = dict(signature_name="serving_default", version_label="canary", output_filter=["logits", "probs"])
    base = codec.encode_sequence_example_requests([("m", None, ctx, fl)] * 2, input_key="seq")
    got = codec.encode_sequence_example_requests([("m", None, ctx, fl)] * 2, input_key="seq", **kw)
    assert got == [with_fields(b, **kw) for b in base]


def test_multi_inference_label_and_task_signatures(codec):
    from min_tfs_client.requests import CLASSIFY_METHOD_NAME, REGRESS_METHOD_NAME, make_multi_inference_request
    from tensorflow_serving.apis import inference_pb2

    rng = np.random.default_rng(14)
    d = {"x": rng.standard_normal((5, 3)).astype(np.float32), "k": rng.integers(0, 99, (5, 1))}
    tasks = [("head_a", CLASSIFY_METHOD_NAME), ("head_b", REGRESS_METHOD_NAME), ("", CLASSIFY_METHOD_NAME)]
    got = codec.encode_example_requests([("m", None, d)], tasks=tasks, version_label="canary")[0]
    base = codec.encode_example_requests([("m", None, d)], tasks=tasks)[0]
    assert got == msg_with_fields(base, inference_pb2.MultiInferenceRequest, version_label="canary")
    ref = make_multi_inference_request("m", None, tasks, d, version_label="canary").SerializeToString(deterministic=True)
    assert got == ref
    # each task's model_spec: name, the task's signature, then the label
    assert bytes.fromhex("0a016d1a06686561645f61220663616e617279") in got
    assert bytes.fromhex("0a016d1a06686561645f62220663616e617279") in got
    with pytest.raises(ValueError, match="per task"):
        codec.encode_example_requests([("m", None, d)], tasks=tasks, signature_name="s")
    with pytest.raises(ValueError, match="PredictRequest"):
        codec.encode_example_requests([("m", None, d)], tasks=tasks, output_filter=["y"])
    with pytest.raises(ValueError, match="per task"):
        make_multi_inference_request("m", None, tasks, d, signature_name="s")


def test_example_errors(codec):
    d = {"x": np.zeros((2, 2), np.float32)}
    with pytest.raises(ValueError, match="PredictRequest"):
        codec.encode_example_requests([("m", None, d)], output_filter=["y"])
    with pytest.raises(ValueError, match="oneof"):
        codec.encode_example_requests([("m", 3, d)], version_label="canary")
    with pytest.raises(ValueError, match="UTF-8"):
        codec.encode_example_requests([("m", None, d)], signature_name=b"\xfe")
    with pytest.raises(ValueError, match="oneof"):
        codec.encode_sequence_example_requests([("m", 1, {}, {"f": np.zeros((2, 3), np.float32)})], input_key="s", version_label="")


def test_host_assembled_example_routes(codec):
    """numpy str columns make the example encodes assemble the request with protobuf on the host: the fields ride along"""
    from tensorflow_serving.apis import classification_pb2

    d = {"w": np.array([["a"], ["bé"]]), "x": np.ones((2, 1), np.float32)}
    kw = dict(signature_name="s", version_label="v")
    got = codec.encode_example_requests([("m", None, d)], **kw)[0]
    assert got == msg_with_fields(codec.encode_example_requests([("m", None, d)])[0], classification_pb2.ClassificationRequest, **kw)
    got = codec.encode_example_requests([("m", None, d)], predict_input="ex", output_filter=["o"], **kw)[0]
    assert got == with_fields(codec.encode_example_requests([("m", None, d)], predict_input="ex")[0], output_filter=["o"], **kw)
    fl = {"f": np.array([[["a"], ["b"]]])}
    got = codec.encode_sequence_example_requests([("m", None, {}, fl)], input_key="s", output_filter=["o"])[0]
    assert got == with_fields(codec.encode_sequence_example_requests([("m", None, {}, fl)], input_key="s")[0], output_filter=["o"])


def test_client_example_methods_send_the_fields():
    """what the server receives from classification_request, regression_request, predict_examples_request and
    predict_sequence_examples_request with the fields, and what the MultiInference serializer writes"""
    from fake_server import IdentityServer
    from min_tfs_client.codec import get_codec
    from min_tfs_client.requests import (CLASSIFY_METHOD_NAME, SpecFields, TensorServingClient, gpu_multi_inference_request_serializer,
                                         make_multi_inference_request)
    from tensorflow_serving.apis import classification_pb2, regression_pb2

    srv = IdentityServer()
    try:
        client = TensorServingClient("127.0.0.1", srv.port)
        d = {"a": np.arange(6, dtype=np.float32).reshape(3, 2)}
        client.classification_request("m", d, signature_name="classification", version_label="canary")
        m = classification_pb2.ClassificationRequest.FromString(srv.received[-1])
        assert (m.model_spec.signature_name, m.model_spec.version_label) == ("classification", "canary")
        client.regression_request("m", d, signature_name="regression")
        assert regression_pb2.RegressionRequest.FromString(srv.received[-1]).model_spec.signature_name == "regression"
        kw = dict(signature_name="predict", version_label="stable", output_filter=["examples"])
        client.predict_examples_request("m", d, **kw)
        assert srv.received[-1] == with_fields(get_codec().encode_example_requests([("m", None, d)], predict_input="examples")[0], **kw)
        fl = {"f": np.ones((2, 3), np.float32)}
        client.predict_sequence_examples_request("m", {}, fl, "seq", **kw)
        assert srv.received[-1] == with_fields(get_codec().encode_sequence_example_requests([("m", None, {}, fl)], input_key="seq")[0],
                                               **kw)
        tasks = [("a", CLASSIFY_METHOD_NAME)]
        wire = gpu_multi_inference_request_serializer(("m", None, tasks, d, None, SpecFields(version_label="canary")))
        assert wire == make_multi_inference_request("m", None, tasks, d, version_label="canary").SerializeToString(deterministic=True)
    finally:
        srv.server.stop(0)
