"""MultiInference on the GPU: MultiInferenceRequests encoded by the tf.Example request kernels (bytes compared with the protobuf
runtime's deterministic serialization of make_multi_inference_request), and batches of MultiInferenceResponses decoded by
mi_index_kernel and the Classify / Regress kernels (compared bit for bit with the definition in multi_inference_corpus)."""
import ctypes as C

import numpy as np
import pytest

import multi_inference_corpus as M
from devutil import Dev
from example_response_corpus import I32, LEN, f32, serialize
from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn
from min_tfs_client.requests import CLASSIFY_METHOD_NAME, REGRESS_METHOD_NAME, make_multi_inference_request

pytestmark = pytest.mark.gpu

CN, RN = CLASSIFY_METHOD_NAME, REGRESS_METHOD_NAME
METHOD = {M.CLASSIFY: CN, M.REGRESS: RN}
TASKS = [("head_c", CN), ("", RN)]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _host(v):
    if isinstance(v, RaggedColumn):
        return RaggedColumn(_host(v.values), _host(v.lengths))
    if isinstance(v, BytesColumn):
        return BytesColumn(_host(v.data), _host(v.offsets), v.shape)
    return v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)


def ref(name, version, tasks, d, ctx=None, grpc_frame=False):
    hd = {k: _host(v) for k, v in d.items()}
    hc = None if ctx is None else {k: _host(v) for k, v in ctx.items()}
    w = make_multi_inference_request(name, version, tasks, hd, hc).SerializeToString(deterministic=True)
    return (b"\x00" + len(w).to_bytes(4, "big") + w) if grpc_frame else w


# ---- encode ----------------------------------------------------------------------------------------------------------------
DTYPES = [np.float32, np.float64, np.float16, np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.bool_]


@pytest.mark.parametrize("dtype", DTYPES, ids=[np.dtype(t).name for t in DTYPES])
def test_every_dtype(codec, dtype):
    rng = np.random.default_rng(1)
    a = (rng.standard_normal((9, 3)) * 1000).astype(dtype) if np.dtype(dtype).kind == "f" else \
        rng.integers(0, 2, (9, 3)).astype(dtype) if dtype is np.bool_ else \
        rng.integers(np.iinfo(dtype).min, np.iinfo(dtype).max, (9, 3), dtype=dtype, endpoint=True)
    d = {"a": a, "f": rng.standard_normal((9, 2)).astype(np.float32)}
    for tasks in (TASKS, [("s", RN)], [("x", CN), ("y", RN), ("z", CN), ("", RN)]):
        assert codec.encode_example_requests([("m", 5, d)], tasks=tasks) == [ref("m", 5, tasks, d)]


def test_ragged_bytes_broadcast_and_context(codec):
    rng = np.random.default_rng(2)
    n = 12
    d = {"r": RaggedColumn(rng.standard_normal((n, 4)).astype(np.float32), rng.integers(0, 5, n)),
         "ids": RaggedColumn(rng.integers(-(1 << 40), 1 << 40, (n, 3)), rng.integers(0, 4, n)),
         "b": BytesColumn.from_array(np.array([f"s{i}-".encode() + b"x" * (i % 5) for i in range(n * 2)]).reshape(n, 2)),
         "w": np.float32(0.5), "k": np.int64(7)}
    ctx = {"q": rng.standard_normal(6).astype(np.float32), "h": rng.integers(0, 1 << 30, 9),
           "s": BytesColumn.from_array(np.array([b"query", b"", "ü".encode()]))}
    for c in (None, ctx, {}):
        for ver in (None, 0, 123456789012):
            assert codec.encode_example_requests([("model", ver, d, c)], tasks=TASKS) == [ref("model", ver, TASKS, d, c)]


def test_order_given_grpc_frame_and_host_route(codec):
    rng = np.random.default_rng(3)
    d = {"z": rng.standard_normal((5, 2)).astype(np.float32), "a": rng.integers(0, 9, (5, 1))}
    got = codec.encode_example_requests([("m", 1, d)], tasks=TASKS, grpc_frame=True)[0]
    assert got == ref("m", 1, TASKS, d, grpc_frame=True)
    given = codec.encode_example_requests([("m", 1, d)], tasks=TASKS, order="given")[0]
    from tensorflow_serving.apis.inference_pb2 import MultiInferenceRequest
    assert MultiInferenceRequest.FromString(given) == make_multi_inference_request("m", 1, TASKS, d)
    assert given.index(b"\x0a\x01z") < given.index(b"\x0a\x01a")       # the first example's map entries, in insertion order
    s = {"t": np.array(["a", "bc", "d", "e", "f"]), "x": d["z"]}      # a numpy str column: the host route
    assert codec.encode_example_requests([("m", 1, s)], tasks=TASKS) == [ref("m", 1, TASKS, s)]
    with pytest.raises(ValueError):
        codec.encode_example_requests([("m", 1, d)], tasks=TASKS, predict_input="examples")
    with pytest.raises(ValueError):
        codec.encode_example_requests([("m", 1, d)], tasks=[("s", "tensorflow/serving/predict")])
    with pytest.raises(ValueError):
        codec.encode_example_requests([("m", 1, d)], tasks=[])


def test_torch_cuda_column(codec):
    torch = pytest.importorskip("torch")
    x = torch.randn(30, 8, device="cuda")
    ids = torch.arange(30, device="cuda", dtype=torch.int64) * 1000
    d = {"x": x, "ids": ids}
    assert codec.encode_example_requests([("m", 2, d)], tasks=TASKS) == [ref("m", 2, TASKS, d)]


def _int_req(lib_keep, dptr, n, m):
    fa = (N.Feature * 1)(N.Feature(data=dptr, src_dtype=9, flags=N.F_DEVICE_DATA, row_elems=m, key=b"ids", key_len=3))
    lib_keep.append(fa)
    return N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_examples=n,
                            n_features=1, flags=0, features=fa)


def _tasks_struct(keep, tasks):
    sigs = [s.encode() for s, _ in tasks]
    arr = (N.InferenceTask * len(tasks))(*[N.InferenceTask(signature_name=s, signature_len=len(s),
                                                             method=N.RESP_CLASSIFY if m == CN else N.RESP_REGRESS)
                                             for s, (_, m) in zip(sigs, tasks)])
    keep += [arr, sigs]
    return N.ExampleTasks(tasks=C.addressof(arr), n_tasks=len(tasks))


def test_graph_replay_over_new_values_and_lengths():
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(4)
        n, m = 60, 5
        keep = []
        a = rng.integers(0, 100, (n, m))
        da = dev.upload(a)
        req = _int_req(keep, da, n, m)
        tk = _tasks_struct(keep, TASKS)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_tasks_arena_size(1, C.byref(req), None, None, None, None, C.byref(tk), C.byref(cap)))
        arena = (dev.malloc(cap.value + 256) + 255) & ~255
        N.check(lib.b200tfs_encode_example_tasks_async(dev.ctx, 1, C.byref(req), None, None, None, None, None, C.byref(tk), arena, cap.value))
        N.check(lib.b200tfs_encode_results(dev.ctx, 1, None, None))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_encode_example_tasks_async(dev.ctx, 1, C.byref(req), None, None, None, None, None, C.byref(tk), arena, cap.value))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        lens = set()
        for rep in range(4):
            a = rng.integers(-(1 << 62), 1 << 62, (n, m)) if rep % 2 else rng.integers(0, 100, (n, m))
            N.check(lib.b200tfs_memcpy_h2d(dev.ctx, da, a.ctypes.data, a.nbytes))
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_encode_results(dev.ctx, 1, off, ln))
            assert dev.download(arena + off[0], ln[0]).tobytes() == ref("m", 3, TASKS, {"ids": a}), rep
            lens.add(ln[0])
        assert len(lens) > 1
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


def test_bad_device_offsets_fail_that_request_only():
    dev = Dev()
    lib = dev.lib
    try:
        n = 10
        keep, reqs, bys = [], [], []
        strs = [f"v{i}".encode() * (i % 3 + 1) for i in range(n)]
        data = np.frombuffer(b"".join(strs), np.uint8)
        offs = np.concatenate([[0], np.cumsum([len(s) for s in strs])]).astype(np.int64)
        bad = offs.copy()
        bad[4] = bad[3] - 1
        dd = dev.upload(data)
        for r in range(3):
            do = dev.upload(bad if r == 1 else offs)
            fa = (N.Feature * 1)(N.Feature(data=dd, src_dtype=7, flags=N.F_DEVICE_DATA, row_elems=1, key=b"s", key_len=1))
            keep.append(fa)
            reqs.append(N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=0, order=N.ORDER_UPB, version=0, n_examples=n,
                                         n_features=1, flags=0, features=fa))
            bys.append(N.Bytes(offsets=do, data_len=len(data), flags=N.F_DEVICE_DATA))
        tk = _tasks_struct(keep, TASKS)
        ra, ba, ta = (N.ExampleRequest * 3)(*reqs), (N.Bytes * 3)(*bys), (N.ExampleTasks * 3)(tk, tk, tk)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_tasks_arena_size(3, ra, ba, None, None, None, ta, C.byref(cap)))
        arena = (dev.malloc(cap.value + 256) + 255) & ~255
        N.check(lib.b200tfs_encode_example_tasks_async(dev.ctx, 3, ra, None, ba, None, None, None, ta, arena, cap.value))
        off, ln = (C.c_uint64 * 3)(), (C.c_uint64 * 3)()
        assert lib.b200tfs_encode_results(dev.ctx, 3, off, ln) == N.E_SHAPE
        assert off[1] == 0 and ln[1] == 0
        want = ref("m", None, TASKS, {"s": BytesColumn(data, offs, (n, 1))})
        for r in (0, 2):
            assert dev.download(arena + off[r], ln[r]).tobytes() == want, r
    finally:
        dev.close()


# ---- decode ----------------------------------------------------------------------------------------------------------------
def _check(codec, kinds, wires, **kw):
    calls = codec.multi_inference_device_calls
    ref_ = M.expected(kinds, wires)
    got = codec.decode_multi_inference_responses(wires, [METHOD[k] for k in kinds], **kw)
    assert len(got) == len(kinds)
    for k, g, (vals, labels, counts, specs) in zip(kinds, got, ref_):
        v = g.values if k == M.REGRESS else g.scores
        host = v.copy_to_host() if hasattr(v, "copy_to_host") else np.asarray(v.cpu() if hasattr(v, "cpu") else v)
        assert host.shape == vals.shape and np.array_equal(_bits(host), _bits(vals))
        assert g.counts.tolist() == counts
        assert [(s.name, s.signature_name, s.has_version, s.version) for s in g.specs] == \
            [(s.name, s.signature_name, s.HasField("version"), s.version.value) for s in specs]
        if k == M.CLASSIFY:
            assert g.labels() == labels
            same = all(r == labels[0] for r in labels)
            assert g.class_labels == ((list(labels[0]) if labels else []) if same else None)
    assert codec.multi_inference_device_calls == calls + 1, "the device route did not finish"
    return got


KINDS = [[M.CLASSIFY], [M.REGRESS], [M.CLASSIFY, M.REGRESS], [M.REGRESS, M.CLASSIFY, M.REGRESS],
         [M.CLASSIFY, M.CLASSIFY, M.REGRESS, M.CLASSIFY]]


@pytest.mark.parametrize("kinds", KINDS, ids=["-".join("cr"[k == M.REGRESS] for k in ks) for ks in KINDS])
def test_batches(codec, kinds):
    rng = np.random.default_rng(len(kinds))
    for n, rows in ((1, 1), (5, 0), (64, 17), (200, 3)):
        _check(codec, kinds, [M.random_response(rng, kinds, rows) for _ in range(n)])
    _check(codec, kinds, [M.random_response(rng, kinds, 4, labels=lambda i: [f"l{i}", "b", ""]) for _ in range(9)])


def test_every_float_pattern_as_value_and_score(codec):
    pats = [0, 0x80000000, 0x7F800001, 0xFFA00000, 0x7FC00000, 0x7F800000, 0xFF800000, 1, 0x807FFFFF, 0x3F800000]
    rng = np.random.default_rng(6)
    pats += rng.integers(0, 1 << 32, 200, dtype=np.uint64).tolist()
    reg = [(1, LEN, [] if b == 0 else [(1, I32, f32(int(b)))]) for b in pats]
    cls = [(1, LEN, [(1, LEN, [(1, LEN, b"a")] + ([] if b == 0 else [(2, I32, f32(int(b)))]))]) for b in pats]
    wire = serialize([M.result(M.REG, reg), M.result(M.CLS, cls)])
    _check(codec, [M.REGRESS, M.CLASSIFY], [wire, wire])


def test_device_and_out(codec):
    from min_tfs_client import device as D
    rng = np.random.default_rng(7)
    kinds = [M.CLASSIFY, M.REGRESS, M.CLASSIFY]
    wires = [M.random_response(rng, kinds, 6) for _ in range(5)]
    got = _check(codec, kinds, wires, device=True)
    assert all(hasattr(g.scores if k == M.CLASSIFY else g.values, "copy_to_host") for k, g in zip(kinds, got))
    pinned = codec.pinned_empty((40,), np.float32)
    dev_out = D.DeviceArray(codec, (30, 2), np.float32)       # cannot be sliced: exactly the rows
    got = _check(codec, kinds, wires, out=[dev_out, pinned, None])
    assert np.shares_memory(np.asarray(got[1].values), pinned)
    with pytest.raises(ValueError):
        codec.decode_multi_inference_responses(wires, [CN, RN])          # a result count other than the tasks
    with pytest.raises(ValueError):
        codec.decode_multi_inference_responses(wires, [CN, RN, CN], out=[None])
    with pytest.raises(ValueError):
        codec.decode_multi_inference_responses(wires, [CN, "tensorflow/serving/predict", CN])


def test_edge_cases_and_mutants_match_the_definition(codec):
    from google.protobuf.message import DecodeError

    cases = [(name, kinds, w) for name, kinds, w in M.edge_cases()] + [(f"mutant {i}", k, w) for i, (k, w) in enumerate(M.mutants())]
    finished = 0
    for name, kinds, wire in cases:
        try:
            M.expected(kinds, [wire])
            raised = None
        except (DecodeError, ValueError) as e:
            raised = type(e)
        calls = codec.multi_inference_device_calls
        if raised is None:
            _check(codec, kinds, [wire])
            finished += 1
        else:
            with pytest.raises(raised):
                codec.decode_multi_inference_responses([wire], [METHOD[k] for k in kinds])
            assert codec.multi_inference_device_calls == calls, name
    # batches mixing good responses with one of every outcome
    rng = np.random.default_rng(8)
    for name, kinds, wire in M.edge_cases():
        good = [M.random_response(rng, kinds, 3) for _ in range(3)]
        wires = good[:2] + [wire] + good[2:]
        try:
            M.expected(kinds, wires)
        except (DecodeError, ValueError) as e:
            with pytest.raises(type(e)):
                codec.decode_multi_inference_responses(wires, [METHOD[k] for k in kinds])
            continue
        _check(codec, kinds, wires)
    assert finished > 50


def _blob(wires):
    blob = b"".join(w.ljust((len(w) + 255) & ~255, b"\0") for w in wires)
    offs = np.cumsum([0] + [(len(w) + 255) & ~255 for w in wires[:-1]]).astype(np.uint64)
    return np.frombuffer(blob, np.uint8), (C.c_uint64 * len(wires))(*offs.tolist()), (C.c_uint64 * len(wires))(*[len(w) for w in wires])


def test_stores_stay_inside_the_used_rows_and_the_capacities():
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(9)
        kinds = [M.CLASSIFY, M.REGRESS, M.CLASSIFY]
        wires = [M.random_response(rng, kinds, k, labels=["a", "bb", "c"]) for k in (4, 0, 6)]
        w, off, ln = _blob(wires)
        rows = 10
        used = [rows * 3, rows, rows * 3]
        canary = np.full(64, 0xA5A5A5A5, np.uint32)
        kv = (C.c_int32 * 3)(*kinds)
        per, batch = (C.c_int64 * 27)(), (C.c_int64 * 15)()
        for caps in ((64, 64, 64), (17, 9, 64), (64, 10, 29), (0, 0, 0)):
            vs = [dev.upload(canary) for _ in range(3)]
            ls = [dev.upload(np.tile(canary, 2)) for _ in range(3)]
            vptr = (C.c_void_p * 3)(*[v if c else None for v, c in zip(vs, caps)])
            lptr = (C.c_void_p * 3)(*[lb if c and k == M.CLASSIFY else None for lb, c, k in zip(ls, caps, kinds)])
            vc = (C.c_uint64 * 3)(*caps)
            lc = (C.c_uint64 * 3)(*[c if k == M.CLASSIFY else 0 for c, k in zip(caps, kinds)])
            N.check(lib.b200tfs_decode_multi_inference_responses_host_async(dev.ctx, 3, kv, w.ctypes.data, 3, off, ln, vptr, vc, lptr, lc))
            N.check(lib.b200tfs_multi_inference_response_results(dev.ctx, 3, 3, per, None, batch))
            for t in range(3):
                got_v, got_l = dev.download(vs[t], 256, np.uint32), dev.download(ls[t], 512, np.uint32)
                assert (got_v[min(used[t], caps[t]):] == 0xA5A5A5A5).all(), (caps, t)
                assert (got_l[2 * (min(used[t], caps[t]) if kinds[t] == M.CLASSIFY else 0):] == 0xA5A5A5A5).all(), (caps, t)
                assert batch[5 * t] == rows and (batch[5 * t + 3] == N.OK) == (used[t] <= caps[t]), (caps, t)
    finally:
        dev.close()


def test_graph_replay_over_new_responses_of_the_same_lengths():
    """Responses padded to one length with an unknown field: a captured decode replayed over new rows, class counts and values."""
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(10)
        kinds = [M.CLASSIFY, M.REGRESS]
        target = 4096

        def pad(w):
            k = target - len(w) - 3
            return w + bytes([15 << 3 | 2]) + bytes([0x80 | (k & 0x7F), k >> 7]) + b"\0" * k

        def batch_of(rows, ncls):
            return [pad(M.random_response(rng, kinds, rows, labels=[f"c{j}" for j in range(ncls)])) for _ in range(3)]
        batches = [batch_of(5, 2), batch_of(20, 4), batch_of(0, 3), batch_of(11, 1)]
        w, off, ln = _blob(batches[0])
        arena = dev.malloc(w.nbytes)
        kv = (C.c_int32 * 2)(*kinds)
        vs = [dev.malloc(4 * 4096) for _ in range(2)]
        lb = dev.malloc(8 * 4096)
        vptr, vc = (C.c_void_p * 2)(*vs), (C.c_uint64 * 2)(4096, 4096)
        lptr, lc = (C.c_void_p * 2)(lb, None), (C.c_uint64 * 2)(4096, 0)
        per, batch = (C.c_int64 * 18)(), (C.c_int64 * 10)()
        N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena, w.ctypes.data, w.nbytes))
        N.check(lib.b200tfs_decode_multi_inference_responses(dev.ctx, 2, kv, arena, 3, off, ln, vptr, vc, lptr, lc))
        N.check(lib.b200tfs_multi_inference_response_results(dev.ctx, 3, 2, per, None, batch))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_decode_multi_inference_responses(dev.ctx, 2, kv, arena, 3, off, ln, vptr, vc, lptr, lc))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        for b in batches:
            w, _, _ = _blob(b)
            N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena, w.ctypes.data, w.nbytes))
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_multi_inference_response_results(dev.ctx, 3, 2, per, None, batch))
            ref_ = M.expected(kinds, b)
            for t in range(2):
                vals, labels, counts, _ = ref_[t]
                assert [per[3 * (3 * t + i) + 1] for i in range(3)] == counts and batch[5 * t + 3] == N.OK
                assert np.array_equal(dev.download(vs[t], 4 * vals.size, np.uint32), _bits(vals).ravel())
            assert batch[1] == ref_[0][0].shape[1]
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


def test_grpc_round_trip():
    """a MultiInference servicer over fake_server's toy model (an example's score: the sum of its float features)"""
    from concurrent import futures

    import grpc
    from min_tfs_client.codec import get_codec
    from min_tfs_client.requests import TensorServingClient
    from tensorflow_serving.apis.inference_pb2 import MultiInferenceRequest, MultiInferenceResponse

    received = []

    def multi(request_bytes, context):
        received.append(request_bytes)
        req = MultiInferenceRequest.FromString(request_bytes)
        resp = MultiInferenceResponse()
        for task in req.tasks:
            res = resp.results.add()
            res.model_spec.CopyFrom(task.model_spec)
            for ex in req.input.example_list.examples:
                s = float(sum(sum(f.float_list.value) for f in ex.features.feature.values()))
                if task.method_name == CN:
                    cl = res.classification_result.classifications.add()
                    cl.classes.add(label="positive", score=s)
                    cl.classes.add(label="negative", score=-s)
                else:
                    res.regression_result.regressions.add(value=s)
        return resp.SerializeToString()

    srv = grpc.server(futures.ThreadPoolExecutor(max_workers=2))
    raw = dict(request_deserializer=lambda b: b, response_serializer=lambda b: b)
    srv.add_generic_rpc_handlers((grpc.method_handlers_generic_handler("tensorflow.serving.PredictionService", {
        "MultiInference": grpc.unary_unary_rpc_method_handler(multi, **raw)}),))
    port = srv.add_insecure_port("127.0.0.1:0")
    srv.start()
    try:
        rng = np.random.default_rng(11)
        d = {"x": rng.standard_normal((20, 3)).astype(np.float32), "id": np.arange(20)}
        client = TensorServingClient("127.0.0.1", port)
        resp = client.multi_inference_request("m", d, TASKS, timeout=30, model_version=4)
        assert received == [ref("m", 4, TASKS, d)]
        kinds = [M.CLASSIFY, M.REGRESS]
        wire = resp.SerializeToString()
        got = _check(get_codec(), kinds, [wire, wire])
        assert got[0].scores.shape == (40, 2) and got[0].class_labels == ["positive", "negative"]
        assert got[0].specs[0].signature_name == "head_c" and got[1].specs[0].version == 4
    finally:
        srv.stop(None)
