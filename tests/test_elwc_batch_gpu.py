"""Predict requests carrying a batch of ExampleListWithContexts (PREDICT_ELWCS) encoded on the GPU: every case compares bytes with
make_predict_elwcs_request(...).SerializeToString(deterministic=True) built from host copies of the same columns."""
import ctypes as C

import numpy as np
import pytest

from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn, _example_columns
from min_tfs_client.requests import make_predict_elwcs_request

pytestmark = pytest.mark.gpu


def _host(v):
    if isinstance(v, RaggedColumn):
        return RaggedColumn(_host(v.values), _host(v.lengths))
    if isinstance(v, BytesColumn):
        return BytesColumn(_host(v.data), _host(v.offsets), v.shape)
    return v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)


def _hostd(d):
    return {k: _host(v) for k, v in d.items()}


def _want(ctx, inp, sizes, key="q", version=2, grpc_frame=False, **fields):
    w = make_predict_elwcs_request("m", version, _hostd(ctx), _hostd(inp), sizes, key, **fields).SerializeToString(deterministic=True)
    return (b"\x00" + len(w).to_bytes(4, "big") + w) if grpc_frame else w


def _check(codec, ctx, inp, sizes, key="q", version=2, **kw):
    got = codec.encode_elwc_requests([("m", version, ctx, inp, sizes)], input_key=key, **kw)[0]
    assert got == _want(ctx, inp, sizes, key, version, **kw)
    return got


def _column(strs, shape=None):
    lens = np.array([len(s) for s in strs], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return BytesColumn(np.frombuffer(b"".join(strs) + b"\xEE\xEE", np.uint8), offsets, shape)


def _strings(rng, m, lo=0, hi=12):
    return [bytes(rng.integers(0, 256, int(k), dtype=np.uint8)) for k in rng.integers(lo, hi + 1, m)]


def _every_dtype(rng, n):
    f = rng.standard_normal((n, 3)).astype(np.float32)
    if n:
        f.view(np.uint32)[0, 0] = 0x7F800001
    return {"f32": f, "f64": rng.standard_normal(n) * 1e300, "f16": rng.standard_normal((n, 2)).astype(np.float16),
            "i8": rng.integers(-128, 128, (n, 2)).astype(np.int8), "i16": rng.integers(-2**15, 2**15, n).astype(np.int16),
            "i32": rng.integers(-2**31, 2**31, (n, 2)).astype(np.int32), "i64": rng.integers(-2**63, 2**63 - 1, (n, 3), dtype=np.int64),
            "u8": rng.integers(0, 256, n).astype(np.uint8), "u16": rng.integers(0, 2**16, n).astype(np.uint16),
            "u32": np.full((n, 1), 2**32 - 1, np.uint32), "u64": np.full(n, 2**64 - 1, np.uint64),
            "b": rng.integers(0, 2, (n, 2)).astype(bool)}


@pytest.mark.parametrize("sizes", [[3, 0, 5, 1], [0, 4], [6, 0], [1], []])
def test_every_dtype_both_sides(codec, sizes):
    rng = np.random.default_rng(len(sizes))
    n, Q = sum(sizes), len(sizes)
    inp = _every_dtype(rng, n)
    inp["k"] = np.int64(-9)
    ctx = _every_dtype(rng, Q)
    ctx["z"] = np.float32(2.5)
    _check(codec, ctx, inp, sizes)
    _check(codec, {}, inp, sizes)
    _check(codec, {"z": np.float32(2.5)}, {"x": inp["f32"]}, sizes)


def test_ragged_and_bytes_on_both_sides(codec):
    rng = np.random.default_rng(2)
    sizes = [4, 0, 7, 1, 3]
    n, Q = sum(sizes), len(sizes)
    inp = {"ids": RaggedColumn(rng.integers(0, 1 << 40, (n, 6)), rng.integers(0, 7, n)), "t": _column(_strings(rng, n * 2), (n, 2)),
           "w": RaggedColumn(_column(_strings(rng, n * 3 * 2), (n, 3, 2)), rng.integers(0, 4, n)),
           "x": rng.standard_normal((n, 4)).astype(np.float32), "s": _column([b"same"], ())}
    ctx = {"query": _column(_strings(rng, Q, 0, 40)), "toks": RaggedColumn(rng.integers(-5, 1 << 33, (Q, 9)), rng.integers(0, 10, Q)),
           "words": RaggedColumn(_column(_strings(rng, Q * 5), (Q, 5)), rng.integers(0, 6, Q)),
           "emb": RaggedColumn(rng.standard_normal((Q, 4, 2)).astype(np.float32), rng.integers(0, 5, Q)), "lang": _column([b"en"], ())}
    _check(codec, ctx, inp, sizes)
    _check(codec, {"emb": ctx["emb"]}, {"x": inp["x"]}, sizes)      # a ragged numeric context alone (kExRagged)


def test_q_0_1_and_1024_and_many_requests(codec):
    rng = np.random.default_rng(3)
    items, wants = [], []
    for sizes in ([], [5], list(rng.integers(0, 4, 1024)), [0] * 7, [2] * 33):
        n, Q = int(np.sum(sizes)), len(sizes)
        inp = {"x": rng.standard_normal((n, 2)).astype(np.float32), "i": rng.integers(0, 1 << 30, n)}
        ctx = {"u": rng.standard_normal((Q, 3)).astype(np.float32), "q": _column(_strings(rng, Q))}
        items.append(("m", 2, ctx, inp, sizes))
        wants.append(_want(ctx, inp, sizes))
    assert codec.encode_elwc_requests(items, input_key="q") == wants


@pytest.mark.parametrize("edge", [128, 16384])
def test_elwc_sizes_straddle_varint_edges(codec, edge):
    """one query whose ELWC is tuned by a string context's length to every size around a 1/2/3-byte varint edge of vi(elwc)"""
    rng = np.random.default_rng(edge)
    x = rng.standard_normal((2, 3)).astype(np.float32)
    base = make_predict_elwcs_request("m", 2, {"s": _column([b""])}, {"x": x}, [2], "q").inputs["q"].string_val[0]
    seen = set()
    for k in range(edge - len(base) - 12, edge - len(base) + 4):
        s = make_predict_elwcs_request("m", 2, {"s": _column([b"a" * k])}, {"x": x}, [2], "q").inputs["q"].string_val[0]
        seen.add(len(s))
        _check(codec, {"s": _column([b"a" * k])}, {"x": x}, [2])
    assert min(seen) < edge <= max(seen)
    _check(codec, {"s": np.full((1, edge // 4), 1.0, np.float32)}, {"x": x}, [2])


def test_large_queries_contexts_and_span_boundaries(codec):
    rng = np.random.default_rng(5)
    # a query larger than the 16 KB emit image, a context larger than 16 KB, and many small queries that one span would have held
    sizes = [40, 1, 0, 2, 3, 1, 1, 60]
    n, Q = sum(sizes), len(sizes)
    inp = {"x": rng.standard_normal((n, 200)).astype(np.float32), "i": rng.integers(-1 << 62, 1 << 62, (n, 3))}
    ctx = {"big": rng.standard_normal((Q, 5000)).astype(np.float32), "b": _column(_strings(rng, Q, 0, 20000))}
    _check(codec, ctx, inp, sizes)
    small = [1] * 300
    _check(codec, {"u": rng.standard_normal((300, 2)).astype(np.float32)}, {"x": rng.standard_normal((300, 2)).astype(np.float32)}, small)
    one = {"x": rng.standard_normal((1, 6000)).astype(np.float32)}             # one example larger than the image
    _check(codec, {}, one, [1])


def test_grpc_frame_and_spec_fields(codec):
    rng = np.random.default_rng(6)
    sizes = [2, 3]
    inp = {"x": rng.standard_normal((5, 2)).astype(np.float32)}
    ctx = {"u": rng.integers(0, 9, (2, 2))}
    _check(codec, ctx, inp, sizes, grpc_frame=True)
    _check(codec, ctx, inp, sizes, version=None, signature_name="rank", version_label="canary", output_filter=["s", "t"])
    _check(codec, ctx, inp, sizes, signature_name="é" * 200, output_filter=["x" * 300])


def test_one_query_equals_the_single_elwc_form(codec):
    rng = np.random.default_rng(7)
    x = {"x": rng.standard_normal((9, 4)).astype(np.float32), "i": rng.integers(0, 1 << 50, 9)}
    u = rng.standard_normal(5).astype(np.float32)
    one = _check(codec, {"u": u[None]}, x, [9], key="in")
    assert one == codec.encode_example_requests([("m", 2, x, {"u": u})], predict_input="in")[0]


def test_host_route_and_device_dtype_errors(codec):
    torch = pytest.importorskip("torch")
    strs = {"s": np.array([b"ab", b"c", b"d"], "S2")}
    _check(codec, {"t": np.array(["x", "y"])}, strs, [1, 2])         # numpy bytes / str: the host route
    with pytest.raises(ValueError):
        codec.encode_elwc_requests([("m", 1, {}, {"x": torch.zeros(3, dtype=torch.complex64, device="cuda")}, [3])], input_key="q")
    with pytest.raises(ValueError):
        codec.encode_elwc_requests([("m", 1, {"u": np.zeros(3)}, {"x": np.zeros(3)}, [1, 2])], input_key="q")


def test_device_columns(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(8)
    sizes = [3, 0, 4]
    n, Q = sum(sizes), len(sizes)
    ids = rng.integers(0, 1 << 40, (n, 5))
    lens = rng.integers(0, 6, n)
    col = _column(_strings(rng, Q * 2, 0, 30), (Q, 2))
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    inp = {"x": dev(rng.standard_normal((n, 3)).astype(np.float32)), "ids": RaggedColumn(dev(ids), dev(lens.astype(np.int64)))}
    ctx = {"u": dev(rng.standard_normal((Q, 2))), "q": BytesColumn(dev(np.asarray(col.data)), dev(col.offsets), col.shape),
           "toks": RaggedColumn(dev(ids[:Q]), dev(lens[:Q].astype(np.int64)))}
    _check(codec, ctx, inp, sizes)


def _c_structs(dev, ids, x, lens, qtok, qlen, col, sizes, lens_dev=None, offs_dev=None):
    """a PREDICT_ELWCS request over device columns: examples "ids" (ragged int64) and "x" (float); contexts "q" (bytes), "t"
    (ragged int64)"""
    n, Q = ids.shape[0], len(sizes)
    di, dx, dl = dev.upload(ids), dev.upload(x), dev.upload(lens)
    dq, dql = dev.upload(qtok), dev.upload(qlen)
    dd = dev.upload(np.asarray(col.data))
    do = offs_dev if offs_dev is not None else dev.upload(col.offsets)
    if lens_dev is not None:
        dql = lens_dev
    fa = (N.Feature * 2)(N.Feature(data=di, src_dtype=9, flags=0, row_elems=ids.shape[1], key=b"ids", key_len=3),
                         N.Feature(data=dx, src_dtype=1, flags=0, row_elems=x.shape[1], key=b"x", key_len=1))
    ca = (N.Feature * 2)(N.Feature(data=dd, src_dtype=7, flags=0, row_elems=1, key=b"q", key_len=1),
                         N.Feature(data=dq, src_dtype=9, flags=0, row_elems=qtok.shape[1], key=b"t", key_len=1))
    rg = [N.Ragged(lengths=dl, max_len=ids.shape[1], unit=1, flags=N.F_DEVICE_DATA), N.Ragged()]
    lrg = [N.Ragged(), N.Ragged(lengths=dql, max_len=qtok.shape[1], unit=1, flags=N.F_DEVICE_DATA)]
    lbs = [N.Bytes(offsets=do, data_len=col.data_len, flags=N.F_DEVICE_DATA), N.Bytes()]
    sz = np.asarray(sizes, np.int64)
    req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=2, n_examples=n,
                           n_features=2, flags=0, features=fa)
    ls = N.ExampleLists(list_sizes=sz.ctypes.data if Q else None, n_lists=Q, context=ca, n_context=2, present=1)
    tg = N.ExampleTarget(kind=N.EXAMPLES_PREDICT_ELWCS, key=b"q", key_len=1)
    return req, tg, ls, rg, lrg, lbs, (fa, ca, sz, di, dx, dl, dq, dql, dd, do)


def _c_ref(ids, x, lens, qtok, qlen, col, sizes):
    return _want({"q": col, "t": RaggedColumn(qtok, qlen)}, {"ids": RaggedColumn(ids, lens), "x": x}, sizes)


def _c_data(rng, sizes, rep=0):
    n, Q = sum(sizes), len(sizes)
    ids = (rng.integers(-(1 << 62), 1 << 62, (n, 6)) if rep % 2 else rng.integers(0, 100, (n, 6))).astype(np.int64)
    lens = rng.integers(0, 7, n).astype(np.int64)
    qtok = rng.integers(0, 1 << (10 + 30 * (rep % 2)), (Q, 4)).astype(np.int64)
    qlen = rng.integers(0, 5, Q).astype(np.int64)
    col = _column(_strings(rng, Q, 0, 5 + 60 * (rep % 2)), (Q, 1))
    return ids, lens, qtok, qlen, col


def test_c_call_mixing_list_string_elwc_and_elwcs(codec):
    """LIST, PREDICT_STRING, PREDICT_ELWC and PREDICT_ELWCS requests in one _host call"""
    import example_ref as ER

    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(9)
        parts, wants = [], []
        for r in range(12):
            k = r % 4
            n = int(rng.integers(0, 20))
            d = {"x": rng.standard_normal((n, 3)).astype(np.float32), "i": rng.integers(-99, 1 << 40, (n, 2))}
            sizes = []
            if k == 3:
                sizes = list(rng.multinomial(n, [0.25] * 4)) if n else [0, 0]
            _, preps = _example_columns(d)
            feats = (N.Feature * 2)(*[p[0] for p in preps])
            req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=5, n_examples=n,
                                   n_features=2, flags=0, features=feats)
            kind = [N.EXAMPLES_LIST, N.EXAMPLES_PREDICT_STRING, N.EXAMPLES_PREDICT_ELWC, N.EXAMPLES_PREDICT_ELWCS][k]
            tg = N.ExampleTarget(kind=kind, key=b"in", key_len=2)
            cx, ls, keep = N.ExampleContext(), N.ExampleLists(), [preps, feats]
            if k == 2:
                ctx = {"q": rng.integers(0, 1 << 20, 3)}
                _, cp = _example_columns(ctx, context=True)
                cf = (N.Feature * 1)(cp[0][0])
                keep += [cp, cf]
                cx = N.ExampleContext(features=cf, n_features=1, present=1)
                wants.append(ER.request_bytes("m", 5, d, key="in", context=ctx))
            elif k == 3:
                Q = len(sizes)
                ctx = {"u": rng.standard_normal((Q, 2)).astype(np.float32)}
                _, cp = _example_columns(ctx)
                cf = (N.Feature * 1)(cp[0][0])
                sz = np.asarray(sizes, np.int64)
                keep += [cp, cf, sz]
                ls = N.ExampleLists(list_sizes=sz.ctypes.data, n_lists=Q, context=cf, n_context=1, present=1)
                wants.append(make_predict_elwcs_request("m", 5, ctx, d, sizes, "in").SerializeToString(deterministic=True))
            else:
                wants.append(ER.request_bytes("m", 5, d, key="in" if k == 1 else None))
            parts.append((req, tg, cx, ls, keep))
        m = len(parts)
        reqs = (N.ExampleRequest * m)(*[p[0] for p in parts])
        tgs = (N.ExampleTarget * m)(*[p[1] for p in parts])
        cxs = (N.ExampleContext * m)(*[p[2] for p in parts])
        lss = (N.ExampleLists * m)(*[p[3] for p in parts])
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_lists_arena_size(m, reqs, None, None, tgs, cxs, None, None, None, None, lss, None, None, C.byref(cap)))
        wire = np.empty(cap.value, np.uint8)
        off, ln = (C.c_uint64 * m)(), (C.c_uint64 * m)()
        N.check(lib.b200tfs_encode_example_lists_host(dev.ctx, m, reqs, None, None, tgs, cxs, None, None, None, None, lss, None, None,
                                                      wire.ctypes.data, cap.value, off, ln))
        for r in range(m):
            assert wire[off[r]: off[r] + ln[r]].tobytes() == wants[r], r
    finally:
        dev.close()


def test_graph_replay_with_new_values_lengths_and_offsets():
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(10)
        sizes = [5, 0, 9, 2, 30]
        n = sum(sizes)
        x = rng.standard_normal((n, 3)).astype(np.float32)
        cap_bytes = 1 << 14
        ids, lens, qtok, qlen, col = _c_data(rng, sizes)
        data = np.zeros(cap_bytes, np.uint8)
        big = BytesColumn(data, col.offsets, col.shape)
        req, tg, ls, rg, lrg, lbs, keep = _c_structs(dev, ids, x, lens, qtok, qlen, big, sizes)
        di, dl, dq, dql, dd, do = keep[3], keep[5], keep[6], keep[7], keep[8], keep[9]
        rga, lrga, lbsa = (N.Ragged * 2)(*rg), (N.Ragged * 2)(*lrg), (N.Bytes * 2)(*lbs)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_lists_arena_size(1, C.byref(req), rga, None, C.byref(tg), None, None, None, None, None, C.byref(ls),
                                                     lrga, lbsa, C.byref(cap)))
        arena = (dev.malloc(cap.value + 256) + 255) & ~255
        args = (dev.ctx, 1, C.byref(req), rga, None, C.byref(tg), None, None, None, None, None, C.byref(ls), lrga, lbsa, arena, cap.value)
        N.check(lib.b200tfs_encode_example_lists_async(*args))
        N.check(lib.b200tfs_encode_results(dev.ctx, 1, None, None))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_encode_example_lists_async(*args))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        seen = set()
        for rep in range(4):
            ids, lens, qtok, qlen, col = _c_data(rng, sizes, rep)
            data = np.zeros(cap_bytes, np.uint8)
            data[: col.data_len] = col.data
            for ptr, a in ((di, ids), (dl, lens), (dq, qtok), (dql, qlen), (dd, data), (do, col.offsets)):
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, ptr, a.ctypes.data, a.nbytes))
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_encode_results(dev.ctx, 1, off, ln))
            assert dev.download(arena + off[0], ln[0]).tobytes() == _c_ref(ids, x, lens, qtok, qlen, col, sizes), rep
            seen.add(ln[0])
        assert len(seen) > 1
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


@pytest.mark.parametrize("case", ["example_length", "context_length", "context_offsets_decreasing", "context_offsets_past_data_len"])
def test_bad_device_lengths_and_offsets(codec, case):
    """The bad request sits in front of good ones in a canary-filled arena with slack: E_SHAPE for it, the others byte-exact,
    and every byte outside every slot keeps the canary."""
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(11)
        sizes = [3, 0, 6, 1, 2]
        n, Q = sum(sizes), len(sizes)
        x = rng.standard_normal((n, 3)).astype(np.float32)
        ids, lens, qtok, qlen, col = _c_data(rng, sizes)
        bl, bq, bo = lens.copy(), qlen.copy(), col.offsets.copy()
        if case == "example_length":
            bl[4] = -(1 << 62)
        elif case == "context_length":
            bq[Q - 1] = 1 << 62
        elif case == "context_offsets_decreasing":
            bo[2] = bo[1] - 1
        else:
            bo[Q] = col.data_len + 1
        parts = []
        for r in range(4):
            p = _c_structs(dev, ids, x, bl if r == 0 else lens, qtok, qlen, col, sizes,
                           lens_dev=dev.upload(bq) if r == 0 else None, offs_dev=dev.upload(bo) if r == 0 else None)
            parts.append(p)
        reqs = (N.ExampleRequest * 4)(*[p[0] for p in parts])
        tga = (N.ExampleTarget * 4)(*[p[1] for p in parts])
        lsa = (N.ExampleLists * 4)(*[p[2] for p in parts])
        rga = (N.Ragged * 8)(*[g for p in parts for g in p[3]])
        lrga = (N.Ragged * 8)(*[g for p in parts for g in p[4]])
        lbsa = (N.Bytes * 8)(*[b for p in parts for b in p[5]])
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_lists_arena_size(4, reqs, rga, None, tga, None, None, None, None, None, lsa, lrga, lbsa, C.byref(cap)))
        slack = 1 << 16
        arena = (dev.malloc(cap.value + slack + 256) + 255) & ~255
        canary = np.full(cap.value + slack, 0xA5, np.uint8)
        N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena, canary.ctypes.data, canary.nbytes))
        N.check(lib.b200tfs_encode_example_lists_async(dev.ctx, 4, reqs, rga, None, tga, None, None, None, None, None, lsa, lrga, lbsa,
                                                       arena, cap.value))
        off, ln = (C.c_uint64 * 4)(), (C.c_uint64 * 4)()
        assert lib.b200tfs_encode_results(dev.ctx, 4, off, ln) == N.E_SHAPE
        assert off[0] == 0 and ln[0] == 0
        want = _c_ref(ids, x, lens, qtok, qlen, col, sizes)
        out = dev.download(arena, cap.value + slack)
        for r in range(1, 4):
            assert out[off[r]: off[r] + ln[r]].tobytes() == want, r
        mask = np.ones(len(out), bool)
        mask[: off[1]] = False
        for r in range(1, 4):
            mask[off[r]: off[r] + ln[r]] = False
        assert (out[mask] == 0xA5).all()
        torch = pytest.importorskip("torch")
        if case == "example_length":
            bad = ({}, {"ids": RaggedColumn(ids, torch.from_numpy(bl).cuda())})
        elif case == "context_length":
            bad = ({"t": RaggedColumn(qtok, torch.from_numpy(bq).cuda())}, {"x": x})
        else:
            bad = ({"q": BytesColumn(torch.from_numpy(np.asarray(col.data)).cuda(), torch.from_numpy(bo).cuda(), col.shape)}, {"x": x})
        with pytest.raises(ValueError):
            codec.encode_elwc_requests([("m", 1, {}, {"x": x}, sizes), ("m", 1, *bad, sizes)], input_key="q")
        _check(codec, {}, {"x": x}, sizes)
    finally:
        dev.close()


def test_predict_round_trip_through_a_servicer():
    """the client's request, parsed by a Predict servicer with ExampleListWithContext.FromString"""
    from fake_server import IdentityServer
    from min_tfs_client.requests import TensorServingClient
    from tensorflow_serving.apis import predict_pb2
    from tensorflow_serving.apis.input_pb2 import ExampleListWithContext

    class RankingServer(IdentityServer):
        def _predict(self, request_bytes, context):
            self.received.append(request_bytes)
            req = predict_pb2.PredictRequest.FromString(request_bytes)
            elwcs = [ExampleListWithContext.FromString(s) for s in req.inputs["elwcs"].string_val]
            out = np.array([len(e.examples) for e in elwcs], np.int64)
            resp = predict_pb2.PredictResponse()
            t = resp.outputs["n"]
            t.dtype = 9
            t.tensor_shape.dim.add().size = len(out)
            t.int64_val.extend(out.tolist())
            resp.model_spec.name = req.model_spec.name
            return resp.SerializeToString()

    srv = RankingServer()
    try:
        client = TensorServingClient("127.0.0.1", srv.port)
        rng = np.random.default_rng(12)
        sizes = [3, 0, 5]
        inp = {"doc": rng.standard_normal((8, 4)).astype(np.float32)}
        ctx = {"user": rng.standard_normal((3, 2)).astype(np.float32)}
        resp = client.predict_elwcs_request("m", ctx, inp, sizes, "elwcs", model_version=3, output_filter=["n"])
        assert resp.to_ndarrays()["n"].tolist() == sizes
        assert srv.received[0] == make_predict_elwcs_request("m", 3, ctx, inp, sizes, "elwcs", output_filter=["n"]).SerializeToString(
            deterministic=True)
    finally:
        srv.stop()
