"""PREDICT_ELWCS requests whose list sizes are in device memory (b200tfs_example_device_lists), encoded on the GPU.  Every case
compares bytes with make_predict_elwcs_request(...).SerializeToString(deterministic=True) built from host copies of the sizes
and of the first sum(sizes) rows; the rows past the sum hold values no sent row has, so a row sent by mistake shows."""
import ctypes as C

import numpy as np
import pytest

from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn, _example_columns, _head_rows
from min_tfs_client.requests import gpu_predict_elwcs_serializer, make_predict_elwcs_request
from test_elwc_batch_gpu import _c_data, _c_structs, _column, _every_dtype, _host, _hostd, _strings

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def _dsizes(sizes):
    return torch.tensor(np.asarray(sizes, np.int64).reshape(-1), dtype=torch.int64, device="cuda")


def _want(ctx, inp, sizes, key="q", version=2, **fields):
    total = int(np.sum(sizes))
    head = {k: _head_rows(_host(v), total) for k, v in inp.items()}
    return make_predict_elwcs_request("m", version, _hostd(ctx), head, list(sizes), key, **fields).SerializeToString(deterministic=True)


def _dcheck(codec, ctx, inp, sizes, **kw):
    got = codec.encode_elwc_requests([("m", 2, ctx, inp, _dsizes(sizes))], input_key="q", **kw)[0]
    assert got == _want(ctx, inp, sizes, **kw)
    return got


def _example_bytes(inp):
    """the worst-case (here: exact) bytes of one example tag 0A included, for dense float columns: ex_max of the planner"""
    s = make_predict_elwcs_request("m", 2, {}, {k: v[:1] for k, v in inp.items()}, [1], "q").inputs["q"].string_val[0]
    from tensorflow_serving.apis.input_pb2 import ExampleListWithContext

    e = ExampleListWithContext.FromString(s).examples[0].ByteSize()
    return 1 + len(_varint(e)) + e


def _varint(v):
    out = bytearray()
    while True:
        b, v = v & 0x7F, v >> 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


@pytest.mark.parametrize("slack", [0, 5])
@pytest.mark.parametrize("sizes", [[3, 0, 5, 1], [0, 4], [6, 0], [1], []])
def test_every_dtype_both_sides(codec, sizes, slack):
    rng = np.random.default_rng(len(sizes) * 10 + slack)
    n, Q = sum(sizes) + slack, len(sizes)
    inp = _every_dtype(rng, n)
    inp["k"] = np.int64(-9)
    ctx = _every_dtype(rng, Q)
    ctx["z"] = np.float32(2.5)
    _dcheck(codec, ctx, inp, sizes)
    _dcheck(codec, {}, inp, sizes)
    _dcheck(codec, {"z": np.float32(2.5)}, {"x": inp["f32"]}, sizes)


@pytest.mark.parametrize("slack", [0, 7])
def test_ragged_and_bytes_on_both_sides(codec, slack):
    rng = np.random.default_rng(2 + slack)
    sizes = [4, 0, 7, 1, 3]
    n, Q = sum(sizes) + slack, len(sizes)
    inp = {"ids": RaggedColumn(rng.integers(0, 1 << 40, (n, 6)), rng.integers(0, 7, n)), "t": _column(_strings(rng, n * 2), (n, 2)),
           "w": RaggedColumn(_column(_strings(rng, n * 3 * 2), (n, 3, 2)), rng.integers(0, 4, n)),
           "x": rng.standard_normal((n, 4)).astype(np.float32), "s": _column([b"same"], ())}
    ctx = {"query": _column(_strings(rng, Q, 0, 40)), "toks": RaggedColumn(rng.integers(-5, 1 << 33, (Q, 9)), rng.integers(0, 10, Q)),
           "words": RaggedColumn(_column(_strings(rng, Q * 5), (Q, 5)), rng.integers(0, 6, Q)),
           "emb": RaggedColumn(rng.standard_normal((Q, 4, 2)).astype(np.float32), rng.integers(0, 5, Q)), "lang": _column([b"en"], ())}
    _dcheck(codec, ctx, inp, sizes)
    _dcheck(codec, {"emb": ctx["emb"]}, {"x": inp["x"]}, sizes)      # kExRagged
    _dcheck(codec, {}, {"t": inp["t"]}, sizes)                       # kExColumns, empty contexts


def test_device_columns_and_device_sizes(codec):
    rng = np.random.default_rng(8)
    sizes = [3, 0, 4]
    n, Q = sum(sizes) + 6, len(sizes)
    ids = rng.integers(0, 1 << 40, (n, 5))
    lens = rng.integers(0, 6, n)
    col = _column(_strings(rng, Q * 2, 0, 30), (Q, 2))
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    inp = {"x": dev(rng.standard_normal((n, 3)).astype(np.float32)), "ids": RaggedColumn(dev(ids), dev(lens.astype(np.int64)))}
    ctx = {"u": dev(rng.standard_normal((Q, 2))), "q": BytesColumn(dev(np.asarray(col.data)), dev(col.offsets), col.shape)}
    _dcheck(codec, ctx, inp, sizes)


def test_size_patterns(codec):
    rng = np.random.default_rng(3)
    x = rng.standard_normal((600, 30)).astype(np.float32)
    per = 16384 // _example_bytes({"x": x})
    assert per > 2
    n = max(4 * per + 8, 2100)
    x = rng.standard_normal((n, 30)).astype(np.float32)
    patterns = [[], [0] * 7, [n], [1] * 300, list(rng.integers(0, 3, 1024)),
                [per], [per + 1], [per - 1, per, per + 1], [2 * per, 2 * per + 1], [0, per, 0, per + 1, 0]]
    for sizes in patterns:
        assert sum(sizes) <= n
        Q = len(sizes)
        ctx = {"u": rng.standard_normal((Q, 3)).astype(np.float32)}
        _dcheck(codec, ctx, {"x": x}, sizes)
        _dcheck(codec, {}, {"x": x}, sizes)
    # a query larger than the 16 KB emit image, and a context larger than it
    big = rng.standard_normal((90, 200)).astype(np.float32)
    _dcheck(codec, {"c": rng.standard_normal((3, 5000)).astype(np.float32)}, {"x": big}, [1, 70, 2])
    # 1024 queries with a ragged column: several warp rounds of the frame kernel over counted rows
    m = 3000
    ids = RaggedColumn(rng.integers(-(1 << 50), 1 << 50, (m, 4)), rng.integers(0, 5, m))
    sizes = list(rng.integers(0, 4, 1024))
    _dcheck(codec, {"u": rng.integers(0, 9, (1024, 2))}, {"ids": ids}, sizes)


def test_many_requests_in_one_call(codec):
    rng = np.random.default_rng(4)
    items, wants = [], []
    for r in range(9):
        Q = int(rng.integers(0, 40))
        sizes = list(rng.integers(0, 10, Q))
        host = r % 3 == 0
        n = int(np.sum(sizes)) + (0 if host else int(rng.integers(0, 20)))
        inp = {"x": rng.standard_normal((n, 2)).astype(np.float32), "i": rng.integers(0, 1 << 30, n)}
        ctx = {"u": rng.standard_normal((Q, 3)).astype(np.float32), "q": _column(_strings(rng, Q))}
        items.append(("m", 2, ctx, inp, sizes if host else _dsizes(sizes)))
        wants.append(_want(ctx, inp, sizes))
    assert codec.encode_elwc_requests(items, input_key="q") == wants


def test_value_errors_and_host_route(codec):
    x = np.arange(20, dtype=np.float32).reshape(10, 2)
    with pytest.raises(ValueError, match="int64"):
        codec.encode_elwc_requests([("m", 1, {}, {"x": x}, _dsizes([1, 2]).to(torch.int32))], input_key="q")
    with pytest.raises(ValueError, match="int64"):
        codec.encode_elwc_requests([("m", 1, {}, {"x": x}, torch.ones((1, 2), dtype=torch.int64, device="cuda"))], input_key="q")
    with pytest.raises(ValueError, match="capacity"):
        codec.encode_elwc_requests([("m", 1, {}, {"k": np.float32(1)}, _dsizes([1, 2]))], input_key="q")
    with pytest.raises(ValueError, match="capacity"):
        codec.encode_elwc_requests([("m", 1, {}, {}, _dsizes([0]))], input_key="q")
    with pytest.raises(ValueError):
        codec.encode_elwc_requests([("m", 1, {}, {"x": x}, _dsizes([3, -1]))], input_key="q")
    with pytest.raises(ValueError):
        codec.encode_elwc_requests([("m", 1, {}, {"x": x}, _dsizes([8, 3]))], input_key="q")
    with pytest.raises(ValueError, match="rows"):       # a context value whose rows are not Q
        codec.encode_elwc_requests([("m", 1, {"u": np.zeros(3)}, {"x": x}, _dsizes([1, 2]))], input_key="q")
    # the codec still works after the refusals
    _dcheck(codec, {}, {"x": x}, [4, 0, 5])
    # an item the host assembles (a numpy bytes column): the sizes come to the host and the rows are cut to their total
    s = np.array([b"row%d" % i for i in range(10)], object).astype("S6")
    for sizes in ([2, 0, 3], [4, 6], []):
        got = codec.encode_elwc_requests([("m", 2, {"c": np.arange(len(sizes))}, {"s": s, "x": x}, _dsizes(sizes))], input_key="q")[0]
        t = int(np.sum(sizes))
        assert got == make_predict_elwcs_request("m", 2, {"c": np.arange(len(sizes))}, {"s": s[:t], "x": x[:t]}, sizes,
                                                 "q").SerializeToString(deterministic=True)
    with pytest.raises(ValueError):
        codec.encode_elwc_requests([("m", 2, {}, {"s": s}, _dsizes([11]))], input_key="q")
    # the serializer takes them through the codec
    assert gpu_predict_elwcs_serializer(("m", 2, {}, {"x": x}, _dsizes([1, 2]), "q")) == _want({}, {"x": x}, [1, 2])


# ---- C ABI: graph replay, bad sizes, mixed calls ------------------------------------------------------------------------------
def _dev_entry(ptr):
    return N.ExampleDeviceLists(sizes=ptr)


def test_graph_replay_with_new_sizes_totals_and_values():
    """capture once; every replay takes new sizes (and a new total), new values, lengths and offsets"""
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(10)
        n, Q = 120, 6
        x = rng.standard_normal((n, 3)).astype(np.float32)
        cap_bytes = 1 << 14
        first = [5, 0, 9, 2, 30, 1]
        ids, lens, qtok, qlen, col = _c_data(rng, [n] + [0] * (Q - 1))
        col = _column(_strings(rng, Q, 0, 5), (Q, 1))
        big = BytesColumn(np.zeros(cap_bytes, np.uint8), col.offsets, col.shape)
        req, tg, ls, rg, lrg, lbs, keep = _c_structs(dev, ids, x, lens, qtok[:Q], qlen[:Q], big, first)
        assert req.n_examples == n
        ls.list_sizes = None
        dsz = dev.upload(np.asarray(first, np.int64))
        dl = _dev_entry(dsz)
        di, dx, dlen, dq, dql, dd, do = keep[3], keep[4], keep[5], keep[6], keep[7], keep[8], keep[9]
        rga, lrga, lbsa = (N.Ragged * 2)(*rg), (N.Ragged * 2)(*lrg), (N.Bytes * 2)(*lbs)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_device_lists_arena_size(1, C.byref(req), rga, None, C.byref(tg), None, None, None, None, None,
                                                            C.byref(ls), lrga, lbsa, C.byref(dl), C.byref(cap)))
        arena = (dev.malloc(cap.value + 256) + 255) & ~255
        args = (dev.ctx, 1, C.byref(req), rga, None, C.byref(tg), None, None, None, None, None, C.byref(ls), lrga, lbsa, C.byref(dl),
                arena, cap.value)
        N.check(lib.b200tfs_encode_example_device_lists_async(*args))
        N.check(lib.b200tfs_encode_results(dev.ctx, 1, None, None))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_encode_example_device_lists_async(*args))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        totals = set()
        for rep in range(5):
            sizes = [int(v) for v in rng.integers(0, 40, Q)] if rep else first
            while sum(sizes) > n:
                sizes[int(np.argmax(sizes))] //= 2
            ids, lens, qtok, qlen, _ = _c_data(rng, [n] + [0] * (Q - 1), rep)
            x = rng.standard_normal((n, 3)).astype(np.float32)
            col = _column(_strings(rng, Q, 0, 5 + 60 * (rep % 2)), (Q, 1))
            data = np.zeros(cap_bytes, np.uint8)
            data[: col.data_len] = col.data
            sz = np.asarray(sizes, np.int64)
            for ptr, a in ((di, ids), (dx, x), (dlen, lens), (dq, qtok[:Q]), (dql, qlen[:Q]), (dd, data), (do, col.offsets), (dsz, sz)):
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, ptr, np.ascontiguousarray(a).ctypes.data, a.nbytes))
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_encode_results(dev.ctx, 1, off, ln))
            t = sum(sizes)
            want = _want({"q": col, "t": RaggedColumn(qtok[:Q], qlen[:Q])}, {"ids": RaggedColumn(ids, lens), "x": x}, sizes)
            assert dev.download(arena + off[0], ln[0]).tobytes() == want, (rep, sizes)
            totals.add(t)
        assert len(totals) >= 3
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


@pytest.mark.parametrize("case", ["negative", "past_n", "one_size_past_n"])
def test_bad_device_sizes(codec, case):
    """The bad request sits in front of good ones (device- and host-sized) in a canary-filled arena with slack: E_SHAPE for it,
    the others byte-exact, and every byte outside its slot and the good records keeps the canary."""
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(11)
        sizes = [3, 0, 6, 1, 2]
        n, Q = sum(sizes) + 4, len(sizes)
        x = rng.standard_normal((n, 3)).astype(np.float32)
        ids, lens, qtok, qlen, col = _c_data(rng, [n] + [0] * (Q - 1))
        qtok, qlen = qtok[:Q], qlen[:Q]
        col = _column(_strings(rng, Q, 0, 5), (Q, 1))
        bad = {"negative": [3, -1, 6, 1, 2], "past_n": [3, 0, 6, 1, 7], "one_size_past_n": [n + 1, 0, 0, 0, 0]}[case]
        parts, dls = [], []
        for r in range(4):
            p = _c_structs(dev, ids, x, lens, qtok, qlen, col, sizes)
            if r == 3:       # host-sized: n_examples is the sum
                p[0].n_examples = sum(sizes)
                dls.append(_dev_entry(None))
            else:
                p[2].list_sizes = None
                dls.append(_dev_entry(dev.upload(np.asarray(bad if r == 0 else sizes, np.int64))))
            parts.append(p)
        reqs = (N.ExampleRequest * 4)(*[p[0] for p in parts])
        tga = (N.ExampleTarget * 4)(*[p[1] for p in parts])
        lsa = (N.ExampleLists * 4)(*[p[2] for p in parts])
        rga = (N.Ragged * 8)(*[g for p in parts for g in p[3]])
        lrga = (N.Ragged * 8)(*[g for p in parts for g in p[4]])
        lbsa = (N.Bytes * 8)(*[b for p in parts for b in p[5]])
        dla = (N.ExampleDeviceLists * 4)(*dls)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_device_lists_arena_size(4, reqs, rga, None, tga, None, None, None, None, None, lsa, lrga, lbsa, dla,
                                                            C.byref(cap)))
        slack = 1 << 16
        arena = (dev.malloc(cap.value + slack + 256) + 255) & ~255
        canary = np.full(cap.value + slack, 0xA5, np.uint8)
        N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena, canary.ctypes.data, canary.nbytes))
        N.check(lib.b200tfs_encode_example_device_lists_async(dev.ctx, 4, reqs, rga, None, tga, None, None, None, None, None, lsa, lrga,
                                                              lbsa, dla, arena, cap.value))
        off, ln = (C.c_uint64 * 4)(), (C.c_uint64 * 4)()
        assert lib.b200tfs_encode_results(dev.ctx, 4, off, ln) == N.E_SHAPE
        assert off[0] == 0 and ln[0] == 0
        want = _want({"q": col, "t": RaggedColumn(qtok, qlen)}, {"ids": RaggedColumn(ids, lens), "x": x}, sizes)
        out = dev.download(arena, cap.value + slack)
        for r in range(1, 4):
            assert out[off[r]: off[r] + ln[r]].tobytes() == want, r
        mask = np.ones(len(out), bool)
        mask[: off[1]] = False       # the bad request's slot
        for r in range(1, 4):
            mask[off[r]: off[r] + ln[r]] = False
        assert (out[mask] == 0xA5).all()
        with pytest.raises(ValueError):
            codec.encode_elwc_requests([("m", 1, {}, {"x": x[:sum(sizes)]}, sizes), ("m", 1, {}, {"x": x}, _dsizes(bad))],
                                       input_key="q")
        _dcheck(codec, {}, {"x": x}, sizes)
    finally:
        dev.close()


def test_c_call_mixing_host_and_device_sizes_list_and_string(codec):
    """LIST, PREDICT_STRING, host-sized and device-sized PREDICT_ELWCS requests in one _host call; the requests without device
    sizes have the bytes of the same call without the device-sized ones"""
    import example_ref as ER

    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(9)
        parts, wants = [], []
        for r in range(16):
            k = r % 4
            n = int(rng.integers(0, 20))
            d = {"x": rng.standard_normal((n, 3)).astype(np.float32), "i": rng.integers(-99, 1 << 40, (n, 2))}
            _, preps = _example_columns(d)
            feats = (N.Feature * 2)(*[p[0] for p in preps])
            req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=5, n_examples=n,
                                   n_features=2, flags=0, features=feats)
            kind = [N.EXAMPLES_LIST, N.EXAMPLES_PREDICT_STRING, N.EXAMPLES_PREDICT_ELWCS, N.EXAMPLES_PREDICT_ELWCS][k]
            tg = N.ExampleTarget(kind=kind, key=b"in", key_len=2)
            ls, dl, keep = N.ExampleLists(), _dev_entry(None), [preps, feats]
            if k >= 2:
                Q = int(rng.integers(0, 6))
                ctx = {"u": rng.standard_normal((Q, 2)).astype(np.float32)}
                total = n if k == 2 else int(rng.integers(0, n + 1))
                sizes = list(rng.multinomial(total, [1 / Q] * Q)) if Q else []
                total = int(np.sum(sizes))
                _, cp = _example_columns(ctx)
                cf = (N.Feature * 1)(cp[0][0])
                sz = np.asarray(sizes, np.int64)
                keep += [cp, cf, sz]
                if k == 2:
                    req.n_examples = total
                    ls = N.ExampleLists(list_sizes=sz.ctypes.data if Q else None, n_lists=Q, context=cf, n_context=1, present=1)
                else:
                    ls = N.ExampleLists(list_sizes=None, n_lists=Q, context=cf, n_context=1, present=1)
                    dl = _dev_entry(dev.upload(sz))
                head = {kk: v[:total] for kk, v in d.items()}
                wants.append(make_predict_elwcs_request("m", 5, ctx, head, sizes, "in").SerializeToString(deterministic=True))
            else:
                wants.append(ER.request_bytes("m", 5, d, key="in" if k == 1 else None))
            parts.append((req, tg, ls, dl, keep))

        def run(sel):
            m = len(sel)
            reqs = (N.ExampleRequest * m)(*[parts[i][0] for i in sel])
            tgs = (N.ExampleTarget * m)(*[parts[i][1] for i in sel])
            lss = (N.ExampleLists * m)(*[parts[i][2] for i in sel])
            dls = (N.ExampleDeviceLists * m)(*[parts[i][3] for i in sel])
            cap = C.c_uint64()
            N.check(lib.b200tfs_example_device_lists_arena_size(m, reqs, None, None, tgs, None, None, None, None, None, lss, None, None,
                                                                dls, C.byref(cap)))
            wire = np.empty(max(cap.value, 1), np.uint8)
            off, ln = (C.c_uint64 * m)(), (C.c_uint64 * m)()
            N.check(lib.b200tfs_encode_example_device_lists_host(dev.ctx, m, reqs, None, None, tgs, None, None, None, None, None, lss,
                                                                 None, None, dls, wire.ctypes.data, cap.value, off, ln))
            return [wire[off[j]: off[j] + ln[j]].tobytes() for j in range(m)]

        allr = list(range(len(parts)))
        got = run(allr)
        for r in allr:
            assert got[r] == wants[r], r
        hosted = [r for r in allr if r % 4 != 3]
        assert run(hosted) == [got[r] for r in hosted]
    finally:
        dev.close()
