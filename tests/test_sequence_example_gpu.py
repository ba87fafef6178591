"""SequenceExample Predict requests encoded on the GPU: every case compares bytes with the numpy writer (sequence_ref.py), which
the CPU tests hold to sequence_examples_from_input_dict + protobuf, through Codec.encode_sequence_example_requests and the C ABI."""
import ctypes as C

import numpy as np
import pytest

import example_ref as ER
import sequence_ref as SR
from devutil import Dev
from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn, _example_columns, _sequence_count
from min_tfs_client.requests import make_predict_sequence_examples_request

pytestmark = pytest.mark.gpu


def _host(v):
    if isinstance(v, RaggedColumn):
        return RaggedColumn(_host(v.values), _host(v.lengths))
    if isinstance(v, BytesColumn):
        return BytesColumn(_host(v.data), _host(v.offsets), v.shape)
    return v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)


def _hostd(d):
    return {k: _host(v) for k, v in d.items()}


def _column(strs, shape=None, tail=3):
    lens = np.array([len(s) for s in strs], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return BytesColumn(np.frombuffer(b"".join(strs) + b"\xEE" * tail, np.uint8), offsets, shape)


def _strings(rng, m, lo=0, hi=12):
    """strings with NUL and high bytes"""
    return [bytes(rng.integers(0, 256, int(k), dtype=np.uint8)) for k in rng.integers(lo, hi + 1, m)]


def _check(codec, ctx, fl, key="seq", version=2, **kw):
    got = codec.encode_sequence_example_requests([("m", version, ctx, fl)], input_key=key, **kw)[0]
    want = SR.request_bytes("m", version, _hostd(ctx), _hostd(fl), key, kw.get("grpc_frame", False), kw.get("order", "deterministic"))
    assert got == want
    return got


def _every_dtype(rng, n, T):
    ctx = {"f32": rng.standard_normal((n, 3)).astype(np.float32), "f64": rng.standard_normal(n) * 1e30,
           "f16": rng.standard_normal((n, 2)).astype(np.float16), "i8": rng.integers(-128, 128, (n, 2)).astype(np.int8),
           "u64": np.full((n, 1), 2**64 - 1, np.uint64), "b": rng.integers(0, 2, n).astype(bool), "k": np.int32(-7)}
    f = rng.standard_normal((n, T, 4)).astype(np.float32)
    f.view(np.uint32)[:, 0, 0] = 0x7F800001                 # a signalling NaN, quieted
    d = rng.standard_normal((n, T)) * 1e300                 # f64 -> f32 rounding and overflow
    d[:, 0] = np.float64(1) + np.float64(2.0**-24)          # a tie, rounded to even
    fl = {"f": f, "d": d, "h": rng.standard_normal((n, T, 2)).astype(np.float16),
          "i64": rng.integers(-2**63, 2**63 - 1, (n, T, 3), dtype=np.int64), "i64x": np.full((n, T), -2**63, np.int64),
          "u8": rng.integers(0, 256, (n, T, 2)).astype(np.uint8), "u32": np.full((n, T), 2**32 - 1, np.uint32),
          "i16": rng.integers(-2**15, 2**15, (n, T)).astype(np.int16), "bo": rng.integers(0, 2, (n, T, 3)).astype(bool)}
    return ctx, fl


@pytest.mark.parametrize("n,T", [(1, 1), (7, 3), (33, 2)])
def test_every_dtype(codec, n, T):
    rng = np.random.default_rng(n)
    ctx, fl = _every_dtype(rng, n, T)
    for grpc in (False, True):
        _check(codec, ctx, fl, grpc_frame=grpc)
    _check(codec, ctx, fl, version=None)
    want = make_predict_sequence_examples_request("m", 2, ctx, fl, "seq").SerializeToString(deterministic=True)
    assert codec.encode_sequence_example_requests([("m", 2, ctx, fl)], input_key="seq")[0] == want


def test_ragged_lists_host_and_device_lengths(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(2)
    n, T = 70, 50
    lens = rng.integers(0, T + 1, n)
    lens[:3] = [0, T, 1]
    ids = rng.integers(-2**40, 2**40, (n, T))
    feats = rng.standard_normal((n, T, 16)).astype(np.float32)
    ctx = {"user": rng.standard_normal((n, 64)).astype(np.float32), "ids": rng.integers(0, 1 << 50, (n, 4)),
           "hist": RaggedColumn(ids, lens)}
    for dev_lengths in (False, True):
        L = torch.from_numpy(lens.astype(np.int64)).cuda() if dev_lengths else lens
        fl = {"item_ids": RaggedColumn(ids, L), "item_feats": RaggedColumn(feats, L), "dense": ids[:, :3]}
        _check(codec, ctx, fl)


def test_bytes_lists_plain_and_ragged(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    n, T, u = 40, 6, 3
    strs = _strings(rng, n * T * u, 0, 40)
    strs[5] = b"\x00" * 7
    col = _column(strs, (n, T, u))
    lens = rng.integers(0, T + 1, n)
    ctx = {"q": _column(_strings(rng, n, 0, 70), (n,))}
    _check(codec, ctx, {"b": col, "r": RaggedColumn(col, lens)})
    dcol = BytesColumn(torch.from_numpy(np.asarray(col.data)).cuda(), torch.from_numpy(col.offsets).cuda(), col.shape)
    _check(codec, ctx, {"b": dcol, "r": RaggedColumn(dcol, torch.from_numpy(lens.astype(np.int64)).cuda())})
    # numpy str values take the host route
    s = np.array([["ab", "wörld"], ["", "c"]])
    got = codec.encode_sequence_example_requests([("m", 2, {}, {"s": s})], input_key="seq")[0]
    assert got == make_predict_sequence_examples_request("m", 2, {}, {"s": s}, "seq").SerializeToString(deterministic=True)


def test_edges(codec):
    rng = np.random.default_rng(4)
    _check(codec, {}, {})                                                       # n = 0
    _check(codec, {"k": np.float32(2)}, {})                                     # one sequence of a 0-d context
    _check(codec, {}, {"x": np.zeros((3, 0, 2), np.float32), "y": np.zeros((3, 0), np.int64)})        # zero steps
    _check(codec, {"c": np.zeros((3, 0), np.int64)}, {"zu": np.zeros((3, 4, 0), np.int32), "zf": np.zeros((3, 2, 0)),
                                                       "zb": _column([], (3, 2, 0))})                   # zero-unit steps
    _check(codec, {"k": np.int64(-1), "v": np.arange(3)}, {"": np.ones((3, 1), np.float32), "a": np.ones((3, 1), np.int8)})
    with pytest.raises(ValueError):
        codec.encode_sequence_example_requests([("m", 1, {}, {"x": np.zeros(3)})], input_key="seq")
    with pytest.raises(ValueError):
        codec.encode_sequence_example_requests([("m", 1, {"c": np.zeros(2)}, {"x": np.zeros((3, 1))})], input_key="seq")


def test_larger_than_the_emit_image(codec):
    """sequences of about 21 KB (200 steps of 8 float lists of 2), a single step of 40 KB, and a bytes step of 70 KB"""
    rng = np.random.default_rng(5)
    n = 9
    fl = {f"l{j}": rng.standard_normal((n, 200, 2)).astype(np.float32) for j in range(8)}
    _check(codec, {"u": rng.standard_normal((n, 8)).astype(np.float32)}, fl)
    _check(codec, {}, {"big": rng.standard_normal((3, 2, 10000)).astype(np.float32), "small": np.ones((3, 1), np.int64)})
    _check(codec, {}, {"s": _column([b"\xff" * 70000, b"", b"a"] * 2, (2, 1, 3))})
    mixed = {"small": np.ones((n, 1), np.float32), "big": RaggedColumn(rng.integers(0, 1 << 60, (n, 3000)), rng.integers(0, 3001, n))}
    _check(codec, {}, mixed)


def test_fifty_thousand_sequences(codec):
    rng = np.random.default_rng(6)
    n, T = 50000, 8
    lens = rng.integers(0, T + 1, n)
    ctx = {"u": rng.standard_normal((n, 2)).astype(np.float32)}
    fl = {"ids": RaggedColumn(rng.integers(0, 1 << 30, (n, T)), lens), "f": rng.standard_normal((n, T)).astype(np.float32)}
    _check(codec, ctx, fl)


def test_order_given_and_grpc_frame(codec):
    rng = np.random.default_rng(7)
    ctx = {"b": rng.standard_normal((4, 2)).astype(np.float32), "a": rng.integers(0, 9, 4)}
    fl = {"y": rng.standard_normal((4, 3, 2)).astype(np.float32), "x": rng.integers(0, 1 << 20, (4, 3))}
    for grpc in (False, True):
        _check(codec, ctx, fl, order="given", grpc_frame=grpc)
        _check(codec, ctx, fl, grpc_frame=grpc)


def test_torch_dlpack_and_pinned_columns(codec):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(8)
    n, T = 12, 5
    f = rng.standard_normal((n, T, 3)).astype(np.float32)
    ids = rng.integers(-1000, 1000, (n, T))
    pinned = codec.pinned_empty((n, T, 3), np.float32)
    pinned[...] = f

    class _DL:     # a DLPack-only producer
        def __init__(self, t):
            self.t = t

        def __dlpack__(self, **kw):
            return self.t.__dlpack__(**kw)

        def __dlpack_device__(self):
            return self.t.__dlpack_device__()

    for fv, iv in ((torch.from_numpy(f).cuda(), torch.from_numpy(ids).cuda()), (_DL(torch.from_numpy(f).cuda()), ids), (pinned, ids)):
        got = codec.encode_sequence_example_requests([("m", 2, {"c": ids[:, 0]}, {"f": fv, "i": iv})], input_key="seq")[0]
        assert got == SR.request_bytes("m", 2, {"c": ids[:, 0]}, {"f": f, "i": ids}, "seq")


def _structs(kind, d, ctx=None, fl=None, key=b"in"):
    """(request, target, ragged entries, bytes entries, context, context bytes, sequence, keep-alive) of one request of the given
    kind, for the _host entry point"""
    keep = []
    if kind == N.EXAMPLES_PREDICT_SEQUENCE:
        n = _sequence_count(d, fl)
        _, cp = _example_columns(d)
        _, lp = _example_columns(fl)
        rg = [p[3] or N.Ragged() for p in cp]
        for p, v in zip(lp, fl.values()):
            g = p[3] or N.Ragged()
            g.max_len, g.unit = v.shape[1], int(np.prod(v.shape[2:], dtype=np.int64))
            rg.append(g)
        preps, seq = cp + lp, N.ExampleSequence(present=1, n_context=len(cp))
    else:
        n, preps = _example_columns(d)
        rg, seq = [p[3] or N.Ragged() for p in preps], N.ExampleSequence()
    feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
    keep += [preps, feats]
    req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=5, n_examples=n,
                           n_features=len(preps), flags=0, features=feats)
    cx, cbs = N.ExampleContext(), []
    if ctx is not None:
        _, cpreps = _example_columns(ctx, context=True)
        cfeats = (N.Feature * max(len(cpreps), 1))(*[p[0] for p in cpreps])
        keep += [cpreps, cfeats]
        cx = N.ExampleContext(features=cfeats, n_features=len(cpreps), present=1)
        cbs = [p.bytes_entry or N.Bytes() for p in cpreps]
    tg = N.ExampleTarget(kind=kind, key=key, key_len=len(key))
    return req, tg, rg, [p.bytes_entry or N.Bytes() for p in preps], cx, cbs, seq, keep


def test_forty_requests_mixing_kinds(codec):
    """sequence, PREDICT_STRING, LIST and Predict-ELWC requests in one call, through the _host entry point"""
    rng = np.random.default_rng(9)
    parts, wants = [], []
    for r in range(40):
        n = int(rng.integers(0, 30))
        d = {"x": rng.standard_normal((n, 3)).astype(np.float32), "i": rng.integers(-99, 1 << 40, (n, 2))}
        k = r % 4
        if k == 0:
            fl = {"ids": RaggedColumn(rng.integers(0, 1 << 35, (n, 6)), rng.integers(0, 7, n)),
                  "s": _column(_strings(rng, n * 2 * 2), (n, 2, 2))}
            parts.append(_structs(N.EXAMPLES_PREDICT_SEQUENCE, d, fl=fl))
            wants.append(SR.request_bytes("m", 5, d, fl, "in"))
        elif k == 1:
            parts.append(_structs(N.EXAMPLES_PREDICT_STRING, d))
            wants.append(ER.request_bytes("m", 5, d, key="in"))
        elif k == 2:
            parts.append(_structs(N.EXAMPLES_LIST, d))
            wants.append(ER.request_bytes("m", 5, d))
        else:
            ctx = {"q": rng.integers(0, 1 << 20, 3)}
            parts.append(_structs(N.EXAMPLES_PREDICT_ELWC, d, ctx=ctx))
            wants.append(ER.request_bytes("m", 5, d, key="in", context=ctx))
    m = len(parts)
    reqs = (N.ExampleRequest * m)(*[p[0] for p in parts])
    tgs = (N.ExampleTarget * m)(*[p[1] for p in parts])
    rgs = [g for p in parts for g in p[2]]
    rga = (N.Ragged * len(rgs))(*rgs)
    bsl = [b for p in parts for b in p[3]]
    bsa = (N.Bytes * len(bsl))(*bsl)
    cxa = (N.ExampleContext * m)(*[p[4] for p in parts])
    cbl = [b for p in parts for b in p[5]]
    cba = (N.Bytes * max(len(cbl), 1))(*cbl) if cbl else None
    sqa = (N.ExampleSequence * m)(*[p[6] for p in parts])
    lib = N.load()
    cap = C.c_uint64()
    N.check(lib.b200tfs_example_sequences_arena_size(m, reqs, rga, bsa, tgs, cxa, cba, None, sqa, C.byref(cap)))
    wire = np.empty(cap.value, np.uint8)
    off, ln = (C.c_uint64 * m)(), (C.c_uint64 * m)()
    N.check(lib.b200tfs_encode_example_sequences_host(codec.ctx, m, reqs, rga, bsa, tgs, cxa, cba, None, sqa, wire.ctypes.data, cap.value,
                                                      off, ln))
    for r in range(m):
        assert wire[off[r]: off[r] + ln[r]].tobytes() == wants[r], r


def _device_sequence(dev, n, T, ids, lens, f, col, lens_dev=None, offs_dev=None):
    """a sequence request over device columns: context "u" (float), lists "ids" (ragged int64), "f" (float) and "s" (bytes)"""
    du, di, df = dev.upload(f[:, 0, :].copy()), dev.upload(ids), dev.upload(f)
    dl = lens_dev if lens_dev is not None else dev.upload(lens.astype(np.int64))
    dd = dev.upload(np.asarray(col.data))
    do = offs_dev if offs_dev is not None else dev.upload(col.offsets)
    fa = (N.Feature * 4)(N.Feature(data=du, src_dtype=1, flags=0, row_elems=f.shape[2], key=b"u", key_len=1),
                         N.Feature(data=di, src_dtype=9, flags=0, row_elems=T, key=b"ids", key_len=3),
                         N.Feature(data=df, src_dtype=1, flags=0, row_elems=T * f.shape[2], key=b"f", key_len=1),
                         N.Feature(data=dd, src_dtype=7, flags=0, row_elems=T * 2, key=b"s", key_len=1))
    rg = [N.Ragged(), N.Ragged(lengths=dl, max_len=T, unit=1, flags=N.F_DEVICE_DATA), N.Ragged(max_len=T, unit=f.shape[2]),
          N.Ragged(lengths=dl, max_len=T, unit=2, flags=N.F_DEVICE_DATA)]
    bs = [N.Bytes(), N.Bytes(), N.Bytes(), N.Bytes(offsets=do, data_len=col.data_len, flags=N.F_DEVICE_DATA)]
    req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=N.ORDER_UPB, version=3, n_examples=n,
                           n_features=4, flags=0, features=fa)
    return req, rg, bs, (fa, di, dl, dd, do, df)


def _seq_ref(n, T, ids, lens, f, col):
    return SR.request_bytes("m", 3, {"u": f[:, 0, :]}, {"ids": RaggedColumn(ids, lens), "f": f, "s": RaggedColumn(col, lens)}, "seq")


def test_graph_replay_with_new_values_lengths_and_offsets():
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(10)
        n, T, cap_bytes = 300, 20, 1 << 19
        f = rng.standard_normal((n, T, 3)).astype(np.float32)

        def make(rep):
            ids = (rng.integers(-(1 << 62), 1 << 62, (n, T)) if rep % 2 else rng.integers(0, 100, (n, T))).astype(np.int64)
            lens = rng.integers(0, T + 1, n).astype(np.int64)
            col = _column(_strings(rng, n * T * 2, 0, 3 + 40 * (rep % 2)), (n, T, 2), tail=0)
            data = np.zeros(cap_bytes, np.uint8)
            data[: col.data_len] = col.data
            return ids, lens, data, col
        ids, lens, data, col = make(0)
        big = BytesColumn(data, col.offsets, col.shape)
        req, rg, bs, keep = _device_sequence(dev, n, T, ids, lens, f, big)
        di, dl, dd, do = keep[1], keep[2], keep[3], keep[4]
        tg = N.ExampleTarget(kind=N.EXAMPLES_PREDICT_SEQUENCE, key=b"seq", key_len=3)
        sq = N.ExampleSequence(present=1, n_context=1)
        rga, bsa = (N.Ragged * 4)(*rg), (N.Bytes * 4)(*bs)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_sequences_arena_size(1, C.byref(req), rga, bsa, C.byref(tg), None, None, None, C.byref(sq), C.byref(cap)))
        arena = (dev.malloc(cap.value + 256) + 255) & ~255
        args = (dev.ctx, 1, C.byref(req), rga, bsa, C.byref(tg), None, None, None, C.byref(sq), arena, cap.value)
        N.check(lib.b200tfs_encode_example_sequences_async(*args))
        N.check(lib.b200tfs_encode_results(dev.ctx, 1, None, None))
        N.check(lib.b200tfs_capture_begin(dev.ctx))
        N.check(lib.b200tfs_encode_example_sequences_async(*args))
        g = C.c_void_p()
        N.check(lib.b200tfs_capture_end(dev.ctx, C.byref(g)))
        off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        seen = set()
        for rep in range(4):
            ids, lens, data, col = make(rep)
            for ptr, a in ((di, ids), (dl, lens), (dd, data), (do, col.offsets)):
                N.check(lib.b200tfs_memcpy_h2d(dev.ctx, ptr, a.ctypes.data, a.nbytes))
            N.check(lib.b200tfs_graph_launch(dev.ctx, g))
            N.check(lib.b200tfs_encode_results(dev.ctx, 1, off, ln))
            assert dev.download(arena + off[0], ln[0]).tobytes() == _seq_ref(n, T, ids, lens, f, col), rep
            seen.add(ln[0])
        assert len(seen) > 1
        N.check(lib.b200tfs_graph_destroy(g))
    finally:
        dev.close()


@pytest.mark.parametrize("case", ["length_negative", "length_past_T", "offsets_decreasing", "offsets_past_data_len"])
def test_bad_device_lengths_and_offsets(codec, case):
    """The bad request sits in front of good ones; the arena is filled with a canary and has slack: E_SHAPE for it, the others
    byte-exact, and every byte outside every record keeps the canary."""
    dev = Dev()
    lib = dev.lib
    try:
        rng = np.random.default_rng(11)
        n, T = 60, 9
        f = rng.standard_normal((n, T, 3)).astype(np.float32)
        ids = rng.integers(0, 1 << 60, (n, T))
        lens = rng.integers(0, T + 1, n).astype(np.int64)
        lens[2] = T                      # sequence 2 reads the offset made to decrease
        col = _column(_strings(rng, n * T * 2, 0, 20), (n, T, 2))
        bl, bo = lens.copy(), col.offsets.copy()
        if case == "length_negative":
            bl[5] = -(1 << 62)
        elif case == "length_past_T":
            bl[n - 1] = 1 << 62
        elif case == "offsets_decreasing":
            bo[40] = bo[39] - 1
        else:
            bo[n * T * 2] = col.data_len + 1
        parts = [_device_sequence(dev, n, T, ids, lens, f, col, lens_dev=dev.upload(bl) if r == 0 else None,
                                  offs_dev=dev.upload(bo) if r == 0 else None) for r in range(4)]
        reqs = (N.ExampleRequest * 4)(*[p[0] for p in parts])
        rga = (N.Ragged * 16)(*[g for p in parts for g in p[1]])
        bsa = (N.Bytes * 16)(*[b for p in parts for b in p[2]])
        tga = (N.ExampleTarget * 4)(*[N.ExampleTarget(kind=N.EXAMPLES_PREDICT_SEQUENCE, key=b"seq", key_len=3)] * 4)
        sqa = (N.ExampleSequence * 4)(*[N.ExampleSequence(present=1, n_context=1)] * 4)
        cap = C.c_uint64()
        N.check(lib.b200tfs_example_sequences_arena_size(4, reqs, rga, bsa, tga, None, None, None, sqa, C.byref(cap)))
        slack = 1 << 20
        arena = (dev.malloc(cap.value + slack + 256) + 255) & ~255
        canary = np.full(cap.value + slack, 0xA5, np.uint8)
        N.check(lib.b200tfs_memcpy_h2d(dev.ctx, arena, canary.ctypes.data, canary.nbytes))
        N.check(lib.b200tfs_encode_example_sequences_async(dev.ctx, 4, reqs, rga, bsa, tga, None, None, None, sqa, arena, cap.value))
        off, ln = (C.c_uint64 * 4)(), (C.c_uint64 * 4)()
        assert lib.b200tfs_encode_results(dev.ctx, 4, off, ln) == N.E_SHAPE
        assert off[0] == 0 and ln[0] == 0
        want = _seq_ref(n, T, ids, lens, f, col)
        out = dev.download(arena, cap.value + slack)
        for r in range(1, 4):
            assert out[off[r]: off[r] + ln[r]].tobytes() == want, r
        # request 0's slot may hold partial bytes; every byte outside the four slots keeps the canary
        mask = np.ones(len(out), bool)
        mask[: off[1]] = False
        for r in range(1, 4):
            mask[off[r]: off[r] + ln[r]] = False
        assert (out[mask] == 0xA5).all()
        torch = pytest.importorskip("torch")
        if case.startswith("length"):
            bad = {"ids": RaggedColumn(ids, torch.from_numpy(bl).cuda())}
        else:
            bad = {"s": BytesColumn(torch.from_numpy(np.asarray(col.data)).cuda(), torch.from_numpy(bo).cuda(), col.shape)}
        with pytest.raises(ValueError):
            codec.encode_sequence_example_requests([("m", 1, {}, {"f": f}), ("m", 1, {}, bad)], input_key="seq")
        _check(codec, {}, {"f": f})
    finally:
        dev.close()


def test_predict_round_trip_through_a_servicer():
    """the client's requests, parsed by a Predict servicer with SequenceExample.FromString"""
    from fake_server import IdentityServer
    from min_tfs_client.requests import TensorServingClient
    from tensorflow.core.example.example_pb2 import SequenceExample
    from tensorflow_serving.apis import predict_pb2

    class SequenceServer(IdentityServer):
        def _predict(self, request_bytes, context):
            self.received.append(request_bytes)
            req = predict_pb2.PredictRequest.FromString(request_bytes)
            seqs = [SequenceExample.FromString(s) for s in req.inputs["sequences"].string_val]
            out = np.array([sum(len(fl.feature) for fl in s.feature_lists.feature_list.values()) for s in seqs], np.int64)
            resp = predict_pb2.PredictResponse()
            t = resp.outputs["steps"]
            t.dtype = 9
            t.tensor_shape.dim.add().size = len(out)
            t.int64_val.extend(out.tolist())
            resp.model_spec.name = req.model_spec.name
            return resp.SerializeToString()

    srv = SequenceServer()
    try:
        client = TensorServingClient("127.0.0.1", srv.port)
        rng = np.random.default_rng(12)
        n, T = 6, 10
        lens = rng.integers(0, T + 1, n)
        ctx = {"user": rng.standard_normal((n, 4)).astype(np.float32)}
        fl = {"clicks": RaggedColumn(rng.integers(0, 1 << 40, (n, T)), lens),
              "dwell": RaggedColumn(rng.standard_normal((n, T, 2)).astype(np.float32), lens)}
        resp = client.predict_sequence_examples_request("m", ctx, fl, "sequences", model_version=3)
        assert resp.to_ndarrays()["steps"].tolist() == (2 * lens).tolist()
        assert srv.received[0] == SR.request_bytes("m", 3, ctx, fl, "sequences")
    finally:
        srv.stop()
