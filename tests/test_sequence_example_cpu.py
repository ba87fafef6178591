"""SequenceExample Predict requests without a GPU: the numpy wire writer (sequence_ref.py) against
sequence_examples_from_input_dict + protobuf, the closed-form size against ByteSize() across varint edges, the arena bound
against the worst case, and every refusal of the *_example_sequences_* entry points (checked before the context is looked at)."""
import ctypes as C

import numpy as np
import pytest

import sequence_ref as SR
from min_tfs_client import _native as N
from min_tfs_client.codec import BytesColumn, RaggedColumn, _example_columns, _sequence_count
from min_tfs_client.requests import make_predict_sequence_examples_request, sequence_examples_from_input_dict


def _ref(ctx, fl, key="seq", version=3, grpc=False):
    wire = make_predict_sequence_examples_request("m", version, ctx, fl, key).SerializeToString(deterministic=True)
    return (b"\x00" + len(wire).to_bytes(4, "big") + wire) if grpc else wire


def _column(strs, shape=None):
    lens = np.array([len(s) for s in strs], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return BytesColumn(np.frombuffer(b"".join(strs) + b"\xEE", np.uint8), offsets, shape)


def _struct(ctx, fl, key=b"seq", grpc=False, order=N.ORDER_UPB):
    """(request, target, ragged entries, bytes entries, sequence entry, keep-alive) as Codec.encode_sequence_example_requests
    builds them"""
    n = _sequence_count(ctx, fl)
    _, cp = _example_columns(ctx)
    _, lp = _example_columns(fl)
    rg = [p[3] or N.Ragged() for p in cp]
    for p, v in zip(lp, fl.values()):
        shape = v.shape
        g = p[3] or N.Ragged()
        g.max_len, g.unit = shape[1], int(np.prod(shape[2:], dtype=np.int64))
        rg.append(g)
    preps = cp + lp
    feats = (N.Feature * max(len(preps), 1))(*[p[0] for p in preps])
    rgs = (N.Ragged * max(len(rg), 1))(*rg)
    bs = (N.Bytes * max(len(preps), 1))(*[p.bytes_entry or N.Bytes() for p in preps])
    req = N.ExampleRequest(model_name=b"m", model_name_len=1, has_version=1, order=order, version=3, n_examples=n,
                           n_features=len(preps), flags=N.RF_GRPC_FRAME if grpc else 0, features=feats)
    tg = N.ExampleTarget(kind=N.EXAMPLES_PREDICT_SEQUENCE, key=key, key_len=len(key))
    sq = N.ExampleSequence(present=1, n_context=len(cp))
    return req, tg, rgs, bs, sq, (preps, feats)


def _rcs(req, tg, rgs, bs, sq, cx=None, tk=None):
    """arena size, _host and _async with no device context: their argument checks, or E_ARG for the missing context"""
    lib = N.load()
    out = C.c_uint64()
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    buf = C.create_string_buffer(256)
    t, s = C.byref(tg) if tg is not None else None, C.byref(sq) if sq is not None else None
    c, k = C.byref(cx) if cx is not None else None, C.byref(tk) if tk is not None else None
    return [lib.b200tfs_example_sequences_arena_size(1, C.byref(req), rgs, bs, t, c, None, k, s, C.byref(out)),
            lib.b200tfs_encode_example_sequences_host(None, 1, C.byref(req), rgs, bs, t, c, None, k, s, buf, 16, off, ln),
            lib.b200tfs_encode_example_sequences_async(None, 1, C.byref(req), rgs, bs, t, c, None, k, s, buf, 16)]


def _size(req, tg, rgs, sq):
    out = C.c_uint64()
    rc = N.load().b200tfs_example_sequences_request_size(C.byref(req), C.byref(tg), None, None, rgs, C.byref(sq), C.byref(out))
    return rc, out.value


def _cases():
    rng = np.random.default_rng(5)
    n = 4
    lens = np.array([0, 3, 1, 2], np.int64)
    ids = rng.integers(-2**63, 2**63 - 1, (n, 3), dtype=np.int64)
    strs = [bytes(rng.integers(0, 256, int(k), dtype=np.uint8)) for k in rng.integers(0, 9, n * 3 * 2)]
    yield "floats", {"u": rng.standard_normal((n, 5)).astype(np.float32)}, {"f": rng.standard_normal((n, 3, 2)).astype(np.float32)}
    yield "dtypes", {"a": np.arange(n, dtype=np.uint8), "b": np.array([True, False, True, True]), "c": np.float64(2.5)}, \
        {"d": rng.standard_normal((n, 2, 3)), "e": rng.standard_normal((n, 3)).astype(np.float16),
         "g": rng.integers(-5, 5, (n, 2, 2)).astype(np.int16), "h": np.full((n, 2), 2**64 - 1, np.uint64),
         "i": np.array([[True, False]] * n), "j": ids}
    yield "ragged", {"r": RaggedColumn(ids, np.array([3, 0, 2, 1]))}, {"rl": RaggedColumn(ids.reshape(n, 3, 1), lens),
                                                                      "rf": RaggedColumn(np.ones((n, 3, 2), np.float32), lens)}
    yield "bytes", {"s": _column(strs[:n], (n,))}, {"bl": _column(strs, (n, 3, 2)),
                                                    "br": RaggedColumn(_column(strs, (n, 3, 2)), lens)}
    yield "zero_steps", {}, {"z": np.zeros((n, 0, 4), np.float32), "zi": np.zeros((n, 0), np.int64)}
    yield "zero_unit", {"c": np.zeros((n, 0), np.float32)}, {"zu": np.zeros((n, 3, 0), np.int32), "zf": np.zeros((n, 2, 0), np.float32),
                                                              "zb": _column([], (n, 2, 0))}
    yield "empty_context", {}, {"f": np.ones((n, 2), np.float32)}
    yield "no_lists", {"u": np.ones((n, 2), np.int64)}, {}
    yield "prefix_keys", {"ab": np.ones(n, np.float32), "a": np.zeros(n, np.int64), "b": np.ones(n, np.int8)}, \
        {"ab": np.ones((n, 1), np.float32), "a": np.ones((n, 2), np.int32), "": np.ones((n, 1), np.float32), "b": np.zeros((n, 1))}
    yield "only_broadcast", {"k": np.int64(7)}, {}
    yield "nothing", {}, {}


@pytest.mark.parametrize("name,ctx,fl", list(_cases()), ids=[c[0] for c in _cases()])
def test_writer_matches_protobuf(name, ctx, fl):
    for grpc in (False, True):
        assert SR.request_bytes("m", 3, ctx, fl, "seq", grpc) == _ref(ctx, fl, grpc=grpc)
    seqs = sequence_examples_from_input_dict(ctx, fl)
    assert [s.SerializeToString(deterministic=True) for s in seqs] == SR.sequences(ctx, fl)


def test_given_order_writer():
    ctx = {"b": np.ones(2, np.float32), "a": np.zeros(2, np.int64)}
    fl = {"y": np.ones((2, 1), np.float32), "x": np.zeros((2, 2), np.int64)}
    given = SR.sequences(ctx, fl, order="given")
    assert given != SR.sequences(ctx, fl)
    # protobuf keeps no insertion order: the same dicts in sorted order give the deterministic bytes
    assert given == SR.sequences({"b": ctx["b"], "a": ctx["a"]}, {"y": fl["y"], "x": fl["x"]}, order="given")
    assert SR.sequences(dict(sorted(ctx.items())), dict(sorted(fl.items())), order="given") == SR.sequences(ctx, fl)


def test_framing_bytes():
    s = sequence_examples_from_input_dict({}, {"f": np.zeros((1, 0), np.float32)})[0].SerializeToString(deterministic=True)
    assert s == b"\x0a\x00\x12\x07\x0a\x05\x0a\x01f\x12\x00"
    s = sequence_examples_from_input_dict({}, {"f": np.zeros((1, 1, 0), np.float32)})[0].SerializeToString(deterministic=True)
    assert s == b"\x0a\x00\x12\x0b\x0a\x09\x0a\x01f\x12\x04\x0a\x02\x12\x00"
    assert SR.request_bytes("m", 3, {}, {}, "seq") == _ref({}, {})            # n = 0: no string_val at all
    assert sequence_examples_from_input_dict({"k": np.zeros((1, 0))}, {})[0].SerializeToString(deterministic=True) == \
        b"\x0a\x09\x0a\x07\x0a\x01k\x12\x02\x12\x00\x12\x00"


def test_count_rule():
    assert _sequence_count({}, {}) == 0
    assert _sequence_count({"k": np.float32(1)}, {}) == 1
    assert _sequence_count({"k": np.float32(1)}, {"f": np.zeros((4, 2))}) == 4
    with pytest.raises(ValueError, match="disagree"):
        _sequence_count({"k": np.zeros(3)}, {"f": np.zeros((4, 2))})
    for bad in (np.zeros(4), np.float32(0)):
        with pytest.raises(ValueError, match="rank >= 2"):
            sequence_examples_from_input_dict({}, {"f": bad})


def test_sequence_mirror():
    assert C.sizeof(N.ExampleSequence) == 8
    assert N.ExampleSequence.n_context.offset == 4
    assert N.EXAMPLES_PREDICT_SEQUENCE == 3


@pytest.mark.parametrize("T,unit,klen,n", [(1, 1, 1, 1), (2, 30, 1, 3), (3, 31, 1, 2), (4, 32, 1, 1), (1, 4095, 1, 2),
                                           (31, 1, 1, 1), (32, 1, 120, 1), (40, 1, 130, 1), (1, 4096, 100, 1), (700, 6, 3, 2),
                                           (9000, 1, 2, 1), (2, 0, 5, 3), (0, 3, 5, 2)])
def test_closed_form_size(T, unit, klen, n):
    """step (unit 30..32 floats), FeatureList, entry (key 120..130), FeatureLists and sequence lengths across their varint edges"""
    key = "k" * klen
    ctx = {"c": np.ones((n, 31), np.float32), key: np.ones((n, unit), np.float16)}
    fl = {key: np.ones((n, T, unit), np.float32), "g": np.ones((n, T), np.float64)}
    req, tg, rgs, bs, sq, keep = _struct(ctx, fl)
    rc, size = _size(req, tg, rgs, sq)
    assert rc == N.OK
    assert size == len(_ref(ctx, fl)) == make_predict_sequence_examples_request("m", 3, ctx, fl, "seq").ByteSize()
    req.flags = N.RF_GRPC_FRAME
    assert _size(req, tg, rgs, sq) == (N.OK, size + 5)


def test_closed_form_refuses_value_dependent_sizes():
    for ctx, fl in [({"i": np.ones(2, np.int64)}, {}), ({}, {"i": np.ones((2, 2), np.int32)}),
                    ({}, {"r": RaggedColumn(np.ones((2, 2), np.float32), np.array([1, 2]))})]:
        req, tg, rgs, bs, sq, keep = _struct(ctx, fl)
        assert _size(req, tg, rgs, sq)[0] == N.E_ARG


def test_arena_bound_covers_worst_case():
    """integer lists at 10-byte varints, ragged lists at T steps and strings at data_len: the slot holds the request"""
    n, T = 3, 5
    strs = [b"x" * 200] * (n * T * 2)
    ctx = {"i": np.full((n, 4), -1, np.int64), "s": _column([b"y" * 300] * n, (n,))}
    fl = {"a": np.full((n, T, 3), -1, np.int64), "r": RaggedColumn(np.full((n, T), -1, np.int64), np.full(n, T)),
          "b": RaggedColumn(_column(strs, (n, T, 2)), np.full(n, T)), "f": np.ones((n, T, 130), np.float32)}
    req, tg, rgs, bs, sq, keep = _struct(ctx, fl)
    out = C.c_uint64()
    assert N.load().b200tfs_example_sequences_arena_size(1, C.byref(req), rgs, bs, C.byref(tg), None, None, None, C.byref(sq),
                                                          C.byref(out)) == N.OK
    assert out.value >= len(_ref(ctx, fl)) + 256


def test_sequence_refusals():
    ctx = {"u": np.zeros((4, 3), np.float32)}
    fl = {"f": np.zeros((4, 2, 3), np.float32), "s": _column([b"ab"] * 8, (4, 2))}
    req, tg, rgs, bs, sq, keep = _struct(ctx, fl)
    assert _rcs(req, tg, rgs, bs, sq) == [N.OK, N.E_ARG, N.E_ARG]       # well-formed: only the device context is missing
    for present in (2, -1):
        sq.present = present
        assert _rcs(req, tg, rgs, bs, sq) == [N.E_ARG] * 3 and "present" in N.last_error()
    sq.present = 1
    # a sequence entry on another kind; PREDICT_SEQUENCE without one
    for kind in (N.EXAMPLES_LIST, N.EXAMPLES_PREDICT_STRING, N.EXAMPLES_PREDICT_ELWC):
        tg.kind = kind
        assert _rcs(req, tg, rgs, bs, sq) == [N.E_ARG] * 3 and "PREDICT_SEQUENCE" in N.last_error()
    assert _rcs(req, None, rgs, bs, sq) == [N.E_ARG] * 3
    tg.kind = N.EXAMPLES_PREDICT_SEQUENCE
    assert _rcs(req, tg, rgs, bs, None) == [N.E_ARG] * 3 and "PREDICT_SEQUENCE" in N.last_error()
    sq.present = 0
    assert _rcs(req, tg, rgs, bs, sq) == [N.E_ARG] * 3
    sq.present = 1
    # with a context or tasks
    cx = N.ExampleContext(features=None, n_features=0, present=1)
    assert _rcs(req, tg, rgs, bs, sq, cx=cx) == [N.E_ARG] * 3 and "context" in N.last_error()
    task = N.InferenceTask(signature_name=b"", signature_len=0, method=N.RESP_CLASSIFY)
    tk = N.ExampleTasks(tasks=C.addressof(task), n_tasks=1)
    assert _rcs(req, tg, rgs, bs, sq, tk=tk) == [N.E_ARG] * 3 and "tasks" in N.last_error()
    # n_context outside [0, n_features]
    for nc in (-1, 4):
        sq.n_context = nc
        assert _rcs(req, tg, rgs, bs, sq) == [N.E_ARG] * 3 and "n_context" in N.last_error()
    sq.n_context = 1
    # a feature list broadcast, without ragged entries, or with row_elems != T * unit
    keep[1][1].flags |= N.F_BROADCAST
    assert _rcs(req, tg, rgs, bs, sq) == [N.E_ARG] * 3 and "broadcast" in N.last_error()
    keep[1][1].flags &= ~N.F_BROADCAST
    assert _rcs(req, tg, None, bs, sq) == [N.E_ARG] * 3 and "ragged" in N.last_error()
    for attr, v in (("max_len", 3), ("unit", 2), ("max_len", -1), ("unit", -6)):
        old = getattr(rgs[1], attr)
        setattr(rgs[1], attr, v)
        assert _rcs(req, tg, rgs, bs, sq) == [N.E_ARG] * 3
        setattr(rgs[1], attr, old)
    rgs[1].flags = 4
    assert _rcs(req, tg, rgs, bs, sq) == [N.E_ARG] * 3 and "flags" in N.last_error()
    rgs[1].flags = 0
    # the context features may not be checked as lists: n_context = 2 makes "f" a context feature with a plain ragged entry
    sq.n_context = 2
    assert _rcs(req, tg, rgs, bs, sq)[0] == N.OK
    sq.n_context = 1
    assert _rcs(req, tg, rgs, bs, sq) == [N.OK, N.E_ARG, N.E_ARG]
    # the older entry points see a PREDICT_SEQUENCE target without sequences
    out = C.c_uint64()
    assert N.load().b200tfs_example_tasks_arena_size(1, C.byref(req), bs, C.byref(tg), None, None, None, C.byref(out)) == N.E_ARG


def test_host_lengths_and_offsets_refused_before_launch():
    """host lengths out of [0, T] and host offsets out of order: E_SHAPE from _host before any launch (no device context)"""
    lib = N.load()
    ids = np.ones((2, 3), np.int64)
    lens = np.array([1, 4], np.int64)
    fl = {"r": RaggedColumn(ids, np.array([1, 2]))}
    req, tg, rgs, bs, sq, keep = _struct({}, fl)
    rgs[0].lengths = lens.ctypes.data
    off, ln = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
    buf = C.create_string_buffer(256)
    assert lib.b200tfs_encode_example_sequences_host(None, 1, C.byref(req), rgs, bs, C.byref(tg), None, None, None, C.byref(sq),
                                                     buf, 256, off, ln) == N.E_SHAPE
    col = _column([b"a", b"bc", b"d", b"ef"], (2, 2))
    col.offsets[2] = 0                   # string 1 ends before it starts
    req, tg, rgs, bs, sq, keep = _struct({}, {"s": col})
    assert lib.b200tfs_encode_example_sequences_host(None, 1, C.byref(req), rgs, bs, C.byref(tg), None, None, None, C.byref(sq),
                                                     buf, 256, off, ln) == N.E_SHAPE
